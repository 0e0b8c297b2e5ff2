"""The block kernel's bus phase evaluates the buses i and i + T of a lane as two independent chains, from words the block plan
packs for it (csrc/b200pf_plan.hpp: o_yword, o_yf32, o_bdesc).  Checked on the host: the packed words decode to the plan's
own arrays, and the emulated block kernel (tests/emu/sparse_emu.cpp) matches the fp64 oracle on topologies with split
substations (case5: 5 to 10 active buses, case14: 14 to 28), which give lanes 1 to 5 buses, with the reference bus, PV buses
and shunts in either chain."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle.c_oracle import COracle
from sparse_emu import BlockEmu
from test_block_ybus_cpu import _grid, _lib as _rows_lib, _plan
from test_sparse_plan_cpu import compare

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
NONE = 0xFFFF


def _lib():
    src = os.path.join(EMU, "bus_words.cpp")
    lib = os.path.join(EMU, "libbus_words.so")
    deps = [src, os.path.join(EMU, "plan_rows.cpp"), os.path.join(HERE, "..", "grid2op_b200", "csrc", "b200pf_plan.hpp")]
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", lib, src])
    h = C.CDLL(lib)
    h.plan_bus_words.restype = C.c_int
    return h


def _words(lib, desc, topo_row, T=8, U=1):
    buf = np.zeros(1 << 20, dtype=np.uint8)
    f = np.zeros(9, dtype=np.int32)
    t = np.ascontiguousarray(topo_row, dtype=np.int8)
    n = lib.plan_bus_words(C.byref(desc), t.ctypes.data_as(C.c_void_p), C.c_int(-1), C.c_int(T), C.c_int(U),
                           buf.ctypes.data_as(C.c_void_p), C.c_int(buf.size), f.ctypes.data_as(C.c_void_p))
    assert n > 0, n
    H = dict(zip(("status", "nb", "ne", "o_yword", "o_yf32", "o_bdesc", "o_colv", "o_shidx", "o_yptr"), f.tolist()))
    return H, buf[:n].tobytes()


def split_cases(gm, n, seed, max_split=None):
    """random topologies with up to max_split substations split (elements to busbar 2 with probability 1/2, and a line end
    on each busbar of a split substation, so that the second bus is seldom an island), a few lines out, injections moved by
    +-10 %"""
    rng = np.random.default_rng(seed)
    is_line = np.zeros(gm.dim_topo, dtype=bool)
    is_line[gm.line_or_pos] = True
    is_line[gm.line_ex_pos] = True
    sub_of = np.zeros(gm.dim_topo, dtype=np.int64)
    sub_of[gm.line_or_pos] = gm.line_or_sub
    sub_of[gm.line_ex_pos] = gm.line_ex_sub
    sub_of[gm.gen_pos] = gm.gen_sub
    sub_of[gm.load_pos] = gm.load_sub
    if gm.n_storage:
        sub_of[gm.storage_pos] = gm.storage_sub
    max_split = gm.n_sub if max_split is None else max_split
    topo = np.tile(gm.default_topo(), (n, 1))
    inj = np.tile(gm.default_inj(), (n, 1))
    sl = gm.inj_slices()
    for i in range(n):
        for s in rng.choice(gm.n_sub, size=rng.integers(0, max_split + 1), replace=False):
            pos = np.flatnonzero(sub_of == s)
            ends = np.flatnonzero(is_line[pos])
            if len(ends) < 2:
                continue
            b = rng.random(len(pos)) < 0.5
            two = rng.choice(ends, size=2, replace=False)
            b[two[0]], b[two[1]] = True, False
            topo[i, pos[b]] = 2
            if gm.n_shunt and rng.random() < 0.5:
                topo[i, gm.dim_topo + np.flatnonzero(np.asarray(gm.shunt_sub) == s)] = 2
        for l in np.flatnonzero(rng.random(gm.n_line) < 0.02):
            topo[i, gm.line_or_pos[l]] = -1
            topo[i, gm.line_ex_pos[l]] = -1
        for k, m in (("load_p", gm.n_load), ("load_q", gm.n_load), ("gen_p", gm.n_gen)):
            inj[i, sl[k]] *= rng.uniform(0.9, 1.1, m)
    return topo, inj


def _chain_roles(H, blob, T):
    """for the plan's buses in the second chain of their lane (i mod 2T >= T): (reference bus, PV bus, shunt) seen"""
    nb = H["nb"]
    desc = np.frombuffer(blob, dtype=np.uint32, count=2 * nb, offset=H["o_bdesc"]).reshape(nb, 2)
    second = (np.arange(nb) % (2 * T)) >= T
    ref = (desc[:, 0] & 0xFFFF) == NONE
    pv = ~ref & ((desc[:, 1] >> 16) == 0)
    sh = (desc[:, 1] & 0xFFFF) != NONE
    return bool((ref & second).any()), bool((pv & second).any()), bool((sh & second).any()), bool((sh & ~second).any())


@pytest.mark.parametrize("name,n", [("rte_case5_example", 64), ("l2rpn_case14_sandbox", 160), ("case14_odd", 96),
                                    ("l2rpn_neurips_2020_track1", 24)])
def test_packed_bus_words_decode_to_the_plan_arrays(name, n):
    gm = _grid(name)
    desc = COracle(gm).desc
    lib, rows = _lib(), _rows_lib()
    topo, _ = split_cases(gm, n, seed=5, max_split=None if gm.n_sub <= 14 else 4)
    nbs = []
    for r in range(n):
        H, blob = _words(lib, desc, topo[r])
        R, rblob, u16 = _plan(rows, desc, topo[r])
        assert rblob == blob                                    # one builder, one blob
        if H["status"] != 0:
            continue
        nb, ne = H["nb"], H["ne"]
        nbs.append(nb)
        ynb, yblk = u16(R["o_ynb"], ne), u16(R["o_yblk"], ne)
        yval = np.frombuffer(blob, dtype=np.float64, count=2 * ne, offset=R["o_yval"])
        colv, shidx = u16(H["o_colv"], nb), u16(H["o_shidx"], nb)
        dcidx, bdpos = u16(R["o_dcidx"], nb), u16(R["o_bdpos"], nb)
        w = np.frombuffer(blob, dtype=np.uint32, count=ne, offset=H["o_yword"]).astype(np.int64)
        assert np.array_equal(w & 0xFFFF, yblk) and np.array_equal((w >> 16) & 0x7FFF, ynb), r
        assert np.array_equal((w >> 31) == 1, colv[ynb] != NONE), r
        yf = np.frombuffer(blob, dtype=np.float32, count=2 * ne, offset=H["o_yf32"])
        assert np.array_equal(yf.view(np.uint32), yval.astype(np.float32).view(np.uint32)), r
        assert H["o_bdesc"] % 8 == 0 and H["o_yf32"] % 8 == 0                  # (uint2 / float2 loads)
        d = np.frombuffer(blob, dtype=np.uint32, count=2 * nb, offset=H["o_bdesc"]).reshape(nb, 2).astype(np.int64)
        assert np.array_equal(d[:, 0] & 0xFFFF, bdpos) and np.array_equal(d[:, 0] >> 16, dcidx), r
        assert np.array_equal(d[:, 1] & 0xFFFF, shidx) and np.array_equal((d[:, 1] >> 16) == 1, colv != NONE), r
        assert np.all(d[:, 1] >> 17 == 0)
    assert len(nbs) >= n // 4
    if name != "rte_case5_example":
        assert max(nbs) > 16, max(nbs)                         # a second group of 2T buses (T = 8)


@pytest.mark.parametrize("name,n,T,U", [("l2rpn_case14_sandbox", 240, 8, 1), ("case14_odd", 160, 8, 1), ("case14_odd", 80, 4, 2),
                                        ("rte_case5_example", 120, 4, 2), ("l2rpn_neurips_2020_track1", 40, 8, 1)])
def test_emulated_bus_chains_vs_oracle(name, n, T, U):
    gm = _grid(name)
    topo, inj = split_cases(gm, n, seed=41, max_split=None if gm.n_sub <= 14 else 4)
    out, status, iters, _ = BlockEmu(gm, T, U).run(topo, inj)
    ref, rstatus, riters, _ = COracle(gm).run(topo, inj)
    assert np.array_equal(status, rstatus)
    bad = status != 0
    assert np.isnan(out[bad]).all()
    ok = ~bad
    assert ok.sum() >= n // 5, ok.sum()
    compare(gm, out, ref, ok)
    assert np.all(iters[ok] >= riters[ok]) and np.all(iters[ok] <= riters[ok] + 1)
    # what the solved instances covered: buses per lane, and the roles of the buses in the second chain
    lib, desc = _lib(), COracle(gm).desc
    per_lane, roles = set(), np.zeros(4, dtype=bool)
    for r in np.flatnonzero(ok):
        H, blob = _words(lib, desc, topo[r], T, U)
        per_lane.add(-(-H["nb"] // T))
        roles |= _chain_roles(H, blob, T)
    want = {("case14_odd", 4): {4, 5}, ("rte_case5_example", 4): {2, 3}}.get((name, T), {2, 3} if "14" in name else {5})
    assert per_lane >= want, per_lane
    if "14" in name:
        assert roles.all(), roles
