"""Admittance rows of the BLOCK plans (csrc/b200pf_plan.hpp): the block kernel's bus lanes compute I = Y V and write their
whole block row of the Jacobian from them.  Checked on the host: every plan's rows against a dense numpy Ybus assembled from
line_y, and the emulated block kernel (tests/emu/sparse_emu.cpp) against the fp64 oracle, on random topologies that include
parallel lines, lines with both ends on one bus, disconnected lines and lines at the reference bus."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from grid2op_b200.gridmodel import GridModel
from oracle.c_oracle import COracle
from sparse_emu import BlockEmu
from test_c_oracle import random_cases
from test_sparse_plan_cpu import compare

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
EMU = os.path.join(HERE, "emu")
NONE = 0xFFFF


def _lib():
    src = os.path.join(EMU, "plan_rows.cpp")
    lib = os.path.join(EMU, "libplan_rows.so")
    deps = [src, os.path.join(HERE, "..", "grid2op_b200", "csrc", "b200pf_plan.hpp")]
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", lib, src])
    h = C.CDLL(lib)
    h.plan_rows_block.restype = C.c_int
    return h


def _grid(name):
    """golden grids; "case14_odd": case14 with line 4 (substations 1-4) moved inside substation 1 (both ends on one bus unless
    the substation is split) and line 5 (2-3) moved onto line 3's substations 1-3 (parallel to it)"""
    if name == "case14_odd":
        gm = GridModel.from_npz(os.path.join(GOLD, "gridmodel_l2rpn_case14_sandbox.npz"))
        gm.line_ex_sub[4] = gm.line_or_sub[4]
        gm.line_or_sub[5], gm.line_ex_sub[5] = gm.line_or_sub[3], gm.line_ex_sub[3]
        return gm
    return GridModel.from_npz(os.path.join(GOLD, f"gridmodel_{name}.npz"))


def _plan(lib, desc, topo_row, T=8, U=1):
    buf = np.zeros(1 << 20, dtype=np.uint8)
    f = np.zeros(18, dtype=np.int32)
    t = np.ascontiguousarray(topo_row, dtype=np.int8)
    n = lib.plan_rows_block(C.byref(desc), t.ctypes.data_as(C.c_void_p), C.c_int(-1), C.c_int(T), C.c_int(U),
                            buf.ctypes.data_as(C.c_void_p), C.c_int(buf.size), f.ctypes.data_as(C.c_void_p))
    assert n > 0, n
    keys = ("status", "nb", "n1", "nblk", "nblkA", "G", "n_bzero", "o_yptr", "o_ynb", "o_yval", "o_yblk", "o_ydiag", "o_dcidx",
            "o_bdpos", "o_bjpos", "o_bzero", "o_brf", "o_brt")
    H = dict(zip(keys, f.tolist()))
    blob = buf[:n].tobytes()
    u16 = lambda off, k: np.frombuffer(blob, dtype=np.uint16, count=k, offset=off).astype(np.int64)   # noqa: E731
    return H, blob, u16


@pytest.mark.parametrize("name,n", [("l2rpn_case14_sandbox", 64), ("case14_odd", 64), ("rte_case5_example", 64),
                                    ("l2rpn_neurips_2020_track1", 24)])
def test_admittance_rows_equal_dense_ybus(name, n):
    gm = _grid(name)
    desc = COracle(gm).desc
    lib = _lib()
    topo, _ = random_cases(gm, n, seed=17, p_disc=0.08)
    nl = gm.n_line
    y8 = np.asarray(gm.line_y, dtype=np.float64).reshape(nl, 8)
    yff, yft, ytf, ytt = (y8[:, 2 * k] + 1j * y8[:, 2 * k + 1] for k in range(4))
    seen = {"parallel": 0, "self": 0, "off": 0, "ref": 0}
    for r in range(n):
        H, blob, u16 = _plan(lib, desc, topo[r])
        if H["status"] != 0:
            continue
        nb, n1, nblk, nblkA = H["nb"], H["n1"], H["nblk"], H["nblkA"]
        brf, brt = u16(H["o_brf"], nl), u16(H["o_brt"], nl)
        dcidx, bdpos = u16(H["o_dcidx"], nb), u16(H["o_bdpos"], nb)
        bjpos = u16(H["o_bjpos"], 2 * nl)
        yptr = u16(H["o_yptr"], nb + 1)
        ne = int(yptr[nb])
        ynb, yblk = u16(H["o_ynb"], ne), u16(H["o_yblk"], ne)
        yval = np.frombuffer(blob, dtype=np.float64, count=2 * ne, offset=H["o_yval"]).reshape(ne, 2)
        ydiag = np.frombuffer(blob, dtype=np.float64, count=2 * nb, offset=H["o_ydiag"]).reshape(nb, 2)
        bzero = u16(H["o_bzero"], H["n_bzero"])
        # dense Ybus of the active buses, shunts excluded (they come with the injections)
        Y = np.zeros((nb, nb), dtype=np.complex128)
        link = np.zeros((nb, nb), dtype=bool)
        for l in range(nl):
            f, t = brf[l], brt[l]
            if f == NONE:
                seen["off"] += 1
                continue
            Y[f, f] += yff[l]; Y[f, t] += yft[l]; Y[t, f] += ytf[l]; Y[t, t] += ytt[l]
            if f == t:
                seen["self"] += 1
            else:
                seen["parallel"] += int(link[f, t])
                link[f, t] = link[t, f] = True
        scale = np.abs(Y).max()
        assert np.allclose(ydiag[:, 0] + 1j * ydiag[:, 1], np.diag(Y), rtol=1e-13, atol=1e-13 * scale)
        written = np.zeros(nblk, dtype=bool)
        written[bdpos[bdpos != NONE]] = True
        assert written.sum() == n1
        for i in range(nb):
            js = ynb[yptr[i]:yptr[i + 1]]
            assert np.array_equal(js, np.flatnonzero(link[i])), (r, i)          # ascending, one entry per neighbour
            yv = yval[yptr[i]:yptr[i + 1]]
            assert np.allclose(yv[:, 0] + 1j * yv[:, 1], Y[i, js], rtol=1e-13, atol=1e-13 * scale), (r, i)
            for e in range(yptr[i], yptr[i + 1]):
                j, b = ynb[e], yblk[e]
                if dcidx[i] == NONE or dcidx[j] == NONE:
                    assert b == nblkA, (r, i, j)                                  # the dummy block
                    seen["ref"] += 1
                else:
                    assert 0 <= b < nblk and not written[b], (r, i, j, b)       # one writer per block
                    written[b] = True
        # the kernel's assembly covers the blocks the per-line positions named, and only the fill is cleared
        for l in range(nl):
            f, t = brf[l], brt[l]
            if f == NONE or f == t or dcidx[f] == NONE or dcidx[t] == NONE:
                continue
            ef = yptr[f] + np.flatnonzero(ynb[yptr[f]:yptr[f + 1]] == t)[0]
            et = yptr[t] + np.flatnonzero(ynb[yptr[t]:yptr[t + 1]] == f)[0]
            assert yblk[ef] == bjpos[2 * l] and yblk[et] == bjpos[2 * l + 1], (r, l)
        assert np.array_equal(np.sort(bzero), np.flatnonzero(~written)), r
    assert seen["off"] > 0 and seen["ref"] > 0
    if name in ("case14_odd", "rte_case5_example", "l2rpn_neurips_2020_track1"):
        assert seen["parallel"] > 0
    if name == "case14_odd":
        assert seen["self"] > 0


@pytest.mark.parametrize("name,n,T,U", [("case14_odd", 200, 8, 1), ("case14_odd", 100, 4, 2), ("rte_case5_example", 200, 4, 2),
                                        ("l2rpn_neurips_2020_track1", 48, 32, 1)])
def test_emulated_block_kernel_vs_oracle_on_odd_lines(name, n, T, U):
    gm = _grid(name)
    topo, inj = random_cases(gm, n, seed=31, p_disc=0.05)
    out, status, iters, _ = BlockEmu(gm, T, U).run(topo, inj)
    ref, rstatus, riters, _ = COracle(gm).run(topo, inj)
    assert np.array_equal(status, rstatus)
    bad = status != 0
    assert np.isnan(out[bad]).all()
    ok = ~bad
    assert ok.sum() >= n // 4
    compare(gm, out, ref, ok)
    assert np.all(iters[ok] >= riters[ok]) and np.all(iters[ok] <= riters[ok] + 1)
