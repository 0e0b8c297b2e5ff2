"""Every solver kernel at its size limits and on grid features no bundled grid has, against the fp64 oracle.

The grids (test_kernel_limits_cpu.py): phase-shifting transformers (y_ft != y_tf, a DC injection per shifted branch), three
busbars per substation (case14: 42 bus slots, more than the warp-per-instance kernel takes; wcci: 354), case14 with a line
inside a substation and a pair of parallel lines, and these combined.  The states: random topologies and injections
(test_c_oracle.random_cases) and heavy connected splits that the oracle solves (test_kernel_limits_cpu.heavy_splits).

The pivoting path picks its kernel from the launch's nb_cap: the warp kernel up to 17 buses on grids of at most 32 bus slots,
else the generic kernel pf_kernel<T, float> with T threads per instance from generic_config (csrc/b200pf.cu), restated here
from the device's opt-in shared-memory limit, clipped matrix included.  Each case asserts the kernel and T that ran, and
ST_TOO_LARGE with NaN records for exactly the instances that exceed the bus arrays or the (clipped) matrix.  The planned
kernels (policy 2) and their pivoting safety net run on the same states; the staged lockstep production branch runs one
heavy split of case14 with three busbars and shifts at batch 4096, and every other block-kernel branch must give its bits.

Every launch prints a "LIMITS" line: kernel, threads per instance, grid variant, mode."""
import numpy as np
import pytest

from grid2op_b200.engine import ST_TOO_LARGE, OutputView, grid_max_active_buses
from oracle.c_oracle import COracle
from test_block_kernel_gpu import _env
from test_c_oracle import random_cases
from test_kernel_limits_cpu import BOUNDARY, _sub_of_input, boundary_states, heavy_splits, solved, variant
from test_waves_gpu import BRANCHES, PROD, _check_oracle, _schedule, _series_inj

pytestmark = pytest.mark.gpu
C14 = "l2rpn_case14_sandbox+psh"
ODD = "case14_odd+psh"
C14B3 = "l2rpn_case14_sandbox+b3"
C14B3P = "l2rpn_case14_sandbox+b3+psh"
T1B3P = "l2rpn_neurips_2020_track1+b3+psh"
WCCI = "l2rpn_wcci_2022_dev+b3+psh"
# variant -> (random states, heavy splits drawn (the oracle-solved ones are kept))
STATES = {C14: (96, 96), ODD: (96, 96), C14B3: (64, 96), C14B3P: (96, 96), T1B3P: (48, 48), WCCI: (8, 0)}


# ---- generic_config / redo_config of csrc/b200pf.cu, restated -------------------------------------------------------
def _a16(x):
    return (int(x) + 15) & ~15


def _ws_fixed(gm, cap):
    """ws_fixed_bytes (csrc/b200pf_kernel.cuh): the bus arrays of a workspace sized for cap buses"""
    return (_a16(17 * cap * 8) + _a16(gm.n_inj * 8) + 2 * _a16(2 * cap * 4) + _a16((gm.n_slot + 13 * cap + 2 * gm.n_line) * 2)
            + _a16(2 * cap + gm.n_slot) + 576)


def _mat_worst(cap, jt):
    d = 2 * cap
    return _a16(max(d * (d + 2) * jt, cap * (cap + 2) * 8))


def _optin():
    import torch
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def pivoting_config(gm, cap):
    """-> (kernel, threads per instance, effective cap, matrix bytes) the pivoting path launches for nb_cap = cap"""
    c = gm.n_slot if cap <= 0 or cap > gm.n_slot else cap
    if max(gm.n_slot, gm.n_line, gm.n_unit, gm.n_load, gm.n_storage, gm.n_shunt) <= 32 and c <= 17:
        return "warp_pivoting", 32, c, None
    jt = 4
    fixed, want = _ws_fixed(gm, c), _mat_worst(c, jt)
    d = 2 * c
    T = 32 if d <= 64 else (128 if d <= 128 else (256 if d <= 256 else 512))
    if fixed + want > _optin():                          # clipped: T follows the largest system that fits
        want = min(want, (_optin() - fixed) & ~15)
        dmax = 1
        while (dmax + 1) * (dmax + 3) * jt <= want:
            dmax += 1
        T = 128 if dmax <= 128 else (256 if dmax <= 256 else 512)
    return "cta_pivoting", T, c, want


def redo_in_global_memory(gm, cap):
    """redo_config: the safety net's fp64 matrix lives in global memory when the worst case of cap buses does not fit on chip"""
    return _ws_fixed(gm, cap) + _mat_worst(cap, 8) > _optin()


def newton_sizes(gm, topo):
    """(DC unknowns n1 = non-reference buses, AC unknowns d = n1 + PQ buses) of every record, as the kernels number them"""
    sub_of = _sub_of_input(gm)
    up, isref = np.asarray(gm.unit_pos), np.asarray(gm.unit_is_ref) != 0
    n1, d = np.zeros(len(topo), dtype=np.int64), np.zeros(len(topo), dtype=np.int64)
    for i, tv in enumerate(topo):
        slot = sub_of * gm.n_busbar + tv.astype(np.int64) - 1
        nb = len(np.unique(slot[tv > 0]))
        on = tv[up] > 0
        ref = np.unique(slot[up][on & isref])
        pv = np.setdiff1d(np.unique(slot[up][on]), ref)
        n1[i] = nb - len(ref)
        d[i] = 2 * n1[i] - len(pv)
    return n1, d


def expected_status(gm, topo, rstatus, cap, want, is_dc, jt=4):
    """the oracle's status, ST_TOO_LARGE where the record has more active buses than the launch's cap or, once it is
    connected, a Newton system the matrix region cannot hold (b200pf_kernel.cuh: the mat_bytes check)"""
    exp = rstatus.copy()
    if want is not None:
        n1, d = newton_sizes(gm, topo)
        over = (n1 * ((n1 + 1) | 1) * 8 > want) | ((not is_dc) & (d * ((d + 1) | 1) * jt > want))
        exp[over & (rstatus <= 1)] = ST_TOO_LARGE
    exp[grid_max_active_buses(gm, topo)[1] > cap] = ST_TOO_LARGE
    return exp


# ---- states ----------------------------------------------------------------------------------------------------------
class _Case:
    def __init__(self, key):
        self.key = key
        self.gm = gm = variant(key)
        n_rand, n_heavy = STATES[key]
        topo, inj = random_cases(gm, n_rand, seed=21)
        if n_heavy:
            ht, hi, _ = solved(gm, heavy_splits(gm, n_heavy, seed=23))
            topo, inj = np.concatenate([topo, ht]), np.concatenate([inj, hi])
        if key in BOUNDARY:
            for c, t in boundary_states(gm, key).items():
                bt, bi, _ = solved(gm, t)
                topo, inj = np.concatenate([topo, bt]), np.concatenate([inj, bi])
        self.topo, self.inj = topo, inj
        self.nb = grid_max_active_buses(gm, topo)[1]
        orc = COracle(gm)
        self.ref = {False: orc.run(topo, inj)[:3], True: orc.run(topo, inj, is_dc=True)[:3]}

    def sub(self, m):
        return self.topo[m], self.inj[m], {dc: tuple(a[m] for a in r) for dc, r in self.ref.items()}


@pytest.fixture(scope="module")
def case(cuda_required):
    cache = {}

    def get(key):
        if key not in cache:
            cache[key] = _Case(key)
        return cache[key]
    return get


def _engine(gm, B, policy, **knobs):
    from grid2op_b200.engine import PowerFlowEngine
    with _env(**knobs):
        eng = PowerFlowEngine(gm, max_batch=B)
    eng.set_kernel_policy(policy)
    return eng


def _log(eng, key, what):
    info = eng.last_launch_info()
    print(f"LIMITS kernel={eng.plan_stats()['last_kernel']} T={info['threads_per_instance']} config={info['config']} "
          f"variant={key} {what}")
    return info


def _run_pivoting(eng, c, key, topo, inj, ref, cap, dc, what):
    """one pivoting launch with nb_cap = cap: the kernel and T of pivoting_config, statuses of expected_status, oracle records"""
    gm = c.gm
    kern, T, ceff, want = pivoting_config(gm, cap)
    out, status, iters, _ = eng.run(topo, inj, is_dc=dc, nb_cap=cap)
    info = _log(eng, key, f"{what} nb_cap={cap} dc={dc}")
    assert eng.plan_stats()["last_kernel"] == kern and info["threads_per_instance"] == T, (kern, T, info)
    exp = expected_status(gm, topo, ref[1], ceff, want, dc)
    _check_oracle(gm, out, status, iters, ref[0], exp, ref[2], dc)
    return status, exp


# ---- 1. the pivoting kernel classes, by the nb_cap argument -----------------------------------------------------------
# (variant, nb_cap): each side of every class boundary — warp kernel / generic T = 32 at 17 / 18 buses, T = 32 / 128 at 33,
# 128 / 256 at 65, and on wcci with three busbars (354 slots) the clipped matrix, whose T follows the largest system that fits
CAPS = [(C14, 17), (C14, 18), (ODD, 17), (ODD, 18), (C14B3P, 32), (C14B3P, 33), (C14B3, 33), (T1B3P, 64), (T1B3P, 65),
        (WCCI, 128), (WCCI, 129), (WCCI, 354)]


@pytest.mark.parametrize("key,cap", CAPS)
def test_pivoting_kernel_class_by_nb_cap(case, key, cap):
    """only instances with at most cap active buses: every one is solved by the class the cap selects (on wcci those whose
    Newton system exceeds a clipped matrix excepted: ST_TOO_LARGE)"""
    c = case(key)
    m = c.nb <= cap
    topo, inj, ref = c.sub(m)
    assert (ref[False][1] == 0).sum() >= 4 and c.nb[m].max() >= min(cap, c.nb.max()) - 4, (c.nb[m].max(), cap)
    eng = _engine(c.gm, len(topo), 1)
    for dc in (False, True):
        status, exp = _run_pivoting(eng, c, key, topo, inj, ref[dc], cap, dc, "by-cap")
        assert (status == 0).sum() >= 4
    eng.close()


# ---- 2. by the real bus counts at the boundaries ----------------------------------------------------------------------
@pytest.mark.parametrize("key", sorted(BOUNDARY))
def test_pivoting_kernel_class_at_real_bus_counts(case, key):
    """Instances with exactly 17 and 18 active buses (case14, two and three busbars) and 128 and 129 (wcci, three busbars),
    each count alone at its tight cap; then both counts in one launch capped at the lower one: the larger instances come
    back ST_TOO_LARGE, the others still match the oracle.  With three busbars case14 has 42 bus slots: 17 buses go to the
    generic kernel, not the warp kernel."""
    c = case(key)
    lo, hi = BOUNDARY[key][0]
    for cnt in (lo, hi):
        topo, inj, ref = c.sub(c.nb == cnt)
        assert len(topo) >= 2, (key, cnt)
        eng = _engine(c.gm, len(topo), 1)
        for dc in (False, True):
            status, _ = _run_pivoting(eng, c, key, topo, inj, ref[dc], cnt, dc, f"real-count={cnt}")
            assert (status == 0).sum() >= 2
        eng.close()
    m = (c.nb == lo) | (c.nb == hi)
    topo, inj, ref = c.sub(m)
    eng = _engine(c.gm, len(topo), 1)
    status, exp = _run_pivoting(eng, c, key, topo, inj, ref[False], lo, False, f"cap-below={lo}")
    assert (status[c.nb[m] == hi] == ST_TOO_LARGE).all() and (status[c.nb[m] == lo] == 0).sum() >= 2
    eng.close()


# ---- 3. nb_cap: tight, every slot, one below the largest instance -----------------------------------------------------
@pytest.mark.parametrize("key", [C14, ODD, C14B3, C14B3P, T1B3P, WCCI])
def test_pivoting_nb_cap_variants(case, key):
    c = case(key)
    tight = int(c.nb.max())
    eng = _engine(c.gm, len(c.topo), 1)
    seen_large = 0
    for cap in (tight, 0, tight - 1):
        for dc in (False, True):
            status, exp = _run_pivoting(eng, c, key, c.topo, c.inj, c.ref[dc], cap, dc, "cap-variant")
            assert (status == 0).sum() >= len(status) // 4
            seen_large += int((status == ST_TOO_LARGE).sum())
    assert seen_large >= 2 * int((c.nb == tight).sum())
    eng.close()


# ---- 4. the planned kernels and their safety net ----------------------------------------------------------------------
def _planned(key, gm):
    """(knobs, expected kernel, expected lanes per instance or None) of the planned runs of a variant"""
    runs = [({}, "planned_block" if gm.n_line <= 32 else "planned_sparse", 8 if gm.n_line <= 32 else None),
            ({"B200PF_BLOCK": 0}, "planned_sparse", None),
            ({"B200PF_BLOCK": 1}, "planned_block", 8 if gm.n_line <= 32 else (32 if gm.n_line <= 64 else 64))]
    if key == T1B3P:      # lanes that own 5 to 8 buses (T = 8) and 3 to 4 (T = 16)
        runs += [({"B200PF_BLOCK": 1, "B200PF_BLOCK_T": t, "B200PF_BLOCK_U": 1}, "planned_block", t) for t in (8, 16)]
    return runs


@pytest.mark.parametrize("key", [C14, ODD, C14B3, C14B3P, T1B3P, WCCI])
def test_planned_kernels_and_safety_net(case, key):
    """Policy 2 on the same states: the default family, the scalar and the block kernel; AC and DC against the oracle.  Then
    the safety net: every third instance forced to give up, so the pivoting re-solve (pf_kernel_redo, fp64, global-memory
    matrix on wcci with three busbars) must give the oracle's status; and with nb_cap one below the largest instance the
    forced instances above it keep the planned kernel's DIVERGED (the re-solve cannot hold them), all others unchanged."""
    c = case(key)
    gm = c.gm
    B = len(c.topo)
    tight = int(c.nb.max())
    for knobs, kern, T in _planned(key, gm):
        eng = _engine(gm, B, 2, **knobs)
        for dc in (False, True):
            out, status, iters, _ = eng.run(c.topo, c.inj, is_dc=dc)
            info = _log(eng, key, f"planned {knobs} dc={dc}")
            assert eng.plan_stats()["last_kernel"] == kern, (knobs, info)
            if T is not None:
                assert info["config"][0] == T, (knobs, info)
            _check_oracle(gm, out, status, iters, *c.ref[dc], dc)
        if knobs:
            eng.close()
            continue
        # the safety net on the same states
        forced = (np.arange(B) % 3 == 0) & (c.ref[False][1] <= 1)
        assert forced.sum() >= 4
        eng.set_debug(3, True)
        n0 = eng.redo_launch_count
        out, status, iters, _ = eng.run(c.topo, c.inj)
        assert eng.redo_launch_count > n0
        print(f"LIMITS kernel=redo global_matrix={redo_in_global_memory(gm, tight)} variant={key} cap={tight}")
        _check_oracle(gm, out, status, iters, *c.ref[False], False)
        n0 = eng.redo_launch_count
        out, status, iters, _ = eng.run(c.topo, c.inj, nb_cap=tight - 1)
        assert eng.redo_launch_count > n0
        exp = np.where(forced & (c.nb > tight - 1), 1, c.ref[False][1])
        assert (forced & (c.nb > tight - 1) & (c.ref[False][1] == 0)).any()
        _check_oracle(gm, out, status, iters, c.ref[False][0], exp, c.ref[False][2], False)
        eng.set_debug(0, True)
        eng.close()
    if key == WCCI:
        assert redo_in_global_memory(gm, tight)


# ---- 5. N-1 on the shifted and odd grids ------------------------------------------------------------------------------
@pytest.mark.parametrize("key", [C14, ODD, C14B3P])
@pytest.mark.parametrize("policy", [1, 2])
def test_n1_sweep_on_shifted_and_odd_grids(case, key, policy):
    c = case(key)
    gm, nl = c.gm, c.gm.n_line
    pick = np.flatnonzero(c.ref[False][1] == 0)[::8][:12]
    topo, inj = c.topo[pick], c.inj[pick]
    nbase = len(topo)
    eng = _engine(gm, nbase * nl, policy)
    rho, status = eng.n1_sweep(topo, inj)
    _log(eng, key, f"n1 policy={policy}")
    assert eng.plan_stats()["last_kernel"].startswith("planned") == (policy == 2)
    eng.close()
    t2, i2 = np.repeat(topo, nl, axis=0), np.repeat(inj, nl, axis=0)
    for b in range(nbase):
        for l in range(nl):
            t2[b * nl + l, gm.line_or_pos[l]] = -1
            t2[b * nl + l, gm.line_ex_pos[l]] = -1
    ref, rs, _, _ = COracle(gm).run(t2, i2)
    rs = rs.reshape(nbase, nl)
    assert np.array_equal(status, rs), np.argwhere(status != rs)[:5]
    ok = status == 0
    assert ok.sum() > ok.size // 2 and np.isnan(rho[~ok]).all()
    want = (OutputView(gm, ref).a_or / gm.thermal_limit_a[None, :]).reshape(nbase, nl, nl)
    assert np.max(np.abs(rho[ok] - want[ok])) <= 2e-5 * max(1.0, float(np.max(want[ok])))
    assert all(np.all(rho[ok[:, l], l, l] == 0.0) for l in range(nl))


# ---- 6. the production branch on a heavy split with three busbars and shifts -----------------------------------------
def test_series_heavy_split_three_busbars_shifts(case):
    """One heavy split of case14 (three busbars, shifted transformers) that the oracle solves on more than 90 % of the
    chronics states, on the series path at batch 4096: the staged lockstep branch of the bench workload (PROD), against the
    oracle; then every other launch_block branch (BRANCHES) bit-equal to it, state by state."""
    import os
    from test_bus_chains_gpu import _run
    c = case(C14B3P)
    gm = c.gm
    gold = os.path.join(os.path.dirname(__file__), "golden")
    chron = np.load(os.path.join(gold, "case14_sandbox_chronics.npz"))["chron"]
    n_rows = chron.shape[1]
    n_state = chron.shape[0] * n_rows
    inj = _series_inj(gm, chron, np.arange(n_state) // n_rows, np.arange(n_state) % n_rows)
    orc = COracle(gm)
    picked = None
    for topo in heavy_splits(gm, 48, seed=29):
        if (topo == 3).sum() < 3:
            continue
        res = orc.run(np.tile(topo, (n_state, 1)), inj)[:3]
        if (res[1] == 0).mean() > 0.9:
            picked = topo, res
            break
    assert picked is not None
    topo, (ref, rstatus, riters) = picked
    nb = grid_max_active_buses(gm, topo[None])[0]
    assert nb >= 19, nb
    tab = [np.full((n_state, gm.n_out), np.nan, dtype=np.float32), np.full(n_state, -1, dtype=np.int32),
           np.full(n_state, -1, dtype=np.int32), np.full((n_state, gm.n_line), np.nan, dtype=np.float32)]
    for st, out, status, iters, rho, info in _run(gm, chron, n_rows, topo, 4096, 2):
        assert info["config"] == PROD[2], info
        print(f"LIMITS kernel=planned_block T=8 config={info['config']} variant={C14B3P} series nb={nb}")
        _check_oracle(gm, out, status, iters, ref[st], rstatus[st], riters[st], False, rho)
        assert (status == 0).mean() > 0.9
        tab[0][st], tab[1][st], tab[2][st], tab[3][st] = out, status, iters, rho
    for knobs, B, cfg in BRANCHES:
        for st, out, status, iters, rho, info in _run(gm, chron, n_rows, topo, B, 1, knobs):
            assert info["config"] == cfg, (knobs, B, info)
            print(f"LIMITS kernel=planned_block T=8 config={info['config']} variant={C14B3P} series-branch B={B}")
            assert (tab[1][st] >= 0).all()
            assert np.array_equal(status, tab[1][st]) and np.array_equal(iters, tab[2][st]), knobs
            assert np.array_equal(out, tab[0][st], equal_nan=True), knobs
            assert np.array_equal(rho, tab[3][st], equal_nan=True), knobs
