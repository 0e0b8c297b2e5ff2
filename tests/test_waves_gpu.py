"""Persistent kernels past their first resident wave, and every dispatch branch of the block kernel, against the fp64 oracle.

Every solver kernel is persistent: the host sizes the grid to what is resident (rounds = ceil(work / resident)) and each warp or
CTA loops over the grid, solving instance group after instance group in the same shared-memory workspace.  The batches here are
chosen so that the loop runs at least twice; each test reads the kernel configuration it targets from the library
(`last_launch_info()["config"]`, b200pf_last_launch_config) and the number of waves it ran,
waves = ceil(batch / (grid * block / threads_per_instance)), instead of assuming them.

Oracle cost is kept small by deduplication.  In series mode with one topology an instance's state is (scenario, row): the oracle
solves the 1728 states of the case14 chronics once, and its results are broadcast.  Every instance that solved the same state
must also have BIT-IDENTICAL records, status, iterations and rho, whatever its lane, warp, CTA or wave.  Batches of random
topologies repeat N states, instance i taking state i mod N, with N coprime to the instances per CTA, so that the copies land
in different positions.  Every launch also checks that a wave is no whole number of repetitions: a warp's next instance is
then another state than its last one, and a value left over in its workspace cannot pass for the right one.
"""
import os

import numpy as np
import pytest

from grid2op_b200.engine import OutputView, grid_max_active_buses
from grid2op_b200.gridmodel import GridModel
from oracle.c_oracle import COracle
from test_block_kernel_gpu import _env
from test_c_oracle import random_cases
from test_engine_random_gpu import _compare
from test_redo_gpu import fast_random_cases

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
NS = 1727               # distinct start states of the series schedule: odd, so copies of a state sit in different lanes


# ---- helpers ---------------------------------------------------------------------------------------------------------
def _check_waves(batch, info, n_states, at_least=2):
    """the launch ran at least `at_least` waves, and a wave is no whole number of repetitions of the n_states states of the
    batch (instance i has state i mod n_states): what a warp solves in its next round is another state than in its last"""
    per_wave = info["grid"] * info["block"] // info["threads_per_instance"]
    assert -(-batch // per_wave) >= at_least and per_wave % n_states != 0, (batch, n_states, info)


def _schedule(batch, n_rows):
    """instance i starts at state s = i mod NS: scenario s mod 3, row s // 3 (s = 1725, 1726 start on the last row)"""
    s = np.arange(batch) % NS
    return (s % 3).astype(np.int32), (s // 3 % n_rows).astype(np.int32)


def _series_inj(gm, chron, scen, rows):
    """the fp64 injection records the series kernels build from chronics rows (test_engine_random_gpu)"""
    r = chron[scen, rows]
    sl = gm.inj_slices()
    nl, ng = gm.n_load, gm.n_gen
    inj = np.tile(gm.default_inj(), (len(scen), 1))
    inj[:, sl["load_p"]] = r[:, :nl]
    inj[:, sl["load_q"]] = r[:, nl:2 * nl]
    inj[:, sl["gen_p"]] = r[:, 2 * nl:2 * nl + ng]
    inj[:, sl["gen_vm"]] = (r[:, 2 * nl + ng:] / gm.prod_pu_to_kv[None, :]).astype(np.float32)
    return inj


def _check_oracle(gm, out, status, iters, ref, rstatus, riters, is_dc, rho=None):
    assert np.array_equal(status, rstatus), np.flatnonzero(status != rstatus)[:10]
    ok = status == 0
    assert np.isnan(out[~ok]).all() and not np.isnan(out[ok]).any()
    _compare(gm, out, ref, ok)
    if not is_dc:
        d = iters[ok].astype(np.int64) - riters[ok]
        assert d.size == 0 or (d.min() >= -1 and d.max() <= 1), (d.min(), d.max())
    if rho is not None:
        assert np.array_equal(rho, OutputView(gm, out).a_or / gm.thermal_limit_a[None, :], equal_nan=True)


def _check_copies(key, *arrays):
    """instances with the same key (state) hold bit-identical values"""
    _, first, inv = np.unique(key, return_index=True, return_inverse=True)
    rep = first[inv]
    for a in arrays:
        if not np.array_equal(a, a[rep], equal_nan=True):
            b = a.reshape(len(a), -1)
            bad = np.flatnonzero(~np.all((b == b[rep]) | (np.isnan(b) & np.isnan(b[rep])), axis=1))
            pytest.fail(f"{len(bad)} instances differ from the first instance of their state: {bad[:10]} vs {rep[bad[:10]]}")


class _Case14:
    def __init__(self):
        self.gm = GridModel.from_npz(os.path.join(GOLD, "gridmodel_l2rpn_case14_sandbox.npz"))
        gm = self.gm
        self.chron = np.load(os.path.join(GOLD, "case14_sandbox_chronics.npz"))["chron"]
        self.n_rows = self.chron.shape[1]
        n_state = self.chron.shape[0] * self.n_rows
        sc, rw = np.arange(n_state) // self.n_rows, np.arange(n_state) % self.n_rows
        topo = np.tile(gm.default_topo(), (n_state, 1))
        inj = _series_inj(gm, self.chron, sc, rw)
        orc = COracle(gm)
        self.ac = orc.run(topo, inj)[:3]
        self.dc = orc.run(topo, inj, is_dc=True)[:3]
        self.tab = None                  # per state: records, status, iterations, rho of the production kernel

    def state(self, scen, rows):
        return scen.astype(np.int64) * self.n_rows + rows % self.n_rows

    def check(self, B, t0, scen, k, res, is_dc=False, tab=True):
        """step k (0-based) of a series bound with (scen, t0): oracle, copies, and bit equality with the production table"""
        out, status, iters, rho = res
        st = self.state(scen[:B], t0[:B] + k)
        ref, rstatus, riters = self.dc if is_dc else self.ac
        _check_oracle(self.gm, out, status, iters, ref[st], rstatus[st], riters[st], is_dc, rho)
        _check_copies(st, out, status, iters, rho)
        if tab:
            self.check_tab(st, out, status, iters, rho)
        return st

    def check_tab(self, st, out, status, iters, rho=None):
        to, ts, ti, tr = self.tab
        assert np.array_equal(out, to[st], equal_nan=True)
        assert np.array_equal(status, ts[st]) and np.array_equal(iters, ti[st])
        if rho is not None:
            assert np.array_equal(rho, tr[st], equal_nan=True)

    def series(self, B, **kw):
        from grid2op_b200.rollout import BatchedDoNothing
        scen, t0 = _schedule(B, self.n_rows)
        return BatchedDoNothing(self.gm, self.chron, B, scen=scen, t0=t0, **kw), scen, t0


@pytest.fixture(scope="module")
def c14(cuda_required):
    """case14 oracle results of all 1728 chronics states, and the production kernel's results of every state (3 steps of
    the bench workload's kernel at batch 32 768, 4 waves) as the table the other kernels must reproduce bit for bit"""
    c = _Case14()
    gm = c.gm
    n_state = c.chron.shape[0] * c.n_rows
    to = np.full((n_state, gm.n_out), np.nan, dtype=np.float32)
    ts = np.full(n_state, -1, dtype=np.int32)
    ti = np.full(n_state, -1, dtype=np.int32)
    tr = np.full((n_state, gm.n_line), np.nan, dtype=np.float32)
    env, scen, t0 = c.series(32768)
    for k in range(3):
        env.step_device()
        out, status, iters, rho = env.fetch()
        assert env.engine.last_launch_info()["config"] == (8, 1, 8, 0, 2, 1, 1, 1)
        st = c.state(scen, t0 + k)
        _, first = np.unique(st, return_index=True)
        to[st[first]], ts[st[first]], ti[st[first]], tr[st[first]] = out[first], status[first], iters[first], rho[first]
    env.close()
    assert (ts >= 0).all(), "the schedule must reach every state"
    c.tab = (to, ts, ti, tr)
    return c


PROD = {2: (8, 1, 8, 0, 2, 1, 1, 1), 4: (8, 1, 4, 0, 4, 1, 1, 1)}        # the stepping kernel of the two WPC branches


def _prod_cfg(B, mode=1):
    return PROD[2 if B <= 32768 else 4][:7] + (mode,)


# ---- 1. the production kernel across waves ---------------------------------------------------------------------------
@pytest.mark.parametrize("B", [32768, 40000, 32772])
def test_production_kernel_across_waves(c14, B):
    """32 768: WPC 2, 4096 instance groups; 40 000: WPC 4; 32 772: the first batch above the WPC switch — 8193 instance groups,
    so the last round of one warp runs alone in its CTA.  The instances with i mod 1727 = 1725 or 1726 start on the last
    chronics row: their second step wraps to row 0."""
    env, scen, t0 = c14.series(B)
    assert (t0 == c14.n_rows - 1).any()
    for k in range(3):
        env.step_device()
        res = env.fetch()
        info = env.engine.last_launch_info()
        assert info["config"] == _prod_cfg(B), info
        _check_waves(B, info, NS)
        c14.check(B, t0, scen, k, res)
    env.close()


# ---- 2. the MODE 0 twins of the staged kernel ------------------------------------------------------------------------
@pytest.mark.parametrize("B", [32768, 40000, 32772])
def test_mode0_staged_twins_across_waves(c14, B):
    """host records of one topology (AC: bit-equal to the series kernel) and the DC series, both on the generic (MODE 0)
    instantiation of the staged lockstep kernel"""
    from grid2op_b200.engine import PowerFlowEngine
    gm = c14.gm
    scen, t0 = _schedule(B, c14.n_rows)
    eng = PowerFlowEngine(gm, max_batch=B)
    out, status, iters, _ = eng.run(np.tile(gm.default_topo(), (B, 1)), _series_inj(gm, c14.chron, scen, t0))
    info = eng.last_launch_info()
    eng.close()
    assert info["config"] == _prod_cfg(B, 0), info
    _check_waves(B, info, NS)
    st = c14.state(scen, t0)
    _check_oracle(gm, out, status, iters, c14.ac[0][st], c14.ac[1][st], c14.ac[2][st], False)
    _check_copies(st, out, status, iters)
    c14.check_tab(st, out, status, iters)
    env, scen, t0 = c14.series(B, is_dc=True)
    for k in range(2):
        env.step_device()
        res = env.fetch()
        info = env.engine.last_launch_info()
        assert info["config"] == _prod_cfg(B, 0), info
        _check_waves(B, info, NS)
        c14.check(B, t0, scen, k, res, is_dc=True, tab=False)
    env.close()


# ---- 3. every launch_block branch gives the same bits ----------------------------------------------------------------
# (knobs, batch, instantiation (T, U, MINB, PROT, WPC, STAGE, UNI, MODE)).  40 000 instances of 8 lanes exceed what 132 SMs of
# 2048 threads can hold (33 792), so every branch runs at least 2 waves there; the default WPC 2 branch needs a batch <= 32 768
# and the free-running one a batch that is not a multiple of 4.
BRANCHES = [
    ({}, 32768, (8, 1, 8, 0, 2, 1, 1, 1)),                                                  # staged lockstep, WPC 2
    ({}, 40000, (8, 1, 4, 0, 4, 1, 1, 1)),                                                  # staged lockstep, WPC 4
    ({"B200PF_BLOCK_WPC": 1}, 40000, (8, 1, 16, 0, 1, 1, 1, 0)),                            # staged lockstep, WPC 1
    ({"B200PF_BLOCK_SPEC": 0}, 32768, (8, 1, 8, 0, 2, 1, 1, 0)),                            # staged, not specialised
    ({"B200PF_BLOCK_UNI": 0}, 40000, (8, 1, 4, 0, 4, 1, 0, 0)),                             # staged free-running
    ({"B200PF_BLOCK_STAGE": 0}, 40000, (8, 1, 16, 0, 1, 0, 1, 0)),                          # unstaged lockstep
    ({"B200PF_BLOCK_STAGE": 0, "B200PF_BLOCK_WPC": 4}, 40000, (8, 1, 4, 0, 4, 0, 0, 0)),    # unstaged free-running, WPC 4
    ({}, 39999, (8, 1, 16, 0, 1, 0, 0, 0)),                                                 # free-running (batch % 4 != 0)
]


def test_every_block_branch_is_bit_equal(c14):
    """The branches only reorganise who solves which instance: each must reproduce the production kernel's table bit for
    bit (so they are bit-equal to each other), and the oracle."""
    seen = set()
    for knobs, B, cfg in BRANCHES:
        with _env(**knobs):
            env, scen, t0 = c14.series(B)
        for k in range(3):
            env.step_device()
            res = env.fetch()
            info = env.engine.last_launch_info()
            assert env.engine.plan_stats()["last_kernel"] == "planned_block"
            assert info["config"] == cfg, (knobs, B, info)
            _check_waves(B, info, NS)
            c14.check(B, t0, scen, k, res)
        env.close()
        seen.add(cfg)
    assert len(seen) == len(BRANCHES)


# ---- 4. a staged launch whose one plan is unsolvable -----------------------------------------------------------------
def test_staged_launch_of_an_unsolvable_plan_advances_rows_once(c14):
    """Every line of substation 3 (load 2, no generator) open: one unsolvable plan for the whole batch, so the staged kernel
    loads no row (row_ahead = 0) and only advances a.t.  Two such steps, then the default topology: every instance solves
    row t0 + 2."""
    gm = c14.gm
    B = 32768
    bad = gm.default_topo().copy()
    m = (gm.line_or_sub == 3) | (gm.line_ex_sub == 3)
    bad[gm.line_or_pos[m]] = -1
    bad[gm.line_ex_pos[m]] = -1
    env, scen, t0 = c14.series(B)
    env.engine.series_set_topo(np.tile(bad, (B, 1)))
    for k in range(2):
        env.step_device()
        out, status, iters, rho = env.fetch()
        info = env.engine.last_launch_info()
        assert info["config"] == PROD[2], info
        _check_waves(B, info, NS)
        st = c14.state(scen, t0 + k)
        _, first = np.unique(st, return_index=True)
        inj = _series_inj(gm, c14.chron, scen[first], (t0[first] + k) % c14.n_rows)
        _, rstatus, _, _ = COracle(gm).run(np.tile(bad, (len(first), 1)), inj)
        assert (rstatus != 0).all()
        assert np.array_equal(status[first], rstatus)
        _check_copies(st, status)
        assert np.isnan(out).all() and np.isnan(rho).all()
    env.engine.series_set_topo(np.tile(gm.default_topo(), (B, 1)))
    env.step_device()
    res = env.fetch()
    assert env.engine.last_launch_info()["config"] == PROD[2]
    c14.check(B, t0, scen, 2, res)
    env.close()


# ---- 5. free-running mixed-plan block kernel -------------------------------------------------------------------------
@pytest.mark.parametrize("grid,n", [("l2rpn_case14_sandbox", 1000), ("rte_case5_example", 300)])
def test_mixed_plan_block_kernel_across_waves(cuda_required, grid, n):
    """Random topologies (a plan per instance): the free-running block kernel with one warp per CTA and 4 instances per
    warp.  N = n + 1 states (odd) repeated over 40 000 instances, a batch that is no multiple of N: a wave is then no whole
    number of repetitions, so over the waves a warp's instances change plans, some from a plan with more buses (a bus split)
    to a smaller one and others the reverse (asserted)."""
    from grid2op_b200.engine import PowerFlowEngine
    gm = GridModel.from_npz(os.path.join(GOLD, f"gridmodel_{grid}.npz"))
    topo, inj = fast_random_cases(gm, n, seed=77)
    extra = gm.default_inj()
    extra[gm.inj_slices()["load_p"]] *= 1.01
    topo, inj = np.concatenate([topo, topo[:1]]), np.concatenate([inj, extra[None]])
    N, B = n + 1, 40000
    idx = np.arange(B) % N
    eng = PowerFlowEngine(gm, max_batch=B)
    eng.set_kernel_policy(2)
    out, status, iters, _ = eng.run(topo[idx], inj[idx])
    info = eng.last_launch_info()
    assert eng.plan_stats()["last_kernel"] == "planned_block"
    assert info["config"] == (8, 1, 16, 0, 1, 0, 0, 0), info
    _check_waves(B, info, N)
    eng.close()
    # the warp of CTA c solves the instance groups c, c + grid, ... of 4 instances each: its largest plan (active buses) in
    # the first two rounds
    n_grp, grid_n = -(-B // 4), info["grid"]
    nb = np.full(4 * max(n_grp, 2 * grid_n), -1)
    nb[:B] = grid_max_active_buses(gm, topo)[1][idx]
    nb = nb.reshape(-1, 4).max(axis=1)
    first, second = nb[:grid_n], nb[grid_n:2 * grid_n]
    both = second >= 0
    assert (first[both] > second[both]).any() and (first[both] < second[both]).any()
    ref, rstatus, riters, _ = COracle(gm).run(topo, inj)
    _check_oracle(gm, out, status, iters, ref[idx], rstatus[idx], riters[idx], False)
    assert (status == 0).any() and (status != 0).any()
    _check_copies(idx, out, status, iters)


# ---- 6. pivoting kernels ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", ["warp_pivoting", "cta_pivoting"])
def test_pivoting_kernels_across_waves(cuda_required, kernel):
    """pf_kernel_small (one warp per instance, case14, >= 3 waves: 132 SMs hold at most 4224 one-warp CTAs) and
    pf_kernel<T, float> (a CTA per instance, 36-substation grid, >= 2 waves), on the random states their own tests use"""
    from grid2op_b200.engine import PowerFlowEngine
    if kernel == "warp_pivoting":
        gm = GridModel.from_npz(os.path.join(GOLD, "gridmodel_l2rpn_case14_sandbox.npz"))
        topo, inj = random_cases(gm, 384, seed=23)
        keep = grid_max_active_buses(gm, topo)[1] <= 17          # what the warp-per-instance kernel takes
        topo, inj = topo[keep], inj[keep]
        B, min_waves = 9000, 3
    else:
        gm = GridModel.from_npz(os.path.join(GOLD, "gridmodel_l2rpn_neurips_2020_track1.npz"))
        topo, inj = random_cases(gm, 128, seed=11)
        B, min_waves = 2600, 2
    N = len(topo)
    idx = np.arange(B) % N
    eng = PowerFlowEngine(gm, max_batch=B)
    eng.set_kernel_policy(1)
    cap = eng.max_active_buses(topo)
    out, status, iters, _ = eng.run(topo[idx], inj[idx], nb_cap=cap)
    info = eng.last_launch_info()
    assert eng.plan_stats()["last_kernel"] == kernel
    assert info["config"] == (-1,) * 8, info
    if kernel == "warp_pivoting":
        assert info["block"] == 32 and info["threads_per_instance"] == 32, info
    _check_waves(B, info, N, min_waves)
    eng.close()
    ref, rstatus, riters, _ = COracle(gm).run(topo, inj)
    _check_oracle(gm, out, status, iters, ref[idx], rstatus[idx], riters[idx], False)
    assert (status == 0).sum() >= B // 4
    _check_copies(idx, out, status, iters)


# ---- 7. the safety net beyond its grid cap ---------------------------------------------------------------------------
def test_safety_net_loops_beyond_its_grid_cap(c14):
    """Every third instance forced to give up at batch 40 000: the re-solve's grid is capped at 8 CTAs of 32 instances per
    SM, so its CTAs loop.  Forced instances (those in the last 32-instance range and those on the last chronics row among them)
    equal the oracle on the row they were due to solve, the others are bit-equal to an undisturbed run, and no row advances
    twice."""
    import torch
    B = 40000
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    redo_grid = min(-(-B // 32), sm * 8)                  # redo_config in csrc/b200pf.cu
    assert -(-B // (32 * redo_grid)) >= 2, (sm, redo_grid)
    env, scen, t0 = c14.series(B)
    eng = env.engine
    forced = np.arange(B) % 3 == 0
    assert forced[B - 32:].any() and (forced & (t0 == c14.n_rows - 1)).any()
    eng.set_debug(3, True)
    n0 = eng.redo_launch_count
    for k in range(3):
        env.step_device()
        out, status, iters, rho = env.fetch()
        assert eng.redo_launch_count == n0 + k + 1
        info = eng.last_launch_info()
        assert info["config"] == PROD[4], info
        _check_waves(B, info, NS)
        st = c14.state(scen, t0 + k)
        _check_oracle(c14.gm, out, status, iters, c14.ac[0][st], c14.ac[1][st], c14.ac[2][st], False, rho)
        assert (status == 0).all()
        u = ~forced
        c14.check_tab(st[u], out[u], status[u], iters[u], rho[u])
        _check_copies(st[forced], out[forced], status[forced], iters[forced], rho[forced])
    eng.set_debug(0, True)
    env.step_device()
    res = env.fetch()
    assert eng.redo_launch_count == n0 + 3
    c14.check(B, t0, scen, 3, res)
    env.close()


# ---- 8. the scalar planned kernel's variants -------------------------------------------------------------------------
@pytest.mark.parametrize("knobs,T,MINB", [({}, 32, 32), ({"B200PF_SPARSE_T": 64}, 64, 10), ({"B200PF_SPARSE_T": 128}, 128, 4),
                                          ({"B200PF_SPARSE_MINB": 28}, 32, 28)])
def test_sparse_kernel_variants_across_waves(c14, knobs, T, MINB):
    """B200PF_BLOCK=0: pf_kernel_sparse<T, MINB>.  The one-warp variant's MINB follows the CTAs per SM the workspace allows
    (case14: 2.5 KB, so 32 — or 28 under its knob); 9000 instances exceed what any variant holds in one wave."""
    import torch
    B = 9000
    with _env(B200PF_BLOCK=0, **knobs):
        env, scen, t0 = c14.series(B)
    for k in range(2):
        env.step_device()
        res = env.fetch()
        info = env.engine.last_launch_info()
        assert env.engine.plan_stats()["last_kernel"] == "planned_sparse"
        per_sm = torch.cuda.get_device_properties(0).shared_memory_per_block_optin // (info["smem_bytes"] + 1024)
        assert info["config"] == (T, -1, MINB, 0, -1, -1, -1, -1), (info, per_sm)
        _check_waves(B, info, NS)
        c14.check(B, t0, scen, k, res, tab=False)
    env.close()
