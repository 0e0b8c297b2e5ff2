"""The block kernel's bus phase and state update on the GPU when a lane has more than two buses: case14 topologies with split
substations (more than 16 active buses, so each of the 8 lanes of an instance runs a second group of two buses), as the
bench workload runs them (series path, one topology for the batch, batch 4096), against the fp64 oracle; and every other
launch_block branch bit-equal to the production kernel on the same topologies."""
import os

import numpy as np
import pytest

from grid2op_b200.engine import grid_max_active_buses
from grid2op_b200.gridmodel import GridModel
from oracle.c_oracle import COracle
from test_block_kernel_gpu import _env
from test_bus_chains_cpu import split_cases
from test_waves_gpu import BRANCHES, PROD, _check_oracle, _schedule, _series_inj

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
N_TOPO = 3


@pytest.fixture(scope="module")
def split14(cuda_required):
    """N_TOPO split topologies of case14 (17 to 20 active buses) that the oracle solves on every chronics state, with the
    oracle's results of all states"""
    gm = GridModel.from_npz(os.path.join(GOLD, "gridmodel_l2rpn_case14_sandbox.npz"))
    chron = np.load(os.path.join(GOLD, "case14_sandbox_chronics.npz"))["chron"]
    n_rows = chron.shape[1]
    n_state = chron.shape[0] * n_rows
    inj = _series_inj(gm, chron, np.arange(n_state) // n_rows, np.arange(n_state) % n_rows)
    cand, _ = split_cases(gm, 400, seed=3)
    nb = grid_max_active_buses(gm, cand)[1]
    orc = COracle(gm)
    picked = []
    for want in (17, 18, 20, 19):
        for r in np.flatnonzero(nb == want):
            res = orc.run(np.tile(cand[r], (n_state, 1)), inj)[:3]
            if (res[1] == 0).mean() > 0.9:
                picked.append((cand[r], int(nb[r]), res))
                break
        if len(picked) == N_TOPO:
            break
    assert len(picked) == N_TOPO, [p[1] for p in picked]
    return gm, chron, n_rows, picked


def _run(gm, chron, n_rows, topo, B, steps, knobs=None):
    from grid2op_b200.rollout import BatchedDoNothing
    scen, t0 = _schedule(B, n_rows)
    with _env(**(knobs or {})):
        env = BatchedDoNothing(gm, chron, B, scen=scen, t0=t0)
    env.engine.series_set_topo(np.tile(topo, (B, 1)))
    res = []
    for k in range(steps):
        env.step_device()
        out, status, iters, rho = env.fetch()
        assert env.engine.plan_stats()["last_kernel"] == "planned_block"
        st = scen.astype(np.int64) * n_rows + (t0 + k) % n_rows
        res.append((st, out, status, iters, rho, env.engine.last_launch_info()))
    env.close()
    return res


def test_production_kernel_on_split_substations(split14):
    gm, chron, n_rows, picked = split14
    for topo, nb, (ref, rstatus, riters) in picked:
        assert nb > 16
        for st, out, status, iters, rho, info in _run(gm, chron, n_rows, topo, 4096, 2):
            assert info["config"] == PROD[2], info
            _check_oracle(gm, out, status, iters, ref[st], rstatus[st], riters[st], False, rho)
            assert (status == 0).mean() > 0.9


def test_every_block_branch_is_bit_equal_on_split_substations(split14):
    """each launch_block branch (tests/test_waves_gpu.py) gives the production kernel's bits, state by state"""
    gm, chron, n_rows, picked = split14
    n_state = chron.shape[0] * n_rows
    for topo, nb, _ in picked[:2]:
        tab = [np.full((n_state, gm.n_out), np.nan, dtype=np.float32), np.full(n_state, -1, dtype=np.int32),
               np.full(n_state, -1, dtype=np.int32), np.full((n_state, gm.n_line), np.nan, dtype=np.float32)]
        for st, out, status, iters, rho, info in _run(gm, chron, n_rows, topo, 4096, 1):
            assert info["config"] == PROD[2], info
            tab[0][st], tab[1][st], tab[2][st], tab[3][st] = out, status, iters, rho
        for knobs, B, cfg in BRANCHES:
            for st, out, status, iters, rho, info in _run(gm, chron, n_rows, topo, B, 1, knobs):
                assert info["config"] == cfg, (knobs, B, info)
                assert (tab[1][st] >= 0).all()
                assert np.array_equal(status, tab[1][st]) and np.array_equal(iters, tab[2][st]), (knobs, nb)
                assert np.array_equal(out, tab[0][st], equal_nan=True), (knobs, nb)
                assert np.array_equal(rho, tab[3][st], equal_nan=True), (knobs, nb)
