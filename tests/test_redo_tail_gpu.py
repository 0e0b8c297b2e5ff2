"""The planned kernels launch their pivoting safety net from the device (csrc/b200pf_redo.cuh): a tail launch that fires only
when a launch leaves an instance as DIVERGED, one per such launch, with one control word per stream.

Case14 series at batch 4096: one topology plan for the whole batch, so every step runs the staged lockstep block kernel.
"""
import os

import numpy as np
import pytest

from grid2op_b200.gridmodel import GridModel
from test_engine_random_gpu import _compare

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
B = 4096


def _case14():
    gm = GridModel.from_npz(os.path.join(GOLD, "gridmodel_l2rpn_case14_sandbox.npz"))
    chron = np.load(os.path.join(GOLD, "case14_sandbox_chronics.npz"))["chron"]
    return gm, chron


def test_tail_launch_fires_once_per_step_with_failures_only(cuda_required):
    from grid2op_b200.rollout import BatchedDoNothing
    gm, chron = _case14()
    ref = BatchedDoNothing(gm, chron, B)
    env = BatchedDoNothing(gm, chron, B)
    eng = env.engine
    # no instance diverges: the planned kernel launches nothing behind itself
    n0 = eng.redo_launch_count
    for _ in range(3):
        ref.step_device(); env.step_device()
        o1, s1, _, r1 = ref.fetch()
        o2, s2, _, r2 = env.fetch()
        assert (s1 == 0).all() and np.array_equal(o1, o2) and np.array_equal(r1, r2)
    info = eng.last_launch_info()
    assert eng.plan_stats()["last_kernel"] == "planned_block" and info["threads_per_instance"] == 8 and info["block"] == 64, info
    assert eng.redo_launch_count == n0
    # every second instance forced to give up: exactly one re-solve per step, and the results of an undisturbed run
    eng.set_debug(2, True)
    for k in range(4):
        ref.step_device(); env.step_device()
        o1, s1, i1, r1 = ref.fetch()
        o2, s2, i2, r2 = env.fetch()
        assert eng.redo_launch_count == n0 + k + 1
        assert (s1 == 0).all() and (s2 == 0).all()            # the row of a re-solved instance is NOT advanced twice
        _compare(gm, o2, o1, s1 == 0)
        assert np.allclose(r1, r2, rtol=1e-5, atol=1e-6)
        assert np.array_equal(o1[1::2], o2[1::2])              # untouched instances: same kernel, bit-equal
    # and back to no failures: no launch
    eng.set_debug(0, True)
    env.step_device()
    assert (env.fetch()[1] == 0).all()
    assert eng.redo_launch_count == n0 + 4
    ref.close(); env.close()


def test_concurrent_group_streams_resolve_their_own_failures(cuda_required):
    """Groups run on streams of their own, concurrently: one stream's armed re-solve must never stand in for another's."""
    from grid2op_b200.rollout import BatchedDoNothing
    gm, chron = _case14()
    ref = BatchedDoNothing(gm, chron, B)
    env = BatchedDoNothing(gm, chron, B)
    for x in (ref, env):
        x.engine.set_kernel_policy(2)
        x.host_groups(2)
    eng = env.engine
    n0 = eng.redo_launch_count
    # (forced failures are chosen at launch time: group 0 with them, group 1 without; then both with different ones)
    for k, mods in enumerate([(2, 0), (0, 3), (2, 3)]):
        for g in (0, 1):
            ref.group_launch(g)
            eng.set_debug(mods[g], True)
            env.group_launch(g)
        for g in (0, 1):
            o1, s1 = ref.group_wait(g)
            o2, s2 = env.group_wait(g)
            assert (s1 == 0).all() and (s2 == 0).all(), (k, g)
            _compare(gm, o2.copy(), o1.copy(), s1 == 0)
            if mods[g] == 0:
                assert np.array_equal(o1, o2), (k, g)
        assert eng.plan_stats()["last_kernel"].startswith("planned")
    assert eng.redo_launch_count == n0 + 4
    ref.close(); env.close()
