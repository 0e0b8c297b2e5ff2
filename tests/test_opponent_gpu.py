"""BatchedEnv's line-attack opponents on the GPU.

* Twin environments, ``step`` (the numpy path) against ``step_tensors`` (csrc/b200pf_opp.cuh inside the apply and reset launches),
  fed the same actions with the opponent on: after every step and every reset they must be bit-equal in environment state, opponent
  state (budget, its dtype flag, counters, the 624 MT19937 words and position), attacked line and duration, rho, status and plan
  counters.  l2rpn_neurips_2020_track1 at batch 1000 with its WeightedRandomOpponent, case14 at batch 4096 with a
  RandomLineOpponent on the lines rte_case14_opponent lists and masked resets; protections off and on.
* The comparison of tests/test_opponent_cpu.py against unmodified grid2op environments, with the CUDA engine on both sides.
"""
import numpy as np
import pytest

from conftest import env_grid

CASE14_LINES = ["1_3_3", "1_4_4", "3_6_15", "9_10_12", "11_12_13", "12_13_14"]            # rte_case14_opponent's config
TRACK1_LINES = ["62_58_180", "62_63_160", "48_50_136", "48_53_141", "41_48_131", "39_41_121", "43_44_125", "44_45_126", "34_35_110",
                "54_58_154"]
TRACK1_NORM = [0.45, 0.45, 0.6, 0.35, 0.3, 0.2, 0.55, 0.3, 0.45, 0.55]


def _opp_compare(k, ref, tst, info_a, info_b, tensor_mode):
    a = ref.opponent_state()
    b = tst.engine.opp_get_state() if tensor_mode else tst.opponent_state()
    for key in a:
        bad = np.argwhere(np.asarray(a[key]) != np.asarray(b[key]))[:5]
        assert not len(bad), (k, key, bad)
    if info_a is not None:
        cv = lambda x: x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)      # noqa: E731
        for key in ("opponent_attack_line", "opponent_attack_duration"):
            assert np.array_equal(info_a[key], cv(info_b[key])), (k, key)
        if tensor_mode:
            assert np.array_equal(a["budget"].view(np.int64), tst._dev["opp_budget"].cpu().numpy().view(np.int64)), k


def _run(ref, tst, steps, seed, reset_every=0, alternate=0):
    import torch
    from test_env_tensor_gpu import _actions, _compare
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(seed)
    t = lambda x: torch.as_tensor(np.asarray(x), device=dev)                     # noqa: E731
    seen = dict(attacks=0, resets=0, illegal=0, game_over=0)
    rho, _, info = ref.reset_step()
    out_b = tst.step_tensors(from_reset=True)
    _compare(-1, ref, (rho, info), tst, (out_b[0], out_b[2]), True)
    for k in range(steps):
        tensor_mode = not alternate or (k // alternate) % 2 == 0
        if reset_every and k and k % reset_every == 0:
            mask = ref.done.copy()
            mask[k % ref.batch::97] = True                       # (live instances too: their opponent restarts, the stream goes on)
            idx = np.flatnonzero(mask)
            rows = (idx * 7 + k) % ref.chron.shape[1]
            ref.reset_instances(idx, rows)
            if tensor_mode:
                r = np.zeros(ref.batch, np.int64); r[idx] = rows
                tst.reset_instances(t(mask), t(r))
            else:
                tst.reset_instances(idx, rows)
            seen["resets"] += len(idx)
            assert ref.engine.plan_counters() == tst.engine.plan_counters(), k
            _opp_compare(k, ref, tst, None, None, tensor_mode)
        sub, bus, line, lst = _actions(ref, rng)
        rho, _, info = ref.step(sub, bus, line, lst)
        if tensor_mode:
            rb, _, ib = tst.step_tensors(t(sub), t(bus), t(line), t(lst))
        else:
            rb, _, ib = tst.step(sub, bus, line, lst)
        _compare(k, ref, (rho, info), tst, (rb, ib), tensor_mode)
        assert ref.engine.plan_counters() == tst.engine.plan_counters(), k
        _opp_compare(k, ref, tst, info, ib, tensor_mode)
        seen["attacks"] += int((info["opponent_attack_line"] >= 0).sum())
        seen["illegal"] += int(np.asarray(info["is_illegal"]).sum())
        seen["game_over"] += int(info["newly_done"].sum())
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("protections", [False, True])
def test_twins_case14_random_line_opponent_batch4096(cuda_required, protections):
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    from test_env_tensor_gpu import _pair
    from grid2op_b200.opponent import opponent_seed
    ref, tst = _pair("l2rpn_case14_sandbox", 4096, protections, observe=False, **({"th_scale": 1.05} if protections else {"thermal": 150.0}))
    seeds = [opponent_seed(s) for s in range(4096)]
    # enable_opponent needs a first step; the twins then start from the same state (_run's reset_step / step_tensors is the next one)
    ref.reset_step(); tst.step(from_reset=True)
    for e in (ref, tst):
        e.enable_opponent("RandomLineOpponent", CASE14_LINES, attack_duration=4, attack_cooldown=6, budget_per_ts=0.5,
                          init_budget=1.0, seeds=seeds)
    seen = _run(ref, tst, 40, seed=31 + protections, reset_every=6, alternate=15)
    assert seen["attacks"] and seen["resets"] and seen["illegal"], seen
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("protections", [False, True])
def test_twins_track1_weighted_random_opponent_batch1000(cuda_required, protections):
    if env_grid("l2rpn_neurips_2020_track1") is None:
        pytest.skip("reference data not available")
    from test_env_tensor_gpu import _pair
    from grid2op_b200.opponent import opponent_seed
    ref, tst = _pair("l2rpn_neurips_2020_track1", 1000, protections, th_scale=1.1, events=True, cd=2, n_scen=2, seed=3)
    seeds = [opponent_seed(s) for s in range(1000)]
    ref.reset_step(); tst.step(from_reset=True)
    for e in (ref, tst):
        e.enable_opponent("WeightedRandomOpponent", TRACK1_LINES, attack_duration=6, attack_cooldown=12, budget_per_ts=0.16667,
                          init_budget=8.0, attack_period=8, rho_normalization=TRACK1_NORM, seeds=seeds)
    seen = _run(ref, tst, 40, seed=21 + protections)
    assert seen["attacks"] and seen["illegal"], seen
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
def test_opponent_vs_reference_env_cuda_engine(cuda_required):
    """tests/test_opponent_cpu.py's comparison against unmodified environments, the CUDA engine on both sides"""
    if env_grid("l2rpn_neurips_2020_track1") is None:
        pytest.skip("reference data not available")
    from grid2op_b200.backend import B200Backend
    from test_opponent_cpu import _track1_kw, run_opponent_vs_reference
    saw = run_opponent_vs_reference("l2rpn_neurips_2020_track1", 150, _track1_kw, seeds=(0, 3, 11), engine_factory=lambda gm: None,
                                    emu=False, backend_class=B200Backend)
    assert saw["refused"] > 0 and saw["whole"] > 0 and saw["illegal_by_attack"] > 0, saw


@pytest.mark.gpu
def test_no_opponent_no_extra_work(cuda_required):
    """without enable_opponent the info keys and the bytes a step moves are what they were"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    import torch
    from test_env_tensor_gpu import _pair
    ref, tst = _pair("l2rpn_case14_sandbox", 256, False, thermal=150.0, observe=False)
    tst.step_tensors(from_reset=True)
    s0 = tst.engine.env_stats()
    _, _, info = tst.step_tensors()
    torch.cuda.synchronize()
    s1 = tst.engine.env_stats()
    assert "opponent_attack_line" not in info and s1["d2h_bytes"] - s0["d2h_bytes"] == 32 and s1["h2d_bytes"] == s0["h2d_bytes"]
    for e in (ref, tst):
        e.close()
