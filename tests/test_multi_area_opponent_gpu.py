"""BatchedEnv's GeometricOpponentMultiArea on the GPU.

* Twin environments, ``step`` (the numpy path) against ``step_tensors`` (csrc/b200pf_opp.cuh inside the apply and reset launches),
  fed the same actions, alternating the two paths: after every step and every masked reset they must be bit-equal in environment
  state, the whole opponent state (budget and its dtype flag, counters, previous_fails, every area's 624 MT19937 words and position,
  schedule, counters, _next_attack_time and remembered line), each area's attacked line and the duration, rho, status and plan
  counters.  l2rpn_idf_2023 at batch 1024 (its three areas) and case14 at batch 4096 (six lines in three areas); protections off
  and on.
* tests/test_multi_area_opponent_cpu.py's comparison against unmodified l2rpn_idf_2023 environments, the CUDA engine on both sides.
* With the multi-area opponent on, a ``step_tensors`` step still moves 32 B device-to-host and nothing host-to-device, and a device
  reset waits on the host as often as without it.
"""
import numpy as np
import pytest

from conftest import env_grid

CASE14_AREAS = [["1_3_3", "1_4_4"], ["3_6_15", "9_10_12"], ["11_12_13", "12_13_14"]]     # tests/test_opponent_gpu.py's lines
SHORT = dict(attack_every_xxx_hour=1.5, average_attack_duration_hour=0.75, minimum_attack_duration_hour=0.25)
MULTI = dict(attack_duration=7, attack_cooldown=1, budget_per_ts=0.5, init_budget=3.0)


def _idf_areas():
    import ast
    import os
    src = open(os.path.join(os.path.dirname(env_grid("l2rpn_idf_2023")), "config.py")).read()
    tree = ast.parse(src)
    for node in tree.body:
        if isinstance(node, ast.Assign) and getattr(node.targets[0], "id", None) == "lines_attacked":
            return ast.literal_eval(node.value)
    raise AssertionError("lines_attacked not found")


def _multi_compare(k, ref, tst, info_a, info_b, tensor_mode):
    a = ref.opponent_state()
    if tensor_mode:
        b = tst.engine.opp_get_state()
        b.update(tst.engine.opp_multi_get_state())
    else:
        b = tst.opponent_state()
    assert set(a) == set(b) and "multi_ctr" in a, (set(a), set(b))
    for key in a:
        bad = np.argwhere(np.asarray(a[key]) != np.asarray(b[key]))[:5]
        assert not len(bad), (k, key, bad)
    assert not a["multi_ctr"][:, :, 3].any(), k                         # no schedule passed the cap
    if info_a is not None:
        cv = lambda x: x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)      # noqa: E731
        for key in ("opponent_attack_line", "opponent_attack_duration"):
            assert np.array_equal(info_a[key], cv(info_b[key])), (k, key)
        assert info_a["opponent_attack_line"].shape == (ref.batch, a["multi_ctr"].shape[1])
        if tensor_mode:
            assert np.array_equal(a["budget"].view(np.int64), tst._dev["opp_budget"].cpu().numpy().view(np.int64)), k


def _run(ref, tst, steps, seed, reset_every=0, alternate=0):
    import torch
    from test_env_tensor_gpu import _actions, _compare
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(seed)
    t = lambda x: torch.as_tensor(np.asarray(x), device=dev)                     # noqa: E731
    seen = dict(attacks=0, multi=0, resets=0, consumed=0, fails=0)
    rho, _, info = ref.reset_step()
    out_b = tst.step_tensors(from_reset=True)
    _compare(-1, ref, (rho, info), tst, (out_b[0], out_b[2]), True)
    for k in range(steps):
        tensor_mode = not alternate or (k // alternate) % 2 == 0
        if reset_every and k and k % reset_every == 0:
            mask = ref.done.copy()
            mask[k % ref.batch::97] = True                       # (live instances too: new schedules, the streams go on)
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
            _multi_compare(k, ref, tst, None, None, tensor_mode)
        sub, bus, line, lst = _actions(ref, rng)
        rho, _, info = ref.step(sub, bus, line, lst)
        if tensor_mode:
            rb, _, ib = tst.step_tensors(t(sub), t(bus), t(line), t(lst))
        else:
            rb, _, ib = tst.step(sub, bus, line, lst)
        _compare(k, ref, (rho, info), tst, (rb, ib), tensor_mode)
        assert ref.engine.plan_counters() == tst.engine.plan_counters(), k
        _multi_compare(k, ref, tst, info, ib, tensor_mode)
        st = ref._opp.get_state()
        n_hit = (info["opponent_attack_line"] >= 0).sum(axis=1)
        seen["attacks"] += int(n_hit.sum())
        seen["multi"] += int((n_hit >= 2).sum())
        seen["consumed"] += int(st["multi_ctr"][:, :, 1].sum())
        seen["fails"] += int(st["multi_fails"].sum())
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("protections", [False, True])
def test_twins_idf_multi_area_opponent_batch1024(cuda_required, protections):
    if env_grid("l2rpn_idf_2023") is None:
        pytest.skip("reference data not available")
    from test_env_tensor_gpu import _pair
    from grid2op_b200.opponent import opponent_seed
    ref, tst = _pair("l2rpn_idf_2023", 1024, protections, th_scale=1.1, seed=5, observe=False)
    seeds = [opponent_seed(s) for s in range(1024)]
    ref.reset_step(); tst.step(from_reset=True)
    for e in (ref, tst):
        e.enable_opponent("GeometricOpponentMultiArea", _idf_areas(), seeds=seeds, **MULTI, **SHORT)
    seen = _run(ref, tst, 30, seed=61 + protections, reset_every=7, alternate=10)
    assert seen["attacks"] and seen["multi"] and seen["resets"] and seen["consumed"] and seen["fails"], seen
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("protections", [False, True])
def test_twins_case14_multi_area_opponent_batch4096(cuda_required, protections):
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    from test_env_tensor_gpu import _pair
    from grid2op_b200.opponent import opponent_seed
    ref, tst = _pair("l2rpn_case14_sandbox", 4096, protections, observe=False, **({"th_scale": 1.05} if protections else {"thermal": 150.0}))
    seeds = [opponent_seed(s) for s in range(4096)]
    ref.reset_step(); tst.step(from_reset=True)
    for e in (ref, tst):
        e.enable_opponent("GeometricOpponentMultiArea", CASE14_AREAS, seeds=seeds, **MULTI, **SHORT)
    seen = _run(ref, tst, 40, seed=71 + protections, reset_every=6, alternate=15)
    assert seen["attacks"] and seen["multi"] and seen["resets"] and seen["consumed"] and seen["fails"], seen
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
def test_multi_area_opponent_vs_reference_env_cuda_engine(cuda_required):
    """tests/test_multi_area_opponent_cpu.py's comparison against unmodified environments, the CUDA engine on both sides"""
    if env_grid("l2rpn_idf_2023") is None:
        pytest.skip("reference data not available")
    from grid2op_b200.backend import B200Backend
    from test_multi_area_opponent_cpu import run_multi_vs_reference
    saw = run_multi_vs_reference(150, (0, 3, 5), 0, engine_factory=lambda gm: None, emu=False, backend_class=B200Backend,
                                 schedule_steps=80)
    assert saw["attack_steps"] > 0 and saw["multi_line"] > 0 and saw["refused_budget"] > 0, saw


@pytest.mark.gpu
def test_multi_area_opponent_no_extra_traffic(cuda_required):
    """with the multi-area opponent on, a step moves the bytes it moved without an opponent, and a device reset waits as often.
    With no budget every combined attack is refused (the schedules, draws and decisions still run), so no topology changes and no
    changed row is copied back: the bytes are the opponent's alone"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    import torch
    from test_env_tensor_gpu import _pair
    from grid2op_b200.opponent import opponent_seed
    ref, tst = _pair("l2rpn_case14_sandbox", 256, False, thermal=150.0, observe=False)
    for e in (ref, tst):
        e.step_tensors(from_reset=True)
    tst.enable_opponent("GeometricOpponentMultiArea", CASE14_AREAS, seeds=[opponent_seed(s) for s in range(256)], attack_duration=7,
                        attack_cooldown=1, budget_per_ts=0.0, init_budget=0.0, **SHORT)
    tst.step_tensors()                                       # (the first step pushes the host state)
    for e in (ref, tst):
        e.step_tensors()
    torch.cuda.synchronize()
    s0 = tst.engine.env_stats()
    _, _, info = tst.step_tensors()
    torch.cuda.synchronize()
    s1 = tst.engine.env_stats()
    assert tuple(info["opponent_attack_line"].shape) == (256, 3) and bool((info["opponent_attack_line"] == -1).all())
    assert s1["d2h_bytes"] - s0["d2h_bytes"] == 32 and s1["h2d_bytes"] == s0["h2d_bytes"]
    assert tst.engine.opp_multi_get_state()["multi_ctr"][:, :, 1].sum() > 0       # (attacks came due and were refused)
    mask = torch.zeros(256, dtype=torch.bool, device="cuda:0")
    mask[::3] = True
    waits = []
    for e in (ref, tst):
        w0 = e.engine.env_stats()["host_waits"]
        e.reset_instances(mask)
        torch.cuda.synchronize()
        waits.append(e.engine.env_stats()["host_waits"] - w0)
    assert waits[0] == waits[1], waits
    assert tst.engine.opp_multi_get_state()["multi_ctr"][::3, :, 1].sum() == 0      # the reset instances start new schedules
    del mask                              # (the resets recorded it on the engines' streams: free it while those streams exist)
    torch.cuda.synchronize()
    for e in (ref, tst):
        e.close()
