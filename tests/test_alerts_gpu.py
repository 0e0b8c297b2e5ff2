"""BatchedEnv's line alerts on the GPU.

* Twin environments, ``step`` (the numpy path, grid2op_b200/alert.py) against ``step_tensors`` (csrc/b200pf_alert.cuh inside the
  post and reset launches), fed the same actions and random alert vectors: after every step and every masked reset the whole alert
  state, the float64 AlertReward, the observation vectors (with the seven alert attributes) and RedispReward are bit-equal.
  l2rpn_idf_2023 at batch 1024 with its multi-area opponent, protections off and on, and case14 at batch 4096 with a
  RandomLineOpponent (one attacked line per instance), the two paths alternating.
* With alerts on, a ``step_tensors`` step moves nothing host-to-device and the same device-to-host bytes and host waits as without.
* A ``raise_alert`` of the wrong shape, dtype or device raises ValueError and changes nothing.
* tests/test_alerts_cpu.py's comparisons with unmodified environments (l2rpn_idf_2023 with timed game overs, and the copy of
  rte_case14_opponent with ``alerts_info.json``), the CUDA engine on both sides.
"""
import numpy as np
import pytest

from conftest import env_grid

SHORT = dict(attack_every_xxx_hour=1.5, average_attack_duration_hour=0.75, minimum_attack_duration_hour=0.25)
MULTI = dict(attack_duration=7, attack_cooldown=1, budget_per_ts=0.5, init_budget=3.0)


CASE14_LINES = ["1_3_3", "1_4_4", "3_6_15", "9_10_12", "11_12_13", "12_13_14"]     # rte_case14_opponent's lines
# (name, batch, opponent kind, its lines, its constants)
CONFIGS = {
    "idf_multi_area": ("l2rpn_idf_2023", 1024, "GeometricOpponentMultiArea", None, dict(MULTI, **SHORT)),
    "case14_random_line": ("l2rpn_case14_sandbox", 4096, "RandomLineOpponent", CASE14_LINES,
                           dict(attack_duration=6, attack_cooldown=4, budget_per_ts=0.5, init_budget=4.0)),
}


def _lines(cfg):
    from test_multi_area_opponent_gpu import _idf_areas
    return CONFIGS[cfg][3] if CONFIGS[cfg][3] is not None else _idf_areas()


def _pair_with_alerts(protections, alerts=True, B=None, cfg="idf_multi_area"):
    from test_env_tensor_gpu import _load, _pair
    name = CONFIGS[cfg][0]
    ref, tst = _pair(name, B or CONFIGS[cfg][1], protections, th_scale=1.1, seed=5, observe=False)
    _, _, env_dir, folders = _load(name, None)
    for e in (ref, tst):
        if alerts:
            e.enable_alerts(_lines(cfg))
        e.enable_observation(env_dir, scenarios=folders)
    return ref, tst


def _compare_alerts(k, ref, tst, ra, rb):
    a, b = ref.alert_state(), tst.engine.alert_get_state() if tst._authority == "device" else tst.alert_state()
    for key in a:
        bad = np.argwhere(np.asarray(a[key]) != np.asarray(b[key]))[:5]
        assert not len(bad), (k, key, bad)
    if ra is not None:
        rb = rb.cpu().numpy() if hasattr(rb, "cpu") else np.asarray(rb)
        assert rb.dtype == np.float64 and np.array_equal(ra.view(np.int64), rb.view(np.int64)), k


def _observe_equal(k, ref, tst):
    oa, ra = ref.observe()
    ob, rb = tst.observe()
    assert np.array_equal(oa.cpu().numpy().view(np.int32), ob.cpu().numpy().view(np.int32)), k
    assert np.array_equal(ra.cpu().numpy().view(np.int32), rb.cpu().numpy().view(np.int32)), k


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,protections", [("idf_multi_area", False), ("idf_multi_area", True), ("case14_random_line", False)])
def test_twins_alerts(cuda_required, cfg, protections):
    if env_grid(CONFIGS[cfg][0]) is None:
        pytest.skip("reference data not available")
    import torch
    from test_env_tensor_gpu import _actions
    from grid2op_b200.opponent import opponent_seed
    ref, tst = _pair_with_alerts(protections, cfg=cfg)
    dev = torch.device("cuda", 0)
    t = lambda x: torch.as_tensor(np.asarray(x), device=dev)                     # noqa: E731
    n = ref._alerts.n
    ref.reset_step(); tst.step_tensors(from_reset=True)
    _observe_equal(-1, ref, tst)
    seeds = [opponent_seed(s) for s in range(ref.batch)]
    for e in (ref, tst):
        e.enable_opponent(CONFIGS[cfg][2], _lines(cfg), seeds=seeds, **CONFIGS[cfg][4])
    rng = np.random.default_rng(71 + protections)
    runs = np.zeros((ref.batch, n), bool)
    seen = dict(rewards=0, resets=0, nonzero_used=0)
    for k in range(40):
        tensor_mode = (k // 10) % 2 == 0
        if k and k % 7 == 0:
            mask = ref.done.copy()
            mask[k % ref.batch::97] = True
            idx = np.flatnonzero(mask)
            rows = (idx * 7 + k) % ref.chron.shape[1]
            ref.reset_instances(idx, rows)
            if tensor_mode:
                r = np.zeros(ref.batch, np.int64); r[idx] = rows
                tst.reset_instances(t(mask), t(r))
            else:
                tst.reset_instances(idx, rows)
            seen["resets"] += len(idx)
            _compare_alerts(k, ref, tst, None, None)
        runs ^= rng.random((ref.batch, n)) < 0.15
        sub, bus, line, lst = _actions(ref, rng)
        _, _, ia = ref.step(sub, bus, line, lst, raise_alert=runs)
        if tensor_mode:
            _, _, ib = tst.step_tensors(t(sub), t(bus), t(line), t(lst), raise_alert=t(runs))
        else:
            _, _, ib = tst.step(sub, bus, line, lst, raise_alert=runs)
        _compare_alerts(k, ref, tst, ia["rewards"]["alert"], ib["rewards"]["alert"])
        _observe_equal(k, ref, tst)
        seen["rewards"] += int((ia["rewards"]["alert"] != 0).sum())
        seen["nonzero_used"] += int((ref._alerts.s["was_used"] != 0).any(axis=1).sum())
    assert seen["rewards"] and seen["resets"] and seen["nonzero_used"], seen
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
def test_alerts_add_no_host_traffic(cuda_required):
    if env_grid("l2rpn_idf_2023") is None:
        pytest.skip("reference data not available")
    import torch
    from test_multi_area_opponent_gpu import _idf_areas
    from grid2op_b200.opponent import opponent_seed
    dev = torch.device("cuda", 0)
    per_step = []
    for alerts in (False, True):
        env, _ = _pair_with_alerts(False, alerts=alerts, B=256)
        env.step_tensors(from_reset=True)
        env.enable_opponent("GeometricOpponentMultiArea", _idf_areas(), seeds=[opponent_seed(s) for s in range(env.batch)], **MULTI, **SHORT)
        up = torch.ones((env.batch, 22), dtype=torch.bool, device=dev) if alerts else None
        env.step_tensors(raise_alert=up)                  # (the first step pushes the host state)
        s0 = env.engine.env_stats()
        for _ in range(5):
            env.step_tensors(raise_alert=up)
            env.observe()
        s1 = env.engine.env_stats()
        per_step.append(tuple(s1[k] - s0[k] for k in ("h2d_bytes", "d2h_bytes", "host_waits")))
        env.close()
    assert per_step[0][0] == per_step[1][0] == 0, per_step
    assert per_step[0] == per_step[1], per_step


@pytest.mark.gpu
def test_step_tensors_rejects_bad_raise_alert(cuda_required):
    """a raise_alert of the wrong shape, dtype or device raises ValueError and changes nothing"""
    if env_grid("l2rpn_idf_2023") is None:
        pytest.skip("reference data not available")
    import torch
    _, env = _pair_with_alerts(False, B=64)
    env.step_tensors(from_reset=True)
    dev = torch.device("cuda", 0)
    up = torch.ones((64, 22), dtype=torch.bool, device=dev)
    env.step_tensors(raise_alert=up)
    before, n0 = env.engine.alert_get_state(), env.n_steps
    for bad in (torch.ones((64, 21), dtype=torch.bool, device=dev), torch.ones((64, 22), dtype=torch.int32, device=dev),
                torch.ones((64, 22), dtype=torch.bool)):
        with pytest.raises(ValueError):
            env.step_tensors(raise_alert=bad)
    after = env.engine.alert_get_state()
    assert env.n_steps == n0 and all(np.array_equal(before[k], after[k]) for k in before)
    env.close()


@pytest.mark.gpu
def test_alerts_vs_reference_env_cuda_engine(cuda_required):
    """tests/test_alerts_cpu.py's comparisons with unmodified environments, the CUDA engine on both sides"""
    if env_grid("l2rpn_idf_2023") is None:
        pytest.skip("reference data not available")
    from grid2op_b200.backend import B200Backend
    from test_alerts_cpu import KILLS, SAW_ALL, run_alerts_vs_reference
    saw = run_alerts_vs_reference(150, (0, 3, 5, 7, 9, 11, 13, 17), kill=KILLS, engine_factory=lambda gm: None,
                                  backend_class=B200Backend, emu=False)
    assert all(saw[k] > 0 for k in SAW_ALL), saw


@pytest.mark.gpu
def test_alerts_single_line_opponent_vs_reference_env_cuda_engine(cuda_required, tmp_path):
    if env_grid("rte_case14_opponent") is None:
        pytest.skip("reference data not available")
    from grid2op_b200.backend import B200Backend
    from test_alerts_cpu import run_case14_alerts_vs_reference
    saw = run_case14_alerts_vs_reference(tmp_path, 80, (1, 2, 4, 8), engine_factory=lambda gm: None, backend_class=B200Backend)
    assert all(saw[k] > 0 for k in saw), saw
