"""BatchedEnv's alarms on the GPU.

* Twin environments, ``step`` (the numpy path, grid2op_b200/alarm.py) against ``step_tensors`` (csrc/b200pf_alarm.cuh inside the
  post and reset launches), fed the same actions and random alarms: after every step and every masked reset the whole alarm state,
  the float64 AlarmReward, is_alarm_illegal, the observation vectors (with the five alarm attributes) and RedispReward are
  bit-equal.  l2rpn_icaps_2021 at batch 1024 with its GeometricOpponent, protections off and on, and case14 at batch 4096 with a
  synthetic three-zone "fixed" alerts_info.json, the two paths alternating.
* With alarms on, a ``step_tensors`` step moves nothing host-to-device and the same device-to-host bytes and host waits as without.
* A ``raise_alarm`` of the wrong shape, dtype or device raises ValueError and changes nothing.
* tests/test_alarms_cpu.py's comparisons with unmodified l2rpn_icaps_2021 environments, the CUDA engine on both sides.
"""
import json

import numpy as np
import pytest

from conftest import env_grid

SHORT = dict(attack_every_xxx_hour=1.5, average_attack_duration_hour=0.75, minimum_attack_duration_hour=0.25)
GEO = dict(attack_duration=7, attack_cooldown=2, budget_per_ts=0.3, init_budget=4.0)
ICAPS_LINES = ["62_58_180", "62_63_160", "48_50_136", "48_53_141", "41_48_131", "39_41_121", "43_44_125", "44_45_126", "34_35_110",
               "54_58_154"]
CASE14_LINES = ["1_3_3", "1_4_4", "3_6_15", "9_10_12", "11_12_13", "12_13_14"]
# a fast refill, so that refusals, the cap and successful alarms all happen within the run
BUDGET = dict(max_budget=3.0, budget_per_ts=0.1, alarm_cost=1.0, init_budget=2.0)
# (name, batch, opponent lines, pair options)
CONFIGS = {
    "icaps": ("l2rpn_icaps_2021", 1024, ICAPS_LINES, dict(th_scale=1.1, seed=5)),
    "case14_zones": ("l2rpn_case14_sandbox", 4096, CASE14_LINES, dict(thermal=150.0)),
}


def _zones(cfg, tmp_path):
    from test_alarms_cpu import three_zones
    from grid2op_b200.alarm import load_alarm_zones
    from grid2op_b200.gridmodel import GridModel
    import os
    grid = env_grid(CONFIGS[cfg][0])
    gm = GridModel(grid)
    if cfg == "icaps":
        return load_alarm_zones(os.path.dirname(grid), gm)
    (tmp_path / "alerts_info.json").write_text(json.dumps(three_zones(gm)))
    return load_alarm_zones(str(tmp_path), gm)


def _pair_with_alarms(protections, tmp_path, alarms=True, B=None, cfg="icaps"):
    from test_env_tensor_gpu import _load, _pair
    name, B0, _, kw = CONFIGS[cfg]
    ref, tst = _pair(name, B or B0, protections, observe=False, **kw)
    _, _, env_dir, folders = _load(name, None)
    zones = _zones(cfg, tmp_path)
    for e in (ref, tst):
        if alarms:
            e.enable_alarms(zones, **BUDGET)
        e.enable_observation(env_dir, scenarios=folders)
    return ref, tst


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _compare_alarms(k, ref, tst, ia=None, ib=None):
    a, b = ref.alarm_state(), tst.engine.alarm_get_state() if tst._authority == "device" else tst.alarm_state()
    for key in a:
        bad = np.argwhere(np.asarray(a[key]).view(np.uint8) != np.asarray(b[key]).view(np.uint8))[:5]
        assert not len(bad), (k, key, bad)
    if ia is not None:
        ra, rb = ia["rewards"]["alarm"], _np(ib["rewards"]["alarm"])
        assert rb.dtype == np.float64 and np.array_equal(ra.view(np.int64), rb.view(np.int64)), k
        assert np.array_equal(ia["is_alarm_illegal"], _np(ib["is_alarm_illegal"]).astype(bool)), k


def _observe_equal(k, ref, tst):
    oa, ra = ref.observe()
    ob, rb = tst.observe()
    assert np.array_equal(_np(oa).view(np.int32), _np(ob).view(np.int32)), k
    assert np.array_equal(_np(ra).view(np.int32), _np(rb).view(np.int32)), k


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,protections", [("icaps", False), ("icaps", True), ("case14_zones", False)])
def test_twins_alarms(cuda_required, tmp_path, cfg, protections):
    if env_grid(CONFIGS[cfg][0]) is None:
        pytest.skip("reference data not available")
    import torch
    from test_env_tensor_gpu import _actions
    from grid2op_b200.opponent import opponent_seed
    ref, tst = _pair_with_alarms(protections, tmp_path, cfg=cfg)
    dev = torch.device("cuda", 0)
    t = lambda x: torch.as_tensor(np.asarray(x), device=dev)                     # noqa: E731
    n = ref._alarms.n
    ref.reset_step(); tst.step_tensors(from_reset=True)
    _observe_equal(-1, ref, tst)
    seeds = [opponent_seed(s) for s in range(ref.batch)]
    for e in (ref, tst):
        e.enable_opponent("GeometricOpponent", CONFIGS[cfg][2], seeds=seeds, **GEO, **SHORT)
    rng = np.random.default_rng(91 + protections)
    seen = dict(ok=0, refused=0, rewards=0, scored=0, resets=0)
    # icaps with the protections on: every 50th instance raises a "west" alarm at step 9 and disconnects CUT at step 21, a game
    # over with a first-round trip 12 steps after the alarm (tests/test_alarms_cpu.py), so that the scoring loop runs on the device
    timed = np.arange(1, ref.batch, 50) if cfg == "icaps" and protections else np.zeros(0, np.int64)
    if len(timed):
        from test_alarms_cpu import CUT
        zones = ref._alarms.names
        west, cut = zones.index("west"), [str(x) for x in ref.gm.name_line].index(CUT)
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
            _compare_alarms(k, ref, tst)
            _observe_equal(k, ref, tst)
        up = rng.random((ref.batch, n)) < np.where(rng.random((ref.batch, 1)) < 0.3, 0.5, 0.0)
        sub, bus, line, lst = _actions(ref, rng)
        if len(timed) and k == 8:
            up[timed] = False
            up[timed, west] = True
        if len(timed) and k == 20:
            sub[timed], line[timed], lst[timed] = -1, cut, -1
        _, _, ia = ref.step(sub, bus, line, lst, raise_alarm=up)
        if tensor_mode:
            _, _, ib = tst.step_tensors(t(sub), t(bus), t(line), t(lst), raise_alarm=t(up))
        else:
            _, _, ib = tst.step(sub, bus, line, lst, raise_alarm=up)
        _compare_alarms(k, ref, tst, ia, ib)
        _observe_equal(k, ref, tst)
        seen["refused"] += int(ia["is_alarm_illegal"].sum())
        seen["ok"] += int((ref._alarms.s["time_last_ok"] == ref.current_step).sum())
        seen["rewards"] += int((ia["rewards"]["alarm"] != 0).sum())
        seen["scored"] += int((ia["rewards"]["alarm"] > 0).sum())
    assert seen["ok"] and seen["refused"] and seen["rewards"] and seen["resets"], seen
    assert seen["scored"] or not len(timed), seen
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
def test_alarms_add_no_host_traffic(cuda_required, tmp_path):
    if env_grid("l2rpn_icaps_2021") is None:
        pytest.skip("reference data not available")
    import torch
    from grid2op_b200.opponent import opponent_seed
    dev = torch.device("cuda", 0)
    per_step = []
    for alarms in (False, True):
        env, _ = _pair_with_alarms(False, tmp_path, alarms=alarms, B=256)
        env.step_tensors(from_reset=True)
        env.enable_opponent("GeometricOpponent", ICAPS_LINES, seeds=[opponent_seed(s) for s in range(env.batch)], **GEO, **SHORT)
        up = torch.ones((env.batch, 3), dtype=torch.bool, device=dev) if alarms else None
        env.step_tensors(raise_alarm=up)                  # (the first step pushes the host state)
        s0 = env.engine.env_stats()
        for _ in range(5):
            env.step_tensors(raise_alarm=up)
            env.observe()
        s1 = env.engine.env_stats()
        per_step.append(tuple(s1[k] - s0[k] for k in ("h2d_bytes", "d2h_bytes", "host_waits")))
        env.close()
    assert per_step[0][0] == per_step[1][0] == 0, per_step
    assert per_step[0] == per_step[1], per_step


@pytest.mark.gpu
def test_step_tensors_rejects_bad_raise_alarm(cuda_required, tmp_path):
    """a raise_alarm of the wrong shape, dtype or device raises ValueError and changes nothing"""
    if env_grid("l2rpn_icaps_2021") is None:
        pytest.skip("reference data not available")
    import torch
    _, env = _pair_with_alarms(False, tmp_path, B=64)
    env.step_tensors(from_reset=True)
    dev = torch.device("cuda", 0)
    up = torch.ones((64, 3), dtype=torch.bool, device=dev)
    env.step_tensors(raise_alarm=up)
    before, n0 = env.engine.alarm_get_state(), env.n_steps
    for bad in (torch.ones((64, 2), dtype=torch.bool, device=dev), torch.ones((64, 3), dtype=torch.int32, device=dev),
                torch.ones((64, 3), dtype=torch.bool), np.ones((64, 3), bool)):
        with pytest.raises(ValueError):
            env.step_tensors(raise_alarm=bad)
    after = env.engine.alarm_get_state()
    assert env.n_steps == n0 and all(np.array_equal(before[k], after[k]) for k in before)
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("protections", [False, True])
def test_alarms_vs_reference_env_cuda_engine(cuda_required, protections):
    """tests/test_alarms_cpu.py's comparisons with unmodified environments, the CUDA engine on both sides"""
    if env_grid("l2rpn_icaps_2021") is None:
        pytest.skip("reference data not available")
    from grid2op_b200.backend import B200Backend
    from test_alarms_cpu import SAW_ALL, SAW_PROT, SEEDS, run_alarms_vs_reference
    saw = run_alarms_vs_reference(150, SEEDS, protections, engine_factory=lambda gm: None, backend_class=B200Backend, emu=False)
    assert all(saw[k] > 0 for k in (SAW_PROT if protections else SAW_ALL)), saw
