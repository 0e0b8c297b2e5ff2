"""The device environment's state handed to the host and back, layer by layer (environment, line-attack opponent, GeometricOpponent,
GeometricOpponentMultiArea, line alerts, alarms), a few ``step_tensors`` steps into small-batch runs of the set-ups of
tests/test_opponent_gpu.py, test_geometric_opponent_gpu.py, test_multi_area_opponent_gpu.py, test_alerts_gpu.py and test_alarms_gpu.py.

* get -> set(the same arrays) -> get returns identical arrays; a get adds exactly the bytes of the arrays it returns to the
  ``d2h_bytes`` of ``env_stats`` and a set the bytes of the arrays it is given to ``h2d_bytes``; a call with some arrays NULL
  copies and counts only the others.
* A set rejected for one bad array (B200PF_E_ARG) changes nothing, the valid arrays passed with it included.
* The get entry points of a layer that is not bound fail with B200PF_E_STATE; so does the GeometricOpponent's after a new opponent
  bind, until its schedules are bound again.

``B200PF_LIB`` selects the library build these calls go to.
"""
import numpy as np
import pytest

from conftest import env_grid

E_ARG, E_STATE = -1, -4
CASE14 = "l2rpn_case14_sandbox"
CASE14_LINES = ["1_3_3", "1_4_4", "3_6_15", "9_10_12", "11_12_13", "12_13_14"]
CASE14_AREAS = [CASE14_LINES[0:2], CASE14_LINES[2:4], CASE14_LINES[4:6]]
SHORT = dict(attack_every_xxx_hour=1.5, average_attack_duration_hour=0.75, minimum_attack_duration_hour=0.25)
OPPONENTS = {
    "RandomLineOpponent": dict(attack_duration=4, attack_cooldown=6, budget_per_ts=0.5, init_budget=1.0),
    "WeightedRandomOpponent": dict(attack_duration=6, attack_cooldown=12, budget_per_ts=0.5, init_budget=8.0, attack_period=8,
                                   rho_normalization=[0.5] * 6),
    "GeometricOpponent": dict(attack_duration=7, attack_cooldown=2, budget_per_ts=0.3, init_budget=4.0, **SHORT),
    "GeometricOpponentMultiArea": dict(attack_duration=7, attack_cooldown=1, budget_per_ts=0.5, init_budget=3.0, **SHORT),
}
B = 64


def _steps(env, n, seed, alerts=0, alarms=0):
    """``n`` step_tensors steps of random actions (and random alerts / alarms when the env has them)"""
    import torch
    from test_env_tensor_gpu import _actions
    rng = np.random.default_rng(seed)
    t = lambda x: torch.as_tensor(np.asarray(x), device="cuda:0")                 # noqa: E731
    for _ in range(n):
        kw = {}
        if alerts:
            kw["raise_alert"] = t(rng.random((B, alerts)) < 0.3)
        if alarms:
            kw["raise_alarm"] = t(rng.random((B, alarms)) < 0.2)
        env.step_tensors(*(t(x) for x in _actions(env, rng)), **kw)
    torch.cuda.synchronize()


def _opponent(env, kind, lines):
    from grid2op_b200.opponent import opponent_seed
    env.enable_opponent(kind, lines, seeds=[opponent_seed(s) for s in range(B)], **OPPONENTS[kind])


def _bytes(env):
    s = env.engine.env_stats()
    return s["d2h_bytes"], s["h2d_bytes"]


def _equal(a, b):
    assert list(a) == list(b)
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), k


def _round_trip(env, get, put, set_keys=None):
    """get -> put(what get returned) -> get; ``set_keys``: the arrays put passes on (default: all)"""
    d0, h0 = _bytes(env)
    a = get()
    d1, h1 = _bytes(env)
    assert (d1 - d0, h1 - h0) == (sum(v.nbytes for v in a.values()), 0)
    put(a)
    d2, h2 = _bytes(env)
    assert (d2 - d1, h2 - h1) == (0, sum(a[k].nbytes for k in (set_keys or a)))
    _equal(a, get())
    return a


def _call(env, fn, *arrays):
    from grid2op_b200.engine import _ptr
    return getattr(env.engine.lib, fn)(env.engine.h, *[_ptr(None if x is None else np.ascontiguousarray(x)) for x in arrays])


def _partial(env, name, full, keep):
    """direct calls of b200pf_<name>_get_state / _set_state with the arrays of ``keep`` alone (the others NULL): only those are copied
    and counted"""
    out = {k: (np.empty_like(v) if k in keep else None) for k, v in full.items()}
    d0, h0 = _bytes(env)
    assert _call(env, f"b200pf_{name}_get_state", *out.values()) == 0
    d1, h1 = _bytes(env)
    nbytes = sum(out[k].nbytes for k in keep)
    assert (d1 - d0, h1 - h0) == (nbytes, 0)
    for k in keep:
        assert np.array_equal(out[k], full[k]), k
    assert _call(env, f"b200pf_{name}_set_state", *out.values()) == 0
    d2, h2 = _bytes(env)
    assert (d2 - d1, h2 - h1) == (0, nbytes)


def _rejected(env, name, get, bad):
    """b200pf_<name>_set_state with the arrays of ``bad`` (all of them changed, one of them out of range) fails with B200PF_E_ARG and
    changes nothing"""
    before = get()
    d0, h0 = _bytes(env)
    assert _call(env, f"b200pf_{name}_set_state", *bad.values()) == E_ARG
    assert _bytes(env) == (d0, h0)
    after = get()
    _equal(before, after)


def _refused(env, name, n):
    assert _call(env, f"b200pf_{name}_get_state", *[None] * n) == E_STATE


def _close(*envs):
    for e in envs:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["RandomLineOpponent", "WeightedRandomOpponent"])
def test_env_and_opponent_state_handoff(cuda_required, kind):
    if env_grid(CASE14) is None:
        pytest.skip("reference data not available")
    from test_env_tensor_gpu import _pair
    ref, env = _pair(CASE14, B, False, thermal=150.0)
    env.step_tensors(from_reset=True)
    _opponent(env, kind, CASE14_LINES)
    _steps(env, 5, seed=1)
    eng = env.engine
    s = _round_trip(env, eng.env_get_state, lambda s: eng.env_set_state(s["topo"], s["nb_inst"], s["cap_dirty"], s["obs_reset"]),
                    set_keys=("topo", "nb_inst", "cap_dirty", "obs_reset"))
    # the environment's get and set take different arrays: a partial get, a partial set, and the observe record (the observation
    # layer is bound: copied and counted)
    out = [None, np.empty_like(s["t"]), None, np.empty_like(s["cap_dirty"]), None]
    d0, h0 = _bytes(env)
    assert _call(env, "b200pf_env_get_state", *out) == 0
    assert _bytes(env) == (d0 + s["t"].nbytes + s["cap_dirty"].nbytes, h0)
    assert np.array_equal(out[1], s["t"]) and np.array_equal(out[3], s["cap_dirty"])
    rec = np.ascontiguousarray(env._obs["host_in"], np.int32)
    assert _call(env, "b200pf_env_set_state", s["topo"], None, None, s["obs_reset"].astype(np.uint8), rec) == 0
    assert _bytes(env) == (d0 + s["t"].nbytes + s["cap_dirty"].nbytes, h0 + s["topo"].nbytes + s["obs_reset"].nbytes + rec.nbytes)
    _equal(s, eng.env_get_state())

    o = _round_trip(env, eng.opp_get_state, eng.opp_set_state)
    _partial(env, "opp", o, ("budget", "mt_pos"))
    bad = {k: v.copy() for k, v in o.items()}
    bad["budget"] += 1.0
    bad["mt"] ^= 1
    bad["mt_pos"][B // 2] = 625
    _rejected(env, "opp", eng.opp_get_state, bad)
    _refused(env, "opp_geo", 3)
    _close(ref, env)


@pytest.mark.gpu
def test_geometric_opponent_state_handoff(cuda_required):
    if env_grid(CASE14) is None:
        pytest.skip("reference data not available")
    from test_env_tensor_gpu import _pair
    ref, env = _pair(CASE14, B, False, thermal=150.0, observe=False)
    env.step_tensors(from_reset=True)
    _opponent(env, "GeometricOpponent", CASE14_LINES)
    _steps(env, 5, seed=2)
    eng = env.engine
    _round_trip(env, eng.opp_get_state, eng.opp_set_state)
    g = _round_trip(env, eng.opp_geo_get_state, eng.opp_geo_set_state)
    _partial(env, "opp_geo", g, ("geo_dur", "geo_ctr"))
    bad = {k: v + 1 for k, v in g.items()}
    bad["geo_ctr"][3, 0] = g["geo_wait"].shape[1] + 1                   # a schedule longer than the cap
    _rejected(env, "opp_geo", eng.opp_geo_get_state, bad)
    # a new opponent bind drops the schedules: refused until they are bound again
    eng.opp_geo_bind = lambda t: None
    env._opp_bind_device()
    _refused(env, "opp_geo", 3)
    del eng.opp_geo_bind
    env._opp_bind_device()
    assert eng.opp_geo_get_state()["geo_wait"].shape == g["geo_wait"].shape
    _close(ref, env)


@pytest.mark.gpu
def test_multi_area_opponent_state_handoff(cuda_required):
    if env_grid(CASE14) is None:
        pytest.skip("reference data not available")
    from test_env_tensor_gpu import _pair
    ref, env = _pair(CASE14, B, False, thermal=150.0, observe=False)
    env.step_tensors(from_reset=True)
    _opponent(env, "GeometricOpponentMultiArea", CASE14_AREAS)
    _steps(env, 5, seed=3)
    eng = env.engine
    _round_trip(env, eng.opp_get_state, eng.opp_set_state)
    m = _round_trip(env, eng.opp_multi_get_state, eng.opp_multi_set_state)
    _partial(env, "opp_multi", m, ("multi_mt_pos", "multi_wait", "multi_fails"))
    bad = {k: v + 1 for k, v in m.items()}
    bad["multi_mt_pos"][:] = 0
    bad["multi_ctr"][5, 2, 1] = -1                                       # attacks consumed < 0
    _rejected(env, "opp_multi", eng.opp_multi_get_state, bad)
    _refused(env, "opp_geo", 3)
    # without the observation layer the observe record is neither copied nor counted
    d0, h0 = _bytes(env)
    eng.env_set_state(obs_in=np.zeros((B, env.gm.n_line + env.gm.n_sub + 3), np.int32))
    assert _bytes(env) == (d0, h0)
    _close(ref, env)


@pytest.mark.gpu
def test_alert_state_handoff(cuda_required):
    if env_grid(CASE14) is None:
        pytest.skip("reference data not available")
    from test_alerts_gpu import _pair_with_alerts
    ref, env = _pair_with_alerts(False, B=B, cfg="case14_random_line")
    env.step_tensors(from_reset=True)
    _opponent(env, "RandomLineOpponent", CASE14_LINES)
    _steps(env, 6, seed=4, alerts=len(CASE14_LINES))
    eng = env.engine
    a = _round_trip(env, eng.alert_get_state, eng.alert_set_state)
    _partial(env, "alert", a, ("already", "tsl_attack", "ts_attack", "cur_id"))
    ring = a["ts_attack"].shape[1]
    bad = {k: v + 1 for k, v in a.items()}
    bad["cur_id"][:] = 0
    bad["cur_id"][B - 1] = ring
    _rejected(env, "alert", eng.alert_get_state, bad)
    _refused(env, "alarm", 10)
    _close(ref, env)


@pytest.mark.gpu
def test_alarm_state_handoff(cuda_required, tmp_path):
    if env_grid(CASE14) is None:
        pytest.skip("reference data not available")
    from test_alarms_gpu import _pair_with_alarms
    ref, env = _pair_with_alarms(False, tmp_path, B=B, cfg="case14_zones")
    env.step_tensors(from_reset=True)
    _opponent(env, "GeometricOpponent", CASE14_LINES)
    _steps(env, 6, seed=5, alarms=env._alarms.n)
    eng = env.engine
    a = _round_trip(env, eng.alarm_get_state, eng.alarm_set_state)
    _partial(env, "alarm", a, ("budget", "last_ok", "ring_mask", "illegal"))
    _refused(env, "alert", 12)
    _close(ref, env)
