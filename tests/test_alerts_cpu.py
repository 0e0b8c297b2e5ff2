"""BatchedEnv's line alerts (grid2op_b200/alert.py, csrc/b200pf_alert.cuh) on the CPU:

* the numpy path next to unmodified l2rpn_idf_2023 environments (host logic on both sides, the multi-area opponent with shortened
  hours and a small budget, random alert vectors with runs of consecutive alerts): after every step the seven alert attributes,
  the AlertReward and the whole ``ObservationIDF2023.to_vect()`` (host build of the observe body) are equal, and the host build
  of the device bodies (tests/emu/alert_emu.cpp) agrees bit for bit;
* ``reset_instances`` gives the state ``env.reset()`` gives, and the observation width without alerts is unchanged;
* the ValueError cases.
"""
import os
import warnings

import numpy as np
import pytest

from conftest import env_grid

ENV = "l2rpn_idf_2023"
ALERT_ATTRS = ("active_alert", "attack_under_alert", "time_since_last_alert", "alert_duration", "total_number_of_alert",
               "time_since_last_attack", "was_alert_used_after_attack")


def _alerts_of(benv, i):
    s, a = benv._alerts.s, benv._alerts
    return dict(active_alert=s["last_alert"][i].astype(bool), attack_under_alert=s["under_alert"][i],
                time_since_last_alert=s["tsl_alert"][i], alert_duration=s["duration"][i], total_number_of_alert=s["total"][i:i + 1],
                time_since_last_attack=s["tsl_attack"][i], was_alert_used_after_attack=s["was_used"][i])


def run_alerts_vs_reference(n_steps, seeds, kill=None, engine_factory=None, backend_class=None, emu=True):
    """-> what the run saw.  ``kill``: {instance: policy} ends that instance's episode by moving every element of one substation to
    busbar 2 (a game over on this grid), timed from the reference observation's ``time_since_last_attack``: ``"alert"`` /
    ``"noalert"`` a few steps after an attack landed, the instance raising every alert / none from step 12 on; ``"noattack"`` when
    no attack lies in the window.  ``engine_factory``: the BatchedEnv engine (default: the host build of the observe body over
    the oracle adapter); ``backend_class``: the reference environments' backend (default: host logic)."""
    import grid2op_b200.backend  # noqa: F401
    import grid2op
    from grid2op.Parameters import Parameters
    from grid2op.Reward import AlertReward
    from alert_emu import COracleAlertObsEngine, EmuAlertEnvState
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import list_scenarios, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    from grid2op_b200.opponent import opponent_seed
    from test_batched_env import _scripted
    from test_geometric_opponent_cpu import _host_logic_backend
    from test_multi_area_opponent_cpu import SHORT, _geo_kw, _make
    grid = env_grid(ENV)
    gm = GridModel(grid)
    env_dir = os.path.dirname(grid)
    cdir = os.path.join(env_dir, "chronics")
    folder = list_scenarios(cdir)[0]
    chron = load_scenarios(cdir, gm, scenarios=[folder])
    B = len(seeds)
    p = Parameters()
    p.NO_OVERFLOW_DISCONNECTION = True
    p.NB_TIMESTEP_COOLDOWN_LINE = 3
    p.NB_TIMESTEP_COOLDOWN_SUB = 2
    e0 = _make("alkw")
    kwo = dict(e0._kwargs_opponent, **SHORT)
    e0.close()
    envs = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for i in range(B):
            e = grid2op.make(ENV, test=True, backend=(backend_class or _host_logic_backend())(), param=p, _add_to_name=f"al{i}", kwargs_opponent=kwo,
                             opponent_init_budget=3.0, opponent_budget_per_ts=0.5, other_rewards={"alert": AlertReward})
            e.seed(int(seeds[i]))
            e.set_id(0)
            obs0 = e.reset()
            envs.append(e)
    sp = envs[0]._oppSpace
    emt = int(sp.opponent.list_opponents[0]._episode_max_time)
    th = np.asarray(envs[0].get_thermal_limit(), dtype=np.float32)
    maint = np.stack([np.asarray(e.chronics_handler.real_data.data.maintenance, dtype=bool) for e in envs])
    benv = BatchedEnv(gm, np.repeat(chron, B, axis=0), B, maintenance=maint, scen=np.arange(B, dtype=np.int32),
                      t0=np.zeros(B, np.int32), thermal_limit_a=th, nb_timestep_cooldown_line=3, nb_timestep_cooldown_sub=2,
                      nb_timestep_reconnection=p.NB_TIMESTEP_RECONNECTION, protections=False,
                      engine=(engine_factory or COracleAlertObsEngine)(gm))
    n = benv.enable_alerts(kwo["lines_attacked"], alert_time_window=p.ALERT_TIME_WINDOW)
    assert n == type(envs[0]).dim_alerts == 22
    assert np.array_equal(benv._alerts.lines, type(envs[0]).alertable_line_ids)
    attrs = list(type(obs0).attr_list_vect)
    n_obs = benv.enable_observation(env_dir, attrs=attrs, scenarios=[folder] * B)
    assert n_obs == obs0.to_vect().size
    seg = benv._obs["tables"]["seg"]
    exact = np.zeros(n_obs, bool)                          # the alert attributes and every integer attribute: bit-equal
    for a, (src, off, ln) in zip(attrs, seg):
        if a in ALERT_ATTRS or a in ("topo_vect", "line_status", "time_before_cooldown_line", "time_before_cooldown_sub", "current_step"):
            exact[off:off + ln] = True

    # The reference's game-over observation is a new object that set_game_over does not fill for attack_under_alert: its
    # values are those of np.empty (baseObservation.py:768, :1680-1687), not a state of the environment.  Not compared there.
    uaa = np.zeros(n_obs, bool)
    for a, (src, off, ln) in zip(attrs, seg):
        uaa[off:off + ln] |= a == "attack_under_alert"

    def same_vector(mine, ob, game_over=False):
        want = ob.to_vect().astype(np.float32)
        keep = ~uaa if game_over else np.ones(n_obs, bool)
        return np.array_equal(mine[exact & keep], want[exact & keep]) and np.allclose(mine[keep], want[keep], rtol=2e-4, atol=2e-3)
    rho, _, _ = benv.reset_step()
    obs = [e.get_obs() for e in envs]
    got = _np(benv.observe()[0])
    for i in range(B):
        assert same_vector(got[i], obs[i]), i              # the reset observation (power flows: the host-logic backends' tolerance)
    benv.enable_opponent("GeometricOpponentMultiArea", kwo["lines_attacked"], attack_duration=sp.attack_max_duration,
                         attack_cooldown=sp.attack_cooldown, budget_per_ts=sp.budget_per_timestep, init_budget=sp.init_budget,
                         seeds=[opponent_seed(int(s)) for s in seeds], delta_time_seconds=envs[0].delta_time_seconds,
                         episode_max_time=emt, **_geo_kw(envs[0], **SHORT))
    em = EmuAlertEnvState(benv) if emu else None
    att = [int(x) for x in benv._opp.lines]
    rngs = [np.random.default_rng(300 + int(s)) for s in seeds]
    is_line_pos = np.zeros(gm.dim_topo, dtype=bool)
    is_line_pos[gm.line_or_pos] = True; is_line_pos[gm.line_ex_pos] = True
    kill_sub = int(np.argmax(benv.sub_size))
    saw = dict(survived_alert=0, survived_no_alert=0, blackout_alert=0, blackout_no_alert=0, blackout_no_attack=0, mixed=0,
               already_kept=0, wrap=0, illegal_alert=0, refused_budget=0)
    kill = kill or {}
    W = p.ALERT_TIME_WINDOW
    alive = np.ones(B, dtype=bool)
    runs = np.zeros((B, n), bool)
    for k in range(n_steps):
        sub_id = np.full(B, -1, np.int64); sub_bus = np.zeros((B, benv.max_sub_size), np.int8)
        line_id = np.full(B, -1, np.int64); line_st = np.zeros(B, np.int64)
        # alerts: runs of consecutive alerts that start and stop at random
        flip = np.stack([r.random(n) < 0.15 for r in rngs])
        runs ^= flip
        raise_alert = runs.copy()
        for i, pol in kill.items():
            if pol in ("alert", "noalert") and k >= 12:
                raise_alert[i] = pol == "alert"
        ref = []
        for i, e in enumerate(envs):
            if not alive[i]:
                ref.append(None)
                continue
            ob = obs[i]
            a = _scripted(k, rngs[i], ob.topo_vect, ob.line_status, ob.time_before_cooldown_line, ob.time_before_cooldown_sub,
                          benv.sub_pos, benv.sub_size, gm.n_line, is_line_pos)
            out = [l for l in att if not ob.line_status[l] and ob.time_before_cooldown_line[l] == 0]
            if k % 2 == 0 and out:
                a = dict(sub=-1, bus=None, line=int(out[0]), status=1)
            tsla = np.asarray(ob.time_since_last_attack)
            if i in kill and ob.time_before_cooldown_sub[kill_sub] == 0 and (
                    (kill[i] in ("alert", "noalert") and k >= 14 and ((tsla >= 1) & (tsla <= 4)).any()) or
                    (kill[i] == "noattack" and k >= 20 and ((tsla == -1) | (tsla > W + 2)).all())):
                a = dict(sub=kill_sub, bus=np.full(int(benv.sub_size[kill_sub]), 2), line=-1, status=0)
            spec = {"raise_alert": [int(x) for x in np.flatnonzero(raise_alert[i])]}
            if a["sub"] >= 0:
                spec["set_bus"] = {"substations_id": [(a["sub"], a["bus"].astype(int).tolist())]}
                sub_id[i] = a["sub"]; sub_bus[i, :len(a["bus"])] = a["bus"]
            if a["line"] >= 0:
                spec["set_line_status"] = [(a["line"], int(a["status"]))]
                line_id[i] = a["line"]; line_st[i] = a["status"]
            already = envs[i]._is_already_attacked.copy()
            o2, r, d, info = e.step(e.action_space(spec))
            obs[i] = o2
            ref.append((d, info, already))
            saw["refused_budget"] += bool(e._oppSpace.previous_fails)
        prev_rho = benv.engine.series_fetch(want_out=False)[3]
        if em is not None:
            assert em.step_apply(sub_id, sub_bus, line_id, line_st, rho=prev_rho)[2] == 0
        rho, done, binfo = benv.step(sub_id, sub_bus, line_id, line_st, raise_alert=raise_alert)
        if em is not None:
            em.step_post(binfo["status"], None, stamp=benv.n_steps, raise_alert=raise_alert)
            st = benv.alert_state()
            for key, v in em.alert_state().items():
                assert np.array_equal(v, st[key]), (k, key)
            assert np.array_equal(em.ast["reward_out"], binfo["rewards"]["alert"]), k
            assert np.array_equal(em.st["obs_in"], benv.observe_inputs()), k
        vec = _np(benv.observe()[0])
        for i in range(B):
            if not alive[i]:
                assert binfo["rewards"]["alert"][i] == 0.0
                continue
            d, info, already = ref[i]
            assert bool(done[i]) == bool(d), (k, i, info["exception"])
            want_r = info["rewards"]["alert"]
            assert binfo["rewards"]["alert"][i] == want_r, (k, i, binfo["rewards"]["alert"][i], want_r)
            ob = obs[i]
            mine = _alerts_of(benv, i)
            if not d:
                for nm in ALERT_ATTRS:
                    assert np.array_equal(np.asarray(getattr(ob, nm)), mine[nm]), (k, i, nm)
            assert same_vector(vec[i], ob, game_over=bool(d)), (k, i)
            la = info["opponent_attack_line"]
            hit = np.zeros(n, bool) if la is None else la[benv._alerts.lines]
            used = np.asarray(ob.was_alert_used_after_attack)           # the reference's: +-1 where a score was given
            assert np.array_equal(used, benv._alerts.s["was_used"][i]), (k, i)
            if used.any():
                if d:
                    saw["blackout_alert" if (used > 0).any() else "blackout_no_alert"] += 1
                else:
                    saw["survived_alert" if (used < 0).any() else "survived_no_alert"] += 1
                saw["mixed"] += bool((used > 0).any() and (used < 0).any())         # a mean strictly between 0 and 1
            elif d:
                assert want_r == 0.0
                saw["blackout_no_attack"] += 1
            if la is not None and (already & ~hit).any():
                saw["already_kept"] += 1
            saw["illegal_alert"] += bool(info["is_illegal"]) and raise_alert[i].any()
            if d:
                alive[i] = False
        saw["wrap"] += int((benv._alerts.s["cur_id"] == 0).any() and k > benv._alerts.ring)
    # env.reset() of every environment against reset_instances: the alert state and the reset observation's alert attributes
    idx = np.arange(B)
    for e in envs:
        e.set_id(0)
    obs = [e.reset() for e in envs]
    benv.reset_instances(idx, rows=np.zeros(B, np.int64))
    vec = _np(benv.observe()[0])
    for i in range(B):
        mine = _alerts_of(benv, i)
        want = obs[i].to_vect().astype(np.float32)
        for nm in ALERT_ATTRS:
            assert np.array_equal(np.asarray(getattr(obs[i], nm)), mine[nm]), (i, nm)
        for a, (src, off, ln) in zip(attrs, seg):
            if a in ALERT_ATTRS:
                assert np.array_equal(vec[i, off:off + ln], want[off:off + ln]), (i, a)
    for e in envs:
        e.close()
    benv.close()
    return saw


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


KILLS = {3: "alert", 4: "noalert", 5: "noattack", 6: "alert", 7: "noalert"}
SAW_ALL = ("survived_alert", "survived_no_alert", "blackout_alert", "blackout_no_alert", "blackout_no_attack", "mixed", "already_kept",
           "wrap", "illegal_alert", "refused_budget")


def test_alerts_vs_reference_env_host_logic():
    if env_grid(ENV) is None:
        pytest.skip("reference data not available")
    saw = run_alerts_vs_reference(150, (0, 3, 5, 7, 9, 11, 13, 17), kill=KILLS)
    assert all(saw[k] > 0 for k in SAW_ALL), saw


# ---- reset and validation ----------------------------------------------------------------------------------------------------
def _small_env(B=2):
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.gridmodel import GridModel
    from oracle_engine import COracleSeriesEngine
    grid = env_grid("l2rpn_case14_sandbox")
    if grid is None:
        pytest.skip("reference data not available")
    from grid2op_b200.chronics import list_scenarios, load_scenarios
    gm = GridModel(grid)
    cdir = os.path.join(os.path.dirname(grid), "chronics")
    chron = load_scenarios(cdir, gm, scenarios=list_scenarios(cdir)[:1])[:, :12]
    return BatchedEnv(gm, chron, B, scen=np.zeros(B, np.int32), t0=np.zeros(B, np.int32), protections=False,
                      engine=COracleSeriesEngine(gm))


@pytest.mark.parametrize("lines,kw", [
    ([0, 999], {}), ([0, -1], {}), (["no such line"], {}), ([0, 1, 0], {}), ([], {}),
    (list(range(65)), {}), ([0, 1], dict(alert_time_window=0)),
])
def test_enable_alerts_rejected(lines, kw):
    benv = _small_env()
    with pytest.raises(ValueError):
        benv.enable_alerts(lines, **kw)
    assert benv._alerts is None


def test_enable_alerts_after_observation_raises_and_width_unchanged():
    from grid2op_b200.observation import COMPLETE_OBSERVATION_ATTRS, attr_sizes, obs_spec
    benv = _small_env()
    gm = benv.gm
    assert attr_sizes(gm) == attr_sizes(gm, 0)
    assert obs_spec(gm)[1] == obs_spec(gm, None, 0)[1]
    assert obs_spec(gm, None, 3)[1] == obs_spec(gm)[1] + 6 * 3 + 1
    assert all(attr_sizes(gm)[a] == 0 for a in ALERT_ATTRS)
    assert set(COMPLETE_OBSERVATION_ATTRS) >= set(ALERT_ATTRS)
    benv._obs = {}                                         # (as enable_observation leaves it)
    with pytest.raises(RuntimeError):
        benv.enable_alerts([0, 1])


def test_raise_alert_checked_and_reset_instances():
    benv = _small_env(B=3)
    benv.enable_alerts([benv.gm.name_line[2], 4, [5, 6]])
    assert list(benv._alerts.lines) == [2, 4, 5, 6]
    benv.reset_step()
    with pytest.raises(ValueError):
        benv.step(raise_alert=np.zeros((3, 3), bool))
    up = np.zeros((3, 4), bool); up[:, 1] = True; up[0, 3] = True
    for _ in range(3):
        _, _, info = benv.step(raise_alert=up)
    st = benv.alert_state()
    assert list(st["total"]) == [6, 3, 3] and list(st["duration"][:, 1]) == [3, 3, 3]
    assert np.array_equal(info["rewards"]["alert"], np.zeros(3))
    assert (st["tsl_attack"] == -1).all() and list(st["cur_id"]) == [3, 3, 3]
    benv.reset_instances([1])
    s2 = benv.alert_state()
    assert s2["total"][1] == 0 and (s2["tsl_alert"][1] == -1).all() and s2["cur_id"][1] == 0 and not s2["launched"][1].any()
    assert s2["total"][0] == 6


# ---- a single-line opponent: rte_case14_opponent with alerts_info.json --------------------------------------------------------
def run_case14_alerts_vs_reference(tmp_dir, n_steps, seeds, engine_factory=None, backend_class=None):
    """a copy of rte_case14_opponent with ``alerts_info.json`` (``"by_line": "opponent"``) written into it: its RandomLineOpponent,
    with multi-step attacks, feeds the alerts.  Unmodified grid2op environments (PlayableAction, AlertReward) next to BatchedEnv;
    the alert state, the reward and was_alert_used_after_attack equal after every step.  -> what the run saw"""
    import json
    import shutil
    import grid2op_b200.backend  # noqa: F401
    import grid2op
    from grid2op.Action import PlayableAction
    from grid2op.Parameters import Parameters
    from grid2op.Reward import AlertReward
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import load_line_events, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    from grid2op_b200.opponent import opponent_seed
    from oracle_engine import COracleSeriesEngine
    from test_batched_env import _scripted
    from test_geometric_opponent_cpu import _host_logic_backend
    src = os.path.dirname(env_grid("rte_case14_opponent"))
    env_dir = os.path.join(str(tmp_dir), "rte_case14_opponent_alerts")
    shutil.copytree(src, env_dir)
    with open(os.path.join(env_dir, "alerts_info.json"), "w") as f:
        json.dump({"by_line": "opponent"}, f)
    gm = GridModel(os.path.join(env_dir, "grid.json"))
    cdir = os.path.join(env_dir, "chronics")
    folder = os.path.join(cdir, sorted(os.listdir(cdir))[0])
    chron = load_scenarios(cdir, gm, scenarios=[folder])
    maint = load_line_events(folder, gm, "maintenance")
    B = len(seeds)
    p = Parameters()
    p.NO_OVERFLOW_DISCONNECTION = True
    p.NB_TIMESTEP_COOLDOWN_LINE = 3
    p.NB_TIMESTEP_COOLDOWN_SUB = 2
    p.ALERT_TIME_WINDOW = 5
    envs = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for i in range(B):
            e = grid2op.make(env_dir, test=True, backend=(backend_class or _host_logic_backend())(), param=p, _add_to_name=f"a14{i}",
                             action_class=PlayableAction, other_rewards={"alert": AlertReward}, opponent_init_budget=1.0,
                             opponent_attack_duration=5, opponent_attack_cooldown=6)
            e.seed(int(seeds[i]))
            e.set_id(0)
            e.reset()
            envs.append(e)
    sp, kwo = envs[0]._oppSpace, envs[0]._kwargs_opponent
    assert type(sp.opponent).__name__ == "RandomLineOpponent" and type(envs[0]).dim_alerts == len(kwo["lines_attacked"])
    th = np.asarray(envs[0].get_thermal_limit(), dtype=np.float32)
    benv = BatchedEnv(gm, chron, B, maintenance=None if maint is None else maint[None], scen=np.zeros(B, np.int32),
                      t0=np.zeros(B, np.int32), thermal_limit_a=th, nb_timestep_cooldown_line=3, nb_timestep_cooldown_sub=2,
                      nb_timestep_reconnection=p.NB_TIMESTEP_RECONNECTION, protections=False,
                      engine=(engine_factory or COracleSeriesEngine)(gm))
    n = benv.enable_alerts(kwo["lines_attacked"], alert_time_window=p.ALERT_TIME_WINDOW)
    assert np.array_equal(benv._alerts.lines, type(envs[0]).alertable_line_ids)
    benv.reset_step()
    obs = [e.get_obs() for e in envs]
    benv.enable_opponent("RandomLineOpponent", kwo["lines_attacked"], attack_duration=sp.attack_max_duration,
                         attack_cooldown=sp.attack_cooldown, budget_per_ts=sp.budget_per_timestep, init_budget=sp.init_budget,
                         seeds=[opponent_seed(int(s)) for s in seeds])
    rngs = [np.random.default_rng(500 + int(s)) for s in seeds]
    is_line_pos = np.zeros(gm.dim_topo, dtype=bool)
    is_line_pos[gm.line_or_pos] = True; is_line_pos[gm.line_ex_pos] = True
    saw = dict(attack_steps=0, long_attack=0, survived_alert=0, survived_no_alert=0)
    alive = np.ones(B, dtype=bool)
    runs = np.zeros((B, n), bool)
    run_len = np.zeros(B, np.int64)
    for k in range(n_steps):
        sub_id = np.full(B, -1, np.int64); sub_bus = np.zeros((B, benv.max_sub_size), np.int8)
        line_id = np.full(B, -1, np.int64); line_st = np.zeros(B, np.int64)
        runs ^= np.stack([r.random(n) < 0.2 for r in rngs])
        ref = []
        for i, e in enumerate(envs):
            if not alive[i]:
                ref.append(None)
                continue
            ob = obs[i]
            a = _scripted(k, rngs[i], ob.topo_vect, ob.line_status, ob.time_before_cooldown_line, ob.time_before_cooldown_sub,
                          benv.sub_pos, benv.sub_size, gm.n_line, is_line_pos)
            spec = {"raise_alert": [int(x) for x in np.flatnonzero(runs[i])]}
            if a["sub"] >= 0:
                spec["set_bus"] = {"substations_id": [(a["sub"], a["bus"].astype(int).tolist())]}
                sub_id[i] = a["sub"]; sub_bus[i, :len(a["bus"])] = a["bus"]
            if a["line"] >= 0:
                spec["set_line_status"] = [(a["line"], int(a["status"]))]
                line_id[i] = a["line"]; line_st[i] = a["status"]
            o2, r, d, info = e.step(e.action_space(spec))
            obs[i] = o2
            ref.append((d, info))
        _, done, binfo = benv.step(sub_id, sub_bus, line_id, line_st, raise_alert=runs)
        rew = _np(binfo["rewards"]["alert"])
        for i in range(B):
            if not alive[i]:
                assert rew[i] == 0.0
                continue
            d, info = ref[i]
            assert bool(done[i]) == bool(d), (k, i, info["exception"])
            assert rew[i] == info["rewards"]["alert"], (k, i, rew[i], info["rewards"]["alert"])
            mine, ob = _alerts_of(benv, i), obs[i]
            if not d:
                for nm in ALERT_ATTRS:
                    assert np.array_equal(np.asarray(getattr(ob, nm)), mine[nm]), (k, i, nm)
            used = np.asarray(ob.was_alert_used_after_attack)
            assert np.array_equal(used, mine["was_alert_used_after_attack"]), (k, i)
            if used.any() and not d:
                saw["survived_alert" if (used < 0).any() else "survived_no_alert"] += 1
            la = info["opponent_attack_line"]
            if la is not None:
                saw["attack_steps"] += 1
                run_len[i] += 1
                saw["long_attack"] += int(run_len[i] == 3)
            else:
                run_len[i] = 0
            if d:
                alive[i] = False
    for e in envs:
        e.close()
    benv.close()
    return saw


def test_alerts_single_line_opponent_vs_reference_env_host_logic(tmp_path):
    if env_grid("rte_case14_opponent") is None:
        pytest.skip("reference data not available")
    saw = run_case14_alerts_vs_reference(tmp_path, 80, (1, 2, 4, 8))
    assert all(saw[k] > 0 for k in saw), saw
