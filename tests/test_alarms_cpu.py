"""BatchedEnv's alarms (grid2op_b200/alarm.py, csrc/b200pf_alarm.cuh) on the CPU:

* the numpy path next to unmodified l2rpn_icaps_2021 environments (host logic on both sides, ActionICAPS2021,
  ObservationICAPS2021, AlarmReward, LinearAttentionBudget with a faster refill, the GeometricOpponent on), protections off and on,
  random alarms on one or two zones and scripted actions: after every step the budget, the four "last alarm" values, the ring
  against ``_all_successful_alarms``, the reward, ``is_alarm_illegal``, ``_is_alarm_used_in_reward``, the five alarm attributes
  and ``to_vect()`` are equal, and the host build of the device bodies (tests/emu/alarm_emu.cpp) agrees bit for bit;
* ``AlarmReward`` itself on scripted game overs (a first-round trip in or out of the alarm's zone, two zones, an alarm too early
  or too late, no trip, no alarm) against the numpy path and the host build, the sticky ``is_alarm_used`` included;
* ``env.reset()`` against ``reset_instances``, ``load_alarm_zones`` against grid2op's zones, and the ValueError cases.
"""
import json
import os
import warnings

import numpy as np
import pytest

from conftest import env_grid

ENV = "l2rpn_icaps_2021"
ALARM_ATTRS = ("is_alarm_illegal", "time_since_last_alarm", "last_alarm", "attention_budget", "was_alarm_used_after_game_over")
# LinearAttentionBudget with a refill of 0.1 per step (not exact in float32) so that the cap is reached within the run
BUDGET = dict(max_budget=3.0, budget_per_ts=0.1, alarm_cost=1.0, init_budget=2.0)
# Timed game overs with a first-round trip (protections on): disconnecting CUT sends about 10 times its flow onto TRIP[0] and 4 times
# onto TRIP[1], the two lines of a load substation; with TRIP[1]'s thermal limit lowered to TRIP_LIMIT_A (rho about 0.8 before)
# both exceed the hard threshold in the cascade's first round, the substation is islanded and the episode ends.  Both lines are
# in the "west" zone.  KILL_AT: the loop iteration of the cut (step KILL_AT + 1); an alarm raised KILL_AT - 12 iterations before
# lies at ALARM_BEST_TIME.
CUT, TRIP, TRIP_LIMIT_A, KILL_AT = "33_36_114", ("34_35_110", "33_35_113"), 65.0, 30
# instance -> how its episode ends (protections on; the other instances act at random)
TIMED = {1: "bonus", 2: "half", 3: "two_zones", 4: "too_early", 5: "too_late", 6: "no_alarm", 7: "no_trip"}


def _alarm_attrs_of(benv, i, game_over):
    """the five attributes as BatchedEnv's record gives them (the observe body's game-over rules)"""
    a = benv._alarms
    rec = a.obs_record(benv.current_step)[i]
    n = a.n
    if game_over:
        return dict(is_alarm_illegal=False, time_since_last_alarm=-1, last_alarm=np.zeros(n, np.int32), attention_budget=np.float32(0),
                    was_alarm_used_after_game_over=bool(rec[3 + n]))
    return dict(is_alarm_illegal=bool(rec[0]), time_since_last_alarm=int(rec[1]), last_alarm=rec[2:2 + n],
                attention_budget=rec[2 + n:3 + n].view(np.float32)[0], was_alarm_used_after_game_over=False)


def _ring_matches(st, i, step, succ, R):
    """the ring of instance i holds exactly the entries of _all_successful_alarms of the last R steps"""
    want = {int(s): np.flatnonzero(m) for s, m in succ if step - int(s) < R}
    got = {int(s): np.flatnonzero([(int(st["ring_mask"][i, r]) >> z) & 1 for z in range(32)])
           for r, s in enumerate(st["ring_step"][i]) if s > 0 and 0 <= step - s < R}
    return want.keys() == got.keys() and all(np.array_equal(want[s], got[s]) for s in want)


def run_alarms_vs_reference(n_steps, seeds, protections, engine_factory=None, backend_class=None, emu=True):
    """-> what the run saw.  Unmodified l2rpn_icaps_2021 environments next to BatchedEnv with ``enable_alarms`` on the zones of
    the environment's alerts_info.json.  ``engine_factory``: the BatchedEnv engine (default: the host build of the observe body
    over the oracle adapter, with the host build of the planned kernel's cascades when ``protections``); ``backend_class``: the
    reference environments' backend (default: host logic)."""
    import grid2op_b200.backend  # noqa: F401
    import grid2op
    from grid2op.Parameters import Parameters
    from alarm_emu import COracleAlarmObsEngine, EmuAlarmEnvState, EmuProtAlarmObsEngine
    from grid2op_b200.alarm import load_alarm_zones
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import list_scenarios, load_line_events, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    from grid2op_b200.opponent import opponent_seed
    from test_batched_env import _scripted
    from test_geometric_opponent_cpu import _geo_kw, _host_logic_backend, short_kw
    grid = env_grid(ENV)
    gm = GridModel(grid)
    env_dir = os.path.dirname(grid)
    cdir = os.path.join(env_dir, "chronics")
    folder = list_scenarios(cdir)[0]
    chron = load_scenarios(cdir, gm, scenarios=[folder])
    maint = load_line_events(folder, gm, "maintenance")
    B = len(seeds)
    p = Parameters()
    p.NO_OVERFLOW_DISCONNECTION = not protections
    p.NB_TIMESTEP_COOLDOWN_LINE = 3
    p.NB_TIMESTEP_COOLDOWN_SUB = 2
    mk = short_kw(ENV)
    names = [str(x) for x in gm.name_line]
    cut, trip = names.index(CUT), [names.index(x) for x in TRIP]
    timed = TIMED if protections else {}
    envs = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for i in range(B):
            e = grid2op.make(ENV, test=True, backend=(backend_class or _host_logic_backend())(), param=p, _add_to_name=f"alarm{i}",
                             kwargs_attention_budget=dict(BUDGET), **mk(i))
            if protections:
                lim = e.get_thermal_limit()
                lim[trip[1]] = TRIP_LIMIT_A
                e.set_thermal_limit(lim)
            e.seed(int(seeds[i]))
            e.set_id(0)
            obs0 = e.reset()
            envs.append(e)
    e0 = envs[0]
    assert type(e0.get_reward_instance()).__name__ == "AlarmReward" and type(e0._attention_budget).__name__ == "LinearAttentionBudget"
    sp, kwo = e0._oppSpace, e0._kwargs_opponent
    th = np.asarray(e0.get_thermal_limit(), dtype=np.float32)                 # (TRIP[1] lowered with the protections on)
    default_engine = EmuProtAlarmObsEngine if protections else COracleAlarmObsEngine
    benv = BatchedEnv(gm, chron, B, maintenance=None if maint is None else maint[None], scen=np.zeros(B, np.int32),
                      t0=np.zeros(B, np.int32), thermal_limit_a=th, nb_timestep_cooldown_line=3, nb_timestep_cooldown_sub=2,
                      nb_timestep_reconnection=p.NB_TIMESTEP_RECONNECTION, protections=protections,
                      engine=(engine_factory or default_engine)(gm))
    zones = load_alarm_zones(env_dir, gm)
    assert zones[0] == list(type(e0).alarms_area_names)
    n = benv.enable_alarms(zones, alarm_best_time=int(p.ALARM_BEST_TIME), alarm_window_size=int(p.ALARM_WINDOW_SIZE), **BUDGET)
    assert n == type(e0).dim_alarms == 3
    assert int(p.ALARM_BEST_TIME) == int(p.ALARM_WINDOW_SIZE) == 12
    west = zones[0].index("west")
    assert all((int(zones[1][l]) >> west) & 1 for l in trip)
    other = next(z for z in range(n) if not any((int(zones[1][l]) >> z) & 1 for l in trip))
    attrs = list(type(obs0).attr_list_vect)
    n_obs = benv.enable_observation(env_dir, attrs=attrs, scenarios=[folder])
    assert n_obs == obs0.to_vect().size
    seg = benv._obs["tables"]["seg"]
    exact = np.zeros(n_obs, bool)                          # the alarm attributes and every integer attribute: bit-equal
    for a, (src, off, ln) in zip(attrs, seg):
        if a in ALARM_ATTRS or a in ("topo_vect", "line_status", "time_before_cooldown_line", "time_before_cooldown_sub", "current_step"):
            exact[off:off + ln] = True

    def same_vector(mine, ob):
        want = ob.to_vect().astype(np.float32)
        return np.array_equal(mine[exact], want[exact]) and np.allclose(mine, want, rtol=2e-4, atol=2e-3)

    benv.reset_step()
    obs = [e.get_obs() for e in envs]
    got = _np(benv.observe()[0])
    for i in range(B):
        assert same_vector(got[i], obs[i]), i              # the reset observation
    benv.enable_opponent("GeometricOpponent", kwo["lines_attacked"], attack_duration=sp.attack_max_duration,
                         attack_cooldown=sp.attack_cooldown, budget_per_ts=sp.budget_per_timestep, init_budget=sp.init_budget,
                         seeds=[opponent_seed(int(s)) for s in seeds], delta_time_seconds=e0.delta_time_seconds,
                         episode_max_time=int(sp.opponent._episode_max_time), pmax_pmin_ratio=kwo.get("pmax_pmin_ratio", 4),
                         **_geo_kw(e0))
    em = EmuAlarmEnvState(benv) if emu else None
    rngs = [np.random.default_rng(700 + int(s)) for s in seeds]
    is_line_pos = np.zeros(gm.dim_topo, dtype=bool)
    is_line_pos[gm.line_or_pos] = True; is_line_pos[gm.line_ex_pos] = True
    kill_sub = int(np.argmax(benv.sub_size))
    load_sub = int(np.intersect1d([gm.line_or_sub[trip[0]], gm.line_ex_sub[trip[0]]], [gm.line_or_sub[trip[1]], gm.line_ex_sub[trip[1]]])[0])
    load_pos = benv.sub_pos[load_sub, :int(benv.sub_size[load_sub])]
    saw = dict(refused_budget=0, illegal_with_alarm=0, capped=0, multi_zone_ok=0, wrap=0, game_over=0, used_before_reset=0,
               **{pol: 0 for pol in TIMED.values()})
    R = benv._alarms.ring
    alive = np.ones(B, dtype=bool)
    for k in range(n_steps):
        sub_id = np.full(B, -1, np.int64); sub_bus = np.zeros((B, benv.max_sub_size), np.int8)
        line_id = np.full(B, -1, np.int64); line_st = np.zeros(B, np.int64)
        raise_alarm = np.zeros((B, n), bool)
        ref = []
        for i, e in enumerate(envs):
            if not alive[i]:
                ref.append(None)
                continue
            ob, rng = obs[i], rngs[i]
            if i in timed:                                    # no action but the scripted alarm and, at KILL_AT, the game over
                pol = timed[i]
                a = dict(sub=-1, bus=None, line=-1, status=0)
                if (pol in ("bonus", "half") and k == KILL_AT - 12) or (pol == "too_late" and k == KILL_AT):
                    raise_alarm[i, west if pol != "half" else other] = True
                elif pol == "two_zones" and k == KILL_AT - 12:
                    raise_alarm[i, [west, other]] = True
                elif pol == "too_early" and k == KILL_AT - 24:
                    raise_alarm[i, west] = True
                if k == KILL_AT and pol != "no_trip":
                    a = dict(sub=-1, bus=None, line=cut, status=-1)
                elif k == KILL_AT:                            # the load of TRIP's substation alone on busbar 2: no trip
                    a = dict(sub=load_sub, bus=np.where(np.isin(load_pos, gm.load_pos), 2, 1).astype(np.int8), line=-1, status=0)
            else:
                u = rng.random() * (1.0 if i >= 2 else 6.0)   # instances 0 and 1 raise few alarms: their budget reaches the cap
                if u < 0.2:
                    raise_alarm[i, rng.integers(n)] = True
                elif u < 0.3:
                    raise_alarm[i, rng.choice(n, 2, replace=False)] = True
                a = _scripted(k, rng, ob.topo_vect, ob.line_status, ob.time_before_cooldown_line, ob.time_before_cooldown_sub,
                              benv.sub_pos, benv.sub_size, gm.n_line, is_line_pos)
                if i % 4 == 3 and k == 40 + 20 * (i // 4) and ob.time_before_cooldown_sub[kill_sub] == 0:
                    a = dict(sub=kill_sub, bus=np.full(int(benv.sub_size[kill_sub]), 2), line=-1, status=0)    # a game over
            spec = {"raise_alarm": [int(x) for x in np.flatnonzero(raise_alarm[i])]}
            if a["sub"] >= 0:
                spec["set_bus"] = {"substations_id": [(a["sub"], a["bus"].astype(int).tolist())]}
                sub_id[i] = a["sub"]; sub_bus[i, :len(a["bus"])] = a["bus"]
            if a["line"] >= 0:
                spec["set_line_status"] = [(a["line"], int(a["status"]))]
                line_id[i] = a["line"]; line_st[i] = a["status"]
            b0 = np.float32(e._attention_budget.current_budget)
            o2, r, d, info = e.step(e.action_space(spec))
            obs[i] = o2
            ref.append((d, r, info, b0))
        prev_rho = benv.engine.series_fetch(want_out=False)[3]
        if em is not None:
            assert em.step_apply(sub_id, sub_bus, line_id, line_st, rho=prev_rho)[2] == 0
        rho, done, binfo = benv.step(sub_id, sub_bus, line_id, line_st, raise_alarm=raise_alarm)
        if em is not None:
            em.step_post(binfo["status"], binfo["disc_lines"], stamp=benv.n_steps, prot=protections, raise_alarm=raise_alarm)
            st = benv.alarm_state()
            for key, v in em.alarm_state().items():
                assert np.array_equal(v, st[key]), (k, key)
            assert np.array_equal(em.ast["reward_out"], binfo["rewards"]["alarm"]), k
            assert np.array_equal(em.st["obs_in"], benv.observe_inputs()), k
        vec = _np(benv.observe()[0])
        st = benv.alarm_state()
        for i in range(B):
            if not alive[i]:
                assert binfo["rewards"]["alarm"][i] == 0.0 and not binfo["is_alarm_illegal"][i]
                continue
            d, r, info, b0 = ref[i]
            e = envs[i]
            ab = e._attention_budget
            assert bool(done[i]) == bool(d), (k, i, info["exception"])
            assert binfo["rewards"]["alarm"][i] == r, (k, i, binfo["rewards"]["alarm"][i], r)
            assert bool(binfo["is_alarm_illegal"][i]) == bool(e._is_alarm_illegal) == (info["reason_alarm_illegal"] is not None), (k, i)
            assert bool(binfo["is_illegal"][i]) == bool(info["is_illegal"]), (k, i)
            assert st["budget"][i] == np.float32(ab.current_budget), (k, i, st["budget"][i], ab.current_budget)
            assert st["time_last"][i] == ab.time_last_alarm_raised and st["time_last_ok"][i] == ab.time_last_successful_alarm_raised, (k, i)
            assert np.array_equal(st["last"][i], ab.last_alarm_raised) and np.array_equal(st["last_ok"][i], ab.last_successful_alarm_raised), (k, i)
            assert _ring_matches(st, i, int(benv.current_step[i]), ab._all_successful_alarms, R), (k, i)
            assert bool(st["any_ok"][i]) == bool(len(ab._all_successful_alarms)), (k, i)
            assert bool(st["used"][i]) == bool(e.get_reward_instance().is_alarm_used), (k, i)
            assert bool(e._is_alarm_used_in_reward) == (bool(st["used"][i]) if d else False), (k, i)
            ob = obs[i]
            mine = _alarm_attrs_of(benv, i, bool(d))
            for nm in ALARM_ATTRS:
                assert np.array_equal(np.asarray(getattr(ob, nm)).ravel(), np.asarray(mine[nm]).ravel()), (k, i, nm)
            assert same_vector(vec[i], ob), (k, i)
            up = raise_alarm[i]
            saw["refused_budget"] += bool(binfo["is_alarm_illegal"][i])
            saw["illegal_with_alarm"] += bool(info["is_illegal"]) and up.any() and st["budget"][i] == b0
            saw["capped"] += bool(not up.any() and not info["is_illegal"] and b0 > np.float32(2.95) and st["budget"][i] == np.float32(3.0))
            saw["multi_zone_ok"] += bool(up.sum() == 2 and st["time_last_ok"][i] == benv.current_step[i] and
                                         st["budget"][i] == b0 - np.float32(1.0))
            if d:
                saw["game_over"] += 1
                alive[i] = False
                if i in timed and k == KILL_AT:               # the outcome each timed game over is scripted for
                    pol, rew = timed[i], binfo["rewards"]["alarm"][i]
                    disc = binfo["disc_lines"][i]
                    first = bool((disc[trip] == 0).any())
                    want = {"bonus": first and rew == 1.0, "half": first and rew == 0.5, "two_zones": first and rew == 0.5,
                            "too_early": first and rew == -1.0 and st["any_ok"][i] and not st["used"][i],
                            "too_late": first and rew == -1.0 and st["any_ok"][i] and not st["used"][i],
                            "no_alarm": first and rew == -1.0 and not st["any_ok"][i],
                            "no_trip": bool((disc == -1).all()) and rew == -1.0}[pol]
                    saw[pol] += int(want)
        saw["wrap"] += int(any(_ring_wrapped(st, i, int(benv.current_step[i]), R) for i in range(B)))
    # env.reset() of every environment against reset_instances: the budget state and the reset observation's alarm attributes
    idx = np.arange(B)
    used_before = benv.alarm_state()["used"].copy()
    saw["used_before_reset"] = int(used_before.sum())
    for e in envs:
        e.set_id(0)
    obs = [e.reset() for e in envs]
    benv.reset_instances(idx, rows=np.zeros(B, np.int64))
    vec = _np(benv.observe()[0])
    st = benv.alarm_state()
    assert np.array_equal(st["used"], used_before)
    for i in range(B):
        ab = envs[i]._attention_budget
        assert st["budget"][i] == np.float32(ab.current_budget) and st["time_last_ok"][i] == -1 and not st["any_ok"][i]
        assert bool(st["used"][i]) == bool(envs[i].get_reward_instance().is_alarm_used)
        want = obs[i].to_vect().astype(np.float32)
        for a, (src, off, ln) in zip(attrs, seg):
            if a in ALARM_ATTRS:
                assert np.array_equal(vec[i, off:off + ln], want[off:off + ln]), (i, a)
    for e in envs:
        e.close()
    benv.close()
    return saw


def _ring_wrapped(st, i, step, R):
    """the ring of instance i holds a successful alarm of the current lap and one of the previous lap"""
    s = st["ring_step"][i]
    return step > R and (s > step - R).any() and ((s > 0) & (s <= step - R)).any()


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


SEEDS = (0, 3, 5, 7, 9, 11, 13, 17)
SAW_ALL = ("refused_budget", "illegal_with_alarm", "capped", "multi_zone_ok", "wrap", "game_over")
# with the protections on, seven instances run the timed game overs: every AlarmReward branch on a game over with a first-round
# trip (full score with the zone bonus, half score without it and for two zones, an alarm at either end of the window, no alarm),
# one without a trip, and AlarmReward.is_alarm_used set before env.reset() / reset_instances (which keep it)
SAW_PROT = ("game_over", "used_before_reset") + tuple(TIMED.values())


@pytest.mark.parametrize("protections", [False, True])
def test_alarms_vs_reference_env_host_logic(protections):
    if env_grid(ENV) is None:
        pytest.skip("reference data not available")
    saw = run_alarms_vs_reference(150, SEEDS, protections)
    assert all(saw[k] > 0 for k in (SAW_PROT if protections else SAW_ALL)), saw


# ---- AlarmReward on scripted game overs --------------------------------------------------------------------------------------
class _Budget:
    def __init__(self, alarms):
        self._all_successful_alarms = alarms


class _Env:
    """what AlarmReward.__call__ reads of the environment"""

    def __init__(self, names, mask, step, disc, alarms):
        self.name_line = [f"l{j}" for j in range(len(mask))]
        self.alarms_area_names = list(names)
        self.alarms_lines_area = {f"l{j}": [names[z] for z in range(len(names)) if (int(m) >> z) & 1] for j, m in enumerate(mask)}
        self.nb_time_step = step
        self._disc_lines = np.asarray(disc, np.int32)
        self._attention_budget = _Budget(alarms)


# (game-over step, disc_lines of 6 lines, successful alarms as (step, zones)); zones: line 0-1 "a", 2-3 "b", 4-5 "c", line 1 also "b"
CASES = [
    ("bonus", 40, [0, -1, -1, -1, -1, -1], [(28, ["a"])]),                 # best time, first-round trip in the zone: 1.0
    ("no_bonus", 40, [-1, -1, 0, -1, -1, -1], [(28, ["a"])]),              # trip elsewhere: half score
    ("two_zones", 40, [0, -1, -1, -1, -1, -1], [(30, ["a", "c"])]),        # two zones: half score, no bonus
    ("later_round", 40, [1, -1, 0, -1, -1, -1], [(31, ["a"])]),            # the zone's line tripped in round 1: no bonus
    ("too_early", 40, [0, -1, -1, -1, -1, -1], [(16, ["a"])]),             # dist = best + W: 0, not used
    ("too_late", 40, [0, -1, -1, -1, -1, -1], [(40, ["a"])]),              # dist = 0 = best - W: 0, not used
    ("inside_early", 40, [0, -1, -1, -1, -1, -1], [(17, ["a"]), (39, ["b"])]),
    ("shared_line", 40, [-1, 0, -1, -1, -1, -1], [(30, ["b"])]),           # line 1 is in "a" and "b"
    ("best_of_many", 60, [-1, -1, -1, -1, 0, 2], [(37, ["c"]), (46, ["c"]), (48, ["a", "b"]), (50, ["c"])]),
    ("no_trip", 40, [-1] * 6, [(28, ["a"])]),                              # -1, is_alarm_used unchanged
    ("no_alarm", 40, [0, -1, -1, -1, -1, -1], []),                         # -1, is_alarm_used unchanged
]


def test_alarm_reward_branches_equal_reference():
    """AlarmReward.__call__ (grid2op) on every branch against BatchedAlarms and the host build of the device body, in one sequence
    on one instance so that the sticky is_alarm_used carries over from case to case (and over reset)"""
    import grid2op_b200.backend  # noqa: F401
    from grid2op.Reward import AlarmReward
    from alarm_emu import AlarmArgs, _lib
    import ctypes as C
    from grid2op_b200.alarm import BatchedAlarms
    names = ["a", "b", "c"]
    mask = np.array([1, 3, 2, 2, 4, 4], np.uint32)
    ref = AlarmReward()
    ref.best_time, ref.window_size = np.int32(12), np.int32(12)
    mine = BatchedAlarms(mask, 3, 1, best_time=12, window_size=12)
    lib = _lib()
    lib.alarm_emu_reward.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    emu = {k: v.copy() for k, v in mine.get_state().items()}
    emu["zone_mask"], emu["raise_"], emu["reward_out"] = mask.copy(), np.zeros((1, 3), np.uint8), np.zeros(1, np.float64)
    am = AlarmArgs(n=3, n_line=6, best_time=12, window=12, ring=24, reward=1)
    for nm, arr in emu.items():
        setattr(am, nm, arr.ctypes.data)
    seen = {}
    for name, step, disc, alarms in CASES:
        mine.reset([0])                                    # (keeps is_alarm_used, as the host build's state does)
        for arr in ("ring_step", "ring_mask", "any_ok"):
            emu[arr][:] = 0
        for s, zs in alarms:
            m = sum(1 << names.index(z) for z in zs)
            mine.s["ring_step"][0, s % 24], mine.s["ring_mask"][0, s % 24], mine.s["any_ok"][0] = s, m, 1
            emu["ring_step"][0, s % 24], emu["ring_mask"][0, s % 24], emu["any_ok"][0] = s, m, 1
        env = _Env(names, mask, step, disc, [(s, np.isin(names, zs)) for s, zs in alarms])
        want = ref(None, env, True, True, False, False)
        got = mine._reward_instance(0, step, np.asarray(disc, np.int32))
        d = np.ascontiguousarray(disc, np.int32)
        assert lib.alarm_emu_reward(C.byref(am), 0, step, d.ctypes.data) == 0
        assert got == want == emu["reward_out"][0], (name, got, want, emu["reward_out"][0])
        assert bool(mine.s["used"][0]) == bool(ref.is_alarm_used) == bool(emu["used"][0]), name
        seen[name] = (float(want), bool(ref.is_alarm_used))
    assert seen["bonus"] == (1.0, True) and seen["no_bonus"] == (0.5, True) and seen["two_zones"][0] == pytest.approx(0.5 * (1 - 4 / 144))
    assert seen["later_round"][0] < 0.5 and seen["too_early"] == (-1.0, False) and seen["too_late"] == (-1.0, False)
    assert seen["inside_early"][1] and seen["shared_line"][0] > 0.9
    # the early returns keep the flag of the case before: set it True first, then both -1 branches
    assert seen["best_of_many"][1] and seen["no_trip"] == (-1.0, True) and seen["no_alarm"] == (-1.0, True)


def test_register_and_reset_keep_the_used_flag():
    """LinearAttentionBudget.register_action restated: cap, refusal, one charge for several zones, an illegal action; reset keeps
    AlarmReward.is_alarm_used"""
    from grid2op_b200.alarm import BatchedAlarms
    a = BatchedAlarms(np.ones(4, np.uint32), 2, 3, max_budget=3.0, budget_per_ts=0.5, alarm_cost=1.0, init_budget=2.0)
    live, ill, go = np.ones(3, bool), np.zeros(3, bool), np.zeros(3, bool)
    up = np.array([[1, 1], [0, 0], [1, 0]], bool)
    a.step(up, live, np.array([False, False, True]), np.full(3, 1), go, None)
    s = a.get_state()
    assert list(s["budget"]) == [1.0, 2.5, 2.0] and list(s["time_last_ok"]) == [1, -1, -1] and list(s["last_ok"][0]) == [1, 1]
    for t in (2, 3):
        a.step(np.zeros((3, 2), bool), live, ill, np.full(3, t), go, None)
    assert list(a.s["budget"]) == [2.0, 3.0, 3.0]
    a.s["budget"][0] = 0.5
    a.step(up, live, ill, np.full(3, 4), go, None)
    assert list(a.s["illegal"]) == [1, 0, 0] and a.s["time_last"][0] == 4 and a.s["time_last_ok"][0] == 1 and list(a.s["last"][0]) == [4, 4]
    a.s["used"][:] = 1
    a.reset([0, 2])
    assert list(a.s["used"]) == [1, 1, 1] and a.s["budget"][0] == 2.0 and a.s["time_last"][0] == -1 and not a.s["ring_step"][0].any()


# ---- zones and validation ----------------------------------------------------------------------------------------------------
def test_load_alarm_zones_equal_reference():
    if env_grid(ENV) is None:
        pytest.skip("reference data not available")
    from test_geometric_opponent_cpu import _make
    from grid2op_b200.alarm import load_alarm_zones
    from grid2op_b200.gridmodel import GridModel
    grid = env_grid(ENV)
    names, mask = load_alarm_zones(os.path.dirname(grid), GridModel(grid))
    e = _make(ENV, "alarmzones")
    assert names == list(e.alarms_area_names)
    for j, ln in enumerate(e.name_line):
        assert [names[z] for z in range(len(names)) if (int(mask[j]) >> z) & 1] == sorted(e.alarms_lines_area[ln]), ln
    assert sum(len(v) for v in e.alarms_area_lines) == sum(bin(int(m)).count("1") for m in mask)
    e.close()


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


def three_zones(gm):
    """a synthetic "fixed" alerts_info.json for case14: three zones over the lines, line 0 in two of them"""
    names = [str(x) for x in gm.name_line]
    return {"fixed": {"z_north": names[:8], "z_mid": names[0:1] + names[8:14], "z_south": names[14:]}}


@pytest.mark.parametrize("content,err", [
    ({"fixed": {"a": ["no such line"]}}, "not in the grid"),
    ("first_only", "in no zone"),
    ({"something": 1}, "no \"fixed\""),
    ({"by_line": "opponent"}, "no \"fixed\""),
    ("many", "at most 32"),
    (None, "no alerts_info.json"),
])
def test_load_alarm_zones_rejected(tmp_path, content, err):
    from grid2op_b200.alarm import load_alarm_zones
    gm = _small_env().gm
    names = [str(x) for x in gm.name_line]
    if content == "first_only":
        content = {"fixed": {"a": names[:3]}}
    elif content == "many":
        content = {"fixed": {f"z{k:02d}": names for k in range(33)}}
    if content is not None:
        (tmp_path / "alerts_info.json").write_text(json.dumps(content))
    with pytest.raises(ValueError, match=err):
        load_alarm_zones(str(tmp_path), gm)


@pytest.mark.parametrize("kw", [dict(alarm_best_time=0), dict(alarm_window_size=-1), dict(alarm_best_time=1000, alarm_window_size=25),
                                dict(zones="no_line"), dict(zones="past_n"), dict(alerts=True)])
def test_enable_alarms_rejected(tmp_path, kw):
    from grid2op_b200.alarm import load_alarm_zones
    benv = _small_env()
    (tmp_path / "alerts_info.json").write_text(json.dumps(three_zones(benv.gm)))
    names, mask = load_alarm_zones(str(tmp_path), benv.gm)
    kw = dict(kw)
    z = kw.pop("zones", None)
    if z == "no_line":
        mask = mask.copy(); mask[3] = 0
    elif z == "past_n":
        mask = mask.copy(); mask[3] = 8
    if kw.pop("alerts", False):
        benv.enable_alerts([0, 1])
    with pytest.raises(ValueError):
        benv.enable_alarms((names, mask), **kw)
    assert benv._alarms is None


def test_enable_alarms_widths_order_and_raise_alarm_checked(tmp_path):
    from grid2op_b200.alarm import load_alarm_zones
    from grid2op_b200.observation import attr_sizes, obs_spec
    benv = _small_env(B=3)
    gm = benv.gm
    assert attr_sizes(gm) == attr_sizes(gm, 0, 0) and attr_sizes(gm, 0, 3)["last_alarm"] == 3
    assert obs_spec(gm, None, 0, 3)[1] == obs_spec(gm)[1] + 3
    (tmp_path / "alerts_info.json").write_text(json.dumps(three_zones(gm)))
    zones = load_alarm_zones(str(tmp_path), gm)
    assert zones[0] == ["z_mid", "z_north", "z_south"] and zones[1][0] == 3
    with pytest.raises(ValueError):
        benv.step(raise_alarm=np.zeros((3, 3), bool))                     # no alarms enabled
    assert benv.enable_alarms(zones) == 3
    with pytest.raises(ValueError):
        benv.enable_alerts([0, 1])
    benv.reset_step()
    with pytest.raises(ValueError):
        benv.step(raise_alarm=np.zeros((3, 2), bool))
    n0 = benv.n_steps
    _, _, info = benv.step(raise_alarm=np.array([[1, 1, 0], [0, 0, 0], [0, 0, 1]], bool))
    st = benv.alarm_state()
    assert benv.n_steps == n0 + 1 and list(st["budget"]) == [1.0, np.float32(2.0) + np.float32(1 / 192), 1.0]
    assert info["rewards"]["alarm"].dtype == np.float64 and info["is_alarm_illegal"].dtype == bool
    benv._obs = {}                                         # (as enable_observation leaves it)
    with pytest.raises(RuntimeError):
        benv.enable_alarms(zones)
