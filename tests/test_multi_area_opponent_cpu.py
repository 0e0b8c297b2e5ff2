"""BatchedEnv's GeometricOpponentMultiArea (grid2op_b200/opponent.py, csrc/b200pf_opp.cuh) on the CPU:

* after ``env.seed(s); env.reset()`` and further OpponentSpace resets, every area's schedule and stream equal those of the
  ``list_opponents[k]`` of an unmodified l2rpn_idf_2023 environment, on the numpy path and in the host build of the device draws;
* the numpy path next to unmodified l2rpn_idf_2023 environments (host logic on both sides), with shortened hours and a small budget:
  attacks in several areas at once, combined attacks refused for budget whose lines come back later, attacks lost to the
  ``~status.all()`` test, a ``previous_fails`` that moves an area's next attack and schedules that run out.  The host build of the
  device body (tests/emu/multi_emu.cpp) runs next to it and must agree bit for bit;
* the ValueError cases, and the unmodified environment raising at ``opponent_attack_cooldown=2``, the reason that cooldown is refused.
"""
import os
import warnings

import numpy as np
import pytest

from conftest import env_grid

ENV = "l2rpn_idf_2023"
# shortened hours (5-minute steps): hazard 1/9, recovery 1/6 over a 3-step minimum
SHORT = dict(attack_every_xxx_hour=1.5, average_attack_duration_hour=0.75, minimum_attack_duration_hour=0.25)


def _make(tag, **kw):
    from test_geometric_opponent_cpu import _host_logic_backend
    import grid2op_b200.backend  # noqa: F401  (locates / bootstraps the grid2op install first)
    import grid2op
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return grid2op.make(ENV, test=True, backend=_host_logic_backend()(), _add_to_name=tag, **kw)


def _areas(env):
    names = list(env.name_line)
    return [[names.index(x) for x in a] for a in env._kwargs_opponent["lines_attacked"]]


def _geo_kw(env, **over):
    kwo = dict(env._kwargs_opponent, **over)
    return {k: kwo[k] for k in ("attack_every_xxx_hour", "average_attack_duration_hour", "minimum_attack_duration_hour", "pmax_pmin_ratio")}


# ---- seeds and schedules ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hours", [None, SHORT])
def test_area_schedules_equal_reference(hours):
    if env_grid(ENV) is None:
        pytest.skip("reference data not available")
    from geo_emu import GeoDraws
    from grid2op_b200.opponent import AREA_COUNTER, AREA_N, AREA_OVERFLOW, BatchedOpponent, opponent_seed
    kw = {}
    if hours is not None:
        e0 = _make("mas0")
        kw = dict(kwargs_opponent=dict(e0._kwargs_opponent, **hours))
        e0.close()
    e = _make(f"mas{hours is None}", **kw)
    areas = _areas(e)
    assert [len(a) for a in areas] == [6, 10, 6]
    max_seed = np.iinfo(np.int32).max
    for s in (0, 5, 77, 2 ** 31 - 2):
        got = e.seed(s)[6]
        top = np.random.RandomState(opponent_seed(s))
        area_seeds = [top.randint(max_seed) for _ in areas]
        assert got == (opponent_seed(s), [(x,) for x in area_seeds]), s
        e.reset()
        mo = e._oppSpace.opponent
        emt = int(mo.list_opponents[0]._episode_max_time)
        assert emt == int(e.max_episode_duration()) == 575
        bo = BatchedOpponent("GeometricOpponentMultiArea", areas, 1, attack_duration=96, attack_cooldown=0, budget_per_ts=0.51,
                             init_budget=1000.0, seeds=[opponent_seed(s)], delta_time_seconds=e.delta_time_seconds, episode_max_time=emt,
                             **_geo_kw(e))
        draws = [GeoDraws(x) for x in area_seeds]
        for r in range(3):
            if r:
                e._oppSpace.reset()
                bo.reset([0])
            st = bo.get_state()
            assert list(mo._new_attack_time_counters) == [-1, -1, -1]
            for k, op in enumerate(mo.list_opponents):
                n = int(op._number_of_attacks)
                w, d = np.asarray(op._attack_waiting_times), np.asarray(op._attack_durations)
                assert st["multi_ctr"][0, k, AREA_N] == n and st["multi_ctr"][0, k, AREA_COUNTER] == 0, (s, r, k)
                assert st["multi_ctr"][0, k, AREA_OVERFLOW] == 0
                assert np.array_equal(w, st["multi_wait"][0, k, :n]) and np.array_equal(d, st["multi_dur"][0, k, :n]), (s, r, k)
                ps = op.space_prng.get_state()
                assert np.array_equal(ps[1], st["multi_mt"][0, k]) and ps[2] == st["multi_mt_pos"][0, k], (s, r, k)
                dw, dd, dropped = draws[k].schedule(bo.hazard_rate, bo.recovery_rate, bo.recovery_min, emt, bo.cap)
                assert dropped == 0 and np.array_equal(dw, w) and np.array_equal(dd, d), (s, r, k)
                assert np.array_equal(draws[k].mt, ps[1]) and draws[k].pos[0] == ps[2], (s, r, k)
    e.close()


# ---- against unmodified grid2op environments -------------------------------------------------------------------------------
def _ref_area_state(op_multi):
    """per area: (attacks consumed, _next_attack_time or the device's None, _new_attack_time_counters)"""
    from grid2op_b200.opponent import NEXT_UNSET
    return [(int(op._attack_counter), NEXT_UNSET if op._next_attack_time is None else int(op._next_attack_time),
             int(op_multi._new_attack_time_counters[k])) for k, op in enumerate(op_multi.list_opponents)]


def run_multi_vs_reference(n_steps, seeds, attack_cooldown, engine_factory, emu: bool, backend_class=None, check_rho_tol=(2e-4, 2e-5),
                           schedule_steps=None):
    """steps unmodified l2rpn_idf_2023 environments (GeometricOpponentMultiArea on, shortened hours, a small budget) and BatchedEnv
    (``enable_opponent`` with the same constants) side by side; -> what the run saw.  Each instance gets the maintenance its
    reference environment generated; ``schedule_steps``: the episode length the first schedules are drawn for (as in
    tests/test_geometric_opponent_cpu.py), so that schedules run out within the run"""
    import grid2op_b200.backend  # noqa: F401
    import grid2op
    from grid2op.Parameters import Parameters
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import list_scenarios, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    from grid2op_b200.opponent import AREA_CLOCK, AREA_COUNTER, AREA_NEXT, opponent_seed
    from test_batched_env import _scripted
    from test_geometric_opponent_cpu import _host_logic_backend
    grid = env_grid(ENV)
    gm = GridModel(grid)
    cdir = os.path.join(os.path.dirname(grid), "chronics")
    folder = list_scenarios(cdir)[0]
    chron = load_scenarios(cdir, gm, scenarios=[folder])
    B = len(seeds)
    p = Parameters()
    p.NO_OVERFLOW_DISCONNECTION = True
    p.NB_TIMESTEP_COOLDOWN_LINE = 3
    p.NB_TIMESTEP_COOLDOWN_SUB = 2
    backend_class = backend_class or _host_logic_backend()
    e0 = _make("maskw")
    kwo = dict(e0._kwargs_opponent, **SHORT)
    e0.close()
    envs = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for i in range(B):
            e = grid2op.make(ENV, test=True, backend=backend_class(), param=p, _add_to_name=f"ma{i}", kwargs_opponent=kwo,
                             opponent_init_budget=3.0, opponent_budget_per_ts=0.5, opponent_attack_cooldown=attack_cooldown)
            if schedule_steps is not None:
                e.set_max_iter(schedule_steps)
                e.reset()
                e.set_max_iter(-1)
            e.seed(int(seeds[i]))
            e.set_id(0)
            e.reset()
            envs.append(e)
    sp = envs[0]._oppSpace
    assert type(sp.opponent).__name__ == "GeometricOpponentMultiArea"
    emt = int(sp.opponent.list_opponents[0]._episode_max_time) if schedule_steps is None else schedule_steps
    th = np.asarray(envs[0].get_thermal_limit(), dtype=np.float32)
    maint = np.stack([np.asarray(e.chronics_handler.real_data.data.maintenance, dtype=bool) for e in envs])
    assert maint.shape == (B, chron.shape[1], gm.n_line)
    benv = BatchedEnv(gm, np.repeat(chron, B, axis=0), B, maintenance=maint, scen=np.arange(B, dtype=np.int32),
                      t0=np.zeros(B, np.int32), thermal_limit_a=th, nb_timestep_cooldown_line=3, nb_timestep_cooldown_sub=2,
                      nb_timestep_reconnection=p.NB_TIMESTEP_RECONNECTION, protections=False, engine=engine_factory(gm))
    rho, _, _ = benv.reset_step()
    obs = [e.get_obs() for e in envs]
    for i in range(B):
        assert np.array_equal(obs[i].topo_vect, benv.topo[i, :gm.dim_topo])
    benv.enable_opponent("GeometricOpponentMultiArea", kwo["lines_attacked"], attack_duration=sp.attack_max_duration,
                         attack_cooldown=sp.attack_cooldown, budget_per_ts=sp.budget_per_timestep, init_budget=sp.init_budget,
                         seeds=[opponent_seed(int(s)) for s in seeds], delta_time_seconds=envs[0].delta_time_seconds,
                         episode_max_time=emt, **_geo_kw(envs[0], **SHORT))
    o = benv._opp
    area_of = np.full(gm.n_line, -1)
    for k in range(len(o.area_off) - 1):
        area_of[o.lines[o.area_off[k]:o.area_off[k + 1]]] = k
    em = None
    if emu:
        from multi_emu import EmuMultiEnvState
        em = EmuMultiEnvState(benv)
    att = [int(x) for x in o.lines]
    rngs = [np.random.default_rng(100 + int(s)) for s in seeds]
    is_line_pos = np.zeros(gm.dim_topo, dtype=bool)
    is_line_pos[gm.line_or_pos] = True; is_line_pos[gm.line_ex_pos] = True
    saw = dict(attack_steps=0, multi_line=0, refused_budget=0, refused_returned=0, lost_status=0, fails_wait=0, schedule_end=0,
               illegal=0)
    alive = np.ones(B, dtype=bool)
    refused = [set() for _ in range(B)]
    ended = np.zeros(B, dtype=bool)
    for k in range(n_steps):
        sub_id = np.full(B, -1, np.int64); sub_bus = np.zeros((B, benv.max_sub_size), np.int8)
        line_id = np.full(B, -1, np.int64); line_st = np.zeros(B, np.int64)
        ref = []
        for i, e in enumerate(envs):
            if not alive[i]:
                ref.append(None)
                continue
            ob = obs[i]
            # one substation or one line per step, never a reconnection through set_bus: RulesByArea and DefaultRules agree
            a = _scripted(k, rngs[i], ob.topo_vect, ob.line_status, ob.time_before_cooldown_line, ob.time_before_cooldown_sub,
                          benv.sub_pos, benv.sub_size, gm.n_line, is_line_pos)
            out = [l for l in att if not ob.line_status[l] and ob.time_before_cooldown_line[l] == 0]
            if k % 2 == 0 and out:
                a = dict(sub=-1, bus=None, line=int(out[0]), status=1)          # reconnect an attackable line (lets attacks land)
            elif k % 16 == 9:
                a = dict(sub=-1, bus=None, line=att[(k // 16 * 5 + i) % len(att)], status=-1)   # an attackable line out: attacks get lost
            spec = {}
            if a["sub"] >= 0:
                spec["set_bus"] = {"substations_id": [(a["sub"], a["bus"].astype(int).tolist())]}
                sub_id[i] = a["sub"]; sub_bus[i, :len(a["bus"])] = a["bus"]
            if a["line"] >= 0:
                spec["set_line_status"] = [(a["line"], int(a["status"]))]
                line_id[i] = a["line"]; line_st[i] = a["status"]
            mo = e._oppSpace.opponent
            before = (_ref_area_state(mo), e._oppSpace.previous_fails)
            o2, r, d, info = e.step(e.action_space(spec))
            obs[i] = o2
            ref.append((d, info, before, _ref_area_state(mo), e._oppSpace.previous_fails, e._oppSpace.budget))
        prev_rho = benv.engine.series_fetch(want_out=False)[3]
        if em is not None:
            ctl = em.step_apply(sub_id, sub_bus, line_id, line_st, rho=prev_rho)
            assert ctl[2] == 0
        rho, done, binfo = benv.step(sub_id, sub_bus, line_id, line_st)
        if em is not None:
            _, status, _, _ = benv.engine.series_fetch(want_out=False)
            em.step_post(status, None, stamp=benv.n_steps)
            st = benv.opponent_state()
            for key, v in em.opponent_state().items():
                assert np.array_equal(v, st[key]), (k, key)
            assert np.array_equal(em.mst["attack_lines"], binfo["opponent_attack_line"]), k
            assert np.array_equal(em.ost["attack_dur"], binfo["opponent_attack_duration"]), k
            assert np.array_equal(em.st["topo"], benv.topo) and np.array_equal(em.st["line_cd"], benv.line_cooldown), k
            assert np.array_equal(em.st["sub_cd"], benv.sub_cooldown) and np.array_equal(em.st["is_illegal"], benv.is_illegal), k
        st = o.get_state()
        for i in range(B):
            if not alive[i]:
                continue
            d, info, (areas0, fails0), areas1, fails, budget = ref[i]
            assert bool(done[i]) == bool(d), (k, i, info["exception"])
            if d:
                alive[i] = False
                continue
            ob = obs[i]
            mo = envs[i]._oppSpace.opponent
            la = info["opponent_attack_line"]
            want = set() if la is None else set(np.flatnonzero(la).tolist())
            got = binfo["opponent_attack_line"][i]
            assert set(int(x) for x in got if x >= 0) == want, (k, i, got, want)
            assert all(x < 0 or area_of[x] == a for a, x in enumerate(got)), (k, i, got)
            assert binfo["opponent_attack_duration"][i] == (info["opponent_attack_duration"] if la is not None else 0), (k, i)
            assert bool(binfo["is_illegal"][i]) == bool(info["is_illegal"]), (k, i)
            saw["illegal"] += bool(info["is_illegal"])
            b = o.budget[i]
            assert b.dtype == np.asarray(budget).dtype and b == budget, (k, i, b, budget)
            assert bool(st["multi_fails"][i]) == bool(fails), (k, i)
            for a, (c, nxt, clock) in enumerate(areas1):
                assert (st["multi_ctr"][i, a, AREA_COUNTER], st["multi_ctr"][i, a, AREA_NEXT], st["multi_ctr"][i, a, AREA_CLOCK]) == \
                    (c, nxt, clock), (k, i, a, st["multi_ctr"][i, a], (c, nxt, clock))
            assert np.array_equal(ob.topo_vect, benv.topo[i, :gm.dim_topo]), (k, i)
            assert np.array_equal(ob.line_status, benv.line_status()[i]), (k, i)
            assert np.array_equal(ob.time_before_cooldown_line, benv.line_cooldown[i]), (k, i)
            assert np.array_equal(ob.time_before_cooldown_sub, benv.sub_cooldown[i]), (k, i)
            assert np.allclose(ob.rho, rho[i], rtol=check_rho_tol[0], atol=check_rho_tol[1]), (k, i)
            # what the step showed
            if want:
                saw["attack_steps"] += 1
                saw["multi_line"] += len(want) >= 2
                if want & refused[i]:
                    saw["refused_returned"] += 1
                    refused[i] -= want
            if fails:
                wanted = {int(mo._previous_attacks[a].line_set_status.argmin()) for a in range(len(areas1))
                          if areas1[a][2] >= 0 and mo._previous_attacks[a] is not None}
                if wanted:
                    saw["refused_budget"] += 1
                    refused[i] |= wanted
            for a, ((c0, _, clock0), (c1, _, clock1)) in enumerate(zip(areas0, areas1)):
                op = mo.list_opponents[a]
                if c1 > c0 and clock1 == -1:
                    saw["lost_status"] += 1                            # consumed, not launched: an area line was out
                if fails0 and clock0 <= 0 and c0 < op._number_of_attacks:
                    saw["fails_wait"] += 1                             # an area asked after a refusal: its next attack moved
            if any(c1 >= mo.list_opponents[a]._number_of_attacks for a, (c1, _, _) in enumerate(areas1)) and not ended[i]:
                ended[i] = True
                saw["schedule_end"] += 1
    saw["alive"] = int(alive.sum())
    for e in envs:
        e.close()
    benv.close()
    return saw


@pytest.mark.parametrize("attack_cooldown,seeds", [(0, (0, 3, 5)), (1, (1, 2, 6))])
def test_multi_area_opponent_vs_reference_env_host_logic(attack_cooldown, seeds):
    if env_grid(ENV) is None:
        pytest.skip("reference data not available")
    from oracle_engine import COracleSeriesEngine
    saw = run_multi_vs_reference(150, seeds, attack_cooldown, engine_factory=COracleSeriesEngine, emu=True, schedule_steps=80)
    assert all(saw[k] > 0 for k in ("attack_steps", "multi_line", "refused_budget", "refused_returned", "lost_status", "fails_wait",
                                    "schedule_end")), saw


# ---- validation ------------------------------------------------------------------------------------------------------------
_OK = dict(attack_duration=96, attack_cooldown=0, budget_per_ts=0.51, init_budget=1000.0, seeds=[0, 1], episode_max_time=575,
           attack_every_xxx_hour=32, average_attack_duration_hour=2, minimum_attack_duration_hour=1)


def test_multi_area_accepts_idf_configuration():
    from grid2op_b200.opponent import BatchedOpponent
    for cd in (0, 1):
        bo = BatchedOpponent("GeometricOpponentMultiArea", [[0, 1, 2], [3], [4, 5]], 2, **dict(_OK, attack_cooldown=cd))
        assert bo.multi and list(bo.area_off) == [0, 3, 4, 6] and len(bo.area_weights) == 6
        assert np.array_equal(bo.area_weights[3:4], [1.0])                     # a one-line area: b_beta 0


@pytest.mark.parametrize("areas,over", [
    ([[0, 1], [2, 3]], dict(attack_cooldown=2)),                               # grid2op's own opponent raises (see below)
    ([[0, 1], [2, 3]], dict(attack_cooldown=12)),
    ([[0, 1], []], {}),                                                        # an empty area
    ([[0, 1], [1, 2]], {}),                                                    # two areas share a line
    ([[k] for k in range(9)], {}),                                             # more than 8 areas
    ([list(range(0, 40)), list(range(40, 65))], {}),                           # more than 64 lines
    ([], {}),                                                                  # no area
    ([[0, 1], [2, 3]], dict(average_attack_duration_hour=1)),                  # the GeometricOpponent's own errors
    ([[0, 1], [2, 3]], dict(attack_every_xxx_hour=2)),
    ([[0, 1], [2, 3]], dict(attack_every_xxx_hour=1e8)),
    ([[0, 1], [2, 3]], dict(pmax_pmin_ratio=0)),
    ([[0, 1], [2, 3]], dict(episode_max_time=None)),
])
def test_multi_area_rejected(areas, over):
    from grid2op_b200.opponent import BatchedOpponent
    with pytest.raises(ValueError):
        BatchedOpponent("GeometricOpponentMultiArea", areas, 2, **dict(_OK, **over))


def test_reference_raises_at_cooldown_2():
    """with opponent_attack_cooldown=2 OpponentSpace skips a step after two attacks and calls the multi-area opponent's
    tell_attack_continues, which raises: the configuration BatchedOpponent refuses"""
    if env_grid(ENV) is None:
        pytest.skip("reference data not available")
    e0 = _make("macd0")
    kwo = dict(e0._kwargs_opponent, **SHORT)
    e0.close()
    for cd, raises in ((2, True), (1, False)):
        e = _make(f"macd{cd}", kwargs_opponent=kwo, opponent_attack_cooldown=cd)
        e.seed(0)
        e.reset()
        got = None
        for _ in range(150):
            try:
                _, _, done, _ = e.step(e.action_space())
            except RuntimeError as err:
                got = err
                break
            if done:
                e.reset()
        e.close()
        assert (got is not None and "should not get there" in str(got)) == raises, (cd, got)
