"""BatchedEnv's GeometricOpponent (grid2op_b200/opponent.py, csrc/b200pf_opp.cuh) on the CPU:

* the host build of the device draws (tests/emu/geo_emu.cpp, libm's log1p) is bit-equal to ``RandomState.geometric`` on both of
  numpy's branches, many seeds and across the 624-word twist;
* the schedules of the numpy path and of the host build equal those of unmodified l2rpn_wcci_2022_dev / l2rpn_icaps_2021
  environments after ``seed(s); reset()`` and after further resets, with their own kwargs and with shortened hours;
* ranks + weight table + choice equal ``GeometricOpponent.attack`` for every number of attackable lines from 1 to 64;
* ``opponent_seed(s)`` is the opponent's seed of ``env.seed(s)`` on both environments;
* the numpy path next to unmodified environments with their GeometricOpponent on (host logic on both sides), with attacks, refusals
  for budget and for a duration above ``attack_max_duration``, attacks lost to the ``~status.all()`` test and schedules that run
  out; the host build of the device body runs next to it and must agree bit for bit;
* the ValueError cases of the constants.
"""
import os
import warnings

import numpy as np
import pytest

from conftest import env_grid

ENVS = ["l2rpn_wcci_2022_dev", "l2rpn_icaps_2021"]
# shortened hours (5-minute steps): hazard 1/9 and recovery 1/6 (inversion), hazard 1/3 (search) and recovery 1/2 (search)
SHORT = [dict(attack_every_xxx_hour=1.5, average_attack_duration_hour=0.75, minimum_attack_duration_hour=0.25),
         dict(attack_every_xxx_hour=0.5, average_attack_duration_hour=0.25, minimum_attack_duration_hour=1 / 12)]


def _host_logic_backend():
    import grid2op_b200.backend as bk
    from oracle_engine import OracleEngine

    class HostLogicBackend(bk.B200Backend):
        def _make_engine(self, gm):
            return OracleEngine(gm)
    return HostLogicBackend


def _make(name, tag, **kw):
    import grid2op_b200.backend  # noqa: F401  (locates / bootstraps the grid2op install first)
    import grid2op
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return grid2op.make(name, test=True, backend=_host_logic_backend()(), _add_to_name=tag, **kw)


def _geo_kw(env, **over):
    kwo = dict(env._kwargs_opponent)
    kwo.update(over)
    return {k: kwo[k] for k in ("attack_every_xxx_hour", "average_attack_duration_hour", "minimum_attack_duration_hour")}


# ---- draws -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [1 / 240, 1 / 36, 1 / (12 * 0.25), 0.5, 0.9])
def test_geometric_bit_equal_to_randomstate(p):
    from geo_emu import GeoDraws
    for seed in range(0, 4000, 61):
        d, r = GeoDraws(seed), np.random.RandomState(seed)
        got = d.geometric(p, 1500)                                       # (> 624 words: crosses the twist)
        want = np.array([r.geometric(p) for _ in range(1500)])
        assert np.array_equal(got, want), (seed, p)
        st = r.get_state()
        assert d.pos[0] == st[2] and np.array_equal(d.mt, st[1]), (seed, p)


# ---- schedules -------------------------------------------------------------------------------------------------------------
def _sched(op):
    return (np.asarray(op._attack_waiting_times), np.asarray(op._attack_durations), int(op._number_of_attacks))


@pytest.mark.parametrize("name", ENVS)
@pytest.mark.parametrize("hours", [None, 0, 1])
def test_schedules_equal_reference(name, hours):
    if env_grid(name) is None:
        pytest.skip("reference data not available")
    from geo_emu import GeoDraws
    from grid2op_b200.opponent import BatchedOpponent, opponent_seed
    kw = {}
    if hours is not None:
        e0 = _make(name, "geos0")
        kwo = dict(e0._kwargs_opponent, **SHORT[hours])
        e0.close()
        kw = dict(kwargs_opponent=kwo)
    e = _make(name, f"geos{hours}", **kw)
    g = _geo_kw(e)
    for s in (0, 5, 77):
        e.seed(s)
        e.reset()
        op = e._oppSpace.opponent
        emt = int(op._episode_max_time)
        assert emt == int(e.max_episode_duration())
        bo = BatchedOpponent("GeometricOpponent", [0, 1], 1, attack_duration=96, attack_cooldown=12, budget_per_ts=0.17, init_budget=144.0,
                             seeds=[opponent_seed(s)], delta_time_seconds=e.delta_time_seconds, episode_max_time=emt, **g)
        dr = GeoDraws(opponent_seed(s))
        # seed + reset, then two more OpponentSpace resets on the continuing stream (env.reset() would first re-seed the opponent
        # from the environment's own stream, which BatchedEnv.reset_instances does not restate for any opponent)
        for r in range(3):
            if r:
                e._oppSpace.reset()
                bo.reset([0])
            w, d, n = _sched(op)
            st = bo.get_state()
            assert n == st["geo_ctr"][0, 0] and st["geo_ctr"][0, 3] == 0, (s, r)
            assert np.array_equal(w, st["geo_wait"][0, :n]) and np.array_equal(d, st["geo_dur"][0, :n]), (s, r)
            assert w.dtype == np.int32 and d.dtype == np.int32
            dw, dd, dropped = dr.schedule(bo.hazard_rate, bo.recovery_rate, bo.recovery_min, emt, bo.cap)
            assert dropped == 0 and np.array_equal(dw, w) and np.array_equal(dd, d), (s, r)
            assert np.array_equal(dr.mt, st["mt"][0]) and dr.pos[0] == st["mt_pos"][0], (s, r)
            assert np.array_equal(op.space_prng.get_state()[1], st["mt"][0]), (s, r)
    e.close()


def test_schedule_cap_drops_and_counts():
    """a cap below the schedule's length writes nothing past it and counts what it dropped; the stream stays numpy's"""
    from geo_emu import GeoDraws
    from grid2op_b200.opponent import BatchedOpponent
    bo = BatchedOpponent("GeometricOpponent", [0, 1], 1, attack_duration=10, attack_cooldown=1, budget_per_ts=1.0, init_budget=1.0,
                         seeds=[3], episode_max_time=2000, **SHORT[1])
    n = int(bo.get_state()["geo_ctr"][0, 0])
    assert 3 < n <= bo.cap
    d = GeoDraws(3)
    w0, d0, dropped = d.schedule(bo.hazard_rate, bo.recovery_rate, bo.recovery_min, 2000, 3)
    assert dropped == n - 3 and np.array_equal(w0, bo.get_state()["geo_wait"][0, :3])
    assert np.array_equal(d.mt, bo.get_state()["mt"][0]) and d.pos[0] == bo.get_state()["mt_pos"][0]


# ---- the choice ------------------------------------------------------------------------------------------------------------
class _Obs:
    def __init__(self, n, rho):
        self.line_status = np.ones(n, dtype=bool)
        self.rho = rho


def test_choice_equal_geometric_opponent_attack():
    import grid2op_b200.backend  # noqa: F401
    from grid2op.Opponent import GeometricOpponent
    from geo_emu import GeoDraws
    g = np.random.default_rng(5)
    for n in range(1, 65):
        b_beta = np.log(4) / (n - 1) if n > 1 else 0.0
        table = np.exp(b_beta * np.arange(n, dtype=np.int64))
        for seed in range(0, 40, 3):
            rho = g.permutation(g.random(n).astype(np.float32) * 1.5)     # distinct values, random order
            if len(np.unique(rho)) != n:
                continue
            op = object.__new__(GeometricOpponent)
            op.space_prng = np.random.RandomState(seed)
            op._lines_ids, op._attacks, op._pmax_pmin_ratio = np.arange(n), np.arange(n), 4
            op._attack_counter, op._number_of_attacks, op._next_attack_time = 0, 1, None
            op._attack_waiting_times, op._attack_durations = np.array([0], np.int32), np.array([5], np.int32)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                want, wdur = op.attack(_Obs(n, rho), None, None, 10.0, False)
            d = GeoDraws(seed)
            line, dur = d.attack(rho, table)
            assert line == int(want) and dur == int(wdur) == 5, (n, seed, line, want)
            st = op.space_prng.get_state()
            assert d.pos[0] == st[2] and np.array_equal(d.mt, st[1]), (n, seed)


# ---- seeds -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ENVS)
def test_opponent_seed_is_env_seed(name):
    if env_grid(name) is None:
        pytest.skip("reference data not available")
    from grid2op_b200.opponent import opponent_seed
    e = _make(name, "geoseed")
    for s in (0, 1, 7, 123, 2 ** 31 - 2):
        assert e.seed(s)[6] == (opponent_seed(s),), s
    e.close()


# ---- against unmodified grid2op environments ---------------------------------------------------------------------------------
def run_geometric_vs_reference(name, n_steps, make_kw, seeds, engine_factory, emu: bool, backend_class=None, check_rho_tol=(2e-4, 2e-5),
                               schedule_steps=None):
    """steps B unmodified environments (GeometricOpponent on, ``make_kw`` overrides) and BatchedEnv (``enable_opponent`` with the
    same constants) side by side; -> what the run saw.  ``schedule_steps``: the episode length the first schedule is drawn for
    (GeometricOpponent.reset draws with the length the previous reset left: a reset under ``set_max_iter(schedule_steps)`` before
    the seeded one sets it, and the episode itself keeps its full length), so that schedules run out within the run"""
    import grid2op_b200.backend  # noqa: F401
    import grid2op
    from grid2op.Parameters import Parameters
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import list_scenarios, load_line_events, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    from grid2op_b200.opponent import opponent_seed
    from test_batched_env import _scripted
    grid = env_grid(name)
    gm = GridModel(grid)
    cdir = os.path.join(os.path.dirname(grid), "chronics")
    folder = list_scenarios(cdir)[0]
    chron = load_scenarios(cdir, gm, scenarios=[folder])
    maint = load_line_events(folder, gm, "maintenance")
    B = len(seeds)
    p = Parameters()
    p.NO_OVERFLOW_DISCONNECTION = True
    p.NB_TIMESTEP_COOLDOWN_LINE = 3
    p.NB_TIMESTEP_COOLDOWN_SUB = 2
    backend_class = backend_class or _host_logic_backend()
    envs = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for i in range(B):
            e = grid2op.make(name, test=True, backend=backend_class(), param=p, _add_to_name=f"geo{i}", **make_kw(i))
            if schedule_steps is not None:
                e.set_max_iter(schedule_steps)
                e.reset()
                e.set_max_iter(-1)
            e.seed(int(seeds[i]))
            e.set_id(0)
            e.reset()
            envs.append(e)
    sp = envs[0]._oppSpace
    assert type(sp.opponent).__name__ == "GeometricOpponent"
    kwo = envs[0]._kwargs_opponent
    emt = int(sp.opponent._episode_max_time) if schedule_steps is None else schedule_steps
    th = np.asarray(envs[0].get_thermal_limit(), dtype=np.float32)
    benv = BatchedEnv(gm, chron, B, maintenance=None if maint is None else maint[None], scen=np.zeros(B, np.int32),
                      t0=np.zeros(B, np.int32), thermal_limit_a=th, nb_timestep_cooldown_line=3, nb_timestep_cooldown_sub=2,
                      nb_timestep_reconnection=p.NB_TIMESTEP_RECONNECTION, protections=False, engine=engine_factory(gm))
    rho, _, _ = benv.reset_step()
    obs = [e.get_obs() for e in envs]
    for i in range(B):
        assert np.array_equal(obs[i].topo_vect, benv.topo[i, :gm.dim_topo])
    benv.enable_opponent("GeometricOpponent", kwo["lines_attacked"], attack_duration=sp.attack_max_duration,
                         attack_cooldown=sp.attack_cooldown, budget_per_ts=sp.budget_per_timestep, init_budget=sp.init_budget,
                         seeds=[opponent_seed(int(s)) for s in seeds], delta_time_seconds=envs[0].delta_time_seconds,
                         episode_max_time=emt, pmax_pmin_ratio=kwo.get("pmax_pmin_ratio", 4), **_geo_kw(envs[0]))
    for i, e in enumerate(envs):
        w, d, n = _sched(e._oppSpace.opponent)
        st = benv._opp.get_state()
        assert n == st["geo_ctr"][i, 0] and np.array_equal(w, st["geo_wait"][i, :n]) and np.array_equal(d, st["geo_dur"][i, :n]), i
    att = [int(x) for x in benv._opp.lines]
    em = None
    if emu:
        from geo_emu import EmuGeoEnvState
        em = EmuGeoEnvState(benv)
    rngs = [np.random.default_rng(100 + int(s)) for s in seeds]
    is_line_pos = np.zeros(gm.dim_topo, dtype=bool)
    is_line_pos[gm.line_or_pos] = True; is_line_pos[gm.line_ex_pos] = True
    saw = dict(attack_steps=0, attacks=0, refused_budget=0, refused_duration=0, fails_wait=0, lost_status=0, schedule_end=0)
    alive = np.ones(B, dtype=bool)
    last_line = np.full(B, -1)
    ended = np.zeros(B, dtype=bool)
    for k in range(n_steps):
        sub_id = np.full(B, -1, np.int64); sub_bus = np.zeros((B, benv.max_sub_size), np.int8)
        line_id = np.full(B, -1, np.int64); line_st = np.zeros(B, np.int64)
        ref = []
        for i, e in enumerate(envs):
            if not alive[i]:
                ref.append(None)
                continue
            o = obs[i]
            a = _scripted(k, rngs[i], o.topo_vect, o.line_status, o.time_before_cooldown_line, o.time_before_cooldown_sub,
                          benv.sub_pos, benv.sub_size, gm.n_line, is_line_pos)
            out = [l for l in att if not o.line_status[l] and o.time_before_cooldown_line[l] == 0]
            if k % 4 == 0 and out:
                a = dict(sub=-1, bus=None, line=int(out[0]), status=1)          # reconnect an attackable line (lets attacks land)
            elif k % 16 == 9:
                a = dict(sub=-1, bus=None, line=att[(k // 16 + i) % len(att)], status=-1)   # an attackable line out: attacks get lost
            spec = {}
            if a["sub"] >= 0:
                spec["set_bus"] = {"substations_id": [(a["sub"], a["bus"].astype(int).tolist())]}
                sub_id[i] = a["sub"]; sub_bus[i, :len(a["bus"])] = a["bus"]
            if a["line"] >= 0:
                spec["set_line_status"] = [(a["line"], int(a["status"]))]
                line_id[i] = a["line"]; line_st[i] = a["status"]
            op = e._oppSpace.opponent
            before = (op._attack_counter, e._oppSpace.previous_fails)
            o2, r, d, info = e.step(e.action_space(spec))
            obs[i] = o2
            ref.append((d, info, before, op._attack_counter, e._oppSpace.previous_fails, e._oppSpace.budget))
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
            assert np.array_equal(em.ost["attack_line"], binfo["opponent_attack_line"]) and np.array_equal(em.ost["attack_dur"], binfo["opponent_attack_duration"]), k
            assert np.array_equal(em.st["topo"], benv.topo) and np.array_equal(em.st["line_cd"], benv.line_cooldown), k
        st = benv._opp.get_state()
        for i in range(B):
            if not alive[i]:
                continue
            d, info, (c0, fails0), c1, fails, budget = ref[i]
            assert bool(done[i]) == bool(d), (k, i, info["exception"])
            if d:
                alive[i] = False
                continue
            o = obs[i]
            op = envs[i]._oppSpace.opponent
            la = info["opponent_attack_line"]
            want_line = -1 if la is None else int(np.flatnonzero(la)[0])
            assert binfo["opponent_attack_line"][i] == want_line, (k, i, binfo["opponent_attack_line"][i], want_line)
            assert binfo["opponent_attack_duration"][i] == (info["opponent_attack_duration"] if la is not None else 0), (k, i)
            b = benv._opp.budget[i]
            assert b.dtype == np.asarray(budget).dtype and b == budget, (k, i, b, budget)
            assert st["geo_ctr"][i, 1] == c1 and bool(st["geo_ctr"][i, 2]) == bool(fails), (k, i)
            nxt = op._next_attack_time
            assert st["ctr"][i, 3] == (-2 ** 31 if nxt is None else int(nxt)), (k, i, st["ctr"][i, 3], nxt)
            assert np.array_equal(o.topo_vect, benv.topo[i, :gm.dim_topo]), (k, i)
            assert np.array_equal(o.line_status, benv.line_status()[i]), (k, i)
            assert np.array_equal(o.time_before_cooldown_line, benv.line_cooldown[i]), (k, i)
            assert np.array_equal(o.time_before_cooldown_sub, benv.sub_cooldown[i]), (k, i)
            assert np.allclose(o.rho, rho[i], rtol=check_rho_tol[0], atol=check_rho_tol[1]), (k, i)
            if want_line >= 0:
                saw["attack_steps"] += 1
                saw["attacks"] += int(c1 > c0)
                last_line[i] = want_line
            elif c1 > c0 and fails:
                if op._attack_durations[c1 - 1] > sp.attack_max_duration:
                    saw["refused_duration"] += 1
                else:
                    saw["refused_budget"] += 1
            elif c1 > c0:
                saw["lost_status"] += 1
            if fails0 and c0 < op._number_of_attacks:
                saw["fails_wait"] += 1                                # the call after a refusal moved the next attack
            if c1 >= op._number_of_attacks and not ended[i]:
                ended[i] = True
                saw["schedule_end"] += 1
    saw["alive"] = int(alive.sum())
    for e in envs:
        e.close()
    benv.close()
    return saw


def short_kw(name):
    """the environment's GeometricOpponent with hazard 1/9 and recovery 1/6 over a 3-step minimum, so that durations above the
    7-step max duration are common; a budget of 0.3 per step from 4 refuses some of the others; a 2-step cooldown"""
    e = _make(name, "geolines")
    kwo = dict(e._kwargs_opponent, **SHORT[0])
    e.close()
    return lambda i: dict(opponent_init_budget=4.0, opponent_budget_per_ts=0.3, opponent_attack_duration=7, opponent_attack_cooldown=2,
                          kwargs_opponent=kwo)


@pytest.mark.parametrize("name,seeds", [("l2rpn_icaps_2021", (0, 3, 5)), ("l2rpn_wcci_2022_dev", (1, 2, 6))])
def test_geometric_opponent_vs_reference_env_host_logic(name, seeds):
    if env_grid(name) is None:
        pytest.skip("reference data not available")
    from oracle_engine import COracleSeriesEngine
    saw = run_geometric_vs_reference(name, 150, short_kw(name), seeds=seeds, engine_factory=COracleSeriesEngine, emu=True,
                                     schedule_steps=80)
    assert all(saw[k] > 0 for k in ("attacks", "refused_budget", "refused_duration", "fails_wait", "lost_status", "schedule_end")), saw


# ---- validation ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [
    dict(attack_every_xxx_hour=24, average_attack_duration_hour=1, minimum_attack_duration_hour=2),       # average < minimum
    dict(attack_every_xxx_hour=24, average_attack_duration_hour=2, minimum_attack_duration_hour=2),       # average == minimum
    dict(attack_every_xxx_hour=4, average_attack_duration_hour=4, minimum_attack_duration_hour=1),        # every <= average
    dict(attack_every_xxx_hour=1e8, average_attack_duration_hour=4, minimum_attack_duration_hour=1),      # hazard draws overflow int32
    dict(attack_every_xxx_hour=1e9, average_attack_duration_hour=1e8, minimum_attack_duration_hour=1),    # recovery draws overflow
    dict(attack_every_xxx_hour=24, average_attack_duration_hour=1.05, minimum_attack_duration_hour=1),    # recovery rate > 1
    dict(attack_every_xxx_hour=24, average_attack_duration_hour=4, minimum_attack_duration_hour=1, pmax_pmin_ratio=0),
    dict(attack_every_xxx_hour=24, average_attack_duration_hour=4),                                       # missing
])
def test_geometric_constants_rejected(kw):
    from grid2op_b200.opponent import BatchedOpponent
    with pytest.raises(ValueError):
        BatchedOpponent("GeometricOpponent", [0, 1], 2, attack_duration=96, attack_cooldown=12, budget_per_ts=0.17, init_budget=144.0,
                        seeds=[0, 1], episode_max_time=8000, **kw)


def test_geometric_needs_episode_max_time():
    from grid2op_b200.opponent import BatchedOpponent
    with pytest.raises(ValueError):
        BatchedOpponent("GeometricOpponent", [0, 1], 1, attack_duration=96, attack_cooldown=12, budget_per_ts=0.17, init_budget=144.0,
                        seeds=[0], attack_every_xxx_hour=24, average_attack_duration_hour=4, minimum_attack_duration_hour=1)
