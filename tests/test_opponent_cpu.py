"""BatchedEnv's line-attack opponents (grid2op_b200/opponent.py, csrc/b200pf_opp.cuh) on the CPU:

* the device restatement of numpy's legacy RandomState draws (host build, tests/emu/opp_emu.cpp) is bit-equal to
  ``np.random.RandomState`` for many seeds, across the 624-word twist;
* ``opponent_seed(s)`` is the opponent's seed of ``env.seed(s)``;
* the numpy path next to unmodified grid2op environments with their opponent ON, stepped with the scripted agent of
  tests/test_batched_env.py (host logic on both sides: oracle adapters): attacked line, duration, line cooldowns, topology, line status
  and the budget (value and dtype) equal after every step, with attacks refused for budget, attacks running to their end and agent
  actions made illegal by an attack's cooldown; the host build of the device body runs next to it and must agree bit for bit.
"""
import os
import warnings

import numpy as np
import pytest

from conftest import env_grid


# ---- RandomState restatement -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 6, 288, 2 ** 31 - 1])
def test_randint_bit_equal_to_randomstate(n):
    from opp_emu import Draws
    for seed in range(0, 3000, 37):
        d, r = Draws(seed), np.random.RandomState(seed)
        got = d.randint(n, 1400)                                      # (> 624 words: crosses the twist)
        want = np.array([r.randint(n) for _ in range(1400)])
        assert np.array_equal(got.astype(np.int64), want), (seed, n)
        assert d.pos[0] == r.get_state()[2] and np.array_equal(d.mt, r.get_state()[1]), (seed, n)


def test_random_sample_and_choice_bit_equal_to_randomstate():
    from opp_emu import Draws
    g = np.random.default_rng(7)
    for seed in range(0, 5000, 53):
        d, r = Draws(seed), np.random.RandomState(seed)
        assert np.array_equal(d.random_sample(700), np.array([r.random_sample() for _ in range(700)])), seed
        for k in range(300):
            n = int(g.integers(1, 13))
            if k % 2:
                assert int(d.randint(n)[0]) == r.choice(np.arange(n)), (seed, k)
            else:
                # the weighted opponent's p: float32 rho over float64 normalisations, some lines at 0
                w = g.random(n).astype(np.float32).astype(np.float64) / g.choice([0.45, 0.3, 0.6, 0.2, 0.55], n)
                w[g.random(n) < 0.2] = 0.0
                if w.sum() <= 0:
                    continue
                assert d.choice_weighted(w) == r.choice(np.arange(n), p=w / w.sum()), (seed, k)
        assert np.array_equal(d.mt, r.get_state()[1]) and d.pos[0] == r.get_state()[2], seed


def _host_logic_backend():
    import grid2op_b200.backend as bk
    from oracle_engine import OracleEngine

    class HostLogicBackend(bk.B200Backend):
        def _make_engine(self, gm):
            return OracleEngine(gm)
    return HostLogicBackend


@pytest.mark.parametrize("name", ["rte_case14_opponent", "l2rpn_neurips_2020_track1"])
def test_opponent_seed_is_env_seed(name):
    if env_grid(name) is None:
        pytest.skip("reference data not available")
    import grid2op_b200.backend  # noqa: F401  (locates / bootstraps the grid2op install first)
    import grid2op
    from grid2op_b200.opponent import opponent_seed
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        e = grid2op.make(name, test=True, backend=_host_logic_backend()(), _add_to_name="oppseed")
    for s in (0, 1, 7, 123, 2 ** 31 - 2):
        assert e.seed(s)[6] == (opponent_seed(s),), s
    e.close()


# ---- against unmodified grid2op environments ----------------------------------------------------------------------------------
def run_opponent_vs_reference(name, n_steps, make_kw, seeds, engine_factory, emu: bool, backend_class=None, check_rho_tol=(2e-4, 2e-5)):
    """steps B unmodified environments (opponent on, ``make_kw`` overrides) and BatchedEnv (``enable_opponent`` with the same
    constants) side by side; -> what the run saw"""
    import grid2op_b200.backend  # noqa: F401  (locates / bootstraps the grid2op install first)
    import grid2op
    from grid2op.Parameters import Parameters
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import load_line_events, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    from grid2op_b200.opponent import opponent_seed
    from test_batched_env import _scripted
    grid = env_grid(name)
    gm = GridModel(grid)
    cdir = os.path.join(os.path.dirname(grid), "chronics")
    folder = os.path.join(cdir, sorted(os.listdir(cdir))[0])
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
            e = grid2op.make(name, test=True, backend=backend_class(), param=p, _add_to_name=f"opp{i}", **make_kw(i))
            e.seed(int(seeds[i]))
            e.set_id(0)
            e.reset()
            envs.append(e)
    sp = envs[0]._oppSpace
    kind = type(sp.opponent).__name__
    kwo = envs[0]._kwargs_opponent
    th = np.asarray(envs[0].get_thermal_limit(), dtype=np.float32)
    benv = BatchedEnv(gm, chron, B, maintenance=None if maint is None else maint[None], scen=np.zeros(B, np.int32),
                      t0=np.zeros(B, np.int32), thermal_limit_a=th, nb_timestep_cooldown_line=3, nb_timestep_cooldown_sub=2,
                      nb_timestep_reconnection=p.NB_TIMESTEP_RECONNECTION, protections=False, engine=engine_factory(gm))
    rho, _, _ = benv.reset_step()
    obs = [e.get_obs() for e in envs]
    for i in range(B):
        assert np.array_equal(obs[i].topo_vect, benv.topo[i, :gm.dim_topo])
        assert np.allclose(obs[i].rho, rho[i], rtol=check_rho_tol[0], atol=check_rho_tol[1])
    benv.enable_opponent(kind, kwo["lines_attacked"], attack_duration=sp.attack_max_duration, attack_cooldown=sp.attack_cooldown,
                         budget_per_ts=sp.budget_per_timestep, init_budget=sp.init_budget, attack_period=kwo.get("attack_period"),
                         rho_normalization=kwo.get("rho_normalization"), seeds=[opponent_seed(int(s)) for s in seeds])
    em = None
    if emu:
        from opp_emu import EmuOppEnvState
        em = EmuOppEnvState(benv)
    rngs = [np.random.default_rng(100 + int(s)) for s in seeds]
    is_line_pos = np.zeros(gm.dim_topo, dtype=bool)
    is_line_pos[gm.line_or_pos] = True; is_line_pos[gm.line_ex_pos] = True
    saw = dict(attack_steps=0, refused=0, whole=0, illegal_by_attack=0, n_illegal=0, back_to_back_same_line=0, budget64=0)
    alive = np.ones(B, dtype=bool)
    run_len = np.zeros(B, dtype=np.int64)
    last_line = np.full(B, -1)
    last_ended = np.full(B, -1)
    for k in range(n_steps):
        sub_id = np.full(B, -1, np.int64); sub_bus = np.zeros((B, benv.max_sub_size), np.int8)
        line_id = np.full(B, -1, np.int64); line_st = np.zeros(B, np.int64)
        ref, try_attacked = [], np.zeros(B, dtype=bool)
        for i, e in enumerate(envs):
            if not alive[i]:
                ref.append(None)
                continue
            o = obs[i]
            a = _scripted(k, rngs[i], o.topo_vect, o.line_status, o.time_before_cooldown_line, o.time_before_cooldown_sub,
                          benv.sub_pos, benv.sub_size, gm.n_line, is_line_pos)
            if k % 4 == 2 and last_line[i] >= 0 and not o.line_status[last_line[i]]:
                a = dict(sub=-1, bus=None, line=int(last_line[i]), status=1)     # reconnect the attacked line (illegal while it runs)
                try_attacked[i] = True
            spec = {}
            if a["sub"] >= 0:
                spec["set_bus"] = {"substations_id": [(a["sub"], a["bus"].astype(int).tolist())]}
                sub_id[i] = a["sub"]; sub_bus[i, :len(a["bus"])] = a["bus"]
            if a["line"] >= 0:
                spec["set_line_status"] = [(a["line"], int(a["status"]))]
                line_id[i] = a["line"]; line_st[i] = a["status"]
            o2, r, d, info = e.step(e.action_space(spec))
            obs[i] = o2
            ref.append((d, info, e._oppSpace.previous_fails, e._oppSpace.budget))
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
            assert np.array_equal(em.st["done"].astype(bool), benv.done) and np.array_equal(em.st["is_illegal"].astype(bool), benv.is_illegal), k
        for i in range(B):
            if not alive[i]:
                continue
            d, info, fails, budget = ref[i]
            assert bool(done[i]) == bool(d), (k, i, info["exception"])
            if d:
                alive[i] = False
                continue
            o = obs[i]
            la = info["opponent_attack_line"]
            want_line = -1 if la is None else int(np.flatnonzero(la)[0])
            assert binfo["opponent_attack_line"][i] == want_line, (k, i, binfo["opponent_attack_line"][i], want_line)
            assert binfo["opponent_attack_duration"][i] == (info["opponent_attack_duration"] if la is not None else 0), (k, i)
            b = benv._opp.budget[i]
            assert b.dtype == np.asarray(budget).dtype and b == budget, (k, i, b, budget)
            assert np.array_equal(o.topo_vect, benv.topo[i, :gm.dim_topo]), (k, i)
            assert np.array_equal(o.line_status, benv.line_status()[i]), (k, i)
            assert np.array_equal(o.time_before_cooldown_line, benv.line_cooldown[i]), (k, i, o.time_before_cooldown_line, benv.line_cooldown[i])
            assert np.array_equal(o.time_before_cooldown_sub, benv.sub_cooldown[i]), (k, i)
            assert np.allclose(o.rho, rho[i], rtol=check_rho_tol[0], atol=check_rho_tol[1]), (k, i)
            saw["n_illegal"] += int(bool(info["is_illegal"]))
            saw["refused"] += int(bool(fails))
            saw["budget64"] += int(b.dtype == np.float64)
            if try_attacked[i] and info["is_illegal"]:
                saw["illegal_by_attack"] += 1
            if want_line >= 0:
                saw["attack_steps"] += 1
                if run_len[i] == 0 and want_line == last_ended[i]:
                    saw["back_to_back_same_line"] += 1
                run_len[i] += 1
                last_line[i] = want_line
                if binfo["opponent_attack_duration"][i] == 1:          # the attack's last step
                    saw["whole"] += int(run_len[i] == int(sp.attack_max_duration))
                    run_len[i] = 0
                    last_ended[i] = want_line
    assert benv.n_illegal == saw["n_illegal"]
    saw["alive"] = int(alive.sum())
    for e in envs:
        e.close()
    benv.close()
    return saw


def _track1_kw(i):
    # the robustness track's opponent with a smaller initial budget and shorter period / duration / cooldown, so that a 150-step
    # run sees attacks refused for budget, whole attacks and the cooldown between them
    return dict(opponent_init_budget=2.0, opponent_attack_duration=6, opponent_attack_cooldown=12,
                kwargs_opponent=dict(lines_attacked=["62_58_180", "62_63_160", "48_50_136", "48_53_141", "41_48_131", "39_41_121",
                                                     "43_44_125", "44_45_126", "34_35_110", "54_58_154"],
                                     rho_normalization=[0.45, 0.45, 0.6, 0.35, 0.3, 0.2, 0.55, 0.3, 0.45, 0.55], attack_period=8))


def test_weighted_random_opponent_vs_reference_env_host_logic():
    name = "l2rpn_neurips_2020_track1"
    if env_grid(name) is None:
        pytest.skip("reference data not available")
    from oracle_engine import COracleSeriesEngine
    saw = run_opponent_vs_reference(name, 150, _track1_kw, seeds=(0, 3, 11), engine_factory=COracleSeriesEngine, emu=True)
    assert saw["refused"] > 0 and saw["whole"] > 0 and saw["illegal_by_attack"] > 0 and saw["budget64"] > 0, saw


def test_random_line_opponent_vs_reference_env_host_logic():
    name = "rte_case14_opponent"
    if env_grid(name) is None:
        pytest.skip("reference data not available")
    from oracle_engine import COracleSeriesEngine
    # the environment's own opponent (RandomLineOpponent on its lines, 0.5 budget per step) with a smaller initial budget and
    # shorter attacks / cooldown, so that the run sees refusals, whole attacks and back-to-back attacks before the scripted agent
    # ends the episodes
    kw = dict(opponent_init_budget=1.0, opponent_attack_duration=5, opponent_attack_cooldown=6)
    saw = run_opponent_vs_reference(name, 80, lambda i: kw, seeds=(1, 2, 4, 8), engine_factory=COracleSeriesEngine, emu=True)
    assert saw["refused"] > 0 and saw["whole"] > 0 and saw["illegal_by_attack"] > 0 and saw["budget64"] > 0, saw
