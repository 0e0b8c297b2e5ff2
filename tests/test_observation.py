"""``BatchedEnv.observe`` (grid2op observation vectors + rewards assembled by csrc/b200pf_obs.cuh) against unmodified grid2op
environments stepped one by one with the same scripted agent: ``obs.to_vect()`` and the reward after every step, after the reset
step, and on the step that ends an episode (the game-over observation).  Integer, boolean and calendar attributes must be equal,
floats within the tolerance of the existing rho / record comparisons (tests/test_batched_env.py).

* CPU (``not gpu``): host logic — the reference environments run B200Backend on the oracle adapter, BatchedEnv runs on the oracle's C
  restatement with the HOST build of the observe kernel body (tests/obs_engines.py);
* GPU (``-m gpu``): the CUDA engine on both sides, protections off and on, on l2rpn_case14_sandbox, l2rpn_neurips_2020_track1 and
  l2rpn_wcci_2022_dev (118 substations, storage units, shunts).
"""
import os
import warnings

import numpy as np
import pytest

from conftest import env_grid

INT_ATTRS = {"year", "month", "day", "hour_of_day", "minute_of_hour", "day_of_week", "line_status", "timestep_overflow", "topo_vect",
             "time_before_cooldown_line", "time_before_cooldown_sub", "time_next_maintenance", "duration_next_maintenance",
             "is_alarm_illegal", "time_since_last_alarm", "last_alarm", "was_alarm_used_after_game_over", "_shunt_bus", "current_step",
             "max_step", "delta_time", "load_detached", "gen_detached", "storage_detached", "timestep_protection_engaged"}


def compare_vect(attrs, sizes, ref, got, what):
    off = 0
    for a in attrs:
        n = sizes[a]
        r, g = ref[off:off + n], got[off:off + n]
        if a in INT_ATTRS:
            assert np.array_equal(r, g, equal_nan=True), (what, a, r, g)
        else:
            atol = 0.05 if a in ("a_or", "a_ex") else 2e-3
            assert np.allclose(r, g, rtol=2e-4, atol=atol, equal_nan=True), (what, a, float(np.nanmax(np.abs(r - g))) if n else 0)
        off += n
    assert off == len(ref) == len(got), (what, off, len(ref), len(got))


def run_observation_vs_reference(env_name, n_steps, backend_factory, engine_factory, protections, B=3, start_row=0, kill_step=None,
                                 kill_sub=None, check_reset=True):
    """Step ``B`` reference environments and one BatchedEnv with the scripted agent of tests/test_batched_env.py; compare
    observe() with obs.to_vect() / the reward after every step.  ``kill_step`` / ``kill_sub``: instance 1 moves every element of
    ``kill_sub`` to busbar 2 at that step (a game over on l2rpn_neurips_2020_track1, see test_batched_env)."""
    import grid2op
    from grid2op.Parameters import Parameters
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import list_scenarios, load_line_events, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    from grid2op_b200.observation import attr_sizes
    from test_batched_env import _scripted
    grid = env_grid(env_name)
    env_dir = os.path.dirname(grid)
    gm = GridModel(grid)
    cdir = os.path.join(env_dir, "chronics")
    folders = list_scenarios(cdir)
    folder = folders[0]
    chron = load_scenarios(cdir, gm, scenarios=[folder])
    maint = load_line_events(folder, gm, "maintenance")
    p = Parameters()
    p.NO_OVERFLOW_DISCONNECTION = not protections
    p.NB_TIMESTEP_COOLDOWN_LINE = 3
    p.NB_TIMESTEP_COOLDOWN_SUB = 2
    envs = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for i in range(B):
            e = grid2op.make(env_name, test=True, backend=backend_factory(), param=p, opponent_init_budget=0., opponent_budget_per_ts=0.,
                             _add_to_name=f"obs{i}_{int(protections)}")
            e.set_id(0)
            envs.append(e)
    attrs = list(type(envs[0].observation_space._template_obj).attr_list_vect)
    reward_name = type(envs[0]._reward_helper.template_reward).__name__
    assert reward_name in ("RedispReward", "L2RPNReward")
    th = np.asarray(envs[0].get_thermal_limit(), dtype=np.float32)
    benv = BatchedEnv(gm, chron, B, maintenance=None if maint is None else maint[None], scen=np.zeros(B, dtype=np.int32),
                      t0=np.zeros(B, dtype=np.int32), thermal_limit_a=th, nb_timestep_cooldown_line=3, nb_timestep_cooldown_sub=2,
                      nb_timestep_reconnection=p.NB_TIMESTEP_RECONNECTION, protections=protections,
                      hard_overflow_threshold=p.HARD_OVERFLOW_THRESHOLD, soft_overflow_threshold=p.SOFT_OVERFLOW_THRESHOLD,
                      nb_timestep_overflow_allowed=p.NB_TIMESTEP_OVERFLOW_ALLOWED, engine=engine_factory(gm))
    benv.enable_observation(env_dir, attrs=attrs, reward=reward_name, scenarios=[folder])
    sizes = attr_sizes(gm)
    np_of = lambda x: x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)        # noqa: E731
    # env.reset() <-> the reset step
    obs = [e.reset() for e in envs]
    benv.reset_step()
    o_b, r_b = benv.observe()
    o_b = np_of(o_b)
    if check_reset:
        for i in range(B):
            compare_vect(attrs, sizes, obs[i].to_vect(), o_b[i], ("reset", i))
    if start_row:
        for i, e in enumerate(envs):
            e.fast_forward_chronics(start_row)
            obs[i] = e.get_obs()
        benv.reset_instances(np.arange(B), rows=np.full(B, start_row + 1))
        benv.current_step[:] = [o.current_step for o in obs]
        for i in range(B):
            benv.line_cooldown[i] = obs[i].time_before_cooldown_line
            benv.sub_cooldown[i] = obs[i].time_before_cooldown_sub
    rngs = [np.random.default_rng(200 + s) for s in range(B)]
    is_line_pos = np.zeros(gm.dim_topo, dtype=bool)
    is_line_pos[gm.line_or_pos] = True; is_line_pos[gm.line_ex_pos] = True
    alive = np.ones(B, dtype=bool)
    go_vect = [None] * B
    saw = dict(illegal=0, maint=0, game_over=0, compared=0, overflow=0)
    for k in range(n_steps):
        sub_id = np.full(B, -1, dtype=np.int64); sub_bus = np.zeros((B, benv.max_sub_size), dtype=np.int8)
        line_id = np.full(B, -1, dtype=np.int64); line_st = np.zeros(B, dtype=np.int64)
        ref = [None] * B
        for i, e in enumerate(envs):
            if not alive[i]:
                continue
            o = obs[i]
            if kill_step is not None and i == 1 and k >= kill_step and o.time_before_cooldown_sub[kill_sub] == 0:
                a = dict(sub=kill_sub, bus=np.full(int(benv.sub_size[kill_sub]), 2), line=-1, status=0)
            else:
                a = _scripted(k, rngs[i], o.topo_vect, o.line_status, o.time_before_cooldown_line, o.time_before_cooldown_sub,
                              benv.sub_pos, benv.sub_size, gm.n_line, is_line_pos)
            spec = {}
            if a["sub"] >= 0:
                spec["set_bus"] = {"substations_id": [(a["sub"], a["bus"].astype(int).tolist())]}
                sub_id[i] = a["sub"]; sub_bus[i, :len(a["bus"])] = a["bus"]
            if a["line"] >= 0:
                spec["set_line_status"] = [(a["line"], int(a["status"]))]
                line_id[i] = a["line"]; line_st[i] = a["status"]
            o2, r, d, info = e.step(e.action_space(spec))
            obs[i] = o2
            ref[i] = (o2, r, d, info)
        rho, done, binfo = benv.step(sub_id, sub_bus, line_id, line_st)
        o_b, r_b = benv.observe()
        o_b, r_b = np_of(o_b), np_of(r_b)
        for i in range(B):
            if not alive[i]:
                # a finished episode keeps reporting its game-over observation
                compare_vect(attrs, sizes, go_vect[i], o_b[i], ("after game over", k, i))
                continue
            o2, r, d, info = ref[i]
            assert bool(done[i]) == bool(d), (k, i, info["exception"], binfo["status"][i])
            assert bool(binfo["is_illegal"][i]) == bool(info["is_illegal"]), (k, i)
            saw["illegal"] += int(bool(info["is_illegal"]))
            v = o2.to_vect()
            compare_vect(attrs, sizes, v, o_b[i], (k, i, bool(d)))
            assert np.isclose(r, r_b[i], rtol=1e-5, atol=1e-4), (k, i, r, r_b[i])
            saw["compared"] += 1
            saw["maint"] += int((o2.time_next_maintenance == 0).any())
            saw["overflow"] += int((o2.timestep_overflow > 0).any())
            if d:
                alive[i] = False; go_vect[i] = v; saw["game_over"] += 1
    for e in envs:
        e.close()
    benv.close()
    return saw


def _host_backend():
    import grid2op_b200.backend as bk
    from oracle_engine import OracleEngine

    class HostLogicBackend(bk.B200Backend):
        def _make_engine(self, gm):
            return OracleEngine(gm)

    return HostLogicBackend


def test_obs_spec_and_tables():
    from grid2op_b200.gridmodel import GridModel
    from grid2op_b200.observation import COMPLETE_OBSERVATION_ATTRS, attr_sizes, obs_spec
    gold = os.path.join(os.path.dirname(__file__), "golden")
    gm = GridModel.from_npz(os.path.join(gold, "gridmodel_l2rpn_case14_sandbox.npz"))
    seg, n = obs_spec(gm)
    sz = attr_sizes(gm)
    assert n == sum(sz[a] for a in COMPLETE_OBSERVATION_ATTRS) and len(seg) == len(COMPLETE_OBSERVATION_ATTRS)
    assert (seg[1:, 1] == np.cumsum(seg[:-1, 2])).all()
    seg2, n2 = obs_spec(gm, ["rho", "topo_vect", "gen_p"])
    assert n2 == gm.n_line + gm.dim_topo + gm.n_gen and seg2[:, 1].tolist() == [0, gm.n_line, gm.n_line + gm.dim_topo]
    with pytest.raises(ValueError):
        obs_spec(gm, ["rho", "theta_or"])


@pytest.mark.parametrize("env_name,kw", [
    ("l2rpn_neurips_2020_track1", dict(n_steps=22, start_row=96, kill_step=8, kill_sub=12)),
    ("rte_case5_example", dict(n_steps=14)),
])
def test_observation_host_logic_vs_reference_env(env_name, kw):
    if env_grid(env_name) is None:
        pytest.skip("reference data not available")
    from obs_engines import COracleObsSeriesEngine
    saw = run_observation_vs_reference(env_name, backend_factory=_host_backend(), engine_factory=COracleObsSeriesEngine, protections=False,
                                       **kw)
    assert saw["compared"] >= 20 and saw["illegal"] >= 1
    if env_name == "l2rpn_neurips_2020_track1":
        assert saw["maint"] and saw["game_over"] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("protections", [False, True])
@pytest.mark.parametrize("env_name,kw", [
    ("l2rpn_case14_sandbox", dict(n_steps=40)),
    ("l2rpn_neurips_2020_track1", dict(n_steps=40, start_row=96, kill_step=10, kill_sub=12)),
    ("l2rpn_wcci_2022_dev", dict(n_steps=16, B=2)),
])
def test_observation_vs_reference_env_gpu(cuda_required, env_name, kw, protections):
    if env_grid(env_name) is None:
        pytest.skip("reference data not available")
    from grid2op_b200.backend import B200Backend
    saw = run_observation_vs_reference(env_name, backend_factory=B200Backend, engine_factory=lambda gm: None, protections=protections, **kw)
    assert saw["compared"] >= 16
