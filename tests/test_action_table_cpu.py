"""BatchedEnv's discrete action ids (grid2op_b200/action_table.py ``ActionTable``, ``BatchedEnv.set_action_table``,
``step(action_id=...)``) on the CPU:

* ``ActionTable.unitary`` row by row against ``IdToAct(env.action_space).init_converter(redispatch=False, curtail=False,
  storage=False)`` on five grids, with each kind of action turned off, and on a three-busbar environment;
* ``ActionTable.from_actions`` through ``IdToAct.save`` and back, and the actions it refuses;
* the numpy path stepping ids next to unmodified environments stepping ``converter.convert_act(id)`` (host logic on both sides);
* the host build of the device bodies with ids, bit-equal to the numpy path;
* the ValueError cases, which change nothing.
"""
import os
import warnings

import numpy as np
import pytest

from conftest import env_grid

GRIDS = ("rte_case5_example", "l2rpn_case14_sandbox", "l2rpn_neurips_2020_track1", "l2rpn_wcci_2022_dev", "l2rpn_idf_2023")
KINDS = ("line_set", "line_change", "topo_set", "topo_change")


def _make(name, suffix, **kw):
    import grid2op_b200.backend  # noqa: F401
    import grid2op
    from test_env_actions_cpu import _host_backend
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return grid2op.make(name, test=True, backend=_host_backend()(), _add_to_name=suffix, **kw)


def _converter(env, all_actions=None, **flags):
    from grid2op.Converter import IdToAct
    c = IdToAct(env.action_space)
    if all_actions is None:
        c.init_converter(redispatch=False, curtail=False, storage=False, **flags)
    else:
        c.init_converter(all_actions=all_actions)
    return c


def _assert_same(conv, T):
    assert conv.n == T.n
    for k, a in enumerate(conv.all_actions):
        assert np.array_equal(a.set_bus, T.set_bus[k]), k
        assert np.array_equal(a.change_bus, T.change_bus[k]), k
        assert np.array_equal(a.line_set_status, T.set_line_status[k]), k
        assert np.array_equal(a.line_change_status, T.change_line_status[k]), k


def _kind(T, k):
    if (T.set_line_status[k] != 0).any():
        return "line_set"
    if T.change_line_status[k].any():
        return "line_change"
    if (T.set_bus[k] != 0).any():
        return "topo_set"
    if T.change_bus[k].any():
        return "topo_change"
    return None


@pytest.mark.parametrize("name", GRIDS)
def test_unitary_table_matches_id_to_act(name):
    if env_grid(name) is None:
        pytest.skip("reference data not available")
    from grid2op_b200.action_table import ActionTable
    from grid2op_b200.gridmodel import GridModel
    env = _make(name, "tab")
    gm = GridModel(env_grid(name))
    _assert_same(_converter(env), ActionTable.unitary(gm))
    if name in ("rte_case5_example", "l2rpn_case14_sandbox"):
        flags = dict(set_line_status=True, change_line_status=True, set_topo_vect=True, change_bus_vect=True)
        for off in flags:
            f = dict(flags, **{off: False})
            _assert_same(_converter(env, **f), ActionTable.unitary(gm, **f))
    env.close()


def test_unitary_table_three_busbars():
    """three busbars per substation: the set enumeration (lines with every pair of busbars, topologies numbered in order) matches,
    and change_bus is refused where grid2op raises"""
    name = "l2rpn_case14_sandbox"
    if env_grid(name) is None:
        pytest.skip("reference data not available")
    from grid2op_b200.action_table import ActionTable
    from grid2op_b200.gridmodel import GridModel
    env = _make(name, "tab3", n_busbar=3)
    from grid2op.Exceptions import Grid2OpException
    gm = GridModel(env_grid(name), n_busbar=3)
    _assert_same(_converter(env, change_bus_vect=False), ActionTable.unitary(gm, change_bus_vect=False))
    with pytest.raises(Grid2OpException):
        _converter(env)
    with pytest.raises(ValueError):
        ActionTable.unitary(gm)
    env.close()


def test_from_actions_round_trip_and_refusals(tmp_path):
    name = "l2rpn_case14_sandbox"
    if env_grid(name) is None:
        pytest.skip("reference data not available")
    from grid2op_b200.action_table import ActionTable
    from grid2op_b200.gridmodel import GridModel
    env = _make(name, "tabio")
    gm = GridModel(env_grid(name))
    conv = _converter(env)
    keep = np.arange(0, conv.n, 3)                        # a filtered list, saved and restored as IdToAct does
    conv.all_actions = [conv.all_actions[k] for k in keep]
    conv.n = len(keep)
    conv.save(str(tmp_path), "acts.npy")
    back = _converter(env, all_actions=os.path.join(str(tmp_path), "acts.npy"))
    T = ActionTable.from_actions(gm, back.all_actions)
    _assert_same(back, T)
    full = ActionTable.unitary(gm)
    for x, y in ((T.set_bus, full.set_bus), (T.change_bus, full.change_bus), (T.set_line_status, full.set_line_status),
                 (T.change_line_status, full.change_line_status)):
        assert np.array_equal(x, y[keep])
    sp = env.action_space
    disp = np.zeros(gm.n_gen); disp[int(np.flatnonzero(type(env).gen_redispatchable)[0])] = 1.0
    with pytest.raises(ValueError):
        ActionTable.from_actions(gm, [sp({}), sp({"redispatch": disp})])
    load0 = int(type(env).load_pos_topo_vect[0])
    sb = np.zeros(gm.dim_topo, int); sb[load0] = -1
    with pytest.raises(ValueError):
        ActionTable.from_actions(gm, [sp({"set_bus": sb})])
    env.close()
    # a storage action and an alarm, on the environments that have them
    if env_grid("l2rpn_wcci_2022_dev") is not None:
        e2 = _make("l2rpn_wcci_2022_dev", "tabsto")
        gm2 = GridModel(env_grid("l2rpn_wcci_2022_dev"))
        st = np.zeros(type(e2).n_storage); st[0] = 1.0
        with pytest.raises(ValueError):
            ActionTable.from_actions(gm2, [e2.action_space({"set_storage": st})])
        with pytest.raises(ValueError):                   # a table for the wrong grid
            ActionTable.from_actions(gm, [e2.action_space({})])
        e2.close()
    if env_grid("l2rpn_icaps_2021") is not None:
        e3 = _make("l2rpn_icaps_2021", "tabalarm")
        gm3 = GridModel(env_grid("l2rpn_icaps_2021"))
        with pytest.raises(ValueError):
            ActionTable.from_actions(gm3, [e3.action_space({"raise_alarm": [0]})])
        e3.close()


def test_table_constructor_refusals():
    from grid2op_b200.action_table import ActionTable
    from grid2op_b200.gridmodel import GridModel
    gm = GridModel.from_npz(os.path.join(os.path.dirname(__file__), "golden", "gridmodel_l2rpn_case14_sandbox.npz"))
    nt, nl = gm.dim_topo, gm.n_line
    T = ActionTable(gm, set_line_status=np.array([[0] * nl, [1] + [0] * (nl - 1)]))
    assert T.n == 2 and T.set_bus.shape == (2, nt) and not T.change_bus.any() and not T.set_bus.flags.writeable
    load = int(np.asarray(gm.load_pos)[0])
    sb = np.zeros((1, nt), np.int8); sb[0, load] = -1
    for kw in (dict(), dict(set_bus=np.full((1, nt), 3)), dict(set_bus=sb), dict(set_bus=np.zeros((1, nt + 1), np.int8)),
               dict(set_bus=np.zeros((1, nt), np.float32)), dict(change_bus=np.zeros((1, nt), np.int8)),
               dict(set_line_status=np.full((1, nl), 2)), dict(set_line_status=np.full((1, nl), 255)),
               dict(set_bus=np.zeros((2, nt), np.int8), set_line_status=np.zeros((1, nl), np.int8))):
        with pytest.raises(ValueError):
            ActionTable(gm, **kw)


def _host_env(B, **kw):
    from test_env_actions_cpu import _small_env
    return _small_env(B, **kw)


def test_id_refusals_change_nothing():
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    from grid2op_b200.action_table import ActionTable
    benv = _host_env(3)
    benv.reset_step()
    gm = benv.gm
    ok = np.zeros(3, np.int64)
    with pytest.raises(ValueError):
        benv.step(action_id=ok)                           # no table
    T = ActionTable.unitary(gm)
    benv.set_action_table(T)
    benv.step(action_id=np.array([1, 2, 3]))
    before = (benv.topo.copy(), benv.line_cooldown.copy(), benv.sub_cooldown.copy(), benv.n_steps)
    for kw in (dict(action_id=np.array([0, T.n, 0])), dict(action_id=np.array([-1, 0, 0])), dict(action_id=np.zeros(3, np.float64)),
               dict(action_id=np.zeros(4, np.int64)), dict(action_id=ok, set_bus=np.zeros((3, gm.dim_topo), np.int8)),
               dict(action_id=ok, sub_id=np.full(3, -1), sub_bus=np.zeros((3, benv.max_sub_size), np.int8)),
               dict(action_id=ok, line_id=np.full(3, -1), line_status=np.zeros(3, np.int64))):
        with pytest.raises(ValueError):
            benv.step(**kw)
    assert np.array_equal(before[0], benv.topo) and np.array_equal(before[1], benv.line_cooldown)
    assert np.array_equal(before[2], benv.sub_cooldown) and before[3] == benv.n_steps
    from grid2op_b200.gridmodel import GridModel
    gold = os.path.join(os.path.dirname(__file__), "golden")
    with pytest.raises(ValueError):
        benv.set_action_table(ActionTable.unitary(GridModel.from_npz(os.path.join(gold, "gridmodel_rte_case5_example.npz"))))
    benv.close()


def test_ids_equal_vectors_and_reset_ignores_ids():
    """ids step as the same rows given as vectors; on a reset step the ids are ignored"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    from grid2op_b200.action_table import ActionTable
    B = 6
    a, b = _host_env(B, nb_timestep_cooldown_line=2, nb_timestep_cooldown_sub=1), _host_env(B, nb_timestep_cooldown_line=2,
                                                                                            nb_timestep_cooldown_sub=1)
    T = ActionTable.unitary(a.gm)
    a.set_action_table(T)
    ra = a.step(from_reset=True, action_id=np.arange(B) + 100)
    rb = b.step(from_reset=True)
    assert np.array_equal(ra[0], rb[0], equal_nan=True) and np.array_equal(a.topo, b.topo)
    rng = np.random.default_rng(3)
    for k in range(20):
        ids = rng.integers(0, T.n, B)
        ra = a.step(action_id=ids)
        rb = b.step(set_bus=T.set_bus[ids], change_bus=T.change_bus[ids], set_line_status=T.set_line_status[ids],
                    change_line_status=T.change_line_status[ids])
        for x, y in ((a.topo, b.topo), (a.last_bus, b.last_bus), (a.line_cooldown, b.line_cooldown), (a.sub_cooldown, b.sub_cooldown),
                     (a.done, b.done), (ra[2]["is_illegal"], rb[2]["is_illegal"]), (ra[2]["is_ambiguous"], rb[2]["is_ambiguous"])):
            assert np.array_equal(x, y), k
        assert np.array_equal(ra[0], rb[0], equal_nan=True), k


def run_ids(env_name, n_steps, B, seed, protections=False, max_sub=3, max_line=2, areas=False, cuda=False):
    """``B`` unmodified environments stepping ``converter.convert_act(id)`` next to one BatchedEnv stepping the same ids through the
    unitary table; a finished instance restarts on both sides (``env.reset()`` / ``reset_instances``).  -> what the run saw"""
    import grid2op_b200.backend as bk
    import grid2op
    from grid2op.Parameters import Parameters
    from grid2op.Rules import RulesByArea
    from obs_engines import COracleObsSeriesEngine, EmuProtObsSeriesEngine
    from grid2op_b200.action_table import ActionTable
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import list_scenarios, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    from grid2op_b200.observation import attr_sizes
    from test_env_actions_cpu import _host_backend
    from test_observation import compare_vect
    grid = env_grid(env_name)
    gm = GridModel(grid)
    env_dir = os.path.dirname(grid)
    cdir = os.path.join(env_dir, "chronics")
    folder = list_scenarios(cdir)[0]
    chron = load_scenarios(cdir, gm, scenarios=[folder])
    p = Parameters()
    p.NO_OVERFLOW_DISCONNECTION = not protections
    p.NB_TIMESTEP_COOLDOWN_LINE = 2
    p.NB_TIMESTEP_COOLDOWN_SUB = 2
    if not areas:
        p.MAX_SUB_CHANGED, p.MAX_LINE_STATUS_CHANGED = max_sub, max_line
    envs = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for i in range(B):
            e = grid2op.make(env_name, test=True, backend=(bk.B200Backend if cuda else _host_backend())(), param=p,
                             opponent_init_budget=0., opponent_budget_per_ts=0., _add_to_name=f"ids{i}_{int(protections)}_{seed}")
            e.set_id(0)
            envs.append(e)
    conv = _converter(envs[0])
    T = ActionTable.unitary(gm)
    rules = envs[0]._game_rules.legal_action
    areas_list = None
    if areas:
        assert isinstance(rules, RulesByArea)
        areas_list = [list(v) for v in rules.substations_id_by_area.values()]
        max_sub, max_line = p.MAX_SUB_CHANGED, p.MAX_LINE_STATUS_CHANGED
    attrs = list(type(envs[0].observation_space._template_obj).attr_list_vect)
    reward_name = type(envs[0]._reward_helper.template_reward).__name__
    th = np.asarray(envs[0].get_thermal_limit(), dtype=np.float32)
    engine_class = EmuProtObsSeriesEngine if protections else COracleObsSeriesEngine
    if type(envs[0]).dim_alerts:
        from alert_emu import COracleAlertObsEngine
        assert not protections
        engine_class = COracleAlertObsEngine
    benv = BatchedEnv(gm, chron, B, scen=np.zeros(B, dtype=np.int32), t0=np.zeros(B, dtype=np.int32), thermal_limit_a=th,
                      nb_timestep_cooldown_line=2, nb_timestep_cooldown_sub=2, nb_timestep_reconnection=p.NB_TIMESTEP_RECONNECTION,
                      protections=protections, hard_overflow_threshold=p.HARD_OVERFLOW_THRESHOLD,
                      soft_overflow_threshold=p.SOFT_OVERFLOW_THRESHOLD, nb_timestep_overflow_allowed=p.NB_TIMESTEP_OVERFLOW_ALLOWED,
                      max_sub_changed=max_sub, max_line_status_changed=max_line, rules_by_area=areas_list,
                      engine=None if cuda else engine_class(gm))
    benv.set_action_table(T)
    if type(envs[0]).dim_alerts:
        benv.enable_alerts(type(envs[0]).alertable_line_ids, alert_time_window=p.ALERT_TIME_WINDOW)
    benv.enable_observation(env_dir, attrs=attrs, reward=reward_name, scenarios=[folder])
    sizes = attr_sizes(gm, benv._alerts.n if benv._alerts is not None else 0)
    obs = [e.reset() for e in envs]
    benv.reset_step()
    benv.observe()
    rng = np.random.default_rng(seed)
    saw = dict(compared=0, cooldown=0, game_over=0, restarted=0, **{k: 0 for k in KINDS})
    for k in range(n_steps):
        ids = rng.integers(0, T.n, B)
        ref = []
        for i, e in enumerate(envs):
            act = conv.convert_act(int(ids[i]))
            aff_l, aff_s = act.get_topological_impact(obs[i].line_status)
            prev_cd = (obs[i].time_before_cooldown_line.copy(), obs[i].time_before_cooldown_sub.copy())
            o2, r, d, info = e.step(act)
            ref.append((o2, r, d, info, aff_l, aff_s, prev_cd))
            obs[i] = o2
        rho, done, binfo = benv.step(action_id=ids)
        o_b, r_b = (x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x) for x in benv.observe())
        restart = []
        for i, (o2, r, d, info, aff_l, aff_s, (cdl, cds)) in enumerate(ref):
            what = (k, i, int(ids[i]), info["exception"])
            assert bool(done[i]) == bool(d), what
            assert bool(binfo["is_illegal"][i]) == bool(info["is_illegal"]), what
            assert bool(binfo["is_ambiguous"][i]) == bool(info["is_ambiguous"]), what
            if info["is_illegal"]:
                saw["cooldown"] += int((cdl[aff_l] > 0).any() or (cds[aff_s] > 0).any())
            elif not d and _kind(T, ids[i]) is not None:
                saw[_kind(T, ids[i])] += 1
            assert np.isclose(r, float(r_b[i]), rtol=1e-5, atol=1e-4), (what, r, float(r_b[i]))
            if d:
                saw["game_over"] += 1
                restart.append(i)
                continue
            assert np.array_equal(o2.topo_vect, benv.topo[i, :gm.dim_topo]), what
            assert np.array_equal(o2.line_status, benv.line_status()[i]), what
            assert np.array_equal(o2.time_before_cooldown_line, benv.line_cooldown[i]), what
            assert np.array_equal(o2.time_before_cooldown_sub, benv.sub_cooldown[i]), what
            assert np.allclose(o2.rho, rho[i], rtol=2e-4, atol=2e-5), what
            compare_vect(attrs, sizes, o2.to_vect(), o_b[i], what)
            saw["compared"] += 1
        if restart:                                       # env.reset() solves row 0: the next step of both sides solves row 1
            for i in restart:
                envs[i].set_id(0)
                obs[i] = envs[i].reset()
            benv.reset_instances(np.asarray(restart), np.ones(len(restart), np.int64))
            saw["restarted"] += len(restart)
    for e in envs:
        e.close()
    benv.close()
    return saw


def test_ids_next_to_reference_case14():
    """case14, MAX_SUB_CHANGED = 3, MAX_LINE_STATUS_CHANGED = 2, cooldowns 2, protections off and on"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    saw = {}
    for protections in (False, True):
        for seed in (0, 1):
            for key, v in run_ids("l2rpn_case14_sandbox", 25, 8, 10 * seed + int(protections), protections=protections).items():
                saw[key] = saw.get(key, 0) + v
    assert saw["compared"] >= 100, saw
    for key in ("cooldown", "game_over", "restarted") + KINDS:
        assert saw[key] > 0, (key, saw)


def test_ids_next_to_reference_idf_2023_rules_by_area():
    if env_grid("l2rpn_idf_2023") is None:
        pytest.skip("reference data not available")
    saw = run_ids("l2rpn_idf_2023", 15, 4, 5, areas=True)
    assert saw["compared"] >= 30, saw
    assert saw["topo_set"] + saw["topo_change"] > 0, saw


@pytest.mark.parametrize("protections", [False, True])
def test_ids_env_bodies(protections):
    """the host build of the device bodies (tests/emu/act_ids_emu.cpp) reading rows of the table by id, next to the numpy path: bit-equal
    at every step and masked reset"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    from act_ids_emu import EmuActIdsEnvState
    from test_env_tensor_cpu import _check, _env, _raw
    from grid2op_b200.action_table import ActionTable
    env, calls = _env("l2rpn_case14_sandbox", 8, protections, max_sub_changed=2, max_line_status_changed=2)
    T = ActionTable.unitary(env.gm)
    env.set_action_table(T)
    tab = (T.set_bus, T.change_bus, T.set_line_status, T.change_line_status)
    emu = EmuActIdsEnvState(env)
    rng = np.random.default_rng(23 + protections)
    seen = dict(illegal=0, ambiguous=0)

    def step(k, ids, from_reset=False):
        del calls[:]
        ctl = emu.step_apply_ids(tab, ids, from_reset=from_reset, tight_cap=env.tight_cap)
        assert ctl[2] == 0
        _, _, info = env.step(from_reset=from_reset, action_id=ids)
        status, disc = _raw(env)
        emu.step_post(status, disc, from_reset=from_reset, stamp=env.n_steps, prot=env.protections)
        assert np.array_equal(emu.st["status_out"], info["status"]), k
        _check(k, env, emu, ctl, len(calls))
        assert np.array_equal(emu.st["is_ambiguous"].astype(bool), env.is_ambiguous), k
        return info

    step(-1, rng.integers(0, T.n, env.batch), from_reset=True)
    for k in range(20):
        if k in (7, 14):
            mask = env.done.copy(); mask[0] = True
            idx = np.flatnonzero(mask)
            env.reset_instances(idx, np.full(len(idx), 3))
            rows = np.zeros(env.batch, np.int32); rows[idx] = 3
            emu.reset(mask, rows)
            for key, arr in (("topo", env.topo), ("last_bus", env.last_bus), ("is_ambiguous", env.is_ambiguous)):
                assert np.array_equal(emu.st[key].astype(arr.dtype), arr), key
        info = step(k, rng.integers(0, T.n, env.batch))
        seen["illegal"] += int(info["is_illegal"].sum())
    # an id out of range: the validation body flags it and the apply body writes nothing
    topo = emu.st["topo"].copy()
    ctl = emu.step_apply_ids(tab, np.full(env.batch, T.n), tight_cap=env.tight_cap)
    assert ctl[2] != 0 and np.array_equal(topo, emu.st["topo"])
    assert seen["illegal"], seen
    env.close()
