"""BatchedEnv's grid2op-native topology action (``set_bus`` / ``change_bus`` / ``set_line_status`` / ``change_line_status`` vectors,
MAX_SUB_CHANGED / MAX_LINE_STATUS_CHANGED, RulesByArea; grid2op_b200/batched_env.py ``_apply_actions``, csrc/b200pf_env.cuh
``act_vec_instance``) on the CPU:

* the numpy path next to unmodified environments (host logic on both sides): random vector actions touching several substations
  and lines, line ends set to -1, reconnections through a busbar and through change_line_status, and a share of deliberately
  ambiguous actions.  After every step: topology, line status, both cooldown vectors, is_illegal, is_ambiguous, done, rho, the
  observation vector and the reward;
* the legacy one-substation / one-line arguments and the same action as vectors give the same state;
* RulesByArea's area tables and the ValueError cases.
"""
import os
import warnings

import numpy as np
import pytest

from conftest import env_grid

AMBIGUITY_KINDS = ("set_change_bus", "set_change_status", "end_minus_one", "disco_with_bus", "reco_with_minus_one")


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _draw(rng, benv, on, n_sub_max, n_line_max):
    """one instance's random vector action -> (set_bus, change_bus, set_status, change_status, ambiguity kind or None)"""
    gm = benv.gm
    sb = np.zeros(gm.dim_topo, np.int8); cb = np.zeros(gm.dim_topo, bool)
    ss = np.zeros(gm.n_line, np.int8); cs = np.zeros(gm.n_line, bool)
    lor, lex = benv.line_or_pos, benv.line_ex_pos
    if rng.random() < 0.1:
        return sb, cb, ss, cs, None
    for s in rng.choice(gm.n_sub, int(rng.integers(1, n_sub_max + 1)), replace=False):
        pos = benv.sub_pos[s, :benv.sub_size[s]]
        if rng.random() < 0.5:
            pick = pos[rng.random(len(pos)) < 0.5]
            sb[pick] = np.where(rng.random(len(pick)) < 0.8, 1, 2)
        else:
            cb[pos[rng.random(len(pos)) < 0.25]] = True
    for l in rng.choice(gm.n_line, int(rng.integers(0, n_line_max + 1)), replace=False):
        r = rng.random()
        if r < 0.3:
            ss[l] = -1 if on[l] else 1
        elif r < 0.5:
            cs[l] = True
        elif r < 0.75:                                    # a line end's busbar: reconnects a disconnected line, else moves the end
            p = lor[l] if rng.random() < 0.5 else lex[l]
            sb[p] = 1 if not on[l] or rng.random() < 0.5 else 2; cb[p] = False
        else:                                             # a line end set to -1 disconnects the line
            p = lor[l] if rng.random() < 0.5 else lex[l]
            sb[p] = -1; cb[p] = False
            q = lex[l] if p == lor[l] else lor[l]
            if sb[q] > 0:
                sb[q] = 0
    off = np.flatnonzero(~on)
    if len(off) and rng.random() < 0.6:                   # reconnect a disconnected line: through one end's busbar or change_status
        l = int(rng.choice(off))
        ss[l] = 0; cb[lor[l]] = cb[lex[l]] = False
        if rng.random() < 0.5:
            sb[lor[l]], sb[lex[l]] = 1, 0
            cs[l] = False
        else:
            sb[lor[l]] = sb[lex[l]] = 0
            cs[l] = True
    # (the random part may already be ambiguous: an end at -1 with its other end or the line's status named)
    kind = None
    if rng.random() < 0.12:
        kind = AMBIGUITY_KINDS[int(rng.integers(len(AMBIGUITY_KINDS)))]
        l = int(rng.integers(gm.n_line))
        if kind == "set_change_bus":
            p = int(rng.integers(gm.dim_topo)); sb[p] = 1; cb[p] = True
        elif kind == "set_change_status":
            ss[l] = 1 if rng.random() < 0.5 else -1; cs[l] = True
        elif kind == "end_minus_one":
            sb[lor[l]] = -1; sb[lex[l]] = 2; cb[lor[l]] = cb[lex[l]] = False
        elif kind == "disco_with_bus":
            ss[l] = -1; cs[l] = False
            if rng.random() < 0.5:
                sb[lor[l]] = 2; cb[lor[l]] = False
            else:
                cb[lex[l]] = True; sb[lex[l]] = 0
        else:
            ss[l] = 1; cs[l] = False
            if rng.random() < 0.5:
                sb[lex[l]] = -1; cb[lex[l]] = False; sb[lor[l]] = min(sb[lor[l]], 0)
            else:
                cb[lor[l]] = True; sb[lor[l]] = 0
    return sb, cb, ss, cs, kind


def _ambiguity_kinds(benv, sb, cb, ss, cs):
    lor, lex = benv.line_or_pos, benv.line_ex_pos
    so, se, ch = sb[lor], sb[lex], cb[lor] | cb[lex]
    return {"set_change_bus": bool(((sb != 0) & cb).any()), "set_change_status": bool(((ss != 0) & cs).any()),
            "end_minus_one": bool((((so == -1) & (se > 0)) | ((se == -1) & (so > 0))).any()),
            "disco_with_bus": bool(((ss == -1) & ((so > 0) | (se > 0) | ch)).any()),
            "reco_with_minus_one": bool(((ss == 1) & ((so == -1) | (se == -1) | ch)).any())}


def _host_backend():
    import grid2op_b200.backend as bk
    from oracle_engine import OracleEngine

    class HostLogicBackend(bk.B200Backend):
        def _make_engine(self, gm):
            return OracleEngine(gm)

    return HostLogicBackend


def run_vector_actions(env_name, n_steps, B, seed, protections=False, max_sub=3, max_line=2, areas=False, maintenance=False,
                       n_sub_max=3, n_line_max=3, cuda=False):
    """-> what the run saw.  ``areas``: the environment's own RulesByArea (l2rpn_idf_2023) on both sides; else LookParam with
    ``max_sub`` / ``max_line`` on both sides.  ``maintenance``: the scenario's maintenance table on both sides.  ``cuda``: the
    CUDA engine on both sides instead of the host logic."""
    import grid2op_b200.backend as bk
    import grid2op
    from grid2op.Parameters import Parameters
    from grid2op.Rules import RulesByArea
    from obs_engines import COracleObsSeriesEngine, EmuProtObsSeriesEngine
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import list_scenarios, load_line_events, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    from grid2op_b200.observation import attr_sizes
    from test_observation import compare_vect
    grid = env_grid(env_name)
    gm = GridModel(grid)
    env_dir = os.path.dirname(grid)
    cdir = os.path.join(env_dir, "chronics")
    folder = list_scenarios(cdir)[0]
    chron = load_scenarios(cdir, gm, scenarios=[folder])
    maint = load_line_events(folder, gm, "maintenance") if maintenance else None
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
            e = grid2op.make(env_name, test=True, backend=(bk.B200Backend if cuda else _host_backend())(), param=p, opponent_init_budget=0., opponent_budget_per_ts=0.,
                             _add_to_name=f"act{i}_{int(protections)}_{seed}")
            e.set_id(0)
            envs.append(e)
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
    if type(envs[0]).dim_alerts:                          # (the host build of the observe body with the alert values)
        from alert_emu import COracleAlertObsEngine
        assert not protections
        engine_class = COracleAlertObsEngine
    benv = BatchedEnv(gm, chron, B, maintenance=None if maint is None else maint[None], scen=np.zeros(B, dtype=np.int32),
                      t0=np.zeros(B, dtype=np.int32), thermal_limit_a=th, nb_timestep_cooldown_line=2, nb_timestep_cooldown_sub=2,
                      nb_timestep_reconnection=p.NB_TIMESTEP_RECONNECTION, protections=protections,
                      hard_overflow_threshold=p.HARD_OVERFLOW_THRESHOLD, soft_overflow_threshold=p.SOFT_OVERFLOW_THRESHOLD,
                      nb_timestep_overflow_allowed=p.NB_TIMESTEP_OVERFLOW_ALLOWED, max_sub_changed=max_sub, max_line_status_changed=max_line,
                      rules_by_area=areas_list,
                      engine=None if cuda else engine_class(gm))
    if areas:                                             # RulesByArea.initialize's line areas
        assert [list(x) for x in benv.lines_id_by_area] == [list(v) for v in rules.lines_id_by_area.values()]
    if type(envs[0]).dim_alerts:                          # (l2rpn_idf_2023's observation carries the alert attributes; no opponent here)
        benv.enable_alerts(type(envs[0]).alertable_line_ids, alert_time_window=p.ALERT_TIME_WINDOW)
    benv.enable_observation(env_dir, attrs=attrs, reward=reward_name, scenarios=[folder])
    sizes = attr_sizes(gm, benv._alerts.n if benv._alerts is not None else 0)
    obs = [e.reset() for e in envs]
    benv.reset_step()
    benv.observe()
    rng = np.random.default_rng(seed)
    alive = np.ones(B, dtype=bool)
    saw = dict(compared=0, count=0, area_count=0, area_allows=0, cooldown=0, multi_sub=0, reco_bus=0, reco_change=0, game_over=0,
               **{k: 0 for k in AMBIGUITY_KINDS})
    for k in range(n_steps):
        SB = np.zeros((B, gm.dim_topo), np.int8); CB = np.zeros((B, gm.dim_topo), bool)
        SS = np.zeros((B, gm.n_line), np.int8); CS = np.zeros((B, gm.n_line), bool)
        ref = [None] * B
        for i, e in enumerate(envs):
            if not alive[i]:
                continue
            on = obs[i].line_status
            sb, cb, ss, cs, _ = _draw(rng, benv, on, n_sub_max, n_line_max)
            SB[i], CB[i], SS[i], CS[i] = sb, cb, ss, cs
            spec = {}
            if (sb != 0).any():
                spec["set_bus"] = sb.astype(int)
            if cb.any():
                spec["change_bus"] = cb
            if (ss != 0).any():
                spec["set_line_status"] = ss.astype(int)
            if cs.any():
                spec["change_line_status"] = cs
            act = e.action_space(spec)
            aff_l, aff_s = act.get_topological_impact(on)
            prev_cd = (obs[i].time_before_cooldown_line.copy(), obs[i].time_before_cooldown_sub.copy())
            o2, r, d, info = e.step(act)
            ref[i] = (o2, r, d, info, aff_l, aff_s, prev_cd, on)
            obs[i] = o2
        rho, done, binfo = benv.step(set_bus=SB, change_bus=CB, set_line_status=SS, change_line_status=CS)
        o_b, r_b = (_np(x) for x in benv.observe())
        for i in range(B):
            if ref[i] is None:
                continue
            o2, r, d, info, aff_l, aff_s, (cdl, cds), on = ref[i]
            what = (k, i, info["exception"])
            assert bool(done[i]) == bool(d), what
            assert bool(binfo["is_illegal"][i]) == bool(info["is_illegal"]), what
            assert bool(binfo["is_ambiguous"][i]) == bool(info["is_ambiguous"]), what
            if info["is_ambiguous"]:
                for kind, hit in _ambiguity_kinds(benv, SB[i], CB[i], SS[i], CS[i]).items():
                    saw[kind] += int(hit)
            elif info["is_illegal"]:
                if areas:
                    over = any(aff_l[v].sum() > max_line for v in rules.lines_id_by_area.values()) or \
                        any(aff_s[v].sum() > max_sub for v in rules.substations_id_by_area.values())
                    saw["area_count"] += int(over)
                else:
                    over = aff_l.sum() > max_line or aff_s.sum() > max_sub
                    saw["count"] += int(over)
                saw["cooldown"] += int(not over and ((cdl[aff_l] > 0).any() or (cds[aff_s] > 0).any()))
            elif not d:
                saw["multi_sub"] += int(aff_s.sum() > 1)
                saw["area_allows"] += int(areas and (aff_s.sum() > max_sub or aff_l.sum() > max_line))
                reco = ~on & o2.line_status
                saw["reco_bus"] += int((reco & ((SB[i][benv.line_or_pos] > 0) | (SB[i][benv.line_ex_pos] > 0))).any())
                saw["reco_change"] += int((reco & CS[i]).any())
            rb = float(r_b[i])
            assert np.isclose(r, rb, rtol=1e-5, atol=1e-4), (what, r, rb)
            if d:
                alive[i] = False; saw["game_over"] += 1
                continue
            assert np.array_equal(o2.topo_vect, benv.topo[i, :gm.dim_topo]), what
            assert np.array_equal(o2.line_status, benv.line_status()[i]), what
            assert np.array_equal(o2.time_before_cooldown_line, benv.line_cooldown[i]), what
            assert np.array_equal(o2.time_before_cooldown_sub, benv.sub_cooldown[i]), what
            assert np.allclose(o2.rho, rho[i], rtol=2e-4, atol=2e-5), what
            compare_vect(attrs, sizes, o2.to_vect(), o_b[i], what)
            saw["compared"] += 1
        if not alive.any():
            break
    for e in envs:
        e.close()
    benv.close()
    return saw


def test_vector_actions_case14():
    """MAX_SUB_CHANGED = 3, MAX_LINE_STATUS_CHANGED = 2, non-zero cooldowns, protections off and on"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    saw = {}
    for protections in (False, True):
        for seed in (0, 1, 2):
            for key, v in run_vector_actions("l2rpn_case14_sandbox", 25, 8, 10 * seed + int(protections), protections=protections).items():
                saw[key] = saw.get(key, 0) + v
    assert saw["compared"] >= 100, saw
    for key in ("count", "cooldown", "multi_sub", "reco_bus", "reco_change") + AMBIGUITY_KINDS:
        assert saw[key] > 0, (key, saw)


def test_vector_actions_idf_2023_rules_by_area():
    if env_grid("l2rpn_idf_2023") is None:
        pytest.skip("reference data not available")
    saw = run_vector_actions("l2rpn_idf_2023", 20, 6, 5, areas=True, n_sub_max=5, n_line_max=4)
    assert saw["compared"] >= 40, saw
    for key in ("area_count", "area_allows", "cooldown", "multi_sub"):
        assert saw[key] > 0, (key, saw)
    assert sum(saw[k] for k in AMBIGUITY_KINDS) > 0, saw


def test_vector_actions_neurips_2020_maintenance():
    if env_grid("l2rpn_neurips_2020_track1") is None:
        pytest.skip("reference data not available")
    saw = run_vector_actions("l2rpn_neurips_2020_track1", 15, 4, 7, maintenance=True, max_sub=2, max_line=2)
    assert saw["compared"] >= 20 and saw["multi_sub"] > 0, saw


def _small_env(B=4, **kw):
    from oracle_engine import COracleSeriesEngine
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import list_scenarios, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    grid = env_grid("l2rpn_case14_sandbox")
    gm = GridModel(grid)
    cdir = os.path.join(os.path.dirname(grid), "chronics")
    chron = load_scenarios(cdir, gm, scenarios=[list_scenarios(cdir)[0]])
    return BatchedEnv(gm, chron, B, scen=np.zeros(B, np.int32), t0=np.zeros(B, np.int32), protections=False,
                      engine=COracleSeriesEngine(gm), **kw)


def test_legacy_and_vector_encodings_agree():
    """one-substation (busbars > 0) and one-line actions through sub_id / line_id and through set_bus / set_line_status"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    from grid2op_b200.batched_env import random_substation_actions
    B = 6
    a = _small_env(B, nb_timestep_cooldown_line=2, nb_timestep_cooldown_sub=1)
    b = _small_env(B, nb_timestep_cooldown_line=2, nb_timestep_cooldown_sub=1)
    a.reset_step(); b.reset_step()
    gm = a.gm
    rng = np.random.default_rng(4)
    n_illegal = 0
    for k in range(30):
        sub, bus = random_substation_actions(a, rng)
        line = np.full(B, -1); st = np.zeros(B, np.int64)
        kind = rng.random(B)
        on = a.line_status()
        sb = np.zeros((B, gm.dim_topo), np.int8); ss = np.zeros((B, gm.n_line), np.int8)
        for i in range(B):
            if kind[i] < 0.5:
                n = a.sub_size[sub[i]]
                sb[i, a.sub_pos[sub[i], :n]] = bus[i, :n]
            else:
                sub[i] = -1
                if kind[i] < 0.85:
                    line[i] = rng.integers(gm.n_line); st[i] = -1 if on[i, line[i]] else 1
                    ss[i, line[i]] = st[i]
        ra = a.step(sub, bus, line, st)
        rb = b.step(set_bus=sb, set_line_status=ss)
        n_illegal += int(ra[2]["is_illegal"].sum())
        assert not rb[2]["is_ambiguous"].any()
        for x, y in ((a.topo, b.topo), (a.last_bus, b.last_bus), (a.line_cooldown, b.line_cooldown), (a.sub_cooldown, b.sub_cooldown),
                     (a.done, b.done), (ra[2]["is_illegal"], rb[2]["is_illegal"])):
            assert np.array_equal(x, y), k
        assert np.array_equal(ra[0], rb[0], equal_nan=True), k
    assert n_illegal > 0


def test_rules_by_area_tables_and_refusals():
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    benv = _small_env(2, rules_by_area=[[3, 0, 1, 2, 2], [4, 5, 6], [7, 8, 9, 10, 11, 12, 13]])
    assert [list(a) for a in benv.areas] == [[0, 1, 2, 3], [4, 5, 6], [7, 8, 9, 10, 11, 12, 13]]
    ls = np.asarray(benv.gm.line_or_sub)
    for k, a in enumerate(benv.areas):
        assert list(benv.lines_id_by_area[k]) == list(np.flatnonzero(np.isin(ls, a)))
        assert ((benv._line_area >> k) & 1).astype(bool).tolist() == np.isin(ls, a).tolist()
    with pytest.raises(ValueError):
        _small_env(2, rules_by_area=[[0, 1, 2], [4, 5, 6]])
    with pytest.raises(ValueError):
        _small_env(2, max_sub_changed=-1)


def test_vector_action_refusals_change_nothing():
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    benv = _small_env(2)
    benv.reset_step()
    gm = benv.gm
    before = (benv.topo.copy(), benv.line_cooldown.copy(), benv.n_steps)
    load_pos = int(np.asarray(gm.load_pos)[0])
    bad = [dict(set_bus=np.zeros((2, gm.dim_topo + 1), np.int8)), dict(set_bus=np.zeros((2, gm.dim_topo), np.float32)),
           dict(change_bus=np.zeros((2, gm.dim_topo), np.int8)), dict(set_line_status=np.zeros((3, gm.n_line), np.int8)),
           dict(set_bus=np.full((2, gm.dim_topo), 3, np.int8)), dict(set_bus=np.full((2, gm.dim_topo), -2, np.int8)),
           dict(set_line_status=np.full((2, gm.n_line), 2, np.int8))]
    sb = np.zeros((2, gm.dim_topo), np.int8); sb[0, load_pos] = -1
    bad.append(dict(set_bus=sb))
    for kw in bad:
        with pytest.raises(ValueError):
            benv.step(**kw)
    with pytest.raises(ValueError):
        benv.step(sub_id=np.full(2, -1), sub_bus=np.zeros((2, benv.max_sub_size), np.int8), set_line_status=np.zeros((2, gm.n_line), np.int8))
    assert np.array_equal(before[0], benv.topo) and np.array_equal(before[1], benv.line_cooldown) and before[2] == benv.n_steps


def test_change_bus_needs_two_busbars():
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.gridmodel import GridModel
    from oracle_engine import COracleSeriesEngine
    gold = os.path.join(os.path.dirname(__file__), "golden")
    gm = GridModel.from_npz(os.path.join(gold, "gridmodel_l2rpn_case14_sandbox.npz"))
    if gm.n_busbar == 2:
        gm.n_busbar = 3
        gm.n_slot = gm.n_sub * 3
    chron = np.zeros((1, 4, 2 * gm.n_load + 2 * gm.n_gen), np.float32)
    try:
        benv = BatchedEnv(gm, chron, 1, scen=np.zeros(1, np.int32), t0=np.zeros(1, np.int32), protections=False,
                          engine=COracleSeriesEngine(gm))
    except Exception as e:                                # (a grid model this engine cannot take: the check is the host path's)
        pytest.skip(f"three-busbar engine unavailable: {e}")
    cb = np.zeros((1, gm.dim_topo), bool); cb[0, 0] = True
    with pytest.raises(ValueError):
        benv.step(change_bus=cb)


@pytest.mark.parametrize("protections,areas", [(False, False), (True, False), (False, True)])
def test_vector_actions_env_bodies(protections, areas):
    """the host build of the device bodies (tests/emu/act_emu.cpp) next to the numpy path, bit-equal at every step and masked
    reset: topology, last busbars, cooldowns, done, is_illegal, is_ambiguous, the observe record's flags and the illegal count"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    from act_emu import EmuActEnvState
    from test_env_actions_gpu import vector_actions
    from test_env_tensor_cpu import _check, _env, _raw
    kw = dict(max_sub_changed=2, max_line_status_changed=2)
    if areas:
        kw = dict(rules_by_area=[[0, 1, 2, 3, 4], [5, 6, 7, 8], [9, 10, 11, 12, 13]])
    env, calls = _env("l2rpn_case14_sandbox", 8, protections, **kw)
    emu = EmuActEnvState(env)
    rng = np.random.default_rng(17 + protections)
    seen = dict(illegal=0, ambiguous=0, over=0)

    def step(k, vecs, from_reset=False):
        del calls[:]
        ctl = emu.step_apply_vec(vecs, from_reset=from_reset, tight_cap=env.tight_cap)
        assert ctl[2] == 0
        if from_reset:
            _, _, info = env.step(from_reset=True)
        else:
            _, _, info = env.step(set_bus=vecs[0], change_bus=vecs[1], set_line_status=vecs[2], change_line_status=vecs[3])
        status, disc = _raw(env)
        emu.step_post(status, disc, from_reset=from_reset, stamp=env.n_steps, prot=env.protections)
        assert np.array_equal(emu.st["status_out"], info["status"]), k
        _check(k, env, emu, ctl, len(calls))
        assert np.array_equal(emu.st["is_ambiguous"].astype(bool), env.is_ambiguous), k
        nl, ns = env.gm.n_line, env.gm.n_sub
        assert np.array_equal((emu.st["obs_in"][:, nl + ns + 2] & 8) != 0, env.is_ambiguous), k
        return info

    step(-1, None, from_reset=True)
    for k in range(20):
        if k in (7, 14):
            mask = env.done.copy(); mask[0] = True
            idx = np.flatnonzero(mask)
            env.reset_instances(idx, np.full(len(idx), 3))
            rows = np.zeros(env.batch, np.int32); rows[idx] = 3
            emu.reset(mask, rows)
            for key, arr in (("topo", env.topo), ("last_bus", env.last_bus), ("is_ambiguous", env.is_ambiguous)):
                assert np.array_equal(emu.st[key].astype(arr.dtype), arr), key
        info = step(k, vector_actions(env, rng))
        seen["illegal"] += int(info["is_illegal"].sum())
        seen["ambiguous"] += int(info["is_ambiguous"].sum())
        seen["over"] += int(info["newly_done"].sum())
    assert seen["illegal"] and seen["ambiguous"], seen
    env.close()


def test_ambiguous_action_registers_no_alarm_icaps_2021():
    """l2rpn_icaps_2021: an ambiguous action that raises an alarm registers nothing in the attention budget (grid2op's
    register_action returns early, attention_budget.py:150), the same alarm with a valid action is charged; budgets, last alarms
    and is_ambiguous equal an unmodified environment's"""
    if env_grid("l2rpn_icaps_2021") is None:
        pytest.skip("reference data not available")
    import grid2op_b200.backend  # noqa: F401
    import grid2op
    from grid2op.Parameters import Parameters
    from oracle_engine import COracleSeriesEngine
    from grid2op_b200.alarm import load_alarm_zones
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import list_scenarios, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    budget = dict(max_budget=3.0, budget_per_ts=0.1, alarm_cost=1.0, init_budget=2.0)
    grid = env_grid("l2rpn_icaps_2021")
    gm = GridModel(grid)
    env_dir = os.path.dirname(grid)
    cdir = os.path.join(env_dir, "chronics")
    folder = list_scenarios(cdir)[0]
    chron = load_scenarios(cdir, gm, scenarios=[folder])
    p = Parameters()
    p.NO_OVERFLOW_DISCONNECTION = True
    B = 2
    envs = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for i in range(B):
            e = grid2op.make("l2rpn_icaps_2021", test=True, backend=_host_backend()(), param=p, _add_to_name=f"amb_alarm{i}",
                             kwargs_attention_budget=dict(budget), opponent_init_budget=0., opponent_budget_per_ts=0.)
            e.set_id(0)
            e.reset()
            envs.append(e)
    th = np.asarray(envs[0].get_thermal_limit(), dtype=np.float32)
    benv = BatchedEnv(gm, chron, B, scen=np.zeros(B, np.int32), t0=np.zeros(B, np.int32), thermal_limit_a=th, protections=False,
                      engine=COracleSeriesEngine(gm))
    benv.enable_alarms(load_alarm_zones(env_dir, gm), **budget, reward=False)
    benv.reset_step()
    sb = np.zeros((B, gm.dim_topo), np.int8); cb = np.zeros((B, gm.dim_topo), bool)
    p0 = int(benv.sub_pos[4, 0])
    sb[0, p0] = 1; cb[0, p0] = True                       # instance 0: set and change on one element, ambiguous
    alarm = np.zeros((B, benv._alarms.n), bool); alarm[:, 0] = True
    ref = []
    for i, e in enumerate(envs):
        spec = {"raise_alarm": [0]}
        if i == 0:
            spec.update(set_bus=sb[0].astype(int), change_bus=cb[0])
        o, r, d, info = e.step(e.action_space(spec))
        ref.append((o, info))
    _, _, binfo = benv.step(set_bus=sb, change_bus=cb, raise_alarm=alarm)
    st = benv.alarm_state()
    assert binfo["is_ambiguous"].tolist() == [True, False] == [bool(x[1]["is_ambiguous"]) for x in ref]
    for i, (o, info) in enumerate(ref):
        assert np.float32(o.attention_budget[0]) == st["budget"][i], (i, o.attention_budget, st["budget"][i])
        assert np.array_equal(o.last_alarm, st["last"][i]), i
    assert st["budget"][0] > st["budget"][1] and (st["last"][0] == -1).all() and st["last"][1][0] > 0
