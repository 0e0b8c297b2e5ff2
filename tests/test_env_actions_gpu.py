"""BatchedEnv's grid2op-native topology action on the tensor path (csrc/b200pf_env.cuh ``act_vec_instance``, ``b200pf_env_step_act``)
against the numpy path (``BatchedEnv._apply_actions``) on twin environments fed the same vector actions: after every step and masked
device reset, the state, rho / status / iterations, the plan counters, the observation and the reward, is_illegal, is_ambiguous
and the alert state are bit-equal.  Also what a vector-action step moves and waits for, the refusals, and a short run of the CUDA
engine next to unmodified environments."""
import ast
import os

import numpy as np
import pytest

from conftest import env_grid
from test_env_tensor_gpu import _compare, _compare_obs, _load


def _idf_rule_areas():
    """the substation areas of l2rpn_idf_2023's ``RulesByArea(...)`` in its config"""
    src = open(os.path.join(os.path.dirname(env_grid("l2rpn_idf_2023")), "config.py")).read()
    for node in ast.walk(ast.parse(src)):
        if isinstance(node, ast.Call) and getattr(node.func, "id", None) == "RulesByArea":
            return ast.literal_eval(node.args[0])
    raise AssertionError("RulesByArea not found")


def _pair(name, B, protections, th_scale=None, n_scen=None, planned=True, **kw):
    from grid2op_b200.batched_env import BatchedEnv
    from test_env_tensor_gpu import _flows
    gm, chron, env_dir, folders = _load(name, n_scen)
    kw = dict(kw, nb_timestep_cooldown_line=2, nb_timestep_cooldown_sub=2, protections=protections)
    if th_scale is not None:
        kw["thermal_limit_a"] = (_flows(gm, chron) * np.float32(th_scale)).astype(np.float32)
    envs = [BatchedEnv(gm, chron, B, **kw) for _ in range(2)]
    for e in envs:
        if protections and planned:
            e.engine.set_kernel_policy(e.engine.KERNEL_PLANNED)
    return envs, env_dir, folders


def vector_actions(env, rng, few=None):
    """random vector actions for the whole batch: a few substations set or changed, line statuses set or changed, line ends at -1,
    reconnections of disconnected lines through a busbar and through change_line_status, and some ambiguous ones.  ``few``: (subs,
    lines) the only substations and lines acted on, each substation set whole to one of two busbar patterns or changed whole, so
    that a large batch reaches few distinct topologies (the planned kernel's plan cache)"""
    B, gm = env.batch, env.gm
    nt, nl = gm.dim_topo, gm.n_line
    lor, lex = env.line_or_pos, env.line_ex_pos
    on = env.line_status()
    if few is None:
        sub = rng.random((B, gm.n_sub)) < 2.0 / gm.n_sub
        touched = sub[:, env.sub_of_pos] & (rng.random((B, nt)) < 0.5)
        use_set = (rng.random((B, gm.n_sub)) < 0.5)[:, env.sub_of_pos]
        sb = np.where(touched & use_set, np.where(rng.random((B, nt)) < 0.8, 1, 2), 0).astype(np.int8)
        cb = touched & ~use_set & (rng.random((B, nt)) < 0.5)
        line_ok = np.ones(nl, bool)
    else:
        subs, lines = few
        patterns = np.stack([np.ones(nt, np.int8), np.where(np.arange(nt) % 2 == 0, 1, 2)])
        sub = np.zeros((B, gm.n_sub), bool)
        sub[:, subs] = rng.random((B, len(subs))) < 0.3
        touched = sub[:, env.sub_of_pos]
        use_set = (rng.random((B, gm.n_sub)) < 0.7)[:, env.sub_of_pos]
        pat = patterns[rng.integers(0, 2, B)]
        sb = np.where(touched & use_set, pat, 0).astype(np.int8)
        cb = touched & ~use_set
        line_ok = np.zeros(nl, bool); line_ok[lines] = True
    pick = (rng.random((B, nl)) < 1.5 / line_ok.sum()) & line_ok[None, :]
    r = rng.random((B, nl))
    ss = np.where(pick & (r < 0.3), np.where(on, -1, 1), 0).astype(np.int8)
    cs = pick & (r >= 0.3) & (r < 0.5)
    minus = pick & (r >= 0.8)
    sb[:, lor] = np.where(minus, -1, sb[:, lor])
    reco = ~on & (rng.random((B, nl)) < 0.3) & line_ok[None, :]
    via_bus = reco & (rng.random((B, nl)) < 0.5)
    sb[:, lor] = np.where(via_bus, 1, sb[:, lor])
    cs |= reco & ~via_bus & (ss == 0)
    amb = rng.random(B) < 0.03                            # set and change on one element
    p = rng.integers(0, nt, B) if few is None else env.sub_pos[few[0][0], 0] * np.ones(B, np.int64)
    sb[amb, p[amb]] = 1; cb[amb, p[amb]] = True
    return sb, cb, ss, cs


def _run(ref, tst, steps, seed, reset_every=5, few=None):
    import torch
    from test_alerts_gpu import _compare_alerts
    dev = torch.device("cuda", 0)
    t = lambda x: torch.as_tensor(np.asarray(x), device=dev)                     # noqa: E731
    rng = np.random.default_rng(seed)
    seen = dict(illegal=0, ambiguous=0, game_over=0, resets=0)
    rho, _, info = ref.reset_step()
    out = tst.step_tensors(from_reset=True)
    _compare(-1, ref, (rho, info), tst, (out[0], out[2]), True)
    _compare_obs(-1, ref, tst)
    alerts = ref._alerts is not None
    for k in range(steps):
        if reset_every and k and k % reset_every == 0 and ref.done.any():
            idx = np.flatnonzero(ref.done)
            rows = (idx * 7 + k) % ref.chron.shape[1]
            ref.reset_instances(idx, rows)
            mask = np.zeros(ref.batch, bool); mask[idx] = True
            rr = np.zeros(ref.batch, np.int64); rr[idx] = rows
            tst.reset_instances(t(mask), t(rr))
            seen["resets"] += len(idx)
            assert ref.engine.plan_counters() == tst.engine.plan_counters(), k
            assert np.array_equal(ref.is_ambiguous, tst._dev["is_ambiguous"].cpu().numpy()), k
            _compare_obs(k, ref, tst)
        sb, cb, ss, cs = vector_actions(ref, rng, few)
        kw = {}
        if alerts:
            kw["raise_alert"] = rng.random((ref.batch, ref._alerts.n)) < 0.1
        rho, _, info = ref.step(set_bus=sb, change_bus=cb, set_line_status=ss, change_line_status=cs, **kw)
        if alerts:
            kw["raise_alert"] = t(kw["raise_alert"])
        rb, _, ib = tst.step_tensors(set_bus=t(sb), change_bus=t(cb), set_line_status=t(ss), change_line_status=t(cs), **kw)
        _compare(k, ref, (rho, info), tst, (rb, ib), True)
        assert np.array_equal(info["is_ambiguous"], ib["is_ambiguous"].cpu().numpy()), k
        assert ref.engine.plan_counters() == tst.engine.plan_counters(), k
        _compare_obs(k, ref, tst)
        if alerts:
            _compare_alerts(k, ref, tst, info["rewards"]["alert"], ib["rewards"]["alert"])
        seen["illegal"] += int(info["is_illegal"].sum())
        seen["ambiguous"] += int(info["is_ambiguous"].sum())
        seen["game_over"] += int(info["newly_done"].sum())
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("protections", [False, True])
def test_vector_twins_case14_batch4096(cuda_required, protections):
    """MAX_SUB_CHANGED = 3, MAX_LINE_STATUS_CHANGED = 2, cooldowns 2, masked resets every 5 steps; with the protections on, thermal
    limits at 1.05 x the flows of the default topology and the planned-kernel policy, the actions on three substations and four lines
    (with fully random multi-substation actions a cascade met a topology the library had no plan for, DESIGN §8)"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    (ref, tst), env_dir, folders = _pair("l2rpn_case14_sandbox", 4096, protections, th_scale=1.05 if protections else None,
                                         max_sub_changed=3, max_line_status_changed=2)
    for e in (ref, tst):
        e.enable_observation(env_dir, scenarios=folders)
    seen = _run(ref, tst, 40, seed=3 + protections, few=([1, 4, 8], [0, 5, 9, 14]) if protections else None)
    assert seen["illegal"] and seen["ambiguous"] and seen["game_over"] and seen["resets"], seen
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
def test_vector_twins_idf_2023_rules_by_area(cuda_required):
    """l2rpn_idf_2023 at batch 1024 with its RulesByArea, its multi-area opponent and its alerts"""
    if env_grid("l2rpn_idf_2023") is None:
        pytest.skip("reference data not available")
    from test_multi_area_opponent_gpu import MULTI, SHORT, _idf_areas
    from grid2op_b200.opponent import opponent_seed
    (ref, tst), env_dir, folders = _pair("l2rpn_idf_2023", 1024, False, n_scen=2, rules_by_area=_idf_rule_areas())
    for e in (ref, tst):
        e.enable_alerts(_idf_areas())
        e.enable_observation(env_dir, scenarios=folders)
    ref.reset_step(); tst.step(from_reset=True)
    for e in (ref, tst):
        e.enable_opponent("GeometricOpponentMultiArea", _idf_areas(), seeds=[opponent_seed(s) for s in range(1024)], **MULTI, **SHORT)
    seen = _run(ref, tst, 25, seed=9)
    assert seen["illegal"] and seen["ambiguous"], seen
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
def test_vector_step_traffic_and_waits(cuda_required):
    """a vector-action step_tensors step copies no host-to-device byte and waits on the host as often as a legacy step with the
    same topology changes"""
    import torch
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    (a, b), _, _ = _pair("l2rpn_case14_sandbox", 512, False)
    dev = torch.device("cuda", 0)
    t = lambda x: torch.as_tensor(np.asarray(x), device=dev)                     # noqa: E731
    for e in (a, b):
        e.step_tensors(from_reset=True)
    rng = np.random.default_rng(1)
    from grid2op_b200.batched_env import random_substation_actions
    gm = a.gm
    for k in range(6):
        sub, bus = random_substation_actions(a, rng)
        sb = np.zeros((a.batch, gm.dim_topo), np.int8)
        for i in range(a.batch):
            n = a.sub_size[sub[i]]
            sb[i, a.sub_pos[sub[i], :n]] = bus[i, :n]
        ts, tb, tsb = t(sub), t(bus), t(sb)
        torch.cuda.synchronize()
        sa, sb0 = a.engine.env_stats(), b.engine.env_stats()
        a.step_tensors(ts, tb)
        b.step_tensors(set_bus=tsb)
        torch.cuda.synchronize()
        sa1, sb1 = a.engine.env_stats(), b.engine.env_stats()
        assert sb1["h2d_bytes"] == sb0["h2d_bytes"], k
        assert sb1["host_waits"] - sb0["host_waits"] == sa1["host_waits"] - sa["host_waits"], k
        assert np.array_equal(a.engine.env_get_state()["topo"], b.engine.env_get_state()["topo"]), k
    for e in (a, b):
        e.close()


@pytest.mark.gpu
def test_vector_step_refusals(cuda_required):
    """bad tensors are refused with nothing changed: wrong dtype / shape / device up front, values by the validation launch"""
    import torch
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    (e, _), _, _ = _pair("l2rpn_case14_sandbox", 64, False)
    gm = e.gm
    dev = torch.device("cuda", 0)
    e.step_tensors(from_reset=True)
    e.step_tensors(set_bus=torch.ones((64, gm.dim_topo), dtype=torch.int8, device=dev))
    torch.cuda.synchronize()
    before = (e.engine.env_get_state()["topo"].copy(), e._dev["line_cd"].clone(), e._dev["is_ambiguous"].clone(), e.n_steps)
    load = int(np.asarray(gm.load_pos)[0])
    sb_load = torch.zeros((64, gm.dim_topo), dtype=torch.int8, device=dev); sb_load[3, load] = -1
    bad = [dict(set_bus=torch.zeros((64, gm.dim_topo), dtype=torch.int32, device=dev)),
           dict(set_bus=torch.zeros((64, gm.dim_topo + 1), dtype=torch.int8, device=dev)),
           dict(set_bus=torch.zeros((64, gm.dim_topo), dtype=torch.int8)),
           dict(change_bus=torch.zeros((64, gm.dim_topo), dtype=torch.uint8, device=dev)),
           dict(set_bus=torch.full((64, gm.dim_topo), 3, dtype=torch.int8, device=dev)),
           dict(set_bus=sb_load),
           dict(set_line_status=torch.full((64, gm.n_line), 2, dtype=torch.int8, device=dev)),
           dict(set_line_status=torch.zeros((64, gm.n_line), dtype=torch.int8, device=dev),
                line_id=torch.zeros(64, dtype=torch.int32, device=dev), line_status=torch.ones(64, dtype=torch.int32, device=dev))]
    for kw in bad:
        with pytest.raises(ValueError):
            e.step_tensors(**kw)
    torch.cuda.synchronize()
    assert np.array_equal(before[0], e.engine.env_get_state()["topo"])
    assert torch.equal(before[1], e._dev["line_cd"]) and torch.equal(before[2], e._dev["is_ambiguous"]) and before[3] == e.n_steps
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,areas", [("l2rpn_case14_sandbox", False), ("l2rpn_idf_2023", True)])
def test_vector_actions_cuda_engine_vs_reference(cuda_required, name, areas):
    """a short run of the numpy path on the CUDA engine next to unmodified environments on the CUDA backend"""
    if env_grid(name) is None:
        pytest.skip("reference data not available")
    from test_env_actions_cpu import run_vector_actions
    saw = run_vector_actions(name, 10, 4, 12, areas=areas, n_sub_max=4 if areas else 3, cuda=True)
    assert saw["compared"] >= 10, saw
