"""BatchedEnv's discrete action ids on the tensor path (``step_tensors(action_id=...)``, ``b200pf_env_step_ids``: each instance reads
its own row of the action table the library holds on the device) against the same actions as the four vectors, gathered from the
table with torch, on twin environments: after every step and masked device reset, the state, info, rho, the plan counters, the
observation and the reward are bit-equal.  Also what an id step moves and waits for, the refusals, and a short run of the CUDA
engine next to unmodified environments."""
import numpy as np
import pytest

from conftest import env_grid
from test_env_actions_gpu import _idf_rule_areas, _pair
from test_env_tensor_gpu import _compare, _compare_obs, _dev_state


def _table(env):
    from grid2op_b200.action_table import ActionTable
    return ActionTable.unitary(env.gm)


def _few_rows(env, T, subs, lines):
    """ids of the rows acting only on the substations ``subs`` (two of each kind per substation) and the lines ``lines``, and
    do nothing: a large batch then reaches few distinct topologies (the planned kernel's plan cache, DESIGN §8)"""
    keep = [0]
    sub_of = env.sub_of_pos
    per = {}
    for k in range(1, T.n):
        pos = np.flatnonzero((T.set_bus[k] != 0) | T.change_bus[k])
        ln = np.flatnonzero((T.set_line_status[k] != 0) | T.change_line_status[k])
        if len(ln):
            if set(ln) <= set(lines):
                keep.append(k)
            continue
        s = set(sub_of[pos].tolist())
        if len(s) == 1 and s <= set(subs):
            key = (s.pop(), bool(T.change_bus[k].any()))
            if per.get(key, 0) < 2:
                per[key] = per.get(key, 0) + 1
                keep.append(k)
    return np.asarray(keep)


def _compare_twins(k, a, b, out_a, out_b):
    import torch
    torch.cuda.synchronize()
    sa, sb = _dev_state(a), _dev_state(b)
    for key in sa:
        assert np.array_equal(sa[key], sb[key]), (k, key)
    (ra, ia), (rb, ib) = out_a, out_b
    assert torch.equal(ra.view(torch.int32), rb.view(torch.int32)), k
    assert ("is_ambiguous" in ia) == ("is_ambiguous" in ib), k   # (a reset step takes no action)
    for key in ("status", "iters", "is_illegal", "newly_done", "is_ambiguous"):
        if key in ia:
            assert torch.equal(ia[key], ib[key]), (k, key)
    if ia["disc_lines"] is not None:
        assert torch.equal(ia["disc_lines"], ib["disc_lines"]), k
    assert a.engine.plan_counters() == b.engine.plan_counters(), k
    assert a.nb_cap == b.nb_cap and a.n_illegal == b.n_illegal, k
    if a._alerts is not None:
        for key, v in a.engine.alert_get_state().items():
            assert np.array_equal(np.asarray(v), np.asarray(b.engine.alert_get_state()[key])), (k, key)
        assert torch.equal(ia["rewards"]["alert"], ib["rewards"]["alert"]), k
    _compare_obs(k, a, b)


def _run(ids_env, vec_env, T, rows, steps, seed, reset_every=5):
    """``ids_env`` steps with ids drawn on the GPU from ``rows``, ``vec_env`` with the same rows gathered by torch"""
    import torch
    dev = torch.device("cuda", 0)
    tab = [torch.as_tensor(np.array(x), device=dev) for x in (T.set_bus, T.change_bus, T.set_line_status, T.change_line_status)]
    rows_d = torch.as_tensor(rows, device=dev)
    g = torch.Generator(device=dev); g.manual_seed(seed)
    seen = dict(illegal=0, ambiguous=0, game_over=0, resets=0)
    a, b = ids_env.step_tensors(from_reset=True), vec_env.step_tensors(from_reset=True)
    _compare_twins(-1, ids_env, vec_env, (a[0], a[2]), (b[0], b[2]))
    alerts = ids_env._alerts is not None
    B = ids_env.batch
    for k in range(steps):
        if reset_every and k and k % reset_every == 0:
            done = ids_env._dev["done"].clone()
            if bool(done.any()):
                rr = (torch.arange(B, device=dev) * 7 + k) % ids_env.chron.shape[1]
                for e in (ids_env, vec_env):
                    e.reset_instances(done, rr)
                seen["resets"] += int(done.sum())
                torch.cuda.synchronize()
                assert ids_env.engine.plan_counters() == vec_env.engine.plan_counters(), k
                _compare_obs(k, ids_env, vec_env)
        ids = rows_d[torch.randint(0, len(rows), (B,), device=dev, generator=g)]
        kw = {}
        if alerts:
            kw["raise_alert"] = torch.rand((B, ids_env._alerts.n), device=dev, generator=g) < 0.1
        ra, _, ia = ids_env.step_tensors(action_id=ids, **kw)
        rb, _, ib = vec_env.step_tensors(set_bus=tab[0][ids], change_bus=tab[1][ids], set_line_status=tab[2][ids],
                                         change_line_status=tab[3][ids], **kw)
        _compare_twins(k, ids_env, vec_env, (ra, ia), (rb, ib))
        seen["illegal"] += int(ia["is_illegal"].sum())
        seen["ambiguous"] += int(ia["is_ambiguous"].sum())
        seen["game_over"] += int(ia["newly_done"].sum())
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("protections", [False, True])
def test_id_twins_case14_batch4096(cuda_required, protections):
    """the unitary table (487 rows), MAX_SUB_CHANGED = 3, MAX_LINE_STATUS_CHANGED = 2, cooldowns 2, masked resets every 5 steps;
    with the protections on, thermal limits at 1.05 x the flows of the default topology, the planned-kernel policy and the rows of
    three substations and four lines, as the vector twins do"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    (a, b), env_dir, folders = _pair("l2rpn_case14_sandbox", 4096, protections, th_scale=1.05 if protections else None,
                                     max_sub_changed=3, max_line_status_changed=2)
    T = _table(a)
    assert T.n == 487
    for e in (a, b):
        e.enable_observation(env_dir, scenarios=folders)
    a.set_action_table(T)
    rows = _few_rows(a, T, [1, 4, 8], [0, 5, 9, 14]) if protections else np.arange(T.n)
    seen = _run(a, b, T, rows, 40, seed=3 + protections)
    assert seen["illegal"] and seen["game_over"] and seen["resets"], seen
    for e in (a, b):
        e.close()


@pytest.mark.gpu
def test_id_twins_idf_2023_full_table(cuda_required):
    """l2rpn_idf_2023 at batch 1024 with the full table (147,260 rows), its RulesByArea, its multi-area opponent and its alerts"""
    if env_grid("l2rpn_idf_2023") is None:
        pytest.skip("reference data not available")
    from test_multi_area_opponent_gpu import MULTI, SHORT, _idf_areas
    from grid2op_b200.opponent import opponent_seed
    (a, b), env_dir, folders = _pair("l2rpn_idf_2023", 1024, False, n_scen=2, rules_by_area=_idf_rule_areas())
    T = _table(a)
    assert T.n == 147260
    for e in (a, b):
        e.enable_alerts(_idf_areas())
        e.enable_observation(env_dir, scenarios=folders)
    a.step(from_reset=True); b.step(from_reset=True)
    for e in (a, b):
        e.enable_opponent("GeometricOpponentMultiArea", _idf_areas(), seeds=[opponent_seed(s) for s in range(1024)], **MULTI, **SHORT)
    a.set_action_table(T)
    seen = _run(a, b, T, np.arange(T.n), 20, seed=9)
    assert seen["illegal"], seen
    for e in (a, b):
        e.close()


@pytest.mark.gpu
def test_ids_alternating_host_and_tensor_paths(cuda_required):
    """one environment alternating step (numpy ids) and step_tensors (device ids) next to the numpy path fed the same rows as
    vectors"""
    import torch
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    (ref, tst), _, _ = _pair("l2rpn_case14_sandbox", 256, False, max_sub_changed=2, max_line_status_changed=2)
    T = _table(ref)
    tst.set_action_table(T)
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(5)
    rho, _, info = ref.reset_step()
    out = tst.step_tensors(from_reset=True)
    _compare(-1, ref, (rho, info), tst, (out[0], out[2]), True)
    n_illegal = 0
    for k in range(24):
        ids = rng.integers(0, T.n, ref.batch)
        rho, _, info = ref.step(set_bus=T.set_bus[ids], change_bus=T.change_bus[ids], set_line_status=T.set_line_status[ids],
                                change_line_status=T.change_line_status[ids])
        if (k // 3) % 2:
            rb, _, ib = tst.step(action_id=ids)
            _compare(k, ref, (rho, info), tst, (rb, ib), False)
            assert np.array_equal(info["is_ambiguous"], ib["is_ambiguous"]), k
        else:
            rb, _, ib = tst.step_tensors(action_id=torch.as_tensor(ids, device=dev))
            _compare(k, ref, (rho, info), tst, (rb, ib), True)
            assert np.array_equal(info["is_ambiguous"], ib["is_ambiguous"].cpu().numpy()), k
        n_illegal += int(info["is_illegal"].sum())
    assert n_illegal > 0
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
def test_id_step_traffic_and_waits(cuda_required):
    """an id step copies no host-to-device byte and no action data device to device, and waits on the host as often as the vector
    step with the same topology changes"""
    import torch
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    (a, b), _, _ = _pair("l2rpn_case14_sandbox", 512, False)
    T = _table(a)
    a.set_action_table(T)
    dev = torch.device("cuda", 0)
    tab = [torch.as_tensor(np.array(x), device=dev) for x in (T.set_bus, T.change_bus, T.set_line_status, T.change_line_status)]
    for e in (a, b):
        e.step_tensors(from_reset=True)
    g = torch.Generator(device=dev); g.manual_seed(1)
    vec_bufs = [a._dev[k].clone() for k in ("act_set_bus", "act_change_bus", "act_set_status", "act_change_status")]
    for k in range(6):
        ids = torch.randint(0, T.n, (a.batch,), device=dev, generator=g, dtype=torch.int32)
        vecs = [x[ids] for x in tab]
        torch.cuda.synchronize()
        sa0, sb0 = a.engine.env_stats(), b.engine.env_stats()
        a.step_tensors(action_id=ids)
        b.step_tensors(set_bus=vecs[0], change_bus=vecs[1], set_line_status=vecs[2], change_line_status=vecs[3])
        torch.cuda.synchronize()
        sa1, sb1 = a.engine.env_stats(), b.engine.env_stats()
        assert sa1["h2d_bytes"] == sa0["h2d_bytes"], k
        assert sa1["host_waits"] - sa0["host_waits"] == sb1["host_waits"] - sb0["host_waits"], k
        assert sa1["d2h_bytes"] - sa0["d2h_bytes"] == sb1["d2h_bytes"] - sb0["d2h_bytes"], k
        assert np.array_equal(a.engine.env_get_state()["topo"], b.engine.env_get_state()["topo"]), k
    # the vector buffers of the id environment were never written: the rows were read from the table in place
    for x, key in zip(vec_bufs, ("act_set_bus", "act_change_bus", "act_set_status", "act_change_status")):
        assert torch.equal(x, a._dev[key]), key
    for e in (a, b):
        e.close()


@pytest.mark.gpu
def test_id_step_refusals(cuda_required):
    """an id out of range from the device is refused by the validation launch with nothing changed; so are ids without a table,
    ids with vectors, a wrong dtype, shape or device; a table with a bad row is refused before anything is bound"""
    import torch
    from grid2op_b200.action_table import ActionTable
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    (e, f), _, _ = _pair("l2rpn_case14_sandbox", 64, False)
    gm = e.gm
    dev = torch.device("cuda", 0)
    e.step_tensors(from_reset=True)
    ok = torch.zeros(64, dtype=torch.int32, device=dev)
    with pytest.raises(ValueError):
        e.step_tensors(action_id=ok)                      # no table yet
    T = ActionTable.unitary(gm)
    e.set_action_table(T)
    e.step_tensors(action_id=torch.full((64,), 30, dtype=torch.int64, device=dev))
    torch.cuda.synchronize()
    before = (e.engine.env_get_state()["topo"].copy(), e._dev["line_cd"].clone(), e._dev["is_ambiguous"].clone(), e.n_steps)
    big = ok.clone(); big[7] = T.n
    neg = ok.clone(); neg[63] = -1
    bad = [dict(action_id=big), dict(action_id=neg), dict(action_id=torch.full((64,), 2 ** 40, dtype=torch.int64, device=dev)),
           dict(action_id=ok.to(torch.int16)), dict(action_id=ok[:32]), dict(action_id=ok.cpu()),
           dict(action_id=ok, set_bus=torch.zeros((64, gm.dim_topo), dtype=torch.int8, device=dev)),
           dict(action_id=ok, line_id=ok, line_status=ok)]
    for kw in bad:
        with pytest.raises(ValueError):
            e.step_tensors(**kw)
    torch.cuda.synchronize()
    assert np.array_equal(before[0], e.engine.env_get_state()["topo"])
    assert torch.equal(before[1], e._dev["line_cd"]) and torch.equal(before[2], e._dev["is_ambiguous"]) and before[3] == e.n_steps
    # the library checks the rows itself: a bad row fails the bind and the bound table stays
    sb = np.zeros((2, gm.dim_topo), np.int8); sb[1, int(np.asarray(gm.load_pos)[0])] = -1
    with pytest.raises(RuntimeError):
        e.engine.act_table_bind(sb, np.zeros((2, gm.dim_topo), bool), np.zeros((2, gm.n_line), np.int8), np.zeros((2, gm.n_line), bool))
    e.step_tensors(action_id=torch.full((64,), T.n - 1, dtype=torch.int32, device=dev))
    # a table built for another grid
    from grid2op_b200.gridmodel import GridModel
    other = GridModel(env_grid("rte_case5_example")) if env_grid("rte_case5_example") else None
    if other is not None:
        with pytest.raises(ValueError):
            f.set_action_table(ActionTable.unitary(other))
    for x in (e, f):
        x.close()


@pytest.mark.gpu
def test_ids_cuda_engine_vs_reference(cuda_required):
    """a short run of the id path on the CUDA engine next to unmodified environments on the CUDA backend stepping
    ``IdToAct.convert_act``"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    from test_action_table_cpu import run_ids
    saw = run_ids("l2rpn_case14_sandbox", 10, 4, 21, cuda=True)
    assert saw["compared"] >= 10, saw
