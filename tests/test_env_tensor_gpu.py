"""BatchedEnv.step_tensors (device environment state, csrc/b200pf_env.cuh) against BatchedEnv.step (the numpy host path) on twin
environments fed the same actions: after every step the device topology, last busbars, cooldowns, done / illegal flags, current step
and chronics row, rho / status / iterations / disc_lines, the kernel configuration of the launch and the observation vectors and
rewards must be bit-equal.  Also the data path of a tensor step: what crosses PCIe and how often the host waits."""
import os

import numpy as np
import pytest

from conftest import env_grid


def _load(name, n_scen=None):
    from grid2op_b200.chronics import list_scenarios, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    grid = env_grid(name)
    gm = GridModel(grid)
    env_dir = os.path.dirname(grid)
    folders = list_scenarios(os.path.join(env_dir, "chronics"))
    if n_scen:
        folders = folders[:n_scen]
    chron = load_scenarios(os.path.join(env_dir, "chronics"), gm, scenarios=folders)
    return gm, chron, env_dir, folders


def _events(chron, gm, seed):
    """synthetic maintenance windows and hazards [n_scen, n_rows, n_line]"""
    rng = np.random.default_rng(seed)
    S, R, nl = chron.shape[0], chron.shape[1], gm.n_line
    m = np.zeros((S, R, nl), bool); h = np.zeros((S, R, nl), bool)
    for s in range(S):
        for _ in range(max(4, R // 12)):
            l, r0 = int(rng.integers(0, nl)), int(rng.integers(0, R - 8))
            (m if rng.random() < 0.5 else h)[s, r0:r0 + int(rng.integers(1, 6)), l] = True
    return m, h


def _flows(gm, chron):
    """largest current of every line (A, at least 1) over the first rows of the scenarios, default topology"""
    from grid2op_b200.batched_env import BatchedEnv
    e = BatchedEnv(gm, chron, 64, thermal_limit_a=np.ones(gm.n_line, np.float32))
    a = np.zeros(gm.n_line, np.float32)
    for _ in range(4):
        rho, _, _ = e.step(None, None)
        a = np.maximum(a, rho.max(0))
    e.close()
    return np.maximum(a, np.float32(1.0))


def _pair(name, B, protections, thermal=None, th_scale=None, events=False, cd=2, n_scen=None, observe=True, seed=0, planned=True):
    """``th_scale``: thermal limits at that multiple of the flows of the default topology (overloads and trips without ending every
    episode at once); ``planned``: with the protections on, the planned-kernel policy (random actions over a large batch reach more
    new topologies per step than the automatic policy builds plans for, and past 17 buses the planned kernel is the only one with
    the protections on); False keeps the automatic policy"""
    from grid2op_b200.batched_env import BatchedEnv
    gm, chron, env_dir, folders = _load(name, n_scen)
    kw = dict(nb_timestep_cooldown_line=cd, nb_timestep_cooldown_sub=cd, protections=protections)
    if thermal is not None:
        kw["thermal_limit_a"] = np.full(gm.n_line, thermal, np.float32)
    if th_scale is not None:
        kw["thermal_limit_a"] = (_flows(gm, chron) * np.float32(th_scale)).astype(np.float32)
    if events:
        kw["maintenance"], kw["hazards"] = _events(chron, gm, seed)
    envs = [BatchedEnv(gm, chron, B, **kw) for _ in range(2)]
    if protections and planned:
        for e in envs:
            e.engine.set_kernel_policy(e.engine.KERNEL_PLANNED)
    if observe:
        for e in envs:
            e.enable_observation(env_dir, scenarios=folders)
    return envs


def _actions(env, rng, line_only=False):
    """random substation and line actions; line statuses +-1 and +-2 (any sign is a valid status); ``line_only``: no substation
    action (the bus count stays that of the default topology)"""
    from grid2op_b200.batched_env import random_substation_actions
    B, gm = env.batch, env.gm
    sub, bus = random_substation_actions(env, rng)
    bus[rng.random((B, env.max_sub_size)) < 0.15] = 0
    sub[(rng.random(B) < 0.55) | line_only] = -1
    line = np.where(rng.random(B) < (0.4 if line_only else 0.25), rng.integers(0, gm.n_line, B), -1)
    lst = np.where(rng.random(B) < 0.5, -1, 1) * rng.integers(1, 3, B)
    return sub, bus, line, lst


def _host_state(e):
    return dict(topo=e.topo.copy(), last_bus=e.last_bus.copy(), line_cd=e.line_cooldown.copy(), sub_cd=e.sub_cooldown.copy(),
                done=e.done.copy(), is_illegal=np.asarray(e.is_illegal).copy(), current_step=e.current_step.copy(),
                row=(e.row % e.chron.shape[1]).astype(np.int32))


def _dev_state(e):
    d = e._dev
    s = e.engine.env_get_state()
    return dict(topo=s["topo"], last_bus=d["last_bus"].cpu().numpy(), line_cd=d["line_cd"].cpu().numpy(), sub_cd=d["sub_cd"].cpu().numpy(),
                done=d["done"].cpu().numpy(), is_illegal=d["is_illegal"].cpu().numpy(), current_step=d["current_step"].cpu().numpy(),
                row=s["t"])


def _compare(k, ref, ref_out, tst, tst_out, tensor_mode):
    import torch
    torch.cuda.synchronize()
    a, b = _host_state(ref), (_dev_state(tst) if tensor_mode else _host_state(tst))
    for key in a:
        bad = np.argwhere(a[key] != b[key])[:5]
        assert not len(bad), (k, key, bad, [(int(a[key][tuple(x)]), int(b[key][tuple(x)])) for x in bad])
    if tensor_mode:            # the device topology is the authority: the host path must agree with it
        assert np.array_equal(tst.engine.env_get_state()["topo"], a["topo"]), k
    rho_a, info_a = ref_out
    rho_b, info_b = tst_out
    cv = lambda x: x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)      # noqa: E731
    assert np.array_equal(rho_a.view(np.int32), cv(rho_b).view(np.int32)), k
    for key in ("status", "iters", "is_illegal", "newly_done"):
        assert np.array_equal(np.asarray(info_a[key]), cv(info_b[key])), (k, key)
    if info_a["disc_lines"] is not None:
        assert np.array_equal(info_a["disc_lines"], cv(info_b["disc_lines"])), k
    assert ref.engine.last_launch_info()["config"] == tst.engine.last_launch_info()["config"], k
    assert ref.nb_cap == tst.nb_cap and ref.n_illegal == tst.n_illegal, (k, ref.nb_cap, tst.nb_cap, ref.n_illegal, tst.n_illegal)


def _run_twins(ref, tst, steps, seed, reset_every=0, alternate=0, line_only=False):
    """``alternate`` > 0: the tensor twin switches between step_tensors and step every ``alternate`` steps.  After a reset both
    twins are observed before the next step too (the reset observation, then the step's)."""
    import torch
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(seed)
    seen = dict(illegal=0, trips=0, game_over=0, resets=0, warp=0)
    t = lambda x: torch.as_tensor(np.asarray(x), device=dev)                     # noqa: E731
    rho, _, info = ref.reset_step()
    out_b = tst.step_tensors(from_reset=True)
    _compare(-1, ref, (rho, info), tst, (out_b[0], out_b[2]), True)
    if ref._obs is not None:
        _compare_obs(-1, ref, tst)
    for k in range(steps):
        tensor_mode = not alternate or (k // alternate) % 2 == 0
        if reset_every and k and k % reset_every == 0 and ref.done.any():
            idx = np.flatnonzero(ref.done)
            rows = (idx * 7 + k) % ref.chron.shape[1]
            ref.reset_instances(idx, rows)
            if tensor_mode:
                mask = np.zeros(ref.batch, bool); mask[idx] = True
                r = np.zeros(ref.batch, np.int64); r[idx] = rows
                tst.reset_instances(t(mask), t(r))
            else:
                tst.reset_instances(idx, rows)
            seen["resets"] += len(idx)
            assert ref.engine.plan_counters() == tst.engine.plan_counters(), k
            if ref._obs is not None:
                _compare_obs(k, ref, tst)
        sub, bus, line, lst = _actions(ref, rng, line_only)
        rho, _, info = ref.step(sub, bus, line, lst)
        if tensor_mode:
            rb, _, ib = tst.step_tensors(t(sub), t(bus), t(line), t(lst))
        else:
            rb, _, ib = tst.step(sub, bus, line, lst)
        _compare(k, ref, (rho, info), tst, (rb, ib), tensor_mode)
        assert ref.engine.plan_counters() == tst.engine.plan_counters(), k
        seen["warp"] += ref.engine.plan_stats()["last_kernel"] == "warp_pivoting"
        if ref._obs is not None:
            _compare_obs(k, ref, tst)
        seen["illegal"] += int(np.asarray(info["is_illegal"]).sum())
        seen["game_over"] += int(info["newly_done"].sum())
        if info["disc_lines"] is not None:
            seen["trips"] += int((info["disc_lines"] >= 0).sum())
    return seen


def _compare_obs(k, ref, tst):
    import torch
    oa, ra = ref.observe()
    ob, rb = tst.observe()
    torch.cuda.synchronize()
    bad = torch.nonzero(oa.view(torch.int32) != ob.view(torch.int32))[:8].tolist()      # (bitwise: NaN records of failed solves)
    assert not bad and torch.equal(ra.view(torch.int32), rb.view(torch.int32)), (k, bad, [(oa[i, j].item(), ob[i, j].item()) for i, j in bad],
                                                                               torch.nonzero(ra.view(torch.int32) != rb.view(torch.int32))[:5].tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("protections", [False, True])
def test_twins_case14_batch4096(cuda_required, protections):
    """case14 at batch 4096, 60 steps, cooldowns 2, masked resets of the finished instances every 5 steps; thermal limits low
    enough for overflows (150 A) or, with the protections on, for trips (1.05 x the flows of the default topology; the planned
    kernel and the host-side cascade)"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    ref, tst = _pair("l2rpn_case14_sandbox", 4096, protections, **({"th_scale": 1.05} if protections else {"thermal": 150.0}))
    seen = _run_twins(ref, tst, 60, seed=11 + protections, reset_every=5)
    assert seen["illegal"] and seen["game_over"] and seen["resets"], seen
    assert seen["trips"] or not protections, seen
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
def test_twins_case14_planned_protections(cuda_required):
    """protections on the planned kernel with the host-side cascade, thermal limits at 0.9 x the flows of the default topology"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    ref, tst = _pair("l2rpn_case14_sandbox", 1024, True, th_scale=0.9)
    seen = _run_twins(ref, tst, 30, seed=5, reset_every=5)
    assert seen["illegal"] and seen["game_over"] and seen["trips"] and seen["resets"], seen
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
def test_twins_neurips_track1_maintenance_hazards(cuda_required):
    """l2rpn_neurips_2020_track1 at batch 1000, 40 steps, maintenance windows and hazards, protections on (the planned kernel and
    the host-side cascade), out-of-service shunts (the isolated-busbar rule)"""
    if env_grid("l2rpn_neurips_2020_track1") is None:
        pytest.skip("reference data not available")
    ref, tst = _pair("l2rpn_neurips_2020_track1", 1000, True, th_scale=1.1, events=True, cd=2, n_scen=2, seed=3)
    seen = _run_twins(ref, tst, 40, seed=21, reset_every=5)
    assert seen["illegal"] and seen["game_over"] and seen["trips"] and seen["resets"], seen
    assert (ref.line_cooldown > 0).any() or ref.done.all()
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,steps", [("rte_case5_example", 512, 30), ("l2rpn_wcci_2022_dev", 256, 12)])
def test_twins_other_grids(cuda_required, name, B, steps):
    """protections on, thermal limits at 1.1 x the flows of the default topology"""
    if env_grid(name) is None:
        pytest.skip("reference data not available")
    ref, tst = _pair(name, B, True, th_scale=1.1, n_scen=2, observe=name != "rte_case5_example")
    seen = _run_twins(ref, tst, steps, seed=2, reset_every=4)
    assert seen["illegal"] and seen["game_over"] and seen["trips"] and seen["resets"], seen
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("alternate", [0, 3])
def test_twins_case14_warp_kernel_device_cascade(cuda_required, alternate):
    """protections on under the automatic kernel policy: line actions only keep every instance within 17 buses, so the warp kernel
    runs and cascades on the device (the library's device topology runs ahead of its host mirror until the next plan lookup); masked
    resets of the finished instances every 5 steps look their plans up in the same calls on both twins.  ``alternate``: the tensor
    twin switches between step_tensors and step every 3 steps."""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    ref, tst = _pair("l2rpn_case14_sandbox", 4096, True, th_scale=1.05, planned=False)
    seen = _run_twins(ref, tst, 40, seed=8, reset_every=5, alternate=alternate, line_only=True)
    assert seen["warp"] >= 30 and seen["illegal"] and seen["game_over"] and seen["trips"] and seen["resets"], seen
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
def test_alternating_host_and_tensor_steps(cuda_required):
    """a run that switches between step_tensors and step every 3 steps stays bit-equal to a host-only twin"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    ref, tst = _pair("l2rpn_case14_sandbox", 2048, True, th_scale=1.05)
    seen = _run_twins(ref, tst, 30, seed=4, reset_every=5, alternate=3)
    assert seen["illegal"] and seen["game_over"] and seen["trips"] and seen["resets"], seen
    for e in (ref, tst):
        e.close()


@pytest.mark.gpu
def test_tensor_step_data_path(cuda_required):
    """a do-nothing tensor step copies nothing host-to-device and only the control words device-to-host, with one host wait; a
    step with actions copies back the wait words plus whole topology rows, never rho, a result record or a cooldown array;
    step_tensors -> observe -> a torch reduction needs no further host synchronisation"""
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    import torch
    dev = torch.device("cuda", 0)
    (env,) = _pair("l2rpn_case14_sandbox", 4096, False)[:1]
    gm, B = env.gm, env.batch
    env.step_tensors(from_reset=True)
    env.observe()
    torch.cuda.synchronize()
    s0, o0 = env.engine.env_stats(), env.engine.obs_stats()
    none = torch.full((B,), -1, dtype=torch.int32, device=dev)
    env.step_tensors(none, torch.zeros((B, env.max_sub_size), dtype=torch.int8, device=dev), none, torch.zeros(B, dtype=torch.int32, device=dev))
    torch.cuda.set_sync_debug_mode("error")          # a torch operation that waits for the device would raise
    try:
        obs, rew = env.observe()
        total = rew.sum()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    s1, o1 = env.engine.env_stats(), env.engine.obs_stats()
    assert s1["h2d_bytes"] == s0["h2d_bytes"] and o1["h2d_bytes"] == o0["h2d_bytes"]
    assert s1["d2h_bytes"] - s0["d2h_bytes"] == 32 and s1["host_waits"] - s0["host_waits"] == 1   # step, observe, sum: one wait
    assert o1["d2h_bytes"] == o0["d2h_bytes"]                   # no series fetch: rho / records / status stay on the device
    assert torch.isfinite(total).item()
    rng = np.random.default_rng(0)
    for _ in range(3):
        sub, bus, line, lst = _actions(env, rng)
        s0 = env.engine.env_stats()
        env.step_tensors(*(torch.as_tensor(x, device=dev) for x in (sub, bus, line, lst)))
        s1 = env.engine.env_stats()
        extra = s1["d2h_bytes"] - s0["d2h_bytes"] - 32
        assert extra % (4 + gm.n_topo_in) == 0 and s1["n_dirty"] <= extra // (4 + gm.n_topo_in) <= B, (extra, s1)
        assert s1["h2d_bytes"] == s0["h2d_bytes"]
    assert env.engine.obs_stats()["d2h_bytes"] == o0["d2h_bytes"]
    env.close()


@pytest.mark.gpu
def test_invalid_actions_leave_the_state_unchanged(cuda_required):
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    import torch
    dev = torch.device("cuda", 0)
    (env,) = _pair("l2rpn_case14_sandbox", 64, False, observe=False)[:1]
    gm, B = env.gm, env.batch
    env.step_tensors(from_reset=True)
    before = _dev_state(env)
    sub = torch.full((B,), -1, dtype=torch.int32, device=dev)
    bus = torch.zeros((B, env.max_sub_size), dtype=torch.int8, device=dev)
    line = torch.full((B,), -1, dtype=torch.int32, device=dev)
    lst = torch.zeros(B, dtype=torch.int32, device=dev)
    bad = [(sub.clone().fill_(gm.n_sub), bus, line, lst), (sub, bus, line.clone().fill_(-2), lst),
           (sub.clone().fill_(1), bus.clone().fill_(3), line, lst), (sub.clone().fill_(1), bus.clone().fill_(-2), line, lst),
           (sub, bus, line.clone().fill_(gm.n_line), lst.clone().fill_(1))]
    for args in bad:
        with pytest.raises(ValueError):
            env.step_tensors(*args)
        after = _dev_state(env)
        for key in before:
            assert np.array_equal(before[key], after[key]), key
    with pytest.raises(ValueError):
        env.step_tensors(sub.to(torch.float32), bus, line, lst)
    with pytest.raises(ValueError):
        env.step_tensors(sub.cpu(), bus, line, lst)
    with pytest.raises(ValueError):
        env.step_tensors(sub[:-1], bus, line, lst)
    env.close()
