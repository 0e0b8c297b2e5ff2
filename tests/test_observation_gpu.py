"""The observe kernel (csrc/b200pf_obs.cuh) against a numpy restatement (tests/obs_engines.py ``restate_obs``) at batch 4096 over 50
steps of random substation and line actions with resets of finished instances, and its data path: it writes into the torch
tensors it is given, the result records never cross to the host, and step -> observe on one stream needs no host synchronisation."""
import os

import numpy as np
import pytest

from conftest import env_grid

ENV = "l2rpn_case14_sandbox"


def _env(B, reward="RedispReward"):
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import list_scenarios, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    grid = env_grid(ENV)
    gm = GridModel(grid)
    env_dir = os.path.dirname(grid)
    folders = list_scenarios(os.path.join(env_dir, "chronics"))
    chron = load_scenarios(os.path.join(env_dir, "chronics"), gm, scenarios=folders)
    a_lim = np.full(gm.n_line, 150.0, dtype=np.float32)          # 150 A: some lines run overloaded, the overflow counters move
    env = BatchedEnv(gm, chron, B, thermal_limit_a=a_lim, nb_timestep_cooldown_line=2, nb_timestep_cooldown_sub=2)
    n_obs = env.enable_observation(env_dir, reward=reward, scenarios=folders)
    return env, n_obs


@pytest.mark.gpu
def test_observe_kernel_equals_numpy_restatement(cuda_required):
    """obs bit-equal to the restatement; the reward within the summation-order difference of the kernel (32 lane partials in fp64
    combined by a butterfly) and the sequential fp64 sums of the restatement: rtol 1e-6."""
    if env_grid(ENV) is None:
        pytest.skip("reference data not available")
    import torch
    from grid2op_b200.batched_env import random_substation_actions
    from grid2op_b200.engine import OutputView
    from obs_engines import restate_obs
    B = 4096
    env, n_obs = _env(B)
    gm = env.gm
    t = env._obs["tables"]
    cnt = dict(ts_over=np.zeros((B, gm.n_line), np.int32), ts_prot=np.zeros((B, gm.n_line), np.int32), stamp=np.full(B, -1, np.int32),
               go_row=np.full(B, -1, np.int32))
    rng = np.random.default_rng(7)
    env.reset_step()
    n_go = n_ill = n_over = 0
    for k in range(52):
        if k:
            sub, bus = random_substation_actions(env, rng)
            sub[rng.random(B) < 0.6] = -1
            line = np.where(rng.random(B) < 0.2, rng.integers(0, gm.n_line, B), -1)
            lst = np.where(rng.random(B) < 0.5, -1, 1)
            env.step(sub, bus, line, lst)
        host_in = env.observe_inputs().copy()
        obs, rew = env.observe()
        torch.cuda.synchronize()
        rec, status, iters, rho = env.engine.series_fetch()
        d = env.engine.series_device_pointers()
        topo = np.empty((B, gm.n_topo_in), np.int8)
        t_next = np.empty(B, np.int32)
        from grid2op_b200.engine import load_library
        import ctypes as C
        lib = load_library()
        assert lib.b200pf_device_read(C.c_void_p(d["t"]), t_next.ctypes.data_as(C.c_void_p), C.c_size_t(t_next.nbytes)) == 0
        topo[:] = env.topo                  # (the device topology mirrors the host's: no protections here)
        ref = restate_obs(env, t, rec, rho, topo, t_next, cnt, host_in)
        got = obs.cpu().numpy()
        bad = np.argwhere(~((got == ref) | (np.isnan(got) & np.isnan(ref))))
        assert len(bad) == 0, (k, bad[:5], got[tuple(bad[0])], ref[tuple(bad[0])])
        # reward restated in fp64
        v = OutputView(gm, rec)
        r = t["reward"]; g = t["gen"]
        gp = v.unit_p[:, gm.n_hidden:].astype(np.float64)
        lp = env.chron[env.scen, np.where(t_next > 0, t_next - 1, env.chron.shape[1] - 1), :gm.n_load].astype(np.float64).sum(axis=1)
        mc = np.where(gp > 0, g["gen_cost_per_MW"][None, :].astype(np.float64), -np.inf).max(axis=1)
        mc = np.where(np.isfinite(mc), mc, 0.0)
        exp = ((r["max_regret"] - (gp.sum(axis=1) - lp) * r["dts_hours"] * mc) / lp).astype(np.float32)
        flags = host_in[:, -1]
        exp = np.where(flags & 1, np.float32(r["reward_illegal"]), exp)
        exp = np.where(flags & 2, np.float32(r["reward_min"]), exp)
        assert np.allclose(rew.cpu().numpy(), exp, rtol=1e-6, atol=0), k
        n_go += int((flags & 2).sum()); n_ill += int((flags & 1).sum()); n_over += int((cnt["ts_over"] > 0).sum())
        done = np.flatnonzero(env.done)
        if len(done) and k % 5 == 4:
            env.reset_instances(done)
    assert n_go > 0 and n_ill > 0 and n_over > 0, (n_go, n_ill, n_over)
    env.close()


@pytest.mark.gpu
def test_observe_data_path(cuda_required):
    """observe() writes into the caller's tensors; only the step's rho / status / iterations travel to the host (the engine's D2H
    byte counter), never a result record; a chain step -> observe -> torch reduction runs without a host synchronisation in between."""
    if env_grid(ENV) is None:
        pytest.skip("reference data not available")
    import torch
    B = 512
    env, n_obs = _env(B, reward="L2RPNReward")
    gm = env.gm
    env.reset_step()
    obs_t = torch.full((B, n_obs), float("nan"), dtype=torch.float32, device="cuda")
    rew_t = torch.full((B,), float("nan"), dtype=torch.float32, device="cuda")
    d2h0 = env.engine.obs_stats()["d2h_bytes"]
    sums = []
    for k in range(5):
        env.step()
        o, r = env.observe(obs_t, rew_t)
        assert o.data_ptr() == obs_t.data_ptr() and r.data_ptr() == rew_t.data_ptr()
        sums.append(o.sum(dim=1) + r)                   # consumed on torch's stream, ordered behind the observe launch
    st = env.engine.obs_stats()
    per_step = B * (4 + 4 + 4 * gm.n_line)              # status + iterations + rho of BatchedEnv.step's fetch
    assert st["d2h_bytes"] - d2h0 == 5 * per_step, (st, per_step)
    assert st["launches"] == 5 and st["h2d_bytes"] == 5 * B * 4 * (gm.n_line + gm.n_sub + 3)
    assert st["bytes_written_per_launch"] == B * (4 * n_obs + 4)
    torch.cuda.synchronize()
    assert torch.isfinite(obs_t).all() and torch.isfinite(rew_t).all()
    assert all(torch.isfinite(s).all() for s in sums)
    env.close()
