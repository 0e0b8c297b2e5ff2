"""The device environment bodies of BatchedEnv.step_tensors (csrc/b200pf_env.cuh) through their host build (tests/emu/env_emu.cpp)
next to the numpy BatchedEnv driven by the oracle adapter engines: after every step the topology, last busbars, both cooldown arrays,
done, is_illegal, current_step, n_illegal, the bus cap, the topology-dirty flag and the observe input record must be equal.  Random
mixed actions with protections off and on (reconnections through set_bus, illegal actions), maintenance windows and hazards, the
out-of-service-shunt busbar rule, resets, and the rejection of out-of-range inputs."""
import os

import numpy as np
import pytest

from conftest import env_grid

ENV = "l2rpn_neurips_2020_track1"


def _env(name, B, protections=False, events=None, cd_line=2, cd_sub=1, **kw):
    from oracle_engine import COracleSeriesEngine, EmuProtSeriesEngine
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import load_scenarios
    from grid2op_b200.gridmodel import GridModel
    grid = env_grid(name)
    gm = GridModel(grid)
    cdir = os.path.join(os.path.dirname(grid), "chronics")
    folder = os.path.join(cdir, sorted(os.listdir(cdir))[0])
    chron = load_scenarios(cdir, gm, scenarios=[folder])
    if events is not None:
        kw["maintenance"], kw["hazards"] = events(chron, gm)
    eng = (EmuProtSeriesEngine if protections else COracleSeriesEngine)(gm)
    env = BatchedEnv(gm, chron, B, scen=np.zeros(B, np.int32), t0=np.full(B, 1, np.int32), nb_timestep_cooldown_line=cd_line,
                     nb_timestep_cooldown_sub=cd_sub, protections=protections, engine=eng, **kw)
    calls = []
    orig = env.engine.series_set_topo
    env.engine.series_set_topo = lambda topo: (calls.append(1), orig(topo))[1]     # counts the host path's plan refreshes
    return env, calls


def _raw(env):
    """status before the isolated-busbar override, and disc_lines, as the library leaves them"""
    _, status, _, _ = env.engine.series_fetch(want_out=False)
    disc = env.fetch_state()["disc_lines"] if env.protections else None
    return status, disc


def _check(k, env, emu, ctl, dirty_calls):
    s, gm = emu.st, env.gm
    assert np.array_equal(s["topo"], env.topo), (k, np.argwhere(s["topo"] != env.topo)[:5])
    assert np.array_equal(s["last_bus"], env.last_bus), k
    assert np.array_equal(s["line_cd"], env.line_cooldown), k
    assert np.array_equal(s["sub_cd"], env.sub_cooldown), k
    assert np.array_equal(s["done"].astype(bool), env.done), k
    assert np.array_equal(s["is_illegal"].astype(bool), np.asarray(env.is_illegal)), k
    assert np.array_equal(s["current_step"], env.current_step), k
    assert np.array_equal(s["t"], env.row % env.chron.shape[1]), k
    assert emu.n_illegal == env.n_illegal, (k, emu.n_illegal, env.n_illegal)
    assert (ctl[0] > 0) == bool(dirty_calls), (k, int(ctl[0]), dirty_calls)
    if env.tight_cap:
        assert emu.bus_cap(ctl, gm.n_slot) == env.nb_cap, (k, emu.bus_cap(ctl, gm.n_slot), env.nb_cap)
    nl, ns = gm.n_line, gm.n_sub
    rec = s["obs_in"]
    assert np.array_equal(rec[:, :nl], env.line_cooldown) and np.array_equal(rec[:, nl:nl + ns], env.sub_cooldown), k
    assert np.array_equal(rec[:, nl + ns], env.current_step) and (rec[:, nl + ns + 1] == env.n_steps).all(), k
    assert np.array_equal(rec[:, nl + ns + 2] & 3, np.asarray(env.is_illegal) * 1 + env.done * 2), k


def _step(k, env, emu, calls, sub=None, bus=None, line=None, lst=None, from_reset=False):
    del calls[:]
    ctl = emu.step_apply(sub, bus, line, lst, from_reset=from_reset, tight_cap=env.tight_cap)
    assert ctl[2] == 0
    rho, done, info = env.step(sub, bus, line, lst, from_reset=from_reset)
    status, disc = _raw(env)
    emu.step_post(status, disc, from_reset=from_reset, stamp=env.n_steps, prot=env.protections)
    assert np.array_equal(emu.st["status_out"], info["status"]), k
    assert np.array_equal(emu.st["newly_done"].astype(bool), info["newly_done"]), k
    _check(k, env, emu, ctl, len(calls))
    return info


def _mixed_actions(env, rng):
    from grid2op_b200.batched_env import random_substation_actions
    B, gm = env.batch, env.gm
    sub, bus = random_substation_actions(env, rng)
    line = np.full(B, -1, np.int64); lst = np.zeros(B, np.int64)
    kind = rng.random(B)
    status = env.line_status()
    for i in range(B):
        if kind[i] >= 0.5:
            sub[i] = -1
            if kind[i] < 0.8:
                line[i] = int(rng.integers(0, gm.n_line))
                lst[i] = (-1 if status[i, line[i]] else 1) * int(rng.integers(1, 3))     # (any magnitude is a valid status)
    return sub, bus, line, lst


@pytest.mark.parametrize("seed,protections", [(0, False), (1, False), (3, False), (0, True), (2, True), (5, True)])
def test_random_mixed_actions_env_bodies(seed, protections):
    if env_grid(ENV) is None:
        pytest.skip("reference data not available")
    from env_emu import EmuEnvState
    env, calls = _env(ENV, 5, protections)
    emu = EmuEnvState(env)
    rng = np.random.default_rng(seed)
    seen = dict(illegal=0, reco=0, over=0, trips=0)
    _step(-1, env, emu, calls, from_reset=True)
    n_reset = 0
    for k in range(14):
        if k == 7:                                         # masked reset of the finished instances and of instance 0
            mask = env.done.copy(); mask[0] = True
            idx = np.flatnonzero(mask)
            env.reset_instances(idx, np.full(len(idx), 3))
            rows = np.zeros(env.batch, np.int32); rows[idx] = 3
            emu.reset(mask, rows)
            n_reset += len(idx)
            for key, arr in (("topo", env.topo), ("last_bus", env.last_bus), ("line_cd", env.line_cooldown), ("current_step", env.current_step)):
                assert np.array_equal(emu.st[key], arr), key
            assert np.array_equal(emu.st["t"], env.row % env.chron.shape[1])
            assert (emu.st["obs_in"][idx, -1] == 4).all() and (emu.st["obs_in"][idx, :-2] == 0).all()
        before = env.topo.copy()
        sub, bus, line, lst = _mixed_actions(env, rng)
        info = _step(k, env, emu, calls, sub, bus, line, lst)
        seen["illegal"] += int(np.asarray(info["is_illegal"]).sum())
        seen["over"] += int(info["newly_done"].sum())
        seen["reco"] += int(((before[:, env.line_or_pos] <= 0) & (env.topo[:, env.line_or_pos] > 0)).sum())
        if info["disc_lines"] is not None:
            seen["trips"] += int((info["disc_lines"] >= 0).sum())
    assert n_reset >= 1 and seen["illegal"] + seen["reco"] + seen["over"] > 0, seen
    assert seen["trips"] or not protections or seen["over"], seen
    env.close()


def test_maintenance_and_hazards_env_bodies():
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    from env_emu import EmuEnvState

    def events(chron, gm):
        R, nl = chron.shape[1], gm.n_line
        h = np.zeros((1, R, nl), bool); m = np.zeros((1, R, nl), bool)
        h[0, 5:9, 3] = True; h[0, 12:14, 7] = True; h[0, 13:20, 3] = True; m[0, 25:30, 10] = True
        return m, h

    env, calls = _env("l2rpn_case14_sandbox", 3, events=events, cd_line=0, cd_sub=0)
    emu = EmuEnvState(env)
    attempts = {7: 3, 10: 3, 15: 7, 22: 3, 27: 10, 31: 10}
    _step(-1, env, emu, calls, from_reset=True)
    for k in range(40):
        lid = np.full(3, -1); lst = np.zeros(3, np.int64)
        if k in attempts:
            lid[:] = attempts[k]; lst[:] = 1
        _step(k, env, emu, calls, line=lid, lst=lst)
    assert env.n_illegal >= 2 and (env.line_cooldown >= 0).all()
    env.close()


def test_isolated_busbar_rule_env_bodies():
    """l2rpn_neurips_2020_track1: every element of a substation whose shunt is out of service moved to busbar 2 ends the episode"""
    if env_grid(ENV) is None:
        pytest.skip("reference data not available")
    from env_emu import EmuEnvState
    env, calls = _env(ENV, 2)
    emu = EmuEnvState(env)
    gm = env.gm
    s_plain = [s for s in range(gm.n_sub) if s not in set(int(x) for x in gm.shunt_sub) and 3 <= env.sub_size[s] <= 5
               and not np.isin(s, gm.gen_sub)]
    sub = np.asarray([12, s_plain[0]], np.int64)
    bus = np.zeros((2, env.max_sub_size), np.int8)
    for i, s in enumerate(sub):
        bus[i, :env.sub_size[s]] = 2
    _step(0, env, emu, calls, sub, bus, np.full(2, -1), np.zeros(2, np.int64))
    assert env.done.tolist() == [True, False] and emu.st["status_out"][0] == 2
    env.close()


def test_out_of_range_inputs_are_rejected_with_the_state_unchanged():
    if env_grid("l2rpn_case14_sandbox") is None:
        pytest.skip("reference data not available")
    from env_emu import EmuEnvState
    env, calls = _env("l2rpn_case14_sandbox", 4)
    emu = EmuEnvState(env)
    gm, B = env.gm, 4
    before = {k: v.copy() for k, v in emu.st.items() if k not in ("ctl", "copy_list", "copy_rows")}
    none, zb = np.full(B, -1), np.zeros((B, env.max_sub_size), np.int8)
    cases = [(np.full(B, gm.n_sub), zb, None, None), (np.full(B, -2), zb, None, None), (np.zeros(B), np.full_like(zb, 3), None, None),
             (np.zeros(B), np.full_like(zb, -2), None, None), (None, None, np.full(B, gm.n_line), np.ones(B)),
             (none, zb, np.full(B, -5), np.ones(B))]
    for sub, bus, line, lst in cases:
        ctl = emu.step_apply(sub, bus, line, lst)
        assert ctl[2] != 0
        for k, v in before.items():
            assert np.array_equal(v, emu.st[k]), k
    ok = emu.step_apply(np.zeros(B), np.full_like(zb, 1), np.full(B, 0), np.full(B, -1))
    assert ok[2] == 0
    ok = emu.step_apply(None, None, np.full(B, 1), np.full(B, 7))           # any line status: > 0 reconnects, as the host path
    assert ok[2] == 0
    env.close()
