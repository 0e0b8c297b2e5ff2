"""TEST INFRASTRUCTURE: the observation layer (``PowerFlowEngine.obs_bind`` / ``observe``) on the host build of its kernel body
(tests/emu/obs_emu.cpp), added to the series stand-ins of tests/oracle_engine.py, so that ``BatchedEnv.observe`` can be stepped next
to unmodified grid2op environments on a machine without a GPU.  Also a numpy restatement of the observation vector for the GPU
kernel to be compared against."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from grid2op_b200.engine import OutputView, make_obs_desc
from grid2op_b200.observation import OBS_SOURCES
from oracle_engine import COracleSeriesEngine, EmuProtSeriesEngine

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
REPO = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libobs_emu.so")


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "obs_emu.cpp")
    deps = [src, os.path.join(REPO, "grid2op_b200", "csrc", "b200pf_obs.cuh"), os.path.join(REPO, "include", "b200pf.h")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++", "-o", LIB, src])
    return LIB


class _ObsHost:
    """obs_bind / observe_host on top of a series stand-in (its topology, chronics row index, records and rho are host arrays)."""

    def obs_bind(self, tables):
        self._obs_lib = C.CDLL(build())
        self._obs_lib.obs_emu_run.restype = C.c_int
        self._obs_desc, self._obs_keep = make_obs_desc(tables)
        gm, B = self.gm, self.B
        self._obs_n = int(tables["n_obs"])
        self._obs_kind = int(tables["reward_kind"])
        self._ts_over = np.zeros((B, gm.n_line), np.int32); self._ts_prot = np.zeros((B, gm.n_line), np.int32)
        self._stamp = np.full(B, -1, np.int32); self._go_row = np.full(B, -1, np.int32)
        self._sizes = np.array([gm.n_line, gm.n_sub, gm.n_gen, gm.n_hidden, gm.n_load, gm.n_storage, gm.n_shunt, gm.dim_topo, gm.n_topo_in,
                                gm.n_out], np.int32)
        self._lpos = np.ascontiguousarray(gm.line_or_pos, np.int32); self._epos = np.ascontiguousarray(gm.line_ex_pos, np.int32)

    def _t_now(self):
        return np.ascontiguousarray(getattr(self, "t32", self.t), dtype=np.int32)

    def observe_host(self, host_in, obs_out=None, reward_out=None):
        gm, B = self.gm, self.B
        obs = obs_out if obs_out is not None else np.empty((B, self._obs_n), np.float32)
        rew = reward_out if reward_out is not None else np.empty(B, np.float32)
        out = np.ascontiguousarray(self.out, np.float32)
        rho = np.ascontiguousarray(getattr(self, "rho", None) if getattr(self, "rho", None) is not None
                                   else OutputView(gm, out).a_or / self.th[None, :], np.float32)
        p = lambda a: a.ctypes.data_as(C.c_void_p)     # noqa: E731
        hin = np.ascontiguousarray(host_in, np.int32)
        topo = np.ascontiguousarray(self.topo, np.int8)
        t = self._t_now()
        scen = np.ascontiguousarray(self.scen, np.int32)
        chron = np.ascontiguousarray(self.chron, np.float32)
        th = np.ascontiguousarray(self.th, np.float32)
        rc = self._obs_lib.obs_emu_run(C.byref(self._obs_desc), p(self._sizes), p(self._lpos), p(self._epos), C.c_int(B), p(out), p(rho),
                                       p(topo), p(t), p(scen), p(chron), C.c_int(chron.shape[1]), p(th), p(hin), p(self._ts_over),
                                       p(self._ts_prot), p(self._stamp), p(self._go_row), p(obs), p(rew))
        assert rc == 0
        return obs, rew


class COracleObsSeriesEngine(_ObsHost, COracleSeriesEngine):
    pass


class EmuProtObsSeriesEngine(_ObsHost, EmuProtSeriesEngine):
    pass


def restate_obs(env, tables, rec, rho, topo, t_next, counters, host_in):
    """numpy restatement of the observation vector of every instance (same per-element float32 operations as the kernel) from the
    result records / rho / device topology fetched from the engine and the BatchedEnv host state.  ``counters``: dict with
    ``ts_over`` / ``ts_prot`` int32 [B, n_line], advanced here exactly as the kernel does."""
    gm, B = env.gm, env.batch
    nl, ns, nh = gm.n_line, gm.n_sub, gm.n_hidden
    v = OutputView(gm, rec)
    f = np.float32
    cd_l, cd_s = host_in[:, :nl], host_in[:, nl:nl + ns]
    cur, stamp, flags = host_in[:, nl + ns], host_in[:, nl + ns + 1], host_in[:, nl + ns + 2]
    go = (flags & 2) != 0
    row = np.where(t_next > 0, t_next - 1, env.chron.shape[1] - 1)
    gr = np.where((flags & 4) != 0, -1, counters["go_row"])
    row = np.where(go & (gr >= 0), gr, row)
    counters["go_row"] = np.where(go, row, -1)
    crow = env.chron[env.scen, row]
    th = env.thermal_limit_a
    adv = counters["stamp"] != stamp
    rst = (flags & 4) != 0
    for arr, thr in ((counters["ts_over"], th), (counters["ts_prot"], (th * f(tables["soft_thr"])).astype(f))):
        base = np.where(rst[:, None], 0, arr)
        up = np.where(v.a_or > thr[None, :], base + 1, 0)
        arr[:] = np.where((adv & ~go)[:, None], up, base)
    counters["stamp"] = stamp.copy()
    gen_p = v.unit_p[:, nh:]
    g = tables["gen"]
    vals = {}
    cal = tables["calendar"][env.scen, row]
    for k, nm in enumerate(("year", "month", "day", "hour_of_day", "minute_of_hour", "day_of_week")):
        vals[nm] = cal[:, k:k + 1].astype(f)
    z = lambda n: np.zeros((B, n), f)             # noqa: E731
    vals.update(gen_p=gen_p, gen_q=v.unit_q[:, nh:], gen_v=v.unit_v[:, nh:], load_p=crow[:, :gm.n_load], load_q=crow[:, gm.n_load:2 * gm.n_load],
                load_v=v.load_v, p_or=v.p_or, q_or=v.q_or, v_or=v.v_or, a_or=v.a_or, p_ex=v.p_ex, q_ex=v.q_ex, v_ex=v.v_ex, a_ex=v.a_ex, rho=rho)
    lo, le = topo[:, gm.line_or_pos], topo[:, gm.line_ex_pos]
    vals["line_status"] = ((lo > 0) & (le > 0)).astype(f)
    vals["timestep_overflow"] = counters["ts_over"].astype(f)
    tv = topo[:, :gm.dim_topo]
    vals["topo_vect"] = np.where(tv > 0, tv, -1).astype(f)
    vals["time_before_cooldown_line"] = cd_l.astype(f); vals["time_before_cooldown_sub"] = cd_s.astype(f)
    if tables.get("maint_time") is not None:
        vals["time_next_maintenance"] = tables["maint_time"][env.scen, row].astype(f)
        vals["duration_next_maintenance"] = tables["maint_dur"][env.scen, row].astype(f)
    else:
        vals["time_next_maintenance"] = np.full((B, nl), -1, f); vals["duration_next_maintenance"] = z(nl)
    st = tables["storage"]
    ch = st["charge0"][None, :] - (cur.astype(f)[:, None] * st["loss_step"][None, :]).astype(f)
    vals["storage_charge"] = np.maximum(ch, f(0))
    vals["gen_p_before_curtail"] = np.where(g["gen_renewable"][None, :], gen_p, f(0)).astype(f)
    vals["curtailment_limit"] = vals["curtailment_limit_effective"] = np.ones((B, gm.n_gen), f)
    vals["time_since_last_alarm"] = np.full((B, 1), -1, f)
    vals.update(_shunt_p=v.shunt_p, _shunt_q=v.shunt_q, _shunt_v=v.shunt_v)
    sb = topo[:, gm.dim_topo:gm.dim_topo + gm.n_shunt]
    vals["_shunt_bus"] = np.where(sb > 0, sb, -1).astype(f)
    vals["current_step"] = cur[:, None].astype(f)
    vals["max_step"] = tables["max_step"][env.scen][:, None].astype(f)
    vals["delta_time"] = np.full((B, 1), tables["delta_time"], f)
    if g["available"]:
        up = np.maximum(np.minimum(g["gen_pmax"][None, :] - gen_p, g["gen_max_ramp_up"][None, :]), f(0))
        dn = np.maximum(np.minimum(gen_p - g["gen_pmin"][None, :], g["gen_max_ramp_down"][None, :]), f(0))
        up[:, g["gen_renewable"]] = 0; dn[:, g["gen_renewable"]] = 0
    else:
        up = dn = z(gm.n_gen)
    vals["gen_margin_up"], vals["gen_margin_down"] = up, dn
    vals["gen_p_delta"] = gen_p - crow[:, 2 * gm.n_load:2 * gm.n_load + gm.n_gen]
    vals["timestep_protection_engaged"] = counters["ts_prot"].astype(f)
    # game over (BaseObservation.set_game_over): zeros, topology / shunt bus -1, maintenance -1, limits 1; calendar and counters of
    # the episode kept
    gozero = [k for k in vals if k not in ("year", "month", "day", "hour_of_day", "minute_of_hour", "day_of_week", "current_step",
                                           "max_step", "delta_time", "curtailment_limit", "curtailment_limit_effective",
                                           "time_since_last_alarm")]
    for k in gozero:
        fill = -1.0 if k in ("topo_vect", "_shunt_bus", "time_next_maintenance") else 0.0
        vals[k] = np.where(go[:, None], f(fill), vals[k]).astype(f)
    obs = np.zeros((B, tables["n_obs"]), f)
    for src, off, ln in tables["seg"]:
        nm = OBS_SOURCES[src]
        if ln and nm in vals:
            obs[:, off:off + ln] = vals[nm]
    return obs
