"""TEST INFRASTRUCTURE: the device environment bodies (csrc/b200pf_env.cuh) through their host build (tests/emu/env_emu.cpp), with
the state in numpy arrays laid out as the CUDA path keeps it on the device.  ``EmuEnvState.from_env`` takes the static tables and
the current state of a numpy :class:`BatchedEnv`, so the two can be stepped side by side."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
REPO = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libenv_emu.so")


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "env_emu.cpp")
    deps = [src, os.path.join(REPO, "grid2op_b200", "csrc", "b200pf_env.cuh")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", LIB, src])
    return LIB


_P, _I = C.c_void_p, C.c_int32


class EnvArgs(C.Structure):
    """``EnvArgs`` of csrc/b200pf_env.cuh, field for field"""
    _fields_ = [(n, _I) for n in ("batch", "n_line", "n_sub", "dim_topo", "n_topo_in", "n_busbar", "n_slot", "max_sub", "n_rows")] + [
        ("sub_pos", _P), ("line_or_pos", _P), ("line_ex_pos", _P), ("line_of_pos", _P), ("other_end_pos", _P), ("elem_pos", _P),
        ("elem_sub", _P), ("n_elem", _I), ("cd_line", _I), ("cd_sub", _I), ("cd_reco", _I),
        ("maint", _P), ("haz", _P), ("maint_time", _P), ("maint_dur", _P), ("haz_dur", _P), ("iso_cols", _P), ("iso_seg", _P),
        ("n_iso_seg", _I), ("n_iso_cols", _I), ("topo0", _P), ("t0", _P), ("scen", _P), ("topo", _P), ("t", _P),
        ("lib_done", _P), ("pcount", _P), ("ts_over", _P), ("lib_disc", _P), ("trip", _P), ("incdone", _P),
        ("last_bus", _P), ("line_cd", _P), ("sub_cd", _P), ("done", _P), ("is_illegal", _P), ("newly_done", _P),
        ("current_step", _P), ("status_out", _P), ("aff_l", _P), ("aff_s", _P), ("row_used", _P), ("stale", _P), ("cap_dirty", _P),
        ("obs_reset", _P), ("nb_inst", _P), ("copy_list", _P), ("copy_rows", _P), ("ctl", _P),
        ("sub_id", _P), ("sub_bus", _P), ("sub_bus_stride", _I), ("sub_bus_cols", _I), ("line_id", _P), ("line_status", _P),
        ("from_reset", _I), ("tight_cap", _I), ("prot", _I), ("status", _P), ("disc", _P), ("obs_in", _P), ("obs_stride", _I),
        ("stamp", _I), ("reset_mask", _P), ("reset_rows", _P)]


class EmuEnvState:
    def __init__(self, env):
        self.lib = C.CDLL(build())
        assert self.lib.env_emu_args_size() == C.sizeof(EnvArgs)
        gm, B = env.gm, env.batch
        self.env, self.gm, self.B = env, gm, B
        i32 = lambda x: np.ascontiguousarray(x, np.int32)          # noqa: E731
        if env._iso_cols is None:
            env._isolated_shunt_busbar()
        epos = np.concatenate([gm.line_or_pos, gm.line_ex_pos, gm.unit_pos, gm.load_pos, gm.storage_pos, gm.dim_topo + np.arange(gm.n_shunt)])
        esub = np.concatenate([gm.line_or_sub, gm.line_ex_sub, gm.unit_sub, gm.load_sub, gm.storage_sub, gm.shunt_sub])
        self.tab = dict(sub_pos=i32(env.sub_pos), line_or_pos=i32(gm.line_or_pos), line_ex_pos=i32(gm.line_ex_pos),
                        line_of_pos=i32(env.line_of_pos), other_end_pos=i32(env.other_end_pos), elem_pos=i32(epos), elem_sub=i32(esub),
                        iso_cols=i32(env._iso_cols), iso_seg=i32(env._iso_seg), topo0=np.ascontiguousarray(env.topo0, np.int8),
                        t0=i32(env.t0), scen=i32(env.scen))
        for nm, arr, dt in (("maint", env._maint, np.uint8), ("haz", env._haz, np.uint8), ("maint_time", env._maint_time, np.int32),
                            ("maint_dur", env._maint_dur, np.int32), ("haz_dur", env._haz_dur, np.int32)):
            self.tab[nm] = None if arr is None else np.ascontiguousarray(arr, dt)
        nl, ns = gm.n_line, gm.n_sub
        self.st = dict(topo=env.topo.copy(), t=i32(env.row % env.chron.shape[1]), last_bus=env.last_bus.copy(),
                       line_cd=i32(env.line_cooldown), sub_cd=i32(env.sub_cooldown), done=env.done.astype(np.uint8),
                       is_illegal=np.asarray(env.is_illegal).astype(np.uint8), newly_done=np.zeros(B, np.uint8), current_step=i32(env.current_step),
                       status_out=np.zeros(B, np.int32), aff_l=np.zeros((B, nl), np.uint8), aff_s=np.full(B, -1, np.int32),
                       row_used=np.zeros(B, np.int32), stale=np.ones(B, np.uint8), cap_dirty=np.ones(B, np.uint8), obs_reset=np.zeros(B, np.uint8),
                       nb_inst=np.zeros(B, np.int32), copy_list=np.zeros(B, np.int32), copy_rows=np.zeros((B, gm.n_topo_in), np.int8),
                       ctl=np.zeros(8, np.int32), obs_in=np.zeros((B, nl + ns + 3), np.int32),
                       lib_done=np.zeros(B, np.int32), pcount=np.zeros((B, nl), np.int32), ts_over=np.zeros((B, nl), np.int32),
                       lib_disc=np.full((B, nl), -1, np.int32), trip=np.zeros((B, nl), np.int8), incdone=np.zeros((B, nl), np.int8))
        self.n_illegal = 0

    def _args(self, **kw):
        gm, env = self.gm, self.env
        a = EnvArgs()
        a.batch, a.n_line, a.n_sub, a.dim_topo, a.n_topo_in = self.B, gm.n_line, gm.n_sub, gm.dim_topo, gm.n_topo_in
        a.n_busbar, a.n_slot, a.max_sub, a.n_rows = gm.n_busbar, gm.n_slot, env.max_sub_size, env.chron.shape[1]
        a.n_elem = len(self.tab["elem_pos"]); a.cd_line, a.cd_sub, a.cd_reco = env.cd_line, env.cd_sub, env.cd_reco
        a.n_iso_seg, a.n_iso_cols = len(self.tab["iso_seg"]), len(self.tab["iso_cols"])
        a.obs_stride = gm.n_line + gm.n_sub + 3
        self._keep = []
        for nm, arr in list(self.tab.items()) + list(self.st.items()):
            if arr is not None and hasattr(EnvArgs, nm):
                setattr(a, nm, arr.ctypes.data)
        for nm, v in kw.items():
            if isinstance(v, np.ndarray):
                self._keep.append(v)
                setattr(a, nm, v.ctypes.data)
            else:
                setattr(a, nm, v)
        return a

    def step_apply(self, sub_id=None, sub_bus=None, line_id=None, line_status=None, from_reset=False, tight_cap=True):
        """validation + apply; -> the control words (n_dirty, cap_max, err, n_copy, n_illegal)"""
        self.st["ctl"][:] = 0
        kw = dict(from_reset=int(from_reset), tight_cap=int(tight_cap))
        if sub_id is not None and not from_reset:
            sb = np.ascontiguousarray(sub_bus, np.int8)
            kw.update(sub_id=np.ascontiguousarray(sub_id, np.int32), sub_bus=sb, sub_bus_stride=sb.shape[1], sub_bus_cols=sb.shape[1])
        if line_id is not None and not from_reset:
            kw.update(line_id=np.ascontiguousarray(line_id, np.int32), line_status=np.ascontiguousarray(line_status, np.int32))
        a = self._args(**kw)
        assert self.lib.env_emu_run(C.byref(a), 0) == 0 and self.lib.env_emu_run(C.byref(a), 1) == 0
        c = self.st["ctl"].copy()
        if not c[2]:
            self.n_illegal += int(c[4])
            if c[0] > 0:                              # the library refreshes its mirror and the plans
                self.st["stale"][:] = 0
        return c

    def step_post(self, status, disc, from_reset=False, stamp=0, prot=False):
        a = self._args(status=np.ascontiguousarray(status, np.int32),
                       disc=np.ascontiguousarray(disc, np.int32) if disc is not None else None, prot=int(prot),
                       from_reset=int(from_reset), stamp=int(stamp))
        if disc is None:
            a.disc = None
        assert self.lib.env_emu_run(C.byref(a), 2) == 0
        self.st["t"][:] = (self.st["t"] + 1) % self.env.chron.shape[1]      # (what the series kernel does)

    def reset(self, mask, rows=None):
        a = self._args(reset_mask=np.ascontiguousarray(mask, np.uint8), reset_rows=None if rows is None else np.ascontiguousarray(rows, np.int32))
        if rows is None:
            a.reset_rows = None
        assert self.lib.env_emu_run(C.byref(a), 3) == 0

    def observed(self):
        """what follows an observe launch: the reset flags are consumed"""
        a = self._args()
        assert self.lib.env_emu_run(C.byref(a), 4) == 0

    @staticmethod
    def bus_cap(ctl, n_slot):
        n = int(ctl[1])
        if n > 17:
            n = (n + 7) // 8 * 8
        return min(n, n_slot)
