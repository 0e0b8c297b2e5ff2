"""TEST INFRASTRUCTURE: the device environment bodies with the action rules and the vector action bound (csrc/b200pf_env.cuh,
``ActArgs``) through their host build (tests/emu/act_emu.cpp), next to a numpy :class:`BatchedEnv` as :class:`env_emu.EmuEnvState`
runs them."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from env_emu import HERE, REPO, EmuEnvState

LIB = os.path.join(HERE, "libact_emu.so")


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "act_emu.cpp")
    deps = [src] + [os.path.join(REPO, "grid2op_b200", "csrc", f) for f in ("b200pf_env.cuh", "b200pf_opp.cuh", "b200pf_alert.cuh",
                                                                              "b200pf_alarm.cuh")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", LIB, src])
    return LIB


_P, _I = C.c_void_p, C.c_int32


class ActArgs(C.Structure):
    """``ActArgs`` of csrc/b200pf_env.cuh, field for field"""
    _fields_ = [("max_sub", _I), ("max_line", _I), ("n_area", _I), ("sub_area", _P), ("line_area", _P), ("sub_of_pos", _P), ("vec", _I),
                ("set_bus", _P), ("change_bus", _P), ("set_status", _P), ("change_status", _P), ("is_ambiguous", _P), ("aff_sub", _P)]


class EmuActEnvState(EmuEnvState):
    def __init__(self, env):
        super().__init__(env)
        self.alib = C.CDLL(build())
        sz = (C.c_int * 2)()
        self.alib.act_emu_sizes(sz)
        assert sz[0] == self.lib.env_emu_args_size() and sz[1] == C.sizeof(ActArgs)
        B, gm = self.B, self.gm
        self.act = dict(sub_of_pos=np.ascontiguousarray(env.sub_of_pos, np.int32),
                        sub_area=None if env.areas is None else np.ascontiguousarray(env._sub_area, np.uint32),
                        line_area=None if env.areas is None else np.ascontiguousarray(env._line_area, np.uint32))
        self.st["is_ambiguous"] = np.zeros(B, np.uint8)
        self.st["aff_sub"] = np.zeros((B, gm.n_sub), np.uint8)
        self.vec = 0

    def _act(self, vecs=None):
        env = self.env
        r = ActArgs(max_sub=env.max_sub_changed, max_line=env.max_line_status_changed, n_area=0 if env.areas is None else len(env.areas))
        for nm, arr in list(self.act.items()) + [("is_ambiguous", self.st["is_ambiguous"]), ("aff_sub", self.st["aff_sub"])]:
            setattr(r, nm, None if arr is None else arr.ctypes.data)
        r.vec = self.vec
        if vecs is not None:
            self._vkeep = [np.ascontiguousarray(v, dt) for v, dt in zip(vecs, (np.int8, np.uint8, np.int8, np.uint8))]
            r.set_bus, r.change_bus, r.set_status, r.change_status = (v.ctypes.data for v in self._vkeep)
        return r

    def step_apply_vec(self, vecs, from_reset=False, tight_cap=True):
        """validation + apply of the vector action ``vecs`` = (set_bus, change_bus, set_status, change_status); -> the control words"""
        self.st["ctl"][:] = 0
        self.vec = 0 if from_reset else 1
        a, r = self._args(from_reset=int(from_reset), tight_cap=int(tight_cap)), self._act(vecs)
        if self.vec:
            assert self.alib.act_emu_run(C.byref(a), C.byref(r), 0) == 0
        assert self.alib.act_emu_run(C.byref(a), C.byref(r), 1) == 0
        c = self.st["ctl"].copy()
        if not c[2]:
            self.n_illegal += int(c[4])
            if c[0] > 0:
                self.st["stale"][:] = 0
        return c

    def step_post(self, status, disc, from_reset=False, stamp=0, prot=False):
        a = self._args(status=np.ascontiguousarray(status, np.int32),
                       disc=np.ascontiguousarray(disc, np.int32) if disc is not None else None, prot=int(prot),
                       from_reset=int(from_reset), stamp=int(stamp))
        if disc is None:
            a.disc = None
        assert self.alib.act_emu_run(C.byref(a), C.byref(self._act()), 2) == 0
        self.st["t"][:] = (self.st["t"] + 1) % self.env.chron.shape[1]

    def reset(self, mask, rows=None):
        a = self._args(reset_mask=np.ascontiguousarray(mask, np.uint8), reset_rows=None if rows is None else np.ascontiguousarray(rows, np.int32))
        if rows is None:
            a.reset_rows = None
        assert self.alib.act_emu_run(C.byref(a), C.byref(self._act()), 3) == 0
