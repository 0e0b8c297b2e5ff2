"""TEST INFRASTRUCTURE: the device environment's validation and apply bodies with the action read by id from an action table
(csrc/b200pf_env.cuh, ``ActIds``) through their host build (tests/emu/act_ids_emu.cpp), next to a numpy :class:`BatchedEnv`; the post
and reset bodies are those of :class:`act_emu.EmuActEnvState`."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from act_emu import ActArgs, EmuActEnvState
from env_emu import HERE, REPO

LIB = os.path.join(HERE, "libact_ids_emu.so")


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "act_ids_emu.cpp")
    deps = [src] + [os.path.join(REPO, "grid2op_b200", "csrc", f) for f in ("b200pf_env.cuh", "b200pf_opp.cuh", "b200pf_alert.cuh",
                                                                              "b200pf_alarm.cuh")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", LIB, src])
    return LIB


class ActIds(C.Structure):
    """``ActIds`` of csrc/b200pf_env.cuh, field for field"""
    _fields_ = [("id", C.c_void_p), ("n", C.c_int32)]


class EmuActIdsEnvState(EmuActEnvState):
    def __init__(self, env):
        super().__init__(env)
        self.ilib = C.CDLL(build())
        sz = (C.c_int * 3)()
        self.ilib.act_ids_emu_sizes(sz)
        assert sz[0] == self.lib.env_emu_args_size() and sz[1] == C.sizeof(ActArgs) and sz[2] == C.sizeof(ActIds)

    def step_apply_ids(self, table, ids, from_reset=False, tight_cap=True):
        """validation + apply with instance i acting with row ``ids[i]`` of ``table`` = (set_bus, change_bus, set_status,
        change_status) [n, ...] (on a reset step: no action); -> the control words"""
        self.st["ctl"][:] = 0
        self.vec = 0 if from_reset else 1
        a, r = self._args(from_reset=int(from_reset), tight_cap=int(tight_cap)), self._act(table)
        keep = np.ascontiguousarray(ids, np.int32)
        q = None if from_reset else ActIds(id=keep.ctypes.data, n=len(self._vkeep[0]))
        qp = None if q is None else C.byref(q)
        if self.vec:
            assert self.ilib.act_ids_emu_run(C.byref(a), C.byref(r), qp, 0) == 0
        assert self.ilib.act_ids_emu_run(C.byref(a), C.byref(r), qp, 1) == 0
        c = self.st["ctl"].copy()
        if not c[2]:
            self.n_illegal += int(c[4])
            if c[0] > 0:
                self.st["stale"][:] = 0
        return c
