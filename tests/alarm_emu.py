"""TEST INFRASTRUCTURE: the device alarms (csrc/b200pf_alarm.cuh) through their host build (tests/emu/alarm_emu.cpp).
``EmuAlarmEnvState`` is :class:`geo_emu.EmuGeoEnvState` with the alarm state in the post and reset bodies and the alarm values in
the observe input record; ``COracleAlarmObsEngine`` / ``EmuProtAlarmObsEngine`` are the host observe engines (without and with
protections) whose input record carries the alarm values."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from geo_emu import EmuGeoEnvState
from obs_engines import COracleObsSeriesEngine, EmuProtObsSeriesEngine

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
REPO = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libalarm_emu.so")

_P, _I, _F = C.c_void_p, C.c_int32, C.c_float


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "alarm_emu.cpp")
    deps = [src, os.path.join(REPO, "include", "b200pf.h")] + [os.path.join(REPO, "grid2op_b200", "csrc", f) for f in
                                                                ("b200pf_env.cuh", "b200pf_opp.cuh", "b200pf_alarm.cuh", "b200pf_obs.cuh")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++", "-o", LIB, src])
    return LIB


class AlarmArgs(C.Structure):
    """``AlarmArgs`` of csrc/b200pf_alarm.cuh, field for field"""
    _fields_ = [("n", _I), ("zone_mask", _P), ("n_line", _I), ("max_budget", _F), ("budget_per_ts", _F), ("alarm_cost", _F),
                ("init_budget", _F), ("best_time", _I), ("window", _I), ("ring", _I), ("reward", _I), ("raise_", _P), ("budget", _P),
                ("time_last", _P), ("time_last_ok", _P), ("last", _P), ("last_ok", _P), ("ring_step", _P), ("ring_mask", _P),
                ("any_ok", _P), ("used", _P), ("illegal", _P), ("reward_out", _P)]


def _lib():
    lib = C.CDLL(build())
    assert lib.alarm_emu_args_size() == C.sizeof(AlarmArgs)
    return lib


class _ObserveWithAlarms:
    def __init__(self, lib):
        self.obs_emu_run = lib.alarm_emu_observe


class COracleAlarmObsEngine(COracleObsSeriesEngine):
    def obs_bind(self, tables):
        super().obs_bind(tables)
        self._obs_lib = _ObserveWithAlarms(_lib())


class EmuProtAlarmObsEngine(EmuProtObsSeriesEngine):
    def obs_bind(self, tables):
        super().obs_bind(tables)
        self._obs_lib = _ObserveWithAlarms(_lib())


class EmuAlarmEnvState(EmuGeoEnvState):
    """the host build of the apply / post / reset bodies with a GeometricOpponent and alarms (``env._alarms``)"""

    def __init__(self, env):
        super().__init__(env)
        self.alib = _lib()
        a = env._alarms
        self.al = a
        self.ast = {k: v.copy() for k, v in a.get_state().items()}
        self.ast["zone_mask"] = np.ascontiguousarray(a.zone_mask, np.uint32)
        self.ast["raise_"] = np.zeros((env.batch, a.n), np.uint8)
        self.ast["reward_out"] = np.zeros(env.batch, np.float64)
        gm = env.gm
        self.stride = gm.n_line + gm.n_sub + 3 + a.n + 4
        self.st["obs_in"] = np.zeros((env.batch, self.stride), np.int32)

    def _args(self, **kw):
        a = super()._args(**kw)
        a.obs_stride = self.stride
        return a

    def _aargs(self):
        a, am = self.al, AlarmArgs()
        am.n, am.n_line = a.n, self.gm.n_line
        am.max_budget, am.budget_per_ts, am.alarm_cost, am.init_budget = a.max_budget, a.budget_per_ts, a.alarm_cost, a.init_budget
        am.best_time, am.window, am.ring, am.reward = a.best_time, a.window, a.ring, int(a.reward)
        for nm, arr in self.ast.items():
            setattr(am, nm, arr.ctypes.data)
        return am

    def step_post(self, status, disc, from_reset=False, stamp=0, prot=False, raise_alarm=None):
        self.ast["raise_"][:] = 0 if raise_alarm is None else np.asarray(raise_alarm, np.uint8)
        a = self._args(status=np.ascontiguousarray(status, np.int32),
                       disc=np.ascontiguousarray(disc, np.int32) if disc is not None else None, prot=int(prot),
                       from_reset=int(from_reset), stamp=int(stamp))
        if disc is None:
            a.disc = None
        assert self.alib.alarm_emu_run(C.byref(a), C.byref(self._oargs()), C.byref(self._gargs()), C.byref(self._aargs()), 2) == 0
        self.st["t"][:] = (self.st["t"] + 1) % self.env.chron.shape[1]

    def reset(self, mask, rows=None):
        a = self._args(reset_mask=np.ascontiguousarray(mask, np.uint8), reset_rows=None if rows is None else np.ascontiguousarray(rows, np.int32))
        if rows is None:
            a.reset_rows = None
        assert self.alib.alarm_emu_run(C.byref(a), C.byref(self._oargs()), C.byref(self._gargs()), C.byref(self._aargs()), 3) == 0

    def alarm_state(self):
        return {k: v for k, v in self.ast.items() if k not in ("zone_mask", "raise_", "reward_out")}
