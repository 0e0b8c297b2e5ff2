"""TEST INFRASTRUCTURE: the device line alerts (csrc/b200pf_alert.cuh) through their host build (tests/emu/alert_emu.cpp).
``EmuAlertEnvState`` is :class:`multi_emu.EmuMultiEnvState` with the alert state in the post and reset bodies and the alert values
in the observe input record; ``COracleAlertObsEngine`` is the host observe engine whose input record carries the alert values."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from multi_emu import EmuMultiEnvState
from obs_engines import COracleObsSeriesEngine

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
REPO = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libalert_emu.so")

_P, _I, _D = C.c_void_p, C.c_int32, C.c_double


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "alert_emu.cpp")
    deps = [src, os.path.join(REPO, "include", "b200pf.h")] + [os.path.join(REPO, "grid2op_b200", "csrc", f) for f in
                                                                ("b200pf_env.cuh", "b200pf_opp.cuh", "b200pf_alert.cuh", "b200pf_obs.cuh")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++", "-o", LIB, src])
    return LIB


class AlertArgs(C.Structure):
    """``AlertArgs`` of csrc/b200pf_alert.cuh, field for field"""
    _fields_ = [("n", _I), ("lines", _P), ("window", _I), ("ring", _I), ("reward", _I), ("min_blackout", _D), ("range_blackout", _D),
                ("max_no_blackout", _D), ("diff_no_blackout", _D), ("raise_", _P), ("attack", _P), ("attack_stride", _I),
                ("last_alert", _P), ("already", _P), ("tsl_alert", _P), ("duration", _P), ("tsl_attack", _P), ("under_alert", _P),
                ("was_used", _P), ("total", _P), ("ts_attack", _P), ("launched", _P), ("current", _P), ("cur_id", _P),
                ("reward_out", _P)]


def _lib():
    lib = C.CDLL(build())
    assert lib.alert_emu_args_size() == C.sizeof(AlertArgs)
    return lib


class _ObserveWithAlerts:
    def __init__(self, lib):
        self.obs_emu_run = lib.alert_emu_observe


class COracleAlertObsEngine(COracleObsSeriesEngine):
    def obs_bind(self, tables):
        super().obs_bind(tables)
        self._obs_lib = _ObserveWithAlerts(_lib())


class EmuAlertEnvState(EmuMultiEnvState):
    """the host build of the apply / post / reset bodies with a GeometricOpponentMultiArea and line alerts (``env._alerts``)"""

    def __init__(self, env):
        super().__init__(env)
        self.alib = _lib()
        a = env._alerts
        self.al = a
        self.ast = {k: v.copy() for k, v in a.get_state().items()}
        self.ast["lines"] = np.ascontiguousarray(a.lines, np.int32)
        self.ast["raise_"] = np.zeros((env.batch, a.n), np.uint8)
        self.ast["reward_out"] = np.zeros(env.batch, np.float64)
        gm = env.gm
        self.stride = gm.n_line + gm.n_sub + 3 + 6 * a.n + 1
        self.st["obs_in"] = np.zeros((env.batch, self.stride), np.int32)

    def _args(self, **kw):
        a = super()._args(**kw)
        a.obs_stride = self.stride
        return a

    def _aargs(self):
        a, al = self.al, AlertArgs()
        al.n, al.window, al.ring, al.reward = a.n, a.window, a.ring, int(a.reward)
        al.min_blackout, al.range_blackout = float(a.min_blackout), float(a.range_blackout)
        al.max_no_blackout, al.diff_no_blackout = float(a.max_no_blackout), float(a.diff_no_blackout)
        for nm, arr in self.ast.items():
            setattr(al, nm, arr.ctypes.data)
        al.attack, al.attack_stride = self.mst["attack_lines"].ctypes.data, self.mst["attack_lines"].shape[1]
        return al

    def step_post(self, status, disc, from_reset=False, stamp=0, prot=False, raise_alert=None):
        self.ast["raise_"][:] = 0 if raise_alert is None else np.asarray(raise_alert, np.uint8)
        a = self._args(status=np.ascontiguousarray(status, np.int32),
                       disc=np.ascontiguousarray(disc, np.int32) if disc is not None else None, prot=int(prot),
                       from_reset=int(from_reset), stamp=int(stamp))
        if disc is None:
            a.disc = None
        assert self.alib.alert_emu_run(C.byref(a), C.byref(self._oargs()), C.byref(self._margs()), C.byref(self._aargs()), 2) == 0
        self.st["t"][:] = (self.st["t"] + 1) % self.env.chron.shape[1]

    def reset(self, mask, rows=None):
        a = self._args(reset_mask=np.ascontiguousarray(mask, np.uint8), reset_rows=None if rows is None else np.ascontiguousarray(rows, np.int32))
        if rows is None:
            a.reset_rows = None
        assert self.alib.alert_emu_run(C.byref(a), C.byref(self._oargs()), C.byref(self._margs()), C.byref(self._aargs()), 3) == 0

    def alert_state(self):
        return {k: v for k, v in self.ast.items() if k not in ("lines", "raise_", "reward_out")}
