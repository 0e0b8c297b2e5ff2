"""TEST INFRASTRUCTURE: the device GeometricOpponentMultiArea (csrc/b200pf_opp.cuh) through its host build (tests/emu/multi_emu.cpp).
``EmuMultiEnvState`` is :class:`opp_emu.EmuOppEnvState` with the multi-area opponent's per-area streams and schedules in the apply
and reset bodies."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from env_emu import EnvArgs
from opp_emu import EmuOppEnvState, OppArgs

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
REPO = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libmulti_emu.so")

_P, _I, _D = C.c_void_p, C.c_int32, C.c_double


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "multi_emu.cpp")
    deps = [src] + [os.path.join(REPO, "grid2op_b200", "csrc", f) for f in ("b200pf_env.cuh", "b200pf_opp.cuh")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", LIB, src])
    return LIB


class OppMultiArgs(C.Structure):
    """``OppMultiArgs`` of csrc/b200pf_opp.cuh, field for field"""
    _fields_ = [("n_area", _I), ("area_off", _I * 9), ("weights", _P), ("p_hazard", _D), ("p_recovery", _D), ("logq_hazard", _D),
                ("logq_recovery", _D), ("recovery_min", _I), ("cap", _I), ("emt", _P), ("mt", _P), ("mt_pos", _P), ("wait", _P),
                ("dur", _P), ("actr", _P), ("fails", _P), ("attack_lines", _P)]


def _lib():
    lib = C.CDLL(build())
    assert lib.multi_emu_args_size() == C.sizeof(OppMultiArgs) and lib.multi_emu_opp_args_size() == C.sizeof(OppArgs)
    assert lib.multi_emu_env_args_size() == C.sizeof(EnvArgs)
    return lib


class EmuMultiEnvState(EmuOppEnvState):
    """the host build of the apply / reset bodies with a GeometricOpponentMultiArea (``env._opp.multi``)"""

    def __init__(self, env):
        super().__init__(env)
        self.mlib = _lib()
        o, s = env._opp, env._opp.get_state()
        self.mst = dict(weights=np.ascontiguousarray(o.area_weights, np.float64), emt=np.ascontiguousarray(o.emt, np.int32),
                        mt=s["multi_mt"].copy(), mt_pos=s["multi_mt_pos"].copy(), wait=s["multi_wait"].copy(), dur=s["multi_dur"].copy(),
                        actr=s["multi_ctr"].copy(), fails=s["multi_fails"].copy(),
                        attack_lines=np.full((env.batch, len(o.area_off) - 1), -1, np.int32))

    def _margs(self):
        o, m = self.o, OppMultiArgs()
        m.n_area = len(o.area_off) - 1
        for k, v in enumerate(o.area_off):
            m.area_off[k] = int(v)
        m.p_hazard, m.p_recovery = float(o.hazard_rate), float(o.recovery_rate)
        m.logq_hazard, m.logq_recovery = o.logq_hazard, o.logq_recovery
        m.recovery_min, m.cap = o.recovery_min, o.cap
        for nm, arr in self.mst.items():
            setattr(m, nm, arr.ctypes.data)
        return m

    def step_apply(self, sub_id=None, sub_bus=None, line_id=None, line_status=None, from_reset=False, tight_cap=True, rho=None):
        self.st["ctl"][:] = 0
        if rho is not None:
            self.ost["rho"][:] = rho
        kw = dict(from_reset=int(from_reset), tight_cap=int(tight_cap))
        if sub_id is not None and not from_reset:
            sb = np.ascontiguousarray(sub_bus, np.int8)
            kw.update(sub_id=np.ascontiguousarray(sub_id, np.int32), sub_bus=sb, sub_bus_stride=sb.shape[1], sub_bus_cols=sb.shape[1])
        if line_id is not None and not from_reset:
            kw.update(line_id=np.ascontiguousarray(line_id, np.int32), line_status=np.ascontiguousarray(line_status, np.int32))
        a, o, m = self._args(**kw), self._oargs(), self._margs()
        assert self.mlib.multi_emu_run(C.byref(a), C.byref(o), C.byref(m), 0) == 0
        assert self.mlib.multi_emu_run(C.byref(a), C.byref(o), C.byref(m), 1) == 0
        c = self.st["ctl"].copy()
        if not c[2]:
            self.n_illegal += int(c[4])
            if c[0] > 0:
                self.st["stale"][:] = 0
        return c

    def reset(self, mask, rows=None):
        a = self._args(reset_mask=np.ascontiguousarray(mask, np.uint8), reset_rows=None if rows is None else np.ascontiguousarray(rows, np.int32))
        if rows is None:
            a.reset_rows = None
        assert self.mlib.multi_emu_run(C.byref(a), C.byref(self._oargs()), C.byref(self._margs()), 3) == 0

    def opponent_state(self):
        s = super().opponent_state()
        s.update(multi_mt=self.mst["mt"], multi_mt_pos=self.mst["mt_pos"], multi_wait=self.mst["wait"], multi_dur=self.mst["dur"],
                 multi_ctr=self.mst["actr"], multi_fails=self.mst["fails"])
        return s
