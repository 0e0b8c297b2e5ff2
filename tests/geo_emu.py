"""TEST INFRASTRUCTURE: the device GeometricOpponent (csrc/b200pf_opp.cuh) through its host build (tests/emu/geo_emu.cpp).
``EmuGeoEnvState`` is :class:`opp_emu.EmuOppEnvState` with the GeometricOpponent's schedules in the apply and reset bodies;
``GeoDraws`` gives its draws, schedules and choice on one RandomState's state."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from env_emu import EnvArgs
from opp_emu import EmuOppEnvState, OppArgs

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
REPO = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libgeo_emu.so")

_P, _I, _D = C.c_void_p, C.c_int32, C.c_double


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "geo_emu.cpp")
    deps = [src] + [os.path.join(REPO, "grid2op_b200", "csrc", f) for f in ("b200pf_env.cuh", "b200pf_opp.cuh")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", LIB, src])
    return LIB


class OppGeoArgs(C.Structure):
    """``OppGeoArgs`` of csrc/b200pf_opp.cuh, field for field"""
    _fields_ = [("weights", _P), ("p_hazard", _D), ("p_recovery", _D), ("logq_hazard", _D), ("logq_recovery", _D),
                ("recovery_min", _I), ("cap", _I), ("emt", _P), ("wait", _P), ("dur", _P), ("gctr", _P)]


def _lib():
    lib = C.CDLL(build())
    assert lib.geo_emu_args_size() == C.sizeof(OppGeoArgs) and lib.geo_emu_opp_args_size() == C.sizeof(OppArgs)
    assert lib.geo_emu_env_args_size() == C.sizeof(EnvArgs)
    lib.geo_emu_geometric.argtypes = [_P, _P, _D, _D, C.c_int, _P]
    lib.geo_emu_sample.argtypes = [_P, _P, _D, _D, _D, _D, C.c_int, _I, C.c_int, _P, _P, _P]
    lib.geo_emu_attack.argtypes = [_P, _P, C.c_int, _P, _P, _P]
    return lib


class GeoDraws:
    """the device restatement's geometric draws, schedules and choice on one RandomState's state"""

    def __init__(self, seed):
        st = np.random.RandomState(seed).get_state()
        self.lib = _lib()
        self.mt = np.array(st[1], dtype=np.uint32)
        self.pos = np.array([st[2]], dtype=np.int32)

    def _s(self):
        return self.mt.ctypes.data, self.pos.ctypes.data

    def geometric(self, p, count=1):
        out = np.empty(count, np.int64)
        self.lib.geo_emu_geometric(*self._s(), float(p), float(np.log(1.0 - float(p))), count, out.ctypes.data)
        return out

    def schedule(self, p_hazard, p_recovery, recovery_min, episode_max_time, cap):
        """-> (waiting times int32 [n], durations int32 [n], entries dropped at the cap)"""
        p_hazard, p_recovery = float(p_hazard), float(p_recovery)
        w, d, dropped = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(1, np.int32)
        n = self.lib.geo_emu_sample(*self._s(), p_hazard, float(np.log(1.0 - p_hazard)), p_recovery,
                                    float(np.log(1.0 - p_recovery)), int(recovery_min), int(episode_max_time), int(cap),
                                    w.ctypes.data, d.ctypes.data, dropped.ctypes.data)
        return w[:n].copy(), d[:n].copy(), int(dropped[0])

    def attack(self, rho, weights):
        """-> (line among 0..n-1, the schedule's duration 5)"""
        r = np.ascontiguousarray(rho, np.float32)
        w = np.ascontiguousarray(weights, np.float64)
        dur = np.zeros(1, np.int32)
        line = self.lib.geo_emu_attack(*self._s(), len(r), r.ctypes.data, w.ctypes.data, dur.ctypes.data)
        return int(line), int(dur[0])


class EmuGeoEnvState(EmuOppEnvState):
    """the host build of the apply / reset bodies with a GeometricOpponent (``env._opp.geometric``)"""

    def __init__(self, env):
        super().__init__(env)
        self.glib = _lib()
        o, s = env._opp, env._opp.get_state()
        self.gst = dict(weights=np.ascontiguousarray(o.geo_weights, np.float64), emt=np.ascontiguousarray(o.emt, np.int32),
                        wait=s["geo_wait"].copy(), dur=s["geo_dur"].copy(), gctr=s["geo_ctr"].copy())

    def _gargs(self):
        o, g = self.o, OppGeoArgs()
        g.p_hazard, g.p_recovery = float(o.hazard_rate), float(o.recovery_rate)
        g.logq_hazard, g.logq_recovery = o.logq_hazard, o.logq_recovery
        g.recovery_min, g.cap = o.recovery_min, o.cap
        for nm, arr in self.gst.items():
            setattr(g, nm, arr.ctypes.data)
        return g

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
        a, o, g = self._args(**kw), self._oargs(), self._gargs()
        assert self.glib.geo_emu_run(C.byref(a), C.byref(o), C.byref(g), 0) == 0
        assert self.glib.geo_emu_run(C.byref(a), C.byref(o), C.byref(g), 1) == 0
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
        assert self.glib.geo_emu_run(C.byref(a), C.byref(self._oargs()), C.byref(self._gargs()), 3) == 0

    def opponent_state(self):
        s = super().opponent_state()
        s.update(geo_wait=self.gst["wait"], geo_dur=self.gst["dur"], geo_ctr=self.gst["gctr"])
        return s
