"""TEST INFRASTRUCTURE: the device opponent (csrc/b200pf_opp.cuh) through its host build (tests/emu/opp_emu.cpp).  ``EmuOppEnvState``
is :class:`env_emu.EmuEnvState` with the opponent of a numpy :class:`BatchedEnv` (``enable_opponent``) in the apply and reset bodies;
``draws`` gives the RandomState restatement one draw at a time."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from env_emu import EmuEnvState, EnvArgs

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
REPO = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libopp_emu.so")

_P, _I, _F = C.c_void_p, C.c_int32, C.c_float


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "opp_emu.cpp")
    deps = [src] + [os.path.join(REPO, "grid2op_b200", "csrc", f) for f in ("b200pf_env.cuh", "b200pf_opp.cuh")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", LIB, src])
    return LIB


class OppArgs(C.Structure):
    """``OppArgs`` of csrc/b200pf_opp.cuh, field for field"""
    _fields_ = [("kind", _I), ("n_attack", _I), ("lines", _P), ("rho_norm", _P), ("attack_period", _I), ("attack_duration", _I),
                ("attack_cooldown", _I), ("budget_per_ts", _F), ("init_budget", _F), ("budget", _P), ("budget64", _P), ("ctr", _P),
                ("mt", _P), ("mt_pos", _P), ("attack_line", _P), ("attack_dur", _P), ("rho", _P)]


def _lib():
    lib = C.CDLL(build())
    assert lib.opp_emu_args_size() == C.sizeof(OppArgs) and lib.opp_emu_env_args_size() == C.sizeof(EnvArgs)
    return lib


class Draws:
    """numpy-legacy draws of the device restatement on one RandomState's state"""

    def __init__(self, seed):
        st = np.random.RandomState(seed).get_state()
        self.lib = _lib()
        self.mt = np.array(st[1], dtype=np.uint32)
        self.pos = np.array([st[2]], dtype=np.int32)

    def randint(self, n, count=1):
        out = np.empty(count, np.uint32)
        self.lib.opp_emu_randint(self.mt.ctypes.data_as(_P), self.pos.ctypes.data_as(_P), C.c_uint32(n), count, out.ctypes.data_as(_P))
        return out

    def random_sample(self, count=1):
        out = np.empty(count, np.float64)
        self.lib.opp_emu_random_sample(self.mt.ctypes.data_as(_P), self.pos.ctypes.data_as(_P), count, out.ctypes.data_as(_P))
        return out

    def choice_weighted(self, w):
        w = np.ascontiguousarray(w, np.float64)
        return int(self.lib.opp_emu_choice_weighted(self.mt.ctypes.data_as(_P), self.pos.ctypes.data_as(_P), w.ctypes.data_as(_P), len(w)))


class EmuOppEnvState(EmuEnvState):
    def __init__(self, env):
        super().__init__(env)
        self.st = {k: v.copy() for k, v in self.st.items()}          # (the base class may share int32 arrays with the environment)
        self.olib = _lib()
        o = env._opp
        s = o.get_state()
        B, nl = env.batch, env.gm.n_line
        self.o = o
        self.ost = dict(lines=np.ascontiguousarray(o.lines, np.int32), rho_norm=np.ascontiguousarray(o.rho_norm, np.float64),
                        budget=s["budget"].copy(), budget64=s["budget64"].copy(), ctr=s["ctr"].copy(), mt=s["mt"].copy(),
                        mt_pos=s["mt_pos"].copy(), attack_line=np.full(B, -1, np.int32), attack_dur=np.zeros(B, np.int32),
                        rho=np.zeros((B, nl), np.float32))

    def _oargs(self):
        o, a = self.o, OppArgs()
        a.kind, a.n_attack, a.attack_period = o.code, len(o.lines), o.attack_period
        a.attack_duration, a.attack_cooldown = int(o.attack_duration), int(o.attack_cooldown)
        a.budget_per_ts, a.init_budget = float(o.budget_per_ts), float(o.init_budget)
        for nm, arr in self.ost.items():
            setattr(a, nm, arr.ctypes.data)
        return a

    def step_apply(self, sub_id=None, sub_bus=None, line_id=None, line_status=None, from_reset=False, tight_cap=True, rho=None):
        """validation + apply with the opponent (``rho``: what the previous step wrote); -> the control words"""
        self.st["ctl"][:] = 0
        if rho is not None:
            self.ost["rho"][:] = rho
        kw = dict(from_reset=int(from_reset), tight_cap=int(tight_cap))
        if sub_id is not None and not from_reset:
            sb = np.ascontiguousarray(sub_bus, np.int8)
            kw.update(sub_id=np.ascontiguousarray(sub_id, np.int32), sub_bus=sb, sub_bus_stride=sb.shape[1], sub_bus_cols=sb.shape[1])
        if line_id is not None and not from_reset:
            kw.update(line_id=np.ascontiguousarray(line_id, np.int32), line_status=np.ascontiguousarray(line_status, np.int32))
        a, o = self._args(**kw), self._oargs()
        assert self.olib.opp_emu_run(C.byref(a), C.byref(o), 0) == 0 and self.olib.opp_emu_run(C.byref(a), C.byref(o), 1) == 0
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
        assert self.olib.opp_emu_run(C.byref(a), C.byref(self._oargs()), 3) == 0

    def opponent_state(self):
        return {k: self.ost[k] for k in ("budget", "budget64", "ctr", "mt", "mt_pos")}
