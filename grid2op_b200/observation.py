"""Static data of the observation layer: what ``BatchedEnv.observe`` needs besides the series state to assemble grid2op
observation vectors and rewards on the device (csrc/b200pf_obs.cuh, ``b200pf_obs_bind`` of include/b200pf.h).

* :func:`obs_spec` — attribute names (``CompleteObservation.attr_list_vect``, grid2op/Observation/completeObservation.py:140-212,
  an environment's own observation class list, or a gym-style subset) -> segments (source, offset, length) and the width;
* :func:`load_gen_charac` — ``prods_charac.csv`` as ``Backend.load_redispacthing_data`` reads it (grid2op/Backend/backend.py:1781-1931);
* :func:`load_calendar` — ``start_datetime.info`` / ``time_interval.info`` of every scenario (grid2op/Chronics/gridValue.py:1024-1060):
  the date of every row, the step length, the real episode length;
* :func:`load_storage` — ``storage_units_charac.csv`` (Emax, Emin, power_loss) and the charge the environment reports when no storage
  is ever set: initial charge (baseEnv.py:1685-1696) minus the loss withdrawn every step (``_withdraw_storage_losses``,
  baseEnv.py:2777-2795);
* :func:`reward_constants` — ``RedispReward.initialize`` (grid2op/Reward/redispReward.py:141-170).
"""
from __future__ import annotations

import csv
import os
from datetime import datetime, timedelta
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .gridmodel import GridModel

__all__ = ["COMPLETE_OBSERVATION_ATTRS", "OBS_SOURCES", "REWARDS", "attr_sizes", "obs_spec", "load_gen_charac", "load_calendar",
           "load_storage", "reward_constants"]

# CompleteObservation.attr_list_vect (grid2op/Observation/completeObservation.py:140-212)
COMPLETE_OBSERVATION_ATTRS = [
    "year", "month", "day", "hour_of_day", "minute_of_hour", "day_of_week", "gen_p", "gen_q", "gen_v", "load_p", "load_q", "load_v",
    "p_or", "q_or", "v_or", "a_or", "p_ex", "q_ex", "v_ex", "a_ex", "rho", "line_status", "timestep_overflow", "topo_vect",
    "time_before_cooldown_line", "time_before_cooldown_sub", "time_next_maintenance", "duration_next_maintenance",
    "target_dispatch", "actual_dispatch", "storage_charge", "storage_power_target", "storage_power", "gen_p_before_curtail",
    "curtailment", "curtailment_limit", "curtailment_limit_effective", "is_alarm_illegal", "time_since_last_alarm", "last_alarm",
    "attention_budget", "was_alarm_used_after_game_over", "_shunt_p", "_shunt_q", "_shunt_v", "_shunt_bus", "current_step",
    "max_step", "delta_time", "gen_margin_up", "gen_margin_down", "active_alert", "attack_under_alert", "time_since_last_alert",
    "alert_duration", "total_number_of_alert", "time_since_last_attack", "was_alert_used_after_attack", "gen_p_delta",
    "load_detached", "gen_detached", "storage_detached", "load_p_detached", "load_q_detached", "gen_p_detached",
    "storage_p_detached", "timestep_protection_engaged",
]

# attribute sources of the kernel, in the order of enum ObsSrc (csrc/b200pf_obs.cuh)
OBS_SOURCES = [
    "year", "month", "day", "hour_of_day", "minute_of_hour", "day_of_week", "gen_p", "gen_q", "gen_v", "load_p", "load_q", "load_v",
    "p_or", "q_or", "v_or", "a_or", "p_ex", "q_ex", "v_ex", "a_ex", "rho", "line_status", "timestep_overflow", "topo_vect",
    "time_before_cooldown_line", "time_before_cooldown_sub", "time_next_maintenance", "duration_next_maintenance",
    "target_dispatch", "actual_dispatch", "storage_charge", "storage_power_target", "storage_power", "gen_p_before_curtail",
    "curtailment", "curtailment_limit", "curtailment_limit_effective", "is_alarm_illegal", "time_since_last_alarm", "last_alarm",
    "attention_budget", "was_alarm_used_after_game_over", "_shunt_p", "_shunt_q", "_shunt_v", "_shunt_bus", "current_step",
    "max_step", "delta_time", "gen_margin_up", "gen_margin_down", "active_alert", "attack_under_alert", "time_since_last_alert",
    "alert_duration", "total_number_of_alert", "time_since_last_attack", "was_alert_used_after_attack", "gen_p_delta",
    "load_detached", "gen_detached", "storage_detached", "load_p_detached", "load_q_detached", "gen_p_detached",
    "storage_p_detached", "timestep_protection_engaged",
]

REWARDS = {None: 0, "none": 0, "RedispReward": 1, "L2RPNReward": 2}


def attr_sizes(gm: GridModel, n_alert: int = 0, n_alarm: int = 0) -> Dict[str, int]:
    """Length of every attribute in the vector of an environment with ``n_alert`` alertable lines (``dim_alerts``; 0: an
    environment without alerts) and ``n_alarm`` alarm zones (``dim_alarms``; 0: an environment without alarms)."""
    nl, ng, nld, ns, nsh, nsub = gm.n_line, gm.n_gen, gm.n_load, gm.n_storage, gm.n_shunt, gm.n_sub
    one = ("year", "month", "day", "hour_of_day", "minute_of_hour", "day_of_week", "is_alarm_illegal", "time_since_last_alarm",
           "attention_budget", "was_alarm_used_after_game_over", "current_step", "max_step", "delta_time")
    sz = {k: 1 for k in one}
    sz.update({k: ng for k in ("gen_p", "gen_q", "gen_v", "target_dispatch", "actual_dispatch", "gen_p_before_curtail", "curtailment",
                              "curtailment_limit", "curtailment_limit_effective", "gen_margin_up", "gen_margin_down", "gen_p_delta",
                              "gen_detached", "gen_p_detached")})
    sz.update({k: nld for k in ("load_p", "load_q", "load_v", "load_detached", "load_p_detached", "load_q_detached")})
    sz.update({k: nl for k in ("p_or", "q_or", "v_or", "a_or", "p_ex", "q_ex", "v_ex", "a_ex", "rho", "line_status", "timestep_overflow",
                              "time_before_cooldown_line", "time_next_maintenance", "duration_next_maintenance",
                              "timestep_protection_engaged")})
    sz.update({k: ns for k in ("storage_charge", "storage_power_target", "storage_power", "storage_detached", "storage_p_detached")})
    sz.update({k: nsh for k in ("_shunt_p", "_shunt_q", "_shunt_v", "_shunt_bus")})
    sz.update({k: 0 for k in ("last_alarm", "active_alert", "attack_under_alert", "time_since_last_alert", "alert_duration",
                             "total_number_of_alert", "time_since_last_attack", "was_alert_used_after_attack")})
    if n_alert:
        sz.update({k: int(n_alert) for k in ("active_alert", "attack_under_alert", "time_since_last_alert", "alert_duration",
                                              "time_since_last_attack", "was_alert_used_after_attack")})
        sz["total_number_of_alert"] = 1
    sz["last_alarm"] = int(n_alarm)
    sz["topo_vect"] = gm.dim_topo
    sz["time_before_cooldown_sub"] = nsub
    return sz


def obs_spec(gm: GridModel, attrs: Optional[Sequence[str]] = None, n_alert: int = 0, n_alarm: int = 0) -> Tuple[np.ndarray, int]:
    """-> (int32 [n_seg, 3] rows (source, offset, length) in the order of ``attrs``, total width).  Unknown name: ValueError."""
    attrs = COMPLETE_OBSERVATION_ATTRS if attrs is None else list(attrs)
    sz = attr_sizes(gm, n_alert, n_alarm)
    seg, off = [], 0
    for a in attrs:
        if a not in sz:
            raise ValueError(f"unknown observation attribute {a!r} (known: CompleteObservation.attr_list_vect)")
        seg.append((OBS_SOURCES.index(a), off, sz[a]))
        off += sz[a]
    return np.asarray(seg, dtype=np.int32).reshape(-1, 3), off


def load_gen_charac(env_dir: str, gm: GridModel, name: str = "prods_charac.csv") -> Dict[str, np.ndarray]:
    """Generator characteristics in backend order (rows matched by name), with the defaults and types of
    ``Backend.load_redispacthing_data``: no file (or a missing mandatory column) -> ``available`` False and the defaults."""
    ng = gm.n_gen
    res = dict(gen_pmin=np.full(ng, 1.0, np.float32), gen_pmax=np.full(ng, 1.0, np.float32), gen_max_ramp_up=np.zeros(ng, np.float32),
               gen_max_ramp_down=np.zeros(ng, np.float32), gen_cost_per_MW=np.full(ng, 1.0, np.float32),
               gen_renewable=np.zeros(ng, bool), gen_redispatchable=np.zeros(ng, bool), available=False)
    path = os.path.join(env_dir, name)
    if not os.path.exists(path):
        return res
    with open(path, newline="") as f:
        rows = list(csv.DictReader(f))
    need = ("type", "Pmax", "Pmin", "max_ramp_up", "max_ramp_down", "start_cost", "shut_down_cost", "marginal_cost", "min_up_time",
            "min_down_time")
    if not rows or any(c not in rows[0] for c in need):
        return res
    by_name = {r["name"]: r for r in rows}
    for i, nm in enumerate(gm.name_gen):
        if nm not in by_name:
            raise ValueError(f"{path}: no row for generator {nm!r} (rows are matched by name)")
        r = by_name[nm]
        res["gen_pmin"][i] = np.float32(float(r["Pmin"])); res["gen_pmax"][i] = np.float32(float(r["Pmax"]))
        ren = r["type"] in ("wind", "solar")
        res["gen_renewable"][i] = ren; res["gen_redispatchable"][i] = not ren
        for col, key in (("max_ramp_up", "gen_max_ramp_up"), ("max_ramp_down", "gen_max_ramp_down")):
            v = np.float32(float(r[col]) if r[col].strip() else np.nan)          # (pandas reads an empty cell as NaN)
            if np.isfinite(v):
                res[key][i] = v
        res["gen_cost_per_MW"][i] = np.float32(float(r["marginal_cost"]))
    res["available"] = True
    return res


def _read_info(path: str, fmts: Sequence[str]):
    with open(path) as f:
        txt = f.read().strip()
    for fmt in fmts:
        try:
            return datetime.strptime(txt, fmt)
        except ValueError:
            pass
    raise ValueError(f"{path}: cannot parse {txt!r}")


def _n_rows(folder: str) -> int:
    from .chronics import read_table
    tbl = read_table(os.path.join(folder, "load_p"))
    if tbl is None:
        raise FileNotFoundError(f"{folder}: no load_p table")
    return len(tbl[1])


def load_calendar(folders: Sequence[str], n_rows: int) -> Tuple[np.ndarray, float, np.ndarray]:
    """-> (int32 [n_scen, n_rows, 6] year, month, day, hour, minute, weekday (Monday = 0) of every row, step length in minutes,
    int32 [n_scen] max_step).  Row r is dated start + (r + 1) x step (GridStateFromFile advances the date before it reads a row,
    gridStateFromFile.py:799).  max_step = the scenario's real row count - 1 (``max_timestep``, gridStateFromFile.py:723-726),
    read from the files: :func:`load_scenarios` pads shorter scenarios.  Defaults of GridValue: 2019-01-01, 5 minutes."""
    cal = np.zeros((len(folders), n_rows, 6), dtype=np.int32)
    max_step = np.zeros(len(folders), dtype=np.int32)
    dts = set()
    for s, folder in enumerate(folders):
        p0, p1 = os.path.join(folder, "start_datetime.info"), os.path.join(folder, "time_interval.info")
        start = _read_info(p0, ("%Y-%m-%d %H:%M", "%Y-%m-%d")) if os.path.exists(p0) else datetime(2019, 1, 1)
        if os.path.exists(p1):
            t = _read_info(p1, ("%H:%M", "%M"))
            dt = timedelta(hours=t.hour, minutes=t.minute)
        else:
            dt = timedelta(minutes=5)
        dts.add(dt)
        for r in range(n_rows):
            d = start + (r + 1) * dt
            cal[s, r] = (d.year, d.month, d.day, d.hour, d.minute, d.weekday())
        max_step[s] = _n_rows(folder) - 1
    if len(dts) != 1:
        raise ValueError("scenarios with different time intervals")
    return cal, dts.pop().total_seconds() / 60.0, max_step


def load_storage(env_dir: str, gm: GridModel, delta_time_min: float, init_capacity: float = 0.5, activate_loss: bool = True,
                 name: str = "storage_units_charac.csv") -> Dict[str, np.ndarray]:
    """Emax / Emin / loss per storage unit (rows matched by name) -> ``charge0`` (float32: the charge after the reset step,
    INIT_STORAGE_CAPACITY x Emax) and ``loss_step`` (float32 MWh withdrawn per step when ACTIVATE_STORAGE_LOSS)."""
    ns = gm.n_storage
    res = dict(Emax=np.zeros(ns, np.float32), Emin=np.zeros(ns, np.float32), loss=np.zeros(ns, np.float32))
    if ns:
        with open(os.path.join(env_dir, name), newline="") as f:
            by_name = {r["name"]: r for r in csv.DictReader(f)}
        for i, nm in enumerate(gm.name_storage):
            r = by_name[nm]
            res["Emax"][i], res["Emin"][i], res["loss"][i] = float(r["Emax"]), float(r["Emin"]), float(r["power_loss"])
    lps = (res["loss"] * np.float32(delta_time_min * 60.0 / 3600.0)).astype(np.float32) if activate_loss else np.zeros(ns, np.float32)
    res["charge0"] = (np.float32(init_capacity) * res["Emax"]).astype(np.float32)
    res["loss_step"] = lps
    return res


def reward_constants(gen: Dict[str, np.ndarray], delta_time_min: float, alpha_redisp: float = 5.0, worst_losses_ratio: float = 0.05,
                     min_reward: float = -10.0, reward_illegal_ambiguous: float = 0.0) -> Dict[str, float]:
    """RedispReward.initialize with the class defaults: max_regret, reward_min, reward_illegal_ambiguous."""
    dts = delta_time_min * 60.0
    worst_marginal_cost = np.max(gen["gen_cost_per_MW"])
    worst_load = gen["gen_pmax"].sum(dtype=np.float32)
    worst_losses = np.float32(worst_losses_ratio) * worst_load
    worst_redisp = alpha_redisp * gen["gen_pmax"].sum()
    max_regret = (worst_losses + worst_redisp) * worst_marginal_cost * dts / 3600.0
    return dict(max_regret=float(max_regret), reward_min=float(np.float32(min_reward)),
                reward_illegal=float(reward_illegal_ambiguous), dts_hours=dts / 3600.0)
