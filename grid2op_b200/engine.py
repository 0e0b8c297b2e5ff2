"""ctypes binding of ``libb200pf.so`` (C ABI declared in ``include/b200pf.h``).

There is no CPU fallback: if the shared library is missing, or no CUDA device is visible,
:class:`PowerFlowEngine` raises :class:`EngineUnavailable`.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Tuple

import numpy as np

from .alarm import ALARM_STATE
from .alert import ALERT_STATE
from .gridmodel import GridModel
from .opponent import MULTI_KEYS

__all__ = ["PowerFlowEngine", "PeerBuffer", "EngineUnavailable", "lib_path", "load_library",
           "ST_CONVERGED", "ST_DIVERGED", "ST_UNSUPPLIED", "ST_NO_REF", "ST_TOO_LARGE", "ABI_SYMBOLS"]

ST_CONVERGED, ST_DIVERGED, ST_UNSUPPLIED, ST_NO_REF, ST_TOO_LARGE = 0, 1, 2, 3, 4
STATUS_TEXT = {
    ST_DIVERGED: "Newton-Raphson did not converge (or singular system)",
    ST_UNSUPPLIED: "an in-service bus is not connected to a reference bus (isolated element / islanded grid)",
    ST_NO_REF: "no reference (slack) unit is in service",
    ST_TOO_LARGE: "more active buses than the launch was sized for",
}

ABI_SYMBOLS = (
    "b200pf_last_error", "b200pf_abi_version", "b200pf_device_count", "b200pf_create", "b200pf_destroy",
    "b200pf_sizes", "b200pf_run_host", "b200pf_run_device", "b200pf_series_bind", "b200pf_series_set_topo",
    "b200pf_series_step", "b200pf_series_results", "b200pf_series_fetch", "b200pf_sync", "b200pf_stream",
    "b200pf_launch_count", "b200pf_last_launch_info", "b200pf_staging", "b200pf_run_staged",
    "b200pf_series_bind_outputs", "b200pf_set_stream", "b200pf_set_static_inj", "b200pf_rows_staging",
    "b200pf_run_rows_staged", "b200pf_set_thermal_limit", "b200pf_n1_host", "b200pf_series_protections",
    "b200pf_series_next_is_reset", "b200pf_series_fetch_state", "b200pf_rows_chunk_launch", "b200pf_rows_chunk_wait",
    "b200pf_rows_chunk_launch_from", "b200pf_pinned_alloc", "b200pf_pinned_free", "b200pf_rows_group_launch", "b200pf_rows_group_wait",
    "b200pf_rows_group_config", "b200pf_set_kernel_policy", "b200pf_plan_stats", "b200pf_run_device_topo",
    "b200pf_set_debug", "b200pf_redo_launch_count",
    "b200pf_device_alloc", "b200pf_device_free", "b200pf_ipc_export", "b200pf_ipc_open", "b200pf_ipc_close", "b200pf_device_read", "b200pf_plan_counters", "b200pf_series_bind_flag",
    "b200pf_series_reset_instances", "b200pf_grid_max_active_buses", "b200pf_obs_bind", "b200pf_observe", "b200pf_obs_stats",
    "b200pf_last_launch_config", "b200pf_env_bind", "b200pf_env_step", "b200pf_env_reset", "b200pf_env_get_state",
    "b200pf_env_set_state", "b200pf_env_pointers", "b200pf_observe_device", "b200pf_env_stats",
    "b200pf_opp_bind", "b200pf_opp_get_state", "b200pf_opp_set_state",
    "b200pf_opp_geo_bind", "b200pf_opp_geo_get_state", "b200pf_opp_geo_set_state",
    "b200pf_opp_multi_bind", "b200pf_opp_multi_get_state", "b200pf_opp_multi_set_state",
    "b200pf_alert_bind", "b200pf_alert_get_state", "b200pf_alert_set_state",
    "b200pf_alarm_bind", "b200pf_alarm_get_state", "b200pf_alarm_set_state", "b200pf_act_bind", "b200pf_env_step_act",
    "b200pf_act_table_bind", "b200pf_env_step_ids",
)


class EngineUnavailable(RuntimeError):
    pass


class _GridDesc(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("n_sub", C.c_int32), ("n_busbar", C.c_int32),
        ("n_line", C.c_int32), ("n_gen", C.c_int32), ("n_hidden", C.c_int32), ("n_load", C.c_int32),
        ("n_storage", C.c_int32), ("n_shunt", C.c_int32), ("dim_topo", C.c_int32),
        ("sn_mva", C.c_double),
        ("line_or_sub", C.c_void_p), ("line_ex_sub", C.c_void_p), ("line_or_pos", C.c_void_p), ("line_ex_pos", C.c_void_p),
        ("line_y", C.c_void_p), ("line_bdc", C.c_void_p), ("line_pshift", C.c_void_p),
        ("line_or_vn", C.c_void_p), ("line_ex_vn", C.c_void_p),
        ("unit_sub", C.c_void_p), ("unit_pos", C.c_void_p), ("unit_is_ref", C.c_void_p),
        ("unit_qmin", C.c_void_p), ("unit_qmax", C.c_void_p), ("unit_vn", C.c_void_p),
        ("load_sub", C.c_void_p), ("load_pos", C.c_void_p), ("load_vn", C.c_void_p),
        ("storage_sub", C.c_void_p), ("storage_pos", C.c_void_p), ("storage_vn", C.c_void_p), ("storage_q", C.c_void_p),
        ("shunt_sub", C.c_void_p), ("shunt_vn", C.c_void_p), ("shunt_vratio", C.c_void_p),
        ("sub_rank", C.c_void_p),
    ]


class ObsDesc(C.Structure):
    """``b200pf_obs_desc`` of include/b200pf.h"""
    _fields_ = [
        ("n_seg", C.c_int32), ("n_obs", C.c_int32), ("seg", C.c_void_p), ("calendar", C.c_void_p), ("max_step", C.c_void_p),
        ("delta_time", C.c_float), ("maint_time", C.c_void_p), ("maint_dur", C.c_void_p),
        ("gen_pmin", C.c_void_p), ("gen_pmax", C.c_void_p), ("gen_ramp_up", C.c_void_p), ("gen_ramp_down", C.c_void_p),
        ("gen_cost", C.c_void_p), ("gen_renewable", C.c_void_p), ("redisp_available", C.c_int32),
        ("sto_charge0", C.c_void_p), ("sto_loss_step", C.c_void_p), ("reward_kind", C.c_int32),
        ("max_regret", C.c_double), ("reward_min", C.c_double), ("reward_illegal", C.c_double), ("dts_hours", C.c_double),
        ("soft_thr", C.c_float), ("n_alert", C.c_int32), ("n_alarm", C.c_int32),
    ]


class EnvDesc(C.Structure):
    """``b200pf_env_desc`` of include/b200pf.h"""
    _fields_ = [
        ("max_sub", C.c_int32), ("sub_pos", C.c_void_p), ("line_of_pos", C.c_void_p), ("other_end_pos", C.c_void_p),
        ("cd_line", C.c_int32), ("cd_sub", C.c_int32), ("cd_reco", C.c_int32),
        ("maint", C.c_void_p), ("haz", C.c_void_p), ("maint_time", C.c_void_p), ("maint_dur", C.c_void_p), ("haz_dur", C.c_void_p),
        ("n_iso_seg", C.c_int32), ("n_iso_cols", C.c_int32), ("iso_seg", C.c_void_p), ("iso_cols", C.c_void_p),
        ("topo0", C.c_void_p), ("t0", C.c_void_p),
        ("last_bus", C.c_void_p), ("line_cd", C.c_void_p), ("sub_cd", C.c_void_p), ("done", C.c_void_p), ("is_illegal", C.c_void_p),
        ("newly_done", C.c_void_p), ("current_step", C.c_void_p), ("status", C.c_void_p),
    ]


class OppDesc(C.Structure):
    """``b200pf_opp_desc`` of include/b200pf.h"""
    _fields_ = [
        ("kind", C.c_int32), ("n_attack", C.c_int32), ("lines", C.c_void_p), ("rho_norm", C.c_void_p), ("attack_period", C.c_int32),
        ("attack_duration", C.c_int32), ("attack_cooldown", C.c_int32), ("budget_per_ts", C.c_float), ("init_budget", C.c_float),
        ("mt", C.c_void_p), ("mt_pos", C.c_void_p), ("attack_line", C.c_void_p), ("attack_dur", C.c_void_p), ("budget", C.c_void_p),
    ]


class OppGeoDesc(C.Structure):
    """``b200pf_opp_geo_desc`` of include/b200pf.h"""
    _fields_ = [
        ("weights", C.c_void_p), ("p_hazard", C.c_double), ("p_recovery", C.c_double), ("logq_hazard", C.c_double),
        ("logq_recovery", C.c_double), ("recovery_min", C.c_int32), ("cap", C.c_int32), ("episode_max_time", C.c_void_p),
        ("wait", C.c_void_p), ("dur", C.c_void_p), ("gctr", C.c_void_p),
    ]


class OppMultiDesc(C.Structure):
    """``b200pf_opp_multi_desc`` of include/b200pf.h"""
    _fields_ = [
        ("n_area", C.c_int32), ("area_off", C.c_void_p), ("weights", C.c_void_p), ("p_hazard", C.c_double), ("p_recovery", C.c_double),
        ("logq_hazard", C.c_double), ("logq_recovery", C.c_double), ("recovery_min", C.c_int32), ("cap", C.c_int32),
        ("episode_max_time", C.c_void_p), ("mt", C.c_void_p), ("mt_pos", C.c_void_p), ("wait", C.c_void_p), ("dur", C.c_void_p),
        ("actr", C.c_void_p), ("fails", C.c_void_p), ("attack_lines", C.c_void_p),
    ]


class AlarmDesc(C.Structure):
    """``b200pf_alarm_desc`` of include/b200pf.h"""
    _fields_ = [
        ("n_zone", C.c_int32), ("zone_mask", C.c_void_p), ("max_budget", C.c_float), ("budget_per_ts", C.c_float),
        ("alarm_cost", C.c_float), ("init_budget", C.c_float), ("best_time", C.c_int32), ("window_size", C.c_int32),
        ("reward", C.c_int32), ("raise_alarm", C.c_void_p), ("reward_out", C.c_void_p), ("is_alarm_illegal", C.c_void_p),
    ]


class ActDesc(C.Structure):
    """``b200pf_act_desc`` of include/b200pf.h"""
    _fields_ = [
        ("max_sub_changed", C.c_int32), ("max_line_status_changed", C.c_int32), ("n_area", C.c_int32), ("sub_area", C.c_void_p),
        ("line_area", C.c_void_p), ("set_bus", C.c_void_p), ("change_bus", C.c_void_p), ("set_status", C.c_void_p),
        ("change_status", C.c_void_p), ("is_ambiguous", C.c_void_p),
    ]


class ActTableDesc(C.Structure):
    """``b200pf_act_table_desc`` of include/b200pf.h"""
    _fields_ = [("n_act", C.c_int32), ("set_bus", C.c_void_p), ("change_bus", C.c_void_p), ("set_status", C.c_void_p),
                ("change_status", C.c_void_p)]


class AlertDesc(C.Structure):
    """``b200pf_alert_desc`` of include/b200pf.h"""
    _fields_ = [
        ("n_alert", C.c_int32), ("lines", C.c_void_p), ("window", C.c_int32), ("reward", C.c_int32),
        ("reward_min_no_blackout", C.c_float), ("reward_min_blackout", C.c_float), ("reward_max_no_blackout", C.c_float),
        ("reward_max_blackout", C.c_float), ("raise_alert", C.c_void_p), ("reward_out", C.c_void_p),
    ]


def make_env_desc(t: dict, state: dict):
    """-> (``b200pf_env_desc`` for the static tables ``t`` (numpy, built by ``BatchedEnv``) and the per-instance device buffers
    ``state`` (integer device addresses), the arrays it points to)"""
    keep = []
    d = EnvDesc()

    def put(name, arr, dtype):
        if arr is None:
            setattr(d, name, None)
            return
        a = np.ascontiguousarray(arr, dtype=dtype)
        if a.size == 0:
            a = np.zeros(1, dtype=dtype)
        keep.append(a)
        setattr(d, name, a.ctypes.data)

    d.max_sub = int(t["sub_pos"].shape[1])
    put("sub_pos", t["sub_pos"], np.int32); put("line_of_pos", t["line_of_pos"], np.int32); put("other_end_pos", t["other_end_pos"], np.int32)
    d.cd_line, d.cd_sub, d.cd_reco = int(t["cd_line"]), int(t["cd_sub"]), int(t["cd_reco"])
    put("maint", t.get("maint"), np.uint8); put("haz", t.get("haz"), np.uint8)
    put("maint_time", t.get("maint_time"), np.int32); put("maint_dur", t.get("maint_dur"), np.int32); put("haz_dur", t.get("haz_dur"), np.int32)
    d.n_iso_seg, d.n_iso_cols = len(t["iso_seg"]), len(t["iso_cols"])
    put("iso_seg", t["iso_seg"], np.int32); put("iso_cols", t["iso_cols"], np.int32)
    put("topo0", t["topo0"], np.int8); put("t0", t["t0"], np.int32)
    for name in ("last_bus", "line_cd", "sub_cd", "done", "is_illegal", "newly_done", "current_step", "status"):
        setattr(d, name, int(state[name]))
    return d, keep


def make_obs_desc(t: dict):
    """-> (``b200pf_obs_desc`` for the tables ``t`` built by ``BatchedEnv.enable_observation``, the arrays it points to)"""
    keep = []
    d = ObsDesc()

    def put(name, arr, dtype):
        if arr is None:
            setattr(d, name, None)
            return
        a = np.ascontiguousarray(arr, dtype=dtype)
        if a.size == 0:
            a = np.zeros(1, dtype=dtype)
        keep.append(a)
        setattr(d, name, a.ctypes.data)

    d.n_seg, d.n_obs = len(t["seg"]), int(t["n_obs"])
    put("seg", t["seg"], np.int32); put("calendar", t["calendar"], np.int32); put("max_step", t["max_step"], np.int32)
    d.delta_time = float(t["delta_time"])
    put("maint_time", t.get("maint_time"), np.int32); put("maint_dur", t.get("maint_dur"), np.int32)
    g = t["gen"]
    put("gen_pmin", g["gen_pmin"], np.float32); put("gen_pmax", g["gen_pmax"], np.float32)
    put("gen_ramp_up", g["gen_max_ramp_up"], np.float32); put("gen_ramp_down", g["gen_max_ramp_down"], np.float32)
    put("gen_cost", g["gen_cost_per_MW"], np.float32); put("gen_renewable", g["gen_renewable"], np.int8)
    d.redisp_available = int(bool(g["available"]))
    put("sto_charge0", t["storage"]["charge0"], np.float32); put("sto_loss_step", t["storage"]["loss_step"], np.float32)
    d.reward_kind = int(t["reward_kind"])
    r = t["reward"]
    d.max_regret, d.reward_min, d.reward_illegal, d.dts_hours = r["max_regret"], r["reward_min"], r["reward_illegal"], r["dts_hours"]
    d.soft_thr = float(t["soft_thr"])
    d.n_alert = int(t.get("n_alert", 0))
    d.n_alarm = int(t.get("n_alarm", 0))
    return d, keep


def lib_path() -> str:
    """The engine library: B200PF_LIB names another build of it (an instrumented copy, or an older build to compare
    against); the default is the one build() leaves next to this file."""
    p = os.environ.get("B200PF_LIB")
    if p:
        return os.path.abspath(p)
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "libb200pf.so")


_LIB = None


def load_library():
    """dlopen the engine and declare the prototypes of include/b200pf.h."""
    global _LIB
    if _LIB is not None:
        return _LIB
    p = lib_path()
    if not os.path.exists(p):
        raise EngineUnavailable(f"{p} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`")
    lib = C.CDLL(p)
    vp, i32, f64 = C.c_void_p, C.c_int, C.c_double
    lib.b200pf_last_error.restype = C.c_char_p
    lib.b200pf_abi_version.restype = i32
    lib.b200pf_device_count.restype = i32
    lib.b200pf_create.argtypes = [C.POINTER(_GridDesc), i32, i32, C.POINTER(vp)]
    lib.b200pf_destroy.argtypes = [vp]
    lib.b200pf_sizes.argtypes = [vp] + [C.POINTER(i32)] * 4
    lib.b200pf_run_host.argtypes = [vp, i32, vp, vp, i32, i32, f64, i32, vp, vp, vp, vp]
    lib.b200pf_run_device.argtypes = [vp, i32, vp, vp, i32, i32, f64, i32, vp, vp, vp, vp]
    lib.b200pf_run_device_topo.argtypes = [vp, i32, vp, vp, vp, i32, i32, f64, i32, vp, vp, vp, vp]
    lib.b200pf_series_bind.argtypes = [vp, vp, i32, i32, vp, vp, i32, vp, vp]
    lib.b200pf_series_set_topo.argtypes = [vp, vp]
    lib.b200pf_series_step.argtypes = [vp, i32, i32, f64, i32]
    lib.b200pf_series_results.argtypes = [vp] + [C.POINTER(vp)] * 5
    lib.b200pf_series_fetch.argtypes = [vp, vp, vp, vp, vp]
    lib.b200pf_sync.argtypes = [vp]
    lib.b200pf_staging.argtypes = [vp] + [C.POINTER(vp)] * 6
    lib.b200pf_run_staged.argtypes = [vp, i32, i32, i32, f64, i32, i32]
    lib.b200pf_series_bind_outputs.argtypes = [vp, vp, vp, vp, vp]
    lib.b200pf_set_stream.argtypes = [vp, C.c_uint64]
    lib.b200pf_set_static_inj.argtypes = [vp, vp]
    lib.b200pf_rows_staging.argtypes = [vp, C.POINTER(vp)]
    lib.b200pf_run_rows_staged.argtypes = [vp, i32, i32, i32, f64, i32]
    lib.b200pf_set_thermal_limit.argtypes = [vp, vp]
    lib.b200pf_n1_host.argtypes = [vp, i32, vp, vp, i32, f64, i32, vp, vp]
    lib.b200pf_series_protections.argtypes = [vp, i32, C.c_float, C.c_float, i32]
    lib.b200pf_series_next_is_reset.argtypes = [vp]
    lib.b200pf_series_fetch_state.argtypes = [vp, vp, vp, vp, vp]
    lib.b200pf_rows_chunk_launch.argtypes = [vp, i32, i32, i32, i32, f64, i32]
    lib.b200pf_rows_chunk_wait.argtypes = [vp]
    lib.b200pf_rows_chunk_launch_from.argtypes = [vp, i32, i32, vp, i32, i32, f64, i32]
    lib.b200pf_pinned_alloc.argtypes = [C.c_size_t, C.POINTER(vp)]
    lib.b200pf_rows_group_launch.argtypes = [vp, i32, i32, i32, vp, i32, i32, f64, i32]
    lib.b200pf_rows_group_wait.argtypes = [vp, i32]
    lib.b200pf_rows_group_config.argtypes = [vp, i32]
    lib.b200pf_pinned_free.argtypes = [vp]
    lib.b200pf_stream.argtypes = [vp]
    lib.b200pf_stream.restype = C.c_uint64
    lib.b200pf_launch_count.argtypes = [vp]
    lib.b200pf_launch_count.restype = C.c_int64
    lib.b200pf_last_launch_info.argtypes = [vp] + [C.POINTER(i32)] * 4
    lib.b200pf_last_launch_config.argtypes = [vp, C.POINTER(i32)]
    lib.b200pf_set_kernel_policy.argtypes = [vp, i32]
    lib.b200pf_plan_stats.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(i32)]
    lib.b200pf_set_debug.argtypes = [vp, i32, i32]
    lib.b200pf_plan_counters.argtypes = [vp, C.POINTER(C.c_int64)]
    lib.b200pf_series_bind_flag.argtypes = [vp, vp]
    lib.b200pf_series_reset_instances.argtypes = [vp, i32, vp, vp, vp]
    lib.b200pf_series_reset_instances.restype = i32
    lib.b200pf_grid_max_active_buses.argtypes = [C.POINTER(_GridDesc), i32, vp, vp, C.POINTER(i32)]
    lib.b200pf_grid_max_active_buses.restype = i32
    lib.b200pf_series_bind_flag.restype = i32
    lib.b200pf_plan_counters.restype = i32
    lib.b200pf_device_alloc.argtypes = [C.c_size_t, C.POINTER(vp)]
    lib.b200pf_device_free.argtypes = [vp]
    lib.b200pf_ipc_export.argtypes = [vp, vp]
    lib.b200pf_ipc_open.argtypes = [vp, C.POINTER(vp)]
    lib.b200pf_ipc_close.argtypes = [vp]
    lib.b200pf_device_read.argtypes = [vp, vp, C.c_size_t]
    lib.b200pf_device_read.restype = i32
    for nm in ("b200pf_set_debug", "b200pf_device_alloc", "b200pf_device_free", "b200pf_ipc_export", "b200pf_ipc_open", "b200pf_ipc_close"):
        getattr(lib, nm).restype = i32
    lib.b200pf_obs_bind.argtypes = [vp, C.POINTER(ObsDesc)]
    lib.b200pf_observe.argtypes = [vp, vp, vp, vp]
    lib.b200pf_obs_stats.argtypes = [vp, C.POINTER(C.c_int64)]
    for nm in ("b200pf_obs_bind", "b200pf_observe", "b200pf_obs_stats"):
        getattr(lib, nm).restype = i32
    lib.b200pf_env_bind.argtypes = [vp, C.POINTER(EnvDesc)]
    lib.b200pf_env_step.argtypes = [vp, vp, vp, i32, i32, vp, vp, i32, i32, i32, f64, i32, i32]
    lib.b200pf_env_reset.argtypes = [vp, vp, vp]
    lib.b200pf_env_get_state.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.b200pf_env_set_state.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.b200pf_env_pointers.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
    lib.b200pf_observe_device.argtypes = [vp, vp, vp]
    lib.b200pf_env_stats.argtypes = [vp, C.POINTER(C.c_int64)]
    lib.b200pf_opp_bind.argtypes = [vp, C.POINTER(OppDesc)]
    lib.b200pf_opp_get_state.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.b200pf_opp_set_state.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.b200pf_opp_geo_bind.argtypes = [vp, C.POINTER(OppGeoDesc)]
    lib.b200pf_opp_geo_get_state.argtypes = [vp, vp, vp, vp]
    lib.b200pf_opp_geo_set_state.argtypes = [vp, vp, vp, vp]
    lib.b200pf_opp_multi_bind.argtypes = [vp, C.POINTER(OppMultiDesc)]
    lib.b200pf_opp_multi_get_state.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.b200pf_opp_multi_set_state.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.b200pf_alert_bind.argtypes = [vp, C.POINTER(AlertDesc)]
    lib.b200pf_alert_get_state.argtypes = [vp] + [vp] * 12
    lib.b200pf_alert_set_state.argtypes = [vp] + [vp] * 12
    lib.b200pf_alarm_bind.argtypes = [vp, C.POINTER(AlarmDesc)]
    lib.b200pf_alarm_get_state.argtypes = [vp] + [vp] * 10
    lib.b200pf_alarm_set_state.argtypes = [vp] + [vp] * 10
    lib.b200pf_act_bind.argtypes = [vp, C.POINTER(ActDesc)]
    lib.b200pf_env_step_act.argtypes = [vp, i32, i32, i32, f64, i32, i32]
    lib.b200pf_act_table_bind.argtypes = [vp, C.POINTER(ActTableDesc)]
    lib.b200pf_env_step_ids.argtypes = [vp, vp, i32, i32, i32, f64, i32, i32]
    for nm in ("b200pf_env_bind", "b200pf_env_step", "b200pf_env_reset", "b200pf_env_get_state", "b200pf_env_set_state",
               "b200pf_env_pointers", "b200pf_observe_device", "b200pf_env_stats", "b200pf_opp_bind", "b200pf_opp_get_state",
               "b200pf_opp_set_state", "b200pf_opp_geo_bind", "b200pf_opp_geo_get_state", "b200pf_opp_geo_set_state",
               "b200pf_opp_multi_bind", "b200pf_opp_multi_get_state", "b200pf_opp_multi_set_state", "b200pf_alert_bind",
               "b200pf_alert_get_state", "b200pf_alert_set_state", "b200pf_alarm_bind", "b200pf_alarm_get_state",
               "b200pf_alarm_set_state", "b200pf_act_bind", "b200pf_env_step_act", "b200pf_act_table_bind", "b200pf_env_step_ids"):
        getattr(lib, nm).restype = i32
    lib.b200pf_redo_launch_count.argtypes = [vp]
    lib.b200pf_redo_launch_count.restype = C.c_int64
    for nm in ("b200pf_create", "b200pf_destroy", "b200pf_sizes", "b200pf_run_host", "b200pf_run_device",
               "b200pf_series_bind", "b200pf_series_set_topo", "b200pf_series_step", "b200pf_series_results",
               "b200pf_series_fetch", "b200pf_sync", "b200pf_last_launch_info", "b200pf_last_launch_config", "b200pf_staging", "b200pf_run_staged",
               "b200pf_series_bind_outputs", "b200pf_set_stream", "b200pf_set_static_inj", "b200pf_rows_staging",
               "b200pf_run_rows_staged", "b200pf_set_thermal_limit", "b200pf_n1_host", "b200pf_series_protections",
               "b200pf_series_next_is_reset", "b200pf_series_fetch_state", "b200pf_rows_chunk_launch", "b200pf_rows_chunk_wait",
               "b200pf_rows_chunk_launch_from", "b200pf_pinned_alloc", "b200pf_pinned_free", "b200pf_rows_group_launch",
               "b200pf_rows_group_wait", "b200pf_rows_group_config"):
        getattr(lib, nm).restype = i32
    _LIB = lib
    return lib


class PeerBuffer:
    """Device buffer of the agent's rank that the other ranks (one process per GPU) map over NVLink (CUDA IPC) and let their
    kernels store results into directly (include/b200pf.h, "Multi-GPU result collection")."""

    def __init__(self, nbytes: int = 0, handle: Optional[bytes] = None):
        self.lib = load_library()
        self.owner = handle is None
        p = C.c_void_p()
        if self.owner:
            rc = self.lib.b200pf_device_alloc(C.c_size_t(int(nbytes)), C.byref(p))
            if rc:
                raise RuntimeError(f"b200pf_device_alloc failed: {self.lib.b200pf_last_error().decode()}")
            buf = (C.c_ubyte * 64)()
            rc = self.lib.b200pf_ipc_export(p, C.cast(buf, C.c_void_p))
            if rc:
                raise RuntimeError(f"b200pf_ipc_export failed: {self.lib.b200pf_last_error().decode()}")
            self.handle = bytes(buf)
        else:
            buf = (C.c_ubyte * 64).from_buffer_copy(handle)
            rc = self.lib.b200pf_ipc_open(C.cast(buf, C.c_void_p), C.byref(p))
            if rc:
                raise RuntimeError(f"b200pf_ipc_open failed: {self.lib.b200pf_last_error().decode()}")
            self.handle = bytes(handle)
        self.ptr = int(p.value)

    def read(self, offset_bytes: int, n_float32: int) -> np.ndarray:
        out = np.empty(int(n_float32), dtype=np.float32)
        rc = self.lib.b200pf_device_read(C.c_void_p(self.ptr + int(offset_bytes)), out.ctypes.data_as(C.c_void_p), C.c_size_t(out.nbytes))
        if rc:
            raise RuntimeError(f"b200pf_device_read failed: {self.lib.b200pf_last_error().decode()}")
        return out

    def close(self):
        if getattr(self, "ptr", 0):
            (self.lib.b200pf_device_free if self.owner else self.lib.b200pf_ipc_close)(C.c_void_p(self.ptr))
            self.ptr = 0


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class OutputView:
    """Named float32 views into the packed result record ``out[batch, n_out]`` (include/b200pf.h)."""

    FIELDS = ("p_or", "q_or", "v_or", "a_or", "theta_or", "p_ex", "q_ex", "v_ex", "a_ex", "theta_ex", "unit_p", "unit_q", "unit_v",
              "unit_theta", "load_v", "load_theta", "storage_v", "shunt_p", "shunt_q", "shunt_v")

    @staticmethod
    def layout(gm: GridModel):
        """-> ((field, start, stop), ...) of the packed record (cached on the grid model)"""
        lay = getattr(gm, "_out_layout_cache", None)
        if lay is None:
            nl, nu, nld, ns, nsh = gm.n_line, gm.n_unit, gm.n_load, gm.n_storage, gm.n_shunt
            sizes = [nl] * 10 + [nu] * 4 + [nld, nld, ns, nsh, nsh, nsh]
            o, lay = 0, []
            for name, n in zip(OutputView.FIELDS, sizes):
                lay.append((name, o, o + n))
                o += n
            assert o == gm.n_out
            lay = gm._out_layout_cache = tuple(lay)
        return lay

    def __init__(self, gm: GridModel, out: np.ndarray):
        for name, a, b in OutputView.layout(gm):
            setattr(self, name, out[:, a:b])


def make_grid_desc(gm: GridModel):
    """-> (``b200pf_grid_desc`` of include/b200pf.h, the arrays it points to — keep them alive as long as the descriptor)"""
    keep = []
    d = _GridDesc()
    d.abi_version = 2
    d.n_sub, d.n_busbar = gm.n_sub, gm.n_busbar
    d.n_line, d.n_gen, d.n_hidden, d.n_load = gm.n_line, gm.n_gen, gm.n_hidden, gm.n_load
    d.n_storage, d.n_shunt, d.dim_topo = gm.n_storage, gm.n_shunt, gm.dim_topo
    d.sn_mva = gm.sn_mva

    def put(name, arr, dtype):
        a = np.ascontiguousarray(arr, dtype=dtype)
        if a.size == 0:
            a = np.zeros(1, dtype=dtype)
        keep.append(a)
        setattr(d, name, a.ctypes.data)

    i32, f64, f32 = np.int32, np.float64, np.float32
    put("line_or_sub", gm.line_or_sub, i32); put("line_ex_sub", gm.line_ex_sub, i32)
    put("line_or_pos", gm.line_or_pos, i32); put("line_ex_pos", gm.line_ex_pos, i32)
    put("line_y", gm.line_y, f64); put("line_bdc", gm.line_bdc, f64); put("line_pshift", gm.line_pshift, f64)
    put("line_or_vn", gm.line_or_vn, f32); put("line_ex_vn", gm.line_ex_vn, f32)
    put("unit_sub", gm.unit_sub, i32); put("unit_pos", gm.unit_pos, i32); put("unit_is_ref", gm.unit_is_ref, i32)
    put("unit_qmin", gm.unit_qmin, f64); put("unit_qmax", gm.unit_qmax, f64); put("unit_vn", gm.unit_vn, f32)
    put("load_sub", gm.load_sub, i32); put("load_pos", gm.load_pos, i32); put("load_vn", gm.load_vn, f32)
    put("storage_sub", gm.storage_sub, i32); put("storage_pos", gm.storage_pos, i32)
    put("storage_vn", gm.storage_vn, f32); put("storage_q", gm.storage_q, f64)
    put("shunt_sub", gm.shunt_sub, i32); put("shunt_vn", gm.shunt_vn, f32); put("shunt_vratio", gm.shunt_vratio, f64)
    put("sub_rank", getattr(gm, "sub_rank", np.arange(gm.n_sub)), i32)
    return d, keep


def grid_max_active_buses(gm: GridModel, topo: np.ndarray, desc=None):
    """Active buses (bus slots with a connected element) of every topology record, int8 [B, n_topo_in] -> (max, int32 [B]).
    Host code of the library (``b200pf_grid_max_active_buses``): needs no device."""
    lib = load_library()
    keep = None
    if desc is None:
        desc, keep = make_grid_desc(gm)
    topo = np.ascontiguousarray(topo, dtype=np.int8).reshape(-1, gm.n_topo_in)
    cnt = np.empty(topo.shape[0], dtype=np.int32)
    best = C.c_int32(0)
    if topo.shape[0]:
        rc = lib.b200pf_grid_max_active_buses(C.byref(desc), topo.shape[0], _ptr(topo), _ptr(cnt), C.byref(best))
        if rc != 0:
            raise RuntimeError(f"b200pf_grid_max_active_buses failed ({rc}): {lib.b200pf_last_error().decode()}")
    del keep
    return int(best.value), cnt


class PowerFlowEngine:
    """One device handle: static grid on the GPU + staging for up to ``max_batch`` instances."""

    def __init__(self, gm: GridModel, max_batch: int = 1, device: int = 0):
        self.gm = gm
        self.device = int(device)
        self.lib = load_library()
        if self.lib.b200pf_abi_version() != 2:
            raise EngineUnavailable("libb200pf ABI version mismatch")
        self.max_batch = int(max_batch)
        d, self._keep = make_grid_desc(gm)
        self._desc = d                      # (its arrays live in self._keep)
        h = C.c_void_p()
        rc = self.lib.b200pf_create(C.byref(d), self.max_batch, int(device), C.byref(h))
        if rc != 0:
            raise EngineUnavailable(f"b200pf_create failed ({rc}): {self.lib.b200pf_last_error().decode()}")
        self.h = h
        n = [C.c_int() for _ in range(4)]
        self.lib.b200pf_sizes(self.h, *[C.byref(v) for v in n])
        assert (n[0].value, n[1].value, n[2].value, n[3].value) == (gm.n_topo_in, gm.n_inj, gm.n_out, gm.n_slot)

    # ------------------------------------------------------------------------------------------
    def _check(self, rc: int, what: str):
        if rc != 0:
            raise RuntimeError(f"{what} failed ({rc}): {self.lib.b200pf_last_error().decode()}")

    def close(self):
        if getattr(self, "h", None) is not None and self.h:
            self.lib.b200pf_destroy(self.h)
            self.h = None
        for p in getattr(self, "_pinned", []):
            self.lib.b200pf_pinned_free(p)
        self._pinned = []

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def max_active_buses(self, topo: np.ndarray, per_instance: bool = False):
        """Largest number of active buses (bus slots with at least one connected element) over a batch of topology records: the
        tight ``nb_cap`` for a launch (0 = unknown -> size for every slot).  ``per_instance``: -> (max, int32 [B]).  Host code of
        the library (``b200pf_grid_max_active_buses``)."""
        gm = self.gm
        topo = np.ascontiguousarray(topo, dtype=np.int8).reshape(-1, gm.n_topo_in)
        n = topo.shape[0]
        cnt = np.empty(n, dtype=np.int32) if per_instance else None
        best = C.c_int32(0)
        if n:
            self._check(self.lib.b200pf_grid_max_active_buses(C.byref(self._desc), n, _ptr(topo), _ptr(cnt), C.byref(best)),
                        "b200pf_grid_max_active_buses")
        return (int(best.value), cnt) if per_instance else int(best.value)

    def run(self, topo: np.ndarray, inj: np.ndarray, is_dc: bool = False, max_iter: int = 10,
            tol_mva: float = 1e-8, nb_cap: int = -1, want_busv: bool = False
            ) -> Tuple[np.ndarray, np.ndarray, np.ndarray, Optional[np.ndarray]]:
        """Host-buffer entry point (H2D + kernel + D2H).  ``topo`` int8 [B, n_topo_in], ``inj`` f64 [B, n_inj].
        ``nb_cap`` < 0: computed from ``topo`` (tight bound -> the warp-per-instance kernel when it applies)."""
        gm = self.gm
        topo = np.ascontiguousarray(topo, dtype=np.int8).reshape(-1, gm.n_topo_in)
        inj = np.ascontiguousarray(inj, dtype=np.float64).reshape(-1, gm.n_inj)
        B = topo.shape[0]
        if nb_cap < 0:
            nb_cap = self.max_active_buses(topo)
        if inj.shape[0] != B:
            raise ValueError("topo / inj batch mismatch")
        out = np.empty((B, gm.n_out), dtype=np.float32)
        status = np.empty(B, dtype=np.int32)
        iters = np.empty(B, dtype=np.int32)
        busv = np.empty((B, 2 * gm.n_slot), dtype=np.float64) if want_busv else None
        rc = self.lib.b200pf_run_host(self.h, B, _ptr(topo), _ptr(inj), int(bool(is_dc)), int(max_iter), float(tol_mva),
                                      int(nb_cap), _ptr(out), _ptr(status), _ptr(iters), _ptr(busv))
        self._check(rc, "b200pf_run_host")
        return out, status, iters, busv

    def run_device(self, batch: int, d_topo: int, d_inj: int, d_out: int, d_status: int, d_iters: int,
                   d_busv: int = 0, is_dc: bool = False, max_iter: int = 10, tol_mva: float = 1e-8, nb_cap: int = 0,
                   host_topo: Optional[np.ndarray] = None):
        """Device-pointer entry point (asynchronous on the handle's stream).  ``host_topo`` (the same records as
        ``d_topo``, as a host array) lets the engine use the planned sparse kernel."""
        if host_topo is not None:
            ht = np.ascontiguousarray(host_topo, dtype=np.int8)
            rc = self.lib.b200pf_run_device_topo(self.h, int(batch), _ptr(ht), C.c_void_p(d_topo), C.c_void_p(d_inj), int(bool(is_dc)),
                                                 int(max_iter), float(tol_mva), int(nb_cap), C.c_void_p(d_out),
                                                 C.c_void_p(d_status), C.c_void_p(d_iters), C.c_void_p(d_busv) if d_busv else None)
            self._check(rc, "b200pf_run_device_topo")
            return
        rc = self.lib.b200pf_run_device(self.h, int(batch), C.c_void_p(d_topo), C.c_void_p(d_inj), int(bool(is_dc)),
                                        int(max_iter), float(tol_mva), int(nb_cap), C.c_void_p(d_out),
                                        C.c_void_p(d_status), C.c_void_p(d_iters), C.c_void_p(d_busv) if d_busv else None)
        self._check(rc, "b200pf_run_device")

    # ---- zero-copy host path ------------------------------------------------------------------
    def staging(self):
        """numpy views of the handle's pinned staging buffers (topo, inj, out, status, iters)."""
        gm, B = self.gm, self.max_batch
        p = [C.c_void_p() for _ in range(6)]
        self._check(self.lib.b200pf_staging(self.h, *[C.byref(v) for v in p]), "b200pf_staging")

        def view(ptr, ctype, shape):
            n = int(np.prod(shape))
            arr = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), shape=(n,))
            return arr.reshape(shape)

        return dict(topo=view(p[0], C.c_int8, (B, gm.n_topo_in)), inj=view(p[1], C.c_double, (B, gm.n_inj)),
                    out=view(p[2], C.c_float, (B, gm.n_out)), status=view(p[3], C.c_int32, (B,)),
                    iters=view(p[4], C.c_int32, (B,)))

    def run_staged(self, batch: int, is_dc: bool = False, max_iter: int = 10, tol_mva: float = 1e-8, nb_cap: int = 0):
        self._check(self.lib.b200pf_run_staged(self.h, int(batch), int(bool(is_dc)), int(max_iter), float(tol_mva),
                                               int(nb_cap), 0), "b200pf_run_staged")

    def rows_staging(self) -> np.ndarray:
        """numpy view of the pinned float32 rows buffer [max_batch, 2 n_load + 2 n_gen]."""
        gm, B = self.gm, self.max_batch
        p = C.c_void_p()
        self._check(self.lib.b200pf_rows_staging(self.h, C.byref(p)), "b200pf_rows_staging")
        ncol = 2 * gm.n_load + 2 * gm.n_gen
        arr = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_float)), shape=(B * ncol,))
        return arr.reshape(B, ncol)

    def set_static_inj(self, static_inj: np.ndarray):
        a = np.ascontiguousarray(static_inj, dtype=np.float64)
        assert a.shape == (self.gm.n_inj,)
        self._check(self.lib.b200pf_set_static_inj(self.h, _ptr(a)), "b200pf_set_static_inj")

    def run_rows_staged(self, batch: int, is_dc: bool = False, max_iter: int = 10, tol_mva: float = 1e-8, nb_cap: int = 0):
        self._check(self.lib.b200pf_run_rows_staged(self.h, int(batch), int(bool(is_dc)), int(max_iter), float(tol_mva),
                                                    int(nb_cap)), "b200pf_run_rows_staged")

    def n1_sweep(self, topo: np.ndarray, inj: np.ndarray, thermal_limit_a: Optional[np.ndarray] = None,
                 max_iter: int = 10, tol_mva: float = 1e-8, nb_cap: int = -1):
        """All single-line outages of every base state in one launch.  Returns ``rho [B, n_line(outage), n_line]``
        and ``status [B, n_line]`` (reference pattern: examples/backend_dependant_code/_obs_with_n1.py:111-125)."""
        gm = self.gm
        topo = np.ascontiguousarray(topo, dtype=np.int8).reshape(-1, gm.n_topo_in)
        inj = np.ascontiguousarray(inj, dtype=np.float64).reshape(-1, gm.n_inj)
        B = topo.shape[0]
        th = np.ascontiguousarray(gm.thermal_limit_a if thermal_limit_a is None else thermal_limit_a, dtype=np.float32)
        self._check(self.lib.b200pf_set_thermal_limit(self.h, _ptr(th)), "b200pf_set_thermal_limit")
        if nb_cap < 0:
            nb_cap = self.max_active_buses(topo)      # an outage can only remove buses
        rho = np.empty((B, gm.n_line, gm.n_line), dtype=np.float32)
        status = np.empty((B, gm.n_line), dtype=np.int32)
        self._check(self.lib.b200pf_n1_host(self.h, B, _ptr(topo), _ptr(inj), int(max_iter), float(tol_mva), int(nb_cap),
                                            _ptr(rho), _ptr(status)), "b200pf_n1_host")
        return rho, status

    def rows_chunk_launch(self, first: int, count: int, is_dc: bool = False, max_iter: int = 10, tol_mva: float = 1e-8,
                          nb_cap: int = 0):
        self._check(self.lib.b200pf_rows_chunk_launch(self.h, int(first), int(count), int(bool(is_dc)), int(max_iter),
                                                      float(tol_mva), int(nb_cap)), "b200pf_rows_chunk_launch")

    def pinned_empty(self, shape, dtype=np.float32) -> np.ndarray:
        """numpy array backed by page-locked host memory (freed with the engine)."""
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        p = C.c_void_p()
        self._check(self.lib.b200pf_pinned_alloc(C.c_size_t(n), C.byref(p)), "b200pf_pinned_alloc")
        self._pinned = getattr(self, "_pinned", []) + [p]
        buf = (C.c_char * n).from_address(p.value)
        return np.frombuffer(buf, dtype=dtype).reshape(shape)

    def rows_chunk_launch_from(self, first: int, count: int, pinned_rows: np.ndarray, is_dc: bool = False, max_iter: int = 10,
                               tol_mva: float = 1e-8, nb_cap: int = 0):
        self._check(self.lib.b200pf_rows_chunk_launch_from(self.h, int(first), int(count), C.c_void_p(pinned_rows.ctypes.data),
                                                           int(bool(is_dc)), int(max_iter), float(tol_mva), int(nb_cap)),
                    "b200pf_rows_chunk_launch_from")

    def rows_group_launch(self, group: int, first: int, count: int, pinned_rows: Optional[np.ndarray] = None, is_dc: bool = False,
                          max_iter: int = 10, tol_mva: float = 1e-8, nb_cap: int = 0):
        """Asynchronous: H2D -> kernel -> D2H of instances [first, first+count) on the stream of ``group``."""
        ptr = C.c_void_p(pinned_rows.ctypes.data) if pinned_rows is not None else None
        self._check(self.lib.b200pf_rows_group_launch(self.h, int(group), int(first), int(count), ptr, int(bool(is_dc)),
                                                      int(max_iter), float(tol_mva), int(nb_cap)), "b200pf_rows_group_launch")

    GROUP_DIRECT_OUT, GROUP_ZEROCOPY_IN, GROUP_DIRECT_STATUS = 1, 2, 4

    def rows_group_config(self, direct_out=False):
        """Flags of include/b200pf.h (an int), or a bool: True = GROUP_DIRECT_OUT (kernels store their results straight
        into the pinned staging buffers, no copy-engine D2H)."""
        flags = int(direct_out) if not isinstance(direct_out, bool) else (1 if direct_out else 0)
        self._check(self.lib.b200pf_rows_group_config(self.h, flags), "b200pf_rows_group_config")

    def rows_group_wait(self, group: int):
        self._check(self.lib.b200pf_rows_group_wait(self.h, int(group)), "b200pf_rows_group_wait")

    def rows_chunk_wait(self):
        self._check(self.lib.b200pf_rows_chunk_wait(self.h), "b200pf_rows_chunk_wait")

    def set_stream(self, stream: int):
        self._check(self.lib.b200pf_set_stream(self.h, C.c_uint64(int(stream))), "b200pf_set_stream")

    def series_bind_outputs(self, d_out: int = 0, d_status: int = 0, d_iters: int = 0, d_rho: int = 0):
        self._check(self.lib.b200pf_series_bind_outputs(self.h, C.c_void_p(d_out or None), C.c_void_p(d_status or None),
                                                        C.c_void_p(d_iters or None), C.c_void_p(d_rho or None)),
                    "b200pf_series_bind_outputs")

    # ---- time series -------------------------------------------------------------------------
    def series_bind(self, chron: np.ndarray, scen: np.ndarray, t0: np.ndarray, static_inj: np.ndarray,
                    thermal_limit_a: np.ndarray):
        gm = self.gm
        chron = np.ascontiguousarray(chron, dtype=np.float32)
        assert chron.ndim == 3 and chron.shape[2] == 2 * gm.n_load + 2 * gm.n_gen
        scen = np.ascontiguousarray(scen, dtype=np.int32)
        t0 = np.ascontiguousarray(t0, dtype=np.int32)
        static_inj = np.ascontiguousarray(static_inj, dtype=np.float64)
        th = np.ascontiguousarray(thermal_limit_a, dtype=np.float32)
        assert static_inj.shape == (gm.n_inj,) and th.shape == (gm.n_line,)
        self._series_batch = int(scen.shape[0])
        rc = self.lib.b200pf_series_bind(self.h, _ptr(chron), chron.shape[0], chron.shape[1], _ptr(scen), _ptr(t0),
                                         self._series_batch, _ptr(static_inj), _ptr(th))
        self._check(rc, "b200pf_series_bind")

    def series_set_topo(self, topo: np.ndarray):
        topo = np.ascontiguousarray(topo, dtype=np.int8).reshape(self._series_batch, self.gm.n_topo_in)
        self._check(self.lib.b200pf_series_set_topo(self.h, _ptr(topo)), "b200pf_series_set_topo")

    def series_step(self, is_dc: bool = False, max_iter: int = 10, tol_mva: float = 1e-8, nb_cap: int = 0):
        self._check(self.lib.b200pf_series_step(self.h, int(bool(is_dc)), int(max_iter), float(tol_mva), int(nb_cap)),
                    "b200pf_series_step")

    def series_fetch(self, want_out=True, want_rho=True):
        gm, B = self.gm, self._series_batch
        out = np.empty((B, gm.n_out), dtype=np.float32) if want_out else None
        status = np.empty(B, dtype=np.int32)
        iters = np.empty(B, dtype=np.int32)
        rho = np.empty((B, gm.n_line), dtype=np.float32) if want_rho else None
        self._check(self.lib.b200pf_series_fetch(self.h, _ptr(out), _ptr(status), _ptr(iters), _ptr(rho)), "b200pf_series_fetch")
        return out, status, iters, rho

    def series_reset_instances(self, idx, t_new=None, topo_rows=None):
        """``env.reset()`` of single instances of the bound series: flags / counters cleared, next chronics row ``t_new``, topology
        ``topo_rows`` (int8 [n, n_topo_in])."""
        idx = np.ascontiguousarray(idx, dtype=np.int32)
        t = None if t_new is None else np.ascontiguousarray(t_new, dtype=np.int32)
        tr = None if topo_rows is None else np.ascontiguousarray(topo_rows, dtype=np.int8).reshape(len(idx), self.gm.n_topo_in)
        self._check(self.lib.b200pf_series_reset_instances(self.h, len(idx), _ptr(idx), _ptr(t), _ptr(tr)), "b200pf_series_reset_instances")

    def series_bind_flag(self, d_flag: int = 0):
        """the device stores the number of series steps done to ``*d_flag`` (device / peer pointer) behind every step"""
        self._check(self.lib.b200pf_series_bind_flag(self.h, C.c_void_p(d_flag or None)), "b200pf_series_bind_flag")

    def series_protections(self, enabled: bool = True, hard_overflow_threshold: float = 2.0,
                           soft_overflow_threshold: float = 1.0, nb_timestep_overflow_allowed: int = 2):
        """Defaults = grid2op.Parameters defaults (Parameters.py:255-270)."""
        self._check(self.lib.b200pf_series_protections(self.h, int(bool(enabled)), float(hard_overflow_threshold),
                                                       float(soft_overflow_threshold), int(nb_timestep_overflow_allowed)),
                    "b200pf_series_protections")

    def series_next_is_reset(self):
        self._check(self.lib.b200pf_series_next_is_reset(self.h), "b200pf_series_next_is_reset")

    def series_fetch_state(self):
        gm, B = self.gm, self._series_batch
        pc = np.empty((B, gm.n_line), dtype=np.int32); tso = np.empty((B, gm.n_line), dtype=np.int32)
        disc = np.empty((B, gm.n_line), dtype=np.int32); done = np.empty(B, dtype=np.int32)
        self._check(self.lib.b200pf_series_fetch_state(self.h, _ptr(pc), _ptr(tso), _ptr(disc), _ptr(done)), "b200pf_series_fetch_state")
        return dict(protection_counter=pc, timestep_overflow=tso, disc_lines=disc, done=done)

    def series_device_pointers(self):
        p = [C.c_void_p() for _ in range(5)]
        self._check(self.lib.b200pf_series_results(self.h, *[C.byref(v) for v in p]), "b200pf_series_results")
        return dict(out=p[0].value, status=p[1].value, iters=p[2].value, rho=p[3].value, t=p[4].value)

    # ---- observation layer -------------------------------------------------------------------
    def obs_bind(self, tables: dict):
        """Static tables of the observation layer for the bound series (``b200pf_obs_bind``; built by BatchedEnv.enable_observation)."""
        d, keep = make_obs_desc(tables)
        self._check(self.lib.b200pf_obs_bind(self.h, C.byref(d)), "b200pf_obs_bind")
        del keep

    def observe(self, host_in: np.ndarray, d_obs: int, d_reward: int = 0):
        """Asynchronous on the handle's stream: H2D of the per-instance host inputs (int32 [batch, n_line + n_sub + 3]), one launch
        writing obs f32 [batch, n_obs] / reward f32 [batch] to the DEVICE pointers ``d_obs`` / ``d_reward``."""
        h = np.ascontiguousarray(host_in, dtype=np.int32)
        self._check(self.lib.b200pf_observe(self.h, _ptr(h), C.c_void_p(d_obs), C.c_void_p(d_reward or None)), "b200pf_observe")

    def obs_stats(self):
        v = (C.c_int64 * 4)()
        self._check(self.lib.b200pf_obs_stats(self.h, v), "b200pf_obs_stats")
        return dict(launches=int(v[0]), h2d_bytes=int(v[1]), d2h_bytes=int(v[2]), bytes_written_per_launch=int(v[3]))

    # ---- device environment state ---------------------------------------------------------------
    def env_bind(self, tables: dict, state: dict):
        """Static tables + caller-owned per-instance device buffers of the device environment (``b200pf_env_bind``; built by
        BatchedEnv)."""
        d, keep = make_env_desc(tables, state)
        self._check(self.lib.b200pf_env_bind(self.h, C.byref(d)), "b200pf_env_bind")
        del keep

    def env_step(self, sub_id: int = 0, sub_bus: int = 0, sub_bus_stride: int = 0, sub_bus_cols: int = 0, line_id: int = 0,
                 line_status: int = 0, from_reset: bool = False, is_dc: bool = False, max_iter: int = 10, tol_mva: float = 1e-8,
                 tight_cap: bool = True, stamp: int = 0):
        """One env step of the bound series from device action buffers (integer addresses, 0 = none); one host wait."""
        v = lambda x: C.c_void_p(int(x) or None)      # noqa: E731
        self._check(self.lib.b200pf_env_step(self.h, v(sub_id), v(sub_bus), int(sub_bus_stride), int(sub_bus_cols), v(line_id),
                                             v(line_status), int(bool(from_reset)), int(bool(is_dc)), int(max_iter), float(tol_mva),
                                             int(bool(tight_cap)), int(stamp)), "b200pf_env_step")

    def env_step_act(self, from_reset: bool = False, is_dc: bool = False, max_iter: int = 10, tol_mva: float = 1e-8, tight_cap: bool = True,
                     stamp: int = 0):
        """:meth:`env_step` with the action taken from the vector buffers :meth:`act_bind` bound (``b200pf_env_step_act``)"""
        self._check(self.lib.b200pf_env_step_act(self.h, int(bool(from_reset)), int(bool(is_dc)), int(max_iter), float(tol_mva),
                                                 int(bool(tight_cap)), int(stamp)), "b200pf_env_step_act")

    def env_step_ids(self, d_action_id: int, from_reset: bool = False, is_dc: bool = False, max_iter: int = 10, tol_mva: float = 1e-8,
                     tight_cap: bool = True, stamp: int = 0):
        """:meth:`env_step_act` with instance i acting with row ``d_action_id[i]`` (device int32 [B]) of the table
        :meth:`act_table_bind` bound (``b200pf_env_step_ids``)"""
        self._check(self.lib.b200pf_env_step_ids(self.h, C.c_void_p(int(d_action_id)), int(bool(from_reset)), int(bool(is_dc)), int(max_iter),
                                                 float(tol_mva), int(bool(tight_cap)), int(stamp)), "b200pf_env_step_ids")

    def act_table_bind(self, set_bus, change_bus, set_line_status, change_line_status):
        """the discrete action table (``b200pf_act_table_bind``): host arrays int8 / bool [n, dim_topo] and int8 / bool [n, n_line],
        checked row by row and copied to device memory the library owns"""
        sb, ss = np.ascontiguousarray(set_bus, np.int8), np.ascontiguousarray(set_line_status, np.int8)
        cb, cs = np.ascontiguousarray(change_bus, np.uint8), np.ascontiguousarray(change_line_status, np.uint8)
        d = ActTableDesc(n_act=len(sb), set_bus=sb.ctypes.data, change_bus=cb.ctypes.data, set_status=ss.ctypes.data,
                         change_status=cs.ctypes.data)
        self._check(self.lib.b200pf_act_table_bind(self.h, C.byref(d)), "b200pf_act_table_bind")

    def act_bind(self, max_sub_changed: int, max_line_status_changed: int, n_area: int, sub_area, line_area, d_set_bus: int,
                 d_change_bus: int, d_set_status: int, d_change_status: int, d_is_ambiguous: int):
        """the agent's action rules and the vector-action buffers of the device environment (``b200pf_act_bind``): ``n_area``
        RulesByArea areas (0: none) with ``sub_area`` / ``line_area`` their uint32 masks [n_sub] / [n_line]; caller-owned device
        buffers int8 / uint8 [B, dim_topo] (set_bus / change_bus), int8 / uint8 [B, n_line] (set / change line status) and uint8
        [B] (is_ambiguous)"""
        sa = la = None
        if n_area:
            sa, la = np.ascontiguousarray(sub_area, np.uint32), np.ascontiguousarray(line_area, np.uint32)
        d = ActDesc(max_sub_changed=int(max_sub_changed), max_line_status_changed=int(max_line_status_changed), n_area=int(n_area),
                    sub_area=None if sa is None else sa.ctypes.data, line_area=None if la is None else la.ctypes.data,
                    set_bus=int(d_set_bus), change_bus=int(d_change_bus), set_status=int(d_set_status), change_status=int(d_change_status),
                    is_ambiguous=int(d_is_ambiguous))
        self._check(self.lib.b200pf_act_bind(self.h, C.byref(d)), "b200pf_act_bind")

    def env_reset(self, d_mask: int, d_rows: int = 0):
        self._check(self.lib.b200pf_env_reset(self.h, C.c_void_p(int(d_mask)), C.c_void_p(int(d_rows) or None)), "b200pf_env_reset")

    def _get_state(self, fn: str, spec):
        """-> {key: array} that the C entry point ``fn`` fills; ``spec``: (key, dtype, shape) in its argument order"""
        s = {k: np.empty(shape, dt) for k, dt, shape in spec}
        self._check(getattr(self.lib, fn)(self.h, *[_ptr(s[k]) for k, _, _ in spec]), fn)
        return s

    def _set_state(self, fn: str, spec, s: dict):
        """``s[key]`` as ``dtype`` of ``shape`` to the C entry point ``fn`` (None: not copied); ``spec`` as for :meth:`_get_state`"""
        a = [None if s[k] is None else np.ascontiguousarray(s[k], dt).reshape(shape) for k, dt, shape in spec]
        self._check(getattr(self.lib, fn)(self.h, *[_ptr(x) for x in a]), fn)

    def env_get_state(self):
        """-> dict(topo int8 [B, n_topo_in], t int32 [B], nb_inst int32 [B], cap_dirty bool [B], obs_reset bool [B])"""
        B = self._series_batch
        s = self._get_state("b200pf_env_get_state", (("topo", np.int8, (B, self.gm.n_topo_in)), ("t", np.int32, B), ("nb_inst", np.int32, B),
                                                      ("cap_dirty", np.uint8, B), ("obs_reset", np.uint8, B)))
        s["cap_dirty"], s["obs_reset"] = s["cap_dirty"].astype(bool), s["obs_reset"].astype(bool)
        return s

    def env_set_state(self, topo=None, nb_inst=None, cap_dirty=None, obs_reset=None, obs_in=None):
        B = self._series_batch
        self._set_state("b200pf_env_set_state", (("topo", np.int8, (B, self.gm.n_topo_in)), ("nb_inst", np.int32, B), ("cap_dirty", np.uint8, B),
                                                 ("obs_reset", np.uint8, B), ("obs_in", np.int32, (B, -1))),
                        dict(topo=topo, nb_inst=nb_inst, cap_dirty=cap_dirty, obs_reset=obs_reset, obs_in=obs_in))

    def env_pointers(self):
        p = [C.c_void_p() for _ in range(3)]
        self._check(self.lib.b200pf_env_pointers(self.h, *[C.byref(x) for x in p]), "b200pf_env_pointers")
        return dict(topo=p[0].value, t=p[1].value, disc=p[2].value)

    def opp_bind(self, t: dict, d_attack_line: int, d_attack_dur: int, d_budget: int):
        """Line-attack opponent of the device environment (``b200pf_opp_bind``): constants and initial random states ``t`` (built
        by BatchedEnv.enable_opponent), caller-owned device outputs int32 / int32 / float64 [batch]."""
        keep = [np.ascontiguousarray(t["lines"], np.int32), np.ascontiguousarray(t["rho_norm"], np.float64),
                np.ascontiguousarray(t["mt"], np.uint32), np.ascontiguousarray(t["mt_pos"], np.int32)]
        d = OppDesc(kind=int(t["kind"]), n_attack=len(keep[0]), lines=keep[0].ctypes.data, rho_norm=keep[1].ctypes.data,
                    attack_period=int(t["attack_period"]), attack_duration=int(t["attack_duration"]), attack_cooldown=int(t["attack_cooldown"]),
                    budget_per_ts=float(t["budget_per_ts"]), init_budget=float(t["init_budget"]), mt=keep[2].ctypes.data,
                    mt_pos=keep[3].ctypes.data, attack_line=int(d_attack_line), attack_dur=int(d_attack_dur), budget=int(d_budget))
        self._check(self.lib.b200pf_opp_bind(self.h, C.byref(d)), "b200pf_opp_bind")
        del keep

    def _opp_spec(self):
        B = self._series_batch
        return (("budget", np.float64, B), ("budget64", np.uint8, B), ("ctr", np.int32, (B, 4)), ("mt", np.uint32, (B, 624)),
                ("mt_pos", np.int32, B))

    def opp_get_state(self):
        """-> dict(budget float64 [B], budget64 uint8 [B], ctr int32 [B, 4], mt uint32 [B, 624], mt_pos int32 [B])"""
        return self._get_state("b200pf_opp_get_state", self._opp_spec())

    def opp_set_state(self, s: dict):
        self._set_state("b200pf_opp_set_state", self._opp_spec(), s)

    def opp_geo_bind(self, t: dict):
        """the GeometricOpponent's constants and first schedules (``b200pf_opp_geo_bind``, after ``opp_bind`` with kind 3): ``t``
        built by BatchedEnv.enable_opponent"""
        keep = [np.ascontiguousarray(t["weights"], np.float64), np.ascontiguousarray(t["episode_max_time"], np.int32),
                np.ascontiguousarray(t["geo_wait"], np.int32), np.ascontiguousarray(t["geo_dur"], np.int32),
                np.ascontiguousarray(t["geo_ctr"], np.int32)]
        cap = int(keep[2].shape[1])
        d = OppGeoDesc(weights=keep[0].ctypes.data, p_hazard=float(t["p_hazard"]), p_recovery=float(t["p_recovery"]),
                       logq_hazard=float(t["logq_hazard"]), logq_recovery=float(t["logq_recovery"]), recovery_min=int(t["recovery_min"]),
                       cap=cap, episode_max_time=keep[1].ctypes.data, wait=keep[2].ctypes.data, dur=keep[3].ctypes.data,
                       gctr=keep[4].ctypes.data)
        self._check(self.lib.b200pf_opp_geo_bind(self.h, C.byref(d)), "b200pf_opp_geo_bind")
        self._opp_geo_cap = cap
        del keep

    def _opp_geo_spec(self):
        B, cap = self._series_batch, getattr(self, "_opp_geo_cap", 0)       # (unbound: the library refuses the call)
        return (("geo_wait", np.int32, (B, cap)), ("geo_dur", np.int32, (B, cap)), ("geo_ctr", np.int32, (B, 4)))

    def opp_geo_get_state(self):
        """-> dict(geo_wait int32 [B, cap], geo_dur int32 [B, cap], geo_ctr int32 [B, 4]) of the GeometricOpponent"""
        return self._get_state("b200pf_opp_geo_get_state", self._opp_geo_spec())

    def opp_geo_set_state(self, s: dict):
        self._set_state("b200pf_opp_geo_set_state", self._opp_geo_spec(), s)

    def opp_multi_bind(self, t: dict, d_attack_lines: int):
        """the GeometricOpponentMultiArea's areas, constants and first state (``b200pf_opp_multi_bind``, after ``opp_bind`` with kind
        4): ``t`` built by BatchedEnv.enable_opponent (the multi_* arrays of BatchedOpponent.get_state); ``d_attack_lines``: device
        int32 [B, n_area] for each step's attacked lines"""
        keep = dict(area_off=np.ascontiguousarray(t["area_off"], np.int32), weights=np.ascontiguousarray(t["weights"], np.float64),
                    emt=np.ascontiguousarray(t["episode_max_time"], np.int32))
        keep.update({k: np.ascontiguousarray(t[k], dt) for k, dt, _ in self._opp_multi_spec()})
        n_area, cap = int(keep["multi_wait"].shape[1]), int(keep["multi_wait"].shape[2])
        d = OppMultiDesc(n_area=n_area, area_off=keep["area_off"].ctypes.data, weights=keep["weights"].ctypes.data,
                         p_hazard=float(t["p_hazard"]), p_recovery=float(t["p_recovery"]), logq_hazard=float(t["logq_hazard"]),
                         logq_recovery=float(t["logq_recovery"]), recovery_min=int(t["recovery_min"]), cap=cap,
                         episode_max_time=keep["emt"].ctypes.data, mt=keep["multi_mt"].ctypes.data,
                         mt_pos=keep["multi_mt_pos"].ctypes.data, wait=keep["multi_wait"].ctypes.data, dur=keep["multi_dur"].ctypes.data,
                         actr=keep["multi_ctr"].ctypes.data, fails=keep["multi_fails"].ctypes.data, attack_lines=d_attack_lines)
        self._check(self.lib.b200pf_opp_multi_bind(self.h, C.byref(d)), "b200pf_opp_multi_bind")
        self._opp_multi_shape = (n_area, cap)
        del keep

    def _opp_multi_spec(self):
        B = self._series_batch
        A, cap = getattr(self, "_opp_multi_shape", (0, 0))                   # (unbound: the library refuses the call)
        return tuple(zip(MULTI_KEYS, (np.uint32,) + (np.int32,) * 5, ((B, A, 624), (B, A), (B, A, cap), (B, A, cap), (B, A, 6), (B,))))

    def opp_multi_get_state(self):
        """-> dict(multi_mt uint32 [B, n_area, 624], multi_mt_pos int32 [B, n_area], multi_wait / multi_dur int32 [B, n_area, cap],
        multi_ctr int32 [B, n_area, 6], multi_fails int32 [B]) of the GeometricOpponentMultiArea"""
        return self._get_state("b200pf_opp_multi_get_state", self._opp_multi_spec())

    def opp_multi_set_state(self, s: dict):
        self._set_state("b200pf_opp_multi_set_state", self._opp_multi_spec(), s)

    def alert_bind(self, a, d_raise: int, d_reward: int):
        """line alerts of the device environment (``b200pf_alert_bind``): ``a`` a :class:`grid2op_b200.alert.BatchedAlerts` (lines,
        window, constants), caller-owned device buffers uint8 [B, n] (the step's raise_alert) and float64 [B] (AlertReward)"""
        lines = np.ascontiguousarray(a.lines, np.int32)
        c = a.constants
        d = AlertDesc(n_alert=len(lines), lines=lines.ctypes.data, window=int(a.window), reward=int(a.reward),
                      reward_min_no_blackout=float(c["reward_min_no_blackout"]), reward_min_blackout=float(c["reward_min_blackout"]),
                      reward_max_no_blackout=float(c["reward_max_no_blackout"]), reward_max_blackout=float(c["reward_max_blackout"]),
                      raise_alert=int(d_raise), reward_out=int(d_reward))
        self._check(self.lib.b200pf_alert_bind(self.h, C.byref(d)), "b200pf_alert_bind")
        self._alert_shape = (len(lines), int(a.ring))

    def _alert_spec(self):
        B = self._series_batch
        n, R = getattr(self, "_alert_shape", (0, 0))                        # (unbound: the library refuses the call)
        return tuple((k, dt, (B,) if k in ("total", "cur_id") else (B, R, n) if k in ("ts_attack", "launched") else (B, n))
                     for k, dt in ALERT_STATE)

    def alert_get_state(self):
        """-> the alert state of every instance, the arrays of :data:`grid2op_b200.alert.ALERT_STATE`"""
        return self._get_state("b200pf_alert_get_state", self._alert_spec())

    def alert_set_state(self, s: dict):
        self._set_state("b200pf_alert_set_state", self._alert_spec(), s)

    def alarm_bind(self, a, d_raise: int, d_reward: int, d_illegal: int):
        """alarms of the device environment (``b200pf_alarm_bind``): ``a`` a :class:`grid2op_b200.alarm.BatchedAlarms` (zones,
        constants), caller-owned device buffers uint8 [B, n] (the step's raise_alarm), float64 [B] (AlarmReward) and uint8 [B]
        (is_alarm_illegal)"""
        zm = np.ascontiguousarray(a.zone_mask, np.uint32)
        d = AlarmDesc(n_zone=int(a.n), zone_mask=zm.ctypes.data, max_budget=float(a.max_budget), budget_per_ts=float(a.budget_per_ts),
                      alarm_cost=float(a.alarm_cost), init_budget=float(a.init_budget), best_time=int(a.best_time),
                      window_size=int(a.window), reward=int(a.reward), raise_alarm=int(d_raise), reward_out=int(d_reward),
                      is_alarm_illegal=int(d_illegal))
        self._check(self.lib.b200pf_alarm_bind(self.h, C.byref(d)), "b200pf_alarm_bind")
        self._alarm_shape = (int(a.n), int(a.ring))

    def _alarm_spec(self):
        B = self._series_batch
        n, R = getattr(self, "_alarm_shape", (0, 0))                        # (unbound: the library refuses the call)
        shapes = dict(last=(B, n), last_ok=(B, n), ring_step=(B, R), ring_mask=(B, R))
        return tuple((k, dt, shapes.get(k, (B,))) for k, dt in ALARM_STATE)

    def alarm_get_state(self):
        """-> the alarm state of every instance, the arrays of :data:`grid2op_b200.alarm.ALARM_STATE`"""
        return self._get_state("b200pf_alarm_get_state", self._alarm_spec())

    def alarm_set_state(self, s: dict):
        self._set_state("b200pf_alarm_set_state", self._alarm_spec(), s)

    def observe_device(self, d_obs: int, d_reward: int = 0):
        self._check(self.lib.b200pf_observe_device(self.h, C.c_void_p(d_obs), C.c_void_p(d_reward or None)), "b200pf_observe_device")

    def env_stats(self):
        v = (C.c_int64 * 8)()
        self._check(self.lib.b200pf_env_stats(self.h, v), "b200pf_env_stats")
        return dict(steps=int(v[0]), h2d_bytes=int(v[1]), d2h_bytes=int(v[2]), host_waits=int(v[3]), n_illegal=int(v[4]),
                    nb_cap=int(v[5]), n_dirty=int(v[6]), plan_refreshes=int(v[7]))

    def sync(self):
        self._check(self.lib.b200pf_sync(self.h), "b200pf_sync")

    @property
    def stream(self) -> int:
        return int(self.lib.b200pf_stream(self.h))

    @property
    def launch_count(self) -> int:
        return int(self.lib.b200pf_launch_count(self.h))

    def last_launch_info(self):
        """Launch configuration of the last planned / pivoting launch.  ``config``: its kernel's template parameters
        (``b200pf_last_launch_config``) — block kernel (T, U, MINB, PROT, WPC, STAGE, UNI, MODE), scalar planned kernel
        (T, -1, MINB, PROT, -1, ...), pivoting kernels all -1."""
        v = [C.c_int() for _ in range(4)]
        self.lib.b200pf_last_launch_info(self.h, *[C.byref(x) for x in v])
        cfg = (C.c_int * 8)()
        self._check(self.lib.b200pf_last_launch_config(self.h, cfg), "b200pf_last_launch_config")
        return dict(smem_bytes=v[0].value, threads_per_instance=v[1].value, grid=v[2].value, block=v[3].value,
                    config=tuple(int(x) for x in cfg))

    KERNEL_AUTO, KERNEL_PIVOTING, KERNEL_PLANNED = 0, 1, 2

    def set_kernel_policy(self, policy: int):
        """0: planned sparse kernel whenever it applies (default); 1: pivoting kernels only; 2: planned kernel
        even when a call has to build many new topology plans."""
        self._check(self.lib.b200pf_set_kernel_policy(self.h, int(policy)), "b200pf_set_kernel_policy")

    def set_debug(self, planned_div_mod: int = 0, redo_enabled: bool = True):
        """TEST knob (include/b200pf.h): make the planned kernel give up on every ``planned_div_mod``-th instance, and / or
        switch the pivoting re-solve off."""
        self._check(self.lib.b200pf_set_debug(self.h, int(planned_div_mod), int(bool(redo_enabled))), "b200pf_set_debug")

    @property
    def redo_launch_count(self) -> int:
        return int(self.lib.b200pf_redo_launch_count(self.h))

    def plan_stats(self):
        n, b, k = C.c_int64(), C.c_int64(), C.c_int()
        self._check(self.lib.b200pf_plan_stats(self.h, C.byref(n), C.byref(b), C.byref(k)), "b200pf_plan_stats")
        return dict(n_plans=n.value, plan_bytes=b.value, last_kernel={0: "none", 1: "warp_pivoting", 2: "cta_pivoting", 3: "planned_sparse", 4: "planned_block"}[k.value])

    def plan_counters(self):
        v = (C.c_int64 * 4)()
        self._check(self.lib.b200pf_plan_counters(self.h, v), "b200pf_plan_counters")
        return dict(lookups=int(v[0]), hits=int(v[1]), built=int(v[2]), cache_resets=int(v[3]))

    def view(self, out: np.ndarray) -> OutputView:
        return OutputView(self.gm, out)
