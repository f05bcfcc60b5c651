"""ctypes binding of ``libt2d_b200.so`` (C ABI: ``include/t2d_b200.h``).

The library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is no
CPU fallback: if the shared object is missing, loading fails loudly, and every compute entry
point needs a CUDA device.
"""

from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("T2D_B200_LIB", os.path.join(_HERE, "libt2d_b200.so"))   # override: A/B builds of the kernels


class T2DError(RuntimeError):
    """A C-ABI call returned a negative code; the message is ``t2d_last_error()``."""


class Config(C.Structure):
    _fields_ = [("interval_ms", C.c_int32), ("delta_t_ms", C.c_int32), ("max_step", C.c_int32),
                ("flags", C.c_int32)]


class TypeParamsC(C.Structure):
    _fields_ = [(n, C.c_float) for n in (
        "half_len", "half_wid", "radius", "lf", "lr", "steer_lo", "steer_hi", "speed_lo", "speed_hi",
        "accel_lo", "accel_hi", "mass", "mass_height", "mu", "I_z", "cf", "cr")] + [
        ("model", C.c_int32), ("shape", C.c_int32)] + [(n, C.c_float) for n in ("wheel_radius", "T_sb", "T_se", "I_yw")]


class MapTileC(C.Structure):
    """``t2d_map_tile``: the static objects and the boundary of one map (host pointers)."""
    _fields_ = [("segments", C.c_void_p), ("n_seg", C.c_int32), ("poly_start", C.c_void_p), ("n_poly", C.c_int32),
                ("bounds", C.c_void_p)]


class ControllerParamsC(C.Structure):
    """``t2d_controller_params``: one configured controller object."""
    _fields_ = [("kind", C.c_int32)] + [(n, C.c_float) for n in (
        "desired_speed", "time_headway", "min_spacing", "max_acceleration", "comfortable_deceleration", "delta",
        "target_speed", "kp", "accel_change_rate", "delta_t", "max_accel", "min_accel", "interval",
        "min_pre_aiming_distance", "pp_interval", "wheel_base")] + [
        ("pid_lateral", C.c_int32), ("pid_longitudinal", C.c_int32)] + [(n, C.c_double) for n in (
        "dt", "kp_lat", "ki_lat", "kd_lat", "max_steering", "kp_lon", "ki_lon", "kd_lon", "derivative_filter_alpha")]


class LaneChangeParamsC(C.Structure):
    """``t2d_lane_change_params``: the MOBIL parameters of a bound lane change."""
    _fields_ = [(n, C.c_double) for n in ("politeness", "threshold", "b_safe", "min_gap")] + [
        ("cooldown", C.c_int32), ("reserved", C.c_int32)]


class YieldParamsC(C.Structure):
    """``t2d_yield_params``: the gap-acceptance parameters of a bound yielding."""
    _fields_ = [(n, C.c_double) for n in ("critical_gap", "commit_decel", "v_min")]


ZONE_DTYPE = [("q", "<i4"), ("reserved", "<i4"), ("s_in_p", "<f8"), ("s_out_p", "<f8"), ("s_in_q", "<f8"),
              ("s_out_q", "<f8")]   # t2d_conflict_zone


class BevStyleC(C.Structure):
    """``t2d_bev_style``: colour, z order and stroke width (points) of one BEV style row."""
    _fields_ = [("r", C.c_uint8), ("g", C.c_uint8), ("b", C.c_uint8), ("z", C.c_int8), ("line_width_pt", C.c_float)]


class LogC(C.Structure):
    """``t2d_log``: a recording's tracks and episode rows (host pointers) + the log_row / type_id device arrays."""
    _fields_ = [("n_tracks", C.c_int32), ("first_ms", C.c_void_p), ("n_frames", C.c_void_p), ("period_ms", C.c_void_p),
                ("type_row", C.c_void_p), ("records", C.c_void_p), ("n_rows", C.c_int32), ("t0_ms", C.c_void_p),
                ("row_track", C.c_void_p), ("log_row", C.c_void_p), ("type_id", C.c_void_p)]


class ReactiveReplayC(C.Structure):
    """``t2d_reactive_replay``: the per-track tables (host pointers) and the per-slot device arrays of a reactive replay."""
    _fields_ = [("n_tracks", C.c_int32), ("track_path", C.c_void_p), ("drive_row", C.c_void_p),
                ("desired_speed", C.c_void_p), ("drive_path", C.c_void_p), ("slot_desired_speed", C.c_void_p)]


class ResetSamplerC(C.Structure):
    """``t2d_reset_sampler``: the seed and options of the sampled resets, the host jitter table, the device row pools and
    the world-owned episode / pool_row / reset_try buffers."""
    _fields_ = [("seed", C.c_uint64), ("sample_rows", C.c_int32), ("tries", C.c_int32), ("avoid_target", C.c_int32),
                ("n_rows", C.c_int32), ("jitter", C.c_void_p), ("pool_type_id", C.c_void_p), ("pool_target", C.c_void_p),
                ("pool_tile_id", C.c_void_p), ("pool_route_id", C.c_void_p), ("episode", C.c_void_p),
                ("pool_row", C.c_void_p), ("reset_try", C.c_void_p)]


class ObsConfigC(C.Structure):
    """``t2d_obs_config``: rows and ranges of the vector observation."""
    _fields_ = [("k_agents", C.c_int32), ("k_segments", C.c_int32), ("agent_range", C.c_float), ("segment_range", C.c_float)]


class HistoryRingC(C.Structure):
    """``t2d_history_ring``: the device arrays of the bound trajectory-history ring."""
    _fields_ = [("length", C.c_int32)] + [(n, C.c_void_p) for n in (
        "x", "y", "heading", "speed", "vx", "vy", "type_id", "track", "count")]


# name -> (restype, argtypes); every symbol include/t2d_b200.h declares
_P = C.c_void_p
SYMBOLS = {
    "t2d_version": (C.c_int, []),
    "t2d_last_error": (C.c_char_p, []),
    "t2d_create": (C.c_int, [C.POINTER(_P), C.c_int, C.c_int, C.c_int, C.POINTER(Config)]),
    "t2d_destroy": (C.c_int, [_P]),
    "t2d_set_config": (C.c_int, [_P, C.POINTER(Config)]),
    "t2d_set_type_table": (C.c_int, [_P, C.POINTER(TypeParamsC), C.c_int]),
    "t2d_set_map": (C.c_int, [_P, _P, C.c_int, _P, C.c_float]),
    "t2d_set_map_polygons": (C.c_int, [_P, _P, C.c_int, _P, C.c_int, _P, C.c_float]),
    "t2d_set_map_table": (C.c_int, [_P, _P, C.c_int, _P, C.c_float]),
    "t2d_bind_state": (C.c_int, [_P] + [_P] * 8),
    "t2d_step": (C.c_int, [_P] + [_P] * 7),
    "t2d_step_host": (C.c_int, [_P] + [_P] * 7),
    "t2d_check_events": (C.c_int, [_P] + [_P] * 4),
    "t2d_set_ego_action": (C.c_int, [_P, _P]),
    "t2d_step_host_ego": (C.c_int, [_P] + [_P] * 8),
    "t2d_env_epilogue": (C.c_int, [_P] + [_P] * 9 + [C.c_int, _P]),
    "t2d_set_goal": (C.c_int, [_P, _P, C.c_float, C.c_int, _P, _P, _P]),
    "t2d_set_agents": (C.c_int, [_P, _P, C.c_int32, _P, C.c_float, C.c_int, _P, _P, _P]),
    "t2d_agents_epilogue": (C.c_int, [_P] + [_P] * 10 + [C.c_int, _P]),
    "t2d_scatter_agent_action": (C.c_int, [_P, _P, C.c_int32, _P, _P, _P]),
    "t2d_step_host_agents": (C.c_int, [_P] + [_P] * 7 + [C.c_int] + [_P] * 6),
    "t2d_reset": (C.c_int, [_P, _P, _P, C.c_int] + [_P] * 7),
    "t2d_set_reset_sampler": (C.c_int, [_P, C.POINTER(ResetSamplerC)]),
    "t2d_reset_sampled": (C.c_int, [_P, _P, C.c_int] + [_P] * 7),
    "t2d_lidar_scan": (C.c_int, [_P, C.c_int, C.c_float, _P, _P, _P]),
    "t2d_lidar_scan_agents": (C.c_int, [_P, _P, C.c_int32, C.c_int, C.c_float, _P, _P, _P]),
    "t2d_set_bev_styles": (C.c_int, [_P, _P, C.c_int, _P, _P, C.c_int, C.c_int]),
    "t2d_bev_render": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int, _P, _P]),
    "t2d_bev_render_agents": (C.c_int, [_P, _P, C.c_int32, _P, C.c_int, C.c_int, _P, C.c_int, _P, _P]),
    "t2d_observe": (C.c_int, [_P, C.POINTER(ObsConfigC), _P, _P, _P, _P]),
    "t2d_observe_agents": (C.c_int, [_P, C.POINTER(ObsConfigC), _P, C.c_int32, _P, _P, _P, _P, _P]),
    "t2d_set_controllers": (C.c_int, [_P, _P, C.c_int, _P, _P, _P, _P]),
    "t2d_set_paths": (C.c_int, [_P, _P, _P, C.c_int]),
    "t2d_control": (C.c_int, [_P, _P, _P]),
    "t2d_set_pid": (C.c_int, [_P, _P, _P]),
    "t2d_set_leader_search": (C.c_int, [_P, C.c_double, C.c_double, _P, _P]),
    "t2d_find_leaders": (C.c_int, [_P, C.c_double, C.c_double, _P, _P, _P]),
    "t2d_set_lane_change": (C.c_int, [_P, _P, _P, _P, _P, _P, _P]),
    "t2d_set_yielding": (C.c_int, [_P, _P, _P, _P, _P, _P, _P]),
    "t2d_find_yields": (C.c_int, [_P, _P, _P, _P]),
    "t2d_set_routes": (C.c_int, [_P, _P, C.c_double, C.c_double, C.c_float]),
    "t2d_bind_route_trackers": (C.c_int, [_P, _P, _P, C.c_int32]),
    "t2d_route_observe": (C.c_int, [_P, _P, C.c_int32, C.c_int, C.c_float, _P, _P]),
    "t2d_set_history": (C.c_int, [_P, C.c_int32]),
    "t2d_observe_history": (C.c_int, [_P, _P, C.c_int32, _P, C.c_int32, _P, _P]),
    "t2d_history_view": (C.c_int, [_P, C.POINTER(HistoryRingC)]),
    "t2d_exchange_create": (C.c_int, [C.POINTER(_P), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "t2d_exchange_connect": (C.c_int, [_P, _P]),
    "t2d_exchange_allgather": (C.c_int, [_P, _P, _P, _P]),
    "t2d_exchange_allgather_lagged": (C.c_int, [_P, _P, _P, C.c_int, _P]),
    "t2d_exchange_status": (C.c_int, [_P, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "t2d_exchange_destroy": (C.c_int, [_P]),
    "t2d_physics_step": (C.c_int, [C.c_int, C.POINTER(TypeParamsC), C.c_int, C.c_int, C.c_int] + [_P] * 11),
    "t2d_bind_wheel_state": (C.c_int, [_P, _P, _P]),
    "t2d_bind_reset_wheel_pool": (C.c_int, [_P, _P, _P]),
    "t2d_set_log": (C.c_int, [_P, C.POINTER(LogC)]),
    "t2d_set_log_schedule": (C.c_int, [_P, C.POINTER(LogC), _P, _P, C.c_int32, _P]),
    "t2d_set_log_reactive": (C.c_int, [_P, C.POINTER(ReactiveReplayC)]),
    "t2d_set_prefetch": (C.c_int, [_P, C.c_int]),
    "t2d_launch_count": (C.c_int64, []),
    "t2d_tick_fixed_count": (C.c_int64, []),
    "t2d_tick_order_fallback_count": (C.c_int64, []),
    "t2d_order_hint": (C.c_int, [_P, _P, _P]),
    "t2d_tick_instance_count": (C.c_int64, [C.c_int]),
}

_lib = None


def load():
    """Load the shared library (once) and declare its prototypes."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc -gencode arch=compute_90a,code=sm_90a).  tactics2d_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(code: int):
    if code != 0:
        msg = load().t2d_last_error()
        raise T2DError(f"t2d error {code}: {msg.decode() if msg else ''}")
