"""The PIDController golden sequences (tests/golden/controllers_pid.npz, tests/make_pid_golden.py) as rows of
the batched controller table."""

import json
import os

import numpy as np

from . import pid_oracle as OC

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "controllers_pid.npz"))
CONFIGS = json.loads(str(G["configs"]))
GAINS = ("dt", "kp_lat", "ki_lat", "kd_lat", "max_steering", "kp_lon", "ki_lon", "kd_lon", "max_accel", "min_accel",
         "derivative_filter_alpha")


def sources(cfg):
    """(pid_lateral, pid_longitudinal) the keywords of a sequence select."""
    lat = {"heading": OC.PID_LAT_HEADING, "cross": OC.PID_LAT_CROSS_TRACK, None: OC.PID_LAT_NONE}[cfg["lateral"]]
    if cfg["control_mode"] == "longitudinal":
        lat = OC.PID_LAT_NONE
    lon = OC.PID_LON_TARGET if cfg["target_speed"] and cfg["control_mode"] != "lateral" else OC.PID_LON_NONE
    return lat, lon


def quirk(cfg):
    """wheel_base <= 0 with a cross-track error: the lateral state advances, the steering is 0 (pid_controller.py:357)."""
    return cfg["lateral"] == "cross" and cfg["wheel_base"] is not None and cfg["wheel_base"] <= 0


def row_dict(cfg):
    """The row as float64 values (the reference's own attributes), for the oracle."""
    lat, lon = sources(cfg)
    wb = cfg["wheel_base"] if cfg["wheel_base"] is not None and cfg["wheel_base"] > 0 else 2.637
    return dict({k: cfg[k] for k in GAINS}, kind=OC.PID, pid_lateral=lat, pid_longitudinal=lon, wheel_base=wb)


def row_c(cfg):
    """The same row as a t2d_controller_params (max_accel, min_accel and wheel_base become fp32)."""
    from tactics2d_b200 import _lib

    return _lib.ControllerParamsC(**{k: v for k, v in row_dict(cfg).items()})


def sequence(cfg):
    """inputs [T, 6] = (x, y, heading, speed, target_speed, lateral target), outputs [T, 2], state [T, 6]."""
    n = cfg["name"]
    return G[f"{n}_inputs"], G[f"{n}_outputs"], G[f"{n}_state"]
