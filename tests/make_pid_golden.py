"""Write tests/golden/controllers_pid.npz from the UNMODIFIED reference's ``PIDController``.

TEST INFRASTRUCTURE ONLY.  Run where a checkout of the reference (WoodOxen/tactics2d @ d7095aa) exists:

    T2D_REFERENCE=<reference checkout> python tests/make_pid_golden.py

``tactics2d.controller`` imports ``shapely.geometry`` (pure_pursuit_controller.py:8); the generator installs the same
stand-in ``oracle/make_golden.py`` uses for ``controllers.npz``, which ``PIDController`` and ``State`` never call.  It has
its own seeded generator and touches no other fixture.
"""

from __future__ import annotations

import os
import sys

import numpy as np

REF = os.environ.get("T2D_REFERENCE")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# PIDController sequences: (name, constructor keywords, driving style, lateral keyword, wheel_base keyword, target_speed
# given, kind of targets).  lateral keyword: "heading" / "cross" / None (missing); wheel_base None: not passed.
PID_SEQUENCES = [
    ("default", dict(), None, "heading", None, True, "plain"),
    ("gains", dict(dt=0.1, kp_lat=2.0, ki_lat=0.1, kd_lat=0.3, max_steering=0.4, kp_lon=1.5, ki_lon=0.2, kd_lon=0.5,
                   max_accel=2.5, min_accel=-4.0, derivative_filter_alpha=0.2), None, "heading", None, True, "plain"),
    ("alpha_one", dict(dt=0.02, derivative_filter_alpha=1.0, ki_lat=0.7, kd_lon=0.05), None, "cross", 2.5, True, "plain"),
    ("lateral_heading", dict(control_mode="lateral"), None, "heading", None, False, "plain"),
    ("lateral_cross", dict(control_mode="lateral", kd_lat=0.2), None, "cross", 2.637, False, "plain"),
    ("longitudinal", dict(control_mode="longitudinal", ki_lon=0.8), None, None, None, True, "plain"),
    ("cross_default_wb", dict(), None, "cross", None, True, "plain"),
    ("wrap", dict(kd_lat=0.05), None, "heading", None, True, "wrap"),
    ("saturation", dict(ki_lon=1.5), None, "heading", None, True, "saturate"),
    ("no_lateral", dict(), None, None, None, True, "plain"),
    ("no_longitudinal", dict(), None, "heading", None, False, "plain"),
    ("wheel_base_quirk", dict(), None, "cross", -1.0, True, "plain"),
    ("style_conservative", dict(), -1.0, "heading", None, True, "saturate"),
    ("style_0_3", dict(), 0.3, "heading", None, True, "saturate"),
    ("style_aggressive", dict(), 1.0, "cross", 2.5, True, "saturate"),
]


def pid_golden(rng=None, T=40):
    """PIDController (pid_controller.py) sequences of the unmodified reference: per sequence the step inputs, the
    (steering, acceleration) of every step and the six state values after it.  Inputs are fp32-representable.  Every
    saturation decision of the longitudinal channel clears its limit (and the fp32 rounding of the limit, which is what a
    batched row holds) by more than 1e-9 relative, so an ulp of libm cannot flip a branch."""
    import json

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    from oracle.make_golden import _shapely_stand_in

    _shapely_stand_in()
    from tactics2d.controller.pid_controller import PIDController
    from tactics2d.participant.trajectory.state import State

    rng = np.random.default_rng(20261017) if rng is None else rng
    f32 = lambda a: np.asarray(a, np.float32).astype(np.float64)
    out, cfgs = {}, []
    for name, kw, style, lat_kw, wb, lon_kw, targets in PID_SEQUENCES:
        c = PIDController(**kw)
        if style is not None:
            c.update_driving_style(style)
        heading = f32(np.cumsum(rng.uniform(-0.3, 0.3, T)) + rng.uniform(-3, 3))
        speed = f32(np.clip(rng.uniform(2, 15) + np.cumsum(rng.uniform(-1, 1, T)), 0, 30))
        tspeed = f32(np.repeat(rng.uniform(0, 20, T // 8 + 1), 8)[:T])
        if targets == "saturate":   # far above and far below the speed: both limits, then the leaky integral
            tspeed = f32(np.where((np.arange(T) // 10) % 2 == 0, speed + rng.uniform(8, 20, T), speed - rng.uniform(8, 20, T)))
        if lat_kw == "cross":
            lat_t = f32(np.cumsum(rng.uniform(-0.4, 0.4, T)) + rng.uniform(-2, 2))
        else:
            lat_t = f32(heading + rng.uniform(-0.6, 0.6, T))
            if targets == "wrap":   # heading errors beyond +-pi in both directions
                lat_t = f32(heading + rng.choice([-1.0, 1.0], T) * rng.uniform(np.pi + 0.05, 3 * np.pi, T))
        xy = f32(rng.uniform(-50, 50, (T, 2)))
        res, states = np.zeros((T, 2)), np.zeros((T, 6))
        for t in range(T):
            kwargs = {}
            if lat_kw == "heading":
                kwargs["target_heading"] = float(lat_t[t])
            elif lat_kw == "cross":
                kwargs["cross_track_error"] = float(lat_t[t])
            if wb is not None:
                kwargs["wheel_base"] = wb
            if lon_kw:
                kwargs["target_speed"] = float(tspeed[t])
            ego = State(frame=0, x=float(xy[t, 0]), y=float(xy[t, 1]), heading=float(heading[t]), speed=float(speed[t]))
            steer, acc = c.step(ego, **kwargs)
            res[t] = (float(steer), float(acc))
            states[t] = (c._lat_integral, c._lat_prev_error, c._lat_prev_derivative, c._lon_integral, c._lon_prev_error,
                         c._lon_prev_derivative)
            if lon_kw and c.control_mode != "lateral":
                out0 = c.kp_lon * states[t, 4] + c.kd_lon * states[t, 5]
                for lim in (c.max_accel, c.min_accel, float(np.float32(c.max_accel)), float(np.float32(c.min_accel))):
                    assert abs(out0 - lim) > 1e-9 * max(1.0, abs(lim)), (name, t, out0, lim)
        out[f"{name}_inputs"] = np.stack([xy[:, 0], xy[:, 1], heading, speed, tspeed, lat_t], 1)
        out[f"{name}_outputs"] = res
        out[f"{name}_state"] = states
        cfgs.append(dict(name=name, control_mode=c.control_mode, dt=c.dt, kp_lat=c.kp_lat, ki_lat=c.ki_lat,
                         kd_lat=c.kd_lat, max_steering=c.max_steering, kp_lon=c.kp_lon, ki_lon=c.ki_lon, kd_lon=c.kd_lon,
                         max_accel=c.max_accel, min_accel=c.min_accel,
                         derivative_filter_alpha=c._derivative_filter_alpha, style=style, lateral=lat_kw,
                         wheel_base=wb, target_speed=lon_kw))
    out["configs"] = np.array(json.dumps(cfgs))
    np.savez(os.path.join(OUT, "controllers_pid.npz"), **out)


if __name__ == "__main__":
    if not REF or not os.path.isdir(os.path.join(REF, "tactics2d")):
        sys.exit("set T2D_REFERENCE to a checkout of the reference (the directory that holds tactics2d/)")
    sys.path.insert(0, REF)
    pid_golden()
    print("golden vectors written to", os.path.normpath(os.path.join(OUT, "controllers_pid.npz")))
