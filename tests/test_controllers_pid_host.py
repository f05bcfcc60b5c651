"""PIDController on the host: the reference's initialisation / driving-style / configure assertions
(tests/test_controllers.py TestPIDController), the t2d_controller_params row it produces, and the row's C layout."""

import ctypes as C

import pytest

from tactics2d_b200 import _lib
from tactics2d_b200.controller import CTRL_PID, PIDController
from tactics2d_b200.controller.controller_base import (PID_LAT_CROSS_TRACK, PID_LAT_HEADING, PID_LAT_NONE,
                                                       PID_LAT_PATH_CROSS_TRACK, PID_LAT_PATH_HEADING, PID_LON_NONE,
                                                       PID_LON_TARGET)


def test_initialization():
    c = PIDController()
    assert (c.dt, c.control_mode, c.kp_lat, c.ki_lat, c.kd_lat, c.max_steering) == (0.05, "combined", 1.5, 0.2, 0.5, 0.5)
    assert (c.kp_lon, c.ki_lon, c.kd_lon, c.max_accel, c.min_accel) == (2.0, 0.3, 0.4, 3.0, -5.0)
    assert c._derivative_filter_alpha == 0.1 and c.lateral_error == "target_heading"
    c = PIDController(dt=0.1, control_mode="lateral", kp_lat=2.0, ki_lat=0.1, kd_lat=0.3, max_steering=0.4, kp_lon=1.5,
                      ki_lon=0.2, kd_lon=0.5, max_accel=2.5, min_accel=-4.0, derivative_filter_alpha=0.2)
    assert (c.dt, c.control_mode, c.kp_lat, c.max_steering, c._derivative_filter_alpha) == (0.1, "lateral", 2.0, 0.4, 0.2)
    with pytest.raises(ValueError, match="control_mode must be one of"):
        PIDController(control_mode="invalid")
    with pytest.raises(ValueError, match="dt must be positive"):
        PIDController(dt=0)
    with pytest.raises(ValueError, match="max_steering must be positive"):
        PIDController(max_steering=0)
    with pytest.raises(ValueError, match="max_accel must be positive"):
        PIDController(max_accel=0)
    with pytest.raises(ValueError, match=r"min_accel must be negative \(deceleration\), got 0.5"):
        PIDController(min_accel=0.5)
    with pytest.raises(ValueError, match=r"derivative_filter_alpha must be in range \(0, 1\], got 1.5"):
        PIDController(derivative_filter_alpha=1.5)
    with pytest.raises(ValueError, match="lateral_error must be one of"):
        PIDController(lateral_error="lane")
    # a fresh controller reads its state without a device
    assert (c._lat_integral, c._lat_prev_error, c._lat_prev_derivative, c._lon_integral, c._lon_prev_error,
            c._lon_prev_derivative) == (0.0,) * 6


def test_update_driving_style():
    c = PIDController()
    c.update_driving_style(-1.0)
    assert (c.kp_lat, c.kp_lon, c.max_steering, c.max_accel, c.min_accel) == (1.0, 1.5, 0.4, 2.5, -4.0)
    c.update_driving_style(1.0)
    assert (c.kp_lat, c.kp_lon, c.max_steering, c.max_accel, c.min_accel) == (2.0, 2.5, 0.6, 3.5, -6.0)
    with pytest.raises(TypeError, match="style_id must be int or float"):
        c.update_driving_style("fast")


def test_configure():
    c = PIDController()
    c.configure(kp_lat=3.0, max_steering=0.4)
    assert (c.kp_lat, c.max_steering) == (3.0, 0.4)
    c.configure(derivative_filter_alpha=0.3)
    assert c._derivative_filter_alpha == 0.3
    with pytest.raises(AttributeError, match="has no parameter"):
        c.configure(invalid_param=1.0)
    with pytest.raises(ValueError, match="dt must be positive"):
        c.configure(dt=-0.1)
    # every key is checked before any is applied
    with pytest.raises(ValueError, match="max_steering must be positive"):
        c.configure(kp_lon=9.0, max_steering=-1.0)
    assert c.kp_lon == 2.0
    with pytest.raises(ValueError, match=r"max_accel \(1.0\) must be greater than min_accel \(2.0\)|min_accel must be"):
        c.configure(max_accel=1.0, min_accel=2.0)
    with pytest.raises(ValueError, match="control_mode must be 'combined', 'lateral', or 'longitudinal'"):
        c.configure(control_mode="both")
    with pytest.raises(ValueError, match="lateral_error must be one of"):
        c.configure(lateral_error="lane")
    c.configure(lateral_error="path_cross_track", control_mode="lateral")
    assert c.params().pid_lateral == PID_LAT_PATH_CROSS_TRACK and c.params().pid_longitudinal == PID_LON_NONE


LAT = {"target_heading": PID_LAT_HEADING, "cross_track_error": PID_LAT_CROSS_TRACK, "path_heading": PID_LAT_PATH_HEADING,
       "path_cross_track": PID_LAT_PATH_CROSS_TRACK}


@pytest.mark.parametrize("mode", ["combined", "lateral", "longitudinal"])
@pytest.mark.parametrize("lateral_error", sorted(LAT))
def test_params_row(mode, lateral_error):
    c = PIDController(control_mode=mode, lateral_error=lateral_error, dt=0.02, kp_lat=1.25, ki_lat=0.3, kd_lat=0.7,
                      max_steering=0.45, kp_lon=1.75, ki_lon=0.35, kd_lon=0.15, max_accel=2.75, min_accel=-4.5,
                      derivative_filter_alpha=0.6)
    r = c.params()
    assert r.kind == CTRL_PID
    assert r.pid_lateral == (PID_LAT_NONE if mode == "longitudinal" else LAT[lateral_error])
    assert r.pid_longitudinal == (PID_LON_NONE if mode == "lateral" else PID_LON_TARGET)
    assert (r.dt, r.kp_lat, r.ki_lat, r.kd_lat, r.max_steering) == (0.02, 1.25, 0.3, 0.7, 0.45)   # doubles: exact
    assert (r.kp_lon, r.ki_lon, r.kd_lon, r.derivative_filter_alpha) == (1.75, 0.35, 0.15, 0.6)
    assert (r.max_accel, r.min_accel) == (2.75, -4.5)
    assert r.wheel_base == pytest.approx(2.637, rel=1e-7)


def test_row_layout():
    """t2d_controller_params: the old fields where they were, then two int32 sources and nine doubles (4 bytes of padding
    before dt)."""
    R = _lib.ControllerParamsC
    assert R.kind.offset == 0 and R.desired_speed.offset == 4 and R.wheel_base.offset == 64
    assert R.pid_lateral.offset == 68 and R.pid_longitudinal.offset == 72
    names = ("dt", "kp_lat", "ki_lat", "kd_lat", "max_steering", "kp_lon", "ki_lon", "kd_lon", "derivative_filter_alpha")
    assert [getattr(R, n).offset for n in names] == [80 + 8 * i for i in range(9)]
    assert all(getattr(R, n).size == 8 for n in names)
    assert C.sizeof(R) == 152 and C.alignment(R) == 8
    assert _lib.SYMBOLS["t2d_set_pid"] == (C.c_int, [C.c_void_p] * 3)
