"""``PIDController`` (tactics2d/controller/pid_controller.py:15-470): PID steering and acceleration with an integral, the
previous error and a low-pass-filtered derivative per channel.

The constructor, attributes, ``update_driving_style``, ``configure`` and ``reset`` are the reference's, with the same
checks and messages.  The controller memory lives on the device: ``step`` runs ``t2d_control`` on a 1 x 2 world and
keeps the state between calls; ``_lat_integral`` ... ``_lon_prev_derivative`` read it back.

``lateral_error`` is the one attribute the reference lacks.  It chooses where a batched row (``params()``, handed to
``BatchedWorld.set_controllers``) takes its lateral error from: ``"target_heading"`` / ``"cross_track_error"`` read
column 1 of ``pid_target``, ``"path_heading"`` / ``"path_cross_track"`` derive it from the slot's ``path_id`` polyline
(DESIGN.md section 1, "PID controller").  ``step`` picks its sources from the keywords it is given, as the reference
does.  A row takes the reference's default wheel base, 2.637 m; set ``row.wheel_base`` on the row ``params()`` returns
for another one.
"""

from __future__ import annotations

import numpy as np

from .. import _lib
from .controller_base import (CTRL_PID, NO_CONTROLLER, PID_LAT_CROSS_TRACK, PID_LAT_HEADING, PID_LAT_NONE,
                              PID_LAT_PATH_CROSS_TRACK, PID_LAT_PATH_HEADING, PID_LON_NONE, PID_LON_TARGET,
                              ControllerBase)

LATERAL_ERRORS = {"target_heading": PID_LAT_HEADING, "cross_track_error": PID_LAT_CROSS_TRACK,
                  "path_heading": PID_LAT_PATH_HEADING, "path_cross_track": PID_LAT_PATH_CROSS_TRACK}
DEFAULT_WHEEL_BASE = 2.637   # pid_controller.py:356
_STATE_NAMES = ("_lat_integral", "_lat_prev_error", "_lat_prev_derivative", "_lon_integral", "_lon_prev_error",
                "_lon_prev_derivative")


def _state_property(k):
    def get(self):
        return float(self._state[0, 0, k]) if self._state is not None else float(self._pending[k])

    def set_(self, value):
        if self._state is not None:
            self._state[0, 0, k] = float(value)
        else:
            self._pending[k] = float(value)

    return property(get, set_)


class PIDController(ControllerBase):
    def __init__(self, dt: float = 0.05, control_mode: str = "combined", kp_lat: float = 1.5, ki_lat: float = 0.2,
                 kd_lat: float = 0.5, max_steering: float = 0.5, kp_lon: float = 2.0, ki_lon: float = 0.3,
                 kd_lon: float = 0.4, max_accel: float = 3.0, min_accel: float = -5.0,
                 derivative_filter_alpha: float = 0.1, lateral_error: str = "target_heading"):
        valid_modes = {"combined", "lateral", "longitudinal"}
        if control_mode not in valid_modes:
            raise ValueError(f"control_mode must be one of {valid_modes}, got '{control_mode}'")
        if dt <= 0:
            raise ValueError(f"dt must be positive, got {dt}")
        if max_steering <= 0:
            raise ValueError(f"max_steering must be positive, got {max_steering}")
        if max_accel <= 0:
            raise ValueError(f"max_accel must be positive, got {max_accel}")
        if min_accel >= 0:
            raise ValueError(f"min_accel must be negative (deceleration), got {min_accel}")
        if max_accel <= min_accel:
            raise ValueError(f"max_accel ({max_accel}) must be greater than min_accel ({min_accel})")
        if derivative_filter_alpha <= 0 or derivative_filter_alpha > 1:
            raise ValueError(f"derivative_filter_alpha must be in range (0, 1], got {derivative_filter_alpha}")
        _check_lateral_error(lateral_error)

        self.dt = dt
        self.control_mode = control_mode
        self.kp_lat = kp_lat
        self.ki_lat = ki_lat
        self.kd_lat = kd_lat
        self.max_steering = max_steering
        self.kp_lon = kp_lon
        self.ki_lon = ki_lon
        self.kd_lon = kd_lon
        self.max_accel = max_accel
        self.min_accel = min_accel
        self._derivative_filter_alpha = derivative_filter_alpha
        self.lateral_error = lateral_error

        self._kp_lat_interpolator = self.create_style_interpolator(1.0, 2.0)
        self._kp_lon_interpolator = self.create_style_interpolator(1.5, 2.5)
        self._max_steering_interpolator = self.create_style_interpolator(0.4, 0.6)
        self._max_accel_interpolator = self.create_style_interpolator(2.5, 3.5)
        self._min_accel_interpolator = self.create_style_interpolator(-4.0, -6.0)

        self._state = None             # fp64 [1, 2, 6] device tensor, created by the first step
        self._pending = np.zeros(6)    # the state until then

    _lat_integral = _state_property(0)
    _lat_prev_error = _state_property(1)
    _lat_prev_derivative = _state_property(2)
    _lon_integral = _state_property(3)
    _lon_prev_error = _state_property(4)
    _lon_prev_derivative = _state_property(5)

    def update_driving_style(self, style_id: float) -> None:
        if not isinstance(style_id, (int, float)):
            raise TypeError("style_id must be int or float")
        self.kp_lat = float(self._kp_lat_interpolator(style_id))
        self.kp_lon = float(self._kp_lon_interpolator(style_id))
        self.max_steering = float(self._max_steering_interpolator(style_id))
        self.max_accel = float(self._max_accel_interpolator(style_id))
        self.min_accel = float(self._min_accel_interpolator(style_id))

    def reset(self) -> None:
        """Clear the integrals, previous errors and derivatives (pid_controller.py:408-418)."""
        if self._state is not None:
            self._state.zero_()
        self._pending[:] = 0.0

    def configure(self, **kwargs) -> None:
        """pid_controller.py:420-470: every key is validated before any is applied."""
        param_map = {"derivative_filter_alpha": "_derivative_filter_alpha"}
        for key, value in kwargs.items():
            internal_key = param_map.get(key, key)
            if not hasattr(self, internal_key):
                raise AttributeError(f"PIDController has no parameter '{key}'")
            if key == "dt" and value <= 0:
                raise ValueError(f"dt must be positive, got {value}")
            elif key == "control_mode" and value not in {"combined", "lateral", "longitudinal"}:
                raise ValueError(f"control_mode must be 'combined', 'lateral', or 'longitudinal', got '{value}'")
            elif key == "max_steering" and value <= 0:
                raise ValueError(f"max_steering must be positive, got {value}")
            elif key == "max_accel" and value <= 0:
                raise ValueError(f"max_accel must be positive, got {value}")
            elif key == "min_accel" and value >= 0:
                raise ValueError(f"min_accel must be negative (deceleration), got {value}")
            elif key == "derivative_filter_alpha" and (value <= 0 or value > 1):
                raise ValueError(f"derivative_filter_alpha must be in range (0, 1], got {value}")
            elif key == "lateral_error":
                _check_lateral_error(value)
        if "max_accel" in kwargs and "min_accel" in kwargs:
            max_val = kwargs["max_accel"]
            min_val = kwargs["min_accel"]
            if max_val <= min_val:
                raise ValueError(f"max_accel ({max_val}) must be greater than min_accel ({min_val})")
        for key, value in kwargs.items():
            setattr(self, param_map.get(key, key), value)

    # ------------------------------------------------------------------ batched path
    def params(self, lateral=None, longitudinal=None) -> "_lib.ControllerParamsC":
        """This controller as one ``t2d_controller_params`` row: ``control_mode`` and ``lateral_error`` give the two
        sources (``lateral`` / ``longitudinal`` override them with ``PID_LAT_*`` / ``PID_LON_*`` codes)."""
        if lateral is None:
            lateral = PID_LAT_NONE if self.control_mode == "longitudinal" else LATERAL_ERRORS[self.lateral_error]
        if longitudinal is None:
            longitudinal = PID_LON_NONE if self.control_mode == "lateral" else PID_LON_TARGET
        return _lib.ControllerParamsC(
            kind=CTRL_PID, max_accel=float(self.max_accel), min_accel=float(self.min_accel), wheel_base=DEFAULT_WHEEL_BASE,
            pid_lateral=int(lateral), pid_longitudinal=int(longitudinal), dt=float(self.dt), kp_lat=float(self.kp_lat),
            ki_lat=float(self.ki_lat), kd_lat=float(self.kd_lat), max_steering=float(self.max_steering),
            kp_lon=float(self.kp_lon), ki_lon=float(self.ki_lon), kd_lon=float(self.kd_lon),
            derivative_filter_alpha=float(self._derivative_filter_alpha))

    def step(self, ego_state, **kwargs):
        """``(steering, acceleration)`` (pid_controller.py:309-406), evaluated by ``t2d_control``.

        Raises where the reference raises.  In ``"combined"`` mode a channel whose keyword is missing or not numeric
        gives 0 and keeps its state; a ``wheel_base <= 0`` there still advances the lateral state and gives steering 0,
        as in the reference.  The keyword values go to the device as fp32."""
        mode = self.control_mode
        lat, lat_target, wheel_base, wheel_base_error = PID_LAT_NONE, 0.0, DEFAULT_WHEEL_BASE, None
        if mode in ("combined", "lateral"):
            try:
                lat, lat_target = _lateral_source(kwargs)
            except (ValueError, TypeError):
                if mode == "lateral":
                    raise
                lat = PID_LAT_NONE
            if lat != PID_LAT_NONE and "cross_track_error" in kwargs:
                wb = kwargs.get("wheel_base", DEFAULT_WHEEL_BASE)
                try:
                    if wb <= 0:
                        raise ValueError(f"wheel_base must be positive, got {wb}")
                    wheel_base = wb
                except (ValueError, TypeError) as e:
                    wheel_base_error = e      # raised (or turned into steering 0) after the state has advanced
        lon, target_speed = PID_LON_NONE, 0.0
        if mode in ("combined", "longitudinal"):
            try:
                if "target_speed" not in kwargs:
                    raise ValueError("Longitudinal control requires 'target_speed' in kwargs")
                target_speed = kwargs["target_speed"]
                if not isinstance(target_speed, (int, float)):
                    raise TypeError("target_speed must be numeric")
                lon = PID_LON_TARGET
            except (ValueError, TypeError):
                if mode == "longitudinal":
                    raise
                lon = PID_LON_NONE
        if lat == PID_LAT_NONE and lon == PID_LON_NONE:
            return 0.0, 0.0

        # a heading error with "cross_track_error" also given takes the cross-track scaling (:355-362): the device runs
        # the heading row, and the steering is rebuilt from the state it leaves
        rescale = lat == PID_LAT_HEADING and "cross_track_error" in kwargs
        row = self.params(lat, lon)
        row.wheel_base = float(wheel_base) if lat == PID_LAT_CROSS_TRACK and wheel_base_error is None else DEFAULT_WHEEL_BASE
        steer, accel = self._step_pid(ego_state, row, float(target_speed), float(lat_target))
        if wheel_base_error is not None:
            if mode == "lateral":
                raise wheel_base_error
            steer = 0.0
        elif rescale:
            integral, e, d = (float(v) for v in self._state[0, 0, :3].tolist())
            out = (self.kp_lat * e + self.kd_lat * d) + self.ki_lat * integral
            steer = float(np.clip(out * (2.0 / wheel_base), -self.max_steering, self.max_steering))
        return steer, accel

    def _step_pid(self, ego_state, row, target_speed, lat_target):
        import torch

        from ..types import TypeParams, TypeTable
        from ..world import BatchedWorld

        w = getattr(self, "_world", None)
        if w is None:
            w = self._world = BatchedWorld(1, 2, TypeTable([TypeParams()]), steer_first=True)
        if self._state is None:
            self._state = torch.zeros((1, 2, 6), dtype=torch.float64, device=w.device)
            self._state[0, 0] = torch.from_numpy(self._pending)
        sp = ego_state.speed
        z = np.zeros((1, 2), np.float32)
        x, y, h, v = z.copy(), z.copy(), z.copy(), z.copy()
        x[0, 0], y[0, 0], h[0, 0], v[0, 0] = ego_state.x, ego_state.y, ego_state.heading, 0.0 if sp is None else sp
        w.set_state(x, y, h, v, type_id=np.array([[0, 255]], np.uint8))
        target = np.array([[[target_speed, lat_target], [0.0, 0.0]]], np.float32)
        w.set_controllers([row], ctrl_id=np.array([[0, NO_CONTROLLER]], np.uint8), pid_target=target,
                          pid_state=self._state)
        act = w.control(torch.zeros((1, 2, 2), dtype=torch.float32, device=w.device))
        steer, accel = act[0, 0].tolist()
        return steer, accel

    def __repr__(self) -> str:
        return f"PIDController(control_mode={self.control_mode!r}, lateral_error={self.lateral_error!r})"


def _check_lateral_error(value):
    if value not in LATERAL_ERRORS:
        raise ValueError(f"lateral_error must be one of {set(LATERAL_ERRORS)}, got '{value}'")


def _lateral_source(kwargs):
    """pid_controller.py:249-283: (source, column-1 target) from the keywords, or the reference's exception."""
    if "target_heading" in kwargs:
        value = kwargs["target_heading"]
        if not isinstance(value, (int, float)):
            raise TypeError("target_heading must be numeric")
        return PID_LAT_HEADING, value
    if "cross_track_error" in kwargs:
        value = kwargs["cross_track_error"]
        if not isinstance(value, (int, float)):
            raise TypeError("cross_track_error must be numeric")
        return PID_LAT_CROSS_TRACK, value
    raise ValueError("Lateral control requires either 'target_heading' or 'cross_track_error' in kwargs")
