"""``IDMController`` (tactics2d/controller/idm_controller.py:16-155): Intelligent Driver Model, longitudinal only; a
batched row may add lane keeping, a PID lateral channel on the slot's path (DESIGN.md section 1 "Lane keeping for IDM
rows")."""

from __future__ import annotations

from typing import Tuple

from .. import _lib
from .controller_base import CTRL_IDM, PID_LAT_PATH_CROSS_TRACK, PID_LAT_PATH_HEADING, ControllerBase


class IDMController(ControllerBase):
    def __init__(self, desired_speed: float = 10.0, time_headway: float = 1.5, min_spacing: float = 2.0,
                 max_acceleration: float = 1.0, comfortable_deceleration: float = 3.0, delta: float = 4.0,
                 lateral=None):
        """``lateral``: None (the reference's IDM, steering 0), or a ``PIDController`` whose ``lateral_error`` is
        ``"path_heading"`` or ``"path_cross_track"``: the batched row then also steers the slot along its path with that
        controller's lateral channel (gains, ``dt``, ``derivative_filter_alpha``, ``max_steering``), on ``pid_state``."""
        if lateral is not None:
            from .pid_controller import PIDController

            if not isinstance(lateral, PIDController) or lateral.lateral_error not in ("path_heading", "path_cross_track"):
                raise ValueError("lateral must be a PIDController with lateral_error 'path_heading' or 'path_cross_track'")
        self.lateral = lateral
        self.desired_speed = desired_speed
        self.time_headway = time_headway
        self.min_spacing = min_spacing
        self.max_acceleration = max_acceleration
        self.comfortable_deceleration = comfortable_deceleration
        self.delta = delta

    def params(self):
        row = _lib.ControllerParamsC(kind=CTRL_IDM, desired_speed=self.desired_speed, time_headway=self.time_headway,
                                     min_spacing=self.min_spacing, max_acceleration=self.max_acceleration,
                                     comfortable_deceleration=self.comfortable_deceleration, delta=self.delta)
        if self.lateral is not None:   # the PID row's lateral fields; its longitudinal ones are not read
            lat = self.lateral.params()
            row.pid_lateral = PID_LAT_PATH_HEADING if self.lateral.lateral_error == "path_heading" else PID_LAT_PATH_CROSS_TRACK
            for k in ("wheel_base", "dt", "kp_lat", "ki_lat", "kd_lat", "max_steering", "derivative_filter_alpha"):
                setattr(row, k, getattr(lat, k))
        return row

    def step(self, ego_state, leading_state=None, **kwargs) -> Tuple[float, float]:
        """``(0.0, acceleration)``: free flow without a leader, car following with one (idm_controller.py:59-92).  The
        lateral channel needs a path and per-slot state, so it is a batched-row feature: this single-state call keeps the
        reference's steering 0 with or without one."""
        _, accel = self._step_one(ego_state, leading_state)
        return 0.0, accel

    def configure(self, **kwargs) -> None:
        for key, value in kwargs.items():
            if hasattr(self, key):
                setattr(self, key, value)
            else:
                raise AttributeError(f"IDMController has no parameter '{key}'")
