"""``ControllerBase`` (tactics2d/controller/controller_base.py:14-95): ``step`` / ``reset`` / ``configure`` and the
driving-style interpolator, plus the hooks the batched path needs (``params`` -> one ``t2d_controller_params`` row)."""

from __future__ import annotations

from abc import ABC, abstractmethod
from typing import Tuple

import numpy as np

from .. import _lib

CTRL_EXTERNAL, CTRL_IDM, CTRL_CRUISE, CTRL_PURE_PURSUIT, CTRL_PID = range(5)
# t2d_controller_params.pid_lateral / pid_longitudinal (T2D_PID_LAT_* / T2D_PID_LON_*)
PID_LAT_NONE, PID_LAT_HEADING, PID_LAT_CROSS_TRACK, PID_LAT_PATH_HEADING, PID_LAT_PATH_CROSS_TRACK = range(5)
PID_LON_NONE, PID_LON_TARGET = range(2)
NO_CONTROLLER = 255


class _StyleInterpolator:
    """``interp1d([x_left, x_right], [y_left, y_right], bounds_error=False, fill_value=(y_left, y_right))``
    (controller_base.py:68-91): linear inside the range, the end values outside."""

    def __init__(self, y_left, y_right, x_left=-1.0, x_right=1.0):
        self.xp, self.fp = (float(x_left), float(x_right)), (float(y_left), float(y_right))

    def __call__(self, style_id):
        return float(np.interp(float(style_id), self.xp, self.fp))


class ControllerBase(ABC):
    @abstractmethod
    def step(self, ego_state, **kwargs) -> Tuple[float, float]:
        """``(steering, acceleration)`` for the ego vehicle (controller_base.py:24-43)."""

    def reset(self) -> None:
        pass

    def configure(self, **kwargs) -> None:
        for key, value in kwargs.items():
            if hasattr(self, key):
                setattr(self, key, value)
            else:
                raise AttributeError(f"Controller {self.__class__.__name__} has no parameter '{key}'")

    @staticmethod
    def create_style_interpolator(y_left: float, y_right: float, x_left: float = -1.0, x_right: float = 1.0):
        return _StyleInterpolator(y_left, y_right, x_left, x_right)

    # ------------------------------------------------------------------ batched path
    def params(self) -> "_lib.ControllerParamsC":
        """This controller as one row of the device controller table."""
        raise NotImplementedError

    def _step_one(self, ego_state, lead_state=None, path=None, wheel_base=None):
        """One ``State`` through ``t2d_control`` (a 1 x 2 batch: the ego and, optionally, its leader)."""
        import torch

        from ..types import TypeParams, TypeTable
        from ..world import BatchedWorld

        w = getattr(self, "_world", None)
        if w is None:
            w = self._world = BatchedWorld(1, 2, TypeTable([TypeParams()]), steer_first=True)
        row = self.params()
        if wheel_base is not None:
            row.wheel_base = float(wheel_base)

        def accel_of(s):
            a = s.accel
            if a is None:   # the reference fails on `None - float` (acceleration_controller.py:96)
                raise TypeError("the state carries no acceleration (State.accel is None)")
            return float(a)

        needs_accel = row.kind in (CTRL_CRUISE, CTRL_PURE_PURSUIT)
        states = [ego_state] + ([lead_state] if lead_state is not None else [])
        z = np.zeros((1, 2), np.float32)
        x, y, h, v, la = z.copy(), z.copy(), z.copy(), z.copy(), z.copy()
        tid = np.full((1, 2), 255, np.uint8)
        for i, s in enumerate(states):
            sp = s.speed
            x[0, i], y[0, i], h[0, i], v[0, i] = s.x, s.y, s.heading, 0.0 if sp is None else sp
            la[0, i] = accel_of(s) if needs_accel else 0.0
            tid[0, i] = 0
        w.set_state(x, y, h, v, type_id=tid)
        w.set_paths([] if path is None else [path])
        w.set_controllers([row], ctrl_id=np.array([[0, NO_CONTROLLER]], np.uint8),
                          lead_index=np.array([[1 if lead_state is not None else -1, -1]], np.int16),
                          path_id=np.array([[0 if path is not None else -1, -1]], np.int16), last_accel=la)
        act = w.control(torch.zeros((1, 2, 2), dtype=torch.float32, device=w.device))
        steer, accel = act[0, 0].tolist()
        return steer, accel

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}()"
