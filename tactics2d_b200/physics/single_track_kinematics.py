"""``SingleTrackKinematics`` - kinematic bicycle, geometry centre as reference point.

Constructor, ``step`` signature / return value and ``verify_state`` follow the reference's
``tactics2d/physics/single_track_kinematics.py`` (:62-124 constructor and range rules, :178-198 ``step`` ->
``(State, accel, delta)`` with the clipped action, :200-250 ``verify_state``).  The integration itself
(:126-176) runs in the sm_90a kernels: a single ``State`` goes through a batch of one; ``step_batch``
advances n participants per launch.
"""

from __future__ import annotations

from typing import Tuple, Union

import numpy as np

from ..participant.trajectory import State
from ..types import MODEL_KINEMATICS, SHAPE_NONE, TypeParams, normalize_range_bicycle
from .physics_model_base import PhysicsModelBase


def _store(rng):
    return None if rng[0] == -np.inf and rng[1] == np.inf else [rng[0], rng[1]]


class SingleTrackKinematics(PhysicsModelBase):
    _MODEL = MODEL_KINEMATICS

    def __init__(self, lf: float, lr: float, steer_range: Union[float, Tuple[float, float]] = None,
                 speed_range: Union[float, Tuple[float, float]] = None,
                 accel_range: Union[float, Tuple[float, float]] = None, interval: int = 100, delta_t: int = None):
        self.lf = lf
        self.lr = lr
        self.wheel_base = lf + lr
        self._steer = normalize_range_bicycle(steer_range)
        self._speed = normalize_range_bicycle(speed_range)
        self._accel = normalize_range_bicycle(accel_range)
        self.steer_range, self.speed_range, self.accel_range = _store(self._steer), _store(self._speed), _store(self._accel)
        self.interval = interval
        self.delta_t = self._effective_delta_t(delta_t, interval)

    # ------------------------------------------------------------------ parameters for the kernels
    def type_params(self, **shape) -> TypeParams:
        kw = dict(lf=self.lf, lr=self.lr, steer_lo=self._steer[0], steer_hi=self._steer[1], speed_lo=self._speed[0],
                  speed_hi=self._speed[1], accel_lo=self._accel[0], accel_hi=self._accel[1], model=self._MODEL,
                  shape=SHAPE_NONE)
        kw.update(shape)
        return TypeParams(**kw)

    # ------------------------------------------------------------------ batched
    def step_batch(self, x, y, heading, speed, accel, delta, interval: int = None):
        """n participants at once.  All arguments are fp32 CUDA tensors of one shape; the state tensors are
        advanced IN PLACE.  Returns ``(vx, vy, accel_applied, delta_applied)`` tensors."""
        import torch

        interval = interval if interval is not None else self.interval
        n = x.numel()
        action = torch.stack([accel.reshape(-1), delta.reshape(-1)], dim=1).contiguous()
        applied = torch.empty_like(action)
        vx, vy = torch.empty_like(x), torch.empty_like(x)
        self._launch(self.type_params(), interval, n, x, y, heading, speed, vx, vy, action, applied)
        return vx, vy, applied[:, 0].reshape(x.shape), applied[:, 1].reshape(x.shape)

    # ------------------------------------------------------------------ reference signature
    def step(self, state: State, accel: float, delta: float, interval: int = None):
        """``(next_state, accel, delta)`` exactly as the reference returns them (:178-198)."""
        import torch

        interval = interval if interval is not None else self.interval
        dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else None
        if dev is None:
            raise RuntimeError("tactics2d_b200 physics needs a CUDA device (no CPU implementation)")
        buf = torch.tensor([[state.x], [state.y], [state.heading], [state.speed]], dtype=torch.float32, device=dev)
        a = torch.tensor([float(accel)], dtype=torch.float32, device=dev)
        d = torch.tensor([float(delta)], dtype=torch.float32, device=dev)
        vx, vy, a_c, d_c = self.step_batch(buf[0], buf[1], buf[2], buf[3], a, d, interval)
        out = torch.cat([buf.reshape(-1), vx, vy, a_c, d_c]).cpu().tolist()
        nxt = State(frame=state.frame + interval, x=out[0], y=out[1], heading=out[2], vx=out[4], vy=out[5], speed=out[3],
                    accel=out[6])
        return nxt, out[6], out[7]

    def verify_state(self, state: State, last_state: State, interval: int = None) -> bool:
        """The reference's rough reachability box (:200-250); host-side, cold."""
        interval = state.frame - last_state.frame if interval is None else interval
        if interval == 0:
            return True
        if None in [self.steer_range, self.speed_range, self.accel_range]:
            return True
        dt = float(interval) / 1000
        v0 = last_state.speed
        steer = np.array(self.steer_range, dtype=np.float64)
        beta = np.arctan(self.lr / self.wheel_base * steer)
        h = np.mod(last_state.heading + v0 / self.wheel_base * np.sin(beta) * dt, 2 * np.pi)
        if h[0] < h[1] and not h[0] <= state.heading <= h[1]:
            return False
        if h[0] > h[1] and not (h[0] <= state.heading or state.heading <= h[1]):
            return False
        sp = np.clip(v0 + np.array(self.accel_range, dtype=np.float64) * dt, *self.speed_range)
        if not sp[0] <= state.speed <= sp[1]:
            return False
        xr = last_state.x + sp * np.cos(last_state.heading + beta) * dt
        yr = last_state.y + sp * np.sin(last_state.heading + beta) * dt
        if not xr[0] < state.x < xr[1] or not yr[0] < state.y < yr[1]:
            return False
        return True
