"""``SingleTrackDrift`` - dynamic bicycle with wheel spin and a Pacejka "magic formula" tyre.

Constructor, ``step(state, omega_wf, omega_wr, accel, delta, interval) -> (State, omega_wf, omega_wr, accel, delta)``
and ``verify_state`` follow the reference's ``tactics2d/physics/single_track_drift.py`` (:98-183, :467-499, :501-556).
The integration (:340-465, tyre forces :185-338) runs in the sm_90a kernels in fp64, with the reference's built-in
``Tire`` coefficients (:14-49; a custom tyre object is not supported - the coefficients are compile-time constants of
the kernel).  Unlike ``SingleTrackDynamics`` this model takes the remainder sub-step (:352-355) and carries the two
wheel speeds from call to call; the returned State has ``vx = vy = None`` (:457-464).
"""

from __future__ import annotations

from typing import Tuple, Union

from ..participant.trajectory import State
from ..types import MODEL_DRIFT
from .single_track_kinematics import SingleTrackKinematics


class Tire:
    """The reference's default tyre (single_track_drift.py:14-49); kept for signature compatibility."""


class SingleTrackDrift(SingleTrackKinematics):
    _MODEL = MODEL_DRIFT

    def __init__(self, lf: float, lr: float, mass: float, mass_height: float, radius: float = 0.344, T_sb: float = 0.76,
                 T_se: float = 1, tire=None, I_z: float = 1500, I_yw: float = 1.7,
                 steer_range: Union[float, Tuple[float, float]] = None, speed_range: Union[float, Tuple[float, float]] = None,
                 accel_range: Union[float, Tuple[float, float]] = None, interval: int = 100, delta_t: int = None):
        if tire is not None and not isinstance(tire, Tire):
            raise NotImplementedError("only the built-in tyre model runs on the device")
        super().__init__(lf, lr, steer_range, speed_range, accel_range, interval, delta_t)
        self.mass, self.mass_height, self.radius, self.T_sb, self.T_se = mass, mass_height, radius, T_sb, T_se
        self.tire = tire if tire is not None else Tire()
        self.I_z, self.I_yw = I_z, I_yw

    def type_params(self, **shape):
        return super().type_params(mass=self.mass, mass_height=self.mass_height, I_z=self.I_z, wheel_radius=self.radius,
                                   T_sb=self.T_sb, T_se=self.T_se, I_yw=self.I_yw, **shape)

    def step_batch(self, x, y, heading, speed, omega_wf, omega_wr, accel, delta, interval: int = None):
        """n participants at once: fp32 CUDA tensors of one shape; state and wheel speeds are advanced IN PLACE.
        Returns ``(vx, vy, accel_applied, delta_applied)``."""
        import torch

        interval = interval if interval is not None else self.interval
        action = torch.stack([accel.reshape(-1), delta.reshape(-1)], dim=1).contiguous()
        applied = torch.empty_like(action)
        vx, vy = torch.empty_like(x), torch.empty_like(x)
        self._launch(self.type_params(), interval, x.numel(), x, y, heading, speed, vx, vy, action, applied, omega_wf, omega_wr)
        return vx, vy, applied[:, 0].reshape(x.shape), applied[:, 1].reshape(x.shape)

    def step(self, state: State, omega_wf: float, omega_wr: float, accel: float, delta: float, interval: int = None):
        """``(next_state, next_omega_wf, next_omega_wr, accel, delta)`` (single_track_drift.py:467-499)."""
        import torch

        interval = interval if interval is not None else self.interval
        if not torch.cuda.is_available():
            raise RuntimeError("tactics2d_b200 physics needs a CUDA device (no CPU implementation)")
        dev = torch.device("cuda", torch.cuda.current_device())
        buf = torch.tensor([[state.x], [state.y], [state.heading], [state.speed], [omega_wf], [omega_wr]], dtype=torch.float32,
                           device=dev)
        a = torch.tensor([float(accel)], dtype=torch.float32, device=dev)
        d = torch.tensor([float(delta)], dtype=torch.float32, device=dev)
        _, _, a_c, d_c = self.step_batch(buf[0], buf[1], buf[2], buf[3], buf[4], buf[5], a, d, interval)
        out = torch.cat([buf.reshape(-1), a_c, d_c]).cpu().tolist()
        nxt = State(frame=state.frame + interval, x=out[0], y=out[1], heading=out[2], speed=out[3], accel=out[6])
        return nxt, out[4], out[5], out[6], out[7]
