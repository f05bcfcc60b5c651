"""``SingleTrackDynamics`` - dynamic bicycle with a linear tyre model.

Constructor (extra ``mass, mass_height, mu=0.7, I_z=1500, cf=cr=20.89``), ``step`` and ``verify_state``
follow the reference's ``tactics2d/physics/single_track_dynamics.py`` (:58-138, :231-251, :253-303).  The
model carries no hidden state between calls (:159-160 re-derive the yaw rate and slip angle per call) and has
no remainder sub-step (:143); the returned State has ``vx = vy = None`` as in the reference (:220-227).
The integration (:140-229) runs in the sm_90a kernels in fp64.
"""

from __future__ import annotations

from typing import Tuple, Union

from ..participant.trajectory import State
from ..types import MODEL_DYNAMICS
from .single_track_kinematics import SingleTrackKinematics


class SingleTrackDynamics(SingleTrackKinematics):
    _MODEL = MODEL_DYNAMICS

    def __init__(self, lf: float, lr: float, mass: float, mass_height: float, mu: float = 0.7, I_z: float = 1500,
                 cf: float = 20.89, cr: float = 20.89, steer_range: Union[float, Tuple[float, float]] = None,
                 speed_range: Union[float, Tuple[float, float]] = None,
                 accel_range: Union[float, Tuple[float, float]] = None, interval: int = 100, delta_t: int = None):
        super().__init__(lf, lr, steer_range, speed_range, accel_range, interval, delta_t)
        self.mass, self.mass_height, self.mu, self.I_z, self.cf, self.cr = mass, mass_height, mu, I_z, cf, cr

    def type_params(self, **shape):
        return super().type_params(mass=self.mass, mass_height=self.mass_height, mu=self.mu, I_z=self.I_z, cf=self.cf,
                                   cr=self.cr, **shape)

    def step(self, state: State, accel: float, delta: float, interval: int = None):
        nxt, a, d = super().step(state, accel, delta, interval)
        nxt.vx = None   # single_track_dynamics.py:220-227: the State is built without vx, vy
        nxt.vy = None
        return nxt, a, d
