"""Sensors on this path: the single-line lidar (the vector observation of the reference's ParkingEnv,
envs/parking.py:303-304,422-429) and the bird's-eye-view camera (its image observation, envs/parking.py:130)."""

from .camera import BEVCamera
from .lidar import SingleLineLidar

__all__ = ["BEVCamera", "SingleLineLidar"]
