"""``SingleLineLidar`` with the reference's constructor parameters (``tactics2d/sensor/lidar.py:33-50``):
``point_density = max(int(freq_detect / freq_scan), 1)`` beams over a full turn, ``angle_resolution = 2 pi /
point_density``, range ``perception_range``.  ``scan(world)`` runs ``_scan_obstacles`` (:128-221) for the ego of
every scenario of a :class:`tactics2d_b200.BatchedWorld` in one kernel launch and returns the [N, point_density]
distance tensor (``inf`` = nothing within range), i.e. the batched ``scan_result``; ``scan_agents(world, observers)``
scans from every row of an observer list instead, [N, Q, point_density]."""

from __future__ import annotations

import numpy as np


class SingleLineLidar:
    def __init__(self, id_: int = 0, perception_range: float = 12.0, freq_scan: float = 10.0, freq_detect: float = 5000.0):
        self.id_ = id_
        self.max_perception_distance = float(perception_range)
        self._freq_scan = freq_scan
        self._freq_detect = freq_detect
        self.point_density = max(int(self._freq_detect / self._freq_scan), 1)
        self.angle_resolution = 2 * np.pi / self.point_density
        self.scan_result = None

    @property
    def freq_scan(self) -> float:
        return self._freq_scan

    @property
    def freq_detect(self) -> float:
        return self._freq_detect

    def scan(self, world):
        self.scan_result = world.lidar_scan(self.point_density, self.max_perception_distance)
        return self.scan_result

    def scan_agents(self, world, observers=None):
        """The same sensor bound to a list of observer slots per scenario (``bind_with(j)`` for each row's slot j;
        ``BatchedWorld.lidar_scan_agents``): fp32 [N, Q, point_density].  ``observers``: int16 [N, Q] device tensor, or
        None for every slot.  Does not touch ``scan_result``, which stays the ego's scan."""
        return world.lidar_scan_agents(self.point_density, self.max_perception_distance, observers)

    def get_points(self, world):
        """Point cloud in the global frame (``_get_points``, lidar.py:223-243): [N, point_density, 2], NaN where no hit."""
        import torch

        d = self.scan_result if self.scan_result is not None else self.scan(world)
        ang = torch.linspace(0, 2 * np.pi, self.point_density + 1, device=d.device, dtype=torch.float32)[:-1]
        th = ang[None, :] + world.heading[:, :1]
        valid = torch.isfinite(d)
        dd = torch.where(valid, d, torch.full_like(d, float("nan")))
        return torch.stack([world.x[:, :1] + dd * torch.cos(th), world.y[:, :1] + dd * torch.sin(th)], -1)
