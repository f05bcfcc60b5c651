"""``ScenarioManager`` - the tick contract of the reference's ``tactics2d/traffic/scenario_manager.py:13-98``
(``update`` -> physics + add_state, ``check_status`` -> priority chain, ``reset``, ``render``) and a concrete
batched manager that drives N scenarios x M participants through one fused kernel launch per tick."""

from __future__ import annotations

from abc import ABC, abstractmethod
from typing import Optional, Tuple

from .status import ScenarioStatus, TrafficStatus


class ScenarioManager(ABC):
    def __init__(self, max_step: int = None, step_size: int = None, render_fps: int = 60, off_screen: bool = False):
        self.render_fps = render_fps
        self.off_screen = off_screen
        self.max_step = max_step
        self.step_size = int(step_size) if step_size is not None else int(1000 / render_fps)   # :50
        self.cnt_step = 0
        self.scenario_status = ScenarioStatus.NORMAL
        self.traffic_status = TrafficStatus.NORMAL
        self.map_ = None
        self.participants = None
        self.render_manager = None
        self.agent = None

    @abstractmethod
    def check_status(self) -> Tuple[ScenarioStatus, TrafficStatus]:
        ...

    @abstractmethod
    def update(self, action):
        ...

    @abstractmethod
    def render(self):
        ...

    @abstractmethod
    def reset(self):
        ...

    def get_active_participants(self, frame: int) -> list:
        return [p.id_ for p in self.participants if p.is_active(frame)]

    def get_observation(self):
        return self.render_manager.get_observation()


class BatchedScenarioManager(ScenarioManager):
    """N scenarios at once.  ``update(action)`` is ``_ParkingScenarioManager.update`` (envs/parking.py:352-359)
    for every participant of every scenario - one ``t2d_step`` launch, which also evaluates the whole
    ``check_status`` chain (:361-392) in the same pass; ``check_status()`` then only reads the result.

    Status tensors (uint8, device): ``scenario_status [N]`` holds ``ScenarioStatus`` codes by the reference's
    priority time-exceed -> out-of-bound -> collision; ``traffic_status [N, M]`` holds ``TrafficStatus`` codes
    (COLLISION_STATIC before COLLISION_DYNAMIC, else NORMAL)."""

    def __init__(self, world, max_step: int = None, step_size: int = None, render_fps: int = 60, off_screen: bool = True):
        super().__init__(max_step, step_size if step_size is not None else world.interval, render_fps, off_screen)
        self.world = world
        world.set_config(interval=self.step_size, max_step=self.max_step or 0)
        self._initial = None
        self._last = None
        self.env_result = None
        self.reset_trackers_on_done = True

    def set_initial_state(self, pool: dict):
        """Pool of initial states ``x, y, heading, speed[, vx, vy]`` [P, M] (device) that ``reset`` draws from."""
        self._initial = pool

    def update(self, action):
        self.cnt_step += 1
        self._last = self.world.step(action)
        return self.get_observation()

    def check_status(self):
        """(scenario_status [N], traffic_status [N, M]) of the last tick.  The priority chain itself ran inside the tick
        (parking.py:361-392); the TrafficStatus codes come from ``t2d_env_epilogue`` - one launch that also leaves the
        reward / terminated / truncated / done vectors of ``ParkingEnv.step`` in ``self.env_result``."""
        r = self._last if self._last is not None else self.world.check_events()
        self.env_result = self.world.env_epilogue(reset_trackers_on_done=self.reset_trackers_on_done)
        return r.status, self.env_result.traffic_status

    def get_observation(self):
        w = self.world
        return dict(x=w.x, y=w.y, heading=w.heading, speed=w.speed, vx=w.vx, vy=w.vy)

    def render(self):
        raise NotImplementedError("rendering is outside this hot path (SURVEY.md section 2, row 13)")

    def reset(self, mask=None, pool_index=None, sample=False):
        """Masked reset (all scenarios when ``mask`` is None) from the initial-state pool.  ``sample``: draw the episodes
        through the world's reset sampler (``BatchedWorld.reset_sampled``: the rows come from its seeded stream, so
        ``pool_index`` is not taken)."""
        import torch

        if self._initial is None:
            raise RuntimeError("call set_initial_state(pool) before reset()")
        if sample and pool_index is not None:
            raise ValueError("a sampled reset draws its rows: pool_index is not taken")
        if mask is None:
            mask = torch.ones(self.world.N, dtype=torch.uint8, device=self.world.device)
            self.cnt_step = 0
        if sample:
            self.world.reset_sampled(mask, self._initial)
        else:
            self.world.reset(mask, self._initial, pool_index)
        self._last = None
