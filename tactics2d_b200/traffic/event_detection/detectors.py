"""Batched event detectors with the reference's class names.

The reference's detectors take ONE shapely pose and return ONE bool
(``tactics2d/traffic/event_detection/{collision,out_bound,time_exceed}.py``).  Both call forms exist here:

* ``update(world)`` takes a :class:`tactics2d_b200.BatchedWorld` and returns device tensors for all N x M
  participants; the arithmetic runs in the fused kernel (``t2d_step`` computes every detector in the same pass as the
  physics; ``t2d_check_events`` evaluates them alone);
* ``update(agent_pose)`` - the reference's signature (collision.py:37, out_bound.py:37, arrival.py:32) - takes ONE pose, the
  (4, 2) corner ring ``Vehicle.get_pose()`` returns (or anything with ``.exterior.coords``, i.e. a shapely Polygon), and
  returns one ``bool``: the pose is put into a one-scenario world and sent through the same kernel
  (``t2d_check_events``), so a reference-style per-agent loop can hand its poses over one at a time.

Semantics kept from the reference:

* ``StaticCollision``  first static object in list order that the pose ``intersects`` (collision.py:37-43);
* ``DynamicCollision`` first other participant in list order whose pose ``intersects`` (collision.py:18-25;
  the reference method as written dereferences ``.geometry`` on shapely objects and cannot run - its intent,
  ego against every other pose with ``break``, is what is implemented, for every participant as the ego);
* ``OutBound``         ``not box.contains(pose)`` with box = (xmin, xmax, ymin, ymax) (out_bound.py:28-48);
* ``TimeExceed``       ``cnt_step += 1; cnt_step > max_step`` (time_exceed.py:26-33);
* ``OffRoute``         ``route.distance(centre) > threshold`` (off_route.py:24-35), the route a polyline.
"""

from __future__ import annotations

from typing import Optional, Sequence

from .event_base import EventBase

F_DYNAMIC, F_STATIC, F_OUTBOUND = 1, 2, 4


def _is_world(obj) -> bool:
    return hasattr(obj, "check_events") and hasattr(obj, "_out")


def _pose_to_rect(pose):
    """(cx, cy, heading, half_len, half_wid) of a pose given as the (4, 2) corner ring of ``get_pose`` - order
    (+l, -w), (+l, +w), (-l, +w), (-l, -w) rotated and moved (vehicle.py:133-140,272-281) - or as a shapely-like polygon."""
    import numpy as np

    if hasattr(pose, "exterior"):
        pose = np.asarray(pose.exterior.coords)[:4]
    elif hasattr(pose, "coords"):
        pose = np.asarray(pose.coords)[:4]
    c = np.asarray(pose, dtype=np.float64).reshape(-1, 2)
    if c.shape[0] < 4:
        raise ValueError("a pose is the ring of 4 corners that get_pose() returns")
    c = c[:4]
    centre = c.mean(0)
    front = 0.5 * (c[0] + c[1]) - centre
    side = 0.5 * (c[1] - c[0])
    return (float(centre[0]), float(centre[1]), float(np.arctan2(front[1], front[0])), float(np.hypot(*front)), float(np.hypot(*side)))


class _PoseProbe:
    """One scenario holding the agent's pose in slot 0 and up to 127 other poses: the single-pose call form."""

    def __init__(self, device="cuda:0"):
        self.device = device
        self._world = None
        self._key = None

    def run(self, rects, segments=None, bounds=None, poly_start=None):
        import numpy as np

        from ...types import MODEL_STATIC, SHAPE_OBB, TypeParams, TypeTable
        from ...world import BatchedWorld

        if len(rects) > 128:
            raise ValueError("at most 127 other agents per call")
        m = 1
        while m < len(rects):
            m *= 2
        m = max(m, 4)
        dims = tuple((round(r[3], 6), round(r[4], 6)) for r in rects)
        rows, ids = [], []
        for d in dims:   # one type row per distinct box size (<= 64 rows)
            if d not in rows:
                rows.append(d)
            ids.append(rows.index(d))
        key = (m, tuple(rows))
        if self._world is None or self._key != key:
            if self._world is not None:
                self._world.close()
            table = TypeTable([TypeParams(half_len=hl, half_wid=hw, model=MODEL_STATIC, shape=SHAPE_OBB) for hl, hw in rows])
            self._world = BatchedWorld(1, m, table, device=self.device)
            self._key = key
        w = self._world
        w.set_map(segments, bounds, poly_start=poly_start)
        x = np.zeros((1, m), np.float32); y = np.zeros((1, m), np.float32); h = np.zeros((1, m), np.float32)
        tid = np.full((1, m), 255, np.uint8)
        for i, r in enumerate(rects):
            x[0, i], y[0, i], h[0, i], tid[0, i] = r[0], r[1], r[2], ids[i]
        w.set_state(x, y, h, np.zeros((1, m), np.float32), type_id=tid)
        r = w.check_events()
        return int(r.flags[0, 0].item()), int(r.hit_index[0, 0].item()), int(r.hit_segment[0, 0].item())


def _events(world, fresh: bool):
    """Flags of the last ``step`` (they were computed in that pass) or a fresh ``check_events`` launch."""
    return world.check_events() if fresh else world._out


class DynamicCollision(EventBase):
    def __init__(self):
        super().__init__()

    def update(self, world, other_agents=None, fresh: bool = True):
        """``update(world)`` -> (collided bool [N, M], first-hit participant index int16 [N, M], -1 = none);
        ``update(agent_pose, other_agents)`` (the reference's call, collision.py:18-25: ``other_agents`` have ``get_pose()``,
        or are poses themselves) -> bool."""
        if not _is_world(world):
            others = [_pose_to_rect(o.get_pose() if hasattr(o, "get_pose") else o) for o in (other_agents or [])]
            if not hasattr(self, "_probe"):
                self._probe = _PoseProbe()
            flags, self.hit_index, _ = self._probe.run([_pose_to_rect(world)] + others)
            self.hit_index = self.hit_index - 1 if self.hit_index > 0 else -1   # index into other_agents
            return bool(flags & F_DYNAMIC)
        r = _events(world, fresh)
        return (r.flags & F_DYNAMIC) != 0, r.hit_index

    def reset(self):
        return


class StaticCollision(EventBase):
    def __init__(self, static_objects: Optional[Sequence] = None):
        self.static_objects = static_objects   # [S, 4] segments (x1, y1, x2, y2) in list order

    def update(self, world, fresh: bool = True):
        """``update(world)`` -> (collided bool [N, M], first-hit object int16 [N, M], -1 = none);
        ``update(agent_pose)`` (collision.py:37-43) -> bool, against ``self.static_objects`` = the [S, 4] segments (with
        ``self.poly_start`` marking the Area polygons among them, see ``tactics2d_b200.map.polygons_to_segments``)."""
        if not _is_world(world):
            if not hasattr(self, "_probe"):
                self._probe = _PoseProbe()
            flags, _, self.hit_object = self._probe.run([_pose_to_rect(world)], self.static_objects, None, getattr(self, "poly_start", None))
            return bool(flags & F_STATIC)
        r = _events(world, fresh)
        return (r.flags & F_STATIC) != 0, r.hit_segment

    def reset(self, static_objects=None, world=None, poly_start=None):
        """Replace the static objects; with ``world`` given the map tile is re-staged on the device."""
        self.static_objects = static_objects
        self.poly_start = poly_start
        if world is not None:
            world.set_map(static_objects, world.bounds, poly_start=poly_start)


class OutBound(EventBase):
    def __init__(self, boundary: tuple = None):
        self.map_boundary = boundary   # (xmin, xmax, ymin, ymax)

    def update(self, world, fresh: bool = True):
        """``update(world)`` -> bool [N, M]; ``update(agent_pose)`` (out_bound.py:37-48) -> bool (False without a boundary)."""
        if not _is_world(world):
            if self.map_boundary is None:
                return False
            if not hasattr(self, "_probe"):
                self._probe = _PoseProbe()
            return bool(self._probe.run([_pose_to_rect(world)], None, self.map_boundary)[0] & F_OUTBOUND)
        r = _events(world, fresh)
        return (r.flags & F_OUTBOUND) != 0

    def reset(self, boundary: tuple = None, world=None):
        self.map_boundary = boundary
        if world is not None:
            world.set_map(world.segments, boundary)


class TimeExceed(EventBase):
    def __init__(self, max_step: int):
        self.max_step = max_step
        self.cnt_step = 0

    def update(self, world=None):
        """Scalar form (reference): ``++cnt > max_step``.  With a world: the per-scenario device counters,
        which ``t2d_step`` increments, compared against ``max_step`` -> bool [N]."""
        if world is None:
            self.cnt_step += 1
            return self.cnt_step > self.max_step
        return world.step_count > self.max_step

    def reset(self, world=None):
        self.cnt_step = 0
        if world is not None:
            world.step_count.zero_()


class Arrival(EventBase):
    """``Arrival`` (reference arrival.py:12-50): IoU of the ego's pose with the target area, completed when
    ``iou >= threshold`` (default 0.95).  Batched: ``reset(target, world)`` installs one target rectangle per
    scenario, ``update(world)`` returns ``(is_completed bool [N], iou fp32 [N])`` of the last ``step``."""

    def __init__(self, target_area=None, threshold: float = 0.95):
        self.target_area = target_area   # [N, 5] = (cx, cy, heading, half_len, half_wid)
        self.threshold = threshold

    def update(self, world):
        """``update(world)`` -> (is_completed bool [N], iou fp32 [N]) of the last ``step``; ``update(agent_pose)``
        (arrival.py:32-47) -> (bool, float) against ``self.target_area`` = one (cx, cy, heading, half_len, half_wid) row or a
        (4, 2) corner ring."""
        if not _is_world(world):
            import numpy as np
            import torch

            from ...types import MODEL_STATIC, SHAPE_OBB, TypeParams, TypeTable
            from ...world import BatchedWorld

            rect = _pose_to_rect(world)
            tgt = np.asarray(self.target_area, dtype=np.float64)
            tgt = np.asarray(_pose_to_rect(tgt)) if tgt.size == 8 else tgt.reshape(-1)[:5]
            w = BatchedWorld(1, 4, TypeTable([TypeParams(half_len=rect[3], half_wid=rect[4], model=MODEL_STATIC, shape=SHAPE_OBB)]))
            tid = np.full((1, 4), 255, np.uint8); tid[0, 0] = 0
            z = np.zeros((1, 4), np.float32)
            x, y, h = z.copy(), z.copy(), z.copy()
            x[0, 0], y[0, 0], h[0, 0] = rect[0], rect[1], rect[2]
            w.set_state(x, y, h, z, type_id=tid)
            w.set_goal(tgt.reshape(1, 5).astype(np.float32), self.threshold, 0)
            r = w.step(torch.zeros((1, 4, 2), device=w.device))
            iou = float(r.iou[0].item())
            w.close()
            return iou >= self.threshold, iou
        r = world._out
        if r.iou is None:
            raise RuntimeError("no target area: call Arrival.reset(target_area, world) / world.set_goal first")
        return r.iou >= self.threshold, r.iou

    def reset(self, target_area=None, world=None, no_action_max_step: int = 100):
        self.target_area = target_area
        if world is not None:
            world.set_goal(target_area, self.threshold, no_action_max_step)


class NoAction(EventBase):
    """``NoAction`` (reference no_action.py:12-58): counts consecutive ticks in which the ego's pose overlaps its
    previous pose with IoU > 0.999; fires when the count exceeds ``max_step``.  The counter lives on the device
    (``world.set_goal(..., no_action_max_step=max_step)``); ``update(world)`` reads it."""

    def __init__(self, max_step=100):
        self.max_step = max_step
        self.cnt_no_action = 0

    def update(self, world):
        if world._goal is None:
            raise RuntimeError("NoAction needs world.set_goal(target, no_action_max_step=...)")
        return world._goal["count"] > self.max_step

    def reset(self, world=None):
        self.cnt_no_action = 0
        if world is not None and world._goal is not None:
            world._goal["count"].zero_()
            world._goal["last_pose"].zero_()


def _route_points(route):
    """[V, 2] float64 vertices of a LineString-like route (anything with ``.coords``) or a list of points."""
    import numpy as np

    try:
        pts = np.asarray(route.coords if hasattr(route, "coords") else route, dtype=np.float64)
    except (TypeError, ValueError):
        pts = None
    if pts is None or pts.ndim != 2 or pts.shape[1] != 2 or pts.shape[0] < 2:
        raise TypeError("The route should be a LineString or a list of points.")
    return pts


class OffRoute(EventBase):
    """``OffRoute`` (reference off_route.py:12-51): off when the distance from the agent's centre to the route exceeds
    ``threshold``.  Batched: ``world.set_routes(route_id, threshold)`` binds one route per slot and the epilogues apply
    the detector (DESIGN.md section 1 "Route following"); ``update(world)`` returns their flags.  ``reset(route)`` /
    ``update(location)`` keep the reference's single-agent form: the location goes through a one-scenario world."""

    def __init__(self, threshold):
        self.threshold = threshold
        self.route = None

    def update(self, location):
        """``update(world)`` -> bool [N, M]: the slots the last epilogue found off route (``agents_epilogue``'s traffic
        status when agents are bound, else ``env_epilogue``'s, which scores the ego); ``update(location)``
        (off_route.py:24-35, a shapely Point or an (x, y) pair) -> bool against the route of ``reset``."""
        if _is_world(location):
            from ..status import TrafficStatus

            w = location
            traffic = w._agents["traffic"] if w._agents is not None else (None if w._env is None else w._env["traffic"])
            if traffic is None:
                raise RuntimeError("no epilogue has run: call env_epilogue or agents_epilogue first")
            return traffic == int(TrafficStatus.OFF_ROUTE)
        if self.route is None:
            raise ValueError("The route should be set before the event detection.")
        import numpy as np

        xy = np.asarray(location.coords[0] if hasattr(location, "coords") else location, dtype=np.float64).reshape(-1)[:2]
        if not hasattr(self, "_probe"):
            self._probe = _RouteProbe()
        return self._probe.run(self.route, float(self.threshold), float(xy[0]), float(xy[1]))

    def reset(self, route):
        """``route``: a LineString-like object or a list of points (off_route.py:37-51); TypeError otherwise."""
        self.route = _route_points(route)


class _RouteProbe:
    """One scenario with one static participant at the location, its route bound: the single-location call form."""

    def __init__(self, device="cuda:0"):
        self.device = device
        self._world = None

    def run(self, route, threshold, x, y):
        import numpy as np

        from ...types import MODEL_STATIC, SHAPE_NONE, TypeParams, TypeTable
        from ...world import BatchedWorld

        if self._world is None:
            table = TypeTable([TypeParams(half_len=0.5, half_wid=0.5, model=MODEL_STATIC, shape=SHAPE_NONE)])
            self._world = BatchedWorld(1, 1, table, device=self.device)
        w = self._world
        w.set_paths([route])
        w.set_routes(np.zeros((1, 1), np.int16), threshold, 0.0, 0.0)
        z = np.zeros((1, 1), np.float32)
        w.set_state(np.full((1, 1), x, np.float32), np.full((1, 1), y, np.float32), z, z, type_id=np.zeros((1, 1), np.uint8))
        w.check_events()
        w._out.status.fill_(1)   # NORMAL: the probe never ticks
        e = w.env_epilogue()
        return bool(e.truncated[0].item())
