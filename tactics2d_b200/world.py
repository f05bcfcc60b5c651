"""BatchedWorld: N scenarios x M participants of structure-of-arrays state in HBM.

This is the object behind the reference-shaped facades (``physics``, ``traffic``, ``envs``): it
owns the fp32 SoA tensors, the C-ABI context, and forwards ``step`` / ``check_events`` / ``reset``
to the sm_90a kernels.  PyTorch is only the device-memory container (``tensor.data_ptr()``) and
the stream provider; there is no eager/CPU implementation behind it.

Replaces the per-object loop of the reference tick: ``ScenarioManager.update`` ->
``physics_model.step`` -> ``agent.add_state`` -> ``check_status`` (envs/parking.py:352-392).
"""

from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, replace
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib
from .types import MODEL_DRIFT, MODEL_STATIC, TYPE_INACTIVE, TypeTable

CFG_ANY_PARTICIPANT = 1
CFG_STEER_FIRST = 2

F_DYNAMIC, F_STATIC, F_OUTBOUND = 1, 2, 4


@dataclass
class StepResult:
    """Device tensors written by one ``step`` (views of buffers owned by the world)."""

    flags: torch.Tensor        # uint8 [N, M]: bit0 dynamic collision, bit1 static collision, bit2 out of bound
    hit_index: torch.Tensor    # int16 [N, M]: lowest colliding participant index or -1
    hit_segment: torch.Tensor  # int16 [N, M]: lowest colliding map segment index or -1
    status: torch.Tensor       # uint8 [N]: ScenarioStatus
    done: torch.Tensor         # uint8 [N]
    iou: Optional[torch.Tensor] = None   # fp32 [N]: IoU(ego pose, target area) when a goal is set (Arrival.update)


@dataclass
class EnvResult:
    """Device tensors written by ``env_epilogue`` (views of buffers owned by the world, overwritten by the next call)."""

    reward: torch.Tensor          # fp32 [N]
    terminated: torch.Tensor      # bool [N]
    truncated: torch.Tensor       # bool [N]
    done: torch.Tensor            # uint8 [N] = terminated | truncated (the mask ``reset`` takes)
    traffic_status: torch.Tensor  # uint8 [N, M] TrafficStatus codes


@dataclass
class AgentEnvResult:
    """Device tensors written by ``agents_epilogue`` (views of buffers owned by the world, overwritten by its next call):
    row (n, q) is the agent observed by slot ``observers[n, q]`` (DESIGN.md section 1 "Per-agent status and reward")."""

    reward: torch.Tensor          # fp32 [N, Q]
    terminated: torch.Tensor      # bool [N, Q]: the row's status is COMPLETED
    truncated: torch.Tensor       # bool [N, Q]: active, not terminated, not NORMAL
    status: torch.Tensor          # uint8 [N, Q] ScenarioStatus codes of the rows, 0 for absent rows
    iou: torch.Tensor             # fp32 [N, Q]: IoU(pose, goal), 0 without the detectors
    done: torch.Tensor            # uint8 [N]: no row of the scenario is NORMAL (the mask ``reset`` takes)
    traffic: torch.Tensor         # uint8 [N, M] TrafficStatus codes


# Columns of the blocks of the vector observation (``BatchedWorld.observe``; DESIGN.md section 1 "Vector observation").
# Positions and velocities are in the ego frame: origin at the ego's centre, +x along its heading; dh = heading - ego heading.
EGO_FIELDS = ("valid", "speed", "v_long", "v_lat", "half_len", "half_wid", "is_disc", "t_frac")
GOAL_FIELDS = ("valid", "ex", "ey", "cos_dh", "sin_dh", "half_len", "half_wid", "dist")
AGENT_FIELDS = ("valid", "ex", "ey", "cos_dh", "sin_dh", "v_x", "v_y", "half_len", "half_wid", "is_disc", "dist")
SEGMENT_FIELDS = ("valid", "ex1", "ey1", "ex2", "ey2", "ecx", "ecy", "dist", "in_ring")
# Leading columns of a row of the route observation (``BatchedWorld.route_observe``; DESIGN.md section 1 "Route
# following"), followed by the look-ahead points (x, y) in the observer's frame.
ROUTE_FIELDS = ("has_route", "lateral", "heading_error", "s_frac", "remaining")
ROUTE_MAX_POINTS = 256
# Columns of every lag of the history observation (``BatchedWorld.observe_history``; DESIGN.md section 1 "Trajectory
# history"): a recorded pose and velocity in the observer's current frame, as an agent row's fields 1..6 put them.
HIST_FIELDS = ("valid", "ex", "ey", "cos_dh", "sin_dh", "v_x", "v_y")
HISTORY_MAX = 64


def vector_obs_width(k_agents: int, k_segments: int) -> int:
    """F, the length of one scenario's row of the vector observation."""
    return len(EGO_FIELDS) + len(GOAL_FIELDS) + len(AGENT_FIELDS) * int(k_agents) + len(SEGMENT_FIELDS) * int(k_segments)


@dataclass
class VectorObservation:
    """Views of one device buffer written by ``BatchedWorld.observe`` (overwritten by its next call with the same config)."""

    flat: torch.Tensor           # fp32 [N, F]: ego, goal, agents, segments back to back
    ego: torch.Tensor            # fp32 [N, 8]   (EGO_FIELDS)
    goal: torch.Tensor           # fp32 [N, 8]   (GOAL_FIELDS; zeros without a goal)
    agents: torch.Tensor         # fp32 [N, K, 11] (AGENT_FIELDS), nearest first
    segments: torch.Tensor       # fp32 [N, S, 9]  (SEGMENT_FIELDS), nearest first
    agent_index: torch.Tensor    # int16 [N, K]: the participant slot of each agent row, -1 for padding
    segment_index: torch.Tensor  # int16 [N, S]: the segment's index in its tile, -1 for padding


@dataclass
class AgentObservation:
    """Views of one device buffer written by ``BatchedWorld.observe_agents`` (overwritten by its next call with the same
    counts): row (n, q) is the vector observation of scenario n seen from slot ``observers[n, q]``."""

    flat: torch.Tensor           # fp32 [N, Q, F]
    ego: torch.Tensor            # fp32 [N, Q, 8]      (EGO_FIELDS, of the observer)
    goal: torch.Tensor           # fp32 [N, Q, 8]      (GOAL_FIELDS)
    agents: torch.Tensor         # fp32 [N, Q, K, 11]  (AGENT_FIELDS), nearest first
    segments: torch.Tensor       # fp32 [N, Q, S, 9]   (SEGMENT_FIELDS), nearest first
    agent_index: torch.Tensor    # int16 [N, Q, K]: the participant slot of each agent row, -1 for padding
    segment_index: torch.Tensor  # int16 [N, Q, S]: the segment's index in its tile, -1 for padding
    observers: Optional[torch.Tensor] = None   # int16 [N, Q] as passed, or None: row q is slot q


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(0 if t is None else t.data_ptr())


class _DeviceArray:
    """A device array the library owns, seen by ``torch.as_tensor`` through the CUDA array interface (no copy)."""

    def __init__(self, ptr: int, shape, typestr: str):
        self.__cuda_array_interface__ = dict(shape=tuple(shape), typestr=typestr, data=(int(ptr), False), version=2)


class BatchedWorld:
    def __init__(self, n_scenarios: int, m_participants: int, type_table: TypeTable, device="cuda:0",
                 interval: int = 100, delta_t: int = 5, max_step: Optional[int] = None,
                 any_participant: bool = False, steer_first: bool = False):
        if not torch.cuda.is_available():
            raise RuntimeError("tactics2d_b200 needs a CUDA device: the batched tick only exists as sm_90a kernels")
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("BatchedWorld lives on a CUDA device")
        self.N, self.M = int(n_scenarios), int(m_participants)
        self.type_table = type_table
        self.interval, self.delta_t = int(interval), int(delta_t)
        self.max_step = int(max_step) if max_step else 0
        self.flags_cfg = (CFG_ANY_PARTICIPANT if any_participant else 0) | (CFG_STEER_FIRST if steer_first else 0)
        self._ctx = C.c_void_p()
        dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.dev_index = dev_index
        cfg = _lib.Config(self.interval, self.delta_t, self.max_step, self.flags_cfg)
        _lib.check(self.lib.t2d_create(C.byref(self._ctx), dev_index, self.N, self.M, C.byref(cfg)))
        arr = type_table.to_c_array()
        _lib.check(self.lib.t2d_set_type_table(self._ctx, arr, len(type_table)))

        f = dict(dtype=torch.float32, device=self.device)
        shape = (self.N, self.M)
        self.x = torch.zeros(shape, **f)
        self.y = torch.zeros(shape, **f)
        self.heading = torch.zeros(shape, **f)
        self.speed = torch.zeros(shape, **f)
        self.vx = torch.zeros(shape, **f)
        self.vy = torch.zeros(shape, **f)
        self.type_id = torch.full(shape, TYPE_INACTIVE, dtype=torch.uint8, device=self.device)
        self.step_count = torch.zeros(self.N, dtype=torch.int32, device=self.device)
        self.frame = 0  # ms; State.frame advances by `interval` per step (single_track_kinematics.py:166)
        self._out = StepResult(
            flags=torch.zeros(shape, dtype=torch.uint8, device=self.device),
            hit_index=torch.full(shape, -1, dtype=torch.int16, device=self.device),
            hit_segment=torch.full(shape, -1, dtype=torch.int16, device=self.device),
            status=torch.ones(self.N, dtype=torch.uint8, device=self.device),
            done=torch.zeros(self.N, dtype=torch.uint8, device=self.device))
        self._bind()
        # SingleTrackDrift participants carry their wheel speeds (single_track_drift.py:467-499)
        self.omega_front = self.omega_rear = None
        if any(r.model == MODEL_DRIFT for r in type_table.rows):
            self.omega_front = torch.zeros(shape, **f)
            self.omega_rear = torch.zeros(shape, **f)
            _lib.check(self.lib.t2d_bind_wheel_state(self._ctx, _ptr(self.omega_front), _ptr(self.omega_rear)))
        self.segments = None
        self.poly_start = None
        self.tiles, self.tile_id = None, None
        self.bounds = None
        self.paths = None
        # what the setters bind (None until they are called) and the output buffers made on first use
        self._goal = self._ctrl = self._log = self._agents = self._ego_action = self._routes = self._sampler = None
        self._history, self._hist_out = 0, {}
        self._route_out = {}
        self._leader = self._leader_out = self._lane = self._reactive = self._yield = self._yield_out = None
        self._env = self._npc_action = self._host_out = self._host_agents = self._lidar = self._bev_out = None
        self._agent_lidar, self._obs_out, self._agent_obs_out, self._agent_bev = {}, {}, {}, {}
        self._seg_style_keys = []
        self._bev_cfg = None

    # ------------------------------------------------------------------ plumbing
    def _bind(self):
        _lib.check(self.lib.t2d_bind_state(self._ctx, _ptr(self.x), _ptr(self.y), _ptr(self.heading), _ptr(self.speed),
                                           _ptr(self.vx), _ptr(self.vy), _ptr(self.type_id), _ptr(self.step_count)))

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _device_tensor(self, name: str, t, dtype: torch.dtype, shape) -> torch.Tensor:
        """``t`` itself, after checking that it is a contiguous ``dtype`` tensor of exactly ``shape`` on the world's device.
        Such a tensor reaches the kernels as a raw pointer: a host tensor, another dtype or shape would be read out of
        bounds."""
        if not (torch.is_tensor(t) and t.device == self.device and t.dtype == dtype and t.shape == shape
                and t.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous {dtype} {list(shape)} tensor on {self.device}")
        return t

    @staticmethod
    def _host_tensor(name: str, a, shape) -> torch.Tensor:
        """``a`` as a contiguous fp32 CPU tensor of exactly ``shape``, for the host steps: any array-like is converted to
        float32, a tensor must already be one."""
        t = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
        if not (t.device.type == "cpu" and t.dtype == torch.float32 and t.shape == shape and t.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous float32 host array {list(shape)}")
        return t

    def _to_device(self, a, dtype: torch.dtype, shape) -> torch.Tensor:
        """``a`` (a tensor on any device, or anything array-like) as a contiguous ``dtype`` tensor of ``shape`` on the
        world's device; a copy unless ``a`` is one already."""
        t = (a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))).to(device=self.device, dtype=dtype)
        return (t if t.shape == shape else t.reshape(shape)).contiguous()

    def _put(self, dst: torch.Tensor, src):
        dst.copy_(self._to_device(src, dst.dtype, dst.shape))

    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self.lib.t2d_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ configuration
    def set_config(self, interval=None, delta_t=None, max_step=None):
        if interval is not None:
            self.interval = int(interval)
        if delta_t is not None:
            self.delta_t = int(delta_t)
        if max_step is not None:
            self.max_step = int(max_step)
        cfg = _lib.Config(self.interval, self.delta_t, self.max_step, self.flags_cfg)
        _lib.check(self.lib.t2d_set_config(self._ctx, C.byref(cfg)))

    def set_type_table(self, type_table: TypeTable):
        """Replace the type table.  The map stays as it was built: its dilated cell lists cover the reach of the table
        that was current at ``set_map``, and a participant whose type reaches further takes the slower exhaustive walk.

        Once BEV styles are chosen (``set_bev_styles``, or the first ``bev``), they are pushed again for the new table
        at once: a table with as many rows keeps the per-type styles, any other falls back on ``default_type_style`` of
        its rows; the target keeps its style."""
        from .sensor.camera import default_type_style

        if any(r.model == MODEL_DRIFT for r in type_table.rows) and self.omega_front is None:
            raise ValueError("a SingleTrackDrift row needs a world created with one (its wheel speeds are allocated there)")
        _lib.check(self.lib.t2d_set_type_table(self._ctx, type_table.to_c_array(), len(type_table)))
        self.type_table = type_table
        self._reactive = None   # the library dropped a bound reactive replay
        if self._bev_cfg is not None:
            type_styles, target = self._bev_cfg
            if len(type_styles) != len(type_table):
                self._bev_cfg = ([default_type_style(r) for r in type_table.rows], target)
            self._push_bev_styles()

    def set_map(self, segments=None, bounds: Optional[Sequence[float]] = None, cell_size: float = 0.0, poly_start=None,
                style=None):
        """Static geometry of the scenario (shared by all N scenarios).

        ``segments``: array [S, 4] of (x1, y1, x2, y2) collidable pieces in list order - what
        ``StaticCollision.reset(static_objects)`` receives (collision.py:45-46), flattened;
        ``bounds``: (xmin, xmax, ymin, ymax) as ``Map.boundary`` / ``OutBound.reset`` take it
        (out_bound.py:50-65), or None;
        ``poly_start``: int array [P + 1] marking the segments that close up to ``Area`` polygons (ring p = segments
        [poly_start[p], poly_start[p + 1])): a pose inside a polygon collides with it even when it touches no edge, and
        ``hit_segment`` then names the first object hit by its first segment (see :func:`polygons_to_segments`);
        ``style``: optional BEV style key of every segment (a ring object is drawn in the style of its first segment;
        :func:`tactics2d_b200.map.segment_style_keys`), default ``obstacle`` for rings and ``road_border`` otherwise."""
        seg = None if segments is None else np.ascontiguousarray(np.asarray(segments, dtype=np.float32).reshape(-1, 4))
        n_seg = 0 if seg is None else seg.shape[0]
        b = None if bounds is None else np.ascontiguousarray(np.asarray(bounds, dtype=np.float32))
        ps = None if poly_start is None else np.ascontiguousarray(np.asarray(poly_start, dtype=np.int32))
        n_poly = 0 if ps is None else len(ps) - 1
        _lib.check(self.lib.t2d_set_map_polygons(
            self._ctx, C.c_void_p(0 if n_seg == 0 else seg.ctypes.data), n_seg, C.c_void_p(0 if n_poly <= 0 else ps.ctypes.data),
            max(0, n_poly), C.c_void_p(0 if b is None else b.ctypes.data), float(cell_size)))
        self.segments = seg
        self.poly_start = ps
        self.bounds = None if b is None else tuple(float(v) for v in b)
        self.tiles, self.tile_id = None, None
        self._seg_style_keys = [self._check_style_keys(style, n_seg)]
        self._push_bev_styles()

    def set_map_table(self, tiles, tile_id, cell_size: float = 0.0):
        """A different map per scenario: ``tiles`` is a list of dicts ``{"segments": [S, 4], "bounds": (4,) or None,
        "poly_start": [P + 1] or None, "style": [S] BEV style keys or None}`` (what ``_ParkingScenarioManager.reset`` builds per episode - the lot's wall and
        obstacle Areas and ``map_.boundary``, envs/parking.py:397-441 - or the reference's ``data/*_map`` files, one tile
        each: ``map.polygons_to_segments(map.load_areas(name, subtypes), [lines])``), ``tile_id`` an integer array [N]: the tile of every scenario.  The ids live in ``self.tile_id`` (uint16
        device tensor) and may be rewritten between ticks."""
        keep, rows = [], (_lib.MapTileC * len(tiles))()
        for i, t in enumerate(tiles):
            seg = t.get("segments")
            seg = None if seg is None or len(seg) == 0 else np.ascontiguousarray(np.asarray(seg, dtype=np.float32).reshape(-1, 4))
            b = t.get("bounds")
            b = None if b is None else np.ascontiguousarray(np.asarray(b, dtype=np.float32))
            ps = t.get("poly_start")
            ps = None if ps is None or len(ps) < 2 else np.ascontiguousarray(np.asarray(ps, dtype=np.int32))
            keep.append((seg, b, ps))
            rows[i].segments = None if seg is None else seg.ctypes.data
            rows[i].n_seg = 0 if seg is None else seg.shape[0]
            rows[i].poly_start = None if ps is None else ps.ctypes.data
            rows[i].n_poly = 0 if ps is None else len(ps) - 1
            rows[i].bounds = None if b is None else b.ctypes.data
        tid = torch.as_tensor(np.asarray(tile_id) if not torch.is_tensor(tile_id) else tile_id).to(torch.int64)
        if tid.numel() != self.N or int(tid.min()) < 0 or int(tid.max()) >= len(tiles):
            raise ValueError(f"tile_id must hold {self.N} indices into the {len(tiles)} tiles")
        tid = self._to_device(tid, torch.int16, tid.shape)   # (bit pattern of uint16 for ids < 32768)
        # a rejected table leaves the previous map bound, and with it the previous tile_id tensor
        _lib.check(self.lib.t2d_set_map_table(self._ctx, rows, len(tiles), _ptr(tid), float(cell_size)))
        self.tile_id = tid
        self.tiles = [dict(segments=k[0], bounds=None if k[1] is None else tuple(float(v) for v in k[1]), poly_start=k[2]) for k in keep]
        self.segments, self.poly_start, self.bounds = None, None, None
        self._seg_style_keys = [self._check_style_keys(t.get("style"), 0 if k[0] is None else k[0].shape[0])
                                for t, k in zip(tiles, keep)]
        self._push_bev_styles()

    def set_goal(self, target=None, arrival_threshold: float = 0.95, no_action_max_step: int = 100):
        """Target area per scenario for the ego (participant 0): array [N, 5] = (cx, cy, heading, half_len, half_wid),
        or None to disable.  Enables ``Arrival`` (IoU >= threshold -> COMPLETED, arrival.py:32-47) and ``NoAction``
        (IoU with the previous pose > 0.999 for more than ``no_action_max_step`` ticks, no_action.py:32-53) inside
        ``step``; ``StepResult.iou`` then holds the ego/target IoU."""
        # the library keeps the pointers of the previous goal until a call succeeds: replace the tensors only then
        if target is None:
            _lib.check(self.lib.t2d_set_goal(self._ctx, _ptr(None), 0.95, 0, _ptr(None), _ptr(None), _ptr(None)))
            self._goal = None
            self._out.iou = None
            return
        g = dict(target=self._to_device(target, torch.float32, (self.N, 5)),
                 iou=torch.zeros(self.N, dtype=torch.float32, device=self.device),
                 last_pose=torch.zeros((self.N, 4), dtype=torch.float32, device=self.device),
                 count=torch.zeros(self.N, dtype=torch.int32, device=self.device))
        _lib.check(self.lib.t2d_set_goal(self._ctx, _ptr(g["target"]), float(arrival_threshold), int(no_action_max_step),
                                         _ptr(g["iou"]), _ptr(g["last_pose"]), _ptr(g["count"])))
        self._goal = g
        self._out.iou = g["iou"]

    # ------------------------------------------------------------------ NPC controllers
    def set_paths(self, paths):
        """Pure-pursuit waypoint polylines: a list of ``[V_p, 2]`` arrays (the ``waypoints`` of
        ``PurePursuitController.step``, pure_pursuit_controller.py:76); ``path_id`` of ``set_controllers`` indexes it."""
        paths = [np.ascontiguousarray(np.asarray(p, dtype=np.float32).reshape(-1, 2)) for p in paths]
        if not paths:
            _lib.check(self.lib.t2d_set_paths(self._ctx, _ptr(None), _ptr(None), 0))
        else:
            xy = np.ascontiguousarray(np.concatenate(paths, 0))
            off = np.zeros(len(paths) + 1, np.int32)
            off[1:] = np.cumsum([len(p) for p in paths])
            _lib.check(self.lib.t2d_set_paths(self._ctx, C.c_void_p(xy.ctypes.data), C.c_void_p(off.ctypes.data), len(paths)))
        self.paths = paths
        self._lane = self._reactive = self._yield = None   # the library dropped a bound lane change, reactive replay and yielding

    def set_controllers(self, controllers, ctrl_id, lead_index=None, path_id=None, last_accel=None, pid_target=None,
                        pid_state=None):
        """Hand the non-ego agents to on-device controllers.  ``controllers``: list of ``tactics2d_b200.controller``
        objects (or ``ControllerParamsC`` rows); ``ctrl_id`` [N, M] uint8: the participant's row, 255 for "action comes
        from the caller"; ``lead_index`` [N, M] int16: its leading vehicle (``leading_state`` / ``front_state``), -1 for
        none; ``path_id`` [N, M] int16: its pure-pursuit path or the PID rows' path (``set_paths``), -1 for none;
        ``last_accel`` [N, M]: ``State.accel`` of the previous tick (default zeros).  ``None`` for ``controllers``
        removes them, and any call drops a bound lane change (``set_lane_change``).  An ``IDMController(lateral=...)``
        row keeps its lane: it steers along its path with a PID lateral channel, on ``pid_state``.  While a leader search is bound (``set_leader_search``), ``control`` ignores ``lead_index`` and
        every controller follows the leader the search finds on the same state in the same call.

        PID rows (``PIDController``): ``pid_target`` [N, M, 2] = (target_speed, target_heading or cross_track_error),
        fp32, read every tick (write new targets into ``self.pid_target`` in place).  Their memory is ``self.pid_state``,
        fp64 [N, M, 6] = (lat_integral, lat_prev_error, lat_prev_derivative, lon_integral, lon_prev_error,
        lon_prev_derivative): a fresh zeroed tensor, or ``pid_state`` when given; ``reset`` zeroes the rows of the
        reset scenarios."""
        if controllers is None:
            _lib.check(self.lib.t2d_set_controllers(self._ctx, _ptr(None), 0, _ptr(None), _ptr(None), _ptr(None), _ptr(None)))
            _lib.check(self.lib.t2d_set_pid(self._ctx, _ptr(None), _ptr(None)))
            self._ctrl = self._lane = self._reactive = self._yield = None
            return
        rows = [c if isinstance(c, _lib.ControllerParamsC) else c.params() for c in controllers]
        arr = (_lib.ControllerParamsC * len(rows))(*rows)
        NM = (self.N, self.M)
        dev = lambda a, dtype: None if a is None else self._to_device(a, dtype, NM)
        cid, lead, pid = dev(ctrl_id, torch.uint8), dev(lead_index, torch.int16), dev(path_id, torch.int16)
        la = dev(last_accel, torch.float32)
        if la is None:
            la = torch.zeros(NM, dtype=torch.float32, device=self.device)
        from .controller.controller_base import CTRL_IDM, CTRL_PID, PID_LAT_NONE

        tgt, st = None, None
        # PID rows and IDM rows with a lateral channel (lane keeping) keep their PID memory in pid_state
        if any(r.kind == CTRL_PID or (r.kind == CTRL_IDM and r.pid_lateral != PID_LAT_NONE) for r in rows):
            if pid_target is not None:
                tgt = self._to_device(pid_target, torch.float32, NM + (2,))
            if pid_state is None:
                st = torch.zeros(NM + (6,), dtype=torch.float64, device=self.device)
            else:
                st = self._device_tensor("pid_state", pid_state, torch.float64, NM + (6,))
        # the controllers first: a rejected table leaves the previous binding, PID arrays included, as it was
        _lib.check(self.lib.t2d_set_controllers(self._ctx, arr, len(rows), _ptr(cid), _ptr(lead), _ptr(pid), _ptr(la)))
        _lib.check(self.lib.t2d_set_pid(self._ctx, _ptr(tgt), _ptr(st)))
        self._ctrl = dict(rows=arr, ctrl_id=cid, lead_index=lead, path_id=pid, last_accel=la, pid_target=tgt, pid_state=st)
        self._lane = self._reactive = self._yield = None   # the library dropped a bound lane change, reactive replay and yielding

    @property
    def last_accel(self) -> Optional[torch.Tensor]:
        return None if self._ctrl is None else self._ctrl["last_accel"]

    @property
    def pid_target(self) -> Optional[torch.Tensor]:
        return None if self._ctrl is None else self._ctrl["pid_target"]

    @property
    def pid_state(self) -> Optional[torch.Tensor]:
        return None if self._ctrl is None else self._ctrl["pid_state"]

    def control(self, action: torch.Tensor) -> torch.Tensor:
        """Fill the rows of ``action`` [N, M, 2] that belong to controlled participants (IN PLACE; the other rows keep
        the caller's values) and refresh ``last_accel`` - ``ControllerBase.step`` of every NPC in one launch.  Call it
        after writing the external (ego) actions and before ``step``."""
        self._device_tensor("action", action, torch.float32, (self.N, self.M, 2))
        _lib.check(self.lib.t2d_control(self._ctx, _ptr(action), self._stream()))
        return action

    # ------------------------------------------------------------------ leader search
    def set_leader_search(self, half_width: Optional[float] = 1.8, max_range: float = 100.0):
        """Find every slot's leader on the device in front of every ``control`` (``t2d_set_leader_search``, K17; DESIGN.md
        section 1 "Leader search"): the nearest participant ahead within ``half_width`` metres of the slot's corridor and
        at most ``max_range`` metres ahead - along the slot's controller path when it has one, else along its heading.
        The controllers then follow these leaders instead of ``lead_index``, so the traffic reacts to every cut-in, reset,
        replayed track and retirement.  The leaders of the last ``control`` are in :attr:`leader` (int16 [N, M], -1 for
        none) and :attr:`leader_gap` (fp32 [N, M], +inf for none).  ``half_width=None`` unbinds, and drops a bound lane
        change.  A rejected call keeps the previous search."""
        if half_width is None:
            _lib.check(self.lib.t2d_set_leader_search(self._ctx, 0.0, 0.0, _ptr(None), _ptr(None)))
            # unbinding the search drops a bound lane change, reactive replay and yielding
            self._leader = self._lane = self._reactive = self._yield = None
            return
        lead = torch.full((self.N, self.M), -1, dtype=torch.int16, device=self.device)
        gap = torch.full((self.N, self.M), float("inf"), dtype=torch.float32, device=self.device)
        _lib.check(self.lib.t2d_set_leader_search(self._ctx, float(half_width), float(max_range), _ptr(lead), _ptr(gap)))
        self._leader = dict(lead=lead, gap=gap, half_width=float(half_width), max_range=float(max_range))

    @property
    def leader(self) -> Optional[torch.Tensor]:
        """int16 [N, M] device tensor: the leaders the bound search found in the last ``control`` (None without one)."""
        return None if self._leader is None else self._leader["lead"]

    @property
    def leader_gap(self) -> Optional[torch.Tensor]:
        """fp32 [N, M] device tensor: the gap to each of those leaders, +inf where there is none."""
        return None if self._leader is None else self._leader["gap"]

    def find_leaders(self, half_width: float = 1.8, max_range: float = 100.0):
        """The leaders of the current state in one launch (``t2d_find_leaders``, K17), with or without a bound search:
        ``(lead, gap)``, int16 and fp32 [N, M] as :attr:`leader` / :attr:`leader_gap`.  The tensors are buffers the next
        call reuses."""
        if self._leader_out is None:
            self._leader_out = (torch.empty((self.N, self.M), dtype=torch.int16, device=self.device),
                                torch.empty((self.N, self.M), dtype=torch.float32, device=self.device))
        lead, gap = self._leader_out
        _lib.check(self.lib.t2d_find_leaders(self._ctx, float(half_width), float(max_range), _ptr(lead), _ptr(gap),
                                             self._stream()))
        return lead, gap

    # ------------------------------------------------------------------ lane changes
    def set_lane_change(self, left, right=None, politeness: float = 0.0, threshold: float = 0.2, b_safe: float = 2.0,
                        min_gap: float = 6.0, cooldown: int = 10):
        """MOBIL lane changes on the device in front of every ``control`` (``t2d_set_lane_change``, K18; DESIGN.md section 1
        "Lane changes").  ``left`` / ``right``: the left and right neighbour of every path of ``set_paths``, -1 for none.
        Every IDM row with a lateral channel (``IDMController(lateral=...)``) that is on its current lane and out of its
        cooldown moves to a neighbour when that gains it more than ``threshold`` m/s^2 (its followers' gains weighted by
        ``politeness``), no car is within ``min_gap`` metres along the target lane, and the new follower brakes no harder
        than ``b_safe``; it then waits ``cooldown`` ticks.  Needs the controllers (with ``path_id``), the paths and a
        leader search, whose corridor it uses.  The current lanes are in :attr:`lane_path` (from ``path_id`` at binding and
        at every reset), the last decisions in :attr:`lane_change` (+1 left, -1 right, 0) and the cooldowns in
        :attr:`lane_cooldown`.  ``left=None`` unbinds; ``set_controllers``, ``set_paths`` and unbinding the search drop it.
        A rejected call keeps the previous binding."""
        if left is None:
            _lib.check(self.lib.t2d_set_lane_change(self._ctx, None, None, None, None, None, None))
            self._lane = None
            return
        n_paths = 0 if self.paths is None else len(self.paths)
        nb = []
        for name, a in (("left", left), ("right", right)):
            a = np.ascontiguousarray(np.asarray(a, dtype=np.int64).reshape(-1))
            if a.shape != (n_paths,) or (a < -32768).any() or (a > 32767).any():   # the library checks the entries
                raise ValueError(f"{name} must hold one int16 neighbour per path of set_paths ({n_paths})")
            nb.append(np.ascontiguousarray(a.astype(np.int16)))
        p = _lib.LaneChangeParamsC(politeness=float(politeness), threshold=float(threshold), b_safe=float(b_safe),
                                   min_gap=float(min_gap), cooldown=int(cooldown))
        NM = (self.N, self.M)
        lane_path = torch.full(NM, -1, dtype=torch.int16, device=self.device)
        cool = torch.zeros(NM, dtype=torch.int16, device=self.device)
        change = torch.zeros(NM, dtype=torch.int8, device=self.device)
        _lib.check(self.lib.t2d_set_lane_change(self._ctx, C.byref(p), C.c_void_p(nb[0].ctypes.data),
                                                C.c_void_p(nb[1].ctypes.data), _ptr(lane_path), _ptr(cool), _ptr(change)))
        self._lane = dict(params=p, left=nb[0], right=nb[1], lane_path=lane_path, cooldown=cool, change=change)

    @property
    def lane_path(self) -> Optional[torch.Tensor]:
        """int16 [N, M] device tensor: every slot's current path while a lane change is bound (None without one)."""
        return None if self._lane is None else self._lane["lane_path"]

    @property
    def lane_change(self) -> Optional[torch.Tensor]:
        """int8 [N, M] device tensor: the decisions of the last ``control``, +1 left, -1 right, 0 none."""
        return None if self._lane is None else self._lane["change"]

    @property
    def lane_cooldown(self) -> Optional[torch.Tensor]:
        """int16 [N, M] device tensor: the ticks each slot still waits before it may change lanes again."""
        return None if self._lane is None else self._lane["cooldown"]

    # ------------------------------------------------------------------ yielding at conflict zones
    def set_yielding(self, priority=None, width: float = 2.0, margin: float = 3.0, critical_gap: float = 3.0,
                     commit_decel: float = 3.0, v_min: float = 0.5):
        """Yield at crossing and merging paths on the device in front of every ``control`` (``t2d_set_yielding``, K19;
        DESIGN.md section 1 "Yielding at conflict zones").  The conflict zones of the bound ``set_paths`` table are built
        once here (:func:`tactics2d_b200.traffic.conflicts.conflict_zones` with ``width`` and ``margin``).
        Every IDM row on a path then stops ``margin`` metres before a zone, as behind a standing leader, while a car on the
        other path is inside it or committed to it (it cannot stop at ``commit_decel`` m/s^2), or reaches it within
        ``critical_gap`` seconds (at its speed, at least ``v_min``) with a higher path ``priority`` (int16 per path,
        default all 0), or with an equal one and nearer its own zone.  A car already committed itself never yields.  The
        yields of the last ``control`` are in :attr:`yield_to` (int16 [N, M], the slot yielded to, -1 for none) and
        :attr:`stop_gap` (fp32 [N, M], the arc length to the stop, +inf for none).  Needs the controllers, the paths and a
        leader search, whose corridor and range it uses; ``set_paths``, ``set_controllers`` and unbinding the search drop
        it, and so does :meth:`unset_yielding`.  A rejected call keeps the previous binding."""
        from .traffic.conflicts import conflict_zones

        n_paths = 0 if self.paths is None else len(self.paths)
        zones = conflict_zones(self.paths or [], width, margin)
        rows = np.zeros(len(zones), _lib.ZONE_DTYPE)
        for k in ("q", "s_in_p", "s_out_p", "s_in_q", "s_out_q"):
            rows[k] = getattr(zones, k)
        off = np.ascontiguousarray(zones.zone_off, np.int32)
        prio = None
        if priority is not None:
            prio = np.asarray(priority, np.int64).reshape(-1)
            if prio.shape != (n_paths,) or (prio < -32768).any() or (prio > 32767).any():
                raise ValueError(f"priority must hold one int16 per path of set_paths ({n_paths})")
            prio = np.ascontiguousarray(prio.astype(np.int16))
        p = _lib.YieldParamsC(critical_gap=float(critical_gap), commit_decel=float(commit_decel), v_min=float(v_min))
        NM = (self.N, self.M)
        yield_to = torch.full(NM, -1, dtype=torch.int16, device=self.device)
        stop_gap = torch.full(NM, float("inf"), dtype=torch.float32, device=self.device)
        host = lambda a: None if a is None or a.size == 0 else C.c_void_p(a.ctypes.data)
        _lib.check(self.lib.t2d_set_yielding(self._ctx, C.byref(p), host(rows), host(off), host(prio), _ptr(yield_to),
                                             _ptr(stop_gap)))
        self._yield = dict(params=p, zones=zones, priority=prio, yield_to=yield_to, stop_gap=stop_gap)

    def unset_yielding(self):
        """Unbind yielding: ``control`` launches K19 no more and K5 runs its other instances."""
        _lib.check(self.lib.t2d_set_yielding(self._ctx, None, None, None, None, None, None))
        self._yield = None

    @property
    def conflict_zones(self):
        """The :class:`~tactics2d_b200.traffic.conflicts.ConflictZones` of the bound yielding (None without one)."""
        return None if self._yield is None else self._yield["zones"]

    @property
    def yield_to(self) -> Optional[torch.Tensor]:
        """int16 [N, M] device tensor: the slot each car yielded to in the last ``control``, -1 for none (None when
        yielding is not bound)."""
        return None if self._yield is None else self._yield["yield_to"]

    @property
    def stop_gap(self) -> Optional[torch.Tensor]:
        """fp32 [N, M] device tensor: the arc length from each yielding car to its stop, +inf where it does not yield."""
        return None if self._yield is None else self._yield["stop_gap"]

    def find_yields(self):
        """The yields of the current state in one launch (``t2d_find_yields``, K19) with the bound yielding:
        ``(yield_to, stop_gap)`` as :attr:`yield_to` / :attr:`stop_gap`.  The tensors are buffers the next call reuses."""
        if self._yield_out is None:
            self._yield_out = (torch.empty((self.N, self.M), dtype=torch.int16, device=self.device),
                               torch.empty((self.N, self.M), dtype=torch.float32, device=self.device))
        yt, sg = self._yield_out
        _lib.check(self.lib.t2d_find_yields(self._ctx, _ptr(yt), _ptr(sg), self._stream()))
        return yt, sg

    # ------------------------------------------------------------------ route following
    def set_routes(self, route_id, threshold: float = None, progress_weight: float = 0.1, off_route_reward: float = -5.0):
        """Give slots a route to follow (``t2d_set_routes``; DESIGN.md section 1 "Route following"): ``route_id`` [N, M]
        indexes the ``set_paths`` table (the one the controllers' ``path_id`` indexes), -1 for none; it is kept as the int16
        device tensor :attr:`route_id`, which may be rewritten between steps.  Every scored participant with a route - the
        ego in ``env_epilogue``, every agent row in ``agents_epilogue`` - is off route (``OffRoute``, off_route.py:24-35)
        when its centre is more than ``threshold`` metres from the route: traffic status OFF_ROUTE, truncated, reward
        ``off_route_reward`` (an extension; default -5, the out-of-bound penalty).  A NORMAL step on the route adds
        ``progress_weight`` x the gain of arc length over the episode's best (default 0.1, the weight of the progress
        towards a target; :attr:`route_s_best` / :attr:`agent_route_s_best` hold the best, fp64).  None unbinds."""
        if route_id is None:
            _lib.check(self.lib.t2d_set_routes(self._ctx, _ptr(None), 0.0, 0.0, 0.0))
            _lib.check(self.lib.t2d_bind_route_trackers(self._ctx, _ptr(None), _ptr(None), 0))
            self._routes = None
            return
        if threshold is None:
            raise ValueError("set_routes needs the OffRoute threshold (metres)")
        if (route_id.numel() if torch.is_tensor(route_id) else np.size(route_id)) != self.N * self.M:
            raise ValueError(f"route_id must hold [{self.N}, {self.M}] path indices")
        rid = self._to_device(route_id, torch.int16, (self.N, self.M))
        # the library keeps the previous routes until a call succeeds: replace the tensors only then
        _lib.check(self.lib.t2d_set_routes(self._ctx, _ptr(rid), float(threshold), float(progress_weight),
                                           float(off_route_reward)))
        self._routes = dict(route_id=rid, threshold=float(threshold), progress_weight=float(progress_weight),
                            off_route_reward=float(off_route_reward),
                            s_best=torch.full((self.N,), -float("inf"), dtype=torch.float64, device=self.device),
                            agent_s_best=None)
        self._bind_route_trackers()

    def _bind_route_trackers(self):
        """(Re)bind the progress trackers: [N] for the ego, [N, Q] for the bound agents' rows."""
        r = self._routes
        if r is None:
            return
        Q = 0 if self._agents is None else self._agents["Q"]
        if Q and (r["agent_s_best"] is None or r["agent_s_best"].shape[1] != Q):
            r["agent_s_best"] = torch.full((self.N, Q), -float("inf"), dtype=torch.float64, device=self.device)
        if not Q:
            r["agent_s_best"] = None
        _lib.check(self.lib.t2d_bind_route_trackers(self._ctx, _ptr(r["s_best"]), _ptr(r["agent_s_best"]), Q))

    @property
    def route_id(self) -> Optional[torch.Tensor]:
        """int16 [N, M] device tensor: the route of every slot (None without routes)."""
        return None if self._routes is None else self._routes["route_id"]

    @property
    def route_s_best(self) -> Optional[torch.Tensor]:
        """fp64 [N] device tensor: the ego's best arc length on its route this episode (-inf before its first step)."""
        return None if self._routes is None else self._routes["s_best"]

    @property
    def agent_route_s_best(self) -> Optional[torch.Tensor]:
        """fp64 [N, Q] device tensor: every agent row's best arc length on its slot's route (None without agents)."""
        return None if self._routes is None else self._routes["agent_s_best"]

    def route_observe(self, n_points: int = 8, spacing: float = 2.0, observers: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The route of each observer in its own frame, in one launch (``t2d_route_observe``, K12): fp32 rows of
        :data:`ROUTE_FIELDS` (has_route, signed lateral offset - positive when the route lies to the left -, heading error
        to the closest segment in (-pi, pi], s / L, L - s) followed by ``n_points`` look-ahead points (x, y) at arc length
        ``min(s + k spacing, L)``, k = 1..n_points.  ``observers=None``: the ego of every scenario, ``[N, F]``; an int16
        ``[N, Q]`` device tensor as in ``observe_agents``: ``[N, Q, F]``.  Rows without a route, or whose observer is out
        of range, empty or retired, are zeros.  The tensor is a buffer the next call with the same shape reuses."""
        P = int(n_points)
        if not 0 <= P <= ROUTE_MAX_POINTS:
            raise ValueError(f"n_points must be in 0..{ROUTE_MAX_POINTS}")
        F = len(ROUTE_FIELDS) + 2 * P
        Q = 1 if observers is None else self._agent_rows(observers, None)
        key = (F, None if observers is None else Q)
        out = self._route_out.get(key)
        if out is None:
            out = self._route_out[key] = torch.empty((self.N, F) if observers is None else (self.N, Q, F),
                                                     dtype=torch.float32, device=self.device)
        _lib.check(self.lib.t2d_route_observe(self._ctx, _ptr(observers), Q, P, float(spacing), _ptr(out), self._stream()))
        return out

    # ------------------------------------------------------------------ trajectory history
    def set_history(self, length: int):
        """Keep the last ``length`` (1..64) states of every slot on the device (``t2d_set_history``; DESIGN.md section 1
        "Trajectory history"; ``Trajectory.add_state`` / ``Trajectory.reset(state)``, trajectory.py:115-149,170-188): every
        step appends the state after its tick, every ``reset`` / ``reset_sampled`` starts the reset scenarios' histories
        again from the state it leaves.  ``set_state``, ``check_events`` and the observations leave the ring alone.  A new
        binding is empty; 0 frees the ring.  A rejected call keeps the previous ring.  It costs N M length 25 bytes (4 more
        per entry with a log schedule)."""
        n = int(length)
        if not 0 <= n <= HISTORY_MAX:
            raise ValueError(f"history length must be in 0..{HISTORY_MAX}")
        _lib.check(self.lib.t2d_set_history(self._ctx, n))
        self._history, self._hist_out = n, {}

    @property
    def history_length(self) -> int:
        """H of the bound history ring, 0 without one."""
        return self._history

    def observe_history(self, agent_index: Optional[torch.Tensor] = None,
                        observers: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The recent past of each observer and of its agents in the observer's CURRENT frame, in one launch
        (``t2d_observe_history``, K16): fp32 ``[..., 1 + K, H, 7]`` of :data:`HIST_FIELDS`, block 0 the observer itself and
        block 1 + k the slot ``agent_index[..., k]``, lag 0 (the newest entry) first; an invalid entry, an absent agent and
        an absent observer give zeros.  Without ``observers`` and with ``agent_index`` None or int16 ``[N, K]`` (what
        ``observe`` returns) the rows are the egos': ``[N, 1 + K, H, 7]``.  With ``observers`` (int16 ``[N, Q]``, as in
        ``observe_agents``) or an ``agent_index`` of ``[N, Q, K]`` (what ``observe_agents`` returns; without ``observers``
        row q is slot q) there is a row per observer: ``[N, Q, 1 + K, H, 7]``.  ``agent_index=None`` is K = 0.  At lag 0,
        while the newest entry is the current state, block 1 + k equals fields 1..6 of the observation's agent row k.  The
        tensor is a buffer the next call with the same shape reuses."""
        if not self._history:
            raise RuntimeError("call set_history before observe_history")
        per_row = observers is not None or (agent_index is not None and torch.is_tensor(agent_index) and agent_index.dim() == 3)
        if per_row:
            if observers is not None:
                Q = self._agent_rows(observers, None)
            else:
                Q = int(agent_index.shape[1])
                if not 1 <= Q <= min(128, self.M):
                    raise ValueError("without observers the agent_index rows are slots: Q must be in 1..min(128, M)")
            lead = (self.N, Q)
        else:
            Q, lead = 0, (self.N,)
        K = 0
        if agent_index is not None:
            if not (torch.is_tensor(agent_index) and agent_index.dim() == len(lead) + 1):
                raise ValueError(f"agent_index must be a contiguous int16 {list(lead) + ['K']} tensor on {self.device}")
            K = int(agent_index.shape[-1])
            if not 0 <= K <= 127:
                raise ValueError("agent_index may name 0..127 agents per row")
            self._device_tensor("agent_index", agent_index, torch.int16, lead + (K,))
        shape = lead + (1 + K, self._history, len(HIST_FIELDS))
        out = self._hist_out.get(shape)
        if out is None:
            out = self._hist_out[shape] = torch.empty(shape, dtype=torch.float32, device=self.device)
        _lib.check(self.lib.t2d_observe_history(self._ctx, _ptr(observers), Q, _ptr(agent_index if K else None), K, _ptr(out),
                                                self._stream()))
        return out

    def _history_ring(self) -> dict:
        """The library's ring as device tensors (views, no copy): x ... vy [N, H, M], type_id, track (or None), count [N]."""
        v = _lib.HistoryRingC()
        _lib.check(self.lib.t2d_history_view(self._ctx, C.byref(v)))
        if v.length == 0:
            raise RuntimeError("no history bound: call set_history first")
        shape = (self.N, v.length, self.M)
        view = lambda ptr, typestr, shp=shape: torch.as_tensor(_DeviceArray(ptr, shp, typestr), device=self.device)
        ring = {k: view(getattr(v, k), "<f4") for k in ("x", "y", "heading", "speed", "vx", "vy")}
        ring["type_id"] = view(v.type_id, "|u1")
        ring["track"] = None if not v.track else view(v.track, "<i4")
        ring["count"] = view(v.count, "<i8", (self.N,))
        return ring

    def history(self) -> dict:
        """Read back the ring (a utility; eager torch): ``x, y, heading, speed, vx, vy`` fp32 and ``type_id`` uint8, each
        ``[N, M, H]`` with lag 0 (the newest entry) first, ``valid`` bool ``[N, M, H]`` (DESIGN.md section 1 "Trajectory
        history": one of the last min(count, H) entries, recorded with the slot's current type - and, with a schedule, its
        current track), zeros (type 255) where not valid, and ``count`` int64 ``[N]``, the entries since each scenario's
        episode began.  Every tensor is a copy."""
        ring = self._history_ring()
        N, M, H = self.N, self.M, self._history
        count = ring["count"].clone()
        lag = torch.arange(H, device=self.device)
        idx = torch.remainder(count[:, None] - 1 - lag[None, :], H)                 # [N, H] ring index of every lag
        recent = lag[None, :] < torch.clamp(count, max=H)[:, None]                  # [N, H]
        pick = lambda a: torch.gather(a, 1, idx[:, :, None].expand(N, H, M)).permute(0, 2, 1).contiguous()
        tid = pick(ring["type_id"])
        valid = recent[:, None, :] & (tid == self.type_id[:, :, None]) & (tid.to(torch.int64) < len(self.type_table))
        if ring["track"] is not None:
            valid &= pick(ring["track"]) == self.replay_track[:, :, None]
        out = {k: torch.where(valid, pick(ring[k]), torch.zeros((), device=self.device))
               for k in ("x", "y", "heading", "speed", "vx", "vy")}
        out["type_id"] = torch.where(valid, tid, torch.full((), TYPE_INACTIVE, dtype=torch.uint8, device=self.device))
        out["valid"], out["count"] = valid, count
        return out

    def trajectory(self, n: int, m: int):
        """Slot m of scenario n's valid history as the reference's ``Trajectory`` of ``State`` objects, oldest first; the
        frame of entry e (counted from the episode's first state) is e x ``interval``."""
        from .participant.trajectory import State, Trajectory

        h = self.history()
        n, m = int(n), int(m)
        if not (0 <= n < self.N and 0 <= m < self.M):
            raise IndexError(f"slot ({n}, {m}) outside the [{self.N}, {self.M}] world")
        cols = {k: h[k][n, m].cpu().numpy() for k in ("x", "y", "heading", "speed", "vx", "vy")}
        valid = h["valid"][n, m].cpu().numpy()
        count = int(h["count"][n])
        traj = Trajectory((n, m), fps=1000.0 / self.interval)
        for lag in range(self._history - 1, -1, -1):
            if valid[lag]:
                c = {k: float(v[lag]) for k, v in cols.items()}
                traj.add_state(State(frame=(count - 1 - lag) * self.interval, x=c["x"], y=c["y"], heading=c["heading"],
                                     vx=c["vx"], vy=c["vy"], speed=c["speed"]))
        return traj

    # ------------------------------------------------------------------ log replay
    def set_log(self, log, t0=None, row_track=None, schedule=None):
        """Replay recorded tracks in the slots bound to them (``t2d_set_log``; DESIGN.md section 1 "Log replay").  ``log``:
        a :class:`tactics2d_b200.dataset_parser.ReplayLog` (or any object with ``first_ms, n_frames, period_ms, type_row``
        [K] and ``records`` [F, 5]) whose type rows are static rows of this world's table, or None to unbind; ``t0`` [P]:
        the start time (ms) of every episode row; exactly one of ``row_track`` [P, M]: the track each slot of a row
        replays, -1 for none, and ``schedule = (slot_off, slot_track)``: slot m of row p replays the tracks
        ``slot_track[slot_off[p * M + m] : slot_off[p * M + m + 1]]`` one after the other (``t2d_set_log_schedule``; their
        presence intervals strictly increasing and disjoint), and :attr:`replay_track` then shows which one each slot holds.
        Before every tick, scenario n's replayed slots take their tracks' state at ``t0[log_row[n]] + (step + 1) *
        interval``; ``reset`` sets ``log_row`` from its ``pool_index`` (pool row p = episode row p) and shows the new row's
        traffic at once.  Replayed slots are checked like any participant; an env over a log keeps the default ego-only
        status (``any_participant=False``)."""
        if log is None:
            _lib.check(self.lib.t2d_set_log(self._ctx, None))
            self._log = self._reactive = None
            return
        if (row_track is None) == (schedule is None):
            raise ValueError("give exactly one of row_track and schedule")
        i32 = lambda a: np.ascontiguousarray(np.asarray(a), dtype=np.int32)
        keep = dict(first=i32(log.first_ms), n_frames=i32(log.n_frames), period=i32(log.period_ms),
                    type_row=np.ascontiguousarray(np.asarray(log.type_row), dtype=np.uint8),
                    records=np.ascontiguousarray(np.asarray(log.records), dtype=np.float32).reshape(-1, 5),
                    t0=i32(t0).reshape(-1), row_track=None if row_track is None else i32(row_track))
        n_rows = keep["t0"].shape[0]
        if row_track is not None and keep["row_track"].shape != (n_rows, self.M):
            raise ValueError(f"row_track must be [{n_rows}, {self.M}] (one row per t0)")
        if schedule is not None:
            keep["slot_off"], keep["slot_track"] = i32(schedule[0]).reshape(-1), i32(schedule[1]).reshape(-1)
            if keep["slot_off"].shape[0] != n_rows * self.M + 1:
                raise ValueError(f"slot_off must hold n_rows * M + 1 = {n_rows * self.M + 1} offsets")
        k = keep["first"].shape[0]
        if not (keep["n_frames"].shape == keep["period"].shape == keep["type_row"].shape == (k,)):
            raise ValueError("first_ms, n_frames, period_ms and type_row need one entry per track")
        if keep["records"].shape[0] != int(keep["n_frames"].astype(np.int64).sum()):
            raise ValueError("records must hold sum(n_frames) rows")
        log_row = torch.arange(self.N, dtype=torch.int32, device=self.device)
        c = self._log_struct(keep, log_row, self.type_id)
        if schedule is None:
            _lib.check(self.lib.t2d_set_log(self._ctx, C.byref(c)))
            track = None
        else:
            track = torch.full((self.N, self.M), -1, dtype=torch.int32, device=self.device)
            p = lambda a: C.c_void_p(a.ctypes.data)
            _lib.check(self.lib.t2d_set_log_schedule(self._ctx, C.byref(c), p(keep["slot_off"]), p(keep["slot_track"]),
                                                     int(keep["slot_track"].shape[0]), _ptr(track)))
        self._log = dict(keep, log_row=log_row, track=track)
        self._reactive = None   # the library dropped a bound reactive replay

    def set_reactive_replay(self, track_path, drive_row=None, desired_speed=None, path_base: int = 0):
        """Let the bound log's reactive tracks react (``t2d_set_log_reactive``; DESIGN.md section 1 "Reactive replay").
        ``track_path`` [K]: the path of every track of the log, -1 for plain replay (``ReplayLog.track_paths``); an entry
        p >= 0 names path ``path_base + p`` of ``set_paths``.  A reactive track is posed from its log at its first sample
        (its handover: the first one after it enters, or the reset), and from then on drives: its slot takes
        ``drive_row[k]`` (default: the non-static row whose static twin is the track's row, ``TypeTable.with_static_twins``),
        the controllers follow :attr:`drive_path` instead of ``path_id``, and the IDM rows take ``desired_speed[k]``
        (default: the track's highest logged speed) from :attr:`slot_desired_speed`.  It leaves at its last stamp, wherever
        it is.  Give the replayed slots an ``IDMController(lateral=PIDController(lateral_error="path_cross_track"))`` row
        first; a leader search, the paths and the log must be bound, no lane change.  The binding takes effect at the next
        ``reset``.  ``track_path=None`` unbinds; ``set_log``, ``set_paths``, ``set_controllers``, ``set_type_table`` and
        unbinding the search drop it.  A rejected call keeps the previous binding."""
        if track_path is None:
            _lib.check(self.lib.t2d_set_log_reactive(self._ctx, None))
            self._reactive = None
            return
        if self._log is None:
            raise ValueError("set_reactive_replay needs a log: call set_log first")
        K = self._log["first"].shape[0]
        tp = np.asarray(track_path, np.int64).reshape(-1)
        if tp.shape != (K,):
            raise ValueError(f"track_path must hold one entry per track of the log ({K})")
        tp = np.where(tp >= 0, tp + int(path_base), -1)
        if (tp > 32767).any():
            raise ValueError("track_path + path_base must fit int16")
        tp = np.ascontiguousarray(tp.astype(np.int16))
        if drive_row is None:
            drive_row = self._class_rows(self._log["type_row"])
        dr = np.asarray(drive_row, np.int64).reshape(-1)
        if dr.shape != (K,) or (dr < 0).any() or (dr > 255).any():
            raise ValueError(f"drive_row must hold one uint8 type row per track ({K})")
        dr = np.ascontiguousarray(dr.astype(np.uint8))
        if desired_speed is None:
            v = self._log["records"].astype(np.float64)
            speed = np.sqrt(v[:, 3] * v[:, 3] + v[:, 4] * v[:, 4])
            bounds = np.concatenate([[0], np.cumsum(self._log["n_frames"].astype(np.int64))])
            desired_speed = [speed[a:b].max() for a, b in zip(bounds[:-1], bounds[1:])]
        ds = np.ascontiguousarray(np.asarray(desired_speed, np.float32).reshape(-1))
        if ds.shape != (K,):
            raise ValueError(f"desired_speed must hold one entry per track ({K})")
        NM = (self.N, self.M)
        drive_path = torch.full(NM, -1, dtype=torch.int16, device=self.device)
        sds = torch.zeros(NM, dtype=torch.float32, device=self.device)
        p = lambda a: C.c_void_p(a.ctypes.data)
        c = _lib.ReactiveReplayC(K, p(tp), p(dr), p(ds), _ptr(drive_path), _ptr(sds))
        _lib.check(self.lib.t2d_set_log_reactive(self._ctx, C.byref(c)))
        self._reactive = dict(track_path=tp, drive_row=dr, desired_speed=ds, drive_path=drive_path,
                              slot_desired_speed=sds)

    def _class_rows(self, type_row):
        """For every static row of ``type_row``, the non-static row it is the twin of (``TypeTable.with_static_twins``)."""
        rows = self.type_table.rows
        out = []
        for r in np.asarray(type_row, np.int64):
            hit = [i for i, q in enumerate(rows) if q.model != MODEL_STATIC and replace(q, model=MODEL_STATIC) == rows[r]]
            if not hit:
                raise ValueError(f"type row {int(r)} is the static twin of no row of the table: pass drive_row")
            out.append(hit[0])
        return out

    @property
    def drive_path(self) -> Optional[torch.Tensor]:
        """int16 [N, M] device tensor: the path every slot showing a reactive track drives along, -1 elsewhere (None
        without a reactive replay).  Every replay rewrites the slots it samples."""
        return None if self._reactive is None else self._reactive["drive_path"]

    @property
    def slot_desired_speed(self) -> Optional[torch.Tensor]:
        """fp32 [N, M] device tensor: the IDM desired speed of every slot showing a reactive track."""
        return None if self._reactive is None else self._reactive["slot_desired_speed"]

    @property
    def reactive(self) -> Optional[torch.Tensor]:
        """bool [N, M] device tensor: the slots that show a reactive track, from its handover to its exit (None without
        a reactive replay)."""
        return None if self._reactive is None else self._reactive["drive_path"] >= 0

    def _log_struct(self, keep, log_row, type_id):
        p = lambda a: C.c_void_p(a.ctypes.data)
        rt = keep.get("row_track")
        return _lib.LogC(keep["first"].shape[0], p(keep["first"]), p(keep["n_frames"]), p(keep["period"]), p(keep["type_row"]),
                         p(keep["records"]), keep["t0"].shape[0], p(keep["t0"]), None if rt is None else p(rt), _ptr(log_row),
                         _ptr(type_id))

    @property
    def replay_track(self) -> Optional[torch.Tensor]:
        """int32 [N, M] device tensor: the track each slot shows, -1 while it shows none or is not replayed (None unless a
        log is bound with a ``schedule``).  Every replay - each tick and each reset of a scenario - rewrites its slots."""
        return None if self._log is None else self._log["track"]

    @property
    def log_row(self) -> Optional[torch.Tensor]:
        """int32 [N] device tensor: the episode row every scenario runs (None without a log).  ``reset`` writes it; it may
        be rewritten between ticks."""
        return None if self._log is None else self._log["log_row"]

    # ------------------------------------------------------------------ state
    def set_wheel_state(self, omega_front, omega_rear):
        """Wheel angular speeds [N, M] of the SingleTrackDrift participants (``omega_wf`` / ``omega_wr``)."""
        if self.omega_front is None:
            raise ValueError("the type table holds no SingleTrackDrift row")
        self._put(self.omega_front, omega_front)
        self._put(self.omega_rear, omega_rear)

    def set_state(self, x, y, heading, speed=None, vx=None, vy=None, type_id=None):
        """Copy host or device arrays [N, M] into the SoA state.  Missing ``vx, vy`` are derived as
        ``State.velocity`` does (state.py:160-165); missing ``speed`` as ``State.speed`` (:143-146)."""
        put = self._put
        put(self.x, x); put(self.y, y); put(self.heading, heading)
        if speed is None and (vx is None or vy is None):
            raise ValueError("give speed, or vx and vy")
        if vx is not None and vy is not None:
            put(self.vx, vx); put(self.vy, vy)
        if speed is not None:
            put(self.speed, speed)
        else:
            self.speed.copy_(torch.sqrt(self.vx * self.vx + self.vy * self.vy))
        if vx is None or vy is None:
            self.vx.copy_(self.speed * torch.cos(self.heading))
            self.vy.copy_(self.speed * torch.sin(self.heading))
        if type_id is not None:
            put(self.type_id, type_id)

    def state_numpy(self) -> dict:
        out = {k: getattr(self, k).detach().cpu().numpy() for k in ("x", "y", "heading", "speed", "vx", "vy")}
        if self.omega_front is not None:
            out["omega_wf"] = self.omega_front.detach().cpu().numpy()
            out["omega_wr"] = self.omega_rear.detach().cpu().numpy()
        return out

    # ------------------------------------------------------------------ the hot path
    def step(self, action: torch.Tensor) -> StepResult:
        """One tick.  ``action``: fp32 device tensor [N, M, 2] = (accel, steer) per bicycle
        (``(steer, accel)`` when built with ``steer_first``), (ax, ay) per point mass."""
        self._device_tensor("action", action, torch.float32, (self.N, self.M, 2))
        o = self._out
        _lib.check(self.lib.t2d_step(self._ctx, _ptr(action), _ptr(o.flags), _ptr(o.hit_index), _ptr(o.hit_segment),
                                     _ptr(o.status), _ptr(o.done), self._stream()))
        self.frame += self.interval
        return o

    @property
    def result(self) -> StepResult:
        """The device-side output arrays of the last ``step`` / ``step_host`` / ``check_events``."""
        return self._out

    def step_host(self, action):
        """One tick for a host-side caller: ``action`` is a float32 ``[N, M, 2]`` NumPy array or CPU tensor (pinned
        memory avoids the driver's staging copy).  Returns ``(done, status)`` as uint8 NumPy arrays [N], valid on
        return; the per-participant flags / hit indices stay on the device in ``self.result`` (whose ``status`` /
        ``done`` tensors this call does not touch).  The copies are
        inside the call (``t2d_step_host``): chunked host->device copy overlapped with the kernel, one
        device->host read-back, one stream synchronisation."""
        a = self._host_tensor("action", action, (self.N, self.M, 2))
        hb = self._host_status()
        o = self._out
        _lib.check(self.lib.t2d_step_host(self._ctx, a.data_ptr(), _ptr(o.flags), _ptr(o.hit_index), _ptr(o.hit_segment),
                                          hb[1].ctypes.data, hb[0].ctypes.data, self._stream()))
        self.frame += self.interval
        return hb[0], hb[1]

    def _host_status(self):
        """The (done, status) host buffers the ego host steps return."""
        if self._host_out is None:
            self._host_out = (np.empty(self.N, np.uint8), np.empty(self.N, np.uint8))
        return self._host_out

    def _npc_zero_action(self) -> torch.Tensor:
        """The internal zero [N, M, 2] action of the host steps called without a device ``action``."""
        if self._npc_action is None:
            self._npc_action = torch.zeros((self.N, self.M, 2), dtype=torch.float32, device=self.device)
        return self._npc_action

    # ------------------------------------------------------------------ env layer
    def set_ego_action(self, ego_action: Optional[torch.Tensor]):
        """Bind the ego's action array: fp32 device tensor [N, 2] (or None to unbind).  While bound, ``control`` and
        ``step`` take the action of participant 0 of every scenario from it - the reference env's single action
        (envs/parking.py:219-239) - instead of row 0 of the full action array."""
        if ego_action is not None:
            self._device_tensor("ego_action", ego_action, torch.float32, (self.N, 2))
        _lib.check(self.lib.t2d_set_ego_action(self._ctx, _ptr(ego_action)))
        self._ego_action = ego_action   # keeps the tensor alive while the library holds its pointer

    def step_host_ego(self, ego_action, action: Optional[torch.Tensor] = None):
        """One tick for a host-side policy that drives only the ego: ``ego_action`` is a float32 ``[N, 2]`` NumPy array
        or CPU tensor; the other participants take the rows of the DEVICE array ``action`` [N, M, 2] (default: an
        internal zero array), which ``set_controllers`` fills on the device.  Per step 8 N bytes go up and 2 N come back
        (``t2d_step_host_ego``).  Returns ``(done, status)`` as uint8 NumPy arrays [N]."""
        a = self._host_tensor("ego_action", ego_action, (self.N, 2))
        if action is None:
            action = self._npc_zero_action()
        else:
            self._device_tensor("action", action, torch.float32, (self.N, self.M, 2))
        hb = self._host_status()
        o = self._out
        _lib.check(self.lib.t2d_step_host_ego(self._ctx, a.data_ptr(), _ptr(action), _ptr(o.flags), _ptr(o.hit_index),
                                              _ptr(o.hit_segment), hb[1].ctypes.data, hb[0].ctypes.data, self._stream()))
        self.frame += self.interval
        return hb[0], hb[1]

    def set_prefetch(self, mode: int):
        """Tuning knob of the tick (``t2d_set_prefetch``), no effect on results: 1 / 0 = ask L2 for the next inputs early or
        not, -1 = the library's policy (on unless a peer-memory done exchange is alive)."""
        _lib.check(self.lib.t2d_set_prefetch(self._ctx, int(mode)))

    def env_epilogue(self, reset_trackers_on_done: bool = True) -> "EnvResult":
        """Reward, terminated, truncated, done and the per-participant TrafficStatus of the last tick in ONE launch
        (``t2d_env_epilogue``: ParkingEnv.step after check_status, envs/parking.py:240-256 and _get_reward :148-190)."""
        e = self._env
        if e is None:
            u8 = dict(dtype=torch.uint8, device=self.device)
            e = self._env = dict(
                reward=torch.zeros(self.N, dtype=torch.float32, device=self.device),
                terminated=torch.zeros(self.N, dtype=torch.bool, device=self.device),
                truncated=torch.zeros(self.N, dtype=torch.bool, device=self.device),
                done=torch.zeros(self.N, **u8), traffic=torch.ones((self.N, self.M), **u8),
                max_iou=torch.full((self.N,), -float("inf"), dtype=torch.float32, device=self.device),
                min_dist=torch.full((self.N,), float("inf"), dtype=torch.float32, device=self.device))
        goal = self._goal is not None
        o = self._out
        _lib.check(self.lib.t2d_env_epilogue(self._ctx, _ptr(o.flags), _ptr(o.status), _ptr(e["reward"]), _ptr(e["terminated"]),
                                             _ptr(e["truncated"]), _ptr(e["traffic"]), _ptr(e["done"]),
                                             _ptr(e["max_iou"] if goal else None), _ptr(e["min_dist"] if goal else None),
                                             1 if reset_trackers_on_done else 0, self._stream()))
        return EnvResult(e["reward"], e["terminated"], e["truncated"], e["done"], e["traffic"])

    def reset_env_trackers(self):
        """``ParkingEnv.reset``: forget the best IoU / distance of the previous episodes (parking.py:276-277)."""
        if self._env is not None:
            self._env["max_iou"].fill_(-float("inf"))
            self._env["min_dist"].fill_(float("inf"))
        if self._routes is not None:
            self._routes["s_best"].fill_(-float("inf"))

    # ------------------------------------------------------------------ per-agent status and reward
    def set_agents(self, observers: Optional[torch.Tensor] = None, goals: Optional[torch.Tensor] = None,
                   arrival_threshold: float = 0.95, no_action_max_step: int = 100):
        """Score every row of an observer list as an agent (``t2d_set_agents``; DESIGN.md section 1 "Per-agent status and
        reward").  ``observers``: int16 ``[N, Q]`` device tensor of slots, Q in 1..128 (a value outside ``[0, M)`` or an
        empty slot gives an absent row; duplicates are allowed), or None for every slot (Q = M); ``goals``: fp32
        ``[N, Q, 5]`` (cx, cy, heading, half_len, half_wid) per row, a NaN cx for none.  A row with a goal whose slot is a
        box gets ``set_goal``'s Arrival / NoAction detectors.  The world owns the detector state, the retired types and the
        outputs of ``agents_epilogue``; a settled row retires its slot (type 255) until ``reset`` restores it."""
        Q = self._agent_rows(observers, goals)
        f32, dev = torch.float32, self.device
        a = dict(
            observers=observers, goals=goals, Q=Q,
            last_pose=torch.zeros((self.N, Q, 4), dtype=f32, device=dev),
            noact_count=torch.zeros((self.N, Q), dtype=torch.int32, device=dev),
            retired_type=torch.full((self.N, self.M), TYPE_INACTIVE, dtype=torch.uint8, device=dev),
            reward=torch.zeros((self.N, Q), dtype=f32, device=dev),
            terminated=torch.zeros((self.N, Q), dtype=torch.bool, device=dev),
            truncated=torch.zeros((self.N, Q), dtype=torch.bool, device=dev),
            status=torch.zeros((self.N, Q), dtype=torch.uint8, device=dev),
            iou=torch.zeros((self.N, Q), dtype=f32, device=dev),
            done=torch.zeros(self.N, dtype=torch.uint8, device=dev),
            traffic=torch.ones((self.N, self.M), dtype=torch.uint8, device=dev),
            max_iou=torch.full((self.N, Q), -float("inf"), dtype=f32, device=dev),
            min_dist=torch.full((self.N, Q), float("inf"), dtype=f32, device=dev))
        _lib.check(self.lib.t2d_set_agents(self._ctx, _ptr(observers), Q, _ptr(goals), float(arrival_threshold),
                                           int(no_action_max_step), _ptr(a["last_pose"]), _ptr(a["noact_count"]),
                                           _ptr(a["retired_type"])))
        self._agents = a
        if self._routes is not None:   # the agents' progress tracker follows their rows
            self._routes["agent_s_best"] = None
            self._bind_route_trackers()

    @property
    def retired_type(self) -> Optional[torch.Tensor]:
        """uint8 [N, M] device tensor: the type of every slot an agent row retired, 255 elsewhere (None without agents)."""
        return None if self._agents is None else self._agents["retired_type"]

    def agents_epilogue(self, reset_trackers_on_done: bool = True) -> AgentEnvResult:
        """Status, reward, terminated, truncated and IoU of every agent row of the last tick, retirement of the slots whose
        rows settled, and the scenarios' done mask (no row NORMAL), in ONE launch (``t2d_agents_epilogue``).  With one row
        per scenario on slot 0 and the ``set_goal`` target as its goal this is ``env_epilogue`` bit for bit."""
        a = self._agents
        if a is None:
            raise RuntimeError("call set_agents before agents_epilogue")
        _lib.check(self.lib.t2d_agents_epilogue(
            self._ctx, _ptr(self._out.flags), _ptr(a["reward"]), _ptr(a["terminated"]), _ptr(a["truncated"]), _ptr(a["status"]),
            _ptr(a["iou"]), _ptr(a["done"]), _ptr(a["max_iou"]), _ptr(a["min_dist"]), _ptr(a["traffic"]),
            1 if reset_trackers_on_done else 0, self._stream()))
        return AgentEnvResult(a["reward"], a["terminated"], a["truncated"], a["status"], a["iou"], a["done"], a["traffic"])

    def reset_agent_trackers(self):
        """Forget every agent row's best IoU / distance of the previous episodes (``reset_env_trackers`` per row)."""
        if self._agents is not None:
            self._agents["max_iou"].fill_(-float("inf"))
            self._agents["min_dist"].fill_(float("inf"))
        if self._routes is not None and self._routes["agent_s_best"] is not None:
            self._routes["agent_s_best"].fill_(-float("inf"))

    # ------------------------------------------------------------------ per-agent action
    def scatter_agent_action(self, agent_action: torch.Tensor, action: torch.Tensor,
                             observers: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Write one action per agent row into its slot of ``action`` [N, M, 2] (IN PLACE; ``t2d_scatter_agent_action``,
        DESIGN.md section 1 "Per-agent action").  ``agent_action``: fp32 ``[N, Q, 2]`` device tensor in the world's action
        order; ``observers``: int16 ``[N, Q]`` as in ``observe_agents`` (None: row q is slot q, Q <= M).  Slot m takes the
        row of the lowest q naming it, when its type is active; every other row of ``action`` keeps its value.  Call it
        before ``control`` and ``step``: a controlled slot then takes its controller's action, and a bound ego action
        still drives slot 0."""
        Q = self._agent_rows(observers, None)
        self._device_tensor("agent_action", agent_action, torch.float32, (self.N, Q, 2))
        self._device_tensor("action", action, torch.float32, (self.N, self.M, 2))
        _lib.check(self.lib.t2d_scatter_agent_action(self._ctx, _ptr(observers), Q, _ptr(agent_action), _ptr(action),
                                                     self._stream()))
        return action

    def step_host_agents(self, agent_action, action: Optional[torch.Tensor] = None, reset_trackers_on_done: bool = True):
        """One multi-agent step for a host-side policy (``t2d_step_host_agents``): ``agent_action`` is a float32
        ``[N, Q, 2]`` NumPy array or CPU tensor, one action per row of the agents bound with ``set_agents``.  It is
        scattered into the DEVICE array ``action`` [N, M, 2] (default: an internal zero array, as ``step_host_ego``), then
        the controllers (if set), the tick and ``agents_epilogue`` run, and the outputs come back in one copy.  Returns
        ``(reward, terminated, truncated, status, done)`` as NumPy arrays ([N, Q] fp32 / bool / bool / uint8 and [N] uint8):
        views of buffers owned by the world that hold their values until the next call.  The flags and hit indices stay on
        the device in ``self.result``; the per-row extrema are those of ``agents_epilogue``, so the two may be mixed.  No
        reset happens inside the call."""
        a_ = self._agents
        if a_ is None:
            raise RuntimeError("call set_agents before step_host_agents")
        Q = a_["Q"]
        a = self._host_tensor("agent_action", agent_action, (self.N, Q, 2))
        if action is None:
            action = self._npc_zero_action()
        else:
            self._device_tensor("action", action, torch.float32, (self.N, self.M, 2))
        hb = self._host_agents
        if hb is None or hb[0].shape[1] != Q:
            hb = self._host_agents = (np.empty((self.N, Q), np.float32), np.empty((self.N, Q), np.bool_),
                                      np.empty((self.N, Q), np.bool_), np.empty((self.N, Q), np.uint8),
                                      np.empty(self.N, np.uint8))
        o = self._out
        _lib.check(self.lib.t2d_step_host_agents(
            self._ctx, a.data_ptr(), _ptr(action), _ptr(o.flags), _ptr(o.hit_index), _ptr(o.hit_segment),
            _ptr(a_["max_iou"]), _ptr(a_["min_dist"]), 1 if reset_trackers_on_done else 0,
            *(h.ctypes.data for h in hb), self._stream()))
        self.frame += self.interval
        return hb

    def check_events(self) -> StepResult:
        """The detectors on the current poses, no physics (``EventBase.update``)."""
        o = self._out
        _lib.check(self.lib.t2d_check_events(self._ctx, _ptr(o.flags), _ptr(o.hit_index), _ptr(o.hit_segment), self._stream()))
        return o

    def lidar_scan(self, n_beams: int = 500, max_range: float = 12.0) -> torch.Tensor:
        """Single-line lidar of every scenario's ego (``SingleLineLidar._scan_obstacles``, sensor/lidar.py:128-221):
        fp32 [N, n_beams] distances, ``inf`` where nothing is hit within ``max_range``.  Defaults are the
        reference's (range 12 m, freq_detect / freq_scan = 5000 / 10 = 500 beams, lidar.py:35-50)."""
        key = (int(n_beams), float(max_range))
        cache = self._lidar
        if cache is None or cache[0] != key:
            scan = torch.empty((self.N, int(n_beams)), dtype=torch.float32, device=self.device)
            self._lidar = cache = (key, self._beam_table(n_beams), scan)
        _lib.check(self.lib.t2d_lidar_scan(self._ctx, int(n_beams), float(max_range), _ptr(cache[1]), _ptr(cache[2]), self._stream()))
        return cache[2]

    def lidar_scan_agents(self, n_beams: int = 500, max_range: float = 12.0,
                          observers: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``lidar_scan`` with the sensor on a list of observer slots per scenario, in one launch
        (``t2d_lidar_scan_agents``; DESIGN.md section 1 "Per-agent lidar"): the reference's ``SingleLineLidar`` bound to
        each row's slot, which sees the map and every other box-shaped participant, slot 0 included.  ``observers``: int16
        ``[N, Q]`` device tensor as in ``observe_agents`` (None: every slot, Q = M); a value outside ``[0, M)`` or an empty
        slot gives a row of ``inf``.  Returns fp32 ``[N, Q, n_beams]``, a buffer per ``(n_beams, max_range, Q)`` that the
        next call with those values reuses.  A row observed by slot 0 equals ``lidar_scan``'s row."""
        Q = self._agent_rows(observers, None)
        key = (int(n_beams), float(max_range), Q)
        entry = self._agent_lidar.get(key)
        if entry is None:
            scan = torch.empty((self.N, Q, int(n_beams)), dtype=torch.float32, device=self.device)
            entry = self._agent_lidar[key] = (self._beam_table(n_beams), scan)
        _lib.check(self.lib.t2d_lidar_scan_agents(self._ctx, _ptr(observers), Q, int(n_beams), float(max_range),
                                                  _ptr(entry[0]), _ptr(entry[1]), self._stream()))
        return entry[1]

    def _beam_table(self, n_beams) -> torch.Tensor:
        """fp64 [n_beams, 2] device tensor: (cos, sin) of every beam's angle, the trig done on the host."""
        theta = np.linspace(0, 2 * np.pi, int(n_beams), endpoint=False)          # lidar.py:160
        return torch.from_numpy(np.stack([np.cos(theta), np.sin(theta)], 1)).to(self.device).contiguous()

    # ------------------------------------------------------------------ BEV observation
    @staticmethod
    def _check_style_keys(keys, n_seg):
        from .sensor.camera import BEV_STYLES

        if keys is None:
            return None
        keys = list(keys)
        if len(keys) != n_seg:
            raise ValueError(f"style needs one key per segment ({n_seg}), got {len(keys)}")
        bad = [k for k in keys if k is not None and k not in BEV_STYLES]
        if bad:
            raise ValueError(f"unknown BEV style keys {sorted(set(bad))}")
        return keys

    def set_bev_styles(self, type_styles=None, target: Optional[str] = "target_area"):
        """Choose how ``bev`` draws each participant type and the goal rectangle, by style key of
        :data:`tactics2d_b200.sensor.camera.BEV_STYLES`.  ``type_styles``: one key (or None = not drawn) per type-table
        row, default from each row's template name (:func:`~tactics2d_b200.sensor.camera.default_type_style`);
        ``target``: the style of the ``set_goal`` rectangle, None = not drawn.  Map segments take the ``style`` given to
        ``set_map`` / ``set_map_table``.  The per-type styles belong to the current table: ``set_type_table`` keeps them
        for a table with as many rows and puts any other table's rows back on their defaults."""
        from .sensor.camera import BEV_STYLES, default_type_style

        if type_styles is None:
            type_styles = [default_type_style(r) for r in self.type_table.rows]
        type_styles = list(type_styles)
        if len(type_styles) != len(self.type_table):
            raise ValueError(f"type_styles needs one key per type-table row ({len(self.type_table)})")
        for k in type_styles + [target]:
            if k is not None and k not in BEV_STYLES:
                raise ValueError(f"unknown BEV style key {k!r}")
        self._bev_cfg = (type_styles, target)
        self._push_bev_styles()

    def _push_bev_styles(self):
        from .sensor.camera import BEV_STYLES, NOT_DRAWN, STYLE_KEYS, style_rgb

        if self._bev_cfg is None:
            return
        type_styles, target = self._bev_cfg
        idx = {k: i for i, k in enumerate(STYLE_KEYS)}
        table = (_lib.BevStyleC * len(STYLE_KEYS))()
        for i, k in enumerate(STYLE_KEYS):
            r, g, b = style_rgb(k)
            table[i] = _lib.BevStyleC(r, g, b, BEV_STYLES[k][1], BEV_STYLES[k][2])
        ts = np.asarray([NOT_DRAWN if k is None else idx[k] for k in type_styles], dtype=np.uint8)
        seg = None
        if any(keys is not None for keys in self._seg_style_keys):
            parts = []
            polys = [self.poly_start] if self.tiles is None else [t["poly_start"] for t in self.tiles]
            for keys, ps in zip(self._seg_style_keys, polys):
                if keys is None:   # this tile keeps the defaults
                    ring = np.zeros(self._tile_nseg(len(parts)), bool)
                    if ps is not None and len(ps) >= 2:
                        ring[ps[0]:ps[-1]] = True
                    parts.append(np.where(ring, idx["obstacle"], idx["road_border"]).astype(np.uint8))
                else:
                    parts.append(np.asarray([NOT_DRAWN if k is None else idx[k] for k in keys], dtype=np.uint8))
            seg = np.ascontiguousarray(np.concatenate(parts)) if parts else None
        n_seg_total = 0 if seg is None else len(seg)
        _lib.check(self.lib.t2d_set_bev_styles(
            self._ctx, table, len(STYLE_KEYS), C.c_void_p(ts.ctypes.data),
            C.c_void_p(0 if seg is None or n_seg_total == 0 else seg.ctypes.data), n_seg_total,
            NOT_DRAWN if target is None else idx[target]))

    def _tile_nseg(self, i):
        if self.tiles is None:
            return 0 if self.segments is None else self.segments.shape[0]
        s = self.tiles[i]["segments"]
        return 0 if s is None else s.shape[0]

    def bev(self, resolution=(200, 200), perception_range=(20.0, 20.0, 20.0, 20.0), rgb: bool = True) -> torch.Tensor:
        """Bird's-eye view of every scenario's ego (``BEVCamera.update`` + ``MatplotlibRenderer``, sensor/camera.py:333-386,
        renderer/matplotlib_renderer.py:542-768) in one launch: ``uint8 [N, H, W, 3]`` RGB, or with ``rgb=False`` the
        style indices ``uint8 [N, H, W]`` (RGB = ``sensor.camera.palette()[index]``).  ``resolution`` = (width, height);
        ``perception_range`` = R or (left, right, front, back) in metres.  The returned tensor is a buffer the world
        reuses on the next call with the same shape.  Uses the default styles until ``set_bev_styles`` is called."""
        if self._bev_cfg is None:
            self.set_bev_styles()
        w, h = int(resolution[0]), int(resolution[1])
        pr = perception_range
        rng = np.ascontiguousarray(np.asarray([pr] * 4 if np.ndim(pr) == 0 else pr, dtype=np.float32).reshape(4))
        key = (w, h, bool(rgb))
        cache = self._bev_out
        if cache is None or cache[0] != key:
            if not (1 <= w <= 1024 and 1 <= h <= 1024):
                raise ValueError("resolution: width and height must be in 1..1024")
            shape = (self.N, h, w, 3) if rgb else (self.N, h, w)
            self._bev_out = cache = (key, torch.empty(shape, dtype=torch.uint8, device=self.device))
        _lib.check(self.lib.t2d_bev_render(self._ctx, w, h, C.c_void_p(rng.ctypes.data), 1 if rgb else 0, _ptr(cache[1]),
                                           self._stream()))
        return cache[1]

    def bev_agents(self, resolution=(200, 200), perception_range=20.0, rgb: bool = True,
                   observers: Optional[torch.Tensor] = None, goals: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``bev`` seen from a list of observer slots per scenario, in one launch (``t2d_bev_render_agents``; DESIGN.md
        section 1 "Per-agent BEV"): the reference's ``BEVCamera`` bound to each row's slot, centred on it with +x along its
        heading, drawing every participant, its own body included.  ``observers``: int16 ``[N, Q]`` device tensor as in
        ``observe_agents`` (None: every slot, Q = M); a value outside ``[0, M)``, an empty or a retired slot gives an
        absent row, all background.  ``goals``: fp32 ``[N, Q, 5]`` per-row goal rectangles (a NaN cx for none); without it
        the rows observed by slot 0 draw the ``set_goal`` target and the others none.  Returns ``uint8 [N, Q, H, W, 3]``, or
        with ``rgb=False`` the style indices ``[N, Q, H, W]``: a buffer per ``(width, height, rgb, Q)`` that the next call
        with those values reuses.  A row observed by slot 0 without ``goals`` equals ``bev``'s image when slot 0 is
        present."""
        Q = self._agent_rows(observers, goals)
        if self._bev_cfg is None:
            self.set_bev_styles()
        w, h = int(resolution[0]), int(resolution[1])
        pr = perception_range
        rng = np.ascontiguousarray(np.asarray([pr] * 4 if np.ndim(pr) == 0 else pr, dtype=np.float32).reshape(4))
        key = (w, h, bool(rgb), Q)
        out = self._agent_bev.get(key)
        if out is None:
            if not (1 <= w <= 1024 and 1 <= h <= 1024):
                raise ValueError("resolution: width and height must be in 1..1024")
            shape = (self.N, Q, h, w, 3) if rgb else (self.N, Q, h, w)
            out = self._agent_bev[key] = torch.empty(shape, dtype=torch.uint8, device=self.device)
        _lib.check(self.lib.t2d_bev_render_agents(self._ctx, _ptr(observers), Q, _ptr(goals), w, h, C.c_void_p(rng.ctypes.data),
                                                  1 if rgb else 0, _ptr(out), self._stream()))
        return out

    # ------------------------------------------------------------------ vector observation
    def observe(self, k_agents: int = 16, k_segments: int = 32, agent_range: float = 50.0,
                segment_range: float = 30.0) -> VectorObservation:
        """The ego-frame vector observation of every scenario's ego (participant 0) in one launch (``t2d_observe``): its
        motion, the ``set_goal`` target, the ``k_agents`` nearest other participants whose centre lies within
        ``agent_range`` metres and the ``k_segments`` nearest segments of its map tile within ``segment_range``, nearest
        first, ties to the lower index; absent rows are zeros with index -1 (DESIGN.md section 1 "Vector observation").
        The tensors are views of one buffer per ``(k_agents, k_segments)`` that the next call with those counts reuses."""
        K, S = int(k_agents), int(k_segments)
        obs = self._obs_out.get((K, S))
        if obs is None:
            obs = self._obs_out[(K, S)] = self._obs_buffer(VectorObservation, (self.N,), K, S)
        cfg = _lib.ObsConfigC(K, S, float(agent_range), float(segment_range))
        _lib.check(self.lib.t2d_observe(self._ctx, C.byref(cfg), _ptr(obs.flat), _ptr(obs.agent_index),
                                        _ptr(obs.segment_index), self._stream()))
        return obs

    def _obs_buffer(self, cls, lead, K: int, S: int):
        """A ``VectorObservation`` / ``AgentObservation`` over one new buffer, leading shape ``lead`` = (N,) or (N, Q)."""
        if not (0 <= K <= 127 and 0 <= S <= 256):
            raise ValueError("k_agents must be in 0..127 and k_segments in 0..256")
        flat = torch.empty(lead + (vector_obs_width(K, S),), dtype=torch.float32, device=self.device)
        a0 = len(EGO_FIELDS) + len(GOAL_FIELDS)
        s0 = a0 + len(AGENT_FIELDS) * K
        i16 = dict(dtype=torch.int16, device=self.device)
        return cls(flat=flat, ego=flat[..., :len(EGO_FIELDS)], goal=flat[..., len(EGO_FIELDS):a0],
                   agents=flat[..., a0:s0].view(lead + (K, len(AGENT_FIELDS))),
                   segments=flat[..., s0:].view(lead + (S, len(SEGMENT_FIELDS))),
                   agent_index=torch.empty(lead + (K,), **i16), segment_index=torch.empty(lead + (S,), **i16))

    def _agent_rows(self, observers, goals) -> int:
        """Q of an observer list (M without one), after checking ``observers`` / ``goals``."""
        if observers is None:
            Q = self.M
        else:
            if not (torch.is_tensor(observers) and observers.dim() == 2):
                raise ValueError(f"observers must be a contiguous int16 [{self.N}, Q] tensor on {self.device}")
            Q = int(observers.shape[1])
            self._device_tensor("observers", observers, torch.int16, (self.N, Q))
        if not 1 <= Q <= 128:
            raise ValueError("the number of observers per scenario must be in 1..128")
        if goals is not None:
            self._device_tensor("goals", goals, torch.float32, (self.N, Q, 5))
        return Q

    def observe_agents(self, k_agents: int = 16, k_segments: int = 32, agent_range: float = 50.0,
                       segment_range: float = 30.0, observers: Optional[torch.Tensor] = None,
                       goals: Optional[torch.Tensor] = None) -> AgentObservation:
        """``observe`` from the point of view of a list of observer slots per scenario, in one launch
        (``t2d_observe_agents``; DESIGN.md section 1 "Per-agent vector observation").  ``observers``: int16 ``[N, Q]``
        device tensor of slots, Q in 1..128 (a value outside ``[0, M)`` or an empty slot gives an absent row; duplicates
        are allowed), or None for every slot (Q = M).  The agents of a row are the nearest other slots, slot 0 included.
        ``goals``: fp32 ``[N, Q, 5]`` (cx, cy, heading, half_len, half_wid) per row, a NaN cx for none; without it the rows
        observed by slot 0 take the ``set_goal`` target and the others none.  A row observed by slot 0 without ``goals``
        equals ``observe``'s row.  The tensors are views of one buffer per ``(k_agents, k_segments, Q)`` that the next call
        with those counts reuses."""
        K, S = int(k_agents), int(k_segments)
        Q = self._agent_rows(observers, goals)
        obs = self._agent_obs_out.get((K, S, Q))
        if obs is None:
            obs = self._agent_obs_out[(K, S, Q)] = self._obs_buffer(AgentObservation, (self.N, Q), K, S)
        obs.observers = observers
        cfg = _lib.ObsConfigC(K, S, float(agent_range), float(segment_range))
        _lib.check(self.lib.t2d_observe_agents(self._ctx, C.byref(cfg), _ptr(observers), Q, _ptr(goals), _ptr(obs.flat),
                                               _ptr(obs.agent_index), _ptr(obs.segment_index), self._stream()))
        return obs

    def _reset_args(self, mask, pool):
        """The checks ``reset`` and ``reset_sampled`` share: the pool columns (fp32 [P, M] on the device, vx / vy and the
        wheel columns in pairs) and the mask; returns (mask as a uint8 [N] device tensor, P)."""
        n_pool = pool["x"].shape[0]
        cols = ["x", "y", "heading", "speed"] + [k for k in ("vx", "vy", "omega_wf", "omega_wr") if pool.get(k) is not None]
        for k in cols:
            self._device_tensor(f"pool[{k!r}]", pool[k], torch.float32, (n_pool, self.M))
        if (pool.get("vx") is None) != (pool.get("vy") is None):
            raise ValueError("give both pool['vx'] and pool['vy'], or neither")
        if self.omega_front is not None and (pool.get("omega_wf") is None) != (pool.get("omega_wr") is None):
            raise ValueError("give both pool['omega_wf'] and pool['omega_wr'], or neither")
        # mask / pool_index reach the kernel as raw pointers: a wrong length would be an illegal address
        if not torch.is_tensor(mask) or mask.numel() != self.N:
            raise ValueError(f"mask must be a tensor of {self.N} scenarios")
        return self._to_device(mask, torch.uint8, (self.N,)), n_pool

    def _bind_wheel_pool(self, pool):
        if self.omega_front is not None:
            _lib.check(self.lib.t2d_bind_reset_wheel_pool(self._ctx, _ptr(pool.get("omega_wf")), _ptr(pool.get("omega_wr"))))

    def reset(self, mask: torch.Tensor, pool: dict, pool_index: Optional[torch.Tensor] = None):
        """Re-initialise the scenarios with ``mask[n] != 0`` from row ``pool_index[n]`` (default n)
        of the pool arrays ``x, y, heading, speed[, vx, vy]`` [P, M] (``ScenarioManager.reset``,
        parking.py:397-441; ``ParticipantBase.reset``, participant_base.py:236-246)."""
        mask, n_pool = self._reset_args(mask, pool)
        if pool_index is not None:
            if not torch.is_tensor(pool_index) or pool_index.numel() != self.N:
                raise ValueError(f"pool_index must be a tensor of {self.N} scenarios")
            pool_index = self._to_device(pool_index, torch.int32, (self.N,))
        if pool_index is None and n_pool < self.N:
            raise ValueError("without pool_index the pool needs one row per scenario")
        self._bind_wheel_pool(pool)
        _lib.check(self.lib.t2d_reset(self._ctx, _ptr(mask), _ptr(pool_index), n_pool, _ptr(pool["x"]), _ptr(pool["y"]),
                                      _ptr(pool["heading"]), _ptr(pool["speed"]), _ptr(pool.get("vx")),
                                      _ptr(pool.get("vy")), self._stream()))

    # ------------------------------------------------------------------ sampled resets
    def set_reset_sampler(self, seed: Optional[int], jitter=None, tries: int = 8, sample_rows: bool = True,
                          avoid_target: bool = False, type_id=None, target=None, tile_id=None, route_id=None):
        """Draw every episode that ``reset_sampled`` starts (``t2d_set_reset_sampler``; DESIGN.md section 1 "Sampled
        resets"; envs/parking.py:397-441, generate_parking_lot.py:231-237).  ``seed`` keys a Philox4x32-10 stream (None
        unbinds); with ``sample_rows`` each reset scenario runs a pool row drawn from it, else its own row n.
        ``jitter`` [M, 4, 2]: the (lo, hi) of dx, dy, dheading, dspeed per slot (a slot of zeros is not moved); up to
        ``tries`` (1..32) drawn start states per slot are checked in slot order with the tick's predicates, and the first
        one that is inside the bounds and meets no map object, no other slot (and, for the ego with ``avoid_target``, not
        the ``set_goal`` target) is taken.  The optional row pools follow the drawn row: ``type_id`` [P, M] into the
        world's type ids, ``target`` [P, 5] into the ``set_goal`` target, ``tile_id`` [P] into the map table's tile ids,
        ``route_id`` [P, M] into ``set_routes``' route ids.  Binding zeroes :attr:`episode_count`."""
        if seed is None:
            _lib.check(self.lib.t2d_set_reset_sampler(self._ctx, None))
            self._sampler = None
            return
        tries = int(tries)
        if not 1 <= tries <= 32:
            raise ValueError("tries must be in 1..32")
        jit = None
        if jitter is not None:
            jit = np.ascontiguousarray(np.asarray(jitter, dtype=np.float32))
            if jit.shape != (self.M, 4, 2):
                raise ValueError(f"jitter must be [{self.M}, 4, 2] (lo, hi) ranges")
            if not (np.isfinite(jit).all() and (jit[..., 0] <= jit[..., 1]).all()):
                raise ValueError("every jitter range must be finite with lo <= hi")
        rows = {}
        for name, a, dtype, tail in (("type_id", type_id, torch.uint8, (self.M,)), ("target", target, torch.float32, (5,)),
                                     ("tile_id", tile_id, torch.int16, ()), ("route_id", route_id, torch.int16, (self.M,))):
            if a is None:
                continue
            t = a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))
            if t.dim() != 1 + len(tail) or tuple(t.shape[1:]) != tail or t.shape[0] < 1:
                raise ValueError(f"the {name} pool must be [P{''.join(', ' + str(d) for d in tail)}]")
            rows[name] = self._to_device(t, dtype, tuple(t.shape))
        n_rows = {t.shape[0] for t in rows.values()}
        if len(n_rows) > 1:
            raise ValueError("the row pools must have the same number of rows")
        if "type_id" in rows:
            tv = rows["type_id"]
            if bool(((tv >= len(self.type_table)) & (tv != TYPE_INACTIVE)).any()):
                raise ValueError("the type_id pool holds ids outside the type table")
        if "target" in rows and self._goal is None:
            raise ValueError("a target pool needs set_goal")
        if "tile_id" in rows:
            if self.tiles is None or len(self.tiles) < 2:
                raise ValueError("a tile_id pool needs a map table of more than one tile")
            tv = rows["tile_id"].to(torch.int64)
            tile_max = int(tv.max())
            if int(tv.min()) < 0 or tile_max >= len(self.tiles):
                raise ValueError(f"the tile_id pool must index the {len(self.tiles)} tiles")
        if "route_id" in rows and self._routes is None:
            raise ValueError("a route_id pool needs set_routes")
        dev = self.device
        s = dict(rows=rows, jitter=jit, tile_max=tile_max if "tile_id" in rows else -1,
                 seed=int(seed) & 0xFFFFFFFFFFFFFFFF, tries=tries, sample_rows=bool(sample_rows),
                 avoid_target=bool(avoid_target), n_rows=n_rows.pop() if n_rows else 0,
                 episode=torch.zeros(self.N, dtype=torch.int32, device=dev),
                 pool_row=torch.arange(self.N, dtype=torch.int32, device=dev),
                 reset_try=torch.full((self.N, self.M), -1, dtype=torch.int8, device=dev))
        c = _lib.ResetSamplerC(s["seed"], int(s["sample_rows"]), tries, int(s["avoid_target"]), s["n_rows"],
                               None if jit is None else jit.ctypes.data, _ptr(rows.get("type_id")),
                               _ptr(rows.get("target")), _ptr(rows.get("tile_id")), _ptr(rows.get("route_id")),
                               _ptr(s["episode"]), _ptr(s["pool_row"]), _ptr(s["reset_try"]))
        # the library keeps the previous sampler until a call succeeds: replace the tensors only then
        _lib.check(self.lib.t2d_set_reset_sampler(self._ctx, C.byref(c)))
        self._sampler = s

    def reset_sampled(self, mask: torch.Tensor, pool: dict):
        """``reset`` of the scenarios with ``mask[n] != 0`` through the bound sampler (``t2d_reset_sampled``): each takes
        the pool row it draws (:attr:`pool_row`), the row-owned columns follow it, then its start states are jittered
        (:attr:`reset_try`) and its :attr:`episode_count` advances.  ``pool`` as ``reset``'s."""
        if self._sampler is None:
            raise RuntimeError("call set_reset_sampler before reset_sampled")
        mask, n_pool = self._reset_args(mask, pool)
        s = self._sampler
        if s["n_rows"] and n_pool != s["n_rows"]:
            raise ValueError(f"the pool must have the row pools' {s['n_rows']} rows")
        if not s["sample_rows"] and n_pool < self.N:
            raise ValueError("without row draws the pool needs one row per scenario")
        # the tile pool was checked against the map bound then; a map table rebound since may hold fewer tiles
        if s["tile_max"] >= 0 and (self.tiles is None or s["tile_max"] >= len(self.tiles)):
            raise ValueError(f"the tile_id pool names tile {s['tile_max']}, beyond the bound map's tiles")
        self._bind_wheel_pool(pool)
        _lib.check(self.lib.t2d_reset_sampled(self._ctx, _ptr(mask), n_pool, _ptr(pool["x"]), _ptr(pool["y"]),
                                              _ptr(pool["heading"]), _ptr(pool["speed"]), _ptr(pool.get("vx")),
                                              _ptr(pool.get("vy")), self._stream()))

    @property
    def pool_row(self) -> Optional[torch.Tensor]:
        """int32 [N] device tensor: the pool row every scenario started its episode from (None without a sampler)."""
        return None if self._sampler is None else self._sampler["pool_row"]

    @property
    def episode_count(self) -> Optional[torch.Tensor]:
        """int32 [N] device tensor holding the uint32 episode counters of the sampler (None without one)."""
        return None if self._sampler is None else self._sampler["episode"]

    @property
    def reset_try(self) -> Optional[torch.Tensor]:
        """int8 [N, M] device tensor: the try that placed each slot at the last sampled reset, -1 where the pool state
        was kept or the slot is not jittered (None without a sampler)."""
        return None if self._sampler is None else self._sampler["reset_try"]
