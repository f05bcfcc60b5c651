"""Seeded synthetic scenario batches for the BASELINE.json configs (host-side NumPy).

The reference has no scenario generator for N x M multi-agent batches (its generators build one
parking lot / racing track, map/generator/*.py, through the global ``np.random``); these are the
synthetic inputs SURVEY.md section 8(d) specifies.  Everything is generated on the CPU from an
explicit seed and rounded to fp32, so the CPU oracle and the GPU see identical bits.
"""

from __future__ import annotations

from dataclasses import dataclass, field
from typing import Optional, Tuple

import numpy as np

from .types import TYPE_INACTIVE, TypeTable


@dataclass
class Scene:
    table: TypeTable
    x: np.ndarray          # fp32 [N, M]
    y: np.ndarray
    heading: np.ndarray
    speed: np.ndarray
    vx: np.ndarray
    vy: np.ndarray
    type_id: np.ndarray    # uint8 [N, M]
    segments: Optional[np.ndarray] = None   # fp32 [S, 4]
    bounds: Optional[Tuple[float, float, float, float]] = None
    name: str = ""
    meta: dict = field(default_factory=dict)

    @property
    def shape(self):
        return self.x.shape

    def state(self) -> dict:
        return dict(x=self.x, y=self.y, heading=self.heading, speed=self.speed, vx=self.vx, vy=self.vy)


def _finish(table, x, y, h, v, tid, segments, bounds, name, **meta) -> Scene:
    f = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    x, y, h, v = f(x), f(y), f(h), f(v)
    vx = f(v.astype(np.float64) * np.cos(h.astype(np.float64)))
    vy = f(v.astype(np.float64) * np.sin(h.astype(np.float64)))
    seg = None if segments is None else np.ascontiguousarray(segments, dtype=np.float32).reshape(-1, 4)
    return Scene(table, x, y, h, v, vx, vy, np.ascontiguousarray(tid, dtype=np.uint8), seg, bounds, name, meta)


def grid_wall_segments(size: float = 200.0, pitch: float = 50.0, wall: float = 16.0) -> np.ndarray:
    """The "synthetic grid map" of config 2: axis-aligned wall pieces of length ``wall`` centred on
    every edge of a ``pitch`` lattice over a ``size`` x ``size`` arena (gaps between pieces let
    traffic through).  The reference's GridMapGenerator is a cost grid, not geometry
    (map/generator/generate_grid_map.py:10-42), so this build defines the map itself."""
    n = int(round(size / pitch))
    segs = []
    for i in range(n + 1):
        c = i * pitch
        for j in range(n):
            m = (j + 0.5) * pitch
            segs.append((c, m - wall / 2, c, m + wall / 2))   # vertical piece on x = c
            segs.append((m - wall / 2, c, m + wall / 2, c))   # horizontal piece on y = c
    return np.asarray(segs, dtype=np.float32)


def random_actions(seed: int, shape, accel=(-4.0, 3.0), steer=(-0.6, 0.6)) -> np.ndarray:
    """Per-step actions [N, M, 2] = (accel, steer); the ranges exceed the models' limits on purpose
    so that clipping is exercised (SURVEY.md 8(d) C1)."""
    rng = np.random.default_rng(seed)
    a = rng.uniform(accel[0], accel[1], shape)
    d = rng.uniform(steer[0], steer[1], shape)
    return np.ascontiguousarray(np.stack([a, d], -1), dtype=np.float32)


def config1(seed: int = 0) -> Scene:
    """C1 (parity gate): 1 scenario x 8 medium cars, SingleTrackKinematics, empty map, bounds
    (-100, 100, -100, 100); 2 x 4 lattice with 6 m pitch and +-1 m jitter so that pairs overlap."""
    rng = np.random.default_rng(seed)
    table = TypeTable.from_templates("kinematics")
    ix, iy = np.meshgrid(np.arange(4), np.arange(2))
    x = (ix.reshape(1, 8) - 1.5) * 6.0 + rng.uniform(-1, 1, (1, 8))
    y = (iy.reshape(1, 8) - 0.5) * 6.0 + rng.uniform(-1, 1, (1, 8))
    h = rng.uniform(0, 2 * np.pi, (1, 8))
    v = rng.uniform(0, 10, (1, 8))
    tid = np.full((1, 8), table.index("medium_car"))
    return _finish(table, x, y, h, v, tid, None, (-100.0, 100.0, -100.0, 100.0), "C1 1x8 kinematics, empty map")


def _arena(rng, n, m, size, jitter, vmax, table, type_choices, heading=None):
    side = int(np.ceil(np.sqrt(m)))
    pitch = size / side
    jitter = pitch / 2 if jitter is None else jitter
    k = np.arange(m)
    gx, gy = (k % side + 0.5) * pitch, (k // side + 0.5) * pitch
    x = gx[None] + rng.uniform(-jitter, jitter, (n, m))
    y = gy[None] + rng.uniform(-jitter, jitter, (n, m))
    h = rng.uniform(0, 2 * np.pi, (n, m)) if heading is None else heading
    v = rng.uniform(0, vmax, (n, m))
    tid = rng.choice(np.asarray(type_choices), size=(n, m))
    return x, y, h, v, tid


def config2(n: int = 4096, m: int = 64, seed: int = 1, size: float = 200.0, jitter: float = None) -> Scene:
    """C2: N x M SingleTrackKinematics vehicles (types sampled from the 9 VEHICLE_TEMPLATE rows) in a
    200 m arena with the synthetic grid map; jitter tuned for a few percent of colliding participants."""
    rng = np.random.default_rng(seed)
    table = TypeTable.vehicles("kinematics")   # the 9 VEHICLE_TEMPLATE rows: a kinematics-only table
    x, y, h, v, tid = _arena(rng, n, m, size, jitter, 15.0, table, list(range(9)))
    return _finish(table, x, y, h, v, tid, grid_wall_segments(size), (-8.0, size + 8.0, -8.0, size + 8.0),
                   f"C2 {n}x{m} kinematics + OBB collision, synthetic grid map")


def config3(n: int = 4096, m: int = 64, seed: int = 3, segments=None, bounds=None) -> Scene:
    """C3: SingleTrackDynamics vehicles driving along a highD-like straight road at 20-40 m/s (away
    from the stiff |v| < 0.5 region); ``segments`` = the map's collidable polylines (highD tiles)."""
    rng = np.random.default_rng(seed)
    table = TypeTable.from_templates("dynamics")
    if bounds is None:
        bounds = (0.0, 668.0, -30.0, 2.0)
    x0, x1, y0, y1 = bounds
    lanes = np.linspace(y0 + 4.0, y1 - 4.0, 8)
    slots = m // 8 + (m % 8 > 0)
    k = np.arange(m)
    x = (x0 + 10.0) + (k // 8 + 0.5)[None] * ((x1 - x0 - 20.0) / slots) + rng.uniform(-6, 6, (n, m))
    y = lanes[k % 8][None] + rng.uniform(-0.8, 0.8, (n, m))
    h = np.where(k % 8 < 4, 0.0, np.pi)[None] + rng.uniform(-0.03, 0.03, (n, m))
    h = np.mod(h, 2 * np.pi)
    v = rng.uniform(20, 40, (n, m))
    tid = rng.integers(0, 9, (n, m))
    return _finish(table, x, y, h, v, tid, segments, bounds, f"C3 {n}x{m} dynamics + map polylines")


def config4(n: int = 16384, m: int = 32, seed: int = 4, segments=None, bounds=None, size: float = 150.0) -> Scene:
    """C4: mixed traffic - 60 % vehicles (kinematics), 20 % cyclists (kinematics, lf = lr = L/2),
    20 % pedestrians (PointMass newton, disc of width/2) on an inD-like intersection."""
    rng = np.random.default_rng(seed)
    table = TypeTable.from_templates("kinematics")
    x, y, h, v, _ = _arena(rng, n, m, size, None, 8.0, table, [0])
    u = rng.uniform(0, 1, (n, m))
    tid = np.where(u < 0.6, rng.integers(0, 9, (n, m)), np.where(u < 0.8, rng.integers(9, 12, (n, m)), rng.integers(12, 16, (n, m))))
    v = np.where(tid >= 12, rng.uniform(0, 2.5, (n, m)), v)
    if bounds is None:
        bounds = (-8.0, size + 8.0, -8.0, size + 8.0)
    else:
        x = x + bounds[0]
        y = y + bounds[2]
    return _finish(table, x, y, h, v, tid, segments, bounds, f"C4 {n}x{m} mixed vehicle/cyclist/pedestrian")


def config5(n: int = 65536, m: int = 128, seed: int = 5, segments=None, bounds=None, size: float = 280.0) -> Scene:
    """C5: broadphase stress - N x 128 kinematic vehicles, rounD-like map."""
    rng = np.random.default_rng(seed)
    table = TypeTable.vehicles("kinematics")
    x, y, h, v, tid = _arena(rng, n, m, size, None, 15.0, table, list(range(9)))
    if bounds is None:
        bounds = (-8.0, size + 8.0, -8.0, size + 8.0)
    else:
        x = x + bounds[0]
        y = y + bounds[2]
    return _finish(table, x, y, h, v, tid, segments, bounds, f"C5 {n}x{m} kinematics + broadphase stress")


def with_inactive(scene: Scene, fraction: float, seed: int = 0) -> Scene:
    """Mark a random subset of slots inactive (ragged scenarios)."""
    rng = np.random.default_rng(seed)
    tid = scene.type_id.copy()
    tid[rng.uniform(0, 1, tid.shape) < fraction] = TYPE_INACTIVE
    return Scene(scene.table, scene.x, scene.y, scene.heading, scene.speed, scene.vx, scene.vy, tid, scene.segments,
                 scene.bounds, scene.name + f" ({fraction:.0%} inactive)", dict(scene.meta))


def replay_episodes(n_rows: int, m: int, n_tracks: int, seed: int = 0, table: Optional[TypeTable] = None, size: float = 200.0,
                    duration_ms: int = 60000, period_ms: int = 40, max_frames: int = 250, horizon_ms: int = 6000):
    """A seeded synthetic recording for log replay (``tactics2d_b200.dataset_parser.ReplayEpisodes``): ``n_tracks`` vehicle
    tracks of 1..``max_frames`` records every ``period_ms`` (a quarter of them starting off the period grid), wandering
    headings that cross 0 / 2 pi, spread over ``duration_ms``; ``n_rows`` episode rows starting on a 20 ms grid, each with a
    random kinematic ego in slot 0 and up to m - 1 of the tracks present in [t0, t0 + horizon_ms] in slots 1.. (random
    picks, -1 when fewer overlap).  Every track's type row is the static twin of a random vehicle row of ``table``
    (default: the 9 vehicle templates)."""
    from .dataset_parser.replay import ReplayEpisodes, ReplayLog
    from .participant.element import Vehicle

    rng = np.random.default_rng(seed)
    base = table if table is not None else TypeTable.vehicles("kinematics")
    veh = [i for i, r in enumerate(base.rows) if r.model == 0 and r.shape == 0]
    table, twin = base.with_static_twins(veh)
    K = int(n_tracks)
    nfr = rng.integers(1, max_frames + 1, K).astype(np.int32)
    first = (rng.integers(-max_frames // 2, duration_ms // period_ms, K) * period_ms).astype(np.int64)
    first += np.where(rng.uniform(0, 1, K) < 0.25, rng.integers(1, period_ms, K), 0)
    cls_row = rng.choice(veh, K)
    recs = []
    for k in range(K):
        n = int(nfr[k])
        h = rng.uniform(0, 2 * np.pi) + np.cumsum(rng.normal(0, 0.08, n))
        v = np.abs(rng.uniform(0, 20) + np.cumsum(rng.normal(0, 0.3, n)))
        vx, vy = v * np.cos(h), v * np.sin(h)
        x = rng.uniform(0, size) + np.cumsum(vx) * period_ms / 1000
        y = rng.uniform(0, size) + np.cumsum(vy) * period_ms / 1000
        recs.append(np.stack([x, y, np.mod(h, 2 * np.pi), vx, vy], 1).astype(np.float32))
    rows = table.rows
    log = ReplayLog(ids=np.arange(K, dtype=np.int64), first_ms=first.astype(np.int32), n_frames=nfr,
                    period_ms=np.full(K, period_ms, np.int32), records=np.ascontiguousarray(np.concatenate(recs)),
                    type_row=np.asarray([twin[int(r)] for r in cls_row], np.uint8), cls=[Vehicle] * K,
                    length=np.asarray([2 * rows[r].half_len for r in cls_row]), width=np.asarray([2 * rows[r].half_wid for r in cls_row]))
    P = int(n_rows)
    t0 = (rng.integers(0, duration_ms // 20, P) * 20).astype(np.int32)
    last = log.last_ms
    row_track = np.full((P, m), -1, np.int32)
    tid = np.full((P, m), TYPE_INACTIVE, np.uint8)
    for p in range(P):
        cand = np.nonzero((last >= t0[p]) & (first <= t0[p] + horizon_ms))[0]
        pick = rng.choice(cand, min(len(cand), m - 1), replace=False)
        row_track[p, 1:1 + len(pick)] = pick
        on = (first[pick] <= t0[p]) & (last[pick] >= t0[p])
        tid[p, 1:1 + len(pick)] = np.where(on, log.type_row[pick], TYPE_INACTIVE)
    x, y, h, v, ego = _arena(rng, P, 1, size, None, 15.0, table, veh)
    z = lambda: np.zeros((P, m))
    px, py, ph, pv = z(), z(), z(), z()
    px[:, 0], py[:, 0], ph[:, 0], pv[:, 0] = x[:, 0], y[:, 0], h[:, 0], v[:, 0]
    tid[:, 0] = ego[:, 0]
    sc = _finish(table, px, py, ph, pv, tid, None, None, "replay")
    pool = sc.state()
    return ReplayEpisodes(log, table, pool, tid, row_track, t0, np.zeros(P, np.int64))


def highway_log(duration_ms: int = 200000, seed: int = 0, rate_per_s: float = 1.85, length_m: float = 420.0,
                speed=(25.0, 38.0), lanes_per_side: int = 3, lane_width: float = 3.75, period_ms: int = 40):
    """A seeded highway-like recording (a :class:`tactics2d_b200.dataset_parser.ReplayLog`, type rows unassigned), modelled
    on highD's traffic (no LevelX data ships with this repository): road users arrive as a Poisson process of
    ``rate_per_s`` per second over ``duration_ms``, each on a random lane of either carriageway (``lanes_per_side`` lanes
    of ``lane_width`` m each side of y = 0; +x above, -x below), and drive straight through the ``length_m`` stretch at
    their own constant speed drawn from ``speed`` (m/s), one record every ``period_ms`` from their arrival (on the period
    grid) until they leave it.  One in eight is a truck (16 m x 2.5 m), the others cars (4.5 m x 1.9 m)."""
    from .dataset_parser.replay import ReplayLog
    from .participant.element import Vehicle

    rng = np.random.default_rng(seed)
    arrivals = []
    t = rng.exponential(1000.0 / rate_per_s)
    while t < duration_ms:
        arrivals.append(t)
        t += rng.exponential(1000.0 / rate_per_s)
    K = len(arrivals)
    first = (np.floor(np.asarray(arrivals) / period_ms) * period_ms).astype(np.int64)
    v = rng.uniform(speed[0], speed[1], K)
    lane = rng.integers(0, 2 * lanes_per_side, K)
    fwd = lane < lanes_per_side
    y = np.where(fwd, -(lane + 0.5), (lane - lanes_per_side + 0.5)) * lane_width
    truck = rng.uniform(0, 1, K) < 0.125
    nfr = (np.floor(length_m / (v * period_ms / 1000.0)) + 1).astype(np.int32)
    recs = []
    for k in range(K):
        s = v[k] * np.arange(nfr[k]) * (period_ms / 1000.0)
        x = s if fwd[k] else length_m - s
        vx = np.full(nfr[k], v[k] if fwd[k] else -v[k])
        h = np.full(nfr[k], 0.0 if fwd[k] else np.pi)
        recs.append(np.stack([x, np.full(nfr[k], y[k]), h, vx, np.zeros(nfr[k])], 1).astype(np.float32))
    return ReplayLog(ids=np.arange(K, dtype=np.int64), first_ms=first.astype(np.int32), n_frames=nfr,
                     period_ms=np.full(K, period_ms, np.int32), records=np.ascontiguousarray(np.concatenate(recs)),
                     type_row=np.full(K, TYPE_INACTIVE, np.uint8), cls=[Vehicle] * K,
                     length=np.where(truck, 16.0, 4.5), width=np.where(truck, 2.5, 1.9))


def highway_episodes(n_rows: int, m: int, seed: int = 0, duration_ms: int = 200000, horizon_ms: Optional[int] = 100000,
                     reuse_slots: bool = True, log=None, **log_kw):
    """Episode rows over :func:`highway_log` (``build_replay_episodes``): row p's ego is a random road user, starting at a
    random frame of the first half of its pass, with ``t0`` in the first ``duration_ms - horizon_ms`` of the log so that
    the window lies inside the recording; the other slots replay the window's tracks, one after the other when
    ``reuse_slots``."""
    from .dataset_parser.replay import build_replay_episodes

    log = highway_log(duration_ms, seed, **log_kw) if log is None else log
    rng = np.random.default_rng(seed + 1)
    span = duration_ms - (horizon_ms or 0)
    ok = np.nonzero(log.first_ms < span)[0]
    ego = rng.choice(ok, int(n_rows))
    t0 = log.first_ms[ego] + rng.integers(0, (log.n_frames[ego] + 1) // 2) * log.period_ms[ego]
    return build_replay_episodes(log, m, t0.tolist(), log.ids[ego].tolist(), horizon_ms=horizon_ms, reuse_slots=reuse_slots)


def idm_highway_log(duration_ms: int = 60000, seed: int = 0, lanes: int = 3, lane_width: float = 3.5,
                    length_m: float = 800.0, period_ms: int = 100, desired=(24.0, 28.0, 32.0), headway_s: float = 3.0):
    """A seeded one-way highway recording made by car following (a :class:`tactics2d_b200.dataset_parser.ReplayLog`, type
    rows unassigned): lane l runs along y = l * ``lane_width`` in +x.  At t = 0 the road holds a car every
    ``headway_s * desired[l]`` metres of lane l, and a new car enters x = 0 about every ``headway_s`` seconds (+-30 %),
    at its own desired speed (the lane's +-10 %).  Every car follows the one ahead in its lane with the IDM (headway
    1.2 s, min spacing 4 m, acceleration 1.5, deceleration 3 m/s^2), integrated in float64 every ``period_ms``, and
    leaves past x = ``length_m``.  Cars are 4.5 m x 1.9 m; heading 0, vy 0."""
    from .dataset_parser.replay import ReplayLog
    from .participant.element import Vehicle

    rng = np.random.default_rng(seed)
    dt = period_ms / 1000.0
    tracks = []                                    # [first_ms, records]
    road = [[] for _ in range(lanes)]              # per lane, front first: [x, v, vd, track]

    def new(l, x, t_ms):
        vd = desired[l] * rng.uniform(0.9, 1.1)
        tracks.append([t_ms, []])
        return [x, vd, vd, len(tracks) - 1]

    for l in range(lanes):
        gap = headway_s * desired[l]
        road[l] = [new(l, x, 0) for x in np.arange(length_m - gap * rng.uniform(0.2, 1.0), 0.0, -gap)]
    due = [rng.uniform(0.0, headway_s) for _ in range(lanes)]
    for step in range(duration_ms // period_ms + 1):
        t_ms = step * period_ms
        for l in range(lanes):
            if t_ms / 1000.0 >= due[l] and (not road[l] or road[l][-1][0] > 30.0):
                road[l].append(new(l, 0.0, t_ms))
                due[l] = t_ms / 1000.0 + headway_s * rng.uniform(0.7, 1.3)
            for c in road[l]:
                tracks[c[3]][1].append((c[0], l * lane_width, 0.0, c[1], 0.0))
            acc = []
            for i, c in enumerate(road[l]):
                x, v, vd = c[0], c[1], c[2]
                a = 1.5 * (1.0 - (v / vd) ** 4)
                if i > 0:
                    lead = road[l][i - 1]
                    s = lead[0] - x - 4.5
                    s_star = 4.0 + v * 1.2 + v * (v - lead[1]) / (2.0 * np.sqrt(1.5 * 3.0))
                    a -= 1.5 * (max(s_star, 4.0) / max(s, 0.1)) ** 2
                acc.append(max(a, -8.0))
            for c, a in zip(road[l], acc):
                v_new = max(c[1] + a * dt, 0.0)
                c[0] += 0.5 * (c[1] + v_new) * dt
                c[1] = v_new
            road[l] = [c for c in road[l] if c[0] <= length_m]
    K = len(tracks)
    recs = [np.asarray(r, np.float32) for _, r in tracks]
    return ReplayLog(ids=np.arange(K, dtype=np.int64), first_ms=np.asarray([f for f, _ in tracks], np.int32),
                     n_frames=np.asarray([len(r) for r in recs], np.int32), period_ms=np.full(K, period_ms, np.int32),
                     records=np.ascontiguousarray(np.concatenate(recs)), type_row=np.full(K, TYPE_INACTIVE, np.uint8),
                     cls=[Vehicle] * K, length=np.full(K, 4.5), width=np.full(K, 1.9))


# ---------------------------------------------------------------------------- scenes with crossing and merging paths
@dataclass
class PathScene:
    """N scenarios of path-following IDM traffic on one ``set_paths`` table: every car is an IDM row that keeps its
    path (``path_controller``), ``path_id`` [N, M] names its path, ``priority`` [n_paths] the paths' priorities for
    ``BatchedWorld.set_yielding``.  Slots with ``path_id == -1`` are empty (``type_id`` 255)."""
    table: TypeTable
    paths: list
    priority: np.ndarray   # int16 [n_paths]
    x: np.ndarray          # fp32 [N, M]
    y: np.ndarray
    heading: np.ndarray
    speed: np.ndarray
    type_id: np.ndarray    # uint8 [N, M]
    path_id: np.ndarray    # int16 [N, M]
    name: str = ""

    @property
    def shape(self):
        return self.x.shape

    @property
    def ctrl_id(self) -> np.ndarray:
        """uint8 [N, M]: row 0 (``path_controller``) for every car."""
        return np.where(self.path_id >= 0, 0, 255).astype(np.uint8)


def path_table() -> TypeTable:
    """One kinematic car type (4.8 m x 1.9 m) that cannot reverse: the reference's IDM keeps braking below 0 m/s."""
    from .types import TypeParams

    return TypeTable([TypeParams(half_len=2.4, half_wid=0.95, lf=1.3, lr=1.3, steer_lo=-0.6, steer_hi=0.6, speed_lo=0.0,
                                 speed_hi=30.0, accel_lo=-8.0, accel_hi=4.0)])


def path_controller():
    """The IDM every car of a :class:`PathScene` drives, with a PID cross-track channel that keeps it on its path."""
    from .controller import IDMController, PIDController

    keep = PIDController(dt=0.1, kp_lat=0.3, ki_lat=0.0, kd_lat=0.3, max_steering=0.6, derivative_filter_alpha=1.0,
                         lateral_error="path_cross_track")
    # the reference's IDM brakes for a closing speed only through min_spacing (its s* subtracts v (v - v_lead) / (2
    # sqrt(a b))): a large min_spacing and max_acceleration make it stop short of a stopped car or a stop point
    return IDMController(desired_speed=10.0, time_headway=1.0, min_spacing=20.0, max_acceleration=8.0,
                         comfortable_deceleration=8.0, lateral=keep)


def _polyline(*pieces):
    return np.ascontiguousarray(np.concatenate([np.asarray(p, np.float64).reshape(-1, 2) for p in pieces]), np.float32)


def _arc(cx, cy, r, a0, a1, n):
    a = np.linspace(a0, a1, n)
    return np.stack([cx + r * np.cos(a), cy + r * np.sin(a)], 1)


def _bezier(p0, p1, p2, n):
    t = np.linspace(0.0, 1.0, n)[:, None]
    p0, p1, p2 = (np.asarray(p, np.float64) for p in (p0, p1, p2))
    return (1 - t) ** 2 * p0 + 2 * t * (1 - t) * p1 + t ** 2 * p2


def _meet(a, u, b, v):
    """The point where the lines a + s u and b + t v meet."""
    a, u, b, v = (np.asarray(q, np.float64) for q in (a, u, b, v))
    cross = lambda p, q: p[0] * q[1] - p[1] * q[0]
    s = cross(b - a, v) / cross(u, v)
    return a + s * u


def _point_at(path, s):
    """(x, y, heading) of ``path`` at arc length s (clamped to its ends)."""
    p = np.asarray(path, np.float64)
    d = np.diff(p, axis=0)
    ln = np.hypot(d[:, 0], d[:, 1])
    cum = np.r_[0.0, np.cumsum(ln)]
    s = np.clip(s, 0.0, cum[-1])
    k = np.clip(np.searchsorted(cum, s, side="right") - 1, 0, len(ln) - 1)
    t = (s - cum[k]) / ln[k]
    return p[k, 0] + t * d[k, 0], p[k, 1] + t * d[k, 1], np.arctan2(d[k, 1], d[k, 0])


def _place(paths, n, m, seed, starts, lane_of, spacing, speed, name, priority):
    """Cars of rank r = 0, 1, ... on the slots of each start lane (``lane_of[slot]``), the first at arc length
    ``starts[lane]`` minus a seeded 0-20 m, the others ``spacing`` (+-3 m) behind it, at seeded speeds in ``speed``."""
    rng = np.random.default_rng(seed)
    lane_of = np.asarray(lane_of)
    x, y, h = (np.zeros((n, m)) for _ in range(3))
    pid = np.full((n, m), -1, np.int16)
    for i in range(n):
        s_lane = {l: starts[l] - rng.uniform(0.0, 20.0) for l in set(lane_of.tolist())}
        for k in range(m):
            l = int(lane_of[k])
            s = s_lane[l]
            s_lane[l] = s - spacing + rng.uniform(-3.0, 3.0)
            if s < 0.0:
                continue   # no room left on this lane
            x[i, k], y[i, k], h[i, k] = _point_at(paths[l], s)
            pid[i, k] = l
    v = rng.uniform(speed[0], speed[1], (n, m))
    tid = np.where(pid >= 0, 0, TYPE_INACTIVE).astype(np.uint8)
    f = lambda a: np.ascontiguousarray(np.where(pid >= 0, a, 0.0), np.float32)
    return PathScene(path_table(), paths, np.asarray(priority, np.int16), f(x), f(y), f(h), f(v), tid, pid, name)


def intersection(n: int, m: int = 8, seed: int = 0, exit_len: float = 200.0, spacing: float = 25.0,
                 speed=(6.0, 10.0)) -> PathScene:
    """A four-arm intersection with one straight-through lane per arm, all four crossing at the centre (right-hand
    traffic, lanes 1.75 m off the axes): path 0 west to east, 1 south to north, 2 east to west, 3 north to south, each
    long enough for its cars before the centre and ``exit_len`` after it, equal priority.  Slot k drives path k % 4; the
    first car of each arm starts 0-20 m further from the centre than 30 m (seeded per scenario and arm), the others
    ``spacing`` metres behind each other.  Without yielding, cars of crossing arms meet at the centre."""
    o = 1.75
    approach = 60.0 + spacing * ((m + 3) // 4)
    paths = [_polyline([[-approach, -o], [exit_len, -o]]), _polyline([[o, -approach], [o, exit_len]]),
             _polyline([[approach, o], [-exit_len, o]]), _polyline([[-o, approach], [-o, -exit_len]])]
    lane_of = [k % 4 for k in range(m)]
    return _place(paths, n, m, seed, {l: approach - 30.0 for l in range(4)}, lane_of, spacing, speed, "intersection",
                  [0, 0, 0, 0])


def t_junction(n: int, m: int = 8, seed: int = 0, speed=(6.0, 10.0), spacing: float = 25.0) -> PathScene:
    """A T-junction merge: path 0 is the main road, west to east along y = 0 (priority 1); path 1 comes up from the south
    along x = 0 and turns right onto it on a 10 m radius (priority 0), sharing its lane from x = 10 m on.  Slot k drives
    path k % 2."""
    side = _polyline([[0.0, -100.0], [0.0, -10.0]], _arc(10.0, -10.0, 10.0, np.pi, np.pi / 2, 12)[1:], [[300.0, 0.0]])
    lane_of = [k % 2 for k in range(m)]
    main = _polyline([[-120.0 - spacing * (m // 2), 0.0], [300.0, 0.0]])
    return _place([main, side], n, m, seed, {0: 80.0 + spacing * (m // 2), 1: 60.0}, lane_of, spacing, speed, "t_junction",
                  [1, 0])


def roundabout(n: int, m: int = 11, seed: int = 0, radius: float = 20.0, arm: float = 80.0, speed=(6.0, 9.0),
               spacing: float = 25.0, ring_cars: int = 3) -> PathScene:
    """A four-arm roundabout (centre 0, ``radius`` m, anticlockwise, right-hand traffic): path 0 is the ring, three
    quarters of a turn from 45 degrees and out on the south-east diagonal (priority 1); paths 1-4 enter from the east,
    north, west and south arms, drive a quarter of the ring and leave by the next arm (priority 0), so that they merge
    into the ring's traffic and diverge from it but never meet each other.  Entries and exits join the ring tangentially
    (quadratic Bezier curves), so that a car that keeps its path stays on it, and each arm's two lanes run 3 m either side
    of its axis.  Slots 0 .. ``ring_cars`` - 1 ride the ring,
    a quarter turn apart from its start; slot k >= ``ring_cars`` enters by arm (k - ``ring_cars``) % 4."""
    o = 3.0                                            # lanes 3 m off each arm's axis: a splitter island between them
    end = 7 * np.pi / 4
    ring = _polyline(_arc(0.0, 0.0, radius, np.pi / 4, end, 64), [[(radius + arm) * np.cos(end), (radius + arm) * np.sin(end)]])
    paths = [ring]
    for a in range(4):
        th = a * np.pi / 2
        c, s = np.cos(th), np.sin(th)
        lane_in = lambda d: (d * c - o * s, d * s + o * c)                    # right of the inbound direction (-c, -s)
        a_in, out = th + 0.45, th + np.pi / 2
        a_out = out - 0.45
        co, so = np.cos(out), np.sin(out)
        lane_out = lambda d: (d * co + o * so, d * so - o * co)               # right of the outbound direction
        ring_at = lambda a: (radius * np.cos(a), radius * np.sin(a))
        tangent = lambda a: (-np.sin(a), np.cos(a))
        join = _bezier(lane_in(radius + 8.0), _meet(lane_in(radius), (-c, -s), ring_at(a_in), tangent(a_in)), ring_at(a_in), 8)
        quarter = _arc(0.0, 0.0, radius, a_in, a_out, 10)
        leave = _bezier(ring_at(a_out), _meet(ring_at(a_out), tangent(a_out), lane_out(radius), (co, so)),
                        lane_out(radius + 8.0), 8)
        paths.append(_polyline([lane_in(radius + arm)], join[:-1], quarter, leave[1:], [lane_out(radius + 200.0)]))
    ring_cars = min(ring_cars, m)
    lane_of = [0] * ring_cars + [1 + (k - ring_cars) % 4 for k in range(ring_cars, m)]
    rng = np.random.default_rng(seed + 7)
    scene = _place(paths, n, m, seed, {0: 0.0, 1: arm - 10.0, 2: arm - 10.0, 3: arm - 10.0, 4: arm - 10.0}, lane_of,
                   spacing, speed, "roundabout", [1, 0, 0, 0, 0])
    for k in range(ring_cars):   # the ring's cars, placed by hand a quarter turn apart
        x, y, h = _point_at(ring, k * radius * np.pi / 2)
        scene.x[:, k], scene.y[:, k], scene.heading[:, k] = x, y, h
        scene.path_id[:, k], scene.type_id[:, k] = 0, 0
        scene.speed[:, k] = rng.uniform(speed[0], speed[1], n)
    return scene


def crossing_log(duration_ms: int = 60000, seed: int = 0, rate_per_s: float = 0.25, speed=(8.0, 12.0),
                 length_m: float = 200.0, period_ms: int = 100):
    """A seeded two-stream crossing recording (a :class:`tactics2d_b200.dataset_parser.ReplayLog`, type rows unassigned):
    one stream drives west to east along y = -1.75, the other south to north along x = 1.75, crossing at the origin, each
    a Poisson process of ``rate_per_s`` arrivals per second at the start of a ``length_m`` approach, at a constant speed
    drawn from ``speed`` (m/s), one record every ``period_ms`` until the car leaves.  The recording ignores the other
    stream: replayed as logged, its cars drive through each other at the crossing.  Cars are 4.5 m x 1.9 m."""
    from .dataset_parser.replay import ReplayLog
    from .participant.element import Vehicle

    rng = np.random.default_rng(seed)
    half = length_m / 2.0
    tracks = []
    for stream in range(2):
        t = rng.exponential(1000.0 / rate_per_s)
        while t < duration_ms:
            tracks.append((stream, t, rng.uniform(speed[0], speed[1])))
            t += max(rng.exponential(1000.0 / rate_per_s), 3000.0)   # at least 3 s apart in a stream
    tracks.sort(key=lambda r: r[1])
    recs, first = [], []
    for stream, t, v in tracks:
        f0 = int(np.floor(t / period_ms)) * period_ms
        nfr = int(np.floor(length_m / (v * period_ms / 1000.0))) + 1
        s = -half + v * np.arange(nfr) * (period_ms / 1000.0)
        if stream == 0:
            r = np.stack([s, np.full(nfr, -1.75), np.zeros(nfr), np.full(nfr, v), np.zeros(nfr)], 1)
        else:
            r = np.stack([np.full(nfr, 1.75), s, np.full(nfr, np.pi / 2), np.zeros(nfr), np.full(nfr, v)], 1)
        recs.append(r.astype(np.float32))
        first.append(f0)
    K = len(recs)
    return ReplayLog(ids=np.arange(K, dtype=np.int64), first_ms=np.asarray(first, np.int32),
                     n_frames=np.asarray([len(r) for r in recs], np.int32), period_ms=np.full(K, period_ms, np.int32),
                     records=np.ascontiguousarray(np.concatenate(recs)), type_row=np.full(K, TYPE_INACTIVE, np.uint8),
                     cls=[Vehicle] * K, length=np.full(K, 4.5), width=np.full(K, 1.9))
