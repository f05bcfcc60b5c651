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
