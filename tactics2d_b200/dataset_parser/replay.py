"""Recorded traffic for log-replay episodes: LevelX tracks -> :class:`ReplayLog` -> :class:`ReplayEpisodes`.

A log-seeded episode keeps its recording: the ego (slot 0) is simulated from its logged state at the episode's start
``t0`` and driven by a policy, and every other slot is bound to a recorded track that ``BatchedWorld.set_log`` replays
on the device before every tick (``Trajectory.get_state(frame)`` of the reference, participant/trajectory/trajectory.py:97-113).
The contract is DESIGN.md section 1 "Log replay"."""

from __future__ import annotations

from dataclasses import dataclass, replace
from typing import Optional, Sequence, Tuple

import numpy as np

from ..types import TYPE_INACTIVE, TypeTable
from .parse_levelx import LevelXParser, template_row

LEVELX_PERIOD_MS = 40   # 25 Hz (parse_levelx.py: time_stamp = frame * 40)


@dataclass
class ReplayLog:
    """Tracks of one recording.  Track k: id ``ids[k]``, records ``records[rec_off[k] : rec_off[k] + n_frames[k]]`` =
    fp32 (x, y, heading, vx, vy) every ``period_ms[k]`` from ``first_ms[k]`` on (no gaps), heading in [0, 2 pi]
    (``fp32(np.mod(h, 2 pi))`` of the float64 heading, as ``initial_state_pool`` stores it); ``type_row[k]``: its row
    of the type table the log is bound with (255 until an episode builder assigns one)."""

    ids: np.ndarray          # int64 [K]
    first_ms: np.ndarray     # int32 [K]
    n_frames: np.ndarray     # int32 [K]
    period_ms: np.ndarray    # int32 [K]
    records: np.ndarray      # float32 [F, 5]
    type_row: np.ndarray     # uint8 [K]
    cls: list                # [K] participant class (Vehicle / Cyclist / Pedestrian)
    length: np.ndarray       # float64 [K]
    width: np.ndarray        # float64 [K]

    @property
    def rec_off(self) -> np.ndarray:
        return np.concatenate([[0], np.cumsum(self.n_frames.astype(np.int64))[:-1]]).astype(np.int64)

    @property
    def last_ms(self) -> np.ndarray:
        return self.first_ms.astype(np.int64) + (self.n_frames.astype(np.int64) - 1) * self.period_ms

    def __len__(self):
        return len(self.ids)

    def index(self, track_id) -> int:
        hit = np.nonzero(self.ids == int(track_id))[0]
        if len(hit) == 0:
            raise KeyError(f"track {track_id} is not in the log")
        return int(hit[0])

    def record(self, k: int, t_ms: int) -> np.ndarray:
        """Track k's record at time stamp ``t_ms`` (must be one of its frames)."""
        d = int(t_ms) - int(self.first_ms[k])
        j, r = divmod(d, int(self.period_ms[k]))
        if r != 0 or not 0 <= j < int(self.n_frames[k]):
            raise KeyError(f"track {int(self.ids[k])} has no frame at {t_ms} ms")
        return self.records[self.rec_off[k] + j]

    def track_paths(self, tolerance: float = 0.1, extend: float = 30.0):
        """Paths for reactive replay (``BatchedWorld.set_reactive_replay``; DESIGN.md section 1 "Reactive replay"):
        ``(paths, track_path, desired_speed)``.  Track k's path is its logged (x, y) without repeated points, simplified
        with Douglas-Peucker at ``tolerance`` metres and extended straight by ``extend`` metres along its last segment
        (so that the lateral controller does not turn back at its end), all in float64, then fp32; ``track_path[k]``
        (int16 [K]) indexes ``paths``.  ``desired_speed[k]`` (fp32 [K]) is the track's highest logged speed.  A track
        whose path has no segment of non-zero length, or whose highest speed is not > 0 (a parked car), stays plain
        replay: ``track_path[k] = -1``.  A logged stop (at a signal, say) is not reproduced: the IDM only stops behind a
        leader, or, with yielding bound (``BatchedWorld.set_yielding``), before a conflict zone of crossing paths."""
        if not tolerance >= 0.0 or not extend >= 0.0:
            raise ValueError("tolerance and extend must be >= 0")
        rec = np.asarray(self.records, np.float32).astype(np.float64)
        speed = np.sqrt(rec[:, 3] * rec[:, 3] + rec[:, 4] * rec[:, 4])
        paths, track_path = [], np.full(len(self), -1, np.int16)
        desired = np.zeros(len(self), np.float32)
        for k, (a, n) in enumerate(zip(self.rec_off, self.n_frames)):
            desired[k] = np.float32(speed[a:a + n].max())
            xy = rec[a:a + n, :2]
            keep = np.concatenate([[True], np.any(xy[1:] != xy[:-1], axis=1)])
            xy = douglas_peucker(xy[keep], tolerance)
            if len(xy) < 2 or not desired[k] > 0.0:
                continue
            d = xy[-1] - xy[-2]
            end = xy[-1] + float(extend) * d / np.hypot(d[0], d[1])
            track_path[k] = len(paths)
            paths.append(np.concatenate([xy, end[None]], 0).astype(np.float32))
        return paths, track_path, desired

    @classmethod
    def from_levelx(cls, parser: LevelXParser, file, folder: str, time_range=None, ids=None) -> "ReplayLog":
        """The tracks of a LevelX recording (``LevelXParser._frames``: highD's box centres and (-pi, pi] headings, the degree
        headings of inD / rounD / exiD / uniD), in ascending id order."""
        t, meta = parser._frames(file, folder, time_range, ids)
        info = {int(r[parser.id_key]): (parser._CLASS_MAPPING[r["class"]], float(r[parser.key_length]), float(r[parser.key_width]))
                for _, r in meta.iterrows()}
        out = dict(ids=[], first_ms=[], n_frames=[], cls=[], length=[], width=[])
        recs = []
        for id_, g in t.groupby(parser.id_key):
            g = g.sort_values("time_stamp")
            ts = g["time_stamp"].to_numpy().astype(np.int64)
            if len(ts) > 1 and not np.all(np.diff(ts) == LEVELX_PERIOD_MS):
                raise ValueError(f"track {int(id_)} has gaps: LevelX tracks are continuous from initialFrame to finalFrame")
            rec = np.stack([g["xCenter"].to_numpy(np.float64), g["yCenter"].to_numpy(np.float64),
                            np.mod(g["heading_"].to_numpy(np.float64), 2 * np.pi), g["xVelocity"].to_numpy(np.float64),
                            g["yVelocity"].to_numpy(np.float64)], 1).astype(np.float32)
            c, L, W = info[int(id_)]
            out["ids"].append(int(id_)); out["first_ms"].append(int(ts[0])); out["n_frames"].append(len(ts))
            out["cls"].append(c); out["length"].append(L); out["width"].append(W)
            recs.append(rec)
        if not recs:
            raise ValueError("no tracks in the selected part of the recording")
        k = len(recs)
        return cls(ids=np.asarray(out["ids"], np.int64), first_ms=np.asarray(out["first_ms"], np.int32),
                   n_frames=np.asarray(out["n_frames"], np.int32), period_ms=np.full(k, LEVELX_PERIOD_MS, np.int32),
                   records=np.ascontiguousarray(np.concatenate(recs, 0)), type_row=np.full(k, TYPE_INACTIVE, np.uint8),
                   cls=out["cls"], length=np.asarray(out["length"]), width=np.asarray(out["width"]))


@dataclass
class ReplayEpisodes:
    """Episode rows over a :class:`ReplayLog`, ready for ``BatchedWorld.reset`` + ``BatchedWorld.set_log`` (or
    ``BatchedTrafficEnv(..., replay=episodes)``): row p starts at ``t0[p]``; ``pool`` / ``type_id`` [P, M] are the initial
    states (slot 0 the ego's logged state at t0, bit for bit, with its class's kinematic row; the replayed slots are
    written by the replay at the reset itself), ``row_track`` [P, M] binds slots to tracks (-1: not replayed),
    ``dropped[p]``: tracks of row p's window that did not fit its M - 1 slots.  Episodes built with slot reuse bind their
    slots with ``schedule = (slot_off [P * M + 1], slot_track [E])`` instead (``BatchedWorld.set_log``) and have no
    ``row_track``."""

    log: ReplayLog
    table: TypeTable
    pool: dict
    type_id: np.ndarray
    row_track: Optional[np.ndarray]
    t0: np.ndarray
    dropped: np.ndarray
    schedule: Optional[Tuple[np.ndarray, np.ndarray]] = None
    ego_track: Optional[np.ndarray] = None   # int64 [P]: the log index of every row's ego track (build_replay_episodes)

    def binding(self) -> dict:
        """The slot binding as ``BatchedWorld.set_log`` keywords: ``row_track=`` or ``schedule=``."""
        return dict(row_track=self.row_track) if self.schedule is None else dict(schedule=self.schedule)

    def ego_routes(self, horizon_ms: Optional[int] = None):
        """Routes that make every row's ego follow its own logged track: ``(paths, route_id)`` for
        ``BatchedWorld.set_paths`` / ``set_routes`` (or ``BatchedTrafficEnv(route=dict(paths=..., route_id=...))``).  Path p
        is the ego track's recorded (x, y) every 40 ms from ``t0[p]`` on, to its end or to ``t0[p] + horizon_ms``;
        ``route_id`` [P, M] int16 routes slot 0 of row p along path p and no other slot.  A track with a single frame left
        gives a path of one repeated point, which has no segment of non-zero length: no route."""
        if self.ego_track is None:
            raise ValueError("these episodes do not know their ego tracks: build them with build_replay_episodes")
        log = self.log
        off, first, period, nf = log.rec_off, log.first_ms.astype(np.int64), log.period_ms.astype(np.int64), log.n_frames
        paths = []
        for p, k in enumerate(self.ego_track):
            k = int(k)
            j0 = (int(self.t0[p]) - int(first[k])) // int(period[k])
            j1 = int(nf[k]) if horizon_ms is None else min(int(nf[k]), j0 + int(horizon_ms) // int(period[k]) + 1)
            xy = np.ascontiguousarray(log.records[off[k] + j0:off[k] + j1, :2], dtype=np.float32)
            paths.append(xy if len(xy) >= 2 else np.repeat(xy, 2, 0))
        M = self.type_id.shape[1]
        route_id = np.full((len(paths), M), -1, np.int16)
        route_id[:, 0] = np.arange(len(paths))
        return paths, route_id

    def scene(self, segments=None, bounds=None, name: str = "replay"):
        """A :class:`tactics2d_b200.synthetic.Scene` of the P rows (one scenario per row) on the given map."""
        from ..synthetic import Scene

        p = self.pool
        seg = None if segments is None else np.ascontiguousarray(segments, dtype=np.float32).reshape(-1, 4)
        return Scene(self.table, p["x"], p["y"], p["heading"], p["speed"], p["vx"], p["vy"], self.type_id, seg, bounds, name,
                     dict(replay=True))


def douglas_peucker(xy, tolerance: float):
    """The Douglas-Peucker simplification of the polyline ``xy`` [V, 2] (float64): the end points, and recursively the
    vertex farthest from the chord between two kept ones (the first of equals) while that distance exceeds
    ``tolerance``.  Distances are to the chord segment."""
    xy = np.asarray(xy, np.float64)
    if len(xy) < 3:
        return xy.copy()
    keep = np.zeros(len(xy), bool)
    keep[0] = keep[-1] = True
    stack = [(0, len(xy) - 1)]
    while stack:
        i, j = stack.pop()
        if j - i < 2:
            continue
        a, b, p = xy[i], xy[j], xy[i + 1:j]
        ab = b - a
        L2 = ab[0] * ab[0] + ab[1] * ab[1]
        t = np.zeros(len(p)) if L2 == 0.0 else np.clip(((p - a) @ ab) / L2, 0.0, 1.0)
        d = np.hypot(*(p - (a + t[:, None] * ab)).T)
        f = int(np.argmax(d))
        if d[f] > tolerance:
            keep[i + 1 + f] = True
            stack += [(i, i + 1 + f), (i + 1 + f, j)]
    return xy[keep]


def _speed(vx, vy):
    vx, vy = np.float64(vx), np.float64(vy)
    return np.float32(np.sqrt(vx * vx + vy * vy))


def build_replay_episodes(log: ReplayLog, m_participants: int, t0s: Sequence[int], ego_tracks: Sequence[int],
                          type_table: Optional[TypeTable] = None, horizon_ms: Optional[int] = None,
                          reuse_slots: bool = False) -> ReplayEpisodes:
    """Row p: the ego is track ``ego_tracks[p]`` (a track id), simulated from its record at ``t0s[p]`` (which must be one of
    its frames); slots 1..M-1 replay the other tracks present somewhere in the window [t0, t0 + horizon_ms] (to the end
    of the log without a horizon), ordered by (first time stamp, id); the ego's own track is never replayed.
    ``type_table`` (default ``TypeTable.from_templates("kinematics")``) gets one static twin per class row the log uses
    (``TypeTable.with_static_twins``): every track's ``type_row`` is the twin of its class row.

    ``reuse_slots``: instead of one track per slot, each slot gets a schedule (``ReplayEpisodes.schedule``): in that same
    order, every track goes to the lowest slot in 1..M-1 whose last track ends strictly before the track's first stamp
    (greedy interval partitioning, so a row uses exactly as many slots as the most tracks of its window present at one
    time), and ``dropped[p]`` counts the tracks that found no such slot.  A slot's initial type is that of its track
    present at t0 (255 if none)."""
    table = type_table if type_table is not None else TypeTable.from_templates("kinematics")
    M = int(m_participants)
    t0s = [int(v) for v in t0s]
    if M < 1:
        raise ValueError("m_participants must be >= 1")
    if len(t0s) != len(ego_tracks) or not t0s:
        raise ValueError("give one ego track per start time (and at least one row)")
    lo, hi = int(log.first_ms.min()), int(log.last_ms.max())
    class_row = np.asarray([template_row(table.rows, c, L, W) for c, L, W in zip(log.cls, log.length, log.width)], np.int64)
    table, twin = table.with_static_twins(class_row)
    type_row = np.asarray([twin[int(r)] for r in class_row], np.uint8)
    first, last = log.first_ms.astype(np.int64), log.last_ms
    order = np.lexsort((log.ids, first))                          # (first stamp, id)
    P = len(t0s)
    pool = {k: np.zeros((P, M), np.float32) for k in ("x", "y", "heading", "speed", "vx", "vy")}
    tid = np.full((P, M), TYPE_INACTIVE, np.uint8)
    row_track = np.full((P, M), -1, np.int32)
    slots = [[[] for _ in range(M)] for _ in range(P)] if reuse_slots else None
    dropped = np.zeros(P, np.int64)
    for p, (t0, ego_id) in enumerate(zip(t0s, ego_tracks)):
        if not lo <= t0 <= hi:
            raise ValueError(f"row {p}: t0 = {t0} ms lies outside the log [{lo}, {hi}] ms")
        e = log.index(ego_id)
        if not first[e] <= t0 <= last[e]:
            raise ValueError(f"row {p}: the ego track {ego_id} is absent at t0 = {t0} ms")
        rec = log.record(e, t0)                                    # KeyError when t0 falls between its frames
        pool["x"][p, 0], pool["y"][p, 0], pool["heading"][p, 0] = rec[0], rec[1], rec[2]
        pool["vx"][p, 0], pool["vy"][p, 0] = rec[3], rec[4]
        pool["speed"][p, 0] = _speed(rec[3], rec[4])
        tid[p, 0] = class_row[e]
        end = np.inf if horizon_ms is None else t0 + int(horizon_ms)
        others = [int(k) for k in order if k != e and last[k] >= t0 and first[k] <= end]
        if reuse_slots:
            free_after = np.full(M, np.iinfo(np.int64).min, np.int64)   # slot m takes a track starting after this
            free_after[0] = np.iinfo(np.int64).max                       # (slot 0 is the ego's)
            for k in others:
                m = int(np.argmax(free_after < first[k]))
                if not free_after[m] < first[k]:
                    dropped[p] += 1
                    continue
                slots[p][m].append(k)
                free_after[m] = last[k]
                if first[k] <= t0 <= last[k]:
                    tid[p, m] = type_row[k]
            continue
        dropped[p] = max(0, len(others) - (M - 1))
        for m, k in enumerate(others[:M - 1], start=1):
            row_track[p, m] = k
            if first[k] <= t0 <= last[k]:
                tid[p, m] = type_row[k]
    t0_arr = np.asarray(t0s, np.int32)
    ego_track = np.asarray([log.index(e) for e in ego_tracks], np.int64)
    if not reuse_slots:
        return ReplayEpisodes(replace(log, type_row=type_row), table, pool, tid, row_track, t0_arr, dropped,
                              ego_track=ego_track)
    flat = [s for row in slots for s in row]
    slot_off = np.concatenate([[0], np.cumsum([len(s) for s in flat])]).astype(np.int32)
    slot_track = np.asarray([k for s in flat for k in s], np.int32)
    return ReplayEpisodes(replace(log, type_row=type_row), table, pool, tid, None, t0_arr, dropped, (slot_off, slot_track),
                          ego_track)
