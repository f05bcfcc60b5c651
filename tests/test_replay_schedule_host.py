"""Slot schedules for log replay on the host: the reusing episode builder's properties on seeded logs, the schedule oracle's
known answers (tests/schedule_oracle.py) and the C ABI's new entry point."""

from types import SimpleNamespace

import numpy as np
import pytest

from oracle import replay as R
from tactics2d_b200 import synthetic
from tactics2d_b200.dataset_parser import build_replay_episodes
from tactics2d_b200.types import TYPE_INACTIVE
from tests import schedule_oracle as S

KEYS = ("x", "y", "heading", "speed", "vx", "vy")


def _ego(log, ep, p):
    """The track whose record at t0 is row p's ego state."""
    t0 = int(ep.t0[p])
    first, last = log.first_ms.astype(np.int64), log.last_ms
    want = [ep.pool[c][p, 0] for c in ("x", "y", "heading", "vx", "vy")]
    hits = [k for k in range(len(log)) if first[k] <= t0 <= last[k] and (t0 - first[k]) % log.period_ms[k] == 0
            and np.array_equal(log.record(k, t0), want)]
    assert len(hits) == 1
    return hits[0]


def _windows(log, ep, horizon_ms):
    """Row p's candidates (the builder's order: (first stamp, id), the ego's track left out)."""
    first, last = log.first_ms.astype(np.int64), log.last_ms
    order = np.lexsort((log.ids, first))
    out = []
    for p in range(len(ep.t0)):
        t0, ego = int(ep.t0[p]), _ego(log, ep, p)
        end = np.inf if horizon_ms is None else t0 + horizon_ms
        out.append((ego, [int(k) for k in order if k != ego and last[k] >= t0 and first[k] <= end]))
    return out


def _slots(ep, p):
    off, trk = ep.schedule
    M = ep.type_id.shape[1]
    return [trk[off[p * M + m]:off[p * M + m + 1]].tolist() for m in range(M)]


def _concurrency(first, last, ks):
    """The most of the intervals [first_k, last_k] holding one instant (a sweep: starts before ends at equal stamps)."""
    ev = sorted([(int(first[k]), 0) for k in ks] + [(int(last[k]), 1) for k in ks])
    cur = best = 0
    for _, end in ev:
        cur += -1 if end else 1
        best = max(best, cur)
    return best


def _first_come(first, last, ks, cap):
    """Tracks refused by a road with ``cap`` places, taken in order: a track gets in when fewer than ``cap`` admitted tracks
    are still present at its first stamp."""
    admitted, refused = [], 0
    for k in ks:
        if sum(1 for a in admitted if last[a] >= first[k]) < cap:
            admitted.append(k)
        else:
            refused += 1
    return refused


@pytest.mark.parametrize("m,seed", [(64, 0), (64, 5), (12, 1), (6, 2)])
def test_reusing_builder_partitions_each_window(m, seed):
    log = synthetic.highway_log(120000, seed)
    ep = synthetic.highway_episodes(24, m, seed=seed, duration_ms=120000, horizon_ms=60000, log=log)
    assert ep.row_track is None
    first, last = ep.log.first_ms.astype(np.int64), ep.log.last_ms
    off, trk = ep.schedule
    assert off.dtype == np.int32 and trk.dtype == np.int32 and off[0] == 0 and off[-1] == len(trk) and (np.diff(off) >= 0).all()
    n_over = 0
    for p, (ego, cand) in enumerate(_windows(ep.log, ep, 60000)):
        slots = _slots(ep, p)
        assert slots[0] == []                                                     # slot 0 is the ego's
        flat = [k for s in slots for k in s]
        assert len(flat) == len(set(flat)) and ego not in flat and set(flat) <= set(cand)
        for s in slots:
            assert all(last[a] < first[b] for a, b in zip(s, s[1:]))            # strictly increasing, disjoint
        conc = _concurrency(first, last, cand)
        if conc <= m - 1:
            assert sum(1 for s in slots if s) == conc and ep.dropped[p] == 0
        else:
            n_over += 1
            assert ep.dropped[p] == _first_come(first, last, cand, m - 1) > 0
            assert len(flat) + ep.dropped[p] == len(cand)
        t0 = int(ep.t0[p])
        for mm, s in enumerate(slots[1:], start=1):                               # the pool's type: the track present at t0
            on = [k for k in s if first[k] <= t0 <= last[k]]
            assert ep.type_id[p, mm] == (ep.log.type_row[on[0]] if on else TYPE_INACTIVE)
    if m < 20:
        assert n_over > 0


def test_reusing_builder_on_a_random_walk_log():
    src = synthetic.replay_episodes(4, 8, 600, seed=3, duration_ms=12000, max_frames=80).log
    first = src.first_ms.astype(np.int64)
    on_grid = np.nonzero(first % 40 == 0)[0][:20]
    t0 = [int(first[k]) for k in on_grid]
    ids = [int(src.ids[k]) for k in on_grid]
    for m in (4, 16, 200):
        ep = build_replay_episodes(src, m, t0, ids, reuse_slots=True)
        a, b = ep.log.first_ms.astype(np.int64), ep.log.last_ms
        for p in range(len(t0)):
            cand = [int(k) for k in np.lexsort((src.ids, a)) if k != on_grid[p] and b[k] >= t0[p]]
            slots = _slots(ep, p)
            conc = _concurrency(a, b, cand)
            if conc <= m - 1:
                assert sum(1 for s in slots if s) == conc and ep.dropped[p] == 0
            else:
                assert ep.dropped[p] == _first_come(a, b, cand, m - 1)


def test_non_reusing_builder_is_unchanged():
    """``reuse_slots=False`` (the default): the first M - 1 candidates, one per slot, in order, as before schedules."""
    log = synthetic.highway_log(60000, 3)
    for reuse in (None, False):
        kw = {} if reuse is None else dict(reuse_slots=reuse)
        rng = np.random.default_rng(0)
        ego = rng.choice(np.nonzero(log.first_ms < 30000)[0], 12)
        t0 = (log.first_ms[ego] + 40 * rng.integers(0, 20, 12)).tolist()
        ep = build_replay_episodes(log, 16, t0, log.ids[ego].tolist(), horizon_ms=20000, **kw)
        assert ep.schedule is None and ep.binding().keys() == {"row_track"}
        first, last = ep.log.first_ms.astype(np.int64), ep.log.last_ms
        order = np.lexsort((log.ids, first))
        for p in range(12):
            cand = [int(k) for k in order if k != ego[p] and last[k] >= t0[p] and first[k] <= t0[p] + 20000]
            want = np.full(16, -1)
            want[1:1 + min(15, len(cand))] = cand[:15]
            assert np.array_equal(ep.row_track[p], want) and ep.dropped[p] == max(0, len(cand) - 15)
            for m in range(1, 16):
                k = want[m]
                on = k >= 0 and first[k] <= t0[p] <= last[k]
                assert ep.type_id[p, m] == (ep.log.type_row[k] if on else TYPE_INACTIVE)
            assert np.array_equal([ep.pool[c][p, 0] for c in ("x", "y", "heading", "vx", "vy")], log.record(ego[p], t0[p]))
        # the reusing builder agrees on everything but the binding (same ego, pool, table and track types)
        ep2 = build_replay_episodes(log, 16, t0, log.ids[ego].tolist(), horizon_ms=20000, reuse_slots=True)
        assert ep2.table.rows == ep.table.rows and np.array_equal(ep2.log.type_row, ep.log.type_row)
        for k in KEYS:
            assert np.array_equal(ep2.pool[k], ep.pool[k])
        assert np.array_equal(ep2.type_id[:, 0], ep.type_id[:, 0])


def test_highway_replay_keeps_every_road_user_for_100_s():
    """M = 64 over a 100 s horizon: with slot reuse every road user present at a tick is in a slot; without it the road
    empties."""
    log = synthetic.highway_log(200000, 0)
    P, M = 40, 64
    ep = synthetic.highway_episodes(P, M, seed=0, log=log)
    ep0 = synthetic.highway_episodes(P, M, seed=0, log=log, reuse_slots=False)
    assert np.array_equal(ep.t0, ep0.t0) and (ep.dropped == 0).all()
    first, last = ep.log.first_ms.astype(np.int64), ep.log.last_ms
    ego = [_ego(ep.log, ep, p) for p in range(P)]
    rows = np.arange(P)
    missing_reuse = missing_plain = present_total = 0
    for step in range(0, 1000, 10):
        t = ep.t0.astype(np.int64) + (step + 1) * 100
        _, track = S.active_track(ep.log, ep.t0, *ep.schedule, rows, np.full(P, step), 100, 1)
        _, pres0, _, _ = R.sample(ep0.log, ep0.t0, ep0.row_track, rows, np.full(P, step), 100, 1)
        for p in range(P):
            here = set(np.nonzero((first <= t[p]) & (t[p] <= last))[0].tolist()) - {ego[p]}
            present_total += len(here)
            shown = set(track[p][track[p] >= 0].tolist())
            assert shown == here, (p, step)
            missing_reuse += len(here - shown)
            plain = set(ep0.row_track[p][pres0[p]].tolist())
            missing_plain += len(here - plain)
    assert missing_reuse == 0 and present_total > 40 * 100 * 10
    assert missing_plain > present_total // 2                                     # the one-track-per-slot episode empties


def _log(first, period, recs, type_row=None):
    recs = [np.asarray(r, np.float32).reshape(-1, 5) for r in recs]
    return SimpleNamespace(first_ms=np.asarray(first, np.int32), period_ms=np.asarray(period, np.int32),
                           n_frames=np.asarray([len(r) for r in recs], np.int32), records=np.concatenate(recs),
                           type_row=np.asarray(type_row if type_row is not None else [7] * len(recs), np.uint8))


def _rec(n, base):
    return [[base + 10.0 * j, base - 2.0 * j, 0.1 * j + 0.05, 3.0 + j, -1.0 + 0.5 * j] for j in range(n)]


def test_oracle_switch_from_a_to_b_across_one_tick():
    # A on [0, 200], B on [240, 400] (B one period after A): at t = 200 A's last record, at t = 300 B between frames
    log = _log([0, 240], [40, 40], [_rec(6, 0.0), _rec(5, 500.0)], [7, 9])
    sched = (np.asarray([0, 2], np.int32), np.asarray([0, 1], np.int32))
    rep, pres, s, tid, trk = S.sample(log, [100], *sched, [0], [0], 100, 1)       # t = 200
    assert rep[0, 0] and pres[0, 0] and trk[0, 0] == 0 and tid[0, 0] == 7
    assert np.array_equal([s[k][0, 0] for k in ("x", "y", "heading", "vx", "vy")], np.asarray(_rec(6, 0.0)[5], np.float32))
    rep, pres, s, tid, trk = S.sample(log, [100], *sched, [0], [1], 100, 1)       # t = 300: B's frames 1 (280), 2 (320)
    assert trk[0, 0] == 1 and tid[0, 0] == 9
    _, _, sb, _ = R.sample(log, [100], [[1]], [0], [1], 100, 1)
    for k in KEYS:
        assert s[k][0, 0].view(np.uint32) == sb[k][0, 0].view(np.uint32), k
    a, b = (np.asarray(_rec(5, 500.0)[j], np.float32).astype(np.float64) for j in (1, 2))
    assert s["x"][0, 0] == np.float32(a[0] + 0.5 * (b[0] - a[0]))


def test_oracle_gap_between_tracks_keeps_the_last_state():
    log = _log([0, 400], [40, 40], [_rec(3, 0.0), _rec(3, 50.0)], [7, 9])       # A on [0, 80], B on [400, 480]
    sched = (np.asarray([0, 2], np.int32), np.asarray([0, 1], np.int32))
    st = {k: np.full((1, 1), -3.0, np.float32) for k in KEYS}
    st1, tid1 = S.apply(st, np.zeros((1, 1), np.uint8), log, [0], *sched, [0], [0], 80, 0)   # t = 0: A
    assert tid1[0, 0] == 7 and st1["x"][0, 0] == 0.0
    st2, tid2 = S.apply(st1, tid1, log, [0], *sched, [0], [2], 80, 0)           # t = 160: in the gap
    assert tid2[0, 0] == TYPE_INACTIVE
    for k in KEYS:
        assert st2[k][0, 0] == st1[k][0, 0]
    _, _, _, _, trk = S.sample(log, [0], *sched, [0], [2], 80, 0)
    assert trk[0, 0] == -1
    st3, tid3 = S.apply(st2, tid2, log, [0], *sched, [0], [5], 80, 0)           # t = 400: B's first record
    assert tid3[0, 0] == 9 and st3["x"][0, 0] == 50.0
    # a slot without entries is not replayed: its type stays
    off = np.asarray([0, 2, 2], np.int32)
    _, t4 = S.apply({k: np.zeros((1, 2), np.float32) for k in KEYS}, np.full((1, 2), 4, np.uint8), log, [0], off, sched[1],
                    [0], [2], 80, 0)
    assert t4.tolist() == [[TYPE_INACTIVE, 4]]


def test_oracle_entry_starting_off_the_period_grid():
    log = _log([0, 213], [40, 40], [_rec(3, 0.0), _rec(4, 70.0)], [7, 9])       # B at 213, 253, 293, 333
    sched = (np.asarray([0, 2], np.int32), np.asarray([0, 1], np.int32))
    for t, want in ((212, -1), (213, 1), (233, 1), (333, 1), (334, -1)):
        _, pres, s, tid, trk = S.sample(log, [t], *sched, [0], [0], 50, 0)
        assert trk[0, 0] == want, t
        if want == 1:
            _, _, sb, _ = R.sample(log, [t], [[1]], [0], [0], 50, 0)
            assert all(s[k][0, 0].view(np.uint32) == sb[k][0, 0].view(np.uint32) for k in KEYS)
    _, _, s, _, _ = S.sample(log, [233], *sched, [0], [0], 50, 0)                # w = 0.5 between B's first two frames
    a, b = (np.asarray(_rec(4, 70.0)[j], np.float32).astype(np.float64) for j in (0, 1))
    assert s["y"][0, 0] == np.float32(a[1] + 0.5 * (b[1] - a[1]))


def test_oracle_long_schedule_and_late_start():
    # 300 tracks of 3 frames, 20 ms apart: [100 i + 7, 100 i + 47]; the slot starts after t0 = 0
    n = 300
    log = _log([100 * i + 7 for i in range(n)], [20] * n, [_rec(3, float(i)) for i in range(n)], [i % 251 for i in range(n)])
    off = np.asarray([0, n], np.int32)
    trk = np.arange(n, dtype=np.int32)
    steps = np.arange(0, 30001, 13)
    _, pres, s, tid, got = S.sample(log, [0], off, trk, np.zeros(len(steps), np.int64), steps, 1, 0)
    want = np.where(((steps - 7) % 100 <= 40) & (steps >= 7) & (steps <= 100 * (n - 1) + 47), (steps - 7) // 100, -1)
    assert np.array_equal(got[:, 0], want) and (want[steps < 7] == -1).all() and (want >= 250).any()
    assert np.array_equal(tid[:, 0], np.where(want >= 0, want % 251, TYPE_INACTIVE).astype(np.uint8))
    on = want >= 0
    _, _, sb, _ = R.sample(log, np.zeros(len(steps), np.int64), np.maximum(want, 0)[:, None], np.arange(len(steps)), steps, 1, 0)
    for k in KEYS:
        assert np.array_equal(s[k][on, 0].view(np.uint32), sb[k][on, 0].view(np.uint32)), k


def test_set_log_schedule_is_part_of_the_abi():
    import ctypes
    from tactics2d_b200 import _lib

    assert "t2d_set_log_schedule" in _lib.SYMBOLS and "t2d_set_log" in _lib.SYMBOLS
    assert ctypes.sizeof(_lib.LogC) == 4 + 4 + 8 * 5 + 4 + 4 + 8 * 4
