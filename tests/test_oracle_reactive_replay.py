"""Reactive replay in float64 (tests/reactive_replay_oracle.py) on known answers - the handover boundaries, the paths
``ReplayLog.track_paths`` builds, parked tracks - and the closed loop of tests/reactive_scenes.py on the CPU: plain
replay drives through a stopped ego, reactive replay stops behind it, and without anything in the way a reactive track
keeps to its log."""

import numpy as np
import pytest

from tactics2d_b200.dataset_parser.replay import ReplayLog, douglas_peucker
from tactics2d_b200.participant.element import Vehicle
from tests import reactive_replay_oracle as RO
from tests import reactive_scenes as RS

INTERVAL = 100


def _log(first, n_frames, period=40, speed=10.0):
    """Straight tracks along +x at ``speed``, one per entry of ``first``."""
    recs = []
    for k, n in enumerate(n_frames):
        s = speed * np.arange(n) * period / 1000.0
        recs.append(np.stack([s, np.full(n, 4.0 * k), np.zeros(n), np.full(n, speed), np.zeros(n)], 1))
    K = len(first)
    return ReplayLog(ids=np.arange(K, dtype=np.int64), first_ms=np.asarray(first, np.int32),
                     n_frames=np.asarray(n_frames, np.int32), period_ms=np.full(K, period, np.int32),
                     records=np.concatenate(recs).astype(np.float32), type_row=np.full(K, 1, np.uint8), cls=[Vehicle] * K,
                     length=np.full(K, 4.5), width=np.full(K, 1.9))


def _world(M):
    w = {k: np.full((1, M), 7.0, np.float32) for k in ("x", "y", "heading", "speed", "vx", "vy")}
    w.update(type_id=np.full((1, M), 200, np.uint8), drive_path=np.full((1, M), 9, np.int16),
             slot_desired_speed=np.full((1, M), 3.0, np.float32), pid_state=np.full((1, M, 6), 5.0),
             last_accel=np.full((1, M), 2.0, np.float32))
    return w


def _k7(log, step, mask=None, t0=0, track_path=None):
    K = len(log)
    tp = np.arange(K, dtype=np.int16) if track_path is None else np.asarray(track_path, np.int16)
    row_track = np.arange(K, dtype=np.int32)[None]
    return RO.apply(_world(K), log, [t0], [0], [step], INTERVAL, tp, np.zeros(K, np.uint8), np.arange(1, K + 1) * 5.0,
                    1 if mask is None else 0, mask, row_track=row_track)


def test_handover_on_the_sample_of_the_first_stamp():
    log = _log([300], [40])
    w = _k7(log, 2)                                   # t = 300: first_k == t
    assert w["handover"][0, 0] and w["type_id"][0, 0] == 1 and w["drive_path"][0, 0] == 0
    assert w["x"][0, 0] == 0.0 and w["slot_desired_speed"][0, 0] == 5.0
    assert (w["pid_state"][0, 0, :3] == 0).all() and (w["pid_state"][0, 0, 3:] == 5).all() and w["last_accel"][0, 0] == 0
    w = _k7(log, 3)                                   # t = 400: simulated, the state is kept
    assert w["simulated"][0, 0] and w["type_id"][0, 0] == 0 and w["x"][0, 0] == 7.0 and w["drive_path"][0, 0] == 0
    assert w["pid_state"][0, 0, 0] == 5.0 and w["last_accel"][0, 0] == 2.0


def test_handover_one_ms_after_the_previous_sample():
    log = _log([201], [40])
    assert not _k7(log, 1)["handover"][0, 0]          # t = 200: not there yet
    assert _k7(log, 1)["type_id"][0, 0] == 255
    w = _k7(log, 2)                                   # t = 300: t - interval = 200 < 201 <= 300
    assert w["handover"][0, 0]
    a, b = np.float64(log.records[2, 0]), np.float64(log.records[3, 0])   # t - first = 99 ms: frame 2 + 19 / 40
    assert w["x"][0, 0] == np.float32(a + (19.0 / 40.0) * (b - a))
    log = _log([200], [40])
    assert _k7(log, 1)["handover"][0, 0] and _k7(log, 2)["simulated"][0, 0]


def test_track_present_at_t0_is_handed_over_by_the_reset():
    log = _log([-400], [40])
    w = _k7(log, 0, mask=np.array([True]))
    assert w["handover"][0, 0] and w["x"][0, 0] == log.records[10, 0]
    assert _k7(log, 0)["simulated"][0, 0]             # the first tick (t = 100) simulates it
    assert not _k7(log, 0, mask=np.array([False]))["handover"].any()


def test_exit_at_the_last_stamp():
    log = _log([0, 0], [18, 19])                      # last stamps 680 and 720
    w = _k7(log, 6)                                   # t = 700
    assert w["type_id"][0].tolist() == [255, 0] and w["drive_path"][0].tolist() == [-1, 1]
    log = _log([0], [18], period=40)
    w = _k7(log, 5, t0=-20)                           # t = 580 ... last 680; t = 680 is the last stamp itself
    assert w["simulated"][0, 0]
    w = _k7(log, 6, t0=-20)                           # t = 680 == last_k: present
    assert w["simulated"][0, 0] and w["type_id"][0, 0] == 0
    w = _k7(log, 6, t0=-19)                           # t = 681 == last_k + 1: gone
    assert w["type_id"][0, 0] == 255 and w["drive_path"][0, 0] == -1


def test_plain_tracks_and_empty_slots_are_replayed_as_before():
    log = _log([0, 0], [40, 40])
    w = _k7(log, 0, track_path=[-1, 0])
    assert w["type_id"][0].tolist() == [1, 0] and w["drive_path"][0].tolist() == [-1, 0]
    assert w["x"][0, 0] == np.float32(10.0 * 0.1) and w["slot_desired_speed"][0, 0] == 3.0


def test_douglas_peucker():
    x = np.linspace(0.0, 100.0, 201)
    assert douglas_peucker(np.stack([x, 0.04 * np.sin(x)], 1), 0.1).shape == (2, 2)
    bend = np.stack([x, np.where(x > 50.0, x - 50.0, 0.0)], 1)
    assert douglas_peucker(bend, 0.1).tolist() == [[0.0, 0.0], [50.0, 0.0], [100.0, 50.0]]
    assert douglas_peucker(np.stack([x, 0.2 * np.sin(x)], 1), 0.1).shape[0] > 10


def test_track_paths_extend_and_take_the_top_speed():
    log = _log([0], [26], speed=10.0)
    log.records[5, 3] = 12.0                          # a faster frame: the desired speed
    paths, tp, ds = log.track_paths(tolerance=0.1, extend=30.0)
    assert tp.tolist() == [0] and ds.tolist() == [12.0]
    assert np.allclose(paths[0], [[0.0, 0.0], [10.0, 0.0], [40.0, 0.0]])


def test_parked_and_single_point_tracks_stay_plain():
    log = _log([0, 0, 0], [30, 30, 1], speed=10.0)
    log.records[30:60, 0] = 5.0                       # track 1 parked: one repeated point, speed 10 in its records
    log.records[30:60, 3] = 0.0
    paths, tp, ds = log.track_paths()
    assert tp.tolist() == [0, -1, -1] and len(paths) == 1
    log = _log([0], [30], speed=0.0)                  # moving points but no logged speed
    log.records[:, 0] = np.arange(30)
    assert log.track_paths()[1].tolist() == [-1]


def _run(scene, reactive, ticks):
    from tactics2d_b200.types import TypeTable  # noqa: F401

    eps = scene[0]
    paths, tp, ds = eps.log.track_paths()
    drive = np.zeros(len(eps.log), np.uint8)
    rows = eps.table.rows
    for k, r in enumerate(eps.log.type_row):
        drive[k] = next(i for i, q in enumerate(rows) if q.model != 4 and q.half_len == rows[r].half_len
                        and q.half_wid == rows[r].half_wid and q.name == rows[r].name)
    return RO.rollout(eps, eps.table, RS.ctab(), paths, tp, drive, ds, ticks, RS.HALF_WIDTH, RS.MAX_RANGE, reactive)


@pytest.fixture(scope="module")
def stopped():
    return RS.stopped_ego()


def test_plain_replay_drives_through_the_stopped_ego(stopped):
    out = _run(stopped, False, 300)
    assert np.any(out["ego_hits"])


def test_reactive_replay_stops_behind_the_stopped_ego(stopped):
    eps, ego_x = stopped
    out = _run(stopped, True, 300)
    assert not out["hits"].any()
    stopped_behind = 0
    for st, tid in zip(out["states"], out["type_id"]):
        lane1 = (np.abs(st["y"][0] - RS.LANE_W) < 1.0) & (tid[0] < 255) & (st["x"][0] < ego_x)
        lane1[0] = False
        gap = ego_x - st["x"][0][lane1]
        slow = st["speed"][0][lane1] < 0.1
        stopped_behind += slow.sum()
        # the reference's IDM (s* falls when closing in) meets a stopped car inside min_spacing: 23 m of 30 here
        assert (gap[slow] >= 0.7 * RS.MIN_SPACING).all()
    assert stopped_behind > 0


def test_reactive_track_with_nothing_in_the_way_keeps_to_its_log():
    eps, k = RS.cruise(period_ms=100)
    out = _run((eps,), True, 150)
    rec = eps.log.records[eps.log.rec_off[k]:eps.log.rec_off[k] + eps.log.n_frames[k]].astype(np.float64)
    h = float(rec[0, 2])
    u = np.array([np.cos(h), np.sin(h)])
    m = 1
    checked = 0
    for i, (st, tid) in enumerate(zip(out["states"], out["type_id"])):
        t = (i + 1) * 100
        if tid[0, m] == 255:
            continue
        j = (t - int(eps.log.first_ms[k])) // 100
        d = np.array([st["x"][0, m], st["y"][0, m]], np.float64) - rec[0, :2]
        along_log = np.dot(rec[j, :2] - rec[0, :2], u)
        assert abs(d[0] * -u[1] + d[1] * u[0]) <= 0.1
        assert abs(np.dot(d, u) - along_log) <= 1.0
        checked += 1
    assert checked > 100
