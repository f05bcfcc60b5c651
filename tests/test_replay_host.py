"""Log replay on the host: ReplayLog against the parser's trajectories, the float64 oracle's known answers (oracle/replay.py)
and the episode builder, on synthetic CSVs in the LevelX schemas (no LevelX data ships with the reference or this repository)."""

from types import SimpleNamespace

import numpy as np
import pandas as pd
import pytest

from oracle import replay as R
from tactics2d_b200.dataset_parser import LevelXParser, ReplayLog, build_replay_episodes
from tactics2d_b200.types import MAX_TYPES, MODEL_KINEMATICS, MODEL_STATIC, TYPE_INACTIVE, TypeParams, TypeTable
from tests.test_levelx_parser import _write_ind


def _write_highd(folder, fid=7):
    rows = []
    for f in range(1, 6):
        rows.append(dict(frame=f, id=5, x=100.0 + f, y=20.0, width=4.5, height=1.8, xVelocity=30.0, yVelocity=0.6 - 0.3 * f,
                         xAcceleration=0.0, yAcceleration=0.0))
        rows.append(dict(frame=f + 1, id=6, x=300.0 - f, y=9.0, width=12.0, height=2.5, xVelocity=-25.0, yVelocity=-0.2 + 0.1 * f,
                         xAcceleration=0.1, yAcceleration=0.0))
    pd.DataFrame(rows).to_csv(folder / f"{fid:02d}_tracks.csv", index=False)
    pd.DataFrame([dict(id=5, width=4.5, height=1.8, initialFrame=1, finalFrame=5, **{"class": "Car"}),
                  dict(id=6, width=12.0, height=2.5, initialFrame=2, finalFrame=6, **{"class": "Truck"})]).to_csv(
        folder / f"{fid:02d}_tracksMeta.csv", index=False)
    pd.DataFrame([dict(id=fid, locationId=1, lowerLaneMarkings="21.0;24.9;28.8", upperLaneMarkings="8.5;12.6;16.4")]).to_csv(
        folder / f"{fid:02d}_recordingMeta.csv", index=False)


@pytest.mark.parametrize("dataset", ["inD", "highD"])
def test_records_equal_parsed_trajectory_states(tmp_path, dataset):
    if dataset == "inD":
        _write_ind(tmp_path)
        fid = 3
    else:
        _write_highd(tmp_path)
        fid = 7
    p = LevelXParser(dataset)
    log = ReplayLog.from_levelx(p, fid, str(tmp_path))
    parts, _ = p.parse_trajectory(fid, str(tmp_path))
    assert sorted(log.ids.tolist()) == sorted(parts) and (log.period_ms == 40).all()
    n = 0
    for k, id_ in enumerate(log.ids):
        traj = parts[int(id_)].trajectory
        assert log.first_ms[k] == traj.first_frame and log.last_ms[k] == traj.last_frame
        for t in range(traj.first_frame, traj.last_frame + 1, 40):
            s = traj.get_state(t)
            want = np.asarray([s.x, s.y, np.mod(s.heading, 2 * np.pi), s.vx, s.vy], np.float64).astype(np.float32)
            assert np.array_equal(log.record(k, t), want), (id_, t)
            n += 1
    assert n == len(log.records)
    assert (log.records[:, 2] >= 0).all() and (log.records[:, 2] <= np.float32(2 * np.pi)).all()
    if dataset == "highD":   # (-pi, pi] headings: the negative ones wrapped
        assert (log.records[:, 2] > np.pi).any()


def _log(first, period, recs, type_row=None):
    recs = [np.asarray(r, np.float32).reshape(-1, 5) for r in recs]
    return SimpleNamespace(first_ms=np.asarray(first, np.int32), period_ms=np.asarray(period, np.int32),
                           n_frames=np.asarray([len(r) for r in recs], np.int32), records=np.concatenate(recs),
                           type_row=np.asarray(type_row if type_row is not None else [7] * len(recs), np.uint8))


def test_oracle_half_way_between_80_and_120_ms():
    rec = [[10.0 * j, -2.0 * j, 0.1 * j, 3.0 + j, -1.0 + 0.5 * j] for j in range(6)]
    log = _log([0], [40], [rec])
    rep, pres, s, tid = R.sample(log, [0], [[0, -1]], [0], [0], 100, 1)         # t = 100 ms: frames 2 (80) and 3 (120), w = 0.5
    assert rep.tolist() == [[True, False]] and pres.tolist() == [[True, False]] and tid[0, 0] == 7
    a, b = np.asarray(rec[2], np.float32).astype(np.float64), np.asarray(rec[3], np.float32).astype(np.float64)
    for c, key in enumerate(("x", "y", "heading", "vx", "vy")):
        assert s[key][0, 0] == np.float32(a[c] + 0.5 * (b[c] - a[c])), key
    vx, vy = np.float64(s["vx"][0, 0]), np.float64(s["vy"][0, 0])
    assert s["speed"][0, 0] == np.float32(np.sqrt(vx * vx + vy * vy))
    # on a frame the record's bits; at reset (offset 0) t = t0
    _, _, s0, _ = R.sample(log, [120], [[0, -1]], [0], [0], 100, 0)
    assert np.array_equal([s0[k][0, 0] for k in ("x", "y", "heading", "vx", "vy")], np.asarray(rec[3], np.float32))


def test_oracle_heading_takes_the_shorter_arc_across_zero():
    rec = [[0, 0, 6.2, 0, 0], [0, 0, 0.1, 0, 0]]
    log = _log([0], [40], [rec])
    _, _, s, _ = R.sample(log, [0], [[0]], [0], [0], 20, 1)                       # w = 0.5
    ha, hb = np.float64(np.float32(6.2)), np.float64(np.float32(0.1))
    h = ha + 0.5 * (hb - ha + 2 * np.pi) - 2 * np.pi
    assert s["heading"][0, 0] == np.float32(h) and 0 < s["heading"][0, 0] < 0.1
    # the other way round, and a result just below 2 pi that rounds to fp32(2 pi) is stored as 0
    log2 = _log([0], [40], [[[0, 0, 0.1, 0, 0], [0, 0, 6.2, 0, 0]]])
    _, _, s2, _ = R.sample(log2, [0], [[0]], [0], [0], 20, 1)
    assert s2["heading"][0, 0] == np.float32(hb + 0.5 * (ha - hb - 2 * np.pi)) and 0 < s2["heading"][0, 0] < 0.1
    log4 = _log([0], [40], [[[0, 0, 0.1, 0, 0], [0, 0, 6.2, 0, 0]]])             # w = 0.75: across 0 to the far side
    _, _, s4, _ = R.sample(log4, [0], [[0]], [0], [0], 30, 1)
    assert s4["heading"][0, 0] == np.float32(hb + 0.75 * (ha - hb - 2 * np.pi) + 2 * np.pi) and s4["heading"][0, 0] > 6.2
    below, top = np.nextafter(np.float32(2 * np.pi), np.float32(0)), np.float32(2 * np.pi)
    log3 = _log([0], [40], [[[0, 0, below, 0, 0], [0, 0, top, 0, 0]]])
    _, _, s3, _ = R.sample(log3, [0], [[0]], [0], [0], 24, 1)                     # w = 0.6: 6.28318529 in float64
    h = np.float64(below) + 0.6 * (np.float64(top) - np.float64(below))
    assert h < 2 * np.pi and np.float32(h) == top and s3["heading"][0, 0] == 0.0


def test_oracle_track_absent_before_first_and_after_last_frame():
    log = _log([200], [40], [[[1, 2, 3, 4, 5], [2, 3, 4, 5, 6]]])                  # present on [200, 240]
    state = {k: np.full((1, 1), -7.0, np.float32) for k in ("x", "y", "heading", "speed", "vx", "vy")}
    for t0, present in ((60, False), (100, True), (120, True), (150, False)):     # t = t0 + 100
        out, tid = R.apply(state, np.zeros((1, 1), np.uint8), log, [t0], [[0]], [0], [0], 100, 1)
        assert (tid[0, 0] != TYPE_INACTIVE) == present, t0
        assert (out["x"][0, 0] == -7.0) == (not present)
    # a slot that replays nothing and a masked-out scenario keep everything
    out, tid = R.apply(state, np.full((1, 1), 3, np.uint8), log, [100], [[-1]], [0], [0], 100, 1)
    assert tid[0, 0] == 3 and out["x"][0, 0] == -7.0
    out, tid = R.apply(state, np.full((1, 1), 3, np.uint8), log, [100], [[0]], [0], [0], 100, 1, mask=[False])
    assert tid[0, 0] == 3 and out["x"][0, 0] == -7.0


def test_episode_builder_order_ego_and_dropped(tmp_path):
    _write_ind(tmp_path)   # tracks: 0 car 0..360 ms, 1 bus 80..360, 2 bicycle 0..200, 3 pedestrian 160..360
    log = ReplayLog.from_levelx(LevelXParser("inD"), 3, str(tmp_path))
    ep = build_replay_episodes(log, 3, [0, 200, 240], [0, 1, 0])
    ids = lambda p: [int(log.ids[k]) if k >= 0 else None for k in ep.row_track[p]]
    assert ids(0) == [None, 2, 1] and ep.dropped[0] == 1                           # (first stamp, id): 2 (0), 1 (80), 3 (160)
    assert ids(1) == [None, 0, 2] and ep.dropped[1] == 1                           # the ego's track 1 is never replayed
    assert ids(2) == [None, 1, 3] and ep.dropped[2] == 0                           # track 2 ended before 240
    assert np.array_equal([ep.pool[k][1, 0] for k in ("x", "y", "heading", "vx", "vy")], log.record(log.index(1), 200))
    vx, vy = np.float64(ep.pool["vx"][1, 0]), np.float64(ep.pool["vy"][1, 0])
    assert ep.pool["speed"][1, 0] == np.float32(np.sqrt(vx * vx + vy * vy))
    rows = ep.table.rows
    assert rows[ep.type_id[0, 0]].model == MODEL_KINEMATICS                        # the ego: its class's kinematic row
    assert ep.type_id[0, 2] == TYPE_INACTIVE and ep.type_id[0, 1] == ep.log.type_row[log.index(2)]   # track 1 appears at 80 ms
    for k in range(len(log)):
        r = rows[ep.log.type_row[k]]
        assert r.model == MODEL_STATIC
    ped = rows[ep.log.type_row[log.index(3)]]
    from tactics2d_b200.participant.element.participant_template import PEDESTRIAN_TEMPLATE
    assert ped.shape == 1 and ped.name in PEDESTRIAN_TEMPLATE                     # a disc, named like its class row
    # a horizon keeps later tracks out of the window
    ep2 = build_replay_episodes(log, 8, [0], [0], horizon_ms=100)
    assert [int(log.ids[k]) for k in ep2.row_track[0] if k >= 0] == [2, 1] and ep2.dropped[0] == 0
    sc = ep.scene()
    assert sc.shape == (3, 3) and sc.table is ep.table


def test_episode_builder_rejects_malformed_input(tmp_path):
    _write_ind(tmp_path)
    log = ReplayLog.from_levelx(LevelXParser("inD"), 3, str(tmp_path))
    with pytest.raises(ValueError, match="absent"):
        build_replay_episodes(log, 4, [40], [3])                                   # pedestrian 3 starts at 160 ms
    with pytest.raises(ValueError, match="outside the log"):
        build_replay_episodes(log, 4, [400], [0])
    with pytest.raises(ValueError, match="outside the log"):
        build_replay_episodes(log, 4, [-40], [0])
    with pytest.raises(KeyError):
        build_replay_episodes(log, 4, [20], [0])                                   # between two frames of the ego
    with pytest.raises(KeyError):
        build_replay_episodes(log, 4, [0], [99])                                   # no such track
    with pytest.raises(ValueError, match="one ego track per start time"):
        build_replay_episodes(log, 4, [0, 40], [0])


def test_static_twins_keep_shape_and_name_within_max_types():
    t = TypeTable.from_templates()
    t2, twin = t.with_static_twins([0, 0, 3, 12])
    assert len(t2) == len(t) + 3 and set(twin) == {0, 3, 12}
    for r, k in twin.items():
        a, b = t.rows[r], t2.rows[k]
        assert b.model == MODEL_STATIC and (a.half_len, a.half_wid, a.radius, a.shape, a.name) == (b.half_len, b.half_wid, b.radius, b.shape, b.name)
    t3, tw3 = t2.with_static_twins([twin[0]])                                     # a static row is its own twin
    assert tw3 == {twin[0]: twin[0]} and len(t3) == len(t2)
    big = TypeTable([TypeParams.vehicle() for _ in range(MAX_TYPES - 1)])
    with pytest.raises(ValueError, match="do not fit"):
        big.with_static_twins([0, 1])


def test_set_log_is_part_of_the_abi():
    from tactics2d_b200 import _lib

    assert "t2d_set_log" in _lib.SYMBOLS
    import ctypes
    assert ctypes.sizeof(_lib.LogC) == 4 + 4 + 8 * 5 + 4 + 4 + 8 * 4   # int32 + pad, 5 pointers, int32 + pad, 4 pointers
