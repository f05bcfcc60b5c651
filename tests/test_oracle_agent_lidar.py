"""The per-agent lidar statement (tests/agent_lidar_oracle.py) against the pinned ego scan (oracle/lidar.py) and against
the unmodified reference's ``SingleLineLidar`` bound to a body k != 0 (tests/golden/lidar_bound.npz, written by
tests/make_lidar_bound_golden.py), plus the rules of DESIGN.md section 1 "Per-agent lidar" that no reference scan exercises."""

import os

import numpy as np
import pytest

from oracle import lidar as OL
from oracle.scenario import CIRCLE, INACTIVE, OBB
from tests import agent_lidar_oracle as AL

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "lidar_bound.npz"))


def _ring_segments(walls):
    return np.concatenate([np.concatenate([w, np.roll(w, -1, 0)], 1) for w in walls], 0)


def _gold_world():
    """The golden scenes as a world: one type-table row per body (each has its own size)."""
    b = GOLD["bodies"]
    S, B = b.shape[:2]
    table = [dict(shape=np.zeros(B, np.int32), half_len=b[k, :, 3], half_wid=b[k, :, 4]) for k in range(S)]
    return b, table


@pytest.mark.parametrize("n_beams,max_range", [(360, 20.0), (500, 12.0), (37, 30.0), (1100, 9.0)])
def test_bound_sensor_equals_reference(n_beams, max_range):
    want = GOLD[f"scan_{n_beams}_{int(max_range)}"]
    b, tables = _gold_world()
    segs = _ring_segments(GOLD["walls"])
    hits = 0
    for k in range(b.shape[0]):
        tid = np.arange(b.shape[1], dtype=np.uint8)[None]
        got = AL.scan_agents(b[k, :, 0][None], b[k, :, 1][None], b[k, :, 2][None], tid, tables[k], n_beams, max_range,
                             observers=[[int(GOLD["bound"][k])]], segments=segs)[0, 0]
        assert np.array_equal(np.isinf(got), np.isinf(want[k]))
        ok = np.isfinite(want[k])
        np.testing.assert_allclose(got[ok], want[k][ok], rtol=1e-12, atol=1e-12)
        hits += int(ok.sum())
    assert hits > 0.2 * want.size


def test_golden_sees_body_zero():
    """The fixture pins the rule: without body 0's ring the bound sensor's scan differs."""
    b, tables = _gold_world()
    segs = _ring_segments(GOLD["walls"])
    want = GOLD["scan_360_20"]
    differs = 0
    for k in range(b.shape[0]):
        tid = np.arange(b.shape[1], dtype=np.uint8)[None]
        tid[0, 0] = INACTIVE
        got = AL.scan_agents(b[k, :, 0][None], b[k, :, 1][None], b[k, :, 2][None], tid, tables[k], 360, 20.0,
                             observers=[[int(GOLD["bound"][k])]], segments=segs)[0, 0]
        differs += int(not np.array_equal(got, want[k]))
    assert differs == b.shape[0]


def _scene(n=6, m=9, seed=0, disc_types=False):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0, 30, (n, m)).astype(np.float32).astype(np.float64)
    y = rng.uniform(0, 30, (n, m)).astype(np.float32).astype(np.float64)
    h = rng.uniform(0, 2 * np.pi, (n, m)).astype(np.float32).astype(np.float64)
    table = dict(shape=np.asarray([OBB, OBB, CIRCLE], np.int32), half_len=np.asarray([2.4, 1.0, 0.3]),
                 half_wid=np.asarray([1.0, 0.4, 0.3]))
    tid = rng.integers(0, 3 if disc_types else 2, (n, m)).astype(np.uint8)
    segs = np.asarray([[0, 0, 30, 0], [30, 0, 30, 30], [0, 15, 12, 15]], np.float64)
    return x, y, h, tid, table, segs


def test_slot_zero_rows_equal_scan_world_bit_for_bit():
    x, y, h, tid, table, segs = _scene(8, 12, seed=1)
    tid[2, 0] = INACTIVE   # a scenario without an ego
    for n_beams, max_range in ((360, 20.0), (1100, 9.0), (37, 30.0)):
        want = OL.scan_world(x, y, h, tid, table, segs, n_beams, max_range)
        got = AL.scan_agents(x, y, h, tid, table, n_beams, max_range, observers=np.zeros((8, 1)), segments=segs)
        assert np.array_equal(got[:, 0], want)
        assert np.isinf(got[2]).all()


def test_absent_rows_and_duplicates():
    x, y, h, tid, table, segs = _scene(4, 9, seed=2)
    tid[:, 3] = INACTIVE   # an empty (or retired) slot
    tid[:, 4] = 7          # a type beyond the table
    obs = np.tile(np.asarray([-1, 9, 3, 4, 5, 5, 2, 300, 5]), (4, 1))
    got = AL.scan_agents(x, y, h, tid, table, 360, 20.0, observers=obs, segments=segs)
    assert np.isinf(got[:, [0, 1, 2, 3, 7]]).all()
    assert np.array_equal(got[:, 4], got[:, 5]) and np.array_equal(got[:, 4], got[:, 8])
    every = AL.scan_agents(x, y, h, tid, table, 360, 20.0, segments=segs)
    assert np.array_equal(every[:, 5], got[:, 4]) and np.array_equal(every[:, 2], got[:, 6])


def test_own_box_unseen_and_slot_zero_seen():
    # two boxes 5 m apart on a line and nothing else: each sees exactly the other one
    x = np.asarray([[0.0, 5.0]]); y = np.zeros((1, 2)); h = np.zeros((1, 2))
    table = dict(shape=np.asarray([OBB], np.int32), half_len=np.asarray([2.0]), half_wid=np.asarray([1.0]))
    tid = np.zeros((1, 2), np.uint8)
    got = AL.scan_agents(x, y, h, tid, table, 360, 20.0)
    # slot 1 looks back along -x (beam 180) at slot 0's front face at x = 2: 3 m; slot 0 sees slot 1's rear face at 3 m
    assert got[0, 1, 180] == pytest.approx(3.0, abs=1e-12) and got[0, 0, 0] == pytest.approx(3.0, abs=1e-12)
    # and only that box: every beam away from it is empty (its own ring around the sensor is never an obstacle)
    assert np.isinf(got[0, 0, 90]) and np.isinf(got[0, 1, 0]) and np.isfinite(got[0]).sum() < 0.2 * got[0].size
    alone = AL.scan_agents(x, y, h, np.asarray([[0, INACTIVE]], np.uint8), table, 360, 20.0)
    assert np.isinf(alone).all()


def test_disc_observer_scans_and_discs_are_not_obstacles():
    x, y, h, tid, table, segs = _scene(5, 10, seed=3, disc_types=True)
    tid[:, 1] = 2   # slot 1 is a disc in every scenario
    got = AL.scan_agents(x, y, h, tid, table, 360, 20.0, observers=np.ones((5, 1)), segments=segs)
    assert np.isfinite(got).any()
    # moving or removing the disc slots changes nothing any row sees
    disc = tid == 2
    x2 = np.where(disc, x + 3.0, x)
    x2[:, 1] = x[:, 1]   # ... except the observer itself, which carries the sensor
    got2 = AL.scan_agents(x2, y, h, tid, table, 360, 20.0, observers=np.ones((5, 1)), segments=segs)
    assert np.array_equal(got, got2)
    every = AL.scan_agents(x, y, h, tid, table, 360, 20.0, segments=segs)
    tid3 = np.where(disc, INACTIVE, tid)
    every3 = AL.scan_agents(x, y, h, tid3, table, 360, 20.0, segments=segs)
    keep = ~disc
    assert np.array_equal(every[keep], every3[keep])


def test_each_scenario_sees_its_own_tile():
    x, y, h, tid, table, segs = _scene(4, 6, seed=4)
    tiles = [segs, np.asarray([[0, 5, 30, 5], [5, 0, 5, 30]], np.float64), None]
    tile_id = np.asarray([0, 1, 2, 1])
    got = AL.scan_agents(x, y, h, tid, table, 360, 20.0, tiles=tiles, tile_id=tile_id)
    for n in range(4):
        one = AL.scan_agents(x[n:n + 1], y[n:n + 1], h[n:n + 1], tid[n:n + 1], table, 360, 20.0,
                             segments=tiles[tile_id[n]])
        assert np.array_equal(got[n], one[0])
    assert not np.array_equal(AL.scan_agents(x, y, h, tid, table, 360, 20.0, tiles=tiles, tile_id=[0, 0, 0, 0])[1],
                              got[1])
