"""The float64 leader search (tests/leader_oracle.py) on known answers, and the closed-loop scene the GPU tests run
(tests/leader_scenes.py) rolled out on the CPU: no collision with every leader found, collisions without leaders."""

import math

import numpy as np
import pytest

from oracle import controllers as OC
from oracle import scenario as O
from tests import leader_oracle as L
from tests import leader_scenes as S

OBB, DISC, NONE = 0, 1, 2


def _find(pts, heading=None, types=None, shapes=(OBB,), hw=1.8, rng=100.0, path_id=None, paths=None):
    pts = np.asarray(pts, np.float64)
    m = len(pts)
    h = np.zeros((1, m)) if heading is None else np.asarray([heading], np.float64)
    tid = np.zeros((1, m), np.uint8) if types is None else np.asarray([types], np.uint8)
    pid = None if path_id is None else np.asarray([path_id], np.int16)
    return L.find(pts[None, :, 0], pts[None, :, 1], h, tid, list(shapes), hw, rng, pid, paths)


def test_same_lane_leader_and_gap():
    r = _find([[0, 0], [30, 0.5], [12, -0.3]])
    assert r["lead"][0].tolist() == [2, -1, 1]
    assert r["gap"][0, 0] == 12.0 and r["gap"][0, 2] == 18.0 and r["gap"][0, 1] == math.inf
    assert (r["frame"][0] == L.HEADING).all() and r["robust"].all()


def test_adjacent_lane_and_behind_are_excluded():
    r = _find([[0, 0], [10, 3.5], [-10, 0]])
    assert r["lead"][0, 0] == -1                 # 3.5 m to the side, and behind
    assert r["lead"][0, 2] == 0                  # the car behind follows slot 0


def test_closed_bounds():
    r = _find([[0, 0], [50, 1.5], [100, 0]], hw=1.5, rng=100.0)
    assert r["lead"][0, 0] == 1                  # |ey| == half_width qualifies
    assert not r["robust"][0, 0]
    r = _find([[0, 0], [100, 0]], rng=100.0)
    assert r["lead"][0, 0] == 1 and r["gap"][0, 0] == 100.0    # gap == max_range qualifies
    r = _find([[0, 0], [100.5, 0]], rng=100.0)
    assert r["lead"][0, 0] == -1


def test_tie_goes_to_the_lower_slot():
    r = _find([[0, 0], [20, 1], [20, -1]])
    assert r["lead"][0, 0] == 1 and not r["robust"][0, 0]


def test_disc_counts_shapeless_and_retired_do_not():
    r = _find([[0, 0], [5, 0], [8, 0], [12, 0]], types=[0, 2, 255, 1], shapes=(OBB, DISC, NONE))
    assert r["lead"][0, 0] == 3                  # slot 1 is shapeless, slot 2 retired
    assert r["lead"][0, 1] == 3                  # a shapeless slot still follows
    assert r["lead"][0, 2] == -1 and r["gap"][0, 2] == math.inf and r["frame"][0, 2] == 0


def test_nan_position_never_qualifies():
    r = _find([[0, 0], [math.nan, 0], [15, 0]])
    assert r["lead"][0, 0] == 2 and r["lead"][0, 1] == -1


def _quarter(radius=50.0, n=33):
    a = np.linspace(0.0, math.pi / 2, n)
    return np.stack([radius * np.sin(a), radius - radius * np.cos(a)], 1).astype(np.float32)


def test_curved_path_finds_the_leader_the_heading_frame_misses():
    arc = _quarter()
    p0, p1 = arc[4].astype(np.float64), arc[20].astype(np.float64)     # far round the bend: off the follower's heading
    pts = [p0, p1]
    r = _find(pts, heading=[math.pi / 16 * 0.5, 0.0], path_id=[-1, -1], paths=[arc])
    assert r["lead"][0, 0] == -1
    r = _find(pts, heading=[math.pi / 16 * 0.5, 0.0], path_id=[0, -1], paths=[arc])
    assert r["lead"][0, 0] == 1 and r["frame"][0, 0] == L.PATH
    assert r["gap"][0, 0] == pytest.approx(50.0 * math.pi / 2 * 16 / 32, rel=1e-3)


def test_follower_without_a_usable_path_takes_the_heading_frame():
    flat = np.array([[0, 0], [0, 0]], np.float32)                     # no segment of non-zero length
    r = _find([[0, 0], [10, 0]], path_id=[0, 0], paths=[flat])
    assert r["frame"][0, 0] == L.HEADING and r["lead"][0, 0] == 1
    r = _find([[0, 0], [10, 0]], path_id=[5, 5], paths=[flat])       # an id outside the table
    assert r["frame"][0, 0] == L.HEADING and r["lead"][0, 0] == 1


def rollout(search, ticks=100):
    """The closed-loop scene in float64: (dynamic-collision flags OR-ed over the rollout, leaders of every tick)."""
    st, tid, cid, pid, paths = S.scene()
    tab = S.table().as_oracle_table()
    rows = [c.params() for c in S.controllers()]
    ctab = [{k: getattr(r, k) for k, _ in r._fields_} for r in rows]
    m = tid.shape[1]
    la = np.zeros((1, m))
    hits = np.zeros((1, m), np.uint8)
    leads = []
    p64 = [p.astype(np.float64) for p in paths]
    for t in range(ticks):
        lead = (L.find(st["x"], st["y"], st["heading"], tid, [OBB], S.HALF_WIDTH, S.MAX_RANGE, pid, paths)["lead"]
                if search else np.full((1, m), -1, np.int16))
        leads.append(lead)
        act, la = OC.control_tick(st, tid, tab, S.script(t, m), cid, ctab, lead, pid, p64, la)
        st = O.physics_tick(st, tid, act, tab, 100, 5)
        st = {k: np.asarray(v, np.float32).astype(np.float64) for k, v in st.items()}
        hits |= O.events(st["x"], st["y"], st["heading"], tid, tab)[0] & O.F_DYNAMIC
    return hits, leads


def test_platoon_and_cut_in_closed_loop():
    hits, leads = rollout(True)
    assert not hits.any()
    assert any(l[0, 1] == S.CUT_IN for l in leads)                    # the lane-0 follower reacts to the cut-in
    hits, _ = rollout(False)
    assert hits[0, S.IDM_SLOTS].any()                                 # without leaders the followers crash
