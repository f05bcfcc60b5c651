"""The float64 MOBIL lane change (tests/lane_change_oracle.py) on known answers, and the closed-loop scenes the GPU tests
run (tests/lane_scenes.py) rolled out on the CPU: overtakes on the left, no collision, every change safe on the state it
was decided on, and a faster lane 0 than without lane changes."""

import math

import numpy as np
import pytest

from tests import lane_change_oracle as LC
from tests import lane_scenes as S

W = S.LANE_W
PATHS = [np.array([[-100.0, W * l], [400.0, W * l]], np.float32) for l in range(3)]
LEFT, RIGHT = [1, 2, -1], [-1, 0, 1]


def _rows(lateral=4):
    idm = dict(kind=1, desired_speed=16.0, time_headway=1.0, min_spacing=20.0, max_acceleration=2.0,
               comfortable_deceleration=6.0, delta=4.0, pid_lateral=lateral)
    slow = dict(idm, desired_speed=8.0, pid_lateral=0)
    return [idm, slow]


def _decide(cars, lanes=None, cool=None, left=LEFT, right=RIGHT, rows=None, **kw):
    """``cars``: (x, lane or y, speed, ctrl row or 255) per slot; an int lane puts the car on the lane's centre line."""
    m = len(cars)
    x = np.array([[c[0] for c in cars]])
    y = np.array([[W * c[1] if isinstance(c[1], int) else c[1] for c in cars]])
    v = np.array([[c[2] for c in cars]])
    cid = np.array([[c[3] for c in cars]], np.uint8)
    lp = np.array([lanes if lanes is not None else [c[1] if isinstance(c[1], int) else 0 for c in cars]], np.int16)
    cd = np.zeros((1, m), np.int16) if cool is None else np.array([cool], np.int16)
    args = dict(politeness=0.0, threshold=0.2, b_safe=4.0, min_gap=8.0, cool_ticks=10)
    args.update(kw)
    return LC.decide(x, y, v, np.zeros((1, m), np.uint8), [0], cid, rows or _rows(), lp, cd, left, right, PATHS, 1.8,
                     100.0, **args)


def test_slow_leader_with_a_free_left_lane_changes_left():
    r = _decide([(0, 0, 14.0, 0), (25, 0, 5.0, 255)])
    assert r["change"][0].tolist() == [1, 0]
    assert r["lane_path"][0].tolist() == [1, 0] and r["cooldown"][0, 0] == 10 and r["robust"].all()


def test_close_fast_new_follower_makes_it_unsafe():
    r = _decide([(0, 0, 14.0, 0), (25, 0, 5.0, 255), (-9, 1, 20.0, 255)])
    assert r["change"][0, 0] == 0
    r = _decide([(0, 0, 14.0, 0), (25, 0, 5.0, 255), (-9, 1, 20.0, 255)], b_safe=7.0)   # the IDM floor is -6
    assert r["change"][0, 0] == 1


def _marginal(politeness):
    # the changer gains a little; its new follower (slot 2, on row 0) loses more than that, weighted by politeness
    return _decide([(0, 0, 12.0, 0), (60, 0, 10.0, 255), (-30, 1, 14.0, 0)], lanes=[0, 0, 1], politeness=politeness,
                   threshold=0.05, b_safe=7.0)


def test_politeness_flips_a_marginal_case():
    assert _marginal(0.0)["change"][0, 0] == 1
    assert _marginal(1.0)["change"][0, 0] == 0


def test_car_alongside_blocks():
    r = _decide([(0, 0, 14.0, 0), (25, 0, 5.0, 255), (5, 1, 14.0, 255)])
    assert r["change"][0, 0] == 0
    r = _decide([(0, 0, 14.0, 0), (25, 0, 5.0, 255), (-9, 1, 14.0, 255)], min_gap=10.0)   # behind within min_gap
    assert r["change"][0, 0] == 0


def test_cooldown_waits_and_counts_down():
    r = _decide([(0, 0, 14.0, 0), (25, 0, 5.0, 255)], cool=[3, 5])
    assert r["change"][0, 0] == 0 and r["cooldown"][0].tolist() == [2, 4]


def test_changer_off_its_own_path_does_not_decide():
    r = _decide([(0, 1.9, 14.0, 0), (25, 0, 5.0, 255)], lanes=[0, 0])
    assert r["change"][0, 0] == 0 and not r["changer"][0, 0]
    r = _decide([(0, 1.7, 14.0, 0), (25, 0, 5.0, 255)], lanes=[0, 0])
    assert r["changer"][0, 0]


def test_missing_neighbour():
    r = _decide([(0, 0, 14.0, 0), (25, 0, 5.0, 255)], left=[-1, 2, -1])
    assert r["change"][0, 0] == 0 and not r["changer"][0, 0]


def test_left_right_tie_goes_left():
    r = _decide([(0, 1, 14.0, 0), (25, 1, 5.0, 255)])
    assert r["change"][0, 0] == 1 and r["lane_path"][0, 0] == 2
    assert not r["robust"][0, 0]                     # the two incentives are equal


def test_follower_without_an_idm_row_takes_the_changers_row():
    cars = [(0, 0, 12.0, 0), (60, 0, 10.0, 255), (-30, 1, 14.0, 255)]

    def incentive(follower_row):
        c = [c[:3] + (follower_row,) if i == 2 else c for i, c in enumerate(cars)]
        r = _decide(c, lanes=[0, 0, 1], politeness=1.0, threshold=-100.0, b_safe=7.0)
        return r["decisions"][0]["incentive"]

    assert incentive(255) == incentive(0)           # no IDM row: the changer's
    assert incentive(1) != incentive(0)             # its own row (desired 8 m/s)


@pytest.mark.parametrize("scene", ["highway", "rings"])
def test_closed_loop_overtakes_on_the_left(scene):
    sc = getattr(S, scene)()
    lane0 = sc[-1]
    with_lc, without = S.rollout(sc, True), S.rollout(sc, False)
    assert not with_lc["hits"].any()
    changes = [d for ds in with_lc["decisions"] for d in ds]
    assert any(d["side"] == 1 and d["slot"] in lane0 for d in changes)
    for d in changes:
        assert d["follower"] is None or d["a_follower"] >= -S.LANE["b_safe"]
    assert with_lc["speed"][:, lane0].mean() > without["speed"][:, lane0].mean() + 0.5
