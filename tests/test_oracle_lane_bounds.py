"""The float64 leader search (tests/leader_oracle.py) and MOBIL decision (tests/lane_change_oracle.py) on the exact scenes
of tests/exact_lane_scenes.py: every bound, tie and clamped projection gives the hand-derived answer, unmasked, and every
K18 case that is not decided by an exact acceleration keeps its incentive at least 0.5 m/s^2 from the threshold."""

import math

import numpy as np
import pytest

from oracle import controllers as OC
from tests import exact_lane_scenes as E
from tests import lane_change_oracle as LC
from tests import leader_oracle as L
from tests import route_oracle as R

LEADER_CASES = E.leader_cases()
LANE_CASES = E.lane_cases()


def _find(cases):
    x, y, h, tid, pid = E.leader_batch(cases)
    return L.find(x, y, h, tid, [E.OBB], E.HW, E.RNG, pid, E.paths())


@pytest.mark.parametrize("case", LEADER_CASES, ids=[c["name"] for c in LEADER_CASES])
def test_leader_case_gives_the_hand_answer(case):
    r = _find([case])
    for slot, (lead, gap) in case["want"].items():
        assert r["lead"][0, slot] == lead, (slot, r["lead"][0, slot])
        assert r["gap"][0, slot] == gap, (slot, r["gap"][0, slot])
        if lead >= 0:
            assert r["frame"][0, slot] == (L.HEADING if case["cars"][0][3] < 0 else L.PATH)


def test_leader_cases_sit_on_their_bounds():
    """The robust filter the random tests apply would hide these cases: the oracle marks them not robust."""
    r = _find(LEADER_CASES)
    names = [c["name"] for c in LEADER_CASES]
    for i, name in enumerate(names):
        if name.startswith("path_corridor") or name.endswith("_closed") or "_tie_" in name:
            followers = [s for s, (lead, _) in LEADER_CASES[i]["want"].items() if lead >= 0]
            assert not r["robust"][i, followers].all(), name


def test_exact_projections():
    """The arc lengths the hand answers rest on: clamped to the lane's ends, and the kinked path's first minimum."""
    lane, kink = (np.asarray(E.paths()[k], np.float64) for k in (0, E.KINK))
    assert R.closest(lane, 513.0, 1.0)[5] == E.L_LANE and R.closest(lane, 500.0, 0.0)[5] == 628.0
    assert R.closest(lane, -129.0, 0.5)[5] == 0.0 and R.closest(lane, 0.0, -1.5)[4] == 1.5
    assert R.closest(kink, 63.0, 101.0)[4:6] == (1.0, 63.0)          # 1 m from both segments: the first one's s
    assert R.closest(kink, 65.0, 99.0)[5] == 64.0                    # the outer wedge: the corner from both segments


def test_corridor_cases_defeat_the_prefilters_they_name():
    """Each corridor case's leader lies outside the Euclidean radius of every prefilter it names and inside the full
    radius d_i + max_range + half_width; together they defeat every prefilter that drops a term of that radius."""
    lane = np.asarray(E.paths()[0], np.float64)
    cases = [c for c in LEADER_CASES if "drops" in c]
    seen = set()
    for c in cases:
        (_, xi, yi, _), (_, xj, yj, _) = c["cars"]
        d_i = R.closest(lane, xi, yi)[4]
        dist = math.hypot(xj - xi, yj - yi)
        radius = dict(disc=E.RNG, no_half_width=d_i + E.RNG, no_d_i=E.RNG + E.HW)
        assert dist <= d_i + E.RNG + E.HW, c["name"]
        assert {k for k, r in radius.items() if dist > r} == set(c["drops"]), c["name"]
        seen |= set(c["drops"])
    assert seen == {"disc", "no_half_width", "no_d_i"}


def _decide(case, **over):
    x, y, v, tid, cid, lane, cool = E.lane_arrays(case)
    left, right = E.neighbours(case)
    kw = dict(case["kw"], **over)
    return LC.decide(x, y, v, tid, [E.OBB], cid, E.ctab(), lane, cool, left, right, E.paths(), E.HW, E.RNG,
                     politeness=kw["politeness"], threshold=kw["threshold"], b_safe=kw["b_safe"], min_gap=kw["min_gap"],
                     cool_ticks=kw["cooldown"])


@pytest.mark.parametrize("case", LANE_CASES, ids=[c["name"] for c in LANE_CASES])
def test_lane_case_gives_the_hand_answer(case):
    r = _decide(case)
    for slot, want in case["want"].items():
        got = (r["lane_path"][0, slot], r["cooldown"][0, slot], r["change"][0, slot])
        assert got == want, (slot, got)
    if "margin" in case:   # the incentive of the one side that decides, read with every side accepted
        slot, side = case["margin"]
        d = [d for d in _decide(case, threshold=-1.0e9)["decisions"] if d["slot"] == slot]
        assert len(d) == 1 and d[0]["side"] == (1 if side == 0 else -1)
        assert abs(d[0]["incentive"] - case["kw"]["threshold"]) >= 0.5, d[0]["incentive"]


def test_free_flow_incentive_is_exactly_zero():
    case = next(c for c in LANE_CASES if c["name"] == "free_tie_goes_left")
    d = _decide(case)["decisions"]
    assert [(x["side"], x["incentive"]) for x in d] == [(1, 0.0)]


def test_fast_follower_is_clipped_to_exactly_minus_b():
    row = E.ctab()[E.STD]
    y0, y1 = np.float32(E.W), np.float32(2 * E.W)
    assert float(OC.idm(40.0, -16.0, y1, True, 10.0, 0.0, y0, row)) == -E.B
    r = _decide(next(c for c in LANE_CASES if c["name"] == "safe_at_the_clip"))
    assert [(d["slot"], d["follower"], d["a_follower"]) for d in r["decisions"]] == [(0, 97, -E.B)]


def test_changer_off_its_path_is_not_a_changer():
    for name, changer in (("own_path_closed", True), ("own_path_past", False), ("free_no_neighbour", False)):
        assert _decide(next(c for c in LANE_CASES if c["name"] == name))["changer"][0, 0] == changer, name


def test_lane_bound_cases_are_not_robust():
    """Every case decided exactly on a bound or a tie is one the random tests' robust filter masks out (a dyadic step
    past a bound is not: it is more than 1e-9 away)."""
    on = {c["name"] for c in LANE_CASES if c["name"].endswith(("_closed", "_at_the_clip", "_at_range")) or "tie" in c["name"]}
    assert len(on) == 10 and "free_threshold_zero" not in on
    for c in LANE_CASES:
        assert _decide(c)["robust"][0, 0] == (c["name"] not in on | {"free_threshold_zero"}), c["name"]
