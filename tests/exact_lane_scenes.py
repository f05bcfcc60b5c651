"""Scenes in which every quantity K17 (the leader search) and K18 (MOBIL lane changes) compare is exact in fp64, with the
answer each must give derived by hand (TEST INFRASTRUCTURE ONLY).

Why they are exact:

* Lanes run parallel to x at y = 0, 3.5 and 7 with vertices at x = -128, 0, 256, 512: every segment length is a power of
  two, so the projection ``t = (x - ax) / len``, the arc length ``s = acc + t len`` and the distance ``|y - y_lane|`` are
  exact for the short dyadic fp32 positions used here.  The kinked path has two 64 m segments.
* Every heading is 0: ``sincos_angle(0)`` is exactly (0, 1), so the heading frame's ``ex = dx`` and ``ey = dy``.
* A bound is crossed by a dyadic step: 2^-7 m past ``max_range``, 2^-20 m past ``half_width``, 2^-10 m inside
  ``min_gap``.
* The accelerations K18 compares on a bound are exact too: free flow on every side makes the incentive
  ``(a_free - a_free) + politeness 0 = 0``, and a fast new follower close behind is clipped to exactly ``-b``.  Every
  other K18 case keeps its incentive at least 0.5 m/s^2 from ``threshold``, so only the intended bound or tie decides.

A leader case is ``dict(name, cars=[(slot, x, y, path)], want={slot: (lead, gap)})`` (path -1: the heading frame); a lane
case is ``dict(name, cars=[(slot, x, y, speed, ctrl row or 255, lane, cooldown)], kw=lane-change parameters,
want={slot: (lane_path, cooldown, change)})``, optionally with its own ``left`` / ``right``.  Slots not listed are empty."""

from __future__ import annotations

import math

import numpy as np

HW, RNG = 1.75, 64.0            # the leader search's half_width and max_range (fp32-exact)
W = 3.5                         # lane spacing
M = 128                         # every slot a warp lane owns: l, l + 32, l + 64, l + 96
OBB = 0
STEP_RANGE, STEP_HW, STEP_GAP = 2.0 ** -7, 2.0 ** -20, 2.0 ** -10
INF = math.inf
KINK = 3                        # (0, 100) -> (64, 100) -> (64, 164): a convex corner at (64, 100)
L_LANE = 640.0                  # the arc length of a lane (128 + 256 + 256)


def paths():
    """Lanes 0..2 (lane l at y = 3.5 l), then the kinked path."""
    lanes = [np.array([[-128.0, W * l], [0.0, W * l], [256.0, W * l], [512.0, W * l]], np.float32) for l in range(3)]
    return lanes + [np.array([[0.0, 100.0], [64.0, 100.0], [64.0, 164.0]], np.float32)]


LEFT, RIGHT = [1, 2, -1, -1], [-1, 0, 1, -1]   # lane 1 has both neighbours, lane 0 only a left one, lane 2 only a right one


# ---------------------------------------------------------------------------------------------------------------- K17
def _lc(name, cars, want, **extra):
    return dict(name=name, cars=cars, want=want, **extra)


def leader_cases():
    cases = []
    for frame, p in (("path", 0), ("heading", -1)):
        # gap == max_range qualifies, 2^-7 m beyond it does not
        cases.append(_lc(f"{frame}_range_closed", [(0, 0.0, 0.0, p), (1, RNG, 0.5, p)], {0: (1, RNG), 1: (-1, INF)}))
        cases.append(_lc(f"{frame}_range_past", [(0, 0.0, 0.0, p), (1, RNG + STEP_RANGE, 0.5, p)], {0: (-1, INF)}))
        # gap == 0 (path: same arc length; heading: ex == 0) does not qualify; the farther candidate does
        cases.append(_lc(f"{frame}_zero_gap", [(0, 0.0, 0.0, p), (1, 0.0, 1.0, p), (2, 8.0, 0.0, p)],
                         {0: (2, 8.0), 1: (2, 8.0), 2: (-1, INF)}))
        # d == half_width (|ey| == half_width) qualifies on either side; 2^-20 m beyond does not
        for sign in (1.0, -1.0):
            tag = "plus" if sign > 0 else "minus"
            cases.append(_lc(f"{frame}_half_width_{tag}",
                             [(0, 0.0, 0.0, p), (1, 16.0, sign * (HW + STEP_HW), p), (2, 24.0, -sign * HW, p)],
                             {0: (2, 24.0)}))
            cases.append(_lc(f"{frame}_half_width_{tag}_closed", [(0, 0.0, 0.0, p), (1, 16.0, sign * HW, p)],
                             {0: (1, 16.0)}))
        # exact ties go to the lower slot, wherever the warp keeps the tied slots
        cases.append(_lc(f"{frame}_tie_2_97", [(40, 0.0, 0.0, p), (97, 20.0, -1.0, p), (2, 20.0, 1.0, p)],
                         {40: (2, 20.0)}))
        cases.append(_lc(f"{frame}_tie_33_64", [(0, 0.0, 0.0, p), (64, 12.0, 0.5, p), (33, 12.0, -0.5, p)],
                         {0: (33, 12.0)}))
        cases.append(_lc(f"{frame}_tie_31_64_127", [(1, 0.0, 0.0, p), (127, 30.0, 0.0, p), (64, 30.0, 1.5, p),
                                                    (31, 30.0, -1.5, p)], {1: (31, 30.0)}))
    # clamped projections: past the end every candidate within half_width of (512, 0) sits at s = L and the lowest slot
    # wins (slot 1, itself past the end, where it has nothing ahead)
    cases.append(_lc("path_end_clamp", [(5, 500.0, 0.0, 0), (70, 513.0, 1.0, 0), (9, 513.0, 0.5, 0), (3, 512.5, -1.0, 0),
                                        (1, 513.5, 0.0, 0)],
                     {5: (1, L_LANE - 128.0 - 500.0), 1: (-1, INF), 3: (-1, INF), 9: (-1, INF), 70: (-1, INF)}))
    # ... and before the start every one sits at s = 0: each sees the same leader, 8 m on
    cases.append(_lc("path_start_clamp", [(66, -129.0, 0.5, 0), (4, -128.5, -1.0, 0), (35, -130.0, 0.0, 0),
                                          (100, -120.0, 0.0, 0)],
                     {66: (100, 8.0), 4: (100, 8.0), 35: (100, 8.0), 100: (-1, INF)}))
    # the kinked path: (63, 101) is 1 m from both segments, and the first strict minimum (the first segment) gives
    # s = 63, not 65; (65, 99) in the corner's outer wedge projects onto the corner from both segments, s = 64
    cases.append(_lc("kink_first_minimum", [(0, 32.0, 100.0, KINK), (1, 63.0, 101.0, KINK), (2, 65.0, 99.0, KINK),
                                            (3, 64.5, 108.0, KINK)],
                     {0: (1, 31.0), 1: (2, 1.0), 2: (3, 8.0), 3: (-1, INF)}))
    cases.append(_lc("kink_outer_wedge", [(0, 63.5, 99.5, KINK), (1, 63.0, 101.0, KINK), (2, 65.0, 99.0, KINK)],
                     {0: (2, 0.5), 1: (0, 0.5)}))
    # the corridor is not a disc: in each case the candidate exactly half_width off the lane and exactly max_range ahead
    # is the leader, and a path-frame prefilter on the Euclidean distance |p_j - p_i| drops it unless its radius is the
    # full d_i + max_range + half_width (d_i the follower's distance to the path).  ``drops`` names the prefilters that
    # get it wrong: "disc" (radius max_range), "no_half_width" (d_i + max_range), "no_d_i" (max_range + half_width).
    cases.append(_lc("path_corridor_disc", [(0, 0.0, -1.5, 0), (1, RNG, HW, 0)], {0: (1, RNG)},
                     drops=("disc",)))                                   # 64.08 m apart
    cases.append(_lc("path_corridor_half_width", [(0, 0.0, 0.0, 0), (1, RNG, HW, 0)], {0: (1, RNG)},
                     drops=("disc", "no_half_width")))                   # 64.02 m apart, d_i = 0
    # 14 m off the lane on either side: 65.91 m apart, more than max_range + half_width = 65.75 m, less than 79.75 m
    cases.append(_lc("path_corridor_d_i_below", [(0, 0.0, -14.0, 0), (1, RNG, HW, 0)], {0: (1, RNG)},
                     drops=("disc", "no_d_i")))
    cases.append(_lc("path_corridor_d_i_above", [(0, 0.0, 14.0, 0), (1, RNG, -HW, 0)], {0: (1, RNG)},
                     drops=("disc", "no_d_i")))
    # a follower 16 m before the lane's start is clamped to s = 0 with d_i = 16: 80.02 m apart, more than
    # d_i + max_range = 80 m and max_range + half_width, less than 81.75 m
    cases.append(_lc("path_corridor_clamped", [(0, -144.0, 0.0, 0), (1, RNG - 128.0, HW, 0)], {0: (1, RNG)},
                     drops=("disc", "no_half_width", "no_d_i")))
    return cases


def leader_batch(cases):
    """``(x, y, heading, type_id, path_id)`` [len(cases), M]: one scenario per case, the other slots empty."""
    n = len(cases)
    x, y = np.zeros((n, M), np.float32), np.zeros((n, M), np.float32)
    tid = np.full((n, M), 255, np.uint8)
    pid = np.full((n, M), -1, np.int16)
    for i, c in enumerate(cases):
        for slot, cx, cy, p in c["cars"]:
            x[i, slot], y[i, slot], tid[i, slot], pid[i, slot] = cx, cy, 0, p
            assert float(np.float32(cx)) == cx and float(np.float32(cy)) == cy, (c["name"], slot)
    return x, y, np.zeros((n, M), np.float32), tid, pid


# ---------------------------------------------------------------------------------------------------------------- K18
B = 6.0                                   # every row's comfortable_deceleration: the IDM clip
BASE_KW = dict(politeness=0.0, threshold=-100.0, b_safe=B, min_gap=8.0, cooldown=5)
STD, FAR = 0, 1                           # the changers' rows


def controllers():
    """Row STD: a lane-keeping IDM; row FAR: the same with a 48 m min_spacing and 4 m/s^2, so a leader 56 - 64 m ahead
    moves the incentive by more than a metre per second squared."""
    from tactics2d_b200.controller import IDMController, PIDController

    keep = PIDController(dt=0.1, kp_lat=0.03, ki_lat=0.0, kd_lat=0.08, max_steering=0.2, derivative_filter_alpha=1.0,
                         lateral_error="path_cross_track")
    return [IDMController(desired_speed=16.0, time_headway=1.0, min_spacing=2.0, max_acceleration=2.0,
                          comfortable_deceleration=B, lateral=keep),
            IDMController(desired_speed=16.0, time_headway=1.0, min_spacing=48.0, max_acceleration=4.0,
                          comfortable_deceleration=B, lateral=keep)]


def ctab():
    return [{k: getattr(r, k) for k, _ in r._fields_} for r in (c.params() for c in controllers())]


def _car(slot, x, lane, v=10.0, row=255, dy=0.0, cool=0):
    return (slot, x, W * lane + dy, v, row, lane, cool)


def _case(name, cars, want, margin=None, **kw):
    c = dict(name=name, cars=cars, want=want, kw=dict(BASE_KW))
    for k in ("left", "right"):
        if k in kw:
            c[k] = kw.pop(k)
    c["kw"].update(kw)
    if margin is not None:
        c["margin"] = margin   # (slot, side): the one incentive that must lie >= 0.5 from threshold
    return c


def lane_cases():
    tiny = -(2.0 ** -10)
    cool = _car(90, 300.0, 0, row=STD, cool=3)   # a lane keeper in its cooldown: counts down, never decides
    cases = [
        # free flow: both incentives are exactly 0
        _case("free_threshold_zero", [_car(0, 0.0, 1, row=STD), cool], {0: (1, 0, 0), 90: (0, 2, 0)}, threshold=0.0),
        _case("free_tie_goes_left", [_car(0, 0.0, 1, row=STD)], {0: (2, 5, 1)}, threshold=tiny),
        _case("free_right_only", [_car(0, 0.0, 2, row=STD)], {0: (1, 5, -1)}, threshold=tiny),
        _case("free_no_neighbour", [_car(0, 0.0, 1, row=STD)], {0: (1, 0, 0)}, threshold=tiny, left=[-1] * 4,
              right=[-1] * 4),
        # blocking: |g| == min_gap does not block, 2^-10 m inside it does (ahead and behind)
        _case("block_ahead_closed", [_car(0, 0.0, 0, row=STD), _car(64, 8.0, 1)], {0: (1, 5, 1)}),
        _case("block_ahead_inside", [_car(0, 0.0, 0, row=STD), _car(64, 8.0 - STEP_GAP, 1)], {0: (0, 0, 0)}),
        _case("block_behind_closed", [_car(0, 0.0, 0, row=STD), _car(33, -8.0, 1)], {0: (1, 5, 1)}),
        _case("block_behind_inside", [_car(0, 0.0, 0, row=STD), _car(33, -8.0 + STEP_GAP, 1)], {0: (0, 0, 0)}),
        # safety: the fast new follower on the left is clipped to exactly -b; b_safe = b is safe (the left wins the tie
        # of two zero incentives), b_safe 2^-20 less is not and the changer goes right
        _case("safe_at_the_clip", [_car(0, 0.0, 1, row=STD), _car(97, -16.0, 2, v=40.0)], {0: (2, 5, 1)}),
        _case("unsafe_past_the_clip", [_car(0, 0.0, 1, row=STD), _car(97, -16.0, 2, v=40.0)], {0: (0, 5, -1)},
              b_safe=B - STEP_HW),
        # the changer's own path: exactly half_width off decides, 2^-20 m further out does not
        _case("own_path_closed", [_car(0, 0.0, 1, row=STD, dy=-HW), cool], {0: (2, 5, 1), 90: (0, 2, 0)}),
        _case("own_path_past", [_car(0, 0.0, 1, row=STD, dy=-HW - STEP_HW), cool], {0: (1, 0, 0), 90: (0, 2, 0)}),
        # the new leader's range: a stopped car exactly max_range ahead on the target costs more than threshold
        _case("new_leader_at_range", [_car(0, 0.0, 0, v=8.0, row=FAR), _car(31, RNG, 1, v=0.0)], {0: (0, 0, 0)},
              margin=(0, 0), threshold=-1.25),
        _case("new_leader_past_range", [_car(0, 0.0, 0, v=8.0, row=FAR), _car(31, RNG + STEP_RANGE, 1, v=0.0)],
              {0: (1, 5, 1)}, threshold=-1.25),
        # ties on the target: the lower slot is the new leader (new follower), and the two choices decide differently
        _case("tie_new_leader_low_slow", [_car(0, 0.0, 0, v=8.0, row=FAR), _car(33, 56.0, 1, v=0.0, dy=0.5),
                                          _car(64, 56.0, 1, v=16.0, dy=-0.5)], {0: (1, 5, 1)}, threshold=-4.0,
              margin=(0, 0)),
        _case("tie_new_leader_low_fast", [_car(0, 0.0, 0, v=8.0, row=FAR), _car(33, 56.0, 1, v=16.0, dy=0.5),
                                          _car(64, 56.0, 1, v=0.0, dy=-0.5)], {0: (0, 0, 0)}, threshold=-4.0,
              margin=(0, 0)),
        _case("tie_new_follower_low_slow", [_car(0, 0.0, 0, row=STD), _car(2, -16.0, 1, v=0.0, dy=0.5),
                                            _car(97, -16.0, 1, v=40.0, dy=-0.5)], {0: (1, 5, 1)}, b_safe=3.0),
        _case("tie_new_follower_low_fast", [_car(0, 0.0, 0, row=STD), _car(2, -16.0, 1, v=40.0, dy=0.5),
                                            _car(97, -16.0, 1, v=0.0, dy=-0.5)], {0: (0, 0, 0)}, b_safe=3.0),
        # simultaneous decisions: both changers take the same empty gap of lane 1 in the same tick
        _case("simultaneous", [_car(0, 0.0, 0, row=STD), _car(127, 0.0, 2, row=STD)], {0: (1, 5, 1), 127: (1, 5, -1)}),
        # K18 -> K17 -> K5 in one call: the changer's leader is the one ahead on its new lane
        _case("same_call_order", [_car(0, 0.0, 0, row=STD), _car(1, 20.0, 0), _car(2, 40.0, 1)], {0: (1, 5, 1)}),
    ]
    return cases


def lane_arrays(case):
    """``(x, y, v, type_id, ctrl_id, lane, cooldown)`` [1, M] of one lane case, the other slots empty."""
    x, y, v = (np.zeros((1, M), np.float32) for _ in range(3))
    tid = np.full((1, M), 255, np.uint8)
    cid = np.full((1, M), 255, np.uint8)
    lane = np.full((1, M), -1, np.int16)
    cool = np.zeros((1, M), np.int16)
    for slot, cx, cy, cv, row, ln, cd in case["cars"]:
        x[0, slot], y[0, slot], v[0, slot], tid[0, slot], cid[0, slot], lane[0, slot], cool[0, slot] = (
            cx, cy, cv, 0, row, ln, cd)
        assert float(np.float32(cx)) == cx and float(np.float32(cy)) == cy, (case["name"], slot)
    return x, y, v, tid, cid, lane, cool


def neighbours(case):
    return case.get("left", LEFT), case.get("right", RIGHT)
