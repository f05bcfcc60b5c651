"""The closed-loop car-following scene of the leader-search tests (TEST INFRASTRUCTURE ONLY): three lanes of IDM cars
behind a scripted ego that brakes hard, and a scripted car that changes from lane 1 into lane 0 between the ego and the
first lane-0 follower, then brakes too.  Every IDM car follows its lane's path, so the search takes the path frame for
them; the two scripted slots take the heading frame.

The reference's IDM shrinks its desired gap while it closes in (``v * (v_lead - v)`` in s*), so ``min_spacing`` is what
keeps a follower off a stopped leader: 20 m, well above the 4.8 m car length.  With every leader found this scene has no
collision; with ``lead_index = -1`` the lane-0 followers drive into the stopped cars."""

from __future__ import annotations

import numpy as np

LANE_W = 3.5
HALF_WIDTH, MAX_RANGE = 1.8, 100.0
EGO, CUT_IN = 0, 10
IDM_SLOTS = list(range(1, 10))
STEER_TICKS = 14


def table():
    from tactics2d_b200.types import TypeParams, TypeTable

    return TypeTable([TypeParams(half_len=2.4, half_wid=0.95, lf=1.3, lr=1.3, steer_lo=-0.6, steer_hi=0.6, speed_lo=0.0,
                                 speed_hi=40.0, accel_lo=-8.0, accel_hi=4.0)])


def controllers():
    from tactics2d_b200.controller import IDMController

    return [IDMController(desired_speed=15.0, time_headway=1.0, min_spacing=20.0, max_acceleration=2.0,
                          comfortable_deceleration=6.0)]


def scene():
    """``(state dict of [1, M] float64 arrays (fp32 values), type_id, ctrl_id, path_id, paths)``."""
    xs, ys, v, ctrl, pid = [100.0], [0.0], [15.0], [255], [-1]
    for lane in range(3):
        for k in range(3):
            xs.append(55.0 - 35.0 * k - 5.0 * lane)
            ys.append(LANE_W * lane)
            v.append(15.0)
            ctrl.append(0)
            pid.append(lane)
    xs.append(80.0); ys.append(LANE_W); v.append(12.0); ctrl.append(255); pid.append(-1)
    m = len(xs)
    z = np.zeros((1, m))
    st = dict(x=np.array([xs]), y=np.array([ys]), heading=z, speed=np.array([v]), vx=z, vy=z)
    st = {k: np.asarray(a, np.float32).astype(np.float64) for k, a in st.items()}
    paths = [np.array([[-50.0, LANE_W * l], [600.0, LANE_W * l]], np.float32) for l in range(3)]
    return st, np.zeros((1, m), np.uint8), np.array([ctrl], np.uint8), np.array([pid], np.int16), paths


def script(t, m):
    """The external (accel, steer) rows of tick t: the ego brakes at -4 m/s^2 from t = 10; the cut-in steers right, then
    back, and brakes once it is in lane 0."""
    a = np.zeros((1, m, 2), np.float32)
    a[0, EGO] = (-4.0 if t >= 10 else 0.0, 0.0)
    a[0, CUT_IN] = (-4.0 if t >= 2 * STEER_TICKS else 0.0,
                    -0.03 if t < STEER_TICKS else (0.03 if t < 2 * STEER_TICKS else 0.0))
    return a
