"""The closed-loop scenes of the lane-change tests (TEST INFRASTRUCTURE ONLY).

``highway``: three straight lanes 3.5 m apart (lane 0 at y = 0, lane 1 to its left, lane 2 left of that).  Slow scripted
cars (no controller, 6 m/s, no action) sit in lanes 0 and 2; faster IDM cars that keep their lane (a PID cross-track
channel) follow them.  As in tests/leader_scenes.py, ``min_spacing`` (20 m) is what keeps the reference's IDM off a slow
leader.  With MOBIL the lane-0 cars overtake through lane 1, on the left.
``rings``: two concentric arcs (radius 150 m and 153.5 m) driven anticlockwise, so the inner ring is the outer ring's left
neighbour; a slow scripted car on the outer ring and IDM cars behind it."""

from __future__ import annotations

import math

import numpy as np

LANE_W = 3.5
HALF_WIDTH, MAX_RANGE = 1.8, 100.0
LANE = dict(politeness=0.2, threshold=0.3, b_safe=4.0, min_gap=10.0, cooldown=30)


def table():
    from tactics2d_b200.types import TypeParams, TypeTable

    return TypeTable([TypeParams(half_len=2.4, half_wid=0.95, lf=1.3, lr=1.3, steer_lo=-0.6, steer_hi=0.6, speed_lo=0.0,
                                 speed_hi=40.0, accel_lo=-8.0, accel_hi=4.0)])


def controllers():
    """Row 0: the IDM with lane keeping every controlled car drives."""
    from tactics2d_b200.controller import IDMController, PIDController

    keep = PIDController(dt=0.1, kp_lat=0.03, ki_lat=0.0, kd_lat=0.08, max_steering=0.2, derivative_filter_alpha=1.0,
                         lateral_error="path_cross_track")
    return [IDMController(desired_speed=16.0, time_headway=1.0, min_spacing=20.0, max_acceleration=2.0,
                          comfortable_deceleration=6.0, lateral=keep)]


def ctab():
    """The rows as the oracles take them."""
    return [{k: getattr(r, k) for k, _ in r._fields_} for r in (c.params() for c in controllers())]


def _state(xs, ys, hs, vs, ctrl, pid):
    m = len(xs)
    z = np.zeros((1, m))
    st = dict(x=np.array([xs]), y=np.array([ys]), heading=np.array([hs]), speed=np.array([vs]), vx=z, vy=z)
    st = {k: np.asarray(a, np.float32).astype(np.float64) for k, a in st.items()}
    return st, np.zeros((1, m), np.uint8), np.array([ctrl], np.uint8), np.array([pid], np.int16)


def highway():
    """``(state dict of [1, M] float64 arrays (fp32 values), type_id, ctrl_id, path_id, paths, left, right, lane-0 IDM
    slots)``."""
    cars = [(90.0, 0, 6.0, 255), (50.0, 0, 13.0, 0), (20.0, 0, 14.0, 0), (-10.0, 0, 14.0, 0),   # lane 0
            (-60.0, 1, 15.0, 0),                                                                  # lane 1
            (140.0, 2, 6.0, 255), (100.0, 2, 12.0, 0)]                                            # lane 2
    xs = [c[0] for c in cars]
    st, tid, cid, pid = _state(xs, [LANE_W * c[1] for c in cars], [0.0] * len(cars), [c[2] for c in cars],
                               [c[3] for c in cars], [c[1] for c in cars])
    paths = [np.array([[-200.0 + 100.0 * k, LANE_W * l] for k in range(13)], np.float32) for l in range(3)]
    return st, tid, cid, pid, paths, [1, 2, -1], [-1, 0, 1], [1, 2, 3]


def _arc(radius, n=129, a0=-0.3, a1=2.0):
    a = np.linspace(a0, a1, n)
    return np.stack([radius * np.cos(a), radius * np.sin(a)], 1).astype(np.float32)


def rings():
    """The same tuple on the two rings: path 0 the outer ring, path 1 the inner one (its left)."""
    r_out, r_in = 150.0 + LANE_W, 150.0
    cars = [(0.45, 0, 5.0, 255), (0.2, 0, 11.0, 0), (-0.05, 0, 11.0, 0)]
    xs = [r_out * math.cos(a) for a, *_ in cars]
    ys = [r_out * math.sin(a) for a, *_ in cars]
    hs = [a + math.pi / 2 for a, *_ in cars]
    st, tid, cid, pid = _state(xs, ys, hs, [c[2] for c in cars], [c[3] for c in cars], [c[1] for c in cars])
    return st, tid, cid, pid, [_arc(r_out), _arc(r_in)], [1, -1], [-1, 0], [1, 2]


def rollout(scene, lanes=True, ticks=150):
    """The scene in float64: IDM with lane keeping, the leader search, the lane change (``lanes``) and the kinematic tick.
    Returns ``dict(hits, speed [ticks, M], lane [ticks, M], change [ticks, M], decisions, states)``: the dynamic-collision
    flags OR-ed over the rollout, the speeds, lanes and decisions of every tick, and the state each was decided on."""
    from oracle import scenario as O
    from tests import lane_change_oracle as LC
    from tests import leader_oracle as L

    st, tid, cid, pid, paths, left, right, _ = scene
    tab = table().as_oracle_table()
    rows = ctab()
    m = tid.shape[1]
    la = np.zeros((1, m))
    ps = np.zeros((1, m, 6))
    lane, cool = pid.copy(), np.zeros((1, m), np.int16)
    hits = np.zeros((1, m), np.uint8)
    out = dict(speed=[], lane=[], change=[], decisions=[], states=[])
    for t in range(ticks):
        if lanes:
            d = LC.decide(st["x"], st["y"], st["speed"], tid, [0], cid, rows, lane, cool, left, right, paths, HALF_WIDTH,
                          MAX_RANGE, **{k: LANE[k] for k in ("politeness", "threshold", "b_safe", "min_gap")},
                          cool_ticks=LANE["cooldown"])
            lane, cool = d["lane_path"], d["cooldown"]
            out["change"].append(d["change"])
            out["decisions"].append(d["decisions"])
        out["states"].append(st)
        lead = L.find(st["x"], st["y"], st["heading"], tid, [0], HALF_WIDTH, MAX_RANGE, lane, paths)["lead"]
        act, la, ps = LC.control_tick(st, tid, tab, np.zeros((1, m, 2), np.float32), cid, rows, lead, lane, paths, la, ps)
        st = O.physics_tick(st, tid, act, tab, 100, 5)
        st = {k: np.asarray(v, np.float32).astype(np.float64) for k, v in st.items()}
        hits |= O.events(st["x"], st["y"], st["heading"], tid, tab)[0] & O.F_DYNAMIC
        out["speed"].append(st["speed"][0].copy())
        out["lane"].append(lane[0].copy())
    out["hits"] = hits
    out["speed"], out["lane"] = np.array(out["speed"]), np.array(out["lane"])
    return out
