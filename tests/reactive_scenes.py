"""The closed-loop scenes of the reactive-replay tests (TEST INFRASTRUCTURE ONLY).

``stopped_ego``: the car-following highway of ``tactics2d_b200.synthetic.idm_highway_log`` (three lanes, 60 s) with the
ego parked in the middle lane, where the recording's cars drive straight through it, as one episode row with slot reuse.
``cruise``: one constant-speed track on a straight diagonal, with the ego parked far away.  Every replayed slot drives
with the IDM and a PID cross-track channel on its track's path."""

from __future__ import annotations

import numpy as np

HALF_WIDTH, MAX_RANGE = 1.8, 100.0
LANE_W = 3.5
MIN_SPACING = 30.0
DESIRED = (12.0, 14.0, 16.0)


def controller():
    from tactics2d_b200.controller import IDMController, PIDController

    keep = PIDController(dt=0.1, kp_lat=0.03, ki_lat=0.0, kd_lat=0.08, max_steering=0.2, derivative_filter_alpha=1.0,
                         lateral_error="path_cross_track")
    # the reference's IDM brakes for a closing speed only through min_spacing (its s* adds v (v_lead - v) / (2 sqrt(a b)),
    # which is negative when closing in): a large min_spacing and max_acceleration make it stop short of a stopped car
    return IDMController(desired_speed=15.0, time_headway=1.0, min_spacing=MIN_SPACING, max_acceleration=8.0,
                         comfortable_deceleration=9.0, lateral=keep)


def ctab():
    """Row 0 as the oracles take it."""
    r = controller().params()
    return [{k: getattr(r, k) for k, _ in r._fields_}]


def _with_parked(log, x, y, heading=0.0):
    """``log`` plus one track parked at (x, y) over the whole recording; returns the new log and the parked track's id."""
    from dataclasses import replace

    first, last = min(int(log.first_ms.min()), 0), int(log.last_ms.max())
    period = int(log.period_ms[0])
    n = (last - first) // period + 1
    rec = np.zeros((n, 5), np.float32)
    rec[:, 0], rec[:, 1], rec[:, 2] = x, y, heading
    pid = int(log.ids.max()) + 1
    out = replace(log, ids=np.append(log.ids, pid), first_ms=np.append(log.first_ms, np.int32(first)),
                  n_frames=np.append(log.n_frames, np.int32(n)), period_ms=np.append(log.period_ms, np.int32(period)),
                  records=np.ascontiguousarray(np.concatenate([log.records, rec])),
                  type_row=np.append(log.type_row, log.type_row[:1]), cls=list(log.cls) + [log.cls[0]],
                  length=np.append(log.length, 4.5), width=np.append(log.width, 1.9))
    return out, pid


def table():
    """The kinematic templates without reverse (``speed_lo = 0``): the reference's IDM keeps braking below 0 m/s, so a car
    that stops inside ``min_spacing`` on a row that can reverse backs away into the car behind it."""
    from dataclasses import replace

    from tactics2d_b200.types import TypeTable

    return TypeTable([replace(r, speed_lo=0.0) for r in TypeTable.from_templates("kinematics").rows])


def stopped_ego(m=64, t0=5000, seed=0):
    """``(episodes, ego_x)``: the ego parked in lane 1 of a 60 s recording at 12 to 16 m/s, a car every 5 s per lane
    (farther apart than the controller's ``min_spacing``), where the nearest car behind
    it at ``t0`` is farthest away (over x in [600, 720] of the 800 m road: the queue behind it stays short, as every car
    still leaves at its logged exit)."""
    from tactics2d_b200.dataset_parser.replay import build_replay_episodes
    from tactics2d_b200.synthetic import idm_highway_log

    log = idm_highway_log(60000, seed, lane_width=LANE_W, desired=DESIRED, headway_s=5.0)
    j = (t0 - log.first_ms.astype(np.int64)) // log.period_ms
    on = (j >= 0) & (j < log.n_frames)
    xs = np.array([log.records[o + jj] for o, jj, k in zip(log.rec_off, j, on) if k])
    lane1 = np.sort(xs[np.abs(xs[:, 1] - LANE_W) < 0.5, 0])
    best, ego_x = -1.0, 450.0
    for x in np.arange(600.0, 720.0, 5.0):
        behind = lane1[lane1 < x]
        ahead = lane1[lane1 >= x]
        clear_ahead = not len(ahead) or ahead[0] - x > 8.0
        d = x - behind[-1] if len(behind) else np.inf
        if clear_ahead and d > best:
            best, ego_x = d, float(x)
    log, ego = _with_parked(log, ego_x, LANE_W)
    eps = build_replay_episodes(log, m, [t0], [ego], table(), reuse_slots=True)
    assert eps.dropped.sum() == 0
    return eps, ego_x


def cruise(m=4, speed=25.0, heading=0.3, period_ms=40):
    """``(episodes, track)``: a constant-speed track on a straight line at ``heading``, entering at 1 s, and the ego parked
    300 m to the side."""
    from tactics2d_b200.dataset_parser.replay import ReplayLog, build_replay_episodes
    from tactics2d_b200.participant.element import Vehicle

    n = 20000 // period_ms + 1
    s = speed * np.arange(n) * period_ms / 1000.0
    c, sn = np.cos(heading), np.sin(heading)
    rec = np.stack([s * c, s * sn, np.full(n, heading), np.full(n, speed * c), np.full(n, speed * sn)], 1).astype(np.float32)
    log = ReplayLog(ids=np.array([0], np.int64), first_ms=np.array([1000], np.int32), n_frames=np.array([n], np.int32),
                    period_ms=np.array([period_ms], np.int32), records=rec, type_row=np.array([255], np.uint8),
                    cls=[Vehicle], length=np.array([4.5]), width=np.array([1.9]))
    log, ego = _with_parked(log, 0.0, 300.0)
    return build_replay_episodes(log, m, [0], [ego], table(), reuse_slots=True), 0
