"""Float64 restatement of ``PIDController`` (tactics2d/controller/pid_controller.py:159-406) and of the path-derived
lateral error of the batched PID rows (DESIGN.md section 1 "PID controller"; no reference counterpart).

Pinned by ``tests/golden/controllers_pid.npz`` (``tests/make_pid_golden.py``, the unmodified reference class).
``control_tick`` is ``oracle.controllers.control_tick`` with PID rows: it evaluates them here and hands every other row to
the existing restatement."""

from __future__ import annotations

import numpy as np

from oracle import controllers as OC

PID = 4
PID_LAT_NONE, PID_LAT_HEADING, PID_LAT_CROSS_TRACK, PID_LAT_PATH_HEADING, PID_LAT_PATH_CROSS_TRACK = 0, 1, 2, 3, 4
PID_LON_NONE, PID_LON_TARGET = 0, 1
PID_DEFAULTS = dict(dt=0.05, kp_lat=1.5, ki_lat=0.2, kd_lat=0.5, max_steering=0.5, kp_lon=2.0, ki_lon=0.3, kd_lon=0.4,
                    max_accel=3.0, min_accel=-5.0, derivative_filter_alpha=0.1, wheel_base=2.637)   # pid_controller.py:41-58, :356


def _clip(x, lo, hi):
    return np.minimum(np.maximum(x, lo), hi)      # np.clip: NaN propagates


def pid_channel(e, s, kp, ki, kd, dt, alpha, limits=None):
    """pid_controller.py:159-234: ``(output, (integral, e, derivative))`` from the error and s = (integral, prev_error,
    prev_derivative).  Python floats: one rounding per operation, in the reference's order."""
    integral, prev_e, prev_d = (float(v) for v in s)
    p_term = kp * e
    raw = (e - prev_e) / dt
    d = alpha * raw + (1 - alpha) * prev_d
    out = p_term + kd * d
    saturated = False
    if limits is not None:
        lo, hi = limits
        if out > hi:
            saturated, out = True, hi
        elif out < lo:
            saturated, out = True, lo
    integral = integral * 0.99 if saturated else integral + e * dt
    out = out + ki * integral
    if limits is not None:
        out = float(_clip(out, limits[0], limits[1]))
    return out, (integral, e, d)


def path_closest(path, x, y):
    """The closest point of a polyline to (x, y) and the unit tangent of its segment: ``(cx, cy, ux, uy)``, or None when
    every segment has zero length.  Segments in order, ``t = clamp(((p - a).(b - a)) / |b - a|^2, 0, 1)``,
    ``c = a + t (b - a)``; the first strict minimum of ``|p - c|^2`` wins.  Python floats, in the kernel's order."""
    path = np.asarray(path, np.float64)
    best = None
    for i in range(len(path) - 1):
        ax, ay = float(path[i, 0]), float(path[i, 1])
        dx, dy = float(path[i + 1, 0]) - ax, float(path[i + 1, 1]) - ay
        l2 = dx * dx + dy * dy
        if not l2 > 0.0:
            continue
        t = min(max(((x - ax) * dx + (y - ay) * dy) / l2, 0.0), 1.0)
        qx, qy = ax + t * dx, ay + t * dy
        ex, ey = x - qx, y - qy
        d2 = ex * ex + ey * ey
        if best is None or d2 < best[0]:
            ln = float(np.sqrt(l2))
            best = (d2, qx, qy, dx / ln, dy / ln)
    return None if best is None else best[1:]


def path_lateral_error(path, x, y, heading, cross):
    """PATH_CROSS_TRACK (``cross``): ``u.x (c.y - y) - u.y (c.x - x)``, positive when the path lies to the left;
    PATH_HEADING: the heading error towards ``atan2(u.y, u.x)``.  None without a usable segment."""
    c = path_closest(path, x, y)
    if c is None:
        return None
    cx, cy, ux, uy = c
    if cross:
        return ux * (cy - y) - uy * (cx - x)
    err = float(np.arctan2(uy, ux)) - heading
    return float(np.arctan2(np.sin(err), np.cos(err)))


def pid_step(p, x, y, heading, speed, target_speed, lat_target, state, path=None):
    """One PIDController.step of one participant (pid_controller.py:309-406): ``(steering, acceleration, state')``.

    ``p`` holds the row (``pid_lateral`` / ``pid_longitudinal`` sources, the gains, ``dt``,
    ``derivative_filter_alpha``, ``max_steering``, ``max_accel`` / ``min_accel``, ``wheel_base``); ``state`` the six
    values (lat integral, previous error, derivative, then the same for lon).  A channel whose source is NONE, or a PATH
    source without a usable ``path``, gives 0 and keeps its half of the state."""
    st = [float(v) for v in state]
    x, y, heading, speed = float(x), float(y), float(heading), float(speed)
    dt, alpha = float(p["dt"]), float(p["derivative_filter_alpha"])
    steer = acc = 0.0
    lat = int(p["pid_lateral"])
    if lat != PID_LAT_NONE:
        e = None
        if lat == PID_LAT_HEADING:
            err = float(lat_target) - heading
            e = float(np.arctan2(np.sin(err), np.cos(err)))
        elif lat == PID_LAT_CROSS_TRACK:
            e = float(lat_target)
        elif path is not None:
            e = path_lateral_error(path, x, y, heading, lat == PID_LAT_PATH_CROSS_TRACK)
        if e is not None:
            out, st[0:3] = pid_channel(e, st[0:3], float(p["kp_lat"]), float(p["ki_lat"]), float(p["kd_lat"]), dt, alpha)
            if lat in (PID_LAT_CROSS_TRACK, PID_LAT_PATH_CROSS_TRACK):
                out = out * (2.0 / float(p["wheel_base"]))
            ms = float(p["max_steering"])
            steer = float(_clip(out, -ms, ms))
    if int(p["pid_longitudinal"]) == PID_LON_TARGET:
        lim = (float(p["min_accel"]), float(p["max_accel"]))
        out, st[3:6] = pid_channel(float(target_speed) - speed, st[3:6], float(p["kp_lon"]), float(p["ki_lon"]),
                                   float(p["kd_lon"]), dt, alpha, lim)
        acc = float(_clip(out, lim[0], lim[1]))
    return steer, acc, st


def control_tick(state, type_id, table, action, ctrl_id, ctrl_table, lead_index, path_id, paths, last_accel,
                 steer_first, pid_target, pid_state):
    """``oracle.controllers.control_tick`` with PID rows: ``(action', last_accel', pid_state')``.

    The PID rows of controlled, active slots are evaluated with ``pid_step`` on their row of ``pid_target`` [N, M, 2] and
    ``pid_state`` [N, M, 6] and written into the action buffer (fp32); the existing restatement then runs every other
    row, keeps the PID rows' actions (they are EXTERNAL to it) and computes ``last_accel'`` from the final buffer."""
    x, y, h, v = (np.asarray(state[k], np.float64) for k in ("x", "y", "heading", "speed"))
    N, M = x.shape
    act = np.array(action, np.float32, copy=True)
    new_state = np.array(pid_state, np.float64, copy=True)
    for n in range(N):
        for m in range(M):
            cid = int(ctrl_id[n, m])
            if cid == 255 or int(type_id[n, m]) == 255 or int(ctrl_table[cid]["kind"]) != PID:
                continue
            pi = -1 if path_id is None else int(path_id[n, m])
            tg = pid_target[n, m]
            steer, acc, new_state[n, m] = pid_step(ctrl_table[cid], x[n, m], y[n, m], h[n, m], v[n, m], tg[0], tg[1],
                                                   new_state[n, m], paths[pi] if 0 <= pi < len(paths) else None)
            act[n, m] = (steer, acc) if steer_first else (acc, steer)
    others = [dict(r, kind=OC.EXTERNAL) if int(r["kind"]) == PID else r for r in ctrl_table]
    out, la = OC.control_tick(state, type_id, table, act, ctrl_id, others, lead_index, path_id, paths, last_accel,
                              steer_first)
    return out, la, new_state
