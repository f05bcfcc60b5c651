"""Float64 restatement of DESIGN.md section 1 "Route following" (TEST INFRASTRUCTURE ONLY): the closest point of a route,
its arc length s and the route's length L, the OffRoute detector and the progress term of both epilogues, and the rows of
K12 (``t2d_route_observe``).

The closest point and its tie rule are ``tests.pid_oracle.path_closest`` (what K5's PATH sources use); ``closest`` adds the
arc length by walking the same segments in the same order, and checks that it lands on the point ``path_closest`` chose.
Python floats: one rounding per operation, in the kernels' order."""

from __future__ import annotations

import math

import numpy as np

from oracle import scenario as O
from tests import pid_oracle as P

OFF_ROUTE = 5
FIELDS = 5


def closest(path, x, y):
    """``(cx, cy, ux, uy, d, s, L)`` of the route ``path`` [V, 2] seen from (x, y), or None when no segment has non-zero
    length."""
    path = np.asarray(path, np.float64)
    x, y = float(x), float(y)
    c = P.path_closest(path, x, y)
    if c is None:
        return None
    best, s, acc = None, None, 0.0
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
        ln = math.sqrt(l2)
        if best is None or d2 < best[0]:
            best = (d2, qx, qy)
            s = acc + t * ln
        acc = acc + ln
    assert (best[1], best[2]) == (c[0], c[1]), "the arc-length walk must pick path_closest's point"
    return c[0], c[1], c[2], c[3], math.sqrt(best[0]), s, acc


def probe(path, x, y, threshold):
    """``(state, s)``: state 0 = no route, 1 = on route, 2 = off route (d > threshold)."""
    if path is None:
        return 0, 0.0
    c = closest(path, x, y)
    if c is None:
        return 0, 0.0
    return (2 if c[4] > threshold else 1), c[5]


def progress(s, best, weight):
    """``(term, best')`` of a NORMAL step on the route: the fp32-rounded ``weight (s - best)`` when s > best (nothing on
    the first step, best = -inf), the tracker after it."""
    if not s > best:
        return 0.0, best
    return (0.0 if best == -np.inf else float(np.float32(weight * (s - best)))), s


def _path(paths, rid):
    return paths[rid] if 0 <= rid < len(paths) else None


def env_epilogue(flags, scn_status, step_count, max_step, x, y, route_id, paths, threshold, weight, off_reward,
                 s_best, reset_trackers=True, **goal):
    """The env epilogue with routes: ``oracle.scenario.env_epilogue`` (``goal`` its goal keywords) on the tick's outputs,
    then OffRoute and the progress term of the ego (slot 0).  ``x``, ``y``, ``route_id`` [N, M]; ``s_best`` [N].  Returns
    its dict plus ``s_best``; ``reward`` is fp32."""
    N = np.asarray(flags).shape[0]
    base = O.env_epilogue(flags, scn_status, step_count, max_step, reset_trackers=reset_trackers, **goal)
    reward = base["reward"].astype(np.float32)
    term, trunc, traffic = base["terminated"].copy(), base["truncated"].copy(), base["traffic_status"].copy()
    s_best = np.array(s_best, np.float64)
    for n in range(N):
        st = int(scn_status[n])
        if st not in (O.NORMAL, O.COMPLETED):
            continue
        state, s = probe(_path(paths, int(route_id[n, 0])), float(np.float32(x[n, 0])), float(np.float32(y[n, 0])),
                         threshold)
        if state == 2:
            traffic[n, 0] = OFF_ROUTE
            term[n], trunc[n] = False, True
            reward[n] = np.float32(off_reward)
        elif state == 1 and st == O.NORMAL:
            t, s_best[n] = progress(s, s_best[n], weight)
            reward[n] = np.float32(reward[n] + np.float32(t))
    done = term | trunc
    if reset_trackers:
        s_best[done] = -np.inf
    return dict(base, reward=reward, terminated=term, truncated=trunc, done=done.astype(np.uint8), traffic_status=traffic,
                s_best=s_best)


def agent_rows(status, x, y, type_id, n_types, route_id, paths, threshold, observers=None):
    """OffRoute per agent row on the statuses K10 gives without routes: ``(status', probe state [N, Q], s [N, Q])``."""
    status = np.array(status)
    N, Q = status.shape
    M = np.asarray(type_id).shape[1]
    state, svals = np.zeros((N, Q), np.int64), np.zeros((N, Q))
    for n in range(N):
        for q in range(Q):
            j = q if observers is None else int(observers[n, q])
            if not (0 <= j < M) or type_id[n, j] >= n_types or status[n, q] not in (O.NORMAL, O.COMPLETED):
                continue
            state[n, q], svals[n, q] = probe(_path(paths, int(route_id[n, j])), float(np.float32(x[n, j])),
                                             float(np.float32(y[n, j])), threshold)
    status[state == 2] = O.FAILED
    return status, state, svals


def observe_row(path, x, y, heading, n_points, spacing):
    """One K12 row (float64, before the fp32 rounding) of an observer at (x, y, heading) on ``path``; zeros without a
    route."""
    F = FIELDS + 2 * n_points
    c = None if path is None else closest(path, float(x), float(y))
    if c is None:
        return np.zeros(F)
    x, y, h = float(x), float(y), float(heading)
    cx, cy, ux, uy, d, s, L = c
    err = math.atan2(uy, ux) - h
    err = math.atan2(math.sin(err), math.cos(err))
    if err == -math.pi:
        err = math.pi
    out = [1.0, ux * (cy - y) - uy * (cx - x), err, s / L, L - s]
    cs, sn = math.cos(h), math.sin(h)
    pts = np.asarray(path, np.float64)
    seg, acc = 0, 0.0
    for k in range(1, n_points + 1):
        sig = min(s + k * float(spacing), L)
        px, py = float(pts[-1, 0]), float(pts[-1, 1])
        while seg + 1 < len(pts):
            ax, ay = float(pts[seg, 0]), float(pts[seg, 1])
            dx, dy = float(pts[seg + 1, 0]) - ax, float(pts[seg + 1, 1]) - ay
            l2 = dx * dx + dy * dy
            if not l2 > 0.0:
                seg += 1
                continue
            ln = math.sqrt(l2)
            end = acc + ln
            if sig <= end:
                t = (sig - acc) / ln
                px, py = ax + t * dx, ay + t * dy
                break
            acc = end
            seg += 1
        ex, ey = px - x, py - y
        out += [ex * cs + ey * sn, ey * cs - ex * sn]
    return np.asarray(out)


def observe(x, y, heading, type_id, n_types, route_id, paths, n_points, spacing, observers=None, Q=None):
    """K12 on the state: [N, Q, F] (``observers`` None: row q is slot q, Q rows)."""
    N, M = np.asarray(x).shape
    Q = (M if Q is None else Q) if observers is None else np.asarray(observers).shape[1]
    out = np.zeros((N, Q, FIELDS + 2 * n_points))
    for n in range(N):
        for q in range(Q):
            j = q if observers is None else int(observers[n, q])
            if not (0 <= j < M) or type_id[n, j] >= n_types:
                continue
            out[n, q] = observe_row(_path(paths, int(route_id[n, j])), np.float32(x[n, j]), np.float32(y[n, j]),
                                    np.float32(heading[n, j]), n_points, spacing)
    return out
