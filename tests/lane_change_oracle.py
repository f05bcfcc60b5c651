"""Float64 restatement of DESIGN.md section 1 "Lane changes" (TEST INFRASTRUCTURE ONLY): the MOBIL decision of K18
(``t2d_set_lane_change``), whether each decision is robust to the last bits of the arithmetic, and the controller pass
with lane keeping (IDM rows with a lateral channel) that the closed-loop rollouts run.

Projections are ``tests.route_oracle.closest`` (K17's ``closest_on_path<true>``), accelerations ``oracle.controllers.idm``
and the lateral channel ``tests.pid_oracle.pid_step``.  Python floats: one rounding per operation, in the kernel's order.
A decision is robust when no quantity it compares lies within ``EPS`` of its bound: a distance to a path against
``half_width``, a gap against 0 and ``max_range``, a blocking distance against ``min_gap``, the best gap against the
runner-up, ``a(n | c)`` against ``-b_safe``, an incentive against ``threshold`` and the two incentives against each other."""

from __future__ import annotations

import numpy as np

from oracle import controllers as OC
from tests import pid_oracle as P
from tests import route_oracle as R

SHAPE_NONE = 2
IDM = OC.IDM
EPS = 1e-9


def _usable(paths, p):
    return 0 <= p < len(paths) and R.closest(np.asarray(paths[p], np.float64), 0.0, 0.0) is not None


def _idm_row(ctab, cid):
    return 0 <= cid < len(ctab) and int(ctab[cid]["kind"]) == IDM


def decide(x, y, v, type_id, shapes, ctrl_id, ctab, lane_path, cooldown, left, right, paths, half_width, max_range,
           politeness=0.0, threshold=0.2, b_safe=2.0, min_gap=6.0, cool_ticks=10, eps=EPS):
    """K18 on one state.  ``x``, ``y``, ``v``, ``type_id``, ``ctrl_id``, ``lane_path``, ``cooldown`` [N, M] (fp32 values);
    ``shapes`` per type row; ``ctab`` the controller rows as dicts; ``left`` / ``right`` per path.  Returns
    ``dict(lane_path, cooldown, change, robust [N, M], changer [N, M], decisions)``; ``decisions`` lists, per change, a
    dict with the slot, the side, the new follower and its predicted ``a(n | c)``."""
    x, y, v = (np.asarray(np.asarray(a, np.float32), np.float64) for a in (x, y, v))
    type_id, ctrl_id = np.asarray(type_id), np.asarray(ctrl_id)
    N, M = x.shape
    shapes = np.asarray(shapes)
    nt = len(shapes)
    hw, rng = float(half_width), float(max_range)
    paths = [np.asarray(p, np.float64) for p in paths]
    lane_out = np.array(lane_path, np.int16, copy=True)
    cool_in = np.asarray(cooldown, np.int64)
    cool_out = np.where(cool_in > 0, cool_in - 1, cool_in).astype(np.int16)
    change = np.zeros((N, M), np.int8)
    robust = np.ones((N, M), bool)
    changer = np.zeros((N, M), bool)
    decisions = []
    for n in range(N):
        active = type_id[n] < nt
        finite = ~(np.isnan(x[n]) | np.isnan(y[n]))
        cand = active & finite & (shapes[np.where(active, type_id[n], 0)] != SHAPE_NONE)
        rows = [int(ctrl_id[n, m]) if _idm_row(ctab, int(ctrl_id[n, m])) else None for m in range(M)]
        proj = {}

        def on(r):   # (s, d) of every slot on path r that is a candidate or may decide
            if r not in proj:
                proj[r] = {k: R.closest(paths[r], x[n, k], y[n, k]) for k in range(M) if active[k] and finite[k]}
            return proj[r]

        def acc(own, f, lead):
            row = ctab[rows[f] if rows[f] is not None else own]
            has = lead is not None
            li = lead if has else f
            return float(OC.idm(v[n, f], x[n, f], y[n, f], has, v[n, li], x[n, li], y[n, li], row))

        for c in range(M):
            cid = int(ctrl_id[n, c])
            p = int(lane_path[n, c])
            if not (active[c] and finite[c] and rows[c] is not None and int(ctab[cid].get("pid_lateral", 0)) != 0
                    and cool_in[n, c] <= 0 and _usable(paths, p)):
                continue
            qs = [int(left[p]), int(right[p])]
            qs = [q if _usable(paths, q) else None for q in qs]
            if qs == [None, None]:
                continue
            ok = True

            def walk(r):
                nonlocal ok
                pr = on(r)
                sc = pr[c][5]
                best_a, best_b, blocked = [], [], False
                for j in range(M):
                    if j == c or not cand[j]:
                        continue
                    d, sj = pr[j][4], pr[j][5]
                    if abs(d - hw) <= eps:
                        ok = False
                    if not d <= hw:
                        continue
                    g, gb = sj - sc, sc - sj
                    if abs(abs(g) - min_gap) <= eps or abs(g) <= eps or abs(g - rng) <= eps or abs(gb - rng) <= eps:
                        ok = False
                    if abs(g) < min_gap:
                        blocked = True
                    if 0.0 < g <= rng:
                        best_a.append((g, j))
                    if 0.0 < gb <= rng:
                        best_b.append((gb, j))
                out = []
                for lst in (best_a, best_b):
                    lst.sort()
                    if len(lst) > 1 and lst[1][0] - lst[0][0] <= eps:
                        ok = False
                    out.append(lst[0][1] if lst else None)
                return out[0], out[1], blocked, pr[c][4]

            l, o, _, dc = walk(p)
            if abs(dc - hw) <= eps:
                robust[n, c] = False
            if not dc <= hw:
                continue
            changer[n, c] = True
            a_c = acc(cid, c, l)
            d_o = (acc(cid, o, l) - acc(cid, o, c)) if o is not None else 0.0
            incs = []
            for side, q in enumerate(qs):
                if q is None:
                    continue
                ln, nn, blocked, _ = walk(q)
                if blocked:
                    continue
                at_c = acc(cid, c, ln)
                d_n, at_n = 0.0, None
                if nn is not None:
                    at_n = acc(cid, nn, c)
                    if abs(at_n + b_safe) <= eps:
                        ok = False
                    if not at_n >= -b_safe:
                        continue
                    d_n = at_n - acc(cid, nn, ln)
                inc = (at_c - a_c) + politeness * (d_n + d_o)
                if abs(inc - threshold) <= eps:
                    ok = False
                if inc > threshold:
                    incs.append((inc, side, q, nn, at_n))
            if len(incs) == 2 and abs(incs[0][0] - incs[1][0]) <= eps:
                ok = False
            robust[n, c] &= ok
            if not incs:
                continue
            pick = incs[0] if len(incs) == 1 or not incs[1][0] > incs[0][0] else incs[1]
            inc, side, q, nn, at_n = pick
            lane_out[n, c] = q
            cool_out[n, c] = cool_ticks
            change[n, c] = 1 if side == 0 else -1
            decisions.append(dict(n=n, slot=c, side=change[n, c], to=q, incentive=inc, follower=nn, a_follower=at_n))
    return dict(lane_path=lane_out, cooldown=cool_out, change=change, robust=robust, changer=changer, decisions=decisions)


def control_tick(state, type_id, table, action, ctrl_id, ctab, lead, lane_path, paths, last_accel, pid_state,
                 steer_first=False):
    """K5 with lane keeping: ``oracle.controllers.control_tick`` on ``lead`` and the current lanes, then the steering of
    every IDM row with a lateral channel from ``tests.pid_oracle.pid_step`` (the lateral half only) on its row of
    ``pid_state``.  Returns ``(action', last_accel', pid_state')``."""
    x, y, h, v = (np.asarray(state[k], np.float64) for k in ("x", "y", "heading", "speed"))
    N, M = x.shape
    paths64 = [np.asarray(p, np.float64) for p in paths]
    out, _ = OC.control_tick(state, type_id, table, action, ctrl_id, ctab, lead, lane_path, paths64, last_accel,
                             steer_first)
    st = np.array(pid_state, np.float64, copy=True)
    si = 0 if steer_first else 1
    for n in range(N):
        for m in range(M):
            cid = int(ctrl_id[n, m])
            if cid == 255 or int(type_id[n, m]) == 255 or not _idm_row(ctab, cid) or int(ctab[cid]["pid_lateral"]) == 0:
                continue
            pi = int(lane_path[n, m])
            row = dict(ctab[cid], pid_longitudinal=P.PID_LON_NONE)
            steer, _, st[n, m] = P.pid_step(row, x[n, m], y[n, m], h[n, m], v[n, m], 0.0, 0.0, st[n, m],
                                            paths64[pi] if 0 <= pi < len(paths64) else None)
            out[n, m, si] = np.float32(steer)
    return out, OC.applied_accel_magnitude(out, type_id, table, steer_first).astype(np.float32), st
