"""Float64 restatement of DESIGN.md section 1 "Yielding at conflict zones" (TEST INFRASTRUCTURE ONLY): whom every slot
yields to (K19, ``t2d_find_yields``), where it stops, whether that answer is robust to the last bits of the arithmetic,
and the acceleration K5's yielding instance gives an IDM row.

Projections use ``tests.route_oracle.closest`` (the closest point and arc length K17 and the route code use).  Python
floats: one rounding per operation, in the kernel's order."""

from __future__ import annotations

import math

import numpy as np

from oracle import controllers as OC
from tests import route_oracle as R

SHAPE_NONE = 2
IDM = OC.IDM
EPS = 1e-9   # a quantity within this of a bound it is compared with: the answer is not robust


def _usable(paths, p):
    return 0 <= p < len(paths) and R.closest(paths[p], 0.0, 0.0) is not None


def point_at(path, s):
    """p's point at arc length clamp(s, 0, L): the library's stop point."""
    s = max(float(s), 0.0)
    acc = 0.0
    x, y = float(path[0, 0]), float(path[0, 1])
    for i in range(len(path) - 1):
        dx, dy = float(path[i + 1, 0]) - float(path[i, 0]), float(path[i + 1, 1]) - float(path[i, 1])
        l2 = dx * dx + dy * dy
        if not l2 > 0.0:
            continue
        ln = math.sqrt(l2)
        t = min((s - acc) / ln, 1.0)
        x, y = float(path[i, 0]) + t * dx, float(path[i, 1]) + t * dy
        if s <= acc + ln:
            break
        acc = acc + ln
    return x, y


def find(x, y, v, type_id, shapes, ctrl_kind, path_id, paths, zones, priority, half_width, max_range,
         critical_gap=3.0, commit_decel=3.0, v_min=0.5, route_id=None, eps=EPS):
    """K19 on one state.  ``x``, ``y``, ``v``, ``type_id``, ``path_id`` (the current paths), ``route_id`` (or None) [N, M];
    ``ctrl_kind`` [N, M] the kind of each slot's controller row (-1: none); ``shapes`` per type row; ``zones`` a
    ``ConflictZones``; ``priority`` per path.  Returns ``dict(yield_to int16, stop_gap float64 (+inf), stop_x, stop_y,
    robust bool, yielder bool)``, all [N, M]."""
    x, y, v = (np.asarray(np.asarray(a, np.float32), np.float64) for a in (x, y, v))
    type_id, path_id = np.asarray(type_id), np.asarray(path_id)
    N, M = x.shape
    shapes = np.asarray(shapes)
    nt = len(shapes)
    paths = [np.asarray(np.asarray(p, np.float32), np.float64) for p in paths]
    prio = np.zeros(len(paths), np.int64) if priority is None else np.asarray(priority, np.int64)
    hw, rng, cg, vmin = float(half_width), float(max_range), float(critical_gap), float(v_min)
    two_cd = 2.0 * float(commit_decel)
    out = dict(yield_to=np.full((N, M), -1, np.int16), stop_gap=np.full((N, M), np.inf), stop_x=np.zeros((N, M)),
               stop_y=np.zeros((N, M)), robust=np.ones((N, M), bool), yielder=np.zeros((N, M), bool))
    off = zones.zone_off
    near = lambda a, b: abs(a - b) <= eps
    for n in range(N):
        spath = np.full(M, -1)
        s = np.zeros(M)
        cand = np.zeros(M, bool)
        own = np.full(M, -1)
        for m in range(M):
            if not (type_id[n, m] < nt) or math.isnan(x[n, m]) or math.isnan(y[n, m]):
                continue
            p = int(path_id[n, m])
            current = _usable(paths, p)
            if not current:
                p = int(route_id[n, m]) if route_id is not None and _usable(paths, int(route_id[n, m])) else -1
            if p < 0:
                continue
            s[m] = R.closest(paths[p], x[n, m], y[n, m])[5]
            spath[m] = p
            cand[m] = shapes[type_id[n, m]] != SHAPE_NONE
            if current and ctrl_kind[n, m] == IDM:
                own[m] = p
        for i in range(M):
            p = int(own[i])
            if p < 0:
                continue
            out["yielder"][n, i] = True
            si, vi = s[i], v[n, i]
            cd = (vi * vi) / two_cd
            rob = True
            found = None
            for z in range(off[p], off[p + 1]):
                di = zones.s_in_p[z] - si
                rob &= not (near(di, cd) or near(di, rng))
                if not (cd < di and di <= rng):
                    continue
                q = int(zones.q[z])
                who = None
                for j in range(M):
                    if not cand[j] or spath[j] != q:
                        continue
                    sj, vj = s[j], v[n, j]
                    rob &= not near(sj, zones.s_out_q[z])
                    if sj > zones.s_out_q[z]:
                        continue
                    dj = zones.s_in_q[z] - sj
                    cdj = (vj * vj) / two_cd
                    tj = max(dj, 0.0) / max(vj, vmin)
                    rob &= not (near(dj, cdj) or near(tj, cg) or near(dj, di))
                    must = dj <= cdj or (tj <= cg and (prio[q] > prio[p] or (
                        prio[q] == prio[p] and (dj < di or (dj == di and j < i)))))
                    if not must:
                        continue
                    c = R.closest(paths[p], x[n, j], y[n, j])
                    rob &= not (near(c[4], hw) or near(c[5], si))
                    if c[4] <= hw and c[5] > si:
                        continue   # excluded: the leader search follows it
                    who = j
                    break
                if who is not None:
                    found = (z, who, di)
                    break
            out["robust"][n, i] = rob
            if found is not None:
                z, who, di = found
                out["yield_to"][n, i] = who
                out["stop_gap"][n, i] = di
                out["stop_x"][n, i], out["stop_y"][n, i] = point_at(paths[p], zones.s_in_p[z])
    return out


def idm_with_stop(v, x, y, has_lead, vl, xl, yl, row, stop):
    """K5's yielding IDM for one slot: ``stop`` = (x, y) of its stop point or None; np.fmin of the two laws."""
    a = float(OC.idm(v, x, y, has_lead, vl, xl, yl, row))
    if stop is None:
        return a
    return float(np.fmin(a, float(OC.idm(v, x, y, True, 0.0, stop[0], stop[1], row))))
