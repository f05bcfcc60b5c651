"""Float64 restatement of DESIGN.md section 1 "Leader search" (TEST INFRASTRUCTURE ONLY): the leader of every slot (K17,
``t2d_find_leaders``) and whether that choice is robust to the last bits of the arithmetic.

The path frame projects with ``tests.route_oracle.closest`` (the closest point and arc length K5's PATH sources and the
route code use); the heading frame takes ``math.cos`` / ``math.sin`` of the follower's fp32 heading, the only
trigonometry.  Python floats and NumPy float64 arrays: one rounding per operation, in the kernel's order."""

from __future__ import annotations

import math

import numpy as np

from tests import route_oracle as R

SHAPE_NONE = 2
EPS = 1e-9       # a candidate within this of a bound, or a runner-up within this of the best gap: the choice is not robust
HEADING, PATH = 1, 2


def usable(paths, pid):
    """The path a follower with controller path ``pid`` is projected on, or None (heading frame)."""
    if paths is None or not 0 <= pid < len(paths):
        return None
    p = np.asarray(paths[pid], np.float64)
    return p if R.closest(p, 0.0, 0.0) is not None else None


def find(x, y, heading, type_id, shapes, half_width, max_range, path_id=None, paths=None, eps=EPS):
    """Leaders of every slot.  ``x``, ``y``, ``heading``, ``type_id`` [N, M] (positions as the fp32 state holds them);
    ``shapes``: the shape id of every type row (n_types = len(shapes)); ``path_id`` [N, M] the controllers' paths and
    ``paths`` the polyline table, or None.  Returns ``dict(lead int16 [N, M], gap float64 [N, M] (+inf: none),
    robust bool [N, M], frame int [N, M] (0: no follower, HEADING, PATH))``."""
    x, y, h = (np.asarray(np.asarray(a, np.float32), np.float64) for a in (x, y, heading))
    type_id = np.asarray(type_id)
    N, M = x.shape
    shapes = np.asarray(shapes)
    nt = len(shapes)
    hw, rng = float(half_width), float(max_range)
    lead = np.full((N, M), -1, np.int16)
    gap = np.full((N, M), np.inf)
    robust = np.ones((N, M), bool)
    frame = np.zeros((N, M), np.int64)
    for n in range(N):
        active = type_id[n] < nt
        finite = ~(np.isnan(x[n]) | np.isnan(y[n]))
        cand = active & finite & (shapes[np.where(active, type_id[n], 0)] != SHAPE_NONE)
        proj = {}
        for i in range(M):
            if not (active[i] and finite[i]):
                continue
            others = cand.copy()
            others[i] = False
            js = np.nonzero(others)[0]
            path = None if path_id is None else usable(paths, int(path_id[n, i]))
            if path is None:
                frame[n, i] = HEADING
                c, s = math.cos(h[n, i]), math.sin(h[n, i])
                dx, dy = x[n, js] - x[n, i], y[n, js] - y[n, i]
                ex = c * dx + s * dy
                ey = -s * dx + c * dy
                ok = (ex > 0.0) & (np.abs(ey) <= hw) & (ex <= rng)
                g = ex
                near = (np.abs(ex) <= eps) | (np.abs(np.abs(ey) - hw) <= eps) | (np.abs(ex - rng) <= eps)
            else:
                frame[n, i] = PATH
                pid = int(path_id[n, i])
                if pid not in proj:   # (s, d) of every candidate and of slot i on this path
                    proj[pid] = {k: R.closest(path, x[n, k], y[n, k]) for k in range(M) if active[k] and finite[k]}
                si = proj[pid][i][5]
                d = np.array([proj[pid][j][4] for j in js])
                g = np.array([proj[pid][j][5] - si for j in js])
                ok = (d <= hw) & (g > 0.0) & (g <= rng)
                near = (np.abs(d - hw) <= eps) | (np.abs(g) <= eps) | (np.abs(g - rng) <= eps)
            if js.size and near.any():
                robust[n, i] = False
            if not ok.any():
                continue
            order = np.lexsort((js[ok], g[ok]))   # smallest (gap, slot)
            lead[n, i] = js[ok][order[0]]
            gap[n, i] = g[ok][order[0]]
            if ok.sum() > 1 and g[ok][order[1]] - g[ok][order[0]] <= eps:
                robust[n, i] = False
    return dict(lead=lead, gap=gap, robust=robust, frame=frame)
