"""Conflict zones between the polylines of a ``set_paths`` table (DESIGN.md section 1 "Yielding at conflict zones").

A zone on path p for path q is a maximal closed arc interval ``[a_p, b_p]`` of p whose points lie within ``width`` of q,
paired with ``[a_q, b_q]``, the hull of the arc lengths of q within ``width`` of that piece of p.  The table is built once,
on the host, from the exact vertex values ``set_paths`` uploads (the fp32 vertices promoted to fp64), with the arc
lengths of K17's closest point (segments of non-zero length only, ``sqrt(dx * dx + dy * dy)`` summed in list order).

Every segment pair is settled in closed form: the points of segment A within ``width`` of segment B are the chord of A's
line through the capsule of B (a rectangle and two discs, a convex set), clipped to A.  The pairs are enumerated on a
sweep over the segments' boxes, so the build stays linear in the number of segment pairs whose boxes overlap.
"""

from __future__ import annotations

from dataclasses import dataclass

import numpy as np


@dataclass
class ConflictZones:
    """The zones of every path, in CSR order by path and sorted by ``(p, s_in_p, q)`` within it.  ``zone_off``
    [n_paths + 1] int32; ``p``, ``q`` [Z] int32; ``s_in_p``, ``s_out_p``, ``s_in_q``, ``s_out_q`` [Z] fp64, the zone's
    arc intervals widened by ``margin`` at both ends."""
    zone_off: np.ndarray
    p: np.ndarray
    q: np.ndarray
    s_in_p: np.ndarray
    s_out_p: np.ndarray
    s_in_q: np.ndarray
    s_out_q: np.ndarray

    def __len__(self):
        return int(self.q.shape[0])


def _segments(paths):
    """The segments of non-zero length of every path: (path, x0, y0, dx, dy, len, cum) as flat arrays."""
    cols = [[] for _ in range(7)]
    for k, poly in enumerate(paths):
        v = np.asarray(np.asarray(poly, np.float32).reshape(-1, 2), np.float64)
        dx, dy = v[1:, 0] - v[:-1, 0], v[1:, 1] - v[:-1, 1]
        l2 = dx * dx + dy * dy
        keep = l2 > 0.0
        if not keep.any():
            continue   # a degenerate path: PathTable::usable fails, nothing is projected on it
        ln = np.sqrt(l2[keep])
        cum = np.zeros(ln.shape[0])
        acc = 0.0
        for i in range(ln.shape[0]):   # the running sum in list order, as closest_on_path accumulates it
            cum[i] = acc
            acc = acc + ln[i]
        for c, a in zip(cols, (np.full(ln.shape[0], k), v[:-1, 0][keep], v[:-1, 1][keep], dx[keep], dy[keep], ln, cum)):
            c.append(a)
    if not cols[0]:
        return [np.zeros(0, np.int64)] + [np.zeros(0) for _ in range(6)]
    return [np.concatenate(c) for c in cols]


def _slab(alpha, beta, lo, hi):
    """The t interval where alpha + beta t lies in [lo, hi] (possibly empty: t0 > t1)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        t0 = (lo - alpha) / beta
        t1 = (hi - alpha) / beta
    a, b = np.minimum(t0, t1), np.maximum(t0, t1)
    flat = beta == 0.0
    inside = (alpha >= lo) & (alpha <= hi)
    a = np.where(flat, np.where(inside, -np.inf, np.inf), a)
    b = np.where(flat, np.where(inside, np.inf, -np.inf), b)
    return a, b


def _disc(ox, oy, dx, dy, cx, cy, w):
    """The t interval where |o + t d - c| <= w (empty: t0 > t1)."""
    ex, ey = ox - cx, oy - cy
    A = dx * dx + dy * dy
    B = ex * dx + ey * dy
    C = ex * ex + ey * ey - w * w
    disc = B * B - A * C
    r = np.sqrt(np.maximum(disc, 0.0))
    t0, t1 = (-B - r) / A, (-B + r) / A
    empty = disc < 0.0
    return np.where(empty, np.inf, t0), np.where(empty, -np.inf, t1)


def _near(ax, ay, adx, ady, bx, by, bdx, bdy, blen, w):
    """For every pair, the parameter interval [t0, t1] of segment A (o + t d, t in [0, 1]) within w of segment B;
    t0 > t1 when there is none."""
    ux, uy = bdx / blen, bdy / blen
    rx, ry = ax - bx, ay - by
    a0, b0 = _slab(rx * ux + ry * uy, adx * ux + ady * uy, 0.0, blen)       # along B
    a1, b1 = _slab(-rx * uy + ry * ux, -adx * uy + ady * ux, -w, w)         # across B
    lo, hi = np.maximum(a0, a1), np.minimum(b0, b1)
    for cx, cy in ((bx, by), (bx + bdx, by + bdy)):
        d0, d1 = _disc(ax, ay, adx, ady, cx, cy, w)
        some = d0 <= d1
        none = lo > hi
        lo = np.where(some, np.where(none, d0, np.minimum(lo, d0)), lo)
        hi = np.where(some, np.where(none, d1, np.maximum(hi, d1)), hi)
    return np.maximum(lo, 0.0), np.minimum(hi, 1.0)


def _close_pairs(P, x0, y0, dx, dy, w):
    """Index pairs of segments of different paths whose boxes, grown by w, overlap: a sweep along the longer side of
    the scene, each box paired with the boxes that start inside its extent there, then the test on the other axis."""
    n = P.shape[0]
    xl, xh = np.minimum(x0, x0 + dx) - w, np.maximum(x0, x0 + dx) + w
    yl, yh = np.minimum(y0, y0 + dy) - w, np.maximum(y0, y0 + dy) + w
    if n and np.ptp(yl) > np.ptp(xl):
        xl, xh, yl, yh = yl, yh, xl, xh
    order = np.argsort(xl, kind="stable")
    start = xl[order]
    cnt = np.searchsorted(start, xh[order], side="right") - np.arange(n) - 1   # the boxes after it that start in it
    cnt = np.maximum(cnt, 0)
    a = np.repeat(np.arange(n), cnt)
    b = a + 1 + (np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt))
    left, right = order[a], order[b]
    keep = (P[left] != P[right]) & (yl[left] <= yh[right]) & (yl[right] <= yh[left])
    return left[keep], right[keep]


def _cummax_by_group(group, v):
    """Running maximum of v restarting at every group (group sorted ascending), exact: on the ranks of v."""
    if not v.size:
        return v
    values, rank = np.unique(v, return_inverse=True)
    stride = np.int64(values.shape[0])
    base = group.astype(np.int64) * stride
    return values[np.maximum.accumulate(base + rank.astype(np.int64)) - base]


def conflict_zones(paths, width: float = 2.0, margin: float = 3.0) -> ConflictZones:
    """The conflict zones of the polylines ``paths`` (a ``set_paths`` table) for cars ``width`` metres apart, each widened
    by ``margin`` metres at both ends.  Zones that begin at the start of both paths (``a_p == a_q == 0``: cars that start
    on the same lane, which the leader search already orders) are dropped, and so are degenerate paths."""
    width, margin = float(width), float(margin)
    if not (np.isfinite(width) and width > 0.0):
        raise ValueError("width must be finite and > 0")
    if not (np.isfinite(margin) and margin >= 0.0):
        raise ValueError("margin must be finite and >= 0")
    n_paths = len(paths)
    P, x0, y0, dx, dy, ln, cum = _segments(paths)
    i, j = _close_pairs(P, x0, y0, dx, dy, width)
    ti0, ti1 = _near(x0[i], y0[i], dx[i], dy[i], x0[j], y0[j], dx[j], dy[j], ln[j], width)   # on segment i, near j
    tj0, tj1 = _near(x0[j], y0[j], dx[j], dy[j], x0[i], y0[i], dx[i], dy[i], ln[i], width)   # on segment j, near i
    ok = (ti0 <= ti1) & (tj0 <= tj1)
    i, j, ti0, ti1, tj0, tj1 = i[ok], j[ok], ti0[ok], ti1[ok], tj0[ok], tj1[ok]
    ai0, ai1 = cum[i] + ti0 * ln[i], cum[i] + ti1 * ln[i]
    aj0, aj1 = cum[j] + tj0 * ln[j], cum[j] + tj1 * ln[j]
    # both directions: (p, q, interval on p, interval on q)
    p = np.r_[P[i], P[j]].astype(np.int64)
    q = np.r_[P[j], P[i]].astype(np.int64)
    lo_p, hi_p = np.r_[ai0, aj0], np.r_[ai1, aj1]
    lo_q, hi_q = np.r_[aj0, ai0], np.r_[aj1, ai1]
    pair = p * max(n_paths, 1) + q
    order = np.lexsort((lo_p, pair))
    pair, p, q, lo_p, hi_p, lo_q, hi_q = (a[order] for a in (pair, p, q, lo_p, hi_p, lo_q, hi_q))
    grp = np.r_[0, np.cumsum(pair[1:] != pair[:-1])] if pair.size else pair
    reach = _cummax_by_group(grp, hi_p)          # the furthest end of the intervals so far in this (p, q) pair
    new = np.r_[True, (grp[1:] != grp[:-1]) | (lo_p[1:] > reach[:-1])] if pair.size else np.zeros(0, bool)
    start = np.flatnonzero(new)
    zp, zq = p[start], q[start]
    a_p = lo_p[start]
    b_p = np.maximum.reduceat(hi_p, start) if start.size else hi_p[:0]
    a_q = np.minimum.reduceat(lo_q, start) if start.size else lo_q[:0]
    b_q = np.maximum.reduceat(hi_q, start) if start.size else hi_q[:0]
    keep = ~((a_p == 0.0) & (a_q == 0.0))
    zp, zq, a_p, b_p, a_q, b_q = zp[keep], zq[keep], a_p[keep], b_p[keep], a_q[keep], b_q[keep]
    s_in_p = a_p - margin
    order = np.lexsort((zq, s_in_p, zp))
    zp, zq, a_p, b_p, a_q, b_q, s_in_p = (a[order] for a in (zp, zq, a_p, b_p, a_q, b_q, s_in_p))
    off = np.zeros(n_paths + 1, np.int32)
    off[1:] = np.cumsum(np.bincount(zp, minlength=n_paths)) if n_paths else off[1:]
    return ConflictZones(zone_off=off, p=zp.astype(np.int32), q=zq.astype(np.int32), s_in_p=s_in_p,
                         s_out_p=b_p + margin, s_in_q=a_q - margin, s_out_q=b_q + margin)
