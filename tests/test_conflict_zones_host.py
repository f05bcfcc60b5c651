"""``tactics2d_b200.traffic.conflicts.conflict_zones`` against brute-force sampling (CPU only).

The reference intervals come from sampling: every path at 1e-2 m to find where it is within ``width`` of the other, then
1e-4 m sampling in a 4e-2 m window around each transition, so every bound is known to 1e-4 m.  The partner interval is
sampled the same way against the piece of p between its bounds."""

import math
import time

import numpy as np
import pytest

from tactics2d_b200 import synthetic as S
from tactics2d_b200.traffic.conflicts import conflict_zones

W, MARGIN, TOL = 2.0, 3.0, 2e-4


def _poly(path):
    p = np.asarray(np.asarray(path, np.float32), np.float64)
    d = np.diff(p, axis=0)
    ln = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1])
    keep = ln > 0.0
    return p[:-1][keep], d[keep], ln[keep], np.r_[0.0, np.cumsum(ln[keep])]


def _at(poly, s):
    a, d, ln, cum = poly
    k = np.clip(np.searchsorted(cum, s, side="right") - 1, 0, len(ln) - 1)
    t = (s - cum[k]) / ln[k]
    return a[k] + t[:, None] * d[k]


def _dist(pts, poly):
    a, d, ln, _ = poly
    best = np.full(len(pts), np.inf)
    for k in range(len(ln)):
        t = np.clip(((pts[:, 0] - a[k, 0]) * d[k, 0] + (pts[:, 1] - a[k, 1]) * d[k, 1]) / (ln[k] * ln[k]), 0.0, 1.0)
        e = pts - (a[k] + t[:, None] * d[k])
        best = np.minimum(best, np.hypot(e[:, 0], e[:, 1]))
    return best


def _sub(poly, lo, hi):
    """The piece of a polyline between arc lengths lo and hi, as a polyline."""
    a, d, ln, cum = poly
    inner = [a[k] for k in range(len(ln)) if lo < cum[k] < hi]
    pts = np.array([_at(poly, np.array([lo]))[0]] + inner + [_at(poly, np.array([hi]))[0]])
    if hi - lo < 1e-12:
        pts = np.array([pts[0], pts[0] + 1e-12])
    return _poly(pts)


def _intervals(poly, other, w):
    """The maximal arc intervals of ``poly`` within w of the polyline ``other``, each bound to 1e-4 m."""
    L = poly[3][-1]
    s = np.r_[np.arange(0.0, L, 1e-2), L]
    inside = _dist(_at(poly, s), other) <= w
    out = []
    edges = np.flatnonzero(np.diff(inside.astype(np.int8)))

    def refine(k, rising):
        f = np.r_[np.arange(s[k], s[k + 1], 1e-4), s[k + 1]]
        ins = _dist(_at(poly, f), other) <= w
        idx = np.flatnonzero(ins)
        return f[idx[0]] if rising else f[idx[-1]]

    lo = 0.0 if inside[0] else None
    for k in edges:
        if not inside[k]:
            lo = refine(k, True)
        else:
            out.append((lo, refine(k, False)))
            lo = None
    if lo is not None:
        out.append((lo, L))
    return out


def _brute(paths, w):
    """Rows (p, q, a_p, b_p, a_q, b_q) by sampling, with the drop rule."""
    polys = [_poly(p) for p in paths]
    rows = []
    for p, pp in enumerate(polys):
        if not len(pp[2]):
            continue
        for q, qq in enumerate(polys):
            if q == p or not len(qq[2]):
                continue
            for a_p, b_p in _intervals(pp, qq, w):
                part = _intervals(qq, _sub(pp, a_p, b_p), w)
                a_q, b_q = min(r[0] for r in part), max(r[1] for r in part)
                if a_p == 0.0 and a_q == 0.0:
                    continue
                rows.append((p, q, a_p, b_p, a_q, b_q))
    return rows


def _table(z):
    return [(int(z.p[k]), int(z.q[k]), z.s_in_p[k] + MARGIN, z.s_out_p[k] - MARGIN, z.s_in_q[k] + MARGIN,
             z.s_out_q[k] - MARGIN) for k in range(len(z))]


def _line(x0, y0, x1, y1):
    return np.array([[x0, y0], [x1, y1]], np.float32)


def _rotated(deg, length=60.0):
    a = math.radians(deg)
    return np.array([[-length * math.cos(a), -length * math.sin(a)], [length * math.cos(a), length * math.sin(a)]],
                    np.float32)


SCENES = {
    "perpendicular": [_line(-50.0, 0.0, 50.0, 0.0), _line(0.0, -50.0, 0.0, 50.0)],
    "crossing_30deg": [_line(-60.0, 0.0, 60.0, 0.0), _rotated(30.0)],
    "merge": S.t_junction(1, 2).paths,
    "roundabout": S.roundabout(1, 2).paths,
    "parallel_inside": [_line(0.0, 0.0, 100.0, 0.0), _line(50.0, W - 1e-6, 150.0, W - 1e-6)],
    "parallel_outside": [_line(0.0, 0.0, 100.0, 0.0), _line(50.0, W + 1e-6, 150.0, W + 1e-6)],
    "identical": [_line(-50.0, 1.0, 50.0, 1.0), _line(-50.0, 1.0, 50.0, 1.0), _line(0.0, -50.0, 0.0, 50.0)],
    "zero_length_segments": [np.array([[-50.0, 0.0], [-50.0, 0.0], [0.0, 0.0], [0.0, 0.0], [50.0, 0.0]], np.float32),
                             np.array([[3.0, -50.0], [3.0, 10.0], [3.0, 10.0], [3.0, 50.0]], np.float32),
                             np.array([[1.0, 1.0], [1.0, 1.0]], np.float32)],
}


@pytest.mark.parametrize("name", sorted(SCENES))
def test_zones_match_sampling(name):
    paths = SCENES[name]
    z = conflict_zones(paths, W, MARGIN)
    got, ref = _table(z), _brute(paths, W)
    assert len(got) == len(ref), (got, ref)
    for g in got:   # same (p, q) rows, bounds to the sampling's resolution
        m = [r for r in ref if r[:2] == g[:2] and all(abs(a - b) <= TOL for a, b in zip(g[2:], r[2:]))]
        assert len(m) == 1, (g, [r for r in ref if r[:2] == g[:2]])
    # CSR by path, sorted by s_in_p
    assert z.zone_off[0] == 0 and z.zone_off[-1] == len(z) and np.all(np.diff(z.zone_off) >= 0)
    for p in range(len(paths)):
        rows = slice(z.zone_off[p], z.zone_off[p + 1])
        assert np.all(z.p[rows] == p) and np.all(np.diff(z.s_in_p[rows]) >= 0.0)
    if name == "parallel_outside":
        assert len(z) == 0
    if name == "parallel_inside":
        assert len(z) == 2
    if name == "identical":   # the two identical lanes start together: only their crossings with path 2 are left
        assert set(zip(z.p.tolist(), z.q.tolist())) == {(0, 2), (2, 0), (1, 2), (2, 1)}
    if name == "zero_length_segments":
        assert 2 not in z.p and 2 not in z.q
        assert len(z) == 2


@pytest.mark.parametrize("name", sorted(SCENES))
def test_partner_side_is_the_matching_rows_own_side(name):
    z = conflict_zones(SCENES[name], W, MARGIN)
    rows = {(int(z.p[k]), int(z.q[k]), z.s_in_p[k], z.s_out_p[k]) for k in range(len(z))}
    for k in range(len(z)):
        assert (int(z.q[k]), int(z.p[k]), z.s_in_q[k], z.s_out_q[k]) in rows


def test_arguments_are_checked():
    with pytest.raises(ValueError):
        conflict_zones(SCENES["perpendicular"], width=0.0)
    with pytest.raises(ValueError):
        conflict_zones(SCENES["perpendicular"], margin=-1.0)
    z = conflict_zones([])
    assert len(z) == 0 and z.zone_off.tolist() == [0]


def test_build_time_for_1000_track_paths():
    """About 1000 reactive-replay track paths: a 9-minute highway log (no zone: its lanes never cross and same-lane
    paths start together, or follow each other) and a 27-minute two-stream crossing log (every crossing pair is a zone)."""
    hw = S.highway_log(duration_ms=540_000).track_paths(0.1, 30.0)[0]
    cx = S.crossing_log(duration_ms=1_600_000, rate_per_s=0.3).track_paths(0.1, 30.0)[0]
    for name, paths in (("highway", hw), ("crossing", cx)):
        conflict_zones(paths)
        t = time.perf_counter()
        z = conflict_zones(paths)
        dt = time.perf_counter() - t
        print(f"conflict_zones: {len(paths)} {name} track paths -> {len(z)} zones in {dt:.3f} s")
    assert len(conflict_zones(hw)) == 0
