"""The float64 restatement of PIDController (tests/pid_oracle.py: pid_step) against the unmodified reference's sequences,
and its path-derived lateral error against sympy's exact segment geometry."""

import numpy as np
import pytest
import sympy
from sympy.geometry import Line2D, Point2D, Segment2D

from . import pid_oracle as OC
from .pid_cases import CONFIGS, quirk, row_dict, sequence


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c["name"] for c in CONFIGS])
def test_oracle_equals_reference_sequences(cfg):
    p = row_dict(cfg)
    inp, want_out, want_state = sequence(cfg)
    st = np.zeros(6)
    for t in range(len(inp)):
        x, y, h, v, ts, lt = inp[t]
        steer, acc, st = OC.pid_step(p, x, y, h, v, ts, lt, st)
        if quirk(cfg):
            steer = 0.0
        np.testing.assert_allclose(st, want_state[t], rtol=1e-13, atol=0)
        np.testing.assert_allclose([steer, acc], want_out[t], rtol=1e-12, atol=1e-12)


def test_sequences_cover_the_issue_cases():
    names = {c["name"] for c in CONFIGS}
    assert {"default", "gains", "lateral_heading", "longitudinal", "saturation", "no_lateral", "no_longitudinal",
            "wheel_base_quirk", "style_conservative", "style_0_3", "style_aggressive"} <= names
    inp, out, st = sequence(next(c for c in CONFIGS if c["name"] == "saturation"))
    assert (out[:, 1] == 3.0).any() and (out[:, 1] == -5.0).any()        # both limits reached
    wrap = sequence(next(c for c in CONFIGS if c["name"] == "wrap"))[0]
    assert (np.abs(wrap[:, 5] - wrap[:, 2]) > np.pi).all()               # every heading error beyond +-pi
    assert (sequence(next(c for c in CONFIGS if c["name"] == "wheel_base_quirk"))[1][:, 0] == 0.0).all()


def _sympy_closest(path, x, y):
    """Distance and closest point by exact rational geometry: the first segment (in order) at the least distance."""
    p = Point2D(sympy.Rational(x), sympy.Rational(y))
    best = None
    for a, b in zip(path[:-1], path[1:]):
        if a[0] == b[0] and a[1] == b[1]:
            continue
        seg = Segment2D(Point2D(sympy.Rational(a[0]), sympy.Rational(a[1])), Point2D(sympy.Rational(b[0]), sympy.Rational(b[1])))
        d = seg.distance(p)
        if best is None or d < best[0]:
            proj = seg.projection(p) if seg.contains(seg.projection(p)) else min(seg.points, key=lambda q: q.distance(p))
            best = (d, proj, seg)
    return best


PATHS = [
    np.array([[0.0, 0.0], [10.0, 0.0], [10.0, 10.0], [0.0, 10.0]]),
    np.array([[-5.0, 2.0], [-5.0, 2.0], [3.0, -4.0], [3.0, -4.0], [12.0, 5.5]]),       # zero-length segments
    np.array([[1.5, 1.5], [4.25, 7.75]]),
]
POINTS = [(5.0, -3.0), (12.0, -2.0), (-3.0, -1.0), (10.0, 0.0), (12.5, 12.0), (5.0, 5.0), (8.0, 3.0), (-9.0, 6.5),
          (20.0, 9.0), (0.5, 0.25), (3.0, 7.0), (-1.0, 12.0)]


@pytest.mark.parametrize("k", range(len(PATHS)))
def test_path_closest_point_matches_sympy(k):
    """Closest point and |cross-track| equal sympy's Segment.distance, including clamps beyond both ends of the path
    and ties at shared vertices; the sign is positive when the path lies to the left of its direction."""
    path = PATHS[k]
    for x, y in POINTS:
        cx, cy, ux, uy = OC.path_closest(path, x, y)
        d, proj, seg = _sympy_closest(path, x, y)
        assert np.hypot(cx - x, cy - y) == pytest.approx(float(d), rel=1e-12, abs=1e-12)
        assert (cx, cy) == pytest.approx((float(proj.x), float(proj.y)), rel=1e-12, abs=1e-12)
        e = OC.path_lateral_error(path, x, y, 0.0, True)
        # the offset across the closest segment: the distance itself where the projection falls inside it, the
        # perpendicular part of it where it is clamped to an end of the path
        assert abs(e) == pytest.approx(float(Line2D(seg.p1, seg.p2).distance(Point2D(sympy.Rational(x), sympy.Rational(y)))),
                                       rel=1e-12, abs=1e-12)
        if seg.contains(seg.projection(Point2D(sympy.Rational(x), sympy.Rational(y)))):
            assert abs(e) == pytest.approx(float(d), rel=1e-12, abs=1e-12)
        side = float((seg.p2.x - seg.p1.x) * (y - seg.p1.y) - (seg.p2.y - seg.p1.y) * (x - seg.p1.x))
        assert side == 0.0 or np.sign(e) == -np.sign(side)     # point right of the path <=> path to its left <=> e > 0


def test_path_tie_at_a_shared_vertex_takes_the_first_segment():
    path = PATHS[0]
    cx, cy, ux, uy = OC.path_closest(path, 12.0, -2.0)       # beyond the corner (10, 0): both segments clamp to it
    assert (cx, cy, ux, uy) == (10.0, 0.0, 1.0, 0.0)
    assert OC.path_lateral_error(path, 12.0, -2.0, 0.0, False) == 0.0   # heading along the first segment
    assert OC.path_closest(np.array([[1.0, 1.0], [1.0, 1.0]]), 0.0, 0.0) is None
