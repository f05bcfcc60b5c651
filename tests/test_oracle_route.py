"""Route following on the host (DESIGN.md section 1 "Route following"): the float64 restatement (tests/route_oracle.py)
against sympy's exact geometry, OffRoute's argument errors, ReplayEpisodes.ego_routes against the log records, and
bench_route.py's argument parsing without a device."""

import math
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest
import sympy
from sympy import Point2D, Rational, Segment2D

from tactics2d_b200.dataset_parser import LevelXParser, ReplayLog, build_replay_episodes
from tactics2d_b200.traffic.event_detection import OffRoute
from tests import route_oracle as RO
from tests.test_levelx_parser import _write_ind

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _exact(path, x, y):
    """Exact (d^2, closest point, arc length) by sympy over the segments of non-zero length, first strict minimum."""
    P = lambda v: Point2D(Rational(Fraction(float(v[0]))), Rational(Fraction(float(v[1]))))
    p = P((x, y))
    best, acc = None, sympy.Integer(0)
    for a, b in zip(path[:-1], path[1:]):
        A, B = P(a), P(b)
        if A == B:
            continue
        seg = Segment2D(A, B)
        d = B - A
        t = min(max(((p - A).dot(d)) / d.dot(d), 0), 1)
        c = A + d * t
        d2 = (p - c).dot(p - c)
        assert sympy.simplify(d2 - seg.distance(p) ** 2) == 0
        if best is None or d2 < best[0]:
            best = (d2, c, acc + t * seg.length)
        acc = acc + seg.length
    return best, acc


CASES = [
    ([(0, 0), (10, 0), (10, 10)], [(5, 3), (12, -1), (10, 0), (-2, 0), (11, 12), (9.5, 0.5)]),          # vertices, ends
    ([(0, 0), (0, 0), (4, 0), (4, 0), (4, 3)], [(2, 1), (5, 5), (0, 0), (4, 0)]),                      # zero-length segments
    ([(0, 0), (10, 10), (10, 0), (0, 10)], [(5, 5), (5, 4.9), (10, 5), (2.5, 2.5)]),                    # self-crossing
    ([(0, 0), (6, 0), (6, 6), (0, 6), (0, 0)], [(3, 3), (0, 0), (7, 7), (3, 2)]),                        # closed
    ([(0, 0), (4, 0), (4, 4), (0, 4)], [(2, 2), (0.5, 2)]),                                              # equidistant ties
]


@pytest.mark.parametrize("path,points", CASES)
def test_closest_point_and_arc_length_against_sympy(path, points):
    path = np.asarray(path, np.float64)
    for x, y in points:
        (d2, c, s), L = _exact(path, x, y)
        cx, cy, ux, uy, d, s_o, L_o = RO.closest(path, x, y)
        assert math.isclose(d, math.sqrt(float(d2)), rel_tol=1e-12, abs_tol=1e-12), (x, y)
        assert math.isclose(cx, float(c.x), abs_tol=1e-12) and math.isclose(cy, float(c.y), abs_tol=1e-12), (x, y)
        assert math.isclose(s_o, float(s), rel_tol=1e-12, abs_tol=1e-12), (x, y)
        assert math.isclose(L_o, float(L), rel_tol=1e-12), (x, y)


def test_ties_take_the_first_segment():
    # (2, 2) is 2 m from three sides of the open square: the first side (arc length 2) wins
    _, _, _, _, d, s, L = RO.closest([(0, 0), (4, 0), (4, 4), (0, 4)], 2.0, 2.0)
    assert d == 2.0 and s == 2.0 and L == 12.0
    # the shared vertex of two segments belongs to the first
    assert RO.closest([(0, 0), (4, 0), (4, 4)], 5.0, -1.0)[5] == 4.0


def test_probe_threshold_and_no_route():
    path = [(0, 0), (10, 0)]
    assert RO.probe(path, 5.0, 2.0, 2.0) == (1, 5.0)          # d == threshold is on route (d > threshold is off)
    assert RO.probe(path, 5.0, 2.5, 2.0)[0] == 2
    assert RO.probe([(1, 1), (1, 1)], 5.0, 2.0, 2.0) == (0, 0.0)
    assert RO.probe(None, 5.0, 2.0, 2.0) == (0, 0.0)
    assert RO.progress(3.0, -np.inf, 0.1) == (0.0, 3.0)       # the first step only records s
    assert RO.progress(2.0, 3.0, 0.1) == (0.0, 3.0)
    assert RO.progress(5.0, 3.0, 0.1) == (float(np.float32(0.1 * 2.0)), 5.0)


def test_observe_row_points_and_frame():
    path = [(0, 0), (10, 0), (10, 10)]
    row = RO.observe_row(path, 2.0, 1.0, 0.0, 4, 5.0)
    assert row[0] == 1.0 and row[1] == -1.0 and row[2] == 0.0          # the route lies 1 m to the right
    assert row[3] == 2.0 / 20.0 and row[4] == 18.0
    pts = row[RO.FIELDS:].reshape(-1, 2)
    assert np.allclose(pts, [(5.0, -1.0), (8.0, 1.0), (8.0, 6.0), (8.0, 9.0)])   # 7, 12, 17, min(22, 20) m
    assert not RO.observe_row(None, 0, 0, 0, 2, 1.0).any() and len(RO.observe_row(None, 0, 0, 0, 2, 1.0)) == 9
    # heading error wraps into (-pi, pi]
    assert RO.observe_row([(0, 0), (-1, 0)], 0.0, 0.0, 0.0, 0, 1.0)[2] == math.pi


def test_off_route_argument_errors():
    d = OffRoute(1.0)
    with pytest.raises(ValueError):
        d.update((0.0, 0.0))                                    # before reset (off_route.py:30-31)
    for bad in (5, "route", [(0, 0)], [[0, 0, 0], [1, 1, 1]], object()):
        with pytest.raises(TypeError):
            d.reset(bad)
    d.reset([(0, 0), (1, 0)])
    assert d.route.shape == (2, 2)

    class Line:
        coords = [(0.0, 0.0), (3.0, 4.0), (3.0, 8.0)]

    d.reset(Line())
    assert d.route.shape == (3, 2)


def test_ego_routes_follow_the_logged_track(tmp_path):
    _write_ind(tmp_path)   # tracks: 0 car 0..360 ms, 1 bus 80..360, 2 bicycle 0..200, 3 pedestrian 160..360
    log = ReplayLog.from_levelx(LevelXParser("inD"), 3, str(tmp_path))
    ep = build_replay_episodes(log, 3, [0, 200, 360], [0, 1, 0])
    paths, rid = ep.ego_routes()
    assert rid.dtype == np.int16 and rid.shape == (3, 3)
    assert (rid[:, 0] == [0, 1, 2]).all() and (rid[:, 1:] == -1).all()
    for p, (t0, tid) in enumerate(zip([0, 200, 360], [0, 1, 0])):
        k = log.index(tid)
        want = [log.record(k, t)[:2] for t in range(t0, int(log.last_ms[k]) + 1, 40)]
        if len(want) == 1:
            want = want * 2                                     # one frame left: a repeated point, no route
        assert np.array_equal(paths[p], np.asarray(want, np.float32)), p
    # the ego starts on its route, at arc length 0
    assert RO.closest(paths[0], ep.pool["x"][0, 0], ep.pool["y"][0, 0])[4:6] == (0.0, 0.0)
    short, _ = ep.ego_routes(horizon_ms=80)
    assert [len(q) for q in short] == [3, 3, 2]
    assert np.array_equal(short[0], paths[0][:3])
    sched = build_replay_episodes(log, 3, [0], [0], reuse_slots=True)
    assert np.array_equal(sched.ego_routes()[0][0], paths[0])


def test_bench_route_help_without_a_device():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench_route.py"), "--help"], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "usage:" in r.stdout
