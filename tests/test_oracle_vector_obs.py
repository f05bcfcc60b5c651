"""The float64 vector-observation oracle (tests/vector_obs_oracle.py) on known answers, and its selection against exact
rational arithmetic.  No GPU needed."""

from fractions import Fraction

import numpy as np

from tests import vector_obs_oracle as V

BOX = dict(shape=V.SHAPE_OBB, half_len=2.5, half_wid=1.0, radius=0.0)
DISC = dict(shape=V.SHAPE_CIRCLE, half_len=0.3, half_wid=0.3, radius=0.3)
NONE = dict(shape=V.SHAPE_NONE, half_len=1.0, half_wid=1.0, radius=0.0)
TABLE = [BOX, DISC, NONE]


def _state(xy, heading=None, types=None):
    """One scenario: the ego (slot 0) at the origin, then the given points."""
    xy = np.asarray([(0.0, 0.0)] + list(xy), np.float32)
    m = len(xy)
    h = np.zeros((1, m), np.float32) if heading is None else np.asarray(heading, np.float32).reshape(1, m)
    st = dict(x=xy[None, :, 0], y=xy[None, :, 1], heading=h, speed=np.zeros((1, m), np.float32),
              vx=np.zeros((1, m), np.float32), vy=np.zeros((1, m), np.float32))
    t = np.zeros((1, m), np.uint8) if types is None else np.asarray(types, np.uint8).reshape(1, m)
    return st, t


def _obs(st, t, k=4, s=0, ra=50.0, rs=30.0, **kw):
    flat, ai, si = V.observe(st, t, TABLE, k, s, ra, rs, **kw)
    ego, goal, agents, segs = V.split(flat, k, s)
    return ego[0], goal[0], agents[0], segs[0], ai[0], si[0]


def test_agent_at_3_4_has_dist_5():
    _, _, ag, _, ai, _ = _obs(*_state([(3.0, 4.0)]))
    assert ag[0, 10] == 5.0 and ag[0, 0] == 1.0 and (ag[0, 1], ag[0, 2]) == (3.0, 4.0)
    assert list(ai) == [1, -1, -1, -1]


def test_heading_half_pi_rotates_x_axis_to_minus_y():
    st, t = _state([(1.0, 0.0)], heading=[np.pi / 2, 0.0])
    _, _, ag, _, _, _ = _obs(st, t)
    assert abs(ag[0, 1]) < 1e-7 and ag[0, 2] == -1.0
    # the heading difference of an agent facing world +x, seen from an ego facing +y: -pi/2
    assert abs(ag[0, 3]) < 1e-7 and ag[0, 4] == -1.0


def test_equal_distances_come_in_slot_order():
    _, _, ag, _, ai, _ = _obs(*_state([(0.0, 1.0), (1.0, 0.0), (-1.0, 0.0), (0.0, -1.0), (0.0, 0.5)]), k=5)
    assert list(ai) == [5, 1, 2, 3, 4]
    assert list(ag[:, 10]) == [0.5, 1.0, 1.0, 1.0, 1.0]


def test_distance_equal_to_range_is_kept():
    st, t = _state([(3.0, 4.0)])
    assert list(_obs(st, t, ra=5.0)[4]) == [1, -1, -1, -1]
    below = float(np.nextafter(np.float32(5.0), np.float32(0.0)))
    assert list(_obs(st, t, ra=below)[4]) == [-1, -1, -1, -1]


def test_shape_none_empty_and_nan_slots_are_excluded():
    st, t = _state([(1.0, 0.0), (2.0, 0.0), (3.0, 0.0), (4.0, 0.0)], types=[0, 2, 255, 0, 1])
    st["x"][0, 3] = np.nan
    _, _, ag, _, ai, _ = _obs(st, t)
    assert list(ai) == [4, -1, -1, -1]   # slot 1 SHAPE_NONE, slot 2 empty, slot 3 NaN
    assert ag[0, 9] == 1.0 and (ag[0, 7], ag[0, 8]) == (np.float32(0.3), np.float32(0.3))


def _seg_obs(segs, poly_start=None, s=4, rs=30.0):
    st, t = _state([])
    tiles = [dict(segments=np.asarray(segs, np.float32), poly_start=poly_start)]
    return _obs(st, t, k=0, s=s, rs=rs, tiles=tiles)


def test_closest_point_endpoint_and_interior():
    _, _, _, sg, _, si = _seg_obs([(2.0, 1.0, 5.0, 1.0), (-2.0, 1.0, 3.0, 1.0)])
    assert list(si) == [1, 0, -1, -1]
    assert (sg[0, 5], sg[0, 6], sg[0, 7]) == (0.0, 1.0, 1.0)                       # interior projection (0, 1)
    assert (sg[1, 5], sg[1, 6], sg[1, 7]) == (2.0, 1.0, np.float32(np.sqrt(5.0)))  # endpoint (2, 1)
    assert tuple(sg[1, 1:5]) == (2.0, 1.0, 5.0, 1.0)


def test_zero_length_segment_has_t_zero():
    _, _, _, sg, _, si = _seg_obs([(1.0, 2.0, 1.0, 2.0)])
    assert si[0] == 0 and (sg[0, 5], sg[0, 6]) == (1.0, 2.0) and sg[0, 7] == np.float32(np.sqrt(5.0))


def test_ring_segments_flagged():
    ring = [(1.0, 1.0, 2.0, 1.0), (2.0, 1.0, 2.0, 2.0), (2.0, 2.0, 1.0, 1.0)]
    _, _, _, sg, _, si = _seg_obs(ring + [(0.0, 3.0, 1.0, 3.0)], poly_start=np.asarray([0, 3], np.int32))
    assert list(si) == [0, 2, 1, 3]
    assert list(sg[:, 8]) == [1.0, 1.0, 1.0, 0.0]


def test_empty_ego_row_is_all_zeros():
    st, t = _state([(1.0, 0.0)], types=[255, 0])
    flat, ai, si = V.observe(st, t, TABLE, 3, 2, 50.0, 30.0, target=np.ones((1, 5), np.float32),
                             tiles=[dict(segments=np.asarray([(0, 1, 1, 1)], np.float32))])
    assert not flat.any() and (ai == -1).all() and (si == -1).all()


def test_padding_rows_are_zeros_with_index_minus_one():
    st, t = _state([(1.0, 0.0)])
    ego, goal, ag, sg, ai, si = _obs(st, t, k=3, s=2, tiles=[dict(segments=np.asarray([(0, 1, 1, 1)], np.float32))])
    assert list(ai) == [1, -1, -1] and list(si) == [0, -1]
    assert not ag[1:].any() and not sg[1:].any()
    assert not goal.any()   # no goal set
    assert ego[0] == 1.0


def test_goal_and_t_frac():
    st, t = _state([])
    target = np.asarray([[0.0, 2.0, 0.5, 2.0, 1.0]], np.float32)
    ego, goal, _, _, _, _ = _obs(st, t, k=0, target=target, step_count=np.asarray([3]), max_step=12)
    assert ego[7] == np.float32(0.25)
    assert goal[0] == 1.0 and (goal[1], goal[2]) == (0.0, 2.0) and goal[7] == 2.0 and (goal[5], goal[6]) == (2.0, 1.0)
    assert goal[3] == np.float32(np.cos(0.5)) and goal[4] == np.float32(np.sin(0.5))
    assert _obs(st, t, k=0, step_count=np.asarray([3]), max_step=0)[0][7] == 0.0


# ---- selection against exact rational arithmetic
def _exact_point(px, py, x0, y0):
    dx, dy = Fraction(float(px)) - Fraction(float(x0)), Fraction(float(py)) - Fraction(float(y0))
    return dx * dx + dy * dy


def _exact_segment(e, x0, y0):
    x1, y1, x2, y2 = (Fraction(float(v)) for v in e)
    ax, ay, ux, uy = x1 - Fraction(float(x0)), y1 - Fraction(float(y0)), x2 - x1, y2 - y1
    uu = ux * ux + uy * uy
    t = min(max(-(ax * ux + ay * uy) / uu, Fraction(0)), Fraction(1)) if uu > 0 else Fraction(0)
    px, py = ax + t * ux, ay + t * uy
    return px * px + py * py


def _separated(values, r2, rel=1e-9):
    v = sorted(values + [r2])
    return all(b - a > rel * max(abs(b), Fraction(1)) for a, b in zip(v, v[1:]))


def test_selection_matches_exact_arithmetic_on_separated_scenes():
    rng = np.random.default_rng(11)
    n, m, K, S, ra, rs = 64, 24, 6, 5, 20.0, 15.0
    x = rng.uniform(-30, 30, (n, m)).astype(np.float32)
    y = rng.uniform(-30, 30, (n, m)).astype(np.float32)
    h = rng.uniform(-np.pi, np.pi, (n, m)).astype(np.float32)
    z = np.zeros((n, m), np.float32)
    types = rng.integers(0, 3, (n, m)).astype(np.uint8)
    types[:, 0] = 0
    segs = rng.uniform(-30, 30, (40, 4)).astype(np.float32)
    st = dict(x=x, y=y, heading=h, speed=z, vx=z, vy=z)
    _, ai, si = V.observe(st, types, TABLE, K, S, ra, rs, tiles=[dict(segments=segs)])
    ra2, rs2 = Fraction(float(np.float32(ra))) ** 2, Fraction(float(np.float32(rs))) ** 2
    checked = 0
    for i in range(n):
        cand = [j for j in range(1, m) if types[i, j] != 2]
        d = {j: _exact_point(x[i, j], y[i, j], x[i, 0], y[i, 0]) for j in cand}
        e = {k: _exact_segment(segs[k], x[i, 0], y[i, 0]) for k in range(len(segs))}
        if not (_separated(list(d.values()), ra2) and _separated(list(e.values()), rs2)):
            continue
        want_a = sorted((v, j) for j, v in d.items() if v <= ra2)[:K]
        want_s = sorted((v, k) for k, v in e.items() if v <= rs2)[:S]
        assert list(ai[i]) == [j for _, j in want_a] + [-1] * (K - len(want_a)), i
        assert list(si[i]) == [k for _, k in want_s] + [-1] * (S - len(want_s)), i
        checked += 1
    assert checked >= n // 2


def test_field_names_match_the_blocks():
    from tactics2d_b200 import AGENT_FIELDS, EGO_FIELDS, GOAL_FIELDS, SEGMENT_FIELDS, vector_obs_width

    assert (len(EGO_FIELDS), len(GOAL_FIELDS), len(AGENT_FIELDS), len(SEGMENT_FIELDS)) == (V.EGO_F, V.GOAL_F, V.AGENT_F, V.SEG_F)
    assert vector_obs_width(16, 32) == V.width(16, 32) == 16 + 11 * 16 + 9 * 32
    assert AGENT_FIELDS[10] == GOAL_FIELDS[7] == SEGMENT_FIELDS[7] == "dist"
