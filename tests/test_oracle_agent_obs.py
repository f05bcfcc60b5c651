"""The float64 per-agent observation oracle (tests/agent_obs_oracle.py) against the vector-observation oracle it generalises,
against exact rational arithmetic on tie scenes, and on known answers.  No GPU needed."""

from fractions import Fraction

import numpy as np

from tests import agent_obs_oracle as A
from tests import vector_obs_oracle as V

BOX = dict(shape=V.SHAPE_OBB, half_len=2.5, half_wid=1.0, radius=0.0)
DISC = dict(shape=V.SHAPE_CIRCLE, half_len=0.3, half_wid=0.3, radius=0.3)
NONE = dict(shape=V.SHAPE_NONE, half_len=1.0, half_wid=1.0, radius=0.0)
TABLE = [BOX, DISC, NONE]


def _scene(seed, n=48, m=20, span=30.0, n_seg=50, empty=0.1):
    """Continuous random scenes: positions, headings, velocities, types (some empty), segments and per-scenario step counts."""
    rng = np.random.default_rng(seed)
    f = lambda *s: rng.uniform(-span, span, s).astype(np.float32)
    st = dict(x=f(n, m), y=f(n, m), heading=rng.uniform(-4, 4, (n, m)).astype(np.float32),
              speed=rng.uniform(0, 20, (n, m)).astype(np.float32), vx=f(n, m) / 3, vy=f(n, m) / 3)
    types = rng.integers(0, 3, (n, m)).astype(np.uint8)
    types[rng.random((n, m)) < empty] = 255
    segs = f(n_seg, 4)
    tiles = [dict(segments=segs, poly_start=np.asarray([0, 6, 12], np.int32))]
    steps = rng.integers(0, 40, n)
    return st, types, tiles, steps


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _both(st, types, K, S, ra, rs, observers=None, **kw):
    return A.observe_agents(st, types, TABLE, K, S, ra, rs, observers=observers, **kw)


def test_observer_zero_is_the_vector_observation_bit_for_bit():
    st, types, tiles, steps = _scene(1)
    n = types.shape[0]
    types[::7, 0] = 255   # scenarios without an ego
    target = np.stack([st["x"][:, 0] + 3, st["y"][:, 0] - 4, np.full(n, 0.7), np.full(n, 2.5), np.full(n, 1.2)], 1)
    for tgt in (None, target.astype(np.float32)):
        for K, S, ra, rs in ((6, 9, 20.0, 15.0), (19, 50, 1e5, 1e5), (0, 3, 5.0, 5.0), (4, 0, 30.0, 30.0)):
            kw = dict(step_count=steps, max_step=40, target=tgt, tiles=tiles)
            ref, ai, si = V.observe(st, types, TABLE, K, S, ra, rs, **kw)
            got, gai, gsi = _both(st, types, K, S, ra, rs, observers=np.zeros((n, 1), np.int64), **kw)
            assert got.shape == (n, 1, V.width(K, S))
            assert np.array_equal(_bits(got[:, 0]), _bits(ref))
            assert np.array_equal(gai[:, 0], ai) and np.array_equal(gsi[:, 0], si)


def _swap(a, j):
    a = np.array(a, copy=True)
    a[:, [0, j]] = a[:, [j, 0]]
    return a


def test_observer_j_is_the_vector_observation_with_slots_0_and_j_swapped():
    st, types, tiles, steps = _scene(2, empty=0.0)   # continuous positions: no distance ties
    n, m = types.shape
    K, S, ra, rs = 8, 12, 25.0, 20.0
    got, gai, gsi = _both(st, types, K, S, ra, rs, step_count=steps, max_step=40, tiles=tiles)
    assert got.shape == (n, m, V.width(K, S))
    for j in (1, 2, 7, m - 1):
        ref, ai, si = V.observe({k: _swap(v, j) for k, v in st.items()}, _swap(types, j), TABLE, K, S, ra, rs,
                                step_count=steps, max_step=40, tiles=tiles)
        ai = ai.astype(np.int64)
        mapped = np.where(ai == j, 0, np.where(ai == 0, j, ai))   # slot 0 of the swapped world is slot j here
        assert np.array_equal(_bits(got[:, j]), _bits(ref)), j
        assert np.array_equal(gai[:, j], mapped) and np.array_equal(gsi[:, j], si), j
        assert (gai[:, j] == 0).any()   # the scenario's slot 0 is among the observed agents


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


def test_selection_on_lattice_ties_matches_exact_arithmetic():
    rng = np.random.default_rng(5)
    n, m, Q = 12, 30, 6
    x = rng.integers(-4, 5, (n, m)).astype(np.float32)
    y = rng.integers(-4, 5, (n, m)).astype(np.float32)
    z = np.zeros((n, m), np.float32)
    st = dict(x=x, y=y, heading=(rng.integers(0, 4, (n, m)) * (np.pi / 2)).astype(np.float32), speed=z, vx=z, vy=z)
    types = rng.integers(0, 3, (n, m)).astype(np.uint8)
    types[rng.random((n, m)) < 0.1] = 255
    g = np.arange(-6, 7, dtype=np.float32)
    segs = np.asarray([(a, b, a + 1, b) for a in g for b in g] + [(a, b, a, b + 1) for a in g for b in g] +
                      [(a, b, a, b) for a in g[::3] for b in g[::3]], np.float32)
    observers = rng.integers(0, m, (n, Q))
    n_types = len(TABLE)
    for K, S, ra, rs in ((5, 7, 3.0, 2.0), (29, 120, 6.0, 3.5)):
        _, ai, si = _both(st, types, K, S, ra, rs, observers=observers, tiles=[dict(segments=segs)])
        ra2, rs2 = Fraction(float(np.float32(ra))) ** 2, Fraction(float(np.float32(rs))) ** 2
        for i in range(n):
            for q in range(Q):
                j = observers[i, q]
                if types[i, j] >= n_types:
                    assert (ai[i, q] == -1).all() and (si[i, q] == -1).all()
                    continue
                d = {k: _exact_point(x[i, k], y[i, k], x[i, j], y[i, j]) for k in range(m)
                     if k != j and types[i, k] < n_types and TABLE[types[i, k]]["shape"] != V.SHAPE_NONE}
                e = {k: _exact_segment(segs[k], x[i, j], y[i, j]) for k in range(len(segs))}
                want_a = sorted((v, k) for k, v in d.items() if v <= ra2)[:K]
                want_s = sorted((v, k) for k, v in e.items() if v <= rs2)[:S]
                assert list(ai[i, q]) == [k for _, k in want_a] + [-1] * (K - len(want_a)), (i, q)
                assert list(si[i, q]) == [k for _, k in want_s] + [-1] * (S - len(want_s)), (i, q)


def test_absent_rows_for_out_of_range_and_empty_observers():
    st, types, tiles, steps = _scene(3, n=6, m=10, empty=0.0)
    types[:] = 0
    types[:, 4] = 255
    obs = np.asarray([[-1, 10, 4, 2, -32768, 32767]] * 6)
    target = np.ones((6, 5), np.float32)
    got, ai, si = _both(st, types, 5, 6, 1e5, 1e5, observers=obs, step_count=steps, max_step=40, target=target,
                        tiles=tiles)
    for q in (0, 1, 2, 4, 5):
        assert not got[:, q].any() and (ai[:, q] == -1).all() and (si[:, q] == -1).all(), q
    assert (got[:, 3, 0] == 1).all() and (ai[:, 3] >= 0).sum(1).min() == 5 and (si[:, 3] >= 0).all()


def test_duplicate_observers_give_equal_rows():
    st, types, tiles, steps = _scene(4, n=8, m=12)
    obs = np.asarray([[3, 5, 3, 0, 5]] * 8)
    got, ai, si = _both(st, types, 6, 8, 30.0, 20.0, observers=obs, tiles=tiles, step_count=steps, max_step=40)
    assert np.array_equal(got[:, 0], got[:, 2]) and np.array_equal(got[:, 1], got[:, 4])
    assert np.array_equal(ai[:, 0], ai[:, 2]) and np.array_equal(si[:, 1], si[:, 4])
    full, fai, _ = _both(st, types, 6, 8, 30.0, 20.0, tiles=tiles, step_count=steps, max_step=40)
    assert np.array_equal(got[:, 0], full[:, 3]) and np.array_equal(ai[:, 1], fai[:, 5])


def test_goals_per_row_and_the_target_for_slot_zero_only():
    st, types, tiles, _ = _scene(6, n=5, m=6, empty=0.0)
    n, m = types.shape
    target = np.tile(np.asarray([[1.0, 2.0, 0.3, 2.0, 1.0]], np.float32), (n, 1))
    got, _, _ = _both(st, types, 2, 2, 30.0, 20.0, target=target, tiles=tiles)
    goal = A.split(got, 2, 2)[1]
    assert (goal[:, 0, 0] == 1).all() and not goal[:, 1:].any()   # only the rows observed by slot 0
    # per-row goals replace the target; a NaN cx is none
    goals = np.random.default_rng(1).uniform(-5, 5, (n, m, 5)).astype(np.float32)
    goals[:, ::2, 0] = np.nan
    got, _, _ = _both(st, types, 2, 2, 30.0, 20.0, target=target, goals=goals, tiles=tiles)
    goal = A.split(got, 2, 2)[1]
    assert not goal[:, ::2].any() and (goal[:, 1::2, 0] == 1).all()
    # a goal row is the target block of that observer: compare with the swapped world's vector observation
    j = 3
    ref, _, _ = V.observe({k: _swap(v, j) for k, v in st.items()}, _swap(types, j), TABLE, 2, 2, 30.0, 20.0,
                          target=goals[:, j], tiles=tiles)
    assert np.array_equal(_bits(got[:, j]), _bits(ref))


def _one(xy, heading=None, types=None):
    xy = np.asarray(xy, np.float32)
    m = len(xy)
    h = np.zeros((1, m), np.float32) if heading is None else np.asarray(heading, np.float32).reshape(1, m)
    z = np.zeros((1, m), np.float32)
    st = dict(x=xy[None, :, 0], y=xy[None, :, 1], heading=h, speed=z, vx=z, vy=z)
    t = np.zeros((1, m), np.uint8) if types is None else np.asarray(types, np.uint8).reshape(1, m)
    return st, t


def test_known_answers():
    # slot 1 at (3, 4) sees slot 0 at distance 5, and slot 2 behind it
    st, t = _one([(0.0, 0.0), (3.0, 4.0), (3.0, 10.0)])
    got, ai, _ = _both(st, t, 3, 0, 50.0, 30.0, observers=np.asarray([[1]]))
    ag = A.split(got, 3, 0)[2][0, 0]
    assert list(ai[0, 0]) == [0, 2, -1]
    assert (ag[0, 10], ag[1, 10]) == (5.0, 6.0) and (ag[0, 1], ag[0, 2]) == (-3.0, -4.0)
    # an observer facing +y sees a slot on its +x side at ey = -1
    st, t = _one([(5.0, 5.0), (4.0, 5.0), (0.0, 0.0)], heading=[0.0, np.pi / 2, 0.0])
    got, ai, _ = _both(st, t, 1, 0, 2.0, 30.0, observers=np.asarray([[1]]))
    ag = A.split(got, 1, 0)[2][0, 0, 0]
    assert ai[0, 0, 0] == 0 and abs(ag[1]) < 1e-6 and ag[2] == -1.0
    # a disc observer's ego block; the segment (0, 1)-(10, 1) is 1 m from slot 2 at (0, 0)
    st, t = _one([(0.0, 5.0), (1.0, 5.0), (0.0, 0.0)], types=[0, 0, 1])
    tiles = [dict(segments=np.asarray([(0, 1, 10, 1)], np.float32))]
    got, _, si = _both(st, t, 0, 1, 50.0, 1.0, observers=np.asarray([[2, 0]]), tiles=tiles)
    ego, _, _, sg = A.split(got, 0, 1)
    assert tuple(ego[0, 0, 4:7]) == (np.float32(0.3), np.float32(0.3), 1.0) and tuple(ego[0, 1, 4:7]) == (2.5, 1.0, 0.0)
    assert si[0, 0, 0] == 0 and sg[0, 0, 0, 7] == 1.0 and si[0, 1, 0] == -1
