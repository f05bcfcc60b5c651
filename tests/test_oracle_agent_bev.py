"""Known answers of the per-agent BEV statement (tests/agent_bev_oracle.py): the slot-0 row is the ego image, absent rows
are background, an observer sees itself on the image centre facing +x, per-row goals land where they are, and duplicate
rows agree."""

import numpy as np

from tests import agent_bev_oracle as AB
from tests import bev_oracle as B

# 0 background, 1 arrow, 2 ring, 3 open, 4 body, 5 disc, 6 target
Z = [-128, 7, 5, 4, 6, 6, 1]
LW = [1.0] * 7
BODY, DISC, TARGET = 4, 5, 6
TABLE = dict(shape=np.array([0, 1, 2]), half_len=np.array([1.0, 0.0, 0.0]), half_wid=np.array([0.5, 0.0, 0.0]),
             radius=np.array([0.0, 0.5, 0.0]))
TS = [BODY, DISC, BODY]          # type 2 is shapeless: never drawn
RES, RNG = (64, 64), (8.0, 8.0, 8.0, 8.0)


def _world():
    """Two scenarios of five slots: boxes, a disc, a shapeless slot and an empty one (scenario 1 has no slot 0)."""
    x = np.array([[0.0, 3.0, -2.5, 1.0, 9.0], [5.0, 6.0, 4.0, 5.5, 0.0]], np.float32)
    y = np.array([[0.0, 1.5, -2.0, -3.0, 9.0], [5.0, 3.0, 7.0, 5.5, 0.0]], np.float32)
    h = np.array([[0.3, -1.1, 0.0, 0.5, 0.0], [0.0, 2.2, 0.0, 1.0, 0.0]], np.float32)
    tid = np.array([[0, 0, 1, 2, 255], [255, 0, 1, 0, 255]], np.uint8)
    seg = np.array([[-6, 4, 6, 4], [-6, -5, -6, 5]], np.float32)
    return dict(x=x, y=y, heading=h), tid, dict(segments=seg, poly_start=None)


def _row(n, j, goal=None, rng=RNG, res=RES):
    st, tid, tile = _world()
    return AB.render_row(n, j, st, tid, TABLE, TS, Z, LW, res[0], res[1], rng, tile, None, goal, TARGET)


def test_slot_zero_row_is_the_ego_image():
    st, tid, tile = _world()
    target = np.array([[2.0, -1.0, 0.2, 1.5, 0.8], [0.0] * 5], np.float32)
    ref = B.render_world_scenario(0, st, tid, TABLE, TS, Z, LW, RES[0], RES[1], RNG, tile, None, target, TARGET)
    rows = AB.render_agents(st, tid, TABLE, TS, Z, LW, RES[0], RES[1], RNG, observers=[[3, 0, 1], [0, 1, 2]],
                            rows=[(0, 1)], tiles=[tile, tile], target=target, target_style=TARGET)
    assert np.array_equal(rows[(0, 1)], ref)
    assert (ref == TARGET).any() and (ref == BODY).any() and (ref == 3).any()


def test_absent_retired_and_out_of_range_rows_are_background():
    st, tid, tile = _world()
    for n, j in ((0, 4), (0, -1), (0, 5), (0, 300), (1, 0), (1, 4)):
        img = AB.render_row(n, j, st, tid, TABLE, TS, Z, LW, RES[0], RES[1], RNG, tile)
        assert img.shape == (RES[1], RES[0]) and not img.any(), (n, j)
    # the ego image of scenario 1 (no slot 0) takes the no-ego view and draws; its slot-0 row does not
    assert B.render_world_scenario(1, st, tid, TABLE, TS, Z, LW, RES[0], RES[1], RNG, tile).any()
    # retiring slot 1 (type 255) empties its row and removes its body from slot 0's row
    tid2 = tid.copy()
    tid2[0, 1] = 255
    assert not AB.render_row(0, 1, st, tid2, TABLE, TS, Z, LW, RES[0], RES[1], RNG, tile).any()
    before = AB.render_row(0, 0, st, tid, TABLE, TS, Z, LW, RES[0], RES[1], RNG, tile)
    after = AB.render_row(0, 0, st, tid2, TABLE, TS, Z, LW, RES[0], RES[1], RNG, tile)
    assert (before == BODY).sum() > (after == BODY).sum()


def test_box_observer_sees_itself_on_the_centre_with_its_arrow_along_plus_x():
    img = _row(0, 1)   # slot 1 at (3, 1.5), heading -1.1
    xmin, ymax, px, py = B.window(RES[0], RES[1], RNG)
    r, c = np.meshgrid(np.arange(RES[1]), np.arange(RES[0]), indexing="ij")
    u, v = xmin + (c + 0.5) * px, ymax - (r + 0.5) * py
    body = (img == BODY) | (img == 1)
    # its own body is the axis-aligned 2 x 1 box about the centre (other slots lie farther than 2 m away)
    near = (np.abs(u) <= 1.5) & (np.abs(v) <= 1.0)
    assert np.array_equal(body & near, (np.abs(u) <= 1.0) & (np.abs(v) <= 0.5))
    arrow = (img == 1) & near
    assert arrow.any() and (u[arrow] >= 0.0).all()
    # the shapeless slot 3 centres a view too, and draws nothing of its own at the centre
    img3 = _row(0, 3)
    assert img3.any() and img3[RES[1] // 2, RES[0] // 2] == 0


def test_per_row_goal_lands_on_its_rectangle_and_nan_draws_nothing():
    st, tid, tile = _world()
    goals = np.full((2, 3, 5), np.nan, np.float32)
    goals[0, 0] = (3.5, -4.0, 0.0, 1.0, 0.75)   # row 0, observed by slot 2 (a disc at (-2.5, -2))
    obs = [[2, 2, 0], [1, 1, 3]]
    target = np.array([[1.0, 1.0, 0.0, 1.0, 1.0], [1.0, 1.0, 0.0, 1.0, 1.0]], np.float32)
    rows = AB.render_agents(st, tid, TABLE, TS, Z, LW, RES[0], RES[1], RNG, observers=obs, tiles=[tile, tile],
                            target=target, goals=goals, target_style=TARGET)
    img = rows[(0, 0)]
    X, Y = B.pixel_centres(B.view_of(-2.5, -2.0, 0.0, True), B.window(RES[0], RES[1], RNG), RES[0], RES[1])
    inside = (np.abs(X - 3.5) <= 1.0) & (np.abs(Y + 4.0) <= 0.75)
    assert np.array_equal(img == TARGET, inside) and inside.sum() > 20
    # NaN goals draw nothing, slot 0's row included (the per-row goals replace the target)
    for key in ((0, 1), (0, 2), (1, 0), (1, 2)):
        assert not (rows[key] == TARGET).any(), key
    # without goals only slot 0's row draws the target
    rows = AB.render_agents(st, tid, TABLE, TS, Z, LW, RES[0], RES[1], RNG, observers=obs, tiles=[tile, tile],
                            target=target, target_style=TARGET)
    assert (rows[(0, 2)] == TARGET).any() and not (rows[(0, 0)] == TARGET).any()


def test_duplicate_rows_are_identical():
    st, tid, tile = _world()
    rows = AB.render_agents(st, tid, TABLE, TS, Z, LW, RES[0], RES[1], RNG, observers=[[1, 2, 1, 1], [2, 3, 3, 2]],
                            tiles=[tile, tile])
    assert np.array_equal(rows[(0, 0)], rows[(0, 2)]) and np.array_equal(rows[(0, 0)], rows[(0, 3)])
    assert np.array_equal(rows[(1, 0)], rows[(1, 3)]) and np.array_equal(rows[(1, 1)], rows[(1, 2)])
    assert not np.array_equal(rows[(0, 0)], rows[(0, 1)])
