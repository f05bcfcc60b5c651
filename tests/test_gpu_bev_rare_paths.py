"""K6 (t2d_bev_render) on the paths tests/test_gpu_bev.py does not take, against the float64 oracle in
tests/bev_oracle.py: every class image bit for bit, and RGB = palette[class] wherever RGB is rendered.

* More than 512 visible primitives: the fallback that rebuilds every candidate at every pixel, in the same launch as
  staged scenarios, with the visible count P of every scenario exact by construction (``count_visible``, whose known
  answers are the one test here that needs no GPU); and the same launch captured in a CUDA graph.
* Image shapes whose 16-pixel runs are short (W * H or a band's pixel count not a multiple of 16) or start at an
  unaligned address (W * H odd: scenario n's image starts at pixel n * W * H), which take the bytewise stores, and
  bands shorter than 16 rows; W = 1024, where a band's mask uses all 64 bins.
* Views without an ego (tile bounds centre or origin), tiles without segments or bounds, a world without a map, and
  ``set_map`` against a one-tile ``set_map_table``.
* Ranges of 0.5 m (one box covers the image, its pixel box runs far past it) and 1e5 m (primitives smaller than a
  pixel), and asymmetric ranges at W != H."""

import numpy as np
import pytest

from tests import bev_oracle as B
from tests.test_gpu_bev import _styles

VEH, CYC, PED, OBS, EMPTY = 0, 1, 2, 3, 255


def _extents(x, y, h, type_id, table, type_style, z, lw, pitch_x, segments=None, poly_start=None, seg_style=None,
             target=None, target_style=B.NOT_DRAWN, ring_style=2, open_style=3):
    """For every primitive of ``bev_oracle.primitives`` (same arguments, same order): the world points whose box the
    kernel culls it by (``make_prim``), and how far in metres the primitive reaches beyond that box (a stroke's half
    width, else 0)."""
    f = lambda v: float(np.float32(v))   # noqa: E731  (device values are float32)
    out = []
    if target is not None and target_style != B.NOT_DRAWN:
        out.append((np.stack(B.box_ring(*(f(v) for v in target[:5])), 1), 0.0))
    seg = np.zeros((0, 4)) if segments is None else np.asarray(segments, np.float32).astype(np.float64)
    ps = [] if poly_start is None or len(poly_start) < 2 else [int(v) for v in poly_start]
    style_of = (lambda s, d: d) if seg_style is None else (lambda s, d: int(seg_style[s]))
    for p in range(len(ps) - 1):
        if style_of(ps[p], ring_style) != B.NOT_DRAWN:   # a ring object: the corners of its vertices' world box
            (x0, y0), (x1, y1) = seg[ps[p]:ps[p + 1], :2].min(0), seg[ps[p]:ps[p + 1], :2].max(0)
            out.append((np.array([[x0, y0], [x0, y1], [x1, y0], [x1, y1]]), 0.0))
    for s in range(len(seg)):
        if ps and ps[0] <= s < ps[-1]:
            continue
        st = style_of(s, open_style)
        if st != B.NOT_DRAWN:
            out.append((seg[s].reshape(2, 2), np.sqrt(B.stroke_hw2(lw[st], pitch_x))))
    for j in range(len(type_id)):
        t = int(type_id[j])
        if t >= len(type_style) or type_style[t] == B.NOT_DRAWN:
            continue
        if table["shape"][t] == B.SHAPE_CIRCLE:   # the corners of the disc's world box
            cx, cy, r = f(x[j]), f(y[j]), table["radius"][t]
            out.append((np.array([[cx - r, cy - r], [cx - r, cy + r], [cx + r, cy - r], [cx + r, cy + r]]), 0.0))
        elif table["shape"][t] == B.SHAPE_OBB:
            rx, ry = B.box_ring(f(x[j]), f(y[j]), f(h[j]), table["half_len"][t], table["half_wid"][t])
            out.append((np.stack([rx, ry], 1), 0.0))
            out.append((np.stack(B.arrow(rx, ry), 1), 0.0))
    return out


def count_visible(args, view, width, height, rng, margin=2.0):
    """The kernel's visible count P for the scene ``bev_oracle.primitives(*args)`` seen from ``view``: P <= 512 takes
    the staged path, more the fallback.  The kernel keeps a primitive whose pixel box, grown by one pixel of slack,
    meets the image; to make P certain, every primitive must lie at least ``margin`` pixels inside the image (counted)
    or beyond one of its edges (not counted).  Raises ValueError for one in between."""
    ext = _extents(*args)
    assert len(ext) == len(B.primitives(*args))
    ex, ey, cs, sn = view
    xmin, ymax, px, py = B.window(width, height, rng)
    n = 0
    for k, (pts, reach) in enumerate(ext):
        dx, dy = pts[:, 0] - ex, pts[:, 1] - ey
        fc = (cs * dx + sn * dy - xmin) / px
        fr = (ymax - (-sn * dx + cs * dy)) / py
        g = reach / min(px, py)
        c0, c1, r0, r1 = fc.min() - g, fc.max() + g, fr.min() - g, fr.max() + g
        if c0 >= margin and c1 <= width - margin and r0 >= margin and r1 <= height - margin:
            n += 1
        elif not (c1 <= -margin or r1 <= -margin or c0 >= width + margin or r0 >= height + margin):
            raise ValueError(f"primitive {k} lies within {margin} px of the image's edge")
    return n


def test_visible_count_inside_outside_and_near_the_edge():
    """CPU known answers of count_visible at 256 x 256 and pitch 0.125 (x = 16 - 0.125 k is k px inside)."""
    rng, view = (16, 16, 16, 16), (0.0, 0.0, 1.0, 0.0)
    table = dict(shape=np.array([0, 1, 2]), half_len=np.array([1.0, 0.0, 0.0]), half_wid=np.array([0.5, 0.0, 0.0]),
                 radius=np.array([0.0, 0.5, 0.0]))
    z, lw = [-128, 7, 5, 4, 6, 6, 1], [1.0] * 7

    def count(parts, seg, target=None, **kw):
        x = [p[0] for p in parts]; y = [p[1] for p in parts]; h = [p[2] for p in parts]; t = [p[3] for p in parts]
        ring = np.array([[-3, -3, -2, -3], [-2, -3, -2, -2], [-2, -2, -3, -3]], np.float32)
        segs = np.concatenate([ring, ring + 100, np.asarray(seg, np.float32).reshape(-1, 4)])
        args = (x, y, h, t, table, [4, 5, 4], z, lw, 0.125, segs, [0, 3, 6], None, target, 6)
        return count_visible(args, view, 256, 256, rng, **kw)

    # inside: a body and its arrow, a disc, one ring, one stroke; beyond the image: a body, a disc, a ring, a stroke;
    # SHAPE_NONE draws nothing
    parts = [(0.0, 0.0, 0.3, 0), (30.0, 0.0, 0.0, 0), (0.0, -40.0, 0.0, 1), (5.0, 5.0, 0.0, 1), (1.0, 1.0, 0.0, 2)]
    seg = [[-1, 5, 1, 5], [40, 40, 41, 41]]
    assert count(parts, seg) == 5
    assert count(parts, seg, target=[-5, -5, 0.0, 1.0, 0.5]) == 6      # the goal moves the count by one
    assert count(parts, seg, target=[-50, -5, 0.0, 1.0, 0.5]) == 5
    # a stroke ending 4 px inside the right edge counts; 3 px inside, its half width (1.39 px) brings it within 2 px
    assert count(parts, seg + [[10, 0, 16 - 4 * 0.125, 0]]) == 6
    with pytest.raises(ValueError):
        count(parts, seg + [[10, 0, 16 - 3 * 0.125, 0]])
    # a box reaching over the top edge, or ending 1 px beyond the left edge, is in neither class; 2 px beyond, it is out
    with pytest.raises(ValueError):
        count(parts + [(0.0, 15.8, 0.0, 0)], seg)
    with pytest.raises(ValueError):
        count(parts + [(-16.125 - 1.0, 0.0, 0.0, 0)], seg)
    assert count(parts + [(-16.25 - 1.0, 0.0, 0.0, 0)], seg) == 5


def _table():
    from tactics2d_b200.types import TypeParams, TypeTable

    return TypeTable([TypeParams.vehicle("medium_car"), TypeParams.cyclist("cyclist"), TypeParams.pedestrian("adult_male"),
                      TypeParams.obstacle(2.0, 1.0)])


def _world(n, m, x, y, h, types, tiles=None, tile_id=None, target=None):
    """A world of the four-row table; ``tiles``: one tile through ``set_map`` (tile_id None) or a map table."""
    from tactics2d_b200 import BatchedWorld

    w = BatchedWorld(n, m, _table())
    if tiles is not None and tile_id is None:
        t = tiles[0]
        w.set_map(t["segments"], t.get("bounds"), poly_start=t.get("poly_start"), style=t.get("style"))
    elif tiles is not None:
        w.set_map_table(tiles, tile_id)
    w.set_state(x, y, h, np.zeros((n, m), np.float32), type_id=types)
    if target is not None:
        w.set_goal(target)
    w.set_bev_styles()
    return w


def _scene(w, n, res, rng, tile=None, target=None):
    """(arguments of ``bev_oracle.primitives``, view) of scenario n of w, as ``bev_oracle.render_world_scenario``
    builds them; ``tile`` as given to set_map / set_map_table."""
    idx, ts, z, lw = _styles(w)
    st, tid, tile = w.state_numpy(), w.type_id.cpu().numpy(), tile or {}
    ss = None if tile.get("style") is None else np.asarray([idx[k] for k in tile["style"]], np.uint8)
    view = B.view_of(st["x"][n, 0], st["y"][n, 0], st["heading"][n, 0], int(tid[n, 0]) < len(ts), tile.get("bounds"))
    args = (st["x"][n], st["y"][n], st["heading"][n], tid[n], w.type_table.as_oracle_table(), ts, z, lw,
            B.window(res[0], res[1], rng)[2], tile.get("segments"), tile.get("poly_start"), ss,
            None if target is None else target[n], B.NOT_DRAWN if target is None else idx["target_area"])
    return args, view


def _check(w, res, rng, tiles=None, target=None):
    """Render class and RGB images; RGB must be palette[class] and every scenario's class image the oracle's.
    ``tiles``: the tile of every scenario, or None without a map.  Returns the class images."""
    import torch
    from tactics2d_b200.sensor.camera import palette

    cls = w.bev(res, rng, rgb=False).clone()
    rgb = w.bev(res, rng, rgb=True)
    assert torch.equal(torch.from_numpy(palette()).to(cls.device)[cls.long()], rgb), (res, rng)
    got = cls.cpu().numpy()
    for n in range(w.N):
        args, view = _scene(w, n, res, rng, None if tiles is None else tiles[n], target)
        ref = B.render(B.primitives(*args), view, res[0], res[1], rng)
        assert np.array_equal(got[n], ref), (res, rng, n, int((got[n] != ref).sum()))
    return got


def _rot(pose, u, v):
    """World coordinates of the point (u, v) in the frame of pose (x, y, heading)."""
    c, s = np.cos(pose[2]), np.sin(pose[2])
    return pose[0] + c * np.asarray(u) - s * np.asarray(v), pose[1] + s * np.asarray(u) + c * np.asarray(v)


def _ring(pose, cu, cv, hu, hv):
    u, v = np.array([cu - hu, cu + hu, cu + hu, cu - hu]), np.array([cv - hv, cv - hv, cv + hv, cv + hv])
    return np.stack(_rot(pose, u, v), 1)


def _tile(pose, rings, strokes, bounds=None):
    """rings: [(vertices, holes, style)]; strokes: [((u1, v1, u2, v2), style)] in the frame of pose."""
    from tactics2d_b200.map import Area, polygons_to_segments

    areas = [Area(i, None, None, r, list(holes)) for i, (r, holes, _) in enumerate(rings)]
    lines = [np.stack(_rot(pose, [s[0], s[2]], [s[1], s[3]]), 1) for s, _ in strokes]
    seg, ps = polygons_to_segments(areas, lines)
    style = [st for p, (_, _, st) in enumerate(rings) for _ in range(ps[p], ps[p + 1])] + [st for _, st in strokes]
    return dict(segments=seg, poly_start=ps, bounds=bounds, style=style)


# ---------------------------------------------------------------------------------------------------- the fallback
# 128 x 96 at range 20: pitch 5/12 m, the view spans u in +-26.7 m, v in +-20 m.  Everything counted lies at least
# 2 px inside the image (|u| <= 25.8, |v| <= 19.1 for its whole extent), everything else 80 m beyond it.
FB_RES, FB_RNG = (128, 96), (20.0, 20.0, 20.0, 20.0)
EGO = (31.0, -12.0, 0.35)
FAR = 80.0


def _dense_tile(rs, n_open):
    """Ring objects (one with a hole) and n_open short strokes of both widths inside the view of EGO, a stroke under
    the body of slot 2, and a ring and strokes far outside: 3 + 1 + n_open visible candidates."""
    rings = [(_ring(EGO, -14, -10, 5, 4), [_ring(EGO, -14, -10, 2, 1.5)], "area"),     # with a hole
             (np.stack(_rot(EGO, [6, 11, 8], [-14, -14, -9]), 1), [], "building"),
             (_ring(EGO, 14, 10, 3, 2), [], "vegetation"),
             (_ring(EGO, FAR + 30, 0, 3, 2), [], "building")]
    strokes = [((-11.5, -12.5, -6.0, -7.5), "curbstone")]                              # under slot 2
    cu, cv = rs.uniform(-23, 23, n_open), rs.uniform(-17, 17, n_open)
    ang, half = rs.uniform(-np.pi, np.pi, n_open), rs.uniform(0.2, 1.5, n_open)
    for k in range(n_open):
        du, dv = half[k] * np.cos(ang[k]), half[k] * np.sin(ang[k])
        strokes.append(((cu[k] - du, cv[k] - dv, cu[k] + du, cv[k] + dv), ("roadline", "curbstone")[k % 2]))
    strokes += [((FAR + 30 + k, -5, FAR + 31 + k, 5), "roadline") for k in range(6)]
    return _tile(EGO, rings, strokes)


def _dense_slots(rs, m, n_fill, n_ped):
    """One scenario's slots around EGO: the ego (2 candidates), a body over the goal, a body across ring 0 and a stroke,
    a car under a cyclist (8), n_ped of 10 pedestrians, obstacles, empty and retired slots (0), two boxes far outside
    (0) and n_fill of the filler cars and cyclists (2 each): 10 + n_ped + 2 n_fill visible candidates."""
    types = np.full(m, EMPTY, np.uint8)
    u, v, hh = np.zeros(m), np.zeros(m), np.zeros(m)

    def put(j, t, uu, vv, hd):
        types[j], u[j], v[j], hh[j] = t, uu, vv, hd

    put(0, VEH, 0.0, 0.0, 0.0)
    put(1, VEH, -15.0, 6.5, 0.6)              # over the goal at (-16, 6)
    put(2, VEH, -9.0, -10.0, np.pi / 2 - 0.2)  # across the right edge of ring 0 and the stroke under it
    put(3, VEH, 6.0, 8.0, 0.1)
    put(4, CYC, 6.8, 8.3, -0.4)               # the later slot, on top of slot 3 at the same z
    for j in range(5, 15):
        uu, vv = (rs.uniform(-23, 23), rs.uniform(-17, 17)) if j - 5 < n_ped else (-FAR - 30, 0.0)
        put(j, PED, uu, vv, 0.0)
    for j in range(15, 20):
        put(j, OBS, rs.uniform(-23, 23), rs.uniform(-17, 17), rs.uniform(-3, 3))
    for j in range(25, 30):                   # retired: type 255 with a pose in view (20..24 stay empty)
        put(j, EMPTY, rs.uniform(-23, 23), rs.uniform(-17, 17), 0.0)
    put(30, VEH, FAR + 30, 10.0, 0.3)
    put(31, CYC, 0.0, -FAR - 25, 1.0)
    for j in range(32, m):
        inside = j - 32 < n_fill
        put(j, (VEH, CYC)[j % 2], rs.uniform(-23, 23) if inside else FAR + 30 + j, rs.uniform(-16, 16),
            rs.uniform(-np.pi, np.pi))
    x, y = _rot(EGO, u, v)
    return x, y, hh + EGO[2], types


@pytest.fixture(scope="module")
def dense_world(cuda_device):
    """Four scenarios of M = 128 in one world: staged (a 100-stroke tile), exactly 512 and 513 visible primitives (the
    same scene without and with its goal), and fallback well past 512."""
    rs = np.random.default_rng(11)
    m = 128
    tiles = [_dense_tile(rs, 100), _dense_tile(rs, 470)]
    plan = [(0, 96, 10, True), (1, 10, 8, False), (1, 10, 8, True), (1, 96, 10, True)]   # tile, fillers, peds, goal
    slots = {}
    x, y, h = (np.zeros((4, m), np.float32) for _ in range(3))
    types = np.zeros((4, m), np.uint8)
    target = np.zeros((4, 5), np.float32)
    for n, (t, n_fill, n_ped, goal) in enumerate(plan):
        key = (n_fill, n_ped)
        if key not in slots:
            slots[key] = _dense_slots(rs, m, n_fill, n_ped)
        x[n], y[n], h[n], types[n] = slots[key]
        gx, gy = _rot(EGO, -16.0 if goal else -FAR - 30, 6.0)
        target[n] = (gx, gy, EGO[2] + 0.2, 2.5, 1.2)
    tid = np.asarray([p[0] for p in plan])
    w = _world(4, m, x, y, h, types, tiles, tid, target)
    yield w, [tiles[t] for t in tid], target
    w.close()


@pytest.mark.gpu
def test_fallback_beyond_512_visible_primitives_next_to_staged_scenarios(dense_world):
    w, tiles, target = dense_world
    P = [count_visible(*_scene(w, n, FB_RES, FB_RNG, tiles[n], target), FB_RES[0], FB_RES[1], FB_RNG) for n in range(4)]
    assert P == [317, 512, 513, 687]   # staged, staged at the limit, fallback at the limit, fallback
    got = _check(w, FB_RES, FB_RNG, tiles, target)
    idx = _styles(w)[0]
    # scenarios 1 and 2 differ by the goal alone; where slot 1's body lies over it, the body stays on top
    diff = got[1] != got[2]
    assert diff.any() and set(np.unique(got[2][diff])) == {idx["target_area"]}
    for n in (2, 3):   # every kind of primitive shows
        assert {idx[k] for k in ("target_area", "area", "building", "vegetation", "roadline", "curbstone", "vehicle",
                                 "cyclist", "pedestrian", "heading_arrow")} <= set(np.unique(got[n]))


@pytest.mark.gpu
def test_fallback_and_staged_launch_under_graph_capture_equals_eager(dense_world):
    import torch

    w, _, _ = dense_world
    for rgb in (False, True):
        eager = w.bev(FB_RES, FB_RNG, rgb=rgb).clone()
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            w.bev(FB_RES, FB_RNG, rgb=rgb)
        torch.cuda.current_stream().wait_stream(s)
        with torch.cuda.graph(g):
            out = w.bev(FB_RES, FB_RNG, rgb=rgb)
        out.fill_(77)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager), rgb


# ---------------------------------------------------------------------------------------------------- image shapes
# Per shape, the bytewise stores it takes: W * H odd puts scenario 1's image at an odd byte (every run unaligned), and
# scenario 2's at 2 W H, which is 16-byte aligned only when W * H is a multiple of 8; a band of min(16, H - row0) rows
# of W pixels not a multiple of 16 ends in a short run.
#   (1, 1), (1, 17), (17, 1), (15, 17), (17, 15), (1023, 15), (1023, 1023): W * H odd
#   (16, 15), (17, 16): W * H = 240 / 272 = 0 mod 16 and every run full: only 16-byte stores; a band of 15 rows, and
#   runs that wrap rows
#   (200, 17): W * H = 3400 = 8 mod 16, scenario 1 unaligned; the last band is one row of 200 = 12 runs + 8 pixels
#   (1024, 17), (17, 1024): W * H = 0 mod 16, only 16-byte stores; 1024 x 17 ends in a band of one row over all 64
#   bins, 17 x 1024 runs through 64 full bands of 272 pixels
SHAPES = [(1, 1), (1, 17), (17, 1), (15, 17), (17, 15), (16, 15), (17, 16), (200, 17), (1023, 15), (1023, 1023), (1024, 17),
          (17, 1024)]


@pytest.fixture(scope="module")
def shape_world(cuda_device):
    """Three scenarios (a car ego at yaw 0, a pedestrian ego at yaw pi/2, no ego: the view centres on the tile's bounds),
    all viewed from the origin, whose participants, goal and map cross both view axes, so that every one-pixel strip
    through the view centre draws."""
    rs = np.random.default_rng(4)
    n, m = 3, 8
    o = (0.0, 0.0, 0.0)
    tile = _tile(o, [(_ring(o, -12, 0, 3, 2), [_ring(o, -12, 0, 1, 0.8)], "area"), (_ring(o, 0, 12, 2, 3), [], "building")],
                 [((-3000, 5, 3000, 5), "roadline"), ((5, -3000, 5, 3000), "curbstone"), ((-6, -7, -2, -3), "roadline"),
                  ((2, -10, 3.5, -15), "curbstone")], bounds=(-60.0, 60.0, -50.0, 50.0))
    x, y, h = (np.zeros((n, m), np.float32) for _ in range(3))
    types = np.full((n, m), EMPTY, np.uint8)
    for k in range(n):
        j = rs.uniform(-0.7, 0.7, (m, 2))
        pts = [(0, 0), (8, 0), (0, 8), (-8, 0), (0, -8), (15, 0), (0, -15), (-15, 0)]
        x[k] = [p[0] + j[i, 0] * (i > 0) for i, p in enumerate(pts)]
        y[k] = [p[1] + j[i, 1] * (i > 0) for i, p in enumerate(pts)]
        h[k] = rs.uniform(-np.pi, np.pi, m)
        types[k] = [(VEH, PED, EMPTY)[k], VEH, CYC, PED, VEH, OBS, CYC, VEH]
    x[:, 0], y[:, 0], h[:, 0] = 0.0, 0.0, [0.0, np.pi / 2, 0.0]
    target = np.asarray([[-4, -3, 0.1, 2.5, 1.2], [3, 2, 0.3, 2.5, 1.2], [-2, 3, -0.2, 2.5, 1.2]], np.float32)
    w = _world(n, m, x, y, h, types, [tile], None, target)
    yield w, tile, target
    w.close()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{a}x{b}" for a, b in SHAPES])
def test_image_shapes_with_short_and_unaligned_runs(shape_world, shape):
    w, tile, target = shape_world
    width, height = shape
    p = 40.0 / max(width, height)          # the long side spans 40 m: thin strips through the view centre
    rng = (width * p / 2, width * p / 2, height * p / 2, height * p / 2)
    got = _check(w, shape, rng, [tile] * w.N, target)
    if width * height > 1:
        assert all(len(np.unique(got[n])) >= 3 for n in range(w.N)), [np.unique(g) for g in got]


# ---------------------------------------------------------------------------------------------------- views and maps
def _participants_around(rs, centres, m):
    """Slot 0 at the first centre, then participants of every drawn kind scattered around each centre in turn."""
    n = len(centres)
    x, y, h = np.zeros((n, m), np.float32), np.zeros((n, m), np.float32), rs.uniform(-3, 3, (n, m)).astype(np.float32)
    types = np.tile(np.asarray([(VEH, CYC, PED, OBS)[j % 4] for j in range(m)], np.uint8), (n, 1))
    for k, (cx, cy) in enumerate(centres):
        x[k], y[k] = cx + rs.uniform(-15, 15, m), cy + rs.uniform(-12, 12, m)
        x[k, 0], y[k, 0] = cx + 1.5, cy - 1.0
    return x, y, h, types


@pytest.mark.gpu
def test_views_without_an_ego_and_tiles_without_bounds_or_segments(cuda_device):
    rs = np.random.default_rng(8)
    a, b = (40.0, -10.0, 0.0), (0.0, 0.0, 0.0)
    tiles = [_tile(a, [(_ring(a, -6, 4, 4, 3), [_ring(a, -6, 4, 1.5, 1)], "area")],
                   [((-15, -8, 12, -6), "roadline"), ((3, 2, 9, 9), "curbstone")], bounds=(20.0, 60.0, -30.0, 10.0)),
             _tile(b, [(_ring(b, 7, -5, 3, 3), [], "building")], [((-12, 6, 10, 7), "roadline")]),
             dict(segments=None, poly_start=None, bounds=(-70.0, -30.0, 20.0, 40.0), style=None),
             dict(segments=None, poly_start=None, bounds=None, style=None)]
    tiles[1]["style"] = None   # default ring and open styles on this tile, given ones on tile 0
    tid = np.asarray([0, 1, 2, 3, 2, 0])
    ego = [False, False, False, False, True, True]
    centres = [(40.0, -10.0), (0.0, 0.0), (-50.0, 30.0), (0.0, 0.0), (-45.0, 28.0), (35.0, -5.0)]
    x, y, h, types = _participants_around(rs, centres, 12)
    types[~np.asarray(ego), 0] = EMPTY
    types[5, 0] = PED
    w = _world(6, 12, x, y, h, types, tiles, tid)
    for res, rng in (((160, 120), (20.0, 20.0, 20.0, 20.0)), ((96, 128), (10.0, 30.0, 25.0, 5.0))):
        got = _check(w, res, rng, [tiles[t] for t in tid])
        assert all(len(np.unique(g)) >= 3 for g in got)
    w.close()


@pytest.mark.gpu
def test_world_without_a_map_before_and_after_one(cuda_device):
    rs = np.random.default_rng(9)
    x, y, h, types = _participants_around(rs, [(0.0, 0.0), (3.0, -2.0)], 10)
    types[0, 0] = EMPTY   # no ego and no map: the view sits at the origin
    w = _world(2, 10, x, y, h, types)
    res, rng = (120, 90), (18.0, 18.0, 18.0, 18.0)
    o = (0.0, 0.0, 0.0)
    tile = _tile(o, [(_ring(o, 5, 5, 3, 2), [], "building")], [((-10, -4, 8, -3), "curbstone")], bounds=(-8.0, 30.0, -6.0, 2.0))
    _check(w, res, rng)
    w.set_map(tile["segments"], tile["bounds"], poly_start=tile["poly_start"], style=tile["style"])
    with_map = _check(w, res, rng, [tile] * 2)   # no ego: the bounds centre (11, -2)
    w.set_map(None)
    without = _check(w, res, rng)
    assert not np.array_equal(with_map[0], without[0])
    w.close()


@pytest.mark.gpu
def test_set_map_equals_a_one_tile_map_table(cuda_device):
    import torch

    rs = np.random.default_rng(10)
    o = (5.0, -3.0, 0.4)
    tile = _tile(o, [(_ring(o, -8, 2, 4, 3), [_ring(o, -8, 2, 2, 1)], "area"), (_ring(o, 6, -6, 2, 2), [], "vegetation")],
                 [((-12, -8, 12, -9), "roadline"), ((2, 3, 9, 10), "curbstone")], bounds=(-20.0, 30.0, -25.0, 15.0))
    x, y, h, types = _participants_around(rs, [(5.0, -3.0), (5.0, -5.0), (0.0, 0.0)], 10)
    types[1, 0] = EMPTY   # no ego: both worlds centre on the tile's bounds
    target = np.asarray([[3, -4, 0.2, 2.5, 1.2]] * 3, np.float32)
    one = _world(3, 10, x, y, h, types, [tile], None, target)
    table = _world(3, 10, x, y, h, types, [tile], np.zeros(3, np.int64), target)
    res, rng = (100, 140), (15.0, 25.0, 20.0, 10.0)
    for rgb in (False, True):
        assert torch.equal(one.bev(res, rng, rgb=rgb), table.bev(res, rng, rgb=rgb)), rgb
    _check(table, res, rng, [tile] * 3, target)
    one.close(); table.close()


# ---------------------------------------------------------------------------------------------------- range extremes
# At 200 x 200 and range 1e5 the pitch is 1000 m and pixel centres sit at 500 + 1000 k (exact in fp64 for a view at the
# origin with yaw 0): a primitive centred on one covers that pixel and nothing else, one between centres covers none.
RANGES = [((256, 160), (0.5, 0.5, 0.5, 0.5)), ((200, 200), (1e5, 1e5, 1e5, 1e5)), ((64, 200), (0.5, 40.0, 3.0, 1.0)),
          ((200, 90), (30.0, 5.0, 2.0, 25.0))]


@pytest.fixture(scope="module")
def range_world(cuda_device):
    n, m = 3, 10
    o = (0.0, 0.0, 0.0)
    tile = _tile(o, [(_ring(o, 30500, 10500, 5, 5), [], "building"), (_ring(o, 31100, 10400, 5, 5), [], "building"),
                     (_ring(o, 0, 0, 40, 30), [], "area")],
                 [((-60505, 500, -60495, 500), "roadline"), ((-3, 0.1, 3, 0.12), "curbstone")], bounds=(-100.0, 100.0, -80.0, 80.0))
    #          ego        on a centre     between centres  on a centre        near the ego (seen at 0.5 m)
    x = np.asarray([0, 500, 700, -1500, -20500, 0.15, -0.1, 3, -6, 2], np.float32)
    y = np.asarray([0, 500, 300, 2500, -40500, 0.1, 0.05, -4, 5, 8], np.float32)
    h = np.asarray([0, 0, 0.3, 0, 0, 1.0, 0.5, 2.0, -1.0, 0.4], np.float32)
    base = np.asarray([VEH, PED, VEH, VEH, CYC, VEH, PED, CYC, VEH, OBS], np.uint8)
    types = np.tile(base, (n, 1))
    types[1, 0], types[2, 0] = PED, EMPTY
    target = np.asarray([[0.1, -0.1, 0.2, 1.0, 0.8]] * n, np.float32)
    w = _world(n, m, np.tile(x, (n, 1)), np.tile(y, (n, 1)), np.tile(h, (n, 1)), types, [tile], None, target)
    yield w, tile, target
    w.close()


@pytest.mark.gpu
@pytest.mark.parametrize("res,rng", RANGES, ids=["0.5m", "1e5m", "asym-64x200", "asym-200x90"])
def test_range_extremes(range_world, res, rng):
    w, tile, target = range_world
    got = _check(w, res, rng, [tile] * w.N, target)
    idx = _styles(w)[0]
    if rng[0] == 0.5 and rng[1] == 0.5:
        assert (got[0] != 0).all()   # the ego's body and arrow cover the whole image
    if rng[0] == 1e5:   # every view is at the origin with yaw 0
        for k in range(w.N):
            cells = lambda style: {tuple(int(v) for v in p) for p in np.argwhere(got[k] == idx[style])}   # noqa: E731
            assert cells("pedestrian") == {(99, 100)}                  # slot 1 at (500, 500): one pixel
            assert cells("heading_arrow") == {(97, 98), (140, 79)}     # slots 3, 4: a centre on the arrow's base edge
            assert not cells("vehicle") and cells("building") == {(89, 130)}   # slot 2 and ring 1 lie between centres
