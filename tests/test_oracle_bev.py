"""Known answers of the float64 BEV oracle (tests/bev_oracle.py), each item of the contract on its own, and its polygon
membership against two independent implementations (OpenCV's pointPolygonTest and sympy.geometry)."""

import numpy as np

from tests import bev_oracle as B

# a small style table: 0 background, 1 arrow, 2 ring, 3 open, 4 body, 5 disc, 6 target, 7 area, 8 low ring
Z = [-128, 7, 5, 4, 6, 6, 1, 2, 1]
LW = [1.0] * 9
BODY, DISC, TARGET, AREA = 4, 5, 6, 7


def _table(hl=1.0, hw=0.5, radius=0.5):
    return dict(shape=np.array([0, 1, 2]), half_len=np.array([hl, 0.0, 0.0]), half_wid=np.array([hw, 0.0, 0.0]),
                radius=np.array([0.0, radius, 0.0]))


def _render(parts, width=256, height=256, rng=(16, 16, 16, 16), view=(0.0, 0.0, 1.0, 0.0), **kw):
    """parts: list of (x, y, h, type); type 0 box, 1 disc, 2 SHAPE_NONE."""
    x = [p[0] for p in parts]; y = [p[1] for p in parts]; h = [p[2] for p in parts]; t = [p[3] for p in parts]
    win = B.window(width, height, rng)
    ts = kw.pop("type_style", [BODY, DISC, BODY])
    prims = B.primitives(x, y, h, t, kw.pop("table", _table()), ts, Z, LW, win[2], **kw)
    return B.render(prims, view, width, height, rng)


def _centre(r, c, width=256, height=256, rng=(16, 16, 16, 16)):
    xmin, ymax, px, py = B.window(width, height, rng)
    return xmin + (c + 0.5) * px, ymax - (r + 0.5) * py


def _cells(img, style):
    return {(int(r), int(c)) for r, c in zip(*np.nonzero(img == style))}


def test_box_and_disc_pixel_sets_with_centres_on_edges():
    # pitch 0.125: a box of half extents (0.9375, 0.4375) at a pixel corner has its edges on centre lines
    img = _render([(4.0, -4.0, 0.0, 0)], type_style=[BODY, DISC, BODY])
    body = _cells(img, BODY) | _cells(img, 1)
    xs = [x for x in np.arange(256) if abs(_centre(0, x)[0] - 4.0) <= 0.9375]
    ys = [r for r in np.arange(256) if abs(_centre(r, 0)[1] + 4.0) <= 0.4375]
    assert body == {(r, c) for r in ys for c in xs}
    assert len(xs) == 16 and len(ys) == 8     # centres exactly on the edges are counted
    # a disc of radius 0.625 about a pixel centre holds the centres at offsets (0.375, 0.5) on its rim
    cx, cy = _centre(100, 60)
    img = _render([(cx, cy, 0.0, 1)], table=_table(radius=0.625))
    disc = _cells(img, DISC)
    expect = {(r, c) for r in range(90, 111) for c in range(50, 71)
              if (_centre(r, c)[0] - cx) ** 2 + (_centre(r, c)[1] - cy) ** 2 <= 0.625 ** 2}
    assert disc == expect and (96, 63) in disc and (96, 64) not in disc


def test_arrow_over_body_points_along_heading_and_ego_faces_plus_x():
    img = _render([(0.0, 0.0, 0.0, 0)])
    arrow = _cells(img, 1)
    assert arrow and all(_centre(r, c)[0] >= 0.0 for r, c in arrow)   # the triangle lies in the front half
    # rotated ego view: a car heading 0.7 rad seen from itself renders as the heading-0 car
    h = 0.7
    v = (0.0, 0.0, np.cos(np.float32(h)), np.sin(np.float32(h)))
    rot = _render([(0.0, 0.0, h, 0)], view=v)
    assert np.mean(rot == img) > 0.999


def test_target_under_areas_and_equal_z_insertion_order():
    seg = np.array([[-2, -2, 2, -2], [2, -2, 2, 2], [2, 2, -2, 2], [-2, 2, -2, -2]], np.float32)
    img = _render([], segments=seg, poly_start=[0, 4], seg_style=[AREA] * 4, target=[0, 0, 0, 3, 3], target_style=TARGET)
    assert TARGET in img and AREA in img and img[128, 128] == AREA    # z 1 target beneath the z 2 area
    # two boxes at equal z: the later slot is drawn on top
    img = _render([(0.0, 0.0, 0.0, 0), (0.5, 0.0, 0.0, 0)], type_style=[BODY, DISC, BODY])
    r, c = 128, 128 + 8          # x = 1.0625 lies in both bodies; the second's arrow is further right
    assert img[r, c] in (BODY, 1)
    prims = B.primitives([0.0, 0.5], [0.0, 0.0], [0.0, 0.0], [0, 0], _table(), [BODY, DISC, BODY], Z, LW, 0.125)
    keys = sorted(prims, key=lambda p: -p[0])
    assert [p[0] & 0xFFFFFF for p in keys][:2] == [B.PARTICIPANT_DRAW_BASE + 3, B.PARTICIPANT_DRAW_BASE + 1]


def test_stroke_width_in_pixels():
    seg = np.array([[-10, 0.0625, 10, 0.0625]], np.float32)   # along a row of centres
    img = _render([], segments=seg)
    col = img[:, 128]
    rows = np.nonzero(col == 3)[0]
    # 1 pt at 200 dpi = 2.78 px wide: the centres within 1.39 px = 0.1736 m of the line, i.e. 3 rows
    assert len(rows) == 3 and set(rows) == {126, 127, 128}
    lw05 = B.primitives([], [], [], [], _table(), [], Z, [1.0, 1.0, 1.0, 0.5], 0.125, segments=seg)
    hw2 = B.stroke_hw2(0.5, 0.125)
    assert abs(np.sqrt(hw2) - 0.5 * 200 / 72 / 2 * 0.125) < 1e-15 and len(lw05) == 1


def test_even_odd_fill_of_area_with_two_holes():
    from tactics2d_b200.map import load_areas, polygons_to_segments

    a = load_areas("inD_2")[1]
    assert len(a.inners) == 2
    seg, ps = polygons_to_segments([a])
    c = a.inners[0].mean(0)
    view = (float(c[0]), float(c[1]), 1.0, 0.0)
    img = _render([], view=view, rng=(40, 40, 40, 40), segments=seg, poly_start=ps, seg_style=[AREA] * len(seg))
    import cv2

    xmin, ymax, px, py = B.window(256, 256, (40, 40, 40, 40))
    outer = a.outer.astype(np.float32); holes = [h.astype(np.float32) for h in a.inners]
    for r in range(0, 256, 5):
        for cc in range(0, 256, 5):
            X = view[0] + (xmin + (cc + 0.5) * px); Y = view[1] + (ymax - (r + 0.5) * py)
            d_out = cv2.pointPolygonTest(outer.reshape(-1, 1, 2), (X, Y), True)
            d_h = [cv2.pointPolygonTest(h.reshape(-1, 1, 2), (X, Y), True) for h in holes]
            if min([abs(d_out)] + [abs(d) for d in d_h]) < 1e-3:
                continue
            inside = d_out > 0 and all(d < 0 for d in d_h)
            assert (img[r, cc] == AREA) == inside, (r, cc)
    assert (img == 0).any() and (img == AREA).any()


def test_aspect_widening_for_asymmetric_ranges_and_non_square_images():
    xmin, ymax, px, py = B.window(200, 100, (10, 30, 5, 5))     # 40 x 10 m into 2:1 -> 40 x 20 about (10, 0)
    assert (xmin, ymax, px, py) == (-10.0, 10.0, 0.2, 0.2)
    xmin, ymax, px, py = B.window(100, 200, (10, 30, 5, 5))     # 40 x 10 into 1:2 -> 40 x 80 about (10, 0)
    assert (xmin, ymax) == (-10.0, 40.0) and px == py == 0.4
    xmin, ymax, px, py = B.window(200, 200, (20, 20, 30, 10))   # front 30 / back 10: the literal y window [-10, 30]
    assert (xmin, ymax) == (-20.0, 30.0)


def test_inactive_ego_view_and_undrawn_types():
    assert B.view_of(5.0, 5.0, 1.0, False, (0.0, 10.0, -4.0, 2.0)) == (5.0, -1.0, 1.0, 0.0)
    assert B.view_of(5.0, 5.0, 1.0, False, None) == (0.0, 0.0, 1.0, 0.0)
    # SHAPE_NONE and a type styled NOT_DRAWN (an obstacle) produce no primitive
    prims = B.primitives([0.0, 1.0], [0.0, 1.0], [0.0, 0.0], [2, 0], _table(), [B.NOT_DRAWN, DISC, BODY], Z, LW, 0.125)
    assert prims == []


def test_polygon_membership_against_opencv_and_sympy():
    import cv2
    import sympy

    rng = np.random.default_rng(0)
    for trial in range(6):
        k = int(rng.integers(3, 9))
        ang = np.sort(rng.uniform(0, 2 * np.pi, k))
        rad = rng.uniform(2, 8, k)
        poly = np.stack([rad * np.cos(ang), rad * np.sin(ang)], 1).astype(np.float32)   # star-shaped, maybe concave
        edges = B.ring_edges(list(poly[:, 0].astype(np.float64)), list(poly[:, 1].astype(np.float64)))
        pts = rng.uniform(-9, 9, (400, 2))
        got = B.in_edges(edges, pts[:, 0], pts[:, 1])
        for (x, y), g in zip(pts, got):
            d = cv2.pointPolygonTest(poly.reshape(-1, 1, 2), (float(x), float(y)), True)
            if abs(d) > 1e-9:
                assert g == (d > 0)
        sp = sympy.Polygon(*[sympy.Point(sympy.Rational(float(a)), sympy.Rational(float(b))) for a, b in poly])
        for (x, y), g in list(zip(pts, got))[:25]:
            p = sympy.Point(sympy.Rational(float(x)), sympy.Rational(float(y)))
            if float(sp.distance(p)) > 1e-9:
                assert g == bool(sp.encloses_point(p))
