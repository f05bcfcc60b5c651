"""Float64 NumPy restatement of the BEV observation (DESIGN.md section 1, "BEV observation") - TEST ONLY.

PARITY UNPINNED: matplotlib is not available to render the reference's image, and the reference's renderer draws
participants at a wrong place anyway (it applies each pose a second time, matplotlib_renderer.py:683-690 with
sensor/camera.py:264,279-281).  This module restates the contract: pixel centre -> world, then every primitive in
descending (z, draw index) order with the coverage formulas of ``t2d_bev.cuh``, evaluated in float64 with one rounding
per operation, so that the device's class image must match it bit for bit.
"""

from __future__ import annotations

import numpy as np

NOT_DRAWN = 255
ARROW = 1
SHAPE_OBB, SHAPE_CIRCLE = 0, 1
PARTICIPANT_DRAW_BASE = 1 + 32767


def window(width, height, rng):
    """(xmin, ymax, pitch_x, pitch_y) of the view window: matplotlib_renderer.py:152-164 and auto_scale :200-224."""
    left, right, front, back = (float(np.float32(v)) for v in rng)
    x_min, x_max, y_min, y_max = -left, right, -back, front
    ww, wh = x_max - x_min, y_max - y_min
    cx, cy = (x_min + x_max) / 2, (y_min + y_max) / 2
    aspect = float(height) / float(width)
    if wh / ww > aspect:
        nw, nh = wh / aspect, wh
    else:
        nw, nh = ww, ww * aspect
    x0, x1, y0, y1 = cx - nw / 2, cx + nw / 2, cy - nh / 2, cy + nh / 2
    return x0, y1, (x1 - x0) / width, (y1 - y0) / height


def stroke_hw2(line_width_pt, pitch_x):
    hw = float(np.float32(line_width_pt)) * 200.0 / 72.0 / 2.0 * pitch_x
    return hw * hw


def pixel_centres(view, win, width, height):
    ex, ey, cs, sn = view
    xmin, ymax, px, py = win
    r, c = np.meshgrid(np.arange(height, dtype=np.float64), np.arange(width, dtype=np.float64), indexing="ij")
    u = xmin + (c + 0.5) * px
    q = ymax - (r + 0.5) * py
    return ex + cs * u - sn * q, ey + sn * u + cs * q


# ---- coverage predicates, in the operation order of t2d_bev.cuh
def ray_crosses(x1, y1, x2, y2, px, py):
    c = (x2 - x1) * (py - y1) - (y2 - y1) * (px - x1)
    return ((y1 > py) != (y2 > py)) & np.where(y2 > y1, c > 0.0, c < 0.0)


def near_segment(x1, y1, x2, y2, px, py, hw2):
    dx, dy, ux, uy = x2 - x1, y2 - y1, px - x1, py - y1
    t = ux * dx + uy * dy
    dd = dx * dx + dy * dy
    vx, vy = px - x2, py - y2
    c = dx * uy - dy * ux
    return np.where(t <= 0.0, ux * ux + uy * uy <= hw2,
                    np.where(t >= dd, vx * vx + vy * vy <= hw2, c * c <= hw2 * dd))


def in_disc(cx, cy, r2, px, py):
    ux, uy = px - cx, py - cy
    return ux * ux + uy * uy <= r2


def in_edges(edges, px, py):
    """Closed even-odd region of a set of edges [(x1, y1, x2, y2)]: inside by parity, or on an edge."""
    inside = np.zeros(px.shape, bool)
    on = np.zeros(px.shape, bool)
    for x1, y1, x2, y2 in edges:
        on |= near_segment(x1, y1, x2, y2, px, py, 0.0)
        inside ^= ray_crosses(x1, y1, x2, y2, px, py)
    return inside | on


def ring_edges(vx, vy):
    n = len(vx)
    return [(vx[i], vy[i], vx[(i + 1) % n], vy[(i + 1) % n]) for i in range(n)]


def box_ring(x, y, h, l, w):
    c, s = np.cos(h), np.sin(h)
    lx, ly = (l, l, -l, -l), (-w, w, w, -w)
    return [x + lx[i] * c - ly[i] * s for i in range(4)], [y + lx[i] * s + ly[i] * c for i in range(4)]


def arrow(rx, ry):
    a, b = (0, 1, 3), (1, 2, 0)
    return [(rx[a[i]] + rx[b[i]]) * 0.5 for i in range(3)], [(ry[a[i]] + ry[b[i]]) * 0.5 for i in range(3)]


def primitives(x, y, h, type_id, table, type_style, z, lw, pitch_x, segments=None, poly_start=None, seg_style=None,
               target=None, target_style=NOT_DRAWN, ring_style=2, open_style=3):
    """The draw list of one scenario: [(key, style, cover(px, py) -> bool array)].  x, y, h, type_id: [M] (float32
    values); table: ``TypeTable.as_oracle_table()``; type_style [n_types]; z / lw: per style; segments float32 [S, 4]."""
    f = lambda v: float(np.float32(v))   # noqa: E731  (device values are float32)
    out = []

    def add(draw, style, cover):
        out.append(((int(z[style]) + 128) << 24 | draw, style, cover))

    if target is not None and target_style != NOT_DRAWN:
        rx, ry = box_ring(f(target[0]), f(target[1]), f(target[2]), f(target[3]), f(target[4]))
        add(0, target_style, lambda px, py, e=ring_edges(rx, ry): in_edges(e, px, py))
    seg = np.zeros((0, 4)) if segments is None else np.asarray(segments, np.float32).astype(np.float64)
    ps = [] if poly_start is None or len(poly_start) < 2 else [int(v) for v in poly_start]
    style_of = (lambda s, d: d) if seg_style is None else (lambda s, d: int(seg_style[s]))
    for p in range(len(ps) - 1):
        st = style_of(ps[p], ring_style)
        if st != NOT_DRAWN:
            e = [tuple(seg[i]) for i in range(ps[p], ps[p + 1])]
            add(1 + ps[p], st, lambda px, py, e=e: in_edges(e, px, py))
    for s in range(len(seg)):
        if ps and ps[0] <= s < ps[-1]:
            continue
        st = style_of(s, open_style)
        if st != NOT_DRAWN:
            hw2 = stroke_hw2(lw[st], pitch_x)
            add(1 + s, st, lambda px, py, g=tuple(seg[s]), hw2=hw2: near_segment(*g, px, py, hw2))
    for j in range(len(type_id)):
        t = int(type_id[j])
        if t >= len(type_style) or type_style[t] == NOT_DRAWN:
            continue
        st = int(type_style[t])
        if table["shape"][t] == SHAPE_CIRCLE:
            r = table["radius"][t]
            add(PARTICIPANT_DRAW_BASE + 2 * j, st, lambda px, py, c=(f(x[j]), f(y[j]), r * r): in_disc(*c, px, py))
        elif table["shape"][t] == SHAPE_OBB:
            rx, ry = box_ring(f(x[j]), f(y[j]), f(h[j]), table["half_len"][t], table["half_wid"][t])
            ax, ay = arrow(rx, ry)
            add(PARTICIPANT_DRAW_BASE + 2 * j, st, lambda px, py, e=ring_edges(rx, ry): in_edges(e, px, py))
            add(PARTICIPANT_DRAW_BASE + 2 * j + 1, ARROW, lambda px, py, e=ring_edges(ax, ay): in_edges(e, px, py))
    return out


def view_of(x0, y0, h0, ego_active, bounds=None):
    """(ex, ey, cos, sin) of the view: the ego, or (sensor_base.py:185-191) the bounds box centre / origin, yaw 0."""
    if ego_active:
        h = float(np.float32(h0))
        return float(np.float32(x0)), float(np.float32(y0)), np.cos(h), np.sin(h)
    if bounds is not None:
        b = [float(np.float32(v)) for v in bounds]
        return (b[0] + b[1]) * 0.5, (b[2] + b[3]) * 0.5, 1.0, 0.0
    return 0.0, 0.0, 1.0, 0.0


def render(prims, view, width, height, rng):
    """Style index image uint8 [H, W] of one scenario."""
    win = window(width, height, rng)
    X, Y = pixel_centres(view, win, width, height)
    img = np.zeros((height, width), np.uint8)
    free = np.ones((height, width), bool)
    for key, style, cover in sorted(prims, key=lambda p: -p[0]):
        if not free.any():
            break
        hit = free & cover(X, Y)
        img[hit] = style
        free &= ~hit
    return img


def render_world_scenario(n, state, type_id, table, type_style, z, lw, width, height, rng, tile=None, seg_style=None,
                          target=None, target_style=NOT_DRAWN):
    """Scenario n of a world: state = dict of [N, M] arrays x, y, heading; tile = dict(segments, poly_start, bounds)."""
    tile = tile or {}
    active = int(type_id[n, 0]) < len(type_style)
    view = view_of(state["x"][n, 0], state["y"][n, 0], state["heading"][n, 0], active, tile.get("bounds"))
    win = window(width, height, rng)
    prims = primitives(state["x"][n], state["y"][n], state["heading"][n], type_id[n], table, type_style, z, lw, win[2],
                       tile.get("segments"), tile.get("poly_start"), seg_style,
                       None if target is None else target[n], target_style)
    return render(prims, view, width, height, rng)
