"""Every instance of the fused tick on its rare paths, against the float64 oracle.

The tick (``t2d_step_kernel<KIN_ONLY, MAP_TABLE, FIXED>``) is compiled as six instances and the host picks one per tick:
fp64 models compiled in or not (a property of the type table), one map tile or a table of tiles, and the instance compiled
for M = 64.  A tick also branches at run time: the one-tile map staged in shared memory or read from global memory (a
blob over 120 KB), vector or scalar loads (M % 4), and one wave of warp tiles or several, where a warp reuses its shared
queue, queue counter and hit minima from one tile to the next.  test_gpu_rare_paths.py forces each rare path in the one
instance its scene selects; here every scene runs in every instance it can reach, and on the runtime axes:

    S1  pair-queue overflow (exhaustive pass), M = 32, 64, 128
    S2  exact-queue overflow (out-of-line exact walk), touching segments only / with a decisive crossing segment
    S3  reach beyond the map's dilation: 1 m cells / the type table replaced after the map
    S4  the edges of the clearance field
    S5  the inD_2 walkway with two holes (containment)
    S6  out of bound at the box edge: extents exactly on each side, 1 ulp inside and outside, around |x| = 1 and 1e4
    S7  exact-queue overflow across two tiles inside one warp (map table only)

Scalar loads take M = 1, 2, 3 (mod 4): empty slots are added, except to the scenes built to overflow the exact queue
(S2), which is trimmed to 61 .. 63 slots so that a warp still holds two scenarios and more undecided pairs than the
queue has entries.

In the two-tile form the scenarios alternate between the scene's tile and a second one that holds the same segments in
reverse order (S5: the same areas in reverse order; S6: another boundary box), so a lane that reads another scenario's
tile finds other segments at the indices it resolves.

Every tick checks flags, hit_index, hit_segment, status and done bit for bit against ``oracle.scenario`` and the state
within 1e-5 (in still scenes x, y and heading bit-unchanged).  The outputs are filled with a sentinel first: the kernel
writes flags, hit_index and hit_segment at every slot of every scenario (empty slots included) and status and done of
every scenario, so no sentinel may be left.  ``t2d_tick_instance_count`` must show that exactly the intended instance
ran, and whether the map was read from global memory.  Within one scene and map form all instances give the same outputs.
"""

import dataclasses
import functools
import os

import numpy as np
import pytest

from oracle import scenario as O
from tests.test_gpu_rare_paths import EXACT_QUEUE, QCAP, _bus_scene, _clearance_scene, _rbound, _tables, _touch_table

INSTANCES = {"kin": 2, "kin_table": 3, "fp64": 0, "fp64_table": 1, "fixed": 4, "fixed_table": 5}   # t2d_tick_instance_count(k)
GLOBAL_MAP = 6          # t2d_tick_instance_count(6): one-tile ticks that read the map from global memory
RESIDENT_WARPS = 16     # per SM at most, at K1's 128 registers per thread: more warp tiles than 16 x SMs take several waves
OUTPUTS = ("flags", "hit_index", "hit_segment", "status", "done")
SENTINEL = {"flags": 0xA5, "hit_index": 0x5A5A, "hit_segment": 0x5A5A, "status": 0xA5, "done": 0xA5}   # never a value


@dataclasses.dataclass
class Scene:
    table: object               # the TypeTable the world ticks with
    x: np.ndarray               # [N, M] fp32, as y, h, v
    y: np.ndarray
    h: np.ndarray
    v: np.ndarray
    tid: np.ndarray             # [N, M] uint8
    tiles: list                 # dict(segments, bounds, poly_start): one tile, or two with tile_id
    acts: list                  # [N, M, 2] action of every tick
    tile_id: np.ndarray = None  # [N] with two tiles
    cell_size: float = 0.0
    map_table: object = None    # the table the map is built for, when the world then ticks with another one (S3)
    rare: np.ndarray = None     # [N] scenarios that take the rare path; the others are sparse
    check: object = None        # check(fl, hi, hs, on0): what the scene is built to show; on0 = scenarios on tile 0
    m_real: int = 0             # participant slots of the scene; slots above it are empty padding
    exact_overflow: bool = False   # every slot of a rare scenario has one undecided (box, segment) pair, and a warp of rare
                                   # scenarios must hold more of them than the exact queue does (S2, S7)


def _group(m):
    """Lanes per scenario (t2d_create): the least power of two that holds m participants at 4 per lane."""
    g = 1
    while 4 * g < m:
        g *= 2
    return g


def _tile(segments=None, bounds=None, poly_start=None):
    seg = None if segments is None else np.ascontiguousarray(segments, dtype=np.float32)
    return dict(segments=seg, bounds=bounds, poly_start=poly_start)


def _scene(table, x, y, h, v, tid, tiles, acts=None, **kw):
    f = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    n, m = np.shape(x)
    acts = acts if acts is not None else [np.zeros((n, m, 2), np.float32)]
    return Scene(table, f(x), f(y), f(h), f(v), np.ascontiguousarray(tid, dtype=np.uint8), tiles, acts, m_real=m, **kw)


def _reversed_tile(sc):
    """The two-tile form: tile 1 holds tile 0's segments in reverse order, and the scenarios alternate between them."""
    t = sc.tiles[0]
    return dataclasses.replace(sc, tiles=[t, dict(t, segments=np.ascontiguousarray(t["segments"][::-1]))],
                               tile_id=np.arange(sc.x.shape[0]) % 2)


# ------------------------------------------------------------------------------------------------ scenes
@functools.lru_cache(None)
def _s1(m):
    """Pair-queue overflow: the first scenario of every other warp is a crowd of M vehicles inside a disc of radius 2 m (all
    M (M - 1) / 2 pairs are candidates, against 192 queue entries per warp); the others are C2 arena scenarios, whose pairs
    the exhaustive pass of a crowded warp resolves as well."""
    from tactics2d_b200 import synthetic

    n = 16
    sc = synthetic.config2(n, m, seed=70 + m, size=60.0)
    dense = np.arange(n) % (2 * (32 // _group(m))) == 0
    rng = np.random.default_rng(m)
    rad, ang = 2.0 * np.sqrt(rng.uniform(0, 1, (n, m))), rng.uniform(0, 2 * np.pi, (n, m))
    x = np.where(dense[:, None], 30.0 + rad * np.cos(ang), sc.x)
    y = np.where(dense[:, None], 30.0 + rad * np.sin(ang), sc.y)
    reach = _rbound(sc.table)[sc.type_id] + _rbound(sc.table).max()
    for s in np.flatnonzero(dense):
        d2 = (x[s, :, None] - x[s, None, :]) ** 2 + (y[s, :, None] - y[s, None, :]) ** 2
        assert np.triu(d2 <= reach[s, :, None] ** 2, 1).sum() > QCAP

    def check(fl, hi, hs, on0):
        for s in np.flatnonzero(dense & on0):
            assert (fl[s] & 1).all() and len(np.unique(hi[s])) > 1, s      # everybody in the crowd hits, not all one partner
        sparse = fl[~dense] & 1
        assert sparse.any() and not sparse.all()                           # the arena scenarios: some collisions, not all

    acts = [synthetic.random_actions(80 + t, (n, m)) for t in range(2)]
    return _scene(sc.table, x, y, sc.heading, sc.speed, sc.type_id, [_tile(sc.segments, sc.bounds)], acts, rare=dense, check=check)


def _touching(k):
    """Box k of a lattice of 2 x 1 m boxes at heading 0, centres on whole metres 12 m apart, and a segment that touches it
    exactly (k % 3: along its top edge, ending on its right edge, meeting its corner): the fp32 filter's margin is exactly
    0, so the pair is undecided and queued for the exact test.  Returns centres [K] and segments [K, 4]."""
    cx, cy = 12.0 * (k % 8), 12.0 * (k // 8)
    cand = np.stack([np.stack([cx - 1, cy + 1, cx + 1, cy + 1], 1), np.stack([cx + 2, cy - 0.5, cx + 4, cy + 0.5], 1),
                     np.stack([cx + 2, cy + 1, cx + 3, cy + 2], 1)])
    return cx, cy, np.ascontiguousarray(cand[k % 3, np.arange(len(k))], dtype=np.float32)


BOX_BOUNDS = (-10.0, 100.0, -10.0, 100.0)


@functools.lru_cache(None)
def _s2(decisive):
    """Exact-queue overflow: two warps of two scenarios of 64 touching boxes each (128 undecided pairs per warp against 64
    exact-queue entries), then two warps whose boxes sit 6 m off every segment.  ``decisive``: every box is also crossed by
    a segment through its centre at a higher index, a decided hit that ends the walk; the touching segment still wins."""
    m, n = 64, 8
    k = np.arange(m)
    cx, cy, seg = _touching(k)
    if decisive:
        seg = np.concatenate([seg, np.stack([cx - 3, cy, cx + 3, cy], 1).astype(np.float32)])
    rare = np.arange(n) < 4
    x = np.where(rare[:, None], cx, cx + 6.0)
    y = np.where(rare[:, None], cy, cy + 6.0)
    z = np.zeros((n, m))

    def check(fl, hi, hs, on0):   # (the slots may have been trimmed: box k is slot k)
        assert (hs[rare & on0] == k[:hs.shape[1]]).all() and (hs[~rare] == -1).all()

    return _scene(_touch_table(), x, y, z, z, np.zeros((n, m)), [_tile(seg, BOX_BOUNDS)], rare=rare, check=check,
                  exact_overflow=True)


@functools.lru_cache(None)
def _s3(form):
    """Buses (bounding radius 6.14 m) reach beyond the map's dilation and take the out-of-line exact walk; those parked
    left of the map have their centres outside the grid.  ``small_cells``: 1 m cells cap the dilation at 1 m;
    ``table_after_map``: the map is built for a table of cars (dilation 2.83 m) and a table with the bus replaces it."""
    small, table = _tables()
    rng = np.random.default_rng(91 if form == "small_cells" else 92)
    n, m = 64, 32
    seg, x, y, h, tid, out = _bus_scene(rng, n, m, 3)
    v = rng.uniform(0, 3, (n, m))

    def check(fl, hi, hs, on0):
        assert (hs[out & on0[:, None]] == 0).mean() > 0.9                 # the buses left of the map reach its left wall

    return _scene(table, x, y, h, v, tid, [_tile(seg, (-40.0, 70.0, -40.0, 70.0))], check=check,
                  cell_size=1.0 if form == "small_cells" else 0.0, map_table=small if form == "table_after_map" else None)


@functools.lru_cache(None)
def _s4():
    """Discs swept across walls at 45 degrees through the corners of the clearance field's fine cells, and centres on
    fine-cell boundaries and in the grid's last row and column (test_gpu_rare_paths._clearance_scene)."""
    table, seg, p, tt, n_swept = _clearance_scene()
    m = 32
    n = -(-len(p) // m)
    pad = n * m - len(p)
    p = np.concatenate([p, np.tile([[-30.0, -30.0]], (pad, 1))])
    tid = np.concatenate([tt, np.full(pad, 255)]).reshape(n, m)
    z = np.zeros((n, m))

    def check(fl, hi, hs, on0):
        if on0.all():
            assert 0.4 < ((fl.reshape(-1)[:n_swept] & 2) != 0).mean() < 0.6      # the sweep straddles contact

    return _scene(table, p[:, 0].reshape(n, m), p[:, 1].reshape(n, m), z, z, tid, [_tile(seg)], check=check)


@functools.lru_cache(None)
def _s5(table_mode):
    """The walkway of inD_2, one Area with two holes, among the map's other areas: boxes inside a hole and clear of every
    edge (free), inside the walkway and clear of every edge (hit by containment alone), and across an inner ring."""
    from oracle.geometry import point_in_ring
    from tactics2d_b200 import TypeParams, TypeTable
    from tactics2d_b200.map import load_areas, polygons_to_segments

    areas = load_areas("inD_2")
    seg, ps = polygons_to_segments(areas)
    k = next(i for i, a in enumerate(areas) if len(a.inners) == 2)
    a, s64 = areas[k], seg.astype(np.float64)
    rng = np.random.default_rng(93)
    pts = rng.uniform(a.outer.min(0), a.outer.max(0), (20000, 2))
    d = pts[:, None, :] - s64[None, :, :2]
    e = s64[None, :, 2:] - s64[None, :, :2]
    t = np.clip((d * e).sum(-1) / np.maximum((e * e).sum(-1), 1e-30), 0, 1)
    clear = np.sqrt(((d - t[..., None] * e) ** 2).sum(-1)).min(1) > 0.6       # beyond the 0.4 x 0.3 box's half diagonal
    px, py = pts[:, 0], pts[:, 1]
    in_area = [point_in_ring(px, py, s64[ps[j]:ps[j + 1]]) for j in range(len(areas))]
    lone = clear & ~np.any([in_area[j] for j in range(len(areas)) if j != k], 0)
    ring = lambda r: np.concatenate([r, np.roll(r, -1, 0)], 1)
    hole = point_in_ring(px, py, ring(a.outer)) & ~in_area[k] & lone
    inside = in_area[k] & lone
    inner = np.concatenate(list(a.inners))
    across = inner[rng.integers(0, len(inner), 64)] + rng.uniform(-0.2, 0.2, (64, 2))
    assert hole.sum() >= 16 and inside.sum() >= 64
    p = np.concatenate([pts[hole][:32], pts[inside][:64], across])
    cls = np.concatenate([np.zeros(min(32, hole.sum())), np.ones(64), np.full(64, 2)])
    m = 32
    n = -(-len(p) // m)
    pad = n * m - len(p)
    p = np.concatenate([p, np.repeat(p[:1], pad, 0)])
    cls = np.concatenate([cls, np.full(pad, -1)]).reshape(n, m)
    h = rng.uniform(0, 6.28, (n, m))                  # below fp32(2 pi): the wrapped heading is the input, so it is still
    table = TypeTable([dataclasses.replace(TypeParams.vehicle("medium_car"), half_len=0.4, half_wid=0.3)])

    def check(fl, hi, hs, on0):
        sel = on0[:, None]
        assert (hs[(cls == 0) & sel] == -1).all() and (hs[(cls == 1) & sel] == ps[k]).all() and (hs[(cls == 2) & sel] >= 0).all()

    z = np.zeros((n, m))
    sc = _scene(table, p[:, 0].reshape(n, m), p[:, 1].reshape(n, m), h, z, np.where(cls < 0, 255, 0), [_tile(seg, None, ps)], check=check)
    if table_mode:
        seg_b, ps_b = polygons_to_segments(areas[::-1])
        sc = dataclasses.replace(sc, tiles=sc.tiles + [_tile(seg_b, None, ps_b)], tile_id=np.arange(n) % 2)
    return sc


EDGE_BOXES = {"a": (-9999.5, 0.875, -0.625, 9998.25), "b": (-0.875, 9999.5, -9998.25, 0.625)}   # every value exact in fp32


def _edge_table():
    from tactics2d_b200 import TypeParams, TypeTable

    car = dataclasses.replace(TypeParams.vehicle("medium_car"), half_len=2.0, half_wid=1.0)
    return TypeTable([car, dataclasses.replace(car, radius=0.75, shape=1)])


def _edge_poses(box):
    """Forty poses against the sides of ``box``, 8 m apart along each side: per side and shape (the 2 x 1 box at heading 0,
    the disc of radius 0.75) the extent exactly on the side (inside: the box is closed), 1 ulp inside, 1 ulp outside, and
    the centre 1 ulp either side of where the clear_in shortcut's fp32 margin (bounding radius * 1.0001 + 1e-3) ends.
    Returns x, y, type ids [40] and which poses are out of bound."""
    f32 = np.float32
    xmin, xmax, ymin, ymax = (f32(b) for b in box)
    rb = _rbound(_edge_table())
    xs, ys, ts, outs = [], [], [], []
    for side, (edge, inward) in enumerate(((xmin, 1), (xmax, -1), (ymin, 1), (ymax, -1))):
        for t, ext in enumerate((2.0 if side < 2 else 1.0, 0.75)):     # half length along x, half width along y
            c = f32(float(edge) + inward * ext)
            assert float(c) - inward * ext == float(edge)                 # the extent lies exactly on the side
            step = lambda v, k: v if k == 0 else step(np.nextafter(v, f32(np.inf * np.sign(k))), k - np.sign(k))
            thr = f32(float(edge) + inward * float(f32(rb[t]) * f32(1.0001) + f32(1e-3)))
            for pos, out in ((c, False), (step(c, inward), False), (step(c, -inward), True), (step(thr, -1), False), (step(thr, 1), False)):
                along = f32(20.0 + 8.0 * (len(xs) % 10)) + (ymin if side < 2 else xmin)
                xs.append(pos if side < 2 else along)
                ys.append(along if side < 2 else pos)
                ts.append(t)
                outs.append(out)
    return np.array(xs, np.float32), np.array(ys, np.float32), np.array(ts), np.array(outs)


@functools.lru_cache(None)
def _s6(box, table_mode):
    """Out of bound at the box edge (the fp32 test's undecided band and its fp64 fallback, and the clear_in shortcut).
    Box a puts x's upper side and y's lower side near 0 and the two others near 1e4; box b the other way round.  In the
    two-tile form the scenarios alternate between the two boxes, each posed against its own box."""
    n, m = 6, 40
    boxes = [box, "b" if box == "a" else "a"] if table_mode else [box]
    tile_id = np.arange(n) % len(boxes)
    poses = [_edge_poses(EDGE_BOXES[b]) for b in boxes]
    x, y, tid, out = (np.stack([poses[i][j] for i in tile_id]) for j in range(4))
    z = np.zeros((n, m))

    def check(fl, hi, hs, on0):
        assert np.array_equal((fl & 4) != 0, out)

    tiles = [_tile(None, EDGE_BOXES[b]) for b in boxes]
    return _scene(_edge_table(), x, y, z, z, tid, tiles, check=check, tile_id=tile_id if table_mode else None)


@functools.lru_cache(None)
def _s7(m):
    """Exact-queue overflow across tiles inside one warp: the touching boxes of S2, M per scenario (one lane per scenario at
    M = 4), 128 undecided pairs per warp against 64 exact-queue entries, scenarios alternating between tile 0 and tile 1,
    which holds tile 0's segments in reverse order: box k touches segment k on tile 0 and 63 - k on tile 1.  Two warps of
    such scenarios, then two warps of boxes 6 m off every segment."""
    spw = 32 // _group(m)
    n = 4 * spw
    k = (np.arange(n)[:, None] * m + np.arange(m)) % 64
    cx, cy, seg = _touching(np.arange(64))
    rare = np.arange(n) < 2 * spw
    x = np.where(rare[:, None], cx[k], cx[k] + 6.0)
    y = np.where(rare[:, None], cy[k], cy[k] + 6.0)
    tile_id = np.arange(n) % 2
    want = np.where(rare[:, None], np.where(tile_id[:, None] == 0, k, 63 - k), -1)

    def check(fl, hi, hs, on0):
        assert np.array_equal(hs, want)

    z = np.zeros((n, m))
    tiles = [_tile(seg, BOX_BOUNDS), _tile(seg[::-1], BOX_BOUNDS)]
    return _scene(_touch_table(), x, y, z, z, np.zeros((n, m)), tiles, rare=rare, check=check, tile_id=tile_id,
                  exact_overflow=True)


SCENES = {
    "s1_m32": lambda tm: _s1(32), "s1_m64": lambda tm: _s1(64), "s1_m128": lambda tm: _s1(128),
    "s2_touch_only": lambda tm: _s2(False), "s2_with_decisive_hit": lambda tm: _s2(True),
    "s3_small_cells": lambda tm: _s3("small_cells"), "s3_table_after_map": lambda tm: _s3("table_after_map"),
    "s4_clearance_edges": lambda tm: _s4(),
    "s5_two_holes": _s5,
    "s6_box_a": lambda tm: _s6("a", tm), "s6_box_b": lambda tm: _s6("b", tm),
    "s7_m4": lambda tm: _s7(4), "s7_m16": lambda tm: _s7(16), "s7_m64": lambda tm: _s7(64),
}
SCENE_M = {"s1_m32": 32, "s1_m64": 64, "s1_m128": 128, "s2_touch_only": 64, "s2_with_decisive_hit": 64, "s3_small_cells": 32,
           "s3_table_after_map": 32, "s4_clearance_edges": 32, "s5_two_holes": 32, "s6_box_a": 40, "s6_box_b": 40, "s7_m4": 4,
           "s7_m16": 16, "s7_m64": 64}
AXES = {   # runtime axis: the scenes it runs
    "smem_map": list(SCENES),
    "global_map": ["s1_m32", "s1_m64", "s1_m128", "s2_touch_only", "s2_with_decisive_hit", "s5_two_holes", "s6_box_a", "s6_box_b"],
    "scalar_m+1": ["s2_touch_only", "s5_two_holes", "s6_box_a"],
    "scalar_m+2": ["s2_touch_only", "s5_two_holes", "s6_box_a"],
    "scalar_m+3": ["s2_touch_only", "s5_two_holes", "s6_box_a"],
    "several_waves": ["s1_m64", "s2_touch_only", "s7_m16"],
}


def _unreachable(scene, axis, instance):
    """Why ``instance`` cannot run ``scene`` on ``axis``, or None."""
    table_mode = instance.endswith("_table")
    if scene.startswith("s7") and not table_mode:
        return "S7 is about two tiles inside one warp: it needs a map table"
    if axis == "global_map" and table_mode:
        return "a map table is always read from global memory: the shared-memory / global-memory axis is one-tile only"
    if instance.startswith("fixed"):
        if axis.startswith("scalar"):
            return "FIXED is compiled for M = 64 with vector loads; scalar loads need M % 4 != 0"
        if SCENE_M[scene] > 64:
            return f"FIXED is compiled for M = 64; this scene has M = {SCENE_M[scene]}"
        if scene.startswith("s7") and SCENE_M[scene] < 64:
            return (f"padded to M = 64, S7 at M = {SCENE_M[scene]} holds 2 scenarios per warp instead of "
                    f"{32 // _group(SCENE_M[scene])}: s7_m64 covers FIXED with a map table")
    return None


def _cases():
    out = []
    for axis, scenes in AXES.items():
        for scene in scenes:
            for instance in INSTANCES:
                why = _unreachable(scene, axis, instance)
                marks = [pytest.mark.skip(reason=why)] if why else []
                out.append(pytest.param(scene, axis, instance, id=f"{scene}-{axis}-{instance}", marks=marks))
    return out


# ------------------------------------------------------------------------------------------------ instances and axes
def _with_dynamics(table):
    """``table`` plus an unused SingleTrackDynamics row, so that the fp64 models are compiled in.  The row is a copy of the
    table's row of largest bounding radius: the largest radius, and with it the map's dilation, do not change."""
    from tactics2d_b200 import TypeTable
    from tactics2d_b200.types import MODEL_DYNAMICS

    big = table.rows[int(np.argmax(_rbound(table)))]
    return TypeTable(table.rows + [dataclasses.replace(big, model=MODEL_DYNAMICS, name="unused dynamics")])


def _pad_slots(sc, k):
    """``k`` empty slots (type 255, zero action) appended to every scenario."""
    if k == 0:
        return sc
    n = sc.x.shape[0]
    pad = lambda a, v: np.concatenate([a, np.full((n, k) + a.shape[2:], v, a.dtype)], 1)
    return dataclasses.replace(sc, x=pad(sc.x, 0), y=pad(sc.y, 0), h=pad(sc.h, 0), v=pad(sc.v, 0), tid=pad(sc.tid, 255),
                               acts=[pad(a, 0) for a in sc.acts])


def _trim_slots(sc, k):
    """The scene without its last ``k`` participant slots."""
    m = sc.x.shape[1] - k
    return dataclasses.replace(sc, x=sc.x[:, :m].copy(), y=sc.y[:, :m].copy(), h=sc.h[:, :m].copy(), v=sc.v[:, :m].copy(),
                               tid=sc.tid[:, :m].copy(), acts=[a[:, :m].copy() for a in sc.acts], m_real=min(sc.m_real, m))


def _far_segments(sc):
    """About 6000 segments of 1 m on a 3 m lattice, 50 m beyond every participant and segment of the scene, at higher
    indices than the scene's own: the one tile's blob exceeds the 120 KB the tick stages into shared memory."""
    xs = [sc.x[sc.tid != 255]] + [t["segments"][:, [0, 2]].ravel() for t in sc.tiles if t["segments"] is not None]
    ys = [sc.y[sc.tid != 255]] + [t["segments"][:, [1, 3]].ravel() for t in sc.tiles if t["segments"] is not None]
    x0, y0 = max(float(v.max()) for v in xs) + 50.0, min(float(v.min()) for v in ys)
    i, j = np.meshgrid(np.arange(78), np.arange(78))
    px, py = (x0 + 3.0 * i).ravel(), (y0 + 3.0 * j).ravel()
    far = np.stack([px, py, px + 1.0, py], 1).astype(np.float32)
    t = sc.tiles[0]
    seg = far if t["segments"] is None else np.concatenate([t["segments"], far])
    return dataclasses.replace(sc, tiles=[dict(t, segments=seg)])


def _waves(sc, sm_count):
    """The scene's warp tiles replicated to an odd N whose warp tiles exceed 16 x the SM count, so that the persistent
    grid runs several waves.  Each replicated tile copies a tile of the scene that holds a rare scenario or one that does
    not, drawn at random tile by tile: whatever the grid's stride, many warps meet a rare tile after a sparse one, and the
    reverse.  Returns idx [N]: the scene's scenario that each replicated one copies."""
    n0, m = sc.x.shape
    spw = 32 // _group(m)
    assert n0 % spw == 0
    base = np.arange(n0 // spw)
    rare_tiles = base[sc.rare.reshape(-1, spw).any(1)]
    sparse_tiles = base[~sc.rare.reshape(-1, spw).any(1)]
    n_tiles = RESIDENT_WARPS * sm_count + 33                       # odd: N is odd also at one scenario per warp
    rng = np.random.default_rng(7)
    pick = np.where(rng.random(n_tiles) < 0.5, rng.choice(rare_tiles, n_tiles), rng.choice(sparse_tiles, n_tiles))
    idx = (pick[:, None] * spw + np.arange(spw)).reshape(-1)[: n_tiles * spw - spw + 1]     # the last tile holds one scenario
    assert len(idx) % 2 == 1 and -(-len(idx) // spw) > RESIDENT_WARPS * sm_count
    assert np.array_equal(np.unique(idx), np.arange(n0))
    return idx


def _events(sc, st, otab):
    """The oracle's events of the scene's scenarios, each on its own tile."""
    n, m = sc.x.shape
    fl, hi, hs = np.zeros((n, m), np.uint8), np.zeros((n, m), np.int16), np.zeros((n, m), np.int16)
    tile_id = np.zeros(n, int) if sc.tile_id is None else sc.tile_id
    for k, t in enumerate(sc.tiles):
        sel = tile_id == k
        n_seg = 0 if t["segments"] is None else len(t["segments"])
        chunk = int(max(1, min(64, 2 ** 21 // (m * max(m, n_seg)))))
        fl[sel], hi[sel], hs[sel] = O.events(st["x"][sel], st["y"][sel], st["heading"][sel], sc.tid[sel], otab, t["segments"],
                                             t["bounds"], chunk=chunk, poly_start=t["poly_start"])
    return fl, hi, hs


def _run(sc, instance, device, idx, global_map):
    """Ticks the scene (its scenarios replicated by ``idx``) in a world that takes ``instance``; returns the outputs of
    every tick on the scene's scenarios and participant slots."""
    import torch

    from tactics2d_b200 import BatchedWorld, _lib
    from tests.util import assert_state_close

    lib = _lib.load()
    n, m = len(idx), sc.x.shape[1]
    _, first = np.unique(idx, return_index=True)         # the replicated scenario the oracle teacher-forces from
    rep = lambda a: np.ascontiguousarray(a[idx])
    if instance.startswith("kin"):
        os.environ["T2D_TICK_GENERIC"] = "1"             # at M = 64 the kinematic instances are FIXED's otherwise
    try:
        w = BatchedWorld(n, m, sc.map_table or sc.table, device=device)
    finally:
        os.environ.pop("T2D_TICK_GENERIC", None)
    outs = []
    try:
        if sc.tile_id is not None:
            w.set_map_table(sc.tiles, rep(sc.tile_id), cell_size=sc.cell_size)
        else:
            t = sc.tiles[0]
            w.set_map(t["segments"], t["bounds"], cell_size=sc.cell_size, poly_start=t["poly_start"])
        if sc.map_table is not None:
            w.set_type_table(sc.table)
        tid = rep(sc.tid)
        w.set_state(rep(sc.x), rep(sc.y), rep(sc.h), rep(sc.v), type_id=tid)
        otab = sc.table.as_oracle_table()
        still = not sc.v.any() and not any(a.any() for a in sc.acts)
        active = tid != 255
        expect = [0] * 7
        expect[INSTANCES[instance]] = 1
        expect[GLOBAL_MAP] = int(global_map)
        o = w.result
        for t, act in enumerate(sc.acts):
            for k, v in SENTINEL.items():
                getattr(o, k).fill_(v)
            before = w.state_numpy()
            c0 = [lib.t2d_tick_instance_count(k) for k in range(7)]
            w.step(torch.from_numpy(rep(act)).to(device))
            torch.cuda.synchronize()
            moved = [lib.t2d_tick_instance_count(k) - c0[k] for k in range(7)]
            assert moved == expect, f"tick {t}: instance launches {moved}, expected {expect}"
            got = w.state_numpy()
            ref = O.physics_tick({k: v[first] for k, v in before.items()}, sc.tid, act, otab, w.interval, w.delta_t)
            assert_state_close(got, {k: v[idx] for k, v in ref.items()}, mask=active, what=f"tick {t}")
            for k in got:
                assert np.array_equal(got[k][~active], before[k][~active]), (t, k)     # empty slots keep their state
            if still:
                for k in ("x", "y", "heading"):
                    assert np.array_equal(got[k], before[k]), (t, k)
            res = {k: getattr(o, k).cpu().numpy() for k in OUTPUTS}
            for k, v in SENTINEL.items():
                left = np.argwhere(res[k] == v)
                assert len(left) == 0, f"tick {t}: {k} not written at {left[:5].tolist()}"
            fl, hi, hs = _events(sc, {k: v[first] for k, v in got.items()}, otab)
            st, done = O.status(fl, sc.tid, w.step_count.cpu().numpy()[first], w.max_step)
            for k, want in zip(OUTPUTS, (fl, hi, hs, st, done)):
                bad = np.argwhere(res[k] != want[idx])
                assert len(bad) == 0, f"tick {t}: {k} differs from the oracle at {bad[:5].tolist()}"
            if sc.check is not None:
                sc.check(fl[:, :sc.m_real], hi[:, :sc.m_real], hs[:, :sc.m_real],
                         np.ones(len(first), bool) if sc.tile_id is None else sc.tile_id == 0)
            outs.append({k: res[k][first][:, :sc.m_real] if res[k].ndim == 2 else res[k][first] for k in OUTPUTS})
    finally:
        w.close()
    return outs


# (scene, map form, participant slots) -> (case, outputs of every tick) of the first such case that ran in this session.
# Each later case of the same key must give the same outputs.  This only makes a disagreement between instances readable:
# a case run alone (or the first one under -k) has nothing to compare with, and every case is held to the oracle anyway.
_SEEN = {}


def _prepare(scene, axis, instance, sm_count):
    """The scene in the form ``instance`` and ``axis`` take, and idx [N]: the scene's scenario each world scenario copies."""
    table_mode = instance.endswith("_table")
    sc = SCENES[scene](table_mode)
    if table_mode and sc.tile_id is None:
        sc = _reversed_tile(sc)
    if instance.startswith("fp64"):
        sc = dataclasses.replace(sc, table=_with_dynamics(sc.table),
                                 map_table=None if sc.map_table is None else _with_dynamics(sc.map_table))
    m = sc.x.shape[1]
    if instance.startswith("fixed"):
        sc = _pad_slots(sc, 64 - m)
    if axis.startswith("scalar"):
        # padded past 64 slots a warp holds one scenario, whose 64 undecided pairs would just fit the exact queue: a scene
        # built to overflow it is trimmed to 61 .. 63 slots instead, two scenarios per warp
        r = int(axis[-1])
        sc = _trim_slots(sc, (m - r) % 4) if sc.exact_overflow else _pad_slots(sc, (r - m) % 4)
        assert sc.x.shape[1] % 4 == r
    if sc.exact_overflow:
        spw = 32 // _group(sc.x.shape[1])
        assert sc.rare.reshape(-1, spw).all(1).any() and spw * sc.m_real > EXACT_QUEUE   # a warp of rare scenarios overflows
    if axis == "global_map":
        sc = _far_segments(sc)
    return sc, _waves(sc, sm_count) if axis == "several_waves" else np.arange(sc.x.shape[0])


def test_instance_counter_is_host_side():
    """The counters need no device: k = 0 .. 6 are counts, any other k is -1, and the FIXED instances' two counts add up
    to t2d_tick_fixed_count."""
    from tactics2d_b200 import _lib

    lib = _lib.load()
    assert lib.t2d_tick_instance_count(-1) == -1 and lib.t2d_tick_instance_count(7) == -1
    counts = [lib.t2d_tick_instance_count(k) for k in range(7)]
    assert min(counts) >= 0 and lib.t2d_tick_fixed_count() == counts[4] + counts[5]


@pytest.mark.gpu
@pytest.mark.parametrize("scene, axis, instance", _cases())
def test_tick_instance_against_the_oracle(cuda_device, scene, axis, instance):
    import torch

    sc, idx = _prepare(scene, axis, instance, torch.cuda.get_device_properties(cuda_device).multi_processor_count)
    outs = _run(sc, instance, cuda_device, idx, axis == "global_map")
    key = (scene, instance.endswith("_table"), sc.m_real)
    case = f"{axis}-{instance}"
    if key not in _SEEN:
        _SEEN[key] = (case, outs)
        return
    seen_case, seen = _SEEN[key]
    for t, (a, b) in enumerate(zip(outs, seen)):
        for k in OUTPUTS:
            assert np.array_equal(a[k], b[k]), f"tick {t}: {k} of {case} differs from {seen_case}"
