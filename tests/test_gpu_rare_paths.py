"""The rare paths of the fused tick (t2d_step_kernel), each forced by a scene built so that it MUST take them, against the
float64 oracle: flags, hit_index, hit_segment, status and done bit-exact, the state within 1e-5.  Dense scenes are where
these paths run in practice (C5 at M = 128, crowds), and a missed collision there would go unseen by the random-scene
parity tests.  Every scene comes with the arithmetic that shows why it takes its path."""

import dataclasses

import numpy as np
import pytest

from oracle import scenario as O

pytestmark = pytest.mark.gpu

QCAP = 192          # candidate pairs one warp can queue (t2d_kernels.cu)
EXACT_QUEUE = 64    # filter-undecided (participant, segment) pairs one warp can queue


def _rbound(table):
    return np.array([r.radius if r.shape == 1 else np.hypot(r.half_len, r.half_wid) * 1.000002 for r in table.rows])


def _tick(w, table, tid, act, segments=None, bounds=None, poly_start=None, still=False):
    """One step of ``w`` against the oracle; returns the oracle's (flags, hit_index, hit_segment)."""
    import torch

    before = w.state_numpy()
    otab = table.as_oracle_table()
    ref = O.physics_tick(before, tid, act, otab, w.interval, w.delta_t)
    r = w.step(torch.from_numpy(np.ascontiguousarray(act, dtype=np.float32)).to(w.device))
    torch.cuda.synchronize()
    got = w.state_numpy()
    for k in ("x", "y", "speed"):
        err = np.abs(got[k] - ref[k]) / np.maximum(np.abs(ref[k]), 1.0)
        assert err.max() <= 1e-5, (k, err.max())
    if still:   # zero speed and action: the poses the scene was built on stay exact
        for k in ("x", "y", "heading"):
            assert np.array_equal(got[k], before[k]), k
    fl, hi, hs = O.events(got["x"], got["y"], got["heading"], tid, otab, segments, bounds, poly_start=poly_start)
    assert np.array_equal(r.flags.cpu().numpy(), fl)
    assert np.array_equal(r.hit_index.cpu().numpy(), hi)
    assert np.array_equal(r.hit_segment.cpu().numpy(), hs)
    st, done = O.status(fl, tid, w.step_count.cpu().numpy(), w.max_step)
    assert np.array_equal(r.status.cpu().numpy(), st)
    assert np.array_equal(r.done.cpu().numpy(), done)
    return fl, hi, hs


def _world(table, x, y, h, v, tid, device, segments=None, bounds=None, cell_size=0.0, poly_start=None):
    from tactics2d_b200 import BatchedWorld

    w = BatchedWorld(*x.shape, table, device=device)
    if segments is not None or bounds is not None:
        w.set_map(segments, bounds, cell_size=cell_size, poly_start=poly_start)
    w.set_state(x, y, h, v, type_id=tid)
    return w


# ------------------------------------------------------------------------------------------------ B1
@pytest.mark.parametrize("m", [32, 64, 128])
def test_pair_queue_overflow_takes_the_exhaustive_pass(cuda_device, m):
    """M vehicles inside a disc of radius 2 m: every pair is at most 4 m apart, below the broadphase reach r_i + r_max
    >= 1.95 + 2.82 m of the vehicle table, so all M (M - 1) / 2 pairs are candidates - 496 at M = 32, 2016 at M = 64,
    8128 at M = 128 - against a queue of 192 per warp.  A warp holds 128 / M scenarios (4, 2, 1): the dense scenario
    shares its warp with sparse arena scenarios, whose pairs the exhaustive pass must resolve as well."""
    from tactics2d_b200 import synthetic

    n = 16
    sc = synthetic.config2(n, m, seed=70 + m, size=60.0)
    rng = np.random.default_rng(m)
    x, y, h, v = sc.x.copy(), sc.y.copy(), sc.heading.copy(), sc.speed.copy()
    spw = 128 // m
    dense = np.arange(n) % (2 * spw) == 0             # one dense scenario in every other warp
    rad, ang = 2.0 * np.sqrt(rng.uniform(0, 1, (n, m))), rng.uniform(0, 2 * np.pi, (n, m))
    x[dense] = (30.0 + rad * np.cos(ang))[dense]
    y[dense] = (30.0 + rad * np.sin(ang))[dense]
    rb = _rbound(sc.table)[sc.type_id]
    reach = rb + rb.max()
    for s in np.nonzero(dense)[0]:
        d2 = (x[s, :, None] - x[s, None, :]) ** 2 + (y[s, :, None] - y[s, None, :]) ** 2
        cand = np.triu(d2 <= reach[s, :, None] ** 2, 1).sum()
        assert cand > QCAP, cand
    w = _world(sc.table, x, y, h, v, sc.type_id, cuda_device, sc.segments, sc.bounds)
    for t in range(2):
        fl, hi, _ = _tick(w, sc.table, sc.type_id, synthetic.random_actions(80 + t, (n, m)), sc.segments, sc.bounds)
        assert (fl[dense] & 1).all()                      # everybody in the crowd collides ...
        assert len(np.unique(hi[dense])) > 1              # ... and not all with the same first partner
        assert (fl[~dense] & 1).any() and not (fl[~dense] & 1).all()
    w.close()


# ------------------------------------------------------------------------------------------------ B2
def _touch_table():
    from tactics2d_b200 import TypeParams, TypeTable

    return TypeTable([dataclasses.replace(TypeParams.vehicle("medium_car"), half_len=2.0, half_wid=1.0)])


@pytest.mark.parametrize("decisive", [False, True], ids=["touch_only", "with_decisive_hit"])
def test_exact_queue_overflow_takes_the_exact_walk(cuda_device, decisive):
    """64 boxes of 2 x 1 half extents at heading 0 on integer centres 12 m apart, every coordinate exact: each box gets a
    segment that touches it exactly - lying on its top edge, ending on its right edge, or meeting its corner.  The filter
    margin of such a pair is exactly 0, inside the +-EPS_LIN band, so every one of them is queued for the exact test: 128
    per warp (2 scenarios of 64) against 64 slots.  With ``decisive`` every box is also crossed by a segment through its
    centre at a higher index (a decided hit that ends the walk): the lower, touching segment must still win."""
    m, n = 64, 4
    table = _touch_table()
    k = np.arange(m)
    cx, cy = (12.0 * (k % 8)).astype(np.float32), (12.0 * (k // 8)).astype(np.float32)
    kind = k % 3
    touch = np.stack([np.where(kind == 0, cx - 1, np.where(kind == 1, cx + 2, cx + 2)),
                      np.where(kind == 0, cy + 1, np.where(kind == 1, cy - 0.5, cy + 1)),
                      np.where(kind == 0, cx + 1, np.where(kind == 1, cx + 4, cx + 3)),
                      np.where(kind == 0, cy + 1, np.where(kind == 1, cy + 0.5, cy + 2))], 1)
    assert 2 * m > EXACT_QUEUE                           # one undecided segment per box, two scenarios per warp
    seg = touch
    if decisive:
        seg = np.concatenate([touch, np.stack([cx - 3, cy, cx + 3, cy], 1)])
    seg = np.ascontiguousarray(seg, dtype=np.float32)
    x, y = np.tile(cx, (n, 1)), np.tile(cy, (n, 1))
    z = np.zeros((n, m), np.float32)
    tid = np.zeros((n, m), np.uint8)
    w = _world(table, x, y, z, z, tid, cuda_device, seg, (-10.0, 100.0, -10.0, 100.0))
    _, _, hs = _tick(w, table, tid, np.zeros((n, m, 2), np.float32), seg, (-10.0, 100.0, -10.0, 100.0), still=True)
    assert np.array_equal(hs, np.tile(k, (n, 1)))        # the touching segment, also where a crossing one follows
    w.close()


# ------------------------------------------------------------------------------------------------ B3
def _bus_scene(rng, n, m, tid_bus):
    """Walls inside a 30 m square and vehicles around it; buses parked with their centres 3.5 - 5.5 m left of the left
    wall (outside the map's grown grid) whose 6 m half length still reaches across it."""
    seg = np.array([(0, 0, 0, 30), (0, 0, 30, 0), (30, 0, 30, 30), (5, 5, 25, 25), (10, 30, 20, 30)], np.float32)
    x = rng.uniform(-8, 38, (n, m)).astype(np.float32)
    y = rng.uniform(-8, 38, (n, m)).astype(np.float32)
    h = rng.uniform(0, 2 * np.pi, (n, m)).astype(np.float32)
    tid = rng.integers(0, 3, (n, m)).astype(np.uint8)
    out = rng.uniform(0, 1, (n, m)) < 0.25
    x[out] = rng.uniform(-5.5, -3.5, out.sum()).astype(np.float32)
    y[out] = rng.uniform(1, 29, out.sum()).astype(np.float32)
    h[out] = rng.uniform(-0.3, 0.3, out.sum()).astype(np.float32)
    tid[out] = tid_bus
    return seg, x, y, h, tid, out


def _tables():
    from tactics2d_b200 import TypeParams, TypeTable

    cars = [TypeParams.vehicle("mini_car"), TypeParams.vehicle("medium_car"), TypeParams.vehicle("luxury_car")]
    bus = dataclasses.replace(TypeParams.vehicle("medium_car"), half_len=6.0, half_wid=1.3, lf=2.8, lr=2.8, name="bus")
    return TypeTable(cars), TypeTable(cars + [bus])


def test_reach_beyond_the_dilation_small_cells(cuda_device):
    """cell_size = 1 m caps the map's dilation at one cell (1 m), so a bus (bounding radius 6.14 m) reaches beyond it and
    every bus near a wall takes the out-of-line exact walk over the cells under its whole bounding box; the buses left of
    the map have their centres outside the grid (which ends about 1 m left of x = 0) and still hit the wall at x = 0."""
    _, table = _tables()
    rng = np.random.default_rng(91)
    n, m = 64, 32
    seg, x, y, h, tid, out = _bus_scene(rng, n, m, 3)
    bounds = (-40.0, 70.0, -40.0, 70.0)
    v = rng.uniform(0, 3, (n, m)).astype(np.float32)
    w = _world(table, x, y, h, v, tid, cuda_device, seg, bounds, cell_size=1.0)
    fl, _, hs = _tick(w, table, tid, np.zeros((n, m, 2), np.float32), seg, bounds)
    assert (hs[out] == 0).mean() > 0.9                   # the buses outside the grid reach the left wall
    assert ((fl & 2) != 0).mean() > 0.3
    w.close()


def test_reach_beyond_the_dilation_table_set_after_the_map(cuda_device):
    """The map is built for a table of cars (reach 2.83 m: the dilation), then a table with a bus row replaces it through
    ``set_type_table``: the buses reach beyond the dilation and take the exact walk; those left of the map have their
    centres outside the grid, which the cars' dilation grew by only 2.83 m."""
    small, table = _tables()
    rng = np.random.default_rng(92)
    n, m = 64, 32
    seg, x, y, h, tid, out = _bus_scene(rng, n, m, 3)
    bounds = (-40.0, 70.0, -40.0, 70.0)
    v = rng.uniform(0, 3, (n, m)).astype(np.float32)
    from tactics2d_b200 import BatchedWorld

    w = BatchedWorld(n, m, small, device=cuda_device)
    w.set_map(seg, bounds)
    w.set_type_table(table)
    w.set_state(x, y, h, v, type_id=tid)
    fl, _, hs = _tick(w, table, tid, np.zeros((n, m, 2), np.float32), seg, bounds)
    assert (hs[out] == 0).mean() > 0.9
    w.close()


# ------------------------------------------------------------------------------------------------ B4
def _clearance_scene():
    """64 short walls at 45 degrees, 12 m apart, the j-th shifted by j / 32 m in x and in y, i.e. by j / 64 of a 2 m fine
    cell; per wall, discs of radius 0.9 and 1.06 swept along the wall's normal from r - 0.25 to r + 0.25 m in 1 mm steps.
    Then centres exactly on fine-cell boundaries near the walls, and in the grid's last row and column.  Returns the table,
    segments, positions [P, 2], type ids [P] and the number of swept poses (first in the list)."""
    from tactics2d_b200 import TypeParams, TypeTable

    radii = (0.9, 1.06)
    table = TypeTable([dataclasses.replace(TypeParams.vehicle("medium_car"), radius=r, shape=1) for r in radii])
    j = np.arange(64)
    cx, cy = 12.0 * (j % 8) + j / 32.0, 12.0 * (j // 8) + j / 32.0
    a = 2.0 / np.sqrt(2.0)
    seg = np.stack([cx - a, cy + a, cx + a, cy - a], 1).astype(np.float32)
    nrm = np.array([1.0, 1.0]) / np.sqrt(2.0)
    d = np.arange(-250, 251) * 1e-3
    pts, types = [], []
    for t, r in enumerate(radii):
        c = np.stack([cx, cy], 1)[:, None, :] - (r + d)[None, :, None] * nrm
        pts.append(c.reshape(-1, 2))
        types.append(np.full(len(c.reshape(-1, 2)), t))
    n_swept = sum(len(p) for p in pts)
    # the grid as the library lays it out: 8 m cells of 4 x 4 fine cells, over the segments' box grown by the reach
    f = np.float32
    xmin, xmax = float(seg[:, [0, 2]].min()), float(seg[:, [0, 2]].max())
    reach = f(max(radii)) * f(1.0002) + f(2e-3)
    margin = f(1e-3) * max(f(1), f(abs(xmin) + abs(xmax)) * f(1e-3))
    x0 = f(xmin) - reach - margin
    g = int(np.floor((f(xmax) + reach + margin - x0) / f(8))) + 1
    b = float(x0) + 2.0 * np.arange(4 * g + 1)
    for k in range(0, 64, 9):                                   # on a vertical boundary, touching and just clear
        xb = b[np.argmin(np.abs(b - (cx[k] - 1.0)))]
        for t, r in enumerate(radii):
            yy = cx[k] + cy[k] - xb - (r + np.array([-0.01, 0.0, 0.01])) * np.sqrt(2.0)
            pts.append(np.stack([np.full(3, xb), yy], 1))
            types.append(np.full(3, t))
    last = np.array([[b[-2] + 0.5, v] for v in b[:-1]] + [[v, b[-2] + 0.5] for v in b[:-1]] + [[b[-1] - 1e-3, b[-1] - 1e-3], [b[-1], b[-1]]])
    pts.append(last)
    types.append(np.arange(len(last)) % 2)
    return table, seg, np.concatenate(pts), np.concatenate(types), n_swept


def test_clearance_field_edges(cuda_device):
    """The byte clearance field decides which participants may reach a wall at all.  Against a wall at 45 degrees a fine
    cell's nearest point is its corner, where the field's bound (centre distance minus the half diagonal, floored to
    0.125 m) is tight to about 5 mm.  A disc whose radius is not a multiple of 0.125 m (0.9, 1.06) and that touches the
    wall from near that corner finds the next multiple above its radius in a byte rounded up instead of down, i.e. would
    be called "far": the 64 sub-cell wall offsets put such corners under the sweep."""
    table, seg, p, tt, n_swept = _clearance_scene()
    m = 32
    n = -(-len(p) // m)
    pad = n * m - len(p)
    p = np.concatenate([p, np.tile([[-30.0, -30.0]], (pad, 1))])
    tt = np.concatenate([tt, np.full(pad, 255)])
    x, y = p[:, 0].reshape(n, m).astype(np.float32), p[:, 1].reshape(n, m).astype(np.float32)
    tid = tt.reshape(n, m).astype(np.uint8)
    z = np.zeros((n, m), np.float32)
    w = _world(table, x, y, z, z, tid, cuda_device, seg, None)
    fl, _, _ = _tick(w, table, tid, np.zeros((n, m, 2), np.float32), seg, None, still=True)
    frac = ((fl.reshape(-1)[:n_swept] & 2) != 0).mean()
    assert 0.4 < frac < 0.6, frac                             # the sweep straddles contact
    w.close()


# ------------------------------------------------------------------------------------------------ B5
def test_area_with_two_holes_on_the_gpu(cuda_device):
    """The walkway of inD_2 with two holes (one Area: exterior and both inner rings back to back) among the map's other
    areas: boxes inside a hole clear of its edges (free), inside the exterior clear of every edge (a hit by containment
    alone), and straddling an inner ring (an edge hit)."""
    from oracle.geometry import point_in_ring
    from tactics2d_b200.map import load_areas, polygons_to_segments
    from tactics2d_b200 import TypeParams, TypeTable

    areas = load_areas("inD_2")
    seg, ps = polygons_to_segments(areas)
    k = [i for i, a in enumerate(areas) if len(a.inners) == 2][0]
    a = areas[k]
    table = TypeTable([dataclasses.replace(TypeParams.vehicle("medium_car"), half_len=0.4, half_wid=0.3)])
    s64 = seg.astype(np.float64)
    rng = np.random.default_rng(93)

    def clearance(pts):
        d = pts[:, None, :] - s64[None, :, :2]
        e = s64[None, :, 2:] - s64[None, :, :2]
        t = np.clip((d * e).sum(-1) / np.maximum((e * e).sum(-1), 1e-30), 0, 1)
        return np.sqrt(((d - t[..., None] * e) ** 2).sum(-1)).min(1)

    mine = s64[ps[k]:ps[k + 1]]
    lo, hi = a.outer.min(0), a.outer.max(0)
    pts = rng.uniform(lo, hi, (40000, 2))
    clear = clearance(pts) > 0.6
    others = np.zeros(len(pts), bool)
    for j in range(len(areas)):
        if j != k:
            others |= point_in_ring(pts[:, 0], pts[:, 1], s64[ps[j]:ps[j + 1]])
    solid = point_in_ring(pts[:, 0], pts[:, 1], mine)
    ring0 = np.concatenate([a.outer, np.roll(a.outer, -1, 0)], 1)
    in_hole = point_in_ring(pts[:, 0], pts[:, 1], ring0) & ~solid & clear & ~others
    inside = solid & clear & ~others
    holes = [np.concatenate([r, np.roll(r, -1, 0)], 1) for r in a.inners]
    hole_v = np.concatenate([r[:, :2] for r in holes])
    straddle = hole_v[rng.integers(0, len(hole_v), 64)] + rng.uniform(-0.2, 0.2, (64, 2))
    assert in_hole.sum() >= 16 and inside.sum() >= 64
    p = np.concatenate([pts[in_hole][:64], pts[inside][:64], straddle])
    cls = np.concatenate([np.zeros(min(64, in_hole.sum())), np.ones(64), np.full(64, 2)])
    m = 32
    n = -(-len(p) // m)
    pad = n * m - len(p)
    p = np.concatenate([p, np.repeat(p[:1], pad, 0)])
    cls = np.concatenate([cls, np.full(pad, -1)])
    x, y = p[:, 0].reshape(n, m).astype(np.float32), p[:, 1].reshape(n, m).astype(np.float32)
    h = rng.uniform(0, 6.28, (n, m)).astype(np.float32)        # below fp32(2 pi): the wrapped heading is the input
    tid = np.where(cls < 0, 255, 0).reshape(n, m).astype(np.uint8)
    z = np.zeros((n, m), np.float32)
    w = _world(table, x, y, h, z, tid, cuda_device, seg, None, poly_start=ps)
    fl, _, hs = _tick(w, table, tid, np.zeros((n, m, 2), np.float32), seg, None, poly_start=ps, still=True)
    hs, cls = hs.reshape(-1), cls.reshape(-1)
    assert (hs[cls == 0] == -1).all()                        # parked in a hole: free
    assert (hs[cls == 1] == ps[k]).all()                     # inside the walkway, touching nothing: the walkway
    assert (hs[cls == 2] >= 0).all()                         # across an inner ring
    w.close()
