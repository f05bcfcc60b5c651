"""The box-culled, warp-compacted partner sweep of the fused tick (t2d_step_kernel): a lane skips the partner words whose
8-slot box lies beyond its own participants' box grown by their reach, and the surviving (lane, word) items are swept by
the whole warp.  A word culled wrongly loses candidate pairs, i.e. collisions, so every scene here compares flags,
hit_index, hit_segment, status and done bit for bit against the float64 oracle, with the poses left exactly as placed
(zero speed, zero action)."""

import dataclasses

import numpy as np
import pytest

from oracle import scenario as O

pytestmark = pytest.mark.gpu

QCAP = 192   # candidate pairs one warp can queue (t2d_kernels.cu)


def _check(table, x, y, h, tid, device, segments=None, bounds=None):
    """One still tick of the scene against the oracle; returns its flags and hit indices."""
    import torch

    from tactics2d_b200 import BatchedWorld

    n, m = x.shape
    z = np.zeros((n, m), np.float32)
    w = BatchedWorld(n, m, table, device=device)
    if segments is not None or bounds is not None:
        w.set_map(segments, bounds)
    w.set_state(x, y, h, z, type_id=tid)
    before = w.state_numpy()
    r = w.step(torch.zeros((n, m, 2), dtype=torch.float32, device=w.device))
    torch.cuda.synchronize()
    got = w.state_numpy()
    for k in ("x", "y", "heading"):
        assert np.array_equal(got[k], before[k]), k
    otab = table.as_oracle_table()
    fl, hi, hs = O.events(got["x"], got["y"], got["heading"], tid, otab, segments, bounds)
    assert np.array_equal(r.flags.cpu().numpy(), fl)
    assert np.array_equal(r.hit_index.cpu().numpy(), hi)
    assert np.array_equal(r.hit_segment.cpu().numpy(), hs)
    st, done = O.status(fl, tid, w.step_count.cpu().numpy(), w.max_step)
    assert np.array_equal(r.status.cpu().numpy(), st)
    assert np.array_equal(r.done.cpu().numpy(), done)
    w.close()
    return fl, hi


def _f32(*a):
    return [np.ascontiguousarray(v, dtype=np.float32) for v in a]


@pytest.mark.parametrize("m", [64, 128])
def test_shuffled_slot_order(cuda_device, m):
    """C2-like arenas with the slot order shuffled in every scenario: neighbours in space are no longer neighbours in slot
    order, so nearly every partner word is needed and the sweep runs the per-lane path; the ordered copy of the same
    scenes runs the compacted list.  Both must find every collision."""
    from tactics2d_b200 import synthetic

    n = 256
    sc = synthetic.config2(n, m, seed=40 + m, size=140.0 if m == 64 else 200.0)
    rng = np.random.default_rng(m)
    perm = np.argsort(rng.uniform(size=(n, m)), axis=1)
    take = lambda a: np.take_along_axis(a, perm, axis=1)
    x, y, h = _f32(sc.x, sc.y, sc.heading)
    tid = sc.type_id.astype(np.uint8)
    fl_o, _ = _check(sc.table, x, y, h, tid, cuda_device, sc.segments, sc.bounds)
    fl_s, _ = _check(sc.table, *_f32(take(x), take(y), take(h)), take(tid), cuda_device, sc.segments, sc.bounds)
    assert (fl_o & 1).any() and (fl_s & 1).any()
    assert np.array_equal(np.sort(take(fl_o), axis=1), np.sort(fl_s, axis=1))   # the same scene, only relabelled


def _disc_table(radius):
    from tactics2d_b200 import TypeParams, TypeTable

    return TypeTable([dataclasses.replace(TypeParams.vehicle("medium_car"), radius=radius, shape=1)])


@pytest.mark.parametrize("origin", [(1.0e4, -1.0e4), (-1.0e4, 1.0e4), (0.0, 0.0)], ids=["pm1e4", "mp1e4", "origin"])
def test_pairs_at_the_reach_across_words_and_box_edges(cuda_device, origin):
    """Discs of radius 1.25 (reach 2.5 to the fp32 broadphase's 1.00001 factor); in each scenario only the pairs
    (a, a + q) are solid, every other slot is inactive, so most 8-slot windows are all-NaN and the boxes a lane and a
    window are tested with are single points: the box edge is the partner itself.  The partner offset q = 1 .. 32 puts
    the partner in every word and on both sides of each word boundary.  Offsets are (2.5, 0), (0, -2.5), (1.5, 2.0) and
    (-2.0, -1.5), all exact at |x| = 1e4 (1 ulp = 2^-10), stretched to a length of 2.5 + k ulps: k = 0 touches (a hit),
    k = 1 is clear and, at 1e4, already beyond the broadphase reach; at the origin k runs across the reach
    (2.5 * (1 + 5e-6)) in steps of 2^-20 (rounded to the float grid of the pair's position)."""
    table = _disc_table(1.25)
    m, n = 64, 128
    ox, oy = origin
    ulp = 2.0 ** -10 if ox else 2.0 ** -20
    vecs = np.array([(2.5, 0.0), (0.0, -2.5), (1.5, 2.0), (-2.0, -1.5)])
    x = np.full((n, m), 0.0)
    y = np.full((n, m), 0.0)
    tid = np.full((n, m), 255, np.uint8)
    expect_hit = np.zeros((n, m), bool)
    for s in range(n):
        q = 1 + s % 32
        ks = (0, 1) if ox else tuple(range(0, 24, 2))
        k = ks[(s // 32) % len(ks)]
        v = vecs[(s // 32 // len(ks) + s) % 4] * ((2.5 + k * ulp) / 2.5)
        for j, a in enumerate(range(0, m - q, 2 * q) if q < m // 2 else [s % (m - q)]):
            b = a + q
            cx, cy = ox + 8.0 * (j % 6), oy + 8.0 * (j // 6)
            x[s, a], y[s, a] = cx, cy
            x[s, b], y[s, b] = cx + v[0], cy + v[1]
            tid[s, [a, b]] = 0
            expect_hit[s, [a, b]] = k == 0
    x, y = _f32(x, y)
    h = np.zeros((n, m), np.float32)
    fl, hi = _check(table, x, y, h, tid, cuda_device)
    assert ((fl & 1) != 0)[expect_hit].all()
    assert ((fl & 1) != 0).sum() >= expect_hit.sum()


@pytest.mark.parametrize("m", [13, 30, 61, 126])
def test_ragged_participant_counts(cuda_device, m):
    """M not a multiple of 4 and below the padded G x 4 (13 of 16, 30 of 32, 61 of 64, 126 of 128): the extended slots
    wrap at M, so the windows straddling the wrap mix the scenario's last and first participants, and the lanes past M
    own nothing (an empty box)."""
    from tactics2d_b200 import synthetic

    sc = synthetic.config2(192, m, seed=60 + m, size=12.0 * np.sqrt(m))
    x, y, h = _f32(sc.x, sc.y, sc.heading)
    fl, _ = _check(sc.table, x, y, h, sc.type_id.astype(np.uint8), cuda_device, sc.segments, sc.bounds)
    assert (fl & 1).any()


def test_all_nan_windows(cuda_device):
    """Scenarios whose slots are inactive except for a few, and scenarios with no solid participant at all (every window
    all-NaN, every lane box empty), beside fully populated ones in the same warps."""
    from tactics2d_b200 import synthetic

    n, m = 128, 64
    sc = synthetic.config2(n, m, seed=77, size=120.0)
    rng = np.random.default_rng(77)
    x, y, h = _f32(sc.x, sc.y, sc.heading)
    tid = sc.type_id.astype(np.uint8)
    kind = np.arange(n) % 4
    tid[kind == 1] = 255                                              # nobody solid
    sparse = (kind == 2)[:, None] & (rng.uniform(size=(n, m)) < 0.85)
    tid[sparse] = 255                                                 # a few solid ones, most windows all-NaN
    block = (kind == 3)[:, None] & ((np.arange(m) // 8) % 2 == 1)[None]
    tid[block] = 255                                                  # every other 8-slot block empty
    fl, _ = _check(sc.table, x, y, h, tid, cuda_device, sc.segments, sc.bounds)
    assert not fl[kind == 1].any()
    assert (fl[kind == 0] & 1).any()


def test_dense_scene_overflows_the_queue(cuda_device):
    """64 vehicles inside a 2 m disc in every fourth scenario: every pair is a candidate (2016 > 192 per warp), so the
    queue overflows and the exhaustive pass resolves the warp; the sparse scenarios sharing those warps are
    ordered arenas whose words the box test culls."""
    from tactics2d_b200 import synthetic

    n, m = 64, 64
    sc = synthetic.config2(n, m, seed=81, size=120.0)
    x, y, h = _f32(sc.x, sc.y, sc.heading)
    tid = sc.type_id.astype(np.uint8)
    rng = np.random.default_rng(81)
    dense = np.arange(n) % 4 == 0
    rad, ang = 2.0 * np.sqrt(rng.uniform(0, 1, (n, m))), rng.uniform(0, 2 * np.pi, (n, m))
    x[dense] = (60.0 + rad * np.cos(ang))[dense]
    y[dense] = (60.0 + rad * np.sin(ang))[dense]
    rb = np.array([np.hypot(r.half_len, r.half_wid) for r in sc.table.rows])[tid]
    for s in np.nonzero(dense)[0]:
        d2 = (x[s, :, None] - x[s, None, :]).astype(np.float64) ** 2 + (y[s, :, None] - y[s, None, :]).astype(np.float64) ** 2
        assert np.triu(d2 <= (rb[s, :, None] + rb.max()) ** 2, 1).sum() > QCAP
    fl, hi = _check(sc.table, x, y, h, tid, cuda_device, sc.segments, sc.bounds)
    assert (fl[dense] & 1).all()
    assert (fl[~dense] & 1).any() and not (fl[~dense] & 1).all()
