"""The x-sorted broadphase of the fused tick (t2d_step_kernel): each scenario's slots are sorted by x and every entry is
paired with the entries after it up to the reach.  It must hand the narrowphase exactly the candidate pairs of the
circular all-partner enumeration, so every scene compares flags, hit_index, hit_segment, status and done bit for bit
against the float64 oracle after still ticks (zero speed, zero action): sorted-order corner cases (one x column, ties,
signed zeros), pairs exactly at the reach at large coordinates, non-solid slots, every group width and slot order, the
map-table and fp64-model variants, and a queue overflow next to sparse scenarios."""

import numpy as np
import pytest

from oracle import scenario as O

from .test_gpu_broadphase_cull import QCAP, _check, _disc_table, _f32

pytestmark = pytest.mark.gpu


def _arena(n, m, seed, spacing=3.4):
    """C2 vehicles at about `spacing` metres apart: a few percent of them touch."""
    from tactics2d_b200 import synthetic

    sc = synthetic.config2(n, m, seed=seed, size=spacing * np.sqrt(m))
    return sc, *_f32(sc.x, sc.y, sc.heading), sc.type_id.astype(np.uint8)


def test_one_x_column_and_ties_in_x(cuda_device):
    """Even scenarios: every participant at the same x (the scan meets every pair); odd ones: x from three values only,
    so most entries tie in x with different y."""
    n, m = 128, 64
    sc, x, y, h, tid = _arena(n, m, 11)
    rng = np.random.default_rng(11)
    y = _f32(rng.uniform(0.0, 2.6 * m, (n, m)))[0]
    x[0::2] = 50.0
    x[1::2] = _f32(50.0 + 2.0 * rng.integers(0, 3, (n // 2, m)))[0]
    fl, _ = _check(sc.table, x, y, h, tid, cuda_device)
    assert (fl[0::2] & 1).any() and (fl[1::2] & 1).any()


def test_signed_zero_coordinates(cuda_device):
    """x and y drawn from {+0.0, -0.0, +-1.5, +-3.0}: -0.0 and +0.0 order differently in the sort key but are equal."""
    n, m = 64, 32
    sc, _, _, h, tid = _arena(n, m, 12)
    rng = np.random.default_rng(12)
    vals = np.array([0.0, -0.0, 1.5, -1.5, 3.0, -3.0], np.float32)
    x = vals[rng.integers(0, 6, (n, m))] * rng.integers(1, 9, (n, m)).astype(np.float32)
    y = vals[rng.integers(0, 6, (n, m))] * rng.integers(1, 9, (n, m)).astype(np.float32)
    x[:, ::5] = np.float32(-0.0)
    fl, _ = _check(sc.table, *_f32(x, y), h, tid, cuda_device)
    assert (fl & 1).any()


@pytest.mark.parametrize("scale", [1.0e4, 1.0e6], ids=["1e4", "1e6"])
@pytest.mark.parametrize("axis", ["x", "y"])
def test_pairs_exactly_at_the_reach(cuda_device, scale, axis):
    """Discs of radius 1.25: pairs 2.5 m apart along one axis touch, 2.5 m + 1 ulp do not; at 1e4 and 1e6 both are on
    the float grid.  The partner's slot offset runs over 1 .. M - 1 (so either end owns the pair, both at M / 2), and the
    pairs sit in columns 40 m apart, the rest of the scenario's slots inactive."""
    table = _disc_table(1.25)
    n, m = 128, 64
    ulp = float(np.spacing(np.float32(scale)))
    x = np.zeros((n, m))
    y = np.zeros((n, m))
    tid = np.full((n, m), 255, np.uint8)
    expect = np.zeros((n, m), bool)
    for s in range(n):
        q = 1 + s % (m - 1)
        k = (s // (m - 1)) % 2
        for j, a in enumerate(range(0, m - q, 2 * q) if q < m // 2 else [s % (m - q)]):
            b = a + q
            c0, c1 = scale + 40.0 * j, scale - 8.0 * (s % 3)
            d = 2.5 + k * ulp
            x[s, a], y[s, a] = c0, c1
            x[s, b], y[s, b] = (c0 + d, c1) if axis == "x" else (c0, c1 - d)
            tid[s, [a, b]] = 0
            expect[s, [a, b]] = k == 0
    x, y = _f32(x, y)
    fl, _ = _check(table, x, y, np.zeros((n, m), np.float32), tid, cuda_device)
    assert np.array_equal((fl & 1) != 0, expect)


def test_inactive_slots_interleaved(cuda_device):
    """Every other slot inactive, then every third, then all but two: the sort puts them last and never scans them."""
    n, m = 96, 64
    sc, x, y, h, tid = _arena(n, m, 13, spacing=2.6)
    k = np.arange(m)
    tid[0::3, 1::2] = 255
    tid[1::3, k % 3 == 0] = 255
    tid[2::3, 2:] = 255
    x[2::3, :2] = x[2::3, :1]
    y[2::3, 1] = y[2::3, 0] + 1.0
    fl, _ = _check(sc.table, x, y, h, tid, cuda_device)
    assert (fl[2::3, :2] & 1).all() and not fl[2::3, 2:].any()


@pytest.mark.parametrize("order", ["ordered", "shuffled", "reversed"])
@pytest.mark.parametrize("m", [1, 2, 3, 5, 31, 32, 33, 63, 64, 65, 127, 128])
def test_group_widths_and_slot_orders(cuda_device, m, order):
    """Every group width G = 1 .. 32 with full and ragged rows, in slot order, shuffled and reversed."""
    n = 96
    sc, x, y, h, tid = _arena(n, m, 100 + m, spacing=2.4)
    if order != "ordered":
        perm = (np.argsort(np.random.default_rng(m).uniform(size=(n, m)), axis=1) if order == "shuffled"
                else np.tile(np.arange(m)[::-1], (n, 1)))
        take = lambda a: np.ascontiguousarray(np.take_along_axis(a, perm, axis=1))
        x, y, h, tid = take(x), take(y), take(h), take(tid)
    fl, _ = _check(sc.table, x, y, h, tid, cuda_device)
    if m >= 5:
        assert (fl & 1).any()


def test_mixed_table_through_a_map_table(cuda_device):
    """C4-like mixed traffic (kinematic vehicles and cyclists, PointMass pedestrians: the fp64-model variant) on a map
    table of two tiles (the MAP_TABLE variant), shuffled slots, one event check per tile against the oracle."""
    import torch

    from tactics2d_b200 import BatchedWorld, synthetic
    from tactics2d_b200.map import load_collidable_segments

    seg, bounds = load_collidable_segments("inD_1")
    tiles = [dict(segments=seg, bounds=bounds, poly_start=None), dict(segments=None, bounds=bounds, poly_start=None)]
    n, m = 128, 32
    sc = synthetic.config4(n, m, seed=14, segments=seg, bounds=bounds, size=60.0)
    perm = np.argsort(np.random.default_rng(14).uniform(size=(n, m)), axis=1)
    take = lambda a: np.ascontiguousarray(np.take_along_axis(a, perm, axis=1))
    x, y, h, v, tid = take(sc.x), take(sc.y), take(sc.heading), take(sc.speed), take(sc.type_id)
    tile_id = np.arange(n) % 2
    w = BatchedWorld(n, m, sc.table, device=cuda_device, any_participant=True)
    w.set_map_table(tiles, tile_id)
    w.set_state(x, y, h, v, type_id=tid)
    r = w.check_events()
    torch.cuda.synchronize()
    table = sc.table.as_oracle_table()
    gfl, ghi, ghs = r.flags.cpu().numpy(), r.hit_index.cpu().numpy(), r.hit_segment.cpu().numpy()
    for t in range(2):
        rows = tile_id == t
        fl, hi, hs = O.events(x[rows], y[rows], h[rows], tid[rows], table, tiles[t]["segments"], tiles[t]["bounds"])
        assert np.array_equal(gfl[rows], fl) and np.array_equal(ghi[rows], hi) and np.array_equal(ghs[rows], hs)
    assert (gfl & 1).any()
    w.close()


def test_queue_overflow_in_one_scenario_of_a_warp(cuda_device):
    """M = 32 (four scenarios per warp): the first scenario of each warp packs its 32 vehicles into a 2 m disc (496
    candidate pairs > the queue), the other three are sparse arenas; the warp takes the exhaustive pass."""
    n, m = 64, 32
    sc, x, y, h, tid = _arena(n, m, 15)
    rng = np.random.default_rng(15)
    dense = np.arange(n) % 4 == 0
    rad, ang = 2.0 * np.sqrt(rng.uniform(0, 1, (n, m))), rng.uniform(0, 2 * np.pi, (n, m))
    x[dense] = _f32(30.0 + rad * np.cos(ang))[0][dense]
    y[dense] = _f32(30.0 + rad * np.sin(ang))[0][dense]
    assert m * (m - 1) // 2 > QCAP
    fl, _ = _check(sc.table, x, y, h, tid, cuda_device)
    assert (fl[dense] & 1).all()
    assert (fl[~dense] & 1).any() and not (fl[~dense] & 1).all()
