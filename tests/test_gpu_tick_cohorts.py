"""The C2-shaped tick (`t2d_step_kernel<.., FIXED>`) splits every CTA's warps into two cohorts: the first half issue
their first tile's loads, then arrive on a named CTA barrier; the second half wait on it before issuing theirs.  Every
thread of the CTA has to reach that barrier exactly once, also the warps of a partial last CTA that have no tile and
the warps of a persistent launch that go on to further tiles.  These shapes run in a world that takes the C2-shaped
instance and in one kept on the generic instance (T2D_TICK_GENERIC=1 at its creation); state and outputs must agree
bit for bit after every tick, and `t2d_tick_fixed_count` must show that the C2-shaped instance ran.

At M = 64 a warp holds 2 scenarios and an 8-warp CTA 16, so N = 1, 3, 9 and 17 leave warps of cohort A, of cohort B or
of both without a tile, 4095 ends on a half tile and 4097 on a CTA with a single tile.  T2D_WPC pins the warps per CTA
(the host picks 2-warp CTAs for small batches on its own); T2D_GRID_LIMIT=1 makes the launch persistent, several tiles
per warp."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

STATE = ("x", "y", "heading", "speed", "vx", "vy")
OUTPUTS = ("flags", "hit_index", "hit_segment", "status", "done")
TICKS = 3


def _world(sc, device, monkeypatch, generic, map_table):
    from tactics2d_b200 import BatchedWorld

    n, m = sc.shape
    with monkeypatch.context() as mp:
        if generic:
            mp.setenv("T2D_TICK_GENERIC", "1")
        w = BatchedWorld(n, m, sc.table, device=device, max_step=7)
    if map_table:
        seg = np.asarray(sc.segments, np.float32)
        tiles = [dict(segments=seg, bounds=sc.bounds), dict(segments=seg[::2] + np.float32(1.5), bounds=sc.bounds)]
        w.set_map_table(tiles, np.arange(n) % 2)
    else:
        w.set_map(sc.segments, sc.bounds)
    w.set_state(sc.x, sc.y, sc.heading, sc.speed, type_id=sc.type_id)
    return w


def _check_pair(n, device, monkeypatch, map_table, seed=21):
    import torch

    from tactics2d_b200 import _lib, synthetic

    lib = _lib.load()
    sc = synthetic.config2(n, 64, seed=seed, size=3.4 * 8.0)   # dense: collisions, drains and status changes
    a = _world(sc, device, monkeypatch, False, map_table)
    b = _world(sc, device, monkeypatch, True, map_table)
    fixed = 0
    try:
        for t in range(TICKS):
            act = torch.from_numpy(synthetic.random_actions(600 + t, sc.shape)).to(device)
            c0 = lib.t2d_tick_fixed_count()
            ra = a.step(act)
            torch.cuda.synchronize()
            fixed += lib.t2d_tick_fixed_count() - c0
            rb = b.step(act)
            torch.cuda.synchronize()
            sa, sb = a.state_numpy(), b.state_numpy()
            for k in STATE:
                assert np.array_equal(sa[k].view(np.uint32), sb[k].view(np.uint32)), (t, k)
            for k in OUTPUTS:
                assert np.array_equal(getattr(ra, k).cpu().numpy(), getattr(rb, k).cpu().numpy()), (t, k)
    finally:
        a.close()
        b.close()
    assert fixed == TICKS


@pytest.mark.parametrize("map_table", [False, True], ids=["one_tile", "map_table"])
@pytest.mark.parametrize("wpc", [None, "8", "3"], ids=["wpc_auto", "wpc8", "wpc3"])
@pytest.mark.parametrize("n", [1, 3, 9, 17, 4095, 4097])
def test_partial_ctas(cuda_device, monkeypatch, n, wpc, map_table):
    if wpc is not None:
        monkeypatch.setenv("T2D_WPC", wpc)
    _check_pair(n, cuda_device, monkeypatch, map_table)


@pytest.mark.parametrize("map_table", [False, True], ids=["one_tile", "map_table"])
@pytest.mark.parametrize("n", [4097, 9001])
def test_persistent_launch(cuda_device, monkeypatch, n, map_table):
    """One CTA per SM: 8-warp CTAs take their tiles in several waves, and a warp reaches the cohort barrier on its
    first tile only."""
    monkeypatch.setenv("T2D_GRID_LIMIT", "1")
    _check_pair(n, cuda_device, monkeypatch, map_table)
