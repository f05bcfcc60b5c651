"""The tick's C2-shaped instance (`t2d_step_kernel<.., FIXED>`): compiled for M = 64, kinematic types only, aligned
state, no ego action and no goal, with the loops over that shape unrolled and the tests for the features it excludes
folded away.  It must compute exactly what the generic instance computes, so
every scene runs in two worlds built alike, one of them kept on the generic instance (T2D_TICK_GENERIC=1 at its
creation), and the state and every output of every tick must agree bit for bit.  Ticks that just miss the shape must
run the generic instance (`t2d_tick_fixed_count` does not move)."""

import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

STATE = ("x", "y", "heading", "speed", "vx", "vy")
OUTPUTS = ("flags", "hit_index", "hit_segment", "status", "done")


def _world(sc, device, generic, interval=100, delta_t=5, map_tiles=None):
    from tactics2d_b200 import BatchedWorld

    n, m = sc.shape
    if generic:
        os.environ["T2D_TICK_GENERIC"] = "1"
    try:
        w = BatchedWorld(n, m, sc.table, device=device, interval=interval, delta_t=delta_t, max_step=7)
    finally:
        os.environ.pop("T2D_TICK_GENERIC", None)
    if map_tiles is None:
        w.set_map(sc.segments, sc.bounds)
    else:
        w.set_map_table(*map_tiles)
    w.set_state(sc.x, sc.y, sc.heading, sc.speed, type_id=sc.type_id)
    return w


def _run_pair(sc, device, ticks=3, ego=False, **kw):
    """Ticks the scene in a world that may take the C2-shaped instance and in one kept generic; asserts bit-identical
    state and outputs after every tick and returns (ticks the C2-shaped instance ran, flags of the last tick)."""
    import torch

    from tactics2d_b200 import _lib, synthetic

    lib = _lib.load()
    n, m = sc.shape
    a, b = _world(sc, device, False, **kw), _world(sc, device, True, **kw)
    fixed = 0
    try:
        for t in range(ticks):
            act = torch.from_numpy(synthetic.random_actions(300 + t, (n, m))).to(device)
            if ego:
                e = torch.from_numpy(synthetic.random_actions(400 + t, (n, 1))[:, 0]).to(device).contiguous()
                a.set_ego_action(e)
                b.set_ego_action(e)
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
        flags = ra.flags.cpu().numpy()
    finally:
        a.close()
        b.close()
    return fixed, flags


def _c2(n, m=64, seed=5, **kw):
    from tactics2d_b200 import synthetic

    return synthetic.config2(n, m, seed=seed, **kw)


@pytest.mark.parametrize("n", [1, 3, 257, 4099])
def test_m64_at_odd_n(cuda_device, n):
    """C2 at M = 64 and odd N: the last warp tile holds one scenario and an empty group."""
    fixed, _ = _run_pair(_c2(n), cuda_device)
    assert fixed == 3


def test_c2_shuffled_slots(cuda_device):
    """The C2 scene with every scenario's slots in a random order (the sort and the sweep see another slot order)."""
    import dataclasses

    sc = _c2(2048, seed=6)
    perm = np.argsort(np.random.default_rng(6).random(sc.shape), axis=1)
    take = lambda v: np.ascontiguousarray(np.take_along_axis(v, perm, axis=1))
    sc = dataclasses.replace(sc, x=take(sc.x), y=take(sc.y), heading=take(sc.heading), speed=take(sc.speed),
                             vx=take(sc.vx), vy=take(sc.vy), type_id=take(sc.type_id))
    fixed, _ = _run_pair(sc, cuda_device)
    assert fixed == 3


def test_dense_scene_with_overlaps(cuda_device):
    """About 3.4 m between vehicles: many pairs touch or nearly touch, so the candidate drain, the fp32 filter's
    undecided pairs and the static phase all run; status goes FAILED in many scenarios."""
    sc = _c2(512, seed=7, size=3.4 * 8.0)
    fixed, flags = _run_pair(sc, cuda_device, ticks=4)
    assert fixed == 4
    assert (flags & 1).any() and (flags & 2).any()


def test_map_table(cuda_device):
    """Every scenario names its own map tile (the map-table variant of the C2-shaped instance)."""
    sc = _c2(300, seed=8)
    seg = np.asarray(sc.segments, np.float32)
    tiles = [dict(segments=seg, bounds=sc.bounds), dict(segments=seg[::2] + np.float32(1.5), bounds=sc.bounds)]
    fixed, _ = _run_pair(sc, cuda_device, map_tiles=(tiles, np.arange(300) % 2))
    assert fixed == 3


@pytest.mark.parametrize("case", ["m63", "m65", "ego_action"])
def test_near_misses_run_generic(cuda_device, case):
    """One shape value off the C2 shape: the generic instance runs (and the two worlds still agree)."""
    m = {"m63": 63, "m65": 65}.get(case, 64)
    fixed, _ = _run_pair(_c2(65, m=m, seed=9), cuda_device, ego=case == "ego_action")
    assert fixed == 0


@pytest.mark.parametrize("interval, delta_t", [(95, 5), (103, 5), (100, 3)], ids=["19_steps", "remainder", "33_steps"])
def test_other_time_steps(cuda_device, interval, delta_t):
    """The sub-step count and the remainder sub-step stay runtime values of the C2-shaped instance."""
    fixed, _ = _run_pair(_c2(65, seed=10), cuda_device, interval=interval, delta_t=delta_t)
    assert fixed == 3


def test_c2_shape_runs_fixed_and_switch_keeps_generic(cuda_device):
    """The gate's positive case at the bench's shape, and the environment switch."""
    import torch

    from tactics2d_b200 import _lib, synthetic

    lib = _lib.load()
    sc = _c2(64)
    act = torch.from_numpy(synthetic.random_actions(1, sc.shape)).to(cuda_device)
    for generic, expect in ((False, 1), (True, 0)):
        w = _world(sc, cuda_device, generic)
        c0 = lib.t2d_tick_fixed_count()
        w.step(act)
        torch.cuda.synchronize()
        assert lib.t2d_tick_fixed_count() - c0 == expect
        w.close()
