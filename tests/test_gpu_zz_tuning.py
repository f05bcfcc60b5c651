"""Tuning knobs of the tick must not change a single bit of its results (run last: nothing here is on the parity path)."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_prefetch_mode_does_not_change_results(cuda_device):
    """``t2d_set_prefetch``: the early L2 prefetch of the tick's inputs on, off, or left to the library's policy - five ticks
    each from the same state with the same actions give identical state, flags, hit indices, status and done."""
    import torch

    from tactics2d_b200 import BatchedWorld, synthetic
    from tactics2d_b200._lib import T2DError

    sc = synthetic.config2(512, 64, seed=61)
    act = torch.from_numpy(synthetic.random_actions(62, sc.shape)).to(cuda_device)
    seen = {}
    for mode in (0, 1, -1):
        w = BatchedWorld(*sc.shape, sc.table, device=cuda_device)
        w.set_map(sc.segments, sc.bounds)
        w.set_state(sc.x, sc.y, sc.heading, sc.speed, type_id=sc.type_id)
        w.set_prefetch(mode)
        for _ in range(5):
            r = w.step(act)
        torch.cuda.synchronize()
        st = w.state_numpy()
        seen[mode] = [st[k].copy() for k in ("x", "y", "heading", "speed", "vx", "vy")] + \
                     [getattr(r, k).cpu().numpy().copy() for k in ("flags", "hit_index", "hit_segment", "status", "done")]
        if mode == -1:
            with pytest.raises(T2DError):
                w.set_prefetch(2)
        w.close()
    for mode in (1, -1):
        for a, b in zip(seen[0], seen[mode]):
            assert np.array_equal(a, b, equal_nan=True) if a.dtype.kind == "f" else np.array_equal(a, b)
    assert seen[0][6].any()          # the comparison saw events, not an empty scene


LAUNCH_SHAPES = [
    {"T2D_WPC": "2"}, {"T2D_WPC": "3"}, {"T2D_WPC": "4"}, {"T2D_WPC": "8"},
    # one CTA of 2 warps per SM: 132 x 2 = 264 warps for the 1024 warp tiles of 2048 x 64, so every persistent CTA loops
    # over about four tiles
    {"T2D_GRID_LIMIT": "1", "T2D_WPC": "2"},
    {"T2D_PDL": "0"},
]


@pytest.mark.parametrize("map_table", [False, True], ids=["one_map", "map_table"])
@pytest.mark.parametrize("kin_only", [True, False], ids=["kin_only", "mixed_models"])
def test_launch_shape_does_not_change_results(cuda_device, monkeypatch, kin_only, map_table):
    """Warps per CTA, the persistent grid's CTA limit and programmatic dependent launch (read at t2d_create, hence set
    before each world is made) must not change a bit of three ticks, for each of the four variants of the tick kernel:
    kinematics-only tables or mixed models (point-mass pedestrians), one map for all scenarios or a tile per scenario."""
    import torch

    from tactics2d_b200 import BatchedWorld, synthetic

    n, m = 2048, 64
    sc = synthetic.config2(n, m, seed=63) if kin_only else synthetic.config4(n, m, seed=64, size=200.0)
    sc_map = synthetic.config2(1, 1, seed=0)
    tiles = [dict(segments=sc_map.segments, bounds=sc_map.bounds),
             dict(segments=sc_map.segments[::2] + np.float32(3.0), bounds=(-20.0, 230.0, -20.0, 230.0))]
    acts = [torch.from_numpy(synthetic.random_actions(65 + t, sc.shape)).to(cuda_device) for t in range(3)]

    def run(env):
        for k in ("T2D_WPC", "T2D_GRID_LIMIT", "T2D_PDL"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        w = BatchedWorld(*sc.shape, sc.table, device=cuda_device)
        if map_table:
            w.set_map_table(tiles, np.arange(n) % 2)
        else:
            w.set_map(tiles[0]["segments"], tiles[0]["bounds"])
        w.set_state(sc.x, sc.y, sc.heading, sc.speed, type_id=sc.type_id)
        out = []
        for a in acts:
            r = w.step(a)
            torch.cuda.synchronize()
            st = w.state_numpy()
            out += [st[k].copy() for k in ("x", "y", "heading", "speed", "vx", "vy")]
            out += [getattr(r, k).cpu().numpy().copy() for k in ("flags", "hit_index", "hit_segment", "status", "done")]
        w.close()
        return out

    base = run({})
    assert base[6].any() and (base[6] & 2).any()     # the comparison saw dynamic and static events
    for env in LAUNCH_SHAPES:
        got = run(env)
        for i, (a, b) in enumerate(zip(base, got)):
            same = np.array_equal(a, b, equal_nan=True) if a.dtype.kind == "f" else np.array_equal(a, b)
            assert same, (env, i)
