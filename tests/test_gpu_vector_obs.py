"""K8, the vector observation (t2d_observe / BatchedWorld.observe), against the float64 oracle in tests/vector_obs_oracle.py:
selection, order, indices, valid, dist, extents, speed, t_frac and in_ring bit-exact for every scenario, the rotated values
within the contract's tolerance.  Also CUDA graph = eager, the C-level rejections, and the env's "vector" observation."""

import ctypes as C

import numpy as np
import pytest

from tests import vector_obs_oracle as V

pytestmark = pytest.mark.gpu


def _check(w, K, S, ra, rs, tiles=(), tile_id=None, target=None):
    """Observes and compares every scenario with the oracle; returns the observation."""
    import torch

    o = w.observe(K, S, ra, rs)
    torch.cuda.synchronize()
    st = w.state_numpy()
    ref, ai, si = V.observe(st, w.type_id.cpu().numpy(), V.table_of(w.type_table), K, S, ra, rs,
                            step_count=w.step_count.cpu().numpy(), max_step=w.max_step, target=target, tiles=tiles,
                            tile_id=tile_id)
    got = o.flat.cpu().numpy()
    assert got.shape == ref.shape == (w.N, V.width(K, S))
    assert np.array_equal(o.agent_index.cpu().numpy(), ai)
    assert np.array_equal(o.segment_index.cpu().numpy(), si)
    V.compare(got, ref, K, S)
    return o


def _c2(n=4096, m=64, seed=1, max_step=50):
    from tactics2d_b200 import BatchedWorld, synthetic

    s = synthetic.config2(n, m, seed=seed)
    w = BatchedWorld(n, m, s.table, max_step=max_step)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    return w, s


def test_c2_bit_exact_with_and_without_goal(cuda_device):
    import torch
    from tactics2d_b200 import synthetic

    w, s = _c2()
    tiles = [dict(segments=s.segments, poly_start=None)]
    o = _check(w, 16, 32, 50.0, 30.0, tiles)
    assert o.flat.shape == (4096, 16 + 11 * 16 + 9 * 32)
    assert (o.agent_index >= 0).sum(1).float().mean() > 4 and (o.segment_index >= 0).any()
    for t in range(3):   # t_frac moves with the ticks
        w.step(torch.from_numpy(synthetic.random_actions(40 + t, (4096, 64))).cuda())
    rng = np.random.default_rng(2)
    x0, y0 = w.x[:, 0].cpu().numpy(), w.y[:, 0].cpu().numpy()
    target = np.stack([x0 + rng.uniform(-30, 30, 4096), y0 + rng.uniform(-30, 30, 4096), rng.uniform(0, 6.3, 4096),
                       np.full(4096, 2.5), np.full(4096, 1.2)], 1).astype(np.float32)
    w.set_goal(target)
    o = _check(w, 16, 32, 50.0, 30.0, tiles, target=target)
    assert (o.goal[:, 0] == 1).all() and (o.ego[:, 7] > 0).all()
    w.set_goal(None)
    o = _check(w, 16, 32, 50.0, 30.0, tiles)
    assert not o.goal.any()
    w.close()


def _ind_tiles():
    from tactics2d_b200.map import load_areas, polygons_to_segments

    tiles = []
    for name in ("inD_1", "inD_2"):
        areas = load_areas(name)
        xy = np.concatenate([a.outer for a in areas])
        b = (float(xy[:, 0].min()), float(xy[:, 0].max()), float(xy[:, 1].min()), float(xy[:, 1].max()))
        seg, ps = polygons_to_segments(areas, [[(b[0] + 5, b[2] + 5), (b[1] - 5, b[3] - 5)]])
        tiles.append(dict(segments=seg, poly_start=ps, bounds=b))
    return tiles


def test_c4_ind_map_table_with_rings_and_tile_rewrite(cuda_device):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    n, m = 16384, 32
    s = synthetic.config4(n, m, seed=4)
    tiles = _ind_tiles()
    assert all(t["poly_start"] is not None and len(t["poly_start"]) > 2 for t in tiles)
    rng = np.random.default_rng(3)
    tid = rng.integers(0, 2, n)
    w = BatchedWorld(n, m, s.table)
    w.set_map_table(tiles, tid)
    cx = np.asarray([(t["bounds"][0] + t["bounds"][1]) / 2 for t in tiles])[tid]
    cy = np.asarray([(t["bounds"][2] + t["bounds"][3]) / 2 for t in tiles])[tid]
    x = (cx[:, None] + rng.uniform(-40, 40, (n, m))).astype(np.float32)
    y = (cy[:, None] + rng.uniform(-40, 40, (n, m))).astype(np.float32)
    types = s.type_id.copy()
    types[rng.random((n, m)) < 0.1] = 255
    types[::97, 0] = 255   # scenarios without an ego
    w.set_state(x, y, s.heading, s.speed, type_id=types)
    for rewrite in (False, True):
        if rewrite:
            tid = 1 - tid
            w.tile_id.copy_(torch.from_numpy(tid.astype(np.int16)).to(cuda_device))
        o = _check(w, 16, 32, 50.0, 30.0, tiles, tile_id=tid)
        assert (o.segments[..., 8] == 1).any() and (o.segments[..., 8] == 0).any()   # ring edges and the open line
        assert (o.agents[..., 9] == 1).any()   # pedestrians are discs
        assert not o.flat[::97].any() and (o.agent_index[::97] == -1).all()
    w.close()


def test_round_1024x128_four_slots_per_lane(cuda_device):
    from tactics2d_b200 import BatchedWorld, synthetic
    from tactics2d_b200.map import load_collidable_segments

    seg, bounds = load_collidable_segments("rounD_0")
    s = synthetic.config5(1024, 128, seed=5, segments=seg, bounds=bounds)
    w = BatchedWorld(1024, 128, s.table)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    tiles = [dict(segments=s.segments, poly_start=None)]
    assert len(s.segments) > 256
    o = _check(w, 127, 256, 1.0e5, 1.0e5, tiles)
    assert (o.agent_index >= 0).sum(1).min() == 127   # every other slot, all four of each lane
    assert (o.segment_index >= 0).sum(1).min() == 256  # the full list, after merges past S
    _check(w, 40, 64, 60.0, 150.0, tiles)
    w.close()


def test_ties_on_lattice_points(cuda_device):
    """Participants and segments on integer lattice points around a lattice ego: many exactly equal distances, including
    across the K-th / S-th cut and across chunk boundaries of the segment merge."""
    from tactics2d_b200 import BatchedWorld, synthetic

    n, m = 256, 96
    s = synthetic.config2(n, m, seed=9)
    rng = np.random.default_rng(4)
    x = rng.integers(-6, 7, (n, m)).astype(np.float32)
    y = rng.integers(-6, 7, (n, m)).astype(np.float32)
    h = (rng.integers(0, 4, (n, m)) * (np.pi / 2)).astype(np.float32)
    g = np.arange(-8, 9, dtype=np.float32)
    segs = np.asarray([(a, b, a + 1, b) for a in g for b in g] + [(a, b, a, b + 1) for a in g for b in g] +
                      [(a, b, a, b) for a in g[::4] for b in g[::4]], np.float32)   # unit edges + zero-length pieces
    w = BatchedWorld(n, m, s.table)
    w.set_map(segs, None)
    w.set_state(x, y, h, s.speed, type_id=s.type_id)
    tiles = [dict(segments=segs, poly_start=None)]
    for K, S, ra, rs in ((5, 7, 3.0, 2.0), (30, 100, 5.0, 4.0), (95, 256, 9.0, 1.5)):
        _check(w, K, S, ra, rs, tiles)
    w.close()


def test_more_rows_than_candidates_and_zero_rows(cuda_device):
    from tactics2d_b200 import BatchedWorld, synthetic

    w, s = _c2(128, 12, seed=3)
    tiles = [dict(segments=s.segments, poly_start=None)]
    o = _check(w, 100, 200, 20.0, 5.0, tiles)
    assert (o.agent_index[:, 11:] == -1).all() and not o.agents[:, 11:].any()
    for K, S in ((0, 0), (0, 9), (7, 0)):
        o = _check(w, K, S, 20.0, 5.0, tiles)
        assert o.flat.shape[1] == 16 + 11 * K + 9 * S
    # no map at all
    w2 = BatchedWorld(128, 12, s.table)
    w2.set_state(s.x[:128], s.y[:128], s.heading[:128], s.speed[:128], type_id=s.type_id[:128])
    o = _check(w2, 4, 4, 20.0, 5.0)
    assert (o.segment_index == -1).all()
    w.close(); w2.close()


def test_scheduled_replay_after_reset_and_track_switches(cuda_device):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    ep = synthetic.highway_episodes(512, 32, seed=4, duration_ms=60000, horizon_ms=20000, length_m=150.0, rate_per_s=4.0)
    P, M = ep.type_id.shape
    w = BatchedWorld(P, M, ep.table, interval=100, max_step=200)
    w.set_log(ep.log, ep.t0, **ep.binding())
    pool = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in ep.pool.items()}
    w.type_id.copy_(torch.from_numpy(ep.type_id).cuda())
    w.reset(torch.ones(P, dtype=torch.uint8, device="cuda"), pool)
    o = _check(w, 12, 0, 60.0, 30.0)
    seen = o.agent_index.cpu().numpy()
    assert (seen >= 0).any()
    track0 = w.replay_track.clone()
    switches = 0
    for t in range(25):
        w.step(torch.zeros((P, M, 2), device="cuda"))
        switches += int((w.replay_track != track0).sum())
        track0 = w.replay_track.clone()
        if t % 6 == 5:
            o = _check(w, 12, 0, 60.0, 30.0)
            ai = o.agent_index.cpu().numpy().astype(np.int64)
            tid = w.type_id.cpu().numpy()
            rows = np.nonzero(ai >= 0)
            assert (tid[rows[0], ai[rows]] != 255).all()   # an absent track is never observed
            trk = w.replay_track.cpu().numpy()
            assert (trk[rows[0], ai[rows]] >= 0).all()
    assert switches > 0
    w.close()


def test_graph_capture_equals_eager(cuda_device):
    import torch

    w, _ = _c2(512, 64)
    eager = w.observe(16, 32).flat.clone()
    idx = w.observe(16, 32).agent_index.clone()
    g = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        w.observe(16, 32)
    torch.cuda.current_stream().wait_stream(st)
    with torch.cuda.graph(g):
        o = w.observe(16, 32)
    o.flat.zero_(); o.agent_index.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(o.flat, eager) and torch.equal(o.agent_index, idx)
    w.close()


def test_c_level_rejections_launch_nothing(cuda_device):
    import torch
    from tactics2d_b200 import _lib

    w, _ = _c2(8, 8)
    lib = w.lib
    out = torch.empty(8 * V.width(127, 256), device=cuda_device)
    ai = torch.empty(8 * 127, dtype=torch.int16, device=cuda_device)
    si = torch.empty(8 * 256, dtype=torch.int16, device=cuda_device)
    p = lambda t: C.c_void_p(t.data_ptr())
    n0 = lib.t2d_launch_count()
    nan, inf = float("nan"), float("inf")
    for K, S, ra, rs in ((-1, 4, 50, 30), (128, 4, 50, 30), (4, -1, 50, 30), (4, 257, 50, 30), (4, 4, 0, 30),
                         (4, 4, -1, 30), (4, 4, nan, 30), (4, 4, inf, 30), (4, 4, 1e6, 30), (4, 4, 50, 0), (4, 4, 50, nan),
                         (4, 4, 50, inf), (4, 4, 50, 2e5)):
        cfg = _lib.ObsConfigC(K, S, ra, rs)
        assert lib.t2d_observe(w._ctx, C.byref(cfg), p(out), p(ai), p(si), None) == -1, (K, S, ra, rs)
    cfg = _lib.ObsConfigC(4, 4, 50, 30)
    assert lib.t2d_observe(w._ctx, C.byref(cfg), None, p(ai), p(si), None) == -1
    assert lib.t2d_observe(w._ctx, None, p(out), p(ai), p(si), None) == -1
    # a context whose state is not bound
    ctx = C.c_void_p()
    _lib.check(lib.t2d_create(C.byref(ctx), 0, 8, 8, C.byref(_lib.Config(100, 5, 0, 0))))
    _lib.check(lib.t2d_set_type_table(ctx, w.type_table.to_c_array(), len(w.type_table)))
    assert lib.t2d_observe(ctx, C.byref(cfg), p(out), p(ai), p(si), None) == -4
    lib.t2d_destroy(ctx)
    assert lib.t2d_launch_count() == n0
    # the limits themselves are accepted, and NULL index arrays are allowed
    assert lib.t2d_observe(w._ctx, C.byref(_lib.ObsConfigC(127, 256, 1e5, 1e5)), p(out), None, None, None) == 0
    with pytest.raises(ValueError):
        w.observe(128, 4)
    with pytest.raises(_lib.T2DError):
        w.observe(4, 4, agent_range=0.0)
    w.close()


def test_env_vector_observation_across_auto_resets(cuda_device):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    s = synthetic.config2(64, 16, seed=2)
    cfg = dict(k_agents=8, k_segments=12, agent_range=40.0, segment_range=25.0)
    env = BatchedTrafficEnv(s, max_step=3, observation="vector", vector_obs=cfg)
    F = 16 + 11 * 8 + 9 * 12
    assert env.observation_space == {"shape": (64, F), "dtype": "float32"}
    obs, _ = env.reset()
    assert obs.shape == (64, F) and obs.dtype == torch.float32
    tiles = [dict(segments=s.segments, poly_start=None)]
    reset_seen = False
    for t in range(5):   # max_step 3: every scenario truncates and auto-resets within these steps
        obs, reward, term, trunc, info = env.step(torch.full((64, 2), 0.1, device=cuda_device))
        got = obs.clone()
        assert torch.equal(got, env.world.observe(**cfg).flat)
        _check(env.world, 8, 12, 40.0, 25.0, tiles)
        reset_seen = reset_seen or bool((env.world.step_count == 0).any())   # observed right after its auto-reset
    assert reset_seen
    env.close()
