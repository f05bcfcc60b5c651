"""K9, the per-agent vector observation (t2d_observe_agents / BatchedWorld.observe_agents), against the float64 oracle in
tests/agent_obs_oracle.py on the [N·Q, F] rows with vector_obs_oracle.compare: selection, order, indices, valid, dist,
extents, speed, t_frac and in_ring bit-exact, the rotated values within the contract's tolerance.  Also the rows observed
by slot 0 against K8, observer lists, CUDA graph = eager, the C-level rejections, the env's "agents" observation and an
output of more than 2^31 elements."""

import ctypes as C

import numpy as np
import pytest

from tests import agent_obs_oracle as A
from tests import vector_obs_oracle as V

pytestmark = pytest.mark.gpu


def _check(w, K, S, ra, rs, observers=None, goals=None, tiles=(), tile_id=None, target=None, scenarios=None):
    """Observes every scenario and compares the scenarios ``scenarios`` (default all) with the oracle."""
    import torch

    o = w.observe_agents(K, S, ra, rs, observers=observers, goals=goals)
    torch.cuda.synchronize()
    sel = np.arange(w.N) if scenarios is None else np.asarray(scenarios)
    st = {k: v[sel] for k, v in w.state_numpy().items()}
    obs = None if observers is None else observers.cpu().numpy()[sel]
    ref, ai, si = A.observe_agents(
        st, w.type_id.cpu().numpy()[sel], V.table_of(w.type_table), K, S, ra, rs, observers=obs,
        step_count=w.step_count.cpu().numpy()[sel], max_step=w.max_step, target=None if target is None else target[sel],
        goals=None if goals is None else goals.cpu().numpy()[sel], tiles=tiles,
        tile_id=None if tile_id is None else np.asarray(tile_id)[sel])
    Q = w.M if observers is None else observers.shape[1]
    F = V.width(K, S)
    idx = torch.from_numpy(sel).to(w.device)
    got = o.flat.index_select(0, idx).cpu().numpy()
    assert o.flat.shape == (w.N, Q, F) and got.shape == ref.shape
    assert np.array_equal(o.agent_index.index_select(0, idx).cpu().numpy(), ai)
    assert np.array_equal(o.segment_index.index_select(0, idx).cpu().numpy(), si)
    V.compare(got.reshape(-1, F), ref.reshape(-1, F), K, S)
    return o


def _c2(n=4096, m=64, seed=1, max_step=50):
    from tactics2d_b200 import BatchedWorld, synthetic

    s = synthetic.config2(n, m, seed=seed)
    w = BatchedWorld(n, m, s.table, max_step=max_step)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    return w, s


def _goals(w, Q, seed, nan_every=3):
    import torch

    rng = np.random.default_rng(seed)
    g = np.stack([rng.uniform(-60, 60, (w.N, Q)), rng.uniform(-60, 60, (w.N, Q)), rng.uniform(-4, 4, (w.N, Q)),
                  np.full((w.N, Q), 2.5), np.full((w.N, Q), 1.2)], -1).astype(np.float32)
    g[:, ::nan_every, 0] = np.nan
    return torch.from_numpy(g).to(w.device)


def test_c2_every_slot_with_and_without_goals_and_k8_identity(cuda_device):
    import torch
    from tactics2d_b200 import synthetic

    w, s = _c2()
    tiles = [dict(segments=s.segments, poly_start=None)]
    for t in range(2):   # t_frac moves with the ticks
        w.step(torch.from_numpy(synthetic.random_actions(40 + t, (4096, 64))).cuda())
    o = _check(w, 16, 32, 50.0, 30.0, tiles=tiles)
    assert o.flat.shape == (4096, 64, 16 + 11 * 16 + 9 * 32) and o.observers is None
    assert (o.agent_index >= 0).sum(2).float().mean() > 4 and (o.segment_index >= 0).any()
    assert (o.agent_index[:, 1:] == 0).any()   # slot 0 is observed by the others
    k8 = w.observe(16, 32)
    assert torch.equal(o.flat[:, 0].contiguous().view(torch.int32), k8.flat.view(torch.int32))
    assert torch.equal(o.agent_index[:, 0], k8.agent_index) and torch.equal(o.segment_index[:, 0], k8.segment_index)
    # the set_goal target: slot 0's rows only, still K8's row
    rng = np.random.default_rng(2)
    x0, y0 = w.x[:, 0].cpu().numpy(), w.y[:, 0].cpu().numpy()
    target = np.stack([x0 + rng.uniform(-30, 30, 4096), y0 + rng.uniform(-30, 30, 4096), rng.uniform(0, 6.3, 4096),
                       np.full(4096, 2.5), np.full(4096, 1.2)], 1).astype(np.float32)
    w.set_goal(target)
    o = _check(w, 16, 32, 50.0, 30.0, tiles=tiles, target=target)
    assert (o.goal[:, 0, 0] == 1).all() and not o.goal[:, 1:].any()
    k8 = w.observe(16, 32)
    assert torch.equal(o.flat[:, 0].contiguous().view(torch.int32), k8.flat.view(torch.int32))
    # per-row goals replace it; a NaN cx gives the zero block
    goals = _goals(w, 64, 3)
    o = _check(w, 16, 32, 50.0, 30.0, goals=goals, tiles=tiles, target=target)
    assert not o.goal[:, ::3].any() and (o.goal[:, 1::3, 0] == 1).all()
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
    w.set_state(x, y, s.heading, s.speed, type_id=types)
    sel = np.arange(0, n, 11)   # the oracle on every 11th scenario
    for rewrite in (False, True):
        if rewrite:
            tid = 1 - tid
            w.tile_id.copy_(torch.from_numpy(tid.astype(np.int16)).to(cuda_device))
        o = _check(w, 16, 32, 50.0, 30.0, tiles=tiles, tile_id=tid, scenarios=sel)
        assert (o.segments[..., 8] == 1).any() and (o.segments[..., 8] == 0).any()   # ring edges and the open line
        assert (o.agents[..., 9] == 1).any()   # pedestrians are discs
        empty = torch.from_numpy(types >= len(w.type_table)).to(cuda_device)
        assert not o.flat[empty].any() and (o.agent_index[empty] == -1).all()
    w.close()


def test_round_1024x128_every_slot_and_full_lists(cuda_device):
    from tactics2d_b200 import BatchedWorld, synthetic
    from tactics2d_b200.map import load_collidable_segments

    seg, bounds = load_collidable_segments("rounD_0")
    s = synthetic.config5(1024, 128, seed=5, segments=seg, bounds=bounds)
    w = BatchedWorld(1024, 128, s.table)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    tiles = [dict(segments=s.segments, poly_start=None)]
    assert len(s.segments) > 256
    _check(w, 16, 32, 50.0, 30.0, tiles=tiles)
    o = _check(w, 127, 256, 1.0e5, 1.0e5, tiles=tiles, scenarios=np.arange(0, 1024, 16))
    assert (o.agent_index >= 0).sum(2).min() == 127 and (o.segment_index >= 0).sum(2).min() == 256
    w.close()


def test_observer_lists(cuda_device):
    import torch

    w, s = _c2(256, 12, seed=3)
    tiles = [dict(segments=s.segments, poly_start=None)]
    rng = np.random.default_rng(6)
    dev = w.device
    lists = [
        rng.integers(0, 12, (256, 5)),                         # random subsets, duplicates included
        np.tile(np.asarray([-1, 0, 12, 11, 300, -7, 5, 5]), (256, 1)),   # -1, out of range, duplicates
        rng.integers(-3, 15, (256, 40)),                       # Q > M with an explicit list
        rng.integers(0, 12, (256, 128)),                       # the largest Q
        np.zeros((256, 1)),                                    # the ego alone
    ]
    for obs in lists:
        t = torch.from_numpy(obs.astype(np.int16)).to(dev)
        o = _check(w, 6, 9, 20.0, 5.0, observers=t, tiles=tiles)
        assert o.observers is t
    # duplicates give equal rows, a list equals the matching rows of the every-slot call
    t = torch.from_numpy(lists[0].astype(np.int16)).to(dev)
    o = w.observe_agents(6, 9, 20.0, 5.0, observers=t)
    part = o.flat.clone()
    full = w.observe_agents(6, 9, 20.0, 5.0).flat
    assert torch.equal(part, torch.gather(full, 1, t.long()[..., None].expand(-1, -1, full.shape[2])))
    # the counts of the every-slot call and the absent rows of empty slots
    empty = np.zeros((256, 12), np.uint8)
    empty[:, 3] = 255
    w.type_id.copy_(torch.from_numpy(np.where(empty == 255, 255, w.type_id.cpu().numpy())).to(dev))
    o = _check(w, 6, 9, 20.0, 5.0, tiles=tiles)
    assert not o.flat[:, 3].any() and (o.agent_index[:, 3] == -1).all() and not (o.agent_index == 3).any()
    w.close()


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
    obs = torch.from_numpy(np.random.default_rng(1).integers(0, M, (P, 8)).astype(np.int16)).cuda()
    o = _check(w, 12, 0, 60.0, 30.0, observers=obs)
    assert (o.agent_index >= 0).any()
    track0 = w.replay_track.clone()
    switches = 0
    for t in range(25):
        w.step(torch.zeros((P, M, 2), device="cuda"))
        switches += int((w.replay_track != track0).sum())
        track0 = w.replay_track.clone()
        if t % 6 == 5:
            o = _check(w, 12, 0, 60.0, 30.0, observers=obs)
            ai = o.agent_index.cpu().numpy().astype(np.int64)
            tid = w.type_id.cpu().numpy()
            n_idx, q_idx, k_idx = np.nonzero(ai >= 0)
            assert (tid[n_idx, ai[n_idx, q_idx, k_idx]] != 255).all()   # an absent track is never observed
            absent = tid[np.arange(P)[:, None], obs.cpu().numpy().astype(np.int64)] == 255
            assert not o.flat[torch.from_numpy(absent).cuda()].any()      # nor does it observe
    assert switches > 0
    w.close()


def test_graph_capture_equals_eager(cuda_device):
    import torch

    w, _ = _c2(512, 64)
    obs = torch.from_numpy(np.random.default_rng(2).integers(-1, 64, (512, 24)).astype(np.int16)).cuda()
    goals = _goals(w, 24, 4)
    for kw in (dict(), dict(observers=obs, goals=goals)):
        o = w.observe_agents(16, 32, **kw)
        eager, idx, sidx = o.flat.clone(), o.agent_index.clone(), o.segment_index.clone()
        g = torch.cuda.CUDAGraph()
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            w.observe_agents(16, 32, **kw)
        torch.cuda.current_stream().wait_stream(st)
        with torch.cuda.graph(g):
            o = w.observe_agents(16, 32, **kw)
        o.flat.zero_(); o.agent_index.zero_(); o.segment_index.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(o.flat, eager) and torch.equal(o.agent_index, idx) and torch.equal(o.segment_index, sidx)
    w.close()


def test_c_level_rejections_launch_nothing(cuda_device):
    import torch
    from tactics2d_b200 import _lib

    w, _ = _c2(8, 8)
    lib = w.lib
    out = torch.empty(8 * 128 * V.width(127, 256), device=cuda_device)
    ai = torch.empty(8 * 128 * 127, dtype=torch.int16, device=cuda_device)
    si = torch.empty(8 * 128 * 256, dtype=torch.int16, device=cuda_device)
    obs = torch.zeros(8 * 128, dtype=torch.int16, device=cuda_device)
    p = lambda t: C.c_void_p(t.data_ptr())
    call = lambda ctx, cfg, o, q, g, out_: lib.t2d_observe_agents(ctx, cfg, o, q, g, out_, p(ai), p(si), None)
    n0 = lib.t2d_launch_count()
    nan, inf = float("nan"), float("inf")
    for K, S, ra, rs in ((-1, 4, 50, 30), (128, 4, 50, 30), (4, -1, 50, 30), (4, 257, 50, 30), (4, 4, 0, 30),
                         (4, 4, -1, 30), (4, 4, nan, 30), (4, 4, inf, 30), (4, 4, 1e6, 30), (4, 4, 50, 0), (4, 4, 50, nan),
                         (4, 4, 50, inf), (4, 4, 50, 2e5)):
        cfg = _lib.ObsConfigC(K, S, ra, rs)
        assert call(w._ctx, C.byref(cfg), p(obs), 4, None, p(out)) == -1, (K, S, ra, rs)
    cfg = _lib.ObsConfigC(4, 4, 50, 30)
    assert call(w._ctx, C.byref(cfg), p(obs), 4, None, None) == -1          # no output
    assert call(w._ctx, None, p(obs), 4, None, p(out)) == -1                # no config
    assert call(None, C.byref(cfg), p(obs), 4, None, p(out)) == -1          # no context
    for q in (0, -1, 129):                                                  # Q outside 1..128
        assert call(w._ctx, C.byref(cfg), p(obs), q, None, p(out)) == -1, q
    assert call(w._ctx, C.byref(cfg), None, 9, None, p(out)) == -1          # every slot, Q > M
    ctx = C.c_void_p()   # a context whose state is not bound
    _lib.check(lib.t2d_create(C.byref(ctx), 0, 8, 8, C.byref(_lib.Config(100, 5, 0, 0))))
    _lib.check(lib.t2d_set_type_table(ctx, w.type_table.to_c_array(), len(w.type_table)))
    assert call(ctx, C.byref(cfg), p(obs), 4, None, p(out)) == -4
    lib.t2d_destroy(ctx)
    assert lib.t2d_launch_count() == n0
    # the limits themselves are accepted, NULL index arrays too, and Q > M with a list
    big = _lib.ObsConfigC(127, 256, 1e5, 1e5)
    assert lib.t2d_observe_agents(w._ctx, C.byref(big), p(obs), 128, None, p(out), None, None, None) == 0
    assert lib.t2d_observe_agents(w._ctx, C.byref(big), None, 8, None, p(out), None, None, None) == 0
    assert lib.t2d_launch_count() == n0 + 2
    # the Python checks keep host tensors, wrong dtypes and shapes away from the kernel
    with pytest.raises(ValueError):
        w.observe_agents(128, 4)
    with pytest.raises(ValueError):
        w.observe_agents(observers=torch.zeros((8, 2), dtype=torch.int16))               # host tensor
    with pytest.raises(ValueError):
        w.observe_agents(observers=torch.zeros((8, 2), dtype=torch.int32, device=cuda_device))
    with pytest.raises(ValueError):
        w.observe_agents(observers=torch.zeros((8, 129), dtype=torch.int16, device=cuda_device))
    with pytest.raises(ValueError):
        w.observe_agents(observers=torch.zeros((4, 2), dtype=torch.int16, device=cuda_device))
    with pytest.raises(ValueError):
        w.observe_agents(goals=torch.zeros((8, 7, 5), device=cuda_device))
    with pytest.raises(ValueError):
        w.observe_agents(goals=torch.zeros((8, 5, 8), device=cuda_device).transpose(1, 2))
    with pytest.raises(_lib.T2DError):
        w.observe_agents(4, 4, agent_range=0.0)
    w.close()


def test_env_agents_observation_across_auto_resets(cuda_device):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    s = synthetic.config2(64, 16, seed=2)
    obs = torch.from_numpy(np.random.default_rng(3).integers(0, 16, (64, 5)).astype(np.int16)).to(cuda_device)
    for cfg, Q in ((dict(k_agents=8, k_segments=12, agent_range=40.0, segment_range=25.0), 16),
                   (dict(k_agents=4, k_segments=6, observers=obs), 5)):
        env = BatchedTrafficEnv(s, max_step=3, observation="agents", vector_obs=cfg)
        F = V.width(cfg["k_agents"], cfg["k_segments"])
        assert env.observation_space == {"shape": (64, Q, F), "dtype": "float32"}
        o, _ = env.reset()
        assert o.shape == (64, Q, F) and o.dtype == torch.float32
        tiles = [dict(segments=s.segments, poly_start=None)]
        reset_seen = False
        for t in range(5):   # max_step 3: every scenario truncates and auto-resets within these steps
            o, reward, term, trunc, info = env.step(torch.full((64, 2), 0.1, device=cuda_device))
            got = o.clone()
            assert torch.equal(got, env.world.observe_agents(**cfg).flat)
            _check(env.world, cfg["k_agents"], cfg["k_segments"], cfg.get("agent_range", 50.0),
                   cfg.get("segment_range", 30.0), observers=cfg.get("observers"), tiles=tiles)
            reset_seen = reset_seen or bool((env.world.step_count == 0).any())
        assert reset_seen
        env.close()
    with pytest.raises(ValueError):
        BatchedTrafficEnv(s, observation="vector", vector_obs=dict(observers=obs))


def test_output_beyond_2_to_the_31_elements(cuda_device):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic
    from tactics2d_b200.map import load_collidable_segments

    free, _ = torch.cuda.mem_get_info()
    if free < 20 * 2**30:
        pytest.skip(f"needs 20 GB of free device memory, {free / 2**30:.1f} GB free")
    n, m, K, S = 4608, 128, 127, 256
    assert n * m * V.width(K, S) > 2**31
    seg, bounds = load_collidable_segments("rounD_0")
    s = synthetic.config5(n, m, seed=7, segments=seg, bounds=bounds)
    w = BatchedWorld(n, m, s.table)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    tiles = [dict(segments=s.segments, poly_start=None)]
    o = _check(w, K, S, 1.0e5, 1.0e5, tiles=tiles, scenarios=np.arange(n - 3, n))
    assert (o.agent_index[-1] >= 0).all() and (o.segment_index[-1] >= 0).all()
    del o
    w.__dict__.pop("_agent_obs_out", None)
    w.close()
    torch.cuda.empty_cache()
