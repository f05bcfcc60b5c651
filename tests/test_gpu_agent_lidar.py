"""The per-agent lidar (K4 over observer rows: t2d_lidar_scan_agents / BatchedWorld.lidar_scan_agents) against the float64
statement in tests/agent_lidar_oracle.py with the lidar tests' criterion (the same inf pattern, hits within
2e-6·R + 1e-6).  Also: rows observed by slot 0 bit-equal to the ego scan, observer lists, dense and touching scenes seen
from a slot other than 0, retirement and reset, CUDA graph = eager, an output of more than 2^31 elements, the C-level
rejections and the env's info["lidar"]."""

import ctypes as C

import numpy as np
import pytest

from tests import agent_lidar_oracle as AL

pytestmark = pytest.mark.gpu


def _check(w, n_beams, max_range, observers=None, scenarios=None, segments=None, tiles=None, tile_id=None, got=None):
    """Scans every scenario (unless ``got`` is given) and compares the scenarios ``scenarios`` (default all) with the
    oracle; returns the device scan and the oracle's rows."""
    import torch

    if got is None:
        got = w.lidar_scan_agents(n_beams, max_range, observers=observers)
    torch.cuda.synchronize()
    sel = np.arange(w.N) if scenarios is None else np.asarray(scenarios)
    st = w.state_numpy()
    f64 = lambda k: st[k][sel].astype(np.float64)
    obs = None if observers is None else observers.cpu().numpy()[sel]
    ref = AL.scan_agents(f64("x"), f64("y"), f64("heading"), w.type_id.cpu().numpy()[sel], w.type_table.as_oracle_table(),
                         n_beams, max_range, observers=obs, segments=segments, tiles=tiles,
                         tile_id=None if tile_id is None else np.asarray(tile_id)[sel])
    idx = torch.from_numpy(sel).to(w.device)
    AL.compare(got.index_select(0, idx).cpu().numpy(), ref, max_range)
    return got, ref


def _c2(n=4096, m=64, seed=1):
    from tactics2d_b200 import BatchedWorld, synthetic

    s = synthetic.config2(n, m, seed=seed)
    w = BatchedWorld(n, m, s.table)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    return w, s


@pytest.mark.parametrize("n_beams,max_range", [(360, 20.0), (500, 12.0), (1100, 9.0)])
def test_c2_every_slot_and_the_ego_scan_bit_for_bit(cuda_device, n_beams, max_range):
    import torch

    w, s = _c2()
    scan = w.lidar_scan_agents(n_beams, max_range).clone()   # (the next call with these arguments reuses the buffer)
    assert scan.shape == (4096, 64, n_beams) and scan.dtype == torch.float32
    ego = w.lidar_scan(n_beams, max_range)
    assert torch.equal(scan[:, 0], ego)
    zeros = torch.zeros((4096, 1), dtype=torch.int16, device=cuda_device)
    assert torch.equal(w.lidar_scan_agents(n_beams, max_range, observers=zeros)[:, 0], ego)
    sel = np.arange(0, 4096, 86)[:48]
    _, ref = _check(w, n_beams, max_range, scenarios=sel, segments=s.segments, got=scan)
    assert np.isfinite(ref).mean() > 0.05
    # slot 0's box is seen by the other rows: scans of the same rows without it differ
    w.type_id[:, 0] = 255
    without = w.lidar_scan_agents(n_beams, max_range)
    assert not torch.equal(without[:, 1:], scan[:, 1:]) and torch.isinf(without[:, 0]).all()
    w.close()


def _tiles():
    from tactics2d_b200 import synthetic

    return [synthetic.grid_wall_segments(60.0, 30.0, 14.0), synthetic.grid_wall_segments(60.0, 20.0, 9.0),
            np.asarray([[10.0, 10.0, 50.0, 12.0], [30.0, 0.0, 31.0, 60.0]], np.float32)]


def test_mixed_traffic_map_table_and_observer_lists(cuda_device):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    n, m = 512, 32
    s = synthetic.with_inactive(synthetic.config4(n, m, seed=41, size=60.0), 0.15, seed=3)
    tiles = _tiles()
    rng = np.random.default_rng(5)
    tid = rng.integers(0, 3, n)
    w = BatchedWorld(n, m, s.table)
    w.set_map_table([dict(segments=t, bounds=s.bounds, poly_start=None) for t in tiles], tid)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    assert (s.type_id == 255).any() and (s.table.as_oracle_table()["shape"][s.type_id[s.type_id < 255]] == 1).any()
    sel = np.arange(0, n, 13)
    lists = [
        None,                                                        # every slot, empty ones included
        np.tile(np.asarray([-1, 0, m, 7, 7, 300, -7, 31, 2, 2]), (n, 1)),   # -1, M, out of range, duplicates
        rng.integers(-3, m + 3, (n, 40)),                            # Q > M with a list
        rng.integers(0, m, (n, 128)),                                # the largest Q
    ]
    for obs in lists:
        t = None if obs is None else torch.from_numpy(obs.astype(np.int16)).to(cuda_device)
        got, ref = _check(w, 360, 20.0, observers=t, scenarios=sel, tiles=tiles, tile_id=tid)
        assert np.isfinite(ref).any()
        if obs is not None:   # absent rows and duplicates
            o = obs[sel]
            absent = (o < 0) | (o >= m) | (s.type_id[sel[:, None], np.clip(o, 0, m - 1)] == 255)
            assert np.isinf(got.cpu().numpy()[sel][absent]).all()
            full = w.lidar_scan_agents(360, 20.0)   # (a buffer of its own: Q = M is none of the lists' Q)
            same = torch.gather(full, 1, t.long().clamp(0, m - 1)[..., None].expand(-1, -1, 360))
            ok = torch.from_numpy(~((obs < 0) | (obs >= m))).to(cuda_device)
            assert torch.equal(got[ok], same[ok])
    w.close()


def test_dense_and_touching_scenes_seen_from_slot_k(cuda_device):
    """The dense-scene cases of the ego scan from a slot k != 0: a box on top of the observer, boxes with the observer's
    centre (edges through the sensor get every beam), windows wrapping beam 0, several 512-beam passes."""
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    n, m, k = 24, 24, 5
    scene = synthetic.config4(n, m, seed=13, size=18.0, segments=synthetic.grid_wall_segments(18.0, 9.0, 5.0))
    scene.type_id[:, [0, k, k + 1]] = 2
    scene.x[:4, k + 1], scene.y[:4, k + 1] = scene.x[:4, k] + 0.3, scene.y[:4, k] - 0.2
    scene.x[4:8, k + 1], scene.y[4:8, k + 1] = scene.x[4:8, k], scene.y[4:8, k]
    scene.x[8:12, 0], scene.y[8:12, 0] = scene.x[8:12, k] - 0.2, scene.y[8:12, k] + 0.1   # slot 0 on top of slot k
    w = BatchedWorld(n, m, scene.table)
    w.set_map(scene.segments, scene.bounds)
    w.set_state(scene.x, scene.y, scene.heading, scene.speed, type_id=scene.type_id)
    obs = torch.from_numpy(np.tile(np.asarray([k, 0, k + 1, 1], np.int16), (n, 1))).to(cuda_device)
    got, ref = _check(w, 1100, 9.0, observers=obs, segments=scene.segments)
    assert np.isfinite(ref[:, 0]).mean() > 0.5
    assert np.isfinite(ref[:8, 0]).all()   # the box on the sensor is hit by every beam
    w.close()


def test_retired_slots_are_absent_and_unseen_until_reset(cuda_device):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    N, M = 512, 16
    s = synthetic.config2(N, M, seed=21)
    w = BatchedWorld(N, M, s.table, max_step=1000)
    w.set_map(s.segments, s.bounds)
    pool = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in s.state().items()}
    w.type_id.copy_(torch.from_numpy(s.type_id).cuda())
    w.reset(torch.ones(N, dtype=torch.uint8, device="cuda"), pool)
    w.set_agents()
    types0 = w.type_id.clone()
    for t in range(6):
        w.step(torch.from_numpy(synthetic.random_actions(900 + t, (N, M))).cuda())
        w.agents_epilogue()
    gone = w.type_id == 255
    assert gone.sum() > 20
    scan = w.lidar_scan_agents(360, 20.0).clone()
    assert torch.isinf(scan[gone]).all()
    sel = torch.nonzero(gone.any(1)).flatten().cpu().numpy()[:40]
    _check(w, 360, 20.0, scenarios=sel, segments=s.segments, got=scan)
    # the same world with the retired slots back in place: some other row saw one of them
    w.type_id.copy_(types0)
    back = w.lidar_scan_agents(360, 20.0).clone()
    assert not torch.equal(back[~gone], scan[~gone])
    w.type_id.copy_(torch.where(gone, torch.full_like(types0, 255), types0))
    mask = torch.zeros(N, dtype=torch.uint8, device=cuda_device)
    mask[::2] = 1
    w.reset(mask, pool)
    m = mask.bool()
    assert torch.equal(w.type_id[m], types0[m])
    after = w.lidar_scan_agents(360, 20.0)
    restored = gone & m[:, None]
    assert restored.any() and torch.isfinite(after[restored]).any()
    _check(w, 360, 20.0, scenarios=sel, segments=s.segments)
    w.close()


def test_graph_capture_equals_eager(cuda_device):
    import torch

    w, _ = _c2(512, 64)
    obs = torch.from_numpy(np.random.default_rng(2).integers(-1, 64, (512, 24)).astype(np.int16)).cuda()
    for kw in (dict(), dict(observers=obs)):
        eager = w.lidar_scan_agents(500, 12.0, **kw).clone()
        g = torch.cuda.CUDAGraph()
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            w.lidar_scan_agents(500, 12.0, **kw)
        torch.cuda.current_stream().wait_stream(st)
        with torch.cuda.graph(g):
            out = w.lidar_scan_agents(500, 12.0, **kw)
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager)
    w.close()


def test_output_beyond_2_to_the_31_elements(cuda_device):
    import torch

    free, _ = torch.cuda.mem_get_info()
    if free < 12 * 2**30:
        pytest.skip(f"needs 12 GB of free device memory, {free / 2**30:.1f} GB free")
    n, q, b = 4096, 128, 4200
    assert n * q * b > 2**31
    w, s = _c2(n, 64, seed=3)
    obs = torch.from_numpy(np.random.default_rng(8).integers(0, 64, (n, q)).astype(np.int16)).to(cuda_device)
    got = w.lidar_scan_agents(b, 20.0, observers=obs)
    _, ref = _check(w, b, 20.0, observers=obs, scenarios=np.arange(n - 2, n), segments=s.segments, got=got)
    assert np.isfinite(ref).any()
    del got
    w.__dict__.pop("_agent_lidar", None)
    w.close()
    torch.cuda.empty_cache()


def test_c_level_rejections_launch_nothing(cuda_device):
    import torch
    from tactics2d_b200 import _lib

    w, _ = _c2(8, 8)
    lib = w.lib
    scan = torch.full((8 * 128 * 64,), 7.0, device=cuda_device)
    cs = torch.zeros((64, 2), dtype=torch.float64, device=cuda_device)
    obs = torch.zeros(8 * 128, dtype=torch.int16, device=cuda_device)
    p = lambda t: C.c_void_p(t.data_ptr())
    call = lambda ctx, o, q, nb, r, c_, s_: lib.t2d_lidar_scan_agents(ctx, o, q, nb, r, c_, s_, None)
    n0 = lib.t2d_launch_count()
    for q in (0, -1, 129):                                                   # Q outside 1..128
        assert call(w._ctx, p(obs), q, 64, 12.0, p(cs), p(scan)) == -1, q
    assert call(w._ctx, None, 9, 64, 12.0, p(cs), p(scan)) == -1             # every slot, Q > M
    for nb in (0, -5):
        assert call(w._ctx, p(obs), 4, nb, 12.0, p(cs), p(scan)) == -1, nb
    for r in (0.0, -1.0, float("nan"), -float("inf")):
        assert call(w._ctx, p(obs), 4, 64, r, p(cs), p(scan)) == -1, r
    assert call(w._ctx, p(obs), 4, 64, 12.0, None, p(scan)) == -1            # no beam table
    assert call(w._ctx, p(obs), 4, 64, 12.0, p(cs), None) == -1              # no output
    assert call(None, p(obs), 4, 64, 12.0, p(cs), p(scan)) == -1             # no context
    ctx = C.c_void_p()   # a context whose state is not bound
    _lib.check(lib.t2d_create(C.byref(ctx), 0, 8, 8, C.byref(_lib.Config(100, 5, 0, 0))))
    _lib.check(lib.t2d_set_type_table(ctx, w.type_table.to_c_array(), len(w.type_table)))
    assert call(ctx, p(obs), 4, 64, 12.0, p(cs), p(scan)) == -4
    lib.t2d_destroy(ctx)
    torch.cuda.synchronize()
    assert lib.t2d_launch_count() == n0 and (scan == 7.0).all()
    # the limits themselves are accepted, and Q > M with a list
    assert call(w._ctx, p(obs), 128, 64, 12.0, p(cs), p(scan)) == 0
    assert call(w._ctx, None, 8, 64, 12.0, p(cs), p(scan)) == 0
    assert lib.t2d_launch_count() == n0 + 2
    # the Python checks keep host tensors, wrong dtypes and shapes away from the kernel
    for bad in (torch.zeros((8, 2), dtype=torch.int16),                              # host tensor
                torch.zeros((8, 2), dtype=torch.int32, device=cuda_device),          # wrong dtype
                torch.zeros((8, 129), dtype=torch.int16, device=cuda_device),        # Q > 128
                torch.zeros((4, 2), dtype=torch.int16, device=cuda_device),          # wrong N
                torch.zeros((8,), dtype=torch.int16, device=cuda_device),            # one dimension
                torch.zeros((2, 8), dtype=torch.int16, device=cuda_device).t()):     # not contiguous
        with pytest.raises(ValueError):
            w.lidar_scan_agents(64, 12.0, observers=bad)
    with pytest.raises(_lib.T2DError):
        w.lidar_scan_agents(64, 0.0)
    w.close()


def test_sensor_scan_agents(cuda_device):
    import torch
    from tactics2d_b200.sensor import SingleLineLidar

    w, _ = _c2(64, 16)
    lidar = SingleLineLidar(perception_range=20.0, freq_scan=10.0, freq_detect=3600.0)
    got = lidar.scan_agents(w)
    assert got.shape == (64, 16, 360) and lidar.scan_result is None
    assert torch.equal(got, w.lidar_scan_agents(360, 20.0))
    assert torch.equal(lidar.scan(w), got[:, 0])
    w.close()


@pytest.mark.parametrize("mode", ["state", "agents"])
def test_env_info_lidar_after_auto_resets(cuda_device, mode):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    n, m = 64, 16
    s = synthetic.config2(n, m, seed=2)
    obs = torch.from_numpy(np.random.default_rng(3).integers(0, m, (n, 5)).astype(np.int16)).to(cuda_device)
    kw = dict(observation=mode, lidar=dict(n_beams=360, max_range=20.0))
    if mode == "agents":
        kw.update(vector_obs=dict(k_agents=4, k_segments=6, observers=obs), agent_rewards=True, agent_actions=True)
    env = BatchedTrafficEnv(s, max_step=3, **kw)
    _, info = env.reset()
    shape = (n, 5, 360) if mode == "agents" else (n, 360)
    assert info["lidar"].shape == shape
    act = torch.full(env.action_space["shape"], 0.1, device=cuda_device)
    reset_seen = False
    for t in range(5):   # max_step 3: every scenario ends and auto-resets within these steps
        out = env.step(act)
        info = out[4]
        got = info["lidar"].clone()
        want = (env.world.lidar_scan_agents(360, 20.0, observers=obs) if mode == "agents" else env.world.lidar_scan(360, 20.0))
        assert got.shape == shape and torch.equal(got, want)
        reset_seen = reset_seen or bool((env.world.step_count == 0).any())
    assert reset_seen
    env.close()
    plain = BatchedTrafficEnv(s, max_step=3)
    _, info = plain.reset()
    assert "lidar" not in info and "lidar" not in plain.step(torch.zeros((n, 2), device=cuda_device))[4]
    plain.close()
    with pytest.raises(ValueError):
        BatchedTrafficEnv(s, lidar=dict(n_beams=360, range=20.0))
