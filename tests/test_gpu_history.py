"""The trajectory history on the device (t2d_set_history / K15 / K16; DESIGN.md section 1 "Trajectory history") against
``tests/history_oracle.py``: the ring after every tick path and reset, bit for bit; a rollout with a ring computing what
one without it computes; validity through retirements, absent replay tracks and schedule switches; K16 at every lag, with
its lag-0 identity to K8 / K9; the env's ``info["history"]`` across auto-resets; and the rejections."""

import ctypes as C

import numpy as np
import pytest

from tests import history_oracle as HO

pytestmark = pytest.mark.gpu

SENTINEL = -7.25


def _world(n=256, m=64, seed=1, max_step=0, **kw):
    from tactics2d_b200 import BatchedWorld, synthetic

    s = synthetic.config2(n, m, seed=seed)
    w = BatchedWorld(n, m, s.table, max_step=max_step, **kw)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    return w, s


def _pool(w):
    import torch

    return {k: getattr(w, k).clone() for k in ("x", "y", "heading", "speed")}, torch.ones(w.N, dtype=torch.uint8, device=w.device)


def _snap(w):
    st = w.state_numpy()
    trk = None if w.replay_track is None else w.replay_track.cpu().numpy()
    return st, w.type_id.cpu().numpy(), trk


def _check_ring(w, ring, what=""):
    """history() equals the oracle ring's view bit for bit (fields, types, valid, count)."""
    st, tid, trk = _snap(w)
    got = {k: v.cpu().numpy() for k, v in w.history().items()}
    ref = ring.view(tid, len(w.type_table), trk)
    assert np.array_equal(got["count"], ref["count"]), what
    assert np.array_equal(got["valid"], ref["valid"]), (what, np.argwhere(got["valid"] != ref["valid"])[:5])
    for k in HO.FIELDS:
        assert np.array_equal(got[k].view(np.uint32), ref[k].view(np.uint32)), (what, k)
    assert np.array_equal(got["type_id"], ref["type_id"]), what


def _tick(w, mode, t, act_all):
    import torch

    a = act_all[t % len(act_all)]
    if mode == "step":
        w.step(torch.from_numpy(a).cuda())
    elif mode == "step_host":
        w.step_host(a)
    elif mode == "step_host_ego":
        w.step_host_ego(np.ascontiguousarray(a[:, 0]))
    elif mode == "step_host_agents":
        w.step_host_agents(np.ascontiguousarray(a[:, :w._agents["Q"]]))
    else:
        raise ValueError(mode)


def _actions(n, m, seed=5, k=8):
    from tactics2d_b200 import synthetic

    return [synthetic.random_actions(seed + i, (n, m)) for i in range(k)]


@pytest.mark.parametrize("H", [1, 2, 7, 64])
@pytest.mark.parametrize("generic", [False, True])
def test_recording_after_every_tick_bit_exact(cuda_device, monkeypatch, H, generic):
    from tactics2d_b200 import _lib

    if generic:
        monkeypatch.setenv("T2D_TICK_GENERIC", "1")
    w, _ = _world()
    lib = _lib.load()
    fixed0 = lib.t2d_tick_fixed_count()
    w.set_history(H)
    ring = HO.Ring(w.N, w.M, H)
    _check_ring(w, ring, "a new binding is empty")
    pool, mask = _pool(w)
    w.reset(mask, pool)
    st, tid, _ = _snap(w)
    ring.restart(np.ones(w.N), st, tid)
    acts = _actions(w.N, w.M)
    checkpoints = {0, 1, H - 1, H, 3 * H + 1}
    _check_ring(w, ring, "R=0")
    for t in range(1, 3 * H + 2):
        _tick(w, "step", t, acts)
        st, tid, _ = _snap(w)
        ring.append(st, tid)
        if t in checkpoints:
            _check_ring(w, ring, f"H={H} R={t}")
    assert (lib.t2d_tick_fixed_count() > fixed0) == (not generic)   # the instance the case is about ran
    w.close()


@pytest.mark.parametrize("mode", ["step_host", "step_host_chunks", "step_host_ego", "step_host_agents"])
def test_recording_through_the_host_steps(cuda_device, monkeypatch, mode):
    if mode == "step_host_chunks":
        monkeypatch.setenv("T2D_HOST_CHUNKS", "3")
        mode = "step_host"
    w, _ = _world(n=257)
    if mode == "step_host_agents":
        w.set_agents(None)
    H = 7
    w.set_history(H)
    ring = HO.Ring(w.N, w.M, H)
    pool, mask = _pool(w)
    w.reset(mask, pool)
    st, tid, _ = _snap(w)
    ring.restart(np.ones(w.N), st, tid)
    acts = _actions(w.N, w.M, seed=9)
    for t in range(1, 3 * H + 2):
        st0, tid0, _ = _snap(w)
        _tick(w, mode, t, acts)
        st, _, _ = _snap(w)
        # K10 (step_host_agents) may retire slots after the append: the ring holds the post-tick types, before K10
        ring.append(st, tid0 if mode == "step_host_agents" else _snap(w)[1])
    _check_ring(w, ring, mode)
    w.close()


def test_env_path_and_host_agents_leave_identical_rings(cuda_device):
    import torch

    ws = []
    for _ in range(2):
        w, _ = _world(n=130)
        w.set_agents(None)
        w.set_history(5)
        pool, mask = _pool(w)
        w.reset(mask, pool)
        ws.append(w)
    acts = _actions(130, 64, seed=21)
    for t in range(9):
        a = acts[t % len(acts)]
        ws[0].step(torch.from_numpy(a).cuda())
        ws[0].agents_epilogue()
        ws[1].step_host_agents(np.ascontiguousarray(a))
    h0, h1 = ws[0].history(), ws[1].history()
    for k in h0:
        assert torch.equal(h0[k], h1[k]), k


def test_history_leaves_the_rollout_alone(cuda_device):
    """A 50-tick C2 rollout with a ring computes exactly what one without it computes."""
    import torch
    from tactics2d_b200 import _lib

    lib = _lib.load()
    acts = _actions(1024, 64, seed=33)
    outs = []
    for H in (0, 16):
        w, _ = _world(n=1024)
        if H:
            w.set_history(H)
        f0 = lib.t2d_tick_order_fallback_count()
        rec = []
        for t in range(50):
            r = w.step(torch.from_numpy(acts[t % len(acts)]).cuda())
            rec.append([r.flags.clone(), r.hit_index.clone(), r.hit_segment.clone(), r.status.clone(), r.done.clone()])
        torch.cuda.synchronize()
        st = w.state_numpy()
        outs.append((st, rec, lib.t2d_tick_order_fallback_count() - f0))
        w.close()
    (s0, r0, f0), (s1, r1, f1) = outs
    for k in s0:
        assert np.array_equal(s0[k].view(np.uint32), s1[k].view(np.uint32)), k
    for a, b in zip(r0, r1):
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    assert f0 == f1


def test_masked_restarts(cuda_device):
    import torch

    w, s = _world(n=200)
    H = 4
    w.set_history(H)
    ring = HO.Ring(w.N, w.M, H)
    pool, mask = _pool(w)
    w.reset(mask, pool)
    st, tid, _ = _snap(w)
    ring.restart(np.ones(w.N), st, tid)
    acts = _actions(w.N, w.M, seed=3)
    for t in range(6):
        _tick(w, "step", t, acts)
        st, tid, _ = _snap(w)
        ring.append(st, tid)
    m = (np.arange(w.N) % 3 == 1).astype(np.uint8)
    w.reset(torch.from_numpy(m).cuda(), pool)
    st, tid, _ = _snap(w)
    ring.restart(m, st, tid)
    _check_ring(w, ring, "reset")
    # a sampled reset with jitter: entry 0 is the placed state
    jit = np.tile(np.array([[-0.5, 0.5], [-0.5, 0.5], [-0.1, 0.1], [-0.5, 0.5]], np.float32), (w.M, 1, 1))
    w.set_reset_sampler(seed=4, jitter=jit, tries=8)
    for t in range(3):
        _tick(w, "step", t, acts)
        st, tid, _ = _snap(w)
        ring.append(st, tid)
    m = (np.arange(w.N) % 4 == 2).astype(np.uint8)
    w.reset_sampled(torch.from_numpy(m).cuda(), pool)
    st, tid, _ = _snap(w)
    ring.restart(m, st, tid)
    assert (w.reset_try.cpu().numpy()[m.astype(bool)] >= 0).any()   # some slots moved
    _check_ring(w, ring, "reset_sampled")
    h = w.history()
    sel = torch.from_numpy(m.astype(bool)).cuda()
    assert (h["count"][sel] == 1).all() and torch.equal(h["x"][sel][:, :, 0], w.x[sel])


def test_retired_slots_lose_their_history(cuda_device):
    import torch

    w, s = _world(n=64)
    w.set_agents(None)
    H = 6
    w.set_history(H)
    pool, mask = _pool(w)
    b = s.bounds
    pool["x"][0, 5] = float(b[1]) + 50.0      # out of bound: K10 retires the slot at the first tick
    w.reset(mask, pool)
    ring = HO.Ring(w.N, w.M, H)
    st, tid, _ = _snap(w)
    ring.restart(np.ones(w.N), st, tid)
    acts = _actions(w.N, w.M, seed=2)
    for t in range(4):
        _tick(w, "step", t, acts)
        st, tid, _ = _snap(w)
        ring.append(st, tid)
        w.agents_epilogue()
    assert int(w.type_id[0, 5]) == 255
    _check_ring(w, ring, "retired")
    assert not w.history()["valid"][0, 5].any()
    w.reset(mask, pool)                        # the type comes back with a fresh history
    assert bool(w.history()["valid"][0, 5, 0]) and not w.history()["valid"][0, 5, 1:].any()


def test_replay_tracks_and_switches(cuda_device):
    from tests.test_gpu_replay_schedule import _walk_episodes, _world as _replay_world

    ep = _walk_episodes(96, 16, seed=3)
    w, pool = _replay_world(ep)
    H = 8
    w.set_history(H)
    import torch

    w.reset(torch.ones(w.N, dtype=torch.uint8, device="cuda"), pool)
    ring = HO.Ring(w.N, w.M, H)
    st, tid, trk = _snap(w)
    ring.restart(np.ones(w.N), st, tid, trk)
    act = torch.zeros((w.N, w.M, 2), dtype=torch.float32, device="cuda")
    switches = appear = 0
    for t in range(30):
        prev_t, prev_k = tid, trk
        w.step(act)
        st, tid, trk = _snap(w)
        ring.append(st, tid, trk)
        switches += int(((prev_k >= 0) & (trk >= 0) & (prev_k != trk)).sum())
        appear += int(((prev_t == 255) & (tid != 255)).sum())
        _check_ring(w, ring, f"t={t}")
    assert switches > 0 and appear > 0   # the cases the track and type checks are about happened


def _obs_check(w, ring, agent_index=None, observers=None, Q=0):
    import torch

    out = w.observe_history(agent_index, observers)
    torch.cuda.synchronize()
    st, tid, trk = _snap(w)
    ai = None if agent_index is None else agent_index.cpu().numpy()
    ob = None if observers is None else observers.cpu().numpy()
    ref, dist = HO.observe(ring, st, tid, len(w.type_table), agent_index=ai, observers=ob, Q=Q, track_now=trk)
    got = out.cpu().numpy().reshape(ref.shape)
    HO.compare(got, ref, dist)
    return out


@pytest.mark.parametrize("n,Q,K", [(7, 128, 127), (4099, 4, 8)])
def test_observation_matches_the_oracle_at_every_lag(cuda_device, n, Q, K):
    import torch

    w, _ = _world(n=n)
    H = 5
    w.set_history(H)
    pool, mask = _pool(w)
    w.reset(mask, pool)
    ring = HO.Ring(w.N, w.M, H)
    st, tid, _ = _snap(w)
    ring.restart(np.ones(w.N), st, tid)
    acts = _actions(w.N, w.M, seed=13)
    for t in range(H + 2):
        _tick(w, "step", t, acts)
        st, tid, _ = _snap(w)
        ring.append(st, tid)
    # K8-style rows and the lag-0 identity with observe
    o = w.observe(16, 0, 50.0, 30.0)
    hist = _obs_check(w, ring, o.agent_index)
    assert hist.shape == (n, 17, H, 7)
    ok = o.agent_index >= 0
    assert torch.equal(hist[:, 1:, 0, 1:7][ok].view(torch.int32), o.agents[..., 1:7][ok].view(torch.int32))
    assert torch.equal(hist[:, 1:, 0, 0][ok], torch.ones_like(hist[:, 1:, 0, 0][ok]))
    _obs_check(w, ring)   # K = 0: the ego's own past only
    # K9-style rows: Q observers with duplicates, -1 and M; K agents with -1 and M mixed in (the oracle holds
    # [N, Q, 1 + K, H] arrays: the largest Q and K at a small N, an odd N with a partial last CTA at a small Q and K)
    rng = np.random.default_rng(n)
    obs = torch.from_numpy(rng.integers(-1, w.M + 1, (n, Q)).astype(np.int16)).cuda()
    oa = w.observe_agents(K, 0, 1e4, 30.0, observers=obs)
    hist = _obs_check(w, ring, oa.agent_index, obs, Q=Q)
    ok = oa.agent_index >= 0
    assert torch.equal(hist[:, :, 1:, 0, 1:7][ok].view(torch.int32), oa.agents[..., 1:7][ok].view(torch.int32))
    ai = oa.agent_index.clone()
    ai[:, :, ::5] = w.M
    _obs_check(w, ring, ai.contiguous(), obs, Q=Q)
    if n < 100:   # without observers an [N, Q, K] index names the rows' slots
        oa = w.observe_agents(8, 0, 50.0, 30.0)
        _obs_check(w, ring, oa.agent_index, None, Q=w.M)
    w.close()


def test_outputs_written_exactly(cuda_device):
    """Every output element is written and nothing past the end (sentinels with a guard tail)."""
    import torch
    from tactics2d_b200 import _lib

    w, _ = _world(n=33)
    H = 3
    w.set_history(H)
    pool, mask = _pool(w)
    w.reset(mask, pool)
    o = w.observe(4, 0)
    K = 4
    size = w.N * (1 + K) * H * 7
    buf = torch.full((size + 64,), SENTINEL, dtype=torch.float32, device="cuda")
    _lib.check(w.lib.t2d_observe_history(w._ctx, None, 0, C.c_void_p(o.agent_index.data_ptr()), K,
                                         C.c_void_p(buf.data_ptr()), w._stream()))
    torch.cuda.synchronize()
    assert not (buf[:size] == SENTINEL).any() and (buf[size:] == SENTINEL).all()


def test_env_history_across_auto_resets(cuda_device):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    s = synthetic.config2(96, 16, seed=2)
    H = 6
    for kw in (dict(observation="vector", vector_obs=dict(k_agents=4, k_segments=0)),
               dict(observation="agents", vector_obs=dict(k_agents=3, k_segments=0), agent_rewards=True),
               dict(observation="state", sampler=dict(seed=3))):
        env = BatchedTrafficEnv(s, max_step=5, history=dict(length=H), **kw)
        obs, info = env.reset(seed=0)
        w = env.world
        assert (w.history()["count"] == 1).all()
        episodes = np.zeros(w.N, np.int64)
        for t in range(13):
            r = env.step(torch.zeros((w.N, 2), dtype=torch.float32, device=w.device))
            info = r[-1]
            done = w.step_count.cpu().numpy() == 0
            st, tid, _ = _snap(w)
            episodes += done
            h = {k: v.cpu().numpy() for k, v in w.history().items()}
            hist = info["history"].cpu().numpy()
            shape = {"vector": (w.N, 5, H, 7), "agents": (w.N, w.M, 4, H, 7), "state": (w.N, 1, H, 7)}[kw["observation"]]
            assert hist.shape == shape
            if not done.any():
                continue
            # a new episode: exactly one valid entry per present slot, the start state (the oracle's restart)
            ring = HO.Ring(int(done.sum()), w.M, H)
            ring.restart(np.ones(int(done.sum())), {k: v[done] for k, v in st.items()}, tid[done])
            ref = ring.view(tid[done], len(w.type_table))
            assert (h["count"][done] == 1).all()
            assert np.array_equal(h["valid"][done], ref["valid"])
            for k in HO.FIELDS:
                assert np.array_equal(h[k][done].view(np.uint32), ref[k].view(np.uint32)), k
            assert (hist[done][..., 1:, 0] == 0).all() and (hist[done][..., 0, 0] <= 1).all()
            if kw["observation"] != "agents":
                assert np.array_equal(hist[done][:, 0, 0, 0], (tid[done][:, 0] < len(w.type_table)).astype(np.float32))
        assert episodes.min() >= 2
        env.close()


def test_rejections_keep_the_old_ring(cuda_device):
    import torch
    from tactics2d_b200 import _lib

    w, _ = _world(n=16)
    with pytest.raises(RuntimeError):
        w.observe_history()
    assert w.lib.t2d_observe_history(w._ctx, None, 0, None, 0, C.c_void_p(1 << 20), None) == -4   # no ring bound
    w.set_history(4)
    pool, mask = _pool(w)
    w.reset(mask, pool)
    w.step(torch.zeros((16, 64, 2), device="cuda"))
    before = w.history()
    for bad in (-1, 65):
        with pytest.raises(ValueError):
            w.set_history(bad)
        assert w.lib.t2d_set_history(w._ctx, bad) == -1
    after = w.history()
    for k in before:
        assert torch.equal(before[k], after[k]), k
    assert int(after["count"][0]) == 2
    o = w.observe(4, 0)
    with pytest.raises(ValueError):
        w.observe_history(o.agent_index.to(torch.int32))
    with pytest.raises(ValueError):
        w.observe_history(o.agent_index[:8])
    with pytest.raises(ValueError):
        w.observe_history(o.agent_index, torch.zeros((16, 2), dtype=torch.int32, device="cuda"))
    out = C.c_void_p(torch.empty(1 << 16, device="cuda").data_ptr())
    lib = w.lib
    assert lib.t2d_observe_history(w._ctx, None, 129, None, 0, out, None) == -1
    assert lib.t2d_observe_history(w._ctx, None, 65, None, 0, out, None) == -1            # no list and Q > M
    assert lib.t2d_observe_history(w._ctx, C.c_void_p(o.agent_index.data_ptr()), 0, None, 0, out, None) == -1
    assert lib.t2d_observe_history(w._ctx, None, 0, None, 128, out, None) == -1
    assert lib.t2d_observe_history(w._ctx, None, 0, None, 3, out, None) == -1              # agent_index NULL
    assert lib.t2d_observe_history(w._ctx, None, 0, None, 0, None, None) == -1
    w.set_history(0)
    with pytest.raises(RuntimeError):
        w.history()
    w.step(torch.zeros((16, 64, 2), device="cuda"))   # no ring: the tick alone
    torch.cuda.synchronize()
