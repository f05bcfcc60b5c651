"""K10, per-agent status / reward / retirement (t2d_agents_epilogue / BatchedWorld.agents_epilogue): bit identity with K1's
status and t2d_env_epilogue for one row on slot 0, teacher-forced parity with the float64 oracle in
tests/agent_reward_oracle.py (every slot, observer lists), retirement through ticks, observations and resets (a log
bound too), CUDA graph = eager, the C-level rejections and the env with agent_rewards=True."""

import ctypes as C

import numpy as np
import pytest

from oracle import scenario as O
from tests import agent_reward_oracle as R

pytestmark = pytest.mark.gpu


def _bits(t):
    """The fp32 bit patterns of a device tensor (-0.0 and NaN payloads compare as bits)."""
    return np.ascontiguousarray(t.cpu().numpy()).view(np.uint32)


def _world(n, m, seed, max_step, ego_still=None, ego_oob=None):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    s = synthetic.config2(n, m, seed=seed)
    w = BatchedWorld(n, m, s.table, max_step=max_step)
    w.set_map(s.segments, s.bounds)
    st = {k: np.array(v) for k, v in s.state().items()}
    if ego_still is not None:   # these egos start at rest
        for k in ("speed", "vx", "vy"):
            st[k][ego_still, 0] = 0.0
    if ego_oob is not None:     # these egos start across the boundary
        st["x"][ego_oob, 0] = np.float32(s.bounds[1] - 0.5)
    pool = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in st.items()}
    w.type_id.copy_(torch.from_numpy(s.type_id).cuda())
    w.reset(torch.ones(n, dtype=torch.uint8, device="cuda"), pool)
    return w, s, pool


def test_one_row_on_slot_zero_is_k1_and_the_env_epilogue_bit_for_bit(cuda_device):
    import torch
    from tactics2d_b200 import synthetic

    N, M = 4096, 64
    idx = np.arange(N)
    still, oob = idx % 3 == 0, idx % 7 == 1
    w, s, pool = _world(N, M, 5, max_step=40, ego_still=still, ego_oob=oob)
    rng = np.random.default_rng(6)
    x0, y0, h0 = (pool[k][:, 0].cpu().numpy() for k in ("x", "y", "heading"))
    exact = idx % 6 == 0
    target = np.stack([x0 + np.where(exact, 0, rng.normal(0, 3, N)), y0 + np.where(exact, 0, rng.normal(0, 3, N)),
                       h0, np.full(N, 2.4), np.full(N, 1.0)], 1).astype(np.float32)
    w.set_goal(target, 0.95, 3)
    w.set_agents(torch.zeros((N, 1), dtype=torch.int16, device=cuda_device), torch.from_numpy(target[:, None]).cuda(), 0.95, 3)
    seen = set()
    for t in range(64):
        act = synthetic.random_actions(300 + t, (N, M))
        act[still, 0] = 0.0
        r = w.step(torch.from_numpy(act).cuda())
        e = w.env_epilogue()
        a = w.agents_epilogue()
        torch.cuda.synchronize()
        assert torch.equal(a.status[:, 0], r.status), t
        assert np.array_equal(_bits(a.iou[:, 0]), _bits(r.iou)), t
        assert np.array_equal(_bits(a.reward[:, 0]), _bits(e.reward)), t
        assert torch.equal(a.terminated[:, 0], e.terminated) and torch.equal(a.truncated[:, 0], e.truncated), t
        assert torch.equal(a.done, e.done) and torch.equal(a.traffic, e.traffic_status), t
        for k in ("max_iou", "min_dist"):
            assert np.array_equal(_bits(w._agents[k][:, 0]), _bits(w._env[k])), (t, k)
        seen |= set(np.unique(r.status.cpu().numpy()).tolist())
        w.reset(e.done, pool)
    assert seen >= {O.NORMAL, O.COMPLETED, O.TIME_EXCEEDED, O.NO_ACTION, O.OUT_BOUND, O.FAILED}, seen
    w.close()


def _goals(w, Q, slot, seed, nan_every=3):
    """Goals near each row's slot (a third NaN)."""
    import torch

    rng = np.random.default_rng(seed)
    sl = np.clip(slot, 0, w.M - 1)
    x, y, h = (np.take_along_axis(getattr(w, k).cpu().numpy(), sl, 1) for k in ("x", "y", "heading"))
    g = np.stack([x + rng.normal(0, 2, x.shape), y + rng.normal(0, 2, x.shape), h, np.full(x.shape, 2.4),
                  np.full(x.shape, 1.0)], -1).astype(np.float32)
    g[:, ::nan_every, 0] = np.nan
    return torch.from_numpy(g).to(w.device)


def _parity(w, pool, observers, goals, steps, sel, seed):
    """Teacher-forced: each step the oracle starts from the device's type ids and row state before K10."""
    import torch
    from tactics2d_b200 import synthetic

    table = w.type_table.as_oracle_table()
    n_types = len(w.type_table)
    a_ = w._agents
    obs = None if observers is None else observers.cpu().numpy()[sel]
    g = goals.cpu().numpy()[sel]
    settled = 0
    for t in range(steps):
        pre = {k: a_[k].cpu().numpy()[sel] for k in ("last_pose", "noact_count", "max_iou", "min_dist", "retired_type")}
        w.step(torch.from_numpy(synthetic.random_actions(seed + t, (w.N, w.M))).cuda())
        pre_type = w.type_id.cpu().numpy()[sel]
        a = w.agents_epilogue()
        torch.cuda.synchronize()
        st = w.state_numpy()
        ref = R.agents_epilogue(w.result.flags.cpu().numpy()[sel], pre_type, st["x"][sel], st["y"][sel], st["heading"][sel],
                                w.step_count.cpu().numpy()[sel], table, n_types, observers=obs, goals=g,
                                last_pose=pre["last_pose"], noact_count=pre["noact_count"], max_iou=pre["max_iou"],
                                min_dist=pre["min_dist"], retired=pre["retired_type"], max_step=w.max_step,
                                threshold=0.95, no_action_max=100)
        iou = a.iou.cpu().numpy()[sel]
        assert np.abs(iou - ref["iou"]).max() <= 2e-6, t
        ok = ~(np.abs(ref["iou"] - 0.95) <= 1e-6).any(1)   # scenarios no IoU puts at the threshold
        for k, got in (("status", a.status), ("terminated", a.terminated), ("truncated", a.truncated)):
            assert np.array_equal(got.cpu().numpy()[sel][ok], ref[k][ok]), (t, k)
        assert np.array_equal(a.done.cpu().numpy()[sel][ok], ref["done"][ok]), t
        assert np.array_equal(w.type_id.cpu().numpy()[sel][ok], ref["type_id"][ok]), t
        assert np.array_equal(a_["retired_type"].cpu().numpy()[sel][ok], ref["retired"][ok]), t
        rw = a.reward.cpu().numpy()[sel][ok]
        assert np.allclose(rw, ref["reward"][ok], rtol=1e-6, atol=5e-6), (t, np.abs(rw - ref["reward"][ok]).max())
        mi, md = a_["max_iou"].cpu().numpy()[sel][ok], a_["min_dist"].cpu().numpy()[sel][ok]
        assert np.allclose(mi, ref["max_iou"][ok], rtol=0, atol=2e-6, equal_nan=False)
        assert np.allclose(md, ref["min_dist"][ok], rtol=1e-6, atol=1e-6)
        assert np.array_equal(a.traffic.cpu().numpy()[sel], ref["traffic"])
        settled += int(((ref["status"] != O.NORMAL) & (ref["status"] != 0)).sum())
        w.reset(a.done, pool)
    return settled


def test_every_slot_against_the_oracle(cuda_device):
    N, M = 4096, 64
    w, s, pool = _world(N, M, 7, max_step=5)
    goals = _goals(w, M, np.broadcast_to(np.arange(M), (N, M)), 8)
    w.set_agents(None, goals, 0.95, 100)
    sel = np.random.default_rng(9).choice(N, 300, replace=False)
    assert _parity(w, pool, None, goals, 8, sel, 500) > 100   # collisions, out of bound and the time limit settle rows
    w.close()


def test_observer_lists_with_duplicates_absent_and_q_above_m(cuda_device):
    import torch

    N, M, Q = 256, 8, 12
    w, s, pool = _world(N, M, 11, max_step=6)
    rng = np.random.default_rng(12)
    obs = rng.integers(-2, M + 2, (N, Q)).astype(np.int16)
    obs[:, 1] = obs[:, 0]   # duplicates
    obs[:4] = -1            # scenarios without a single agent: done at every step
    observers = torch.from_numpy(obs).cuda()
    goals = _goals(w, Q, obs.astype(np.int64), 13)
    w.set_agents(observers, goals, 0.95, 100)
    _parity(w, pool, observers, goals, 6, np.arange(N), 700)
    a = w.agents_epilogue()
    assert (a.done[:4] == 1).all() and (a.status[:4] == 0).all()
    w.close()


def test_retirement_through_ticks_observations_and_resets(cuda_device):
    import torch
    from tactics2d_b200 import synthetic

    N, M = 512, 16
    w, s, pool = _world(N, M, 21, max_step=1000)
    w.set_agents()
    types0 = w.type_id.clone()
    retired_any = torch.zeros((N, M), dtype=torch.bool, device=cuda_device)
    for t in range(6):
        w.step(torch.from_numpy(synthetic.random_actions(900 + t, (N, M))).cuda())
        pre = w.type_id.clone()
        a = w.agents_epilogue()
        settled = (a.status != O.NORMAL) & (a.status != 0)   # row q = slot q
        assert torch.equal(w.type_id[settled], torch.full_like(w.type_id[settled], 255))
        assert torch.equal(w.retired_type[settled], pre[settled])
        assert torch.equal(w.type_id[~settled], pre[~settled])
        retired_any |= settled
        # the retired slots neither move nor collide on the next tick, and the observation shows their rows absent
        gone = w.type_id == 255
        xy = (w.x.clone(), w.y.clone())
        r = w.step(torch.from_numpy(synthetic.random_actions(950 + t, (N, M))).cuda())
        assert torch.equal(w.x[gone], xy[0][gone]) and torch.equal(w.y[gone], xy[1][gone])
        assert not r.flags[gone].any()
        hit = r.hit_index.long()
        assert not (gone.gather(1, hit.clamp(min=0)) & (hit >= 0)).any()
        o = w.observe_agents(4, 4)
        assert not o.flat[gone].any() and (o.agent_index[gone] == -1).all()
    assert retired_any.sum() > 20
    mask = torch.zeros(N, dtype=torch.uint8, device=cuda_device)
    mask[::2] = 1
    keep = w.type_id.clone()
    w.reset(mask, pool)
    m = mask.bool()
    assert torch.equal(w.type_id[m], types0[m]) and (w.retired_type[m] == 255).all()
    assert torch.equal(w.type_id[~m], keep[~m])
    assert (w._agents["last_pose"][m][..., 3] == 0).all() and (w._agents["noact_count"][m] == 0).all()
    w.close()


def test_env_resets_restore_types_with_and_without_a_log(cuda_device):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    s = synthetic.config2(128, 16, seed=31)
    env = BatchedTrafficEnv(s, max_step=50, observation="agents", vector_obs=dict(k_agents=4, k_segments=4),
                            agent_rewards=True)
    env.reset(seed=1)
    for t in range(8):
        env.step(torch.from_numpy(synthetic.random_actions(40 + t, (128, 16))).cuda())
    assert (env.world.type_id == 255).any()
    env.reset(seed=2, options={"shuffle": True})
    assert torch.equal(env.world.type_id, env._type_id) and (env.world.retired_type == 255).all()
    env.close()
    # a log bound: the reset runs K2 then K7, and the ego (never replayed) gets its row's type back
    N, M = 128, 16
    ep = synthetic.replay_episodes(N, M, 1200, seed=8, size=100.0, duration_ms=10000, max_frames=120)
    env = BatchedTrafficEnv(None, replay=ep, max_step=6, observation="agents", vector_obs=dict(k_agents=4, k_segments=4),
                            agent_rewards=True)
    env.reset(seed=1, options={"shuffle": True})
    w = env.world
    resets = 0
    for t in range(10):
        _, reward, term, trunc, info = env.step(torch.from_numpy(np.random.default_rng(t).uniform(-.5, .5, (N, 2))
                                                                 .astype(np.float32)).cuda())
        done = w._agents["done"].bool()
        resets += int(done.sum())
        row = w.log_row.long()
        ego_type = torch.from_numpy(ep.type_id[:, 0]).cuda()[row]
        assert torch.equal(w.type_id[done, 0], ego_type[done]) and (w.retired_type[done] == 255).all()
    assert resets >= N
    env.reset(seed=3, options={"shuffle": True})
    assert torch.equal(w.type_id[:, 0], torch.from_numpy(ep.type_id[:, 0]).cuda()[w.log_row.long()])
    env.close()


def test_graph_of_tick_epilogue_and_reset_equals_eager(cuda_device):
    import torch
    from tactics2d_b200 import synthetic

    N, M = 512, 16
    worlds = [_world(N, M, 41, max_step=7) for _ in range(2)]
    act = torch.from_numpy(synthetic.random_actions(42, (N, M))).cuda()
    for w, s, pool in worlds:
        w.set_agents(None, _goals(w, M, np.broadcast_to(np.arange(M), (N, M)), 43), 0.95, 2)

    def step(w, pool):
        w.step(act)
        a = w.agents_epilogue()
        w.reset(a.done, pool)
        return a

    (we, _, pe), (wg, _, pg) = worlds
    step(we, pe)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(wg, pg)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ag = step(wg, pg)
    for t in range(10):
        ae = step(we, pe)
        g.replay()
        torch.cuda.synchronize()
        for k in ("reward", "terminated", "truncated", "status", "iou", "done", "traffic"):
            assert torch.equal(getattr(ae, k), getattr(ag, k)), (t, k)
        for k in ("x", "y", "heading", "type_id", "step_count", "retired_type"):
            assert torch.equal(getattr(we, k), getattr(wg, k)), (t, k)
    for w, _, _ in worlds:
        w.close()


def test_c_level_rejections_launch_nothing(cuda_device):
    import torch
    from tactics2d_b200 import _lib

    w, s, pool = _world(8, 8, 1, max_step=10)
    lib = w.lib
    p = lambda t: C.c_void_p(t.data_ptr())
    f32 = lambda *sh: torch.zeros(sh, dtype=torch.float32, device=cuda_device)
    u8 = lambda *sh: torch.zeros(sh, dtype=torch.uint8, device=cuda_device)
    obs = torch.zeros((8, 128), dtype=torch.int16, device=cuda_device)
    lp, cnt, ret = f32(8, 128, 4), torch.zeros((8, 128), dtype=torch.int32, device=cuda_device), u8(8, 8)
    out = dict(reward=f32(8, 128), term=u8(8, 128), trunc=u8(8, 128), st=u8(8, 128), iou=f32(8, 128), done=u8(8),
               mi=f32(8, 128), md=f32(8, 128))
    o = [p(out[k]) for k in ("reward", "term", "trunc", "st", "iou", "done", "mi", "md")]
    epi = lambda ctx, *a: lib.t2d_agents_epilogue(ctx, p(w.result.flags), *a, None, 1, None)
    n0 = lib.t2d_launch_count()
    assert epi(w._ctx, *o) == -4                                                    # before t2d_set_agents
    seta = lambda o_, q, *st: lib.t2d_set_agents(w._ctx, o_, q, None, 0.95, 3, *st)
    for q in (0, -1, 129):
        assert seta(p(obs), q, p(lp), p(cnt), p(ret)) == -1, q                     # Q outside 1..128
    assert seta(None, 9, p(lp), p(cnt), p(ret)) == -1                               # every slot, Q > M
    for i in range(3):                                                              # a NULL state array
        st = [p(lp), p(cnt), p(ret)]
        st[i] = None
        assert seta(p(obs), 4, *st) == -1, i
    assert lib.t2d_set_agents(w._ctx, p(obs), 4, p(lp), 1.5, 3, p(lp), p(cnt), p(ret)) == -1   # threshold with goals
    assert seta(p(obs), 128, p(lp), p(cnt), p(ret)) == 0
    for i in range(8):                                                              # a NULL output
        a = list(o)
        a[i] = None
        assert epi(w._ctx, *a) == -1, i
    assert lib.t2d_agents_epilogue(None, p(w.result.flags), *o, None, 1, None) == -1
    assert lib.t2d_agents_epilogue(w._ctx, None, *o, None, 1, None) == -1
    ctx = C.c_void_p()   # a context whose state is not bound
    _lib.check(lib.t2d_create(C.byref(ctx), 0, 8, 8, C.byref(_lib.Config(100, 5, 0, 0))))
    _lib.check(lib.t2d_set_type_table(ctx, w.type_table.to_c_array(), len(w.type_table)))
    assert lib.t2d_set_agents(ctx, p(obs), 4, None, 0.95, 3, p(lp), p(cnt), p(ret)) == 0
    assert epi(ctx, *o) == -4
    lib.t2d_destroy(ctx)
    assert lib.t2d_launch_count() == n0
    assert epi(w._ctx, *o) == 0 and lib.t2d_launch_count() == n0 + 1
    assert seta(None, 0, None, None, None) == 0                                     # unbind
    assert epi(w._ctx, *o) == -4
    with pytest.raises(ValueError):
        w.set_agents(observers=torch.zeros((8, 2), dtype=torch.int16))               # host tensor
    with pytest.raises(ValueError):
        w.set_agents(goals=torch.zeros((8, 7, 5), device=cuda_device))
    w.close()


def test_env_with_agent_rewards(cuda_device):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    N, M, Q = 64, 16, 6
    s = synthetic.config2(N, M, seed=2)
    obs = torch.from_numpy(np.random.default_rng(3).integers(0, M, (N, Q)).astype(np.int16)).to(cuda_device)
    goals = torch.from_numpy(np.stack([s.x[:, :Q], s.y[:, :Q], s.heading[:, :Q], np.full((N, Q), 2.4), np.full((N, Q), 1.0)],
                                      -1).astype(np.float32)).to(cuda_device)
    cfg = dict(k_agents=4, k_segments=6, observers=obs, goals=goals)
    env = BatchedTrafficEnv(s, max_step=4, observation="agents", vector_obs=cfg, agent_rewards=True)
    o, _ = env.reset()
    assert (o[..., 0] == 1).all()   # every agent is present
    resets = 0
    for t in range(9):
        o, reward, term, trunc, info = env.step(torch.full((N, 2), 0.1, device=cuda_device))
        assert reward.shape == term.shape == trunc.shape == (N, Q) and o.shape[:2] == (N, Q)
        assert reward.dtype == torch.float32 and term.dtype == trunc.dtype == torch.bool
        assert info["agent_status"].shape == (N, Q) and info["agent_iou"].shape == (N, Q)
        assert info["traffic_status"].shape == (N, M) and "scenario_status" in info
        done = env.world._agents["done"].bool()
        assert (o[done][..., 0] == 1).all()   # after the auto-reset every agent shows again
        resets += int(done.sum())
    assert resets >= N   # max_step 4: every scenario reset at least once
    env.close()
    with pytest.raises(ValueError):
        BatchedTrafficEnv(s, observation="agents", vector_obs=cfg, agent_rewards=True, target=np.zeros((N, 5), np.float32))
    with pytest.raises(ValueError):
        BatchedTrafficEnv(s, observation="vector", agent_rewards=True)
