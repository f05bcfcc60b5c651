"""K11, per-agent actions (t2d_scatter_agent_action / BatchedWorld.scatter_agent_action) and the host-buffer multi-agent
step (t2d_step_host_agents / BatchedWorld.step_host_agents): K11 against tests/agent_action_oracle.py bit for bit,
rollouts driven by the scatter against rollouts fed the oracle-scattered [N, M, 2] (retirement, resets, controllers),
controller and ego precedence, identity with the ego action for one row on slot 0, the host step against the device path,
CUDA graph = eager, the C-level rejections and the env with agent_actions=True."""

import ctypes as C

import numpy as np
import pytest

from tests.agent_action_oracle import owner_rows, scatter_agent_action

pytestmark = pytest.mark.gpu


def _bits(t):
    """The fp32 bit patterns of a device tensor or array (-0.0 and NaN payloads compare as bits)."""
    a = t.cpu().numpy() if hasattr(t, "cpu") else t
    return np.ascontiguousarray(a).view(np.uint32)


def _random_bits(rng, shape):
    """fp32 values from random bit patterns (NaN payloads, infinities, -0.0, subnormals among them)."""
    b = rng.integers(0, 2**32, shape, dtype=np.uint64).astype(np.uint32)
    b.reshape(-1)[:4] = [0x80000000, 0x7FC00001, 0xFFBADBAD, 0x00000001]
    return b.view(np.float32)


def _world(n, m, seed, max_step=0, scene=None, empty_every=11, **kw):
    """A C2-style world (or the given scene) whose every empty_every-th slot (slot 0 excepted) is empty."""
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    s = scene if scene is not None else synthetic.config2(n, m, seed=seed)
    w = BatchedWorld(n, m, s.table, max_step=max_step, **kw)
    w.set_map(s.segments, s.bounds)
    tid = s.type_id.copy()
    if empty_every:
        flat = tid.reshape(-1)
        flat[3::empty_every] = 255
        tid[:, 0] = s.type_id[:, 0]
    pool = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in s.state().items()}
    w.type_id.copy_(torch.from_numpy(tid).cuda())
    w.reset(torch.ones(n, dtype=torch.uint8, device="cuda"), pool)
    return w, pool


def _observer_list(rng, n, m, q):
    """int16 [n, q] with duplicates, -1, values >= M and rows on empty slots."""
    obs = rng.integers(-1, m + 2, (n, q)).astype(np.int16)
    if q > 1:
        obs[:, 1] = obs[:, 0]              # a duplicate in every scenario
    obs[::5, -1] = m                       # one past the end
    obs[::7, 0] = -1
    return obs


def _check_k11(w, Q, observers, seed):
    import torch

    rng = np.random.default_rng(seed)
    base = _random_bits(rng, (w.N, w.M, 2))
    rows = _random_bits(rng, (w.N, Q, 2))
    act = torch.from_numpy(base.copy()).cuda()
    rows_t = torch.from_numpy(rows).cuda()
    if observers is None and Q < w.M:   # rows 0..Q-1 on slots 0..Q-1: only the C call takes Q < M without a list
        assert w.lib.t2d_scatter_agent_action(w._ctx, None, Q, C.c_void_p(rows_t.data_ptr()), C.c_void_p(act.data_ptr()),
                                              w._stream()) == 0
    else:
        w.scatter_agent_action(rows_t, act, None if observers is None else torch.from_numpy(observers).cuda())
    torch.cuda.synchronize()
    types = w.type_id.cpu().numpy()
    ref = scatter_agent_action(base, rows, types, len(w.type_table), observers)
    assert np.array_equal(_bits(act), _bits(ref))
    written = (owner_rows(types, Q, observers) < Q) & (types < len(w.type_table))
    assert written.any() and (~written).any()
    return written


@pytest.mark.parametrize("case", ["every_slot", "list", "one_row", "q128"])
def test_k11_against_the_oracle_c2(cuda_device, case):
    N, M = 4096, 64
    w, _ = _world(N, M, 3)
    rng = np.random.default_rng(4)
    # retired slots of a K10 run look like empty ones: type 255
    w.type_id[5::9, 7] = 255
    if case == "every_slot":
        _check_k11(w, M, None, 10)
    elif case == "list":
        _check_k11(w, 40, _observer_list(rng, N, M, 40), 11)
    elif case == "one_row":
        _check_k11(w, 1, rng.integers(-1, M + 1, (N, 1)).astype(np.int16), 12)
        _check_k11(w, 1, None, 13)
    else:
        _check_k11(w, 128, _observer_list(rng, N, M, 128), 14)
    w.close()


def test_k11_against_the_oracle_c4_ind(cuda_device):
    from tactics2d_b200 import synthetic
    from tactics2d_b200.map import load_collidable_segments

    seg, b = load_collidable_segments("inD_1")
    s = synthetic.config4(16384, 32, seed=4, segments=seg, bounds=b)
    w, _ = _world(16384, 32, 0, scene=s)
    rng = np.random.default_rng(5)
    _check_k11(w, 32, None, 20)
    _check_k11(w, 48, _observer_list(rng, 16384, 32, 48), 21)
    w.close()


def _idm(w, observers, seed):
    """IDM on every slot no row names, each following a random slot that a row names (an agent leader)."""
    from tactics2d_b200.controller import IDMController

    rng = np.random.default_rng(seed)
    named = owner_rows(w.type_id.cpu().numpy(), observers.shape[1], observers) < observers.shape[1]
    cid = np.where(named, 255, 0).astype(np.uint8)
    lead = np.full((w.N, w.M), -1, np.int16)
    for n in range(w.N):
        agents = np.nonzero(named[n])[0]
        if len(agents):
            lead[n] = rng.choice(agents, w.M)
    w.set_controllers([IDMController()], cid, lead_index=lead)
    return named, cid


STATE = ("x", "y", "heading", "speed", "vx", "vy", "type_id", "step_count")
AGENT_OUT = ("reward", "terminated", "truncated", "status", "iou", "done", "traffic", "max_iou", "min_dist", "retired_type",
             "last_pose", "noact_count")


def _same_worlds(wa, wb, t, action=None):
    import torch

    for k in STATE:
        assert torch.equal(getattr(wa, k), getattr(wb, k)), (t, k)
    for k in ("flags", "hit_index", "hit_segment", "status", "done"):
        assert torch.equal(getattr(wa.result, k), getattr(wb.result, k)), (t, k)
    for k in AGENT_OUT:
        assert np.array_equal(_bits(wa._agents[k]) if wa._agents[k].dtype == torch.float32 else wa._agents[k].cpu().numpy(),
                              _bits(wb._agents[k]) if wb._agents[k].dtype == torch.float32 else wb._agents[k].cpu().numpy()), (t, k)
    if wa.last_accel is not None:
        assert np.array_equal(_bits(wa.last_accel), _bits(wb.last_accel)), t


@pytest.mark.parametrize("controllers", [False, True])
def test_rollout_scatter_equals_the_oracle_scattered_action(cuda_device, controllers):
    import torch
    from tactics2d_b200 import synthetic

    N, M, Q = 1024, 16, 10
    rng = np.random.default_rng(30)
    obs = _observer_list(rng, N, M, Q)
    obs_t = torch.from_numpy(obs).cuda()
    (wa, pa), (wb, pb) = _world(N, M, 31, max_step=12), _world(N, M, 31, max_step=12)
    for w in (wa, wb):
        w.set_agents(obs_t)
        if controllers:
            named, _ = _idm(w, obs, 32)
    act_a = torch.zeros((N, M, 2), device=cuda_device)
    act_b = np.zeros((N, M, 2), np.float32)
    settled = resets = 0
    for t in range(40):
        rows = synthetic.random_actions(400 + t, (N, Q))
        wa.scatter_agent_action(torch.from_numpy(rows).cuda(), act_a, obs_t)
        act_b = scatter_agent_action(act_b, rows, wb.type_id.cpu().numpy(), len(wb.type_table), obs)
        full_b = torch.from_numpy(act_b).cuda()
        for w, a in ((wa, act_a), (wb, full_b)):
            if controllers:
                w.control(a)
            w.step(a)
        ea, eb = wa.agents_epilogue(), wb.agents_epilogue()
        torch.cuda.synchronize()
        act_b = full_b.cpu().numpy()   # what the controllers wrote stays in the buffer, as in act_a
        assert np.array_equal(_bits(act_a), _bits(act_b)), t
        _same_worlds(wa, wb, t)
        settled += int(((ea.status != 1) & (ea.status != 0)).sum())
        resets += int(ea.done.sum())
        wa.reset(ea.done, pa)
        wb.reset(eb.done, pb)
    assert settled > 100 and resets >= N   # retirement and masked resets both happened
    if controllers:
        assert (wa.last_accel.cpu().numpy()[~named] > 0).any()
    for w in (wa, wb):
        w.close()


def test_controller_and_ego_precedence(cuda_device):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.controller import IDMController

    N, M = 256, 8
    rows = torch.from_numpy(synthetic.random_actions(50, (N, M))).cuda()
    # a controlled agent slot takes its controller's action
    worlds = [_world(N, M, 51, empty_every=0)[0] for _ in range(2)]
    cid = np.full((N, M), 255, np.uint8)
    cid[:, 2::3] = 0
    for w in worlds:
        w.set_controllers([IDMController()], cid)
    act_a, act_b = torch.zeros((N, M, 2), device=cuda_device), torch.zeros((N, M, 2), device=cuda_device)
    worlds[0].scatter_agent_action(rows, act_a)
    worlds[0].control(act_a)
    worlds[1].control(act_b)
    torch.cuda.synchronize()
    ctl = torch.from_numpy(cid != 255).cuda()
    assert torch.equal(act_a[ctl], act_b[ctl]) and not torch.equal(act_a[ctl], rows[ctl])
    assert torch.equal(act_a[~ctl], rows[~ctl])
    for w in worlds:
        w.close()
    # a bound ego action drives slot 0 whatever the scatter wrote there
    (wa, _), (wb, _), (wc, _) = (_world(N, M, 52) for _ in range(3))
    ego = torch.from_numpy(synthetic.random_actions(53, (N, 1))[:, 0]).cuda()
    for w in (wa, wb):
        w.set_ego_action(ego)
    act_a, act_c = torch.zeros((N, M, 2), device=cuda_device), torch.zeros((N, M, 2), device=cuda_device)
    act_b = torch.zeros((N, M, 2), device=cuda_device)
    act_b[:, 1:] = rows[:, 1:]
    wa.scatter_agent_action(rows, act_a)
    wc.scatter_agent_action(rows, act_c)
    for w, a in ((wa, act_a), (wb, act_b), (wc, act_c)):
        w.step(a)
    torch.cuda.synchronize()
    for k in ("x", "y", "heading", "speed"):
        assert torch.equal(getattr(wa, k), getattr(wb, k)), k
    assert not torch.equal(wa.x[:, 0], wc.x[:, 0])
    for w in (wa, wb, wc):
        w.close()


@pytest.mark.parametrize("controllers", [False, True])
def test_one_row_on_slot_zero_is_the_ego_action(cuda_device, controllers):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.controller import IDMController

    N, M = 2048, 16
    (wa, pa), (wb, pb) = _world(N, M, 60, max_step=20), _world(N, M, 60, max_step=20)
    zero = torch.zeros((N, 1), dtype=torch.int16, device=cuda_device)
    for w in (wa, wb):
        w.set_agents(zero)
        if controllers:   # everyone but the ego follows the slot in front of it, slot 1 the ego
            cid = np.zeros((N, M), np.uint8)
            cid[:, 0] = 255
            w.set_controllers([IDMController()], cid, lead_index=np.tile(np.arange(M, dtype=np.int16) - 1, (N, 1)))
    act_a, act_b = torch.zeros((N, M, 2), device=cuda_device), torch.zeros((N, M, 2), device=cuda_device)
    ego = torch.zeros((N, 2), device=cuda_device)
    wb.set_ego_action(ego)
    resets = 0
    for t in range(40):
        ego.copy_(torch.from_numpy(synthetic.random_actions(600 + t, (N, 1))[:, 0]))
        wa.scatter_agent_action(ego[:, None].contiguous(), act_a, zero)
        for w, a in ((wa, act_a), (wb, act_b)):
            if controllers:
                w.control(a)
            w.step(a)
        ea, eb = wa.agents_epilogue(), wb.agents_epilogue()
        torch.cuda.synchronize()
        _same_worlds(wa, wb, t)
        if controllers:
            assert torch.equal(act_a, act_b), t
        resets += int(ea.done.sum())
        wa.reset(ea.done, pa)
        wb.reset(eb.done, pb)
    assert resets >= N
    for w in (wa, wb):
        w.close()


def test_step_host_agents_equals_the_device_path(cuda_device):
    import torch
    from tactics2d_b200 import synthetic

    N, M, Q = 1024, 16, 12
    rng = np.random.default_rng(70)
    obs = torch.from_numpy(_observer_list(rng, N, M, Q)).cuda()
    (wa, pa), (wb, pb), (wc, pc) = (_world(N, M, 71, max_step=10) for _ in range(3))
    for w in (wa, wb, wc):
        w.set_agents(obs)
    act_a, act_b, act_c = (torch.zeros((N, M, 2), device=cuda_device) for _ in range(3))
    done_c = np.zeros(N, np.uint8)
    p = lambda t: C.c_void_p(0 if t is None else t.data_ptr())
    resets = 0
    for t in range(36):
        rows = synthetic.random_actions(700 + t, (N, Q))
        reward, term, trunc, status, done = wa.step_host_agents(rows, act_a)
        wb.scatter_agent_action(torch.from_numpy(rows).cuda(), act_b, obs)
        wb.step(act_b)
        e = wb.agents_epilogue()
        # every host output but done NULL, and no flags, hit indices or traffic status of the caller's
        rc = wc.lib.t2d_step_host_agents(wc._ctx, C.c_void_p(rows.ctypes.data), p(act_c), None, None, None,
                                         p(wc._agents["max_iou"]), p(wc._agents["min_dist"]), 1, None, None, None, None,
                                         C.c_void_p(done_c.ctypes.data), wc._stream())
        assert rc == 0
        torch.cuda.synchronize()
        assert np.array_equal(_bits(reward), _bits(e.reward)), t
        assert np.array_equal(term, e.terminated.cpu().numpy()) and np.array_equal(trunc, e.truncated.cpu().numpy()), t
        assert np.array_equal(status, e.status.cpu().numpy()) and np.array_equal(done, e.done.cpu().numpy()), t
        assert np.array_equal(done_c, done), t
        assert term.dtype == trunc.dtype == np.bool_ and reward.shape == (N, Q) and done.shape == (N,)
        for k in STATE:
            assert torch.equal(getattr(wa, k), getattr(wb, k)) and torch.equal(getattr(wc, k), getattr(wb, k)), (t, k)
        for k in ("flags", "hit_index", "hit_segment"):
            assert torch.equal(getattr(wa.result, k), getattr(wb.result, k)), (t, k)
        for k in ("max_iou", "min_dist", "retired_type", "last_pose", "noact_count"):
            assert torch.equal(wa._agents[k], wb._agents[k]) and torch.equal(wc._agents[k], wb._agents[k]), (t, k)
        assert torch.equal(act_a, act_b) and torch.equal(act_c, act_b), t
        resets += int(done.sum())
        mask = torch.from_numpy(done.copy()).cuda()
        for w, pool in ((wa, pa), (wb, pb), (wc, pc)):
            w.reset(mask, pool)
    assert resets >= N
    assert not wc.result.flags.any()   # K10 read the library's own flags: the world's were never passed
    for w in (wa, wb, wc):
        w.close()


def test_graph_of_scatter_control_tick_and_epilogue_equals_eager(cuda_device):
    import torch
    from tactics2d_b200 import synthetic

    N, M, Q = 512, 16, 9
    obs_np = _observer_list(np.random.default_rng(80), N, M, Q)
    obs = torch.from_numpy(obs_np).cuda()
    rows = torch.from_numpy(synthetic.random_actions(81, (N, Q))).cuda()
    worlds = [_world(N, M, 82, max_step=8) for _ in range(2)]
    acts = [torch.zeros((N, M, 2), device=cuda_device) for _ in range(2)]
    for w, _ in worlds:
        w.set_agents(obs)
        _idm(w, obs_np, 83)

    def step(w, pool, act):
        w.scatter_agent_action(rows, act, obs)
        w.control(act)
        w.step(act)
        a = w.agents_epilogue()
        w.reset(a.done, pool)
        return a

    (we, pe), (wg, pg) = worlds
    step(we, pe, acts[0])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(wg, pg, acts[1])
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ag = step(wg, pg, acts[1])
    for t in range(12):
        ae = step(we, pe, acts[0])
        g.replay()
        torch.cuda.synchronize()
        for k in ("reward", "terminated", "truncated", "status", "done"):
            assert torch.equal(getattr(ae, k), getattr(ag, k)), (t, k)
        for k in STATE:
            assert torch.equal(getattr(we, k), getattr(wg, k)), (t, k)
        assert torch.equal(acts[0], acts[1]) and torch.equal(we.last_accel, wg.last_accel), t
    for w, _ in worlds:
        w.close()


def test_c_level_rejections_launch_nothing(cuda_device):
    import torch
    from tactics2d_b200 import _lib

    w, _ = _world(8, 8, 1, max_step=10)
    lib = w.lib
    p = lambda t: C.c_void_p(t.data_ptr())
    f32 = lambda *sh: torch.zeros(sh, dtype=torch.float32, device=cuda_device)
    obs = torch.zeros((8, 128), dtype=torch.int16, device=cuda_device)
    rows, act = f32(8, 128, 2), f32(8, 8, 2)
    odd = C.c_void_p(act.data_ptr() + 4)
    host = np.zeros((8, 128, 2), np.float32)
    hp = C.c_void_p(host.ctypes.data)
    mi, md = f32(8, 128), f32(8, 128)
    outs = [np.zeros((8, 128), np.float32), np.zeros((8, 128), np.uint8), np.zeros((8, 128), np.uint8),
            np.zeros((8, 128), np.uint8), np.zeros(8, np.uint8)]
    op = [C.c_void_p(o.ctypes.data) for o in outs]
    host_step = lambda ctx, a, ac, m1, m2, done: lib.t2d_step_host_agents(ctx, a, ac, None, None, None, m1, m2, 1,
                                                                          *op[:4], done, None)
    n0 = lib.t2d_launch_count()
    sc = lib.t2d_scatter_agent_action
    assert sc(None, p(obs), 4, p(rows), p(act), None) == -1                        # NULL context
    for q in (0, -1, 129):
        assert sc(w._ctx, p(obs), q, p(rows), p(act), None) == -1, q                # Q outside 1..128
    assert sc(w._ctx, None, 9, p(rows), p(act), None) == -1                         # every slot, Q > M
    assert sc(w._ctx, p(obs), 4, None, p(act), None) == -1                          # NULL arrays
    assert sc(w._ctx, p(obs), 4, p(rows), None, None) == -1
    assert sc(w._ctx, p(obs), 4, C.c_void_p(rows.data_ptr() + 4), p(act), None) == -1   # not 8-byte aligned
    assert sc(w._ctx, p(obs), 4, p(rows), odd, None) == -1
    # the host step: before t2d_set_agents, then every NULL argument and a misaligned action
    assert host_step(w._ctx, hp, p(act), p(mi), p(md), op[4]) == -4
    w.set_agents(obs[:, :4].contiguous())
    assert host_step(None, hp, p(act), p(mi), p(md), op[4]) == -1
    for i in range(5):
        a = [hp, p(act), p(mi), p(md), op[4]]
        a[i] = None
        assert host_step(w._ctx, *a) == -1, i
    assert host_step(w._ctx, hp, odd, p(mi), p(md), op[4]) == -1
    ctx = C.c_void_p()   # a context whose state is not bound
    _lib.check(lib.t2d_create(C.byref(ctx), 0, 8, 8, C.byref(_lib.Config(100, 5, 0, 0))))
    _lib.check(lib.t2d_set_type_table(ctx, w.type_table.to_c_array(), len(w.type_table)))
    assert sc(ctx, p(obs), 4, p(rows), p(act), None) == -4
    assert host_step(ctx, hp, p(act), p(mi), p(md), op[4]) == -4
    lib.t2d_destroy(ctx)
    assert lib.t2d_launch_count() == n0
    assert sc(w._ctx, p(obs), 128, p(rows), p(act), None) == 0 and lib.t2d_launch_count() == n0 + 1
    assert sc(w._ctx, None, 8, p(rows), p(act), None) == 0 and lib.t2d_launch_count() == n0 + 2
    # the Python layer checks the tensors before their pointers reach the kernel
    for bad in (torch.zeros((8, 4, 2)), f32(8, 5, 2), f32(8, 4, 2).double(), f32(8, 2, 4).transpose(1, 2)):
        with pytest.raises(ValueError):
            w.scatter_agent_action(bad, act, obs[:, :4].contiguous())
    with pytest.raises(ValueError):
        w.scatter_agent_action(f32(8, 4, 2), f32(8, 7, 2), obs[:, :4].contiguous())
    with pytest.raises(ValueError):
        w.scatter_agent_action(f32(8, 4, 2), act, obs[:, :4].cpu())
    with pytest.raises(ValueError):
        w.step_host_agents(np.zeros((8, 5, 2), np.float32))
    w.close()


def _env_pair(s, n, m, observers, rewards, seed=0):
    from tactics2d_b200.envs import BatchedTrafficEnv

    cfg = dict(k_agents=4, k_segments=6)
    if observers is not None:
        cfg["observers"] = observers
    kw = dict(max_step=6, observation="agents", vector_obs=cfg, agent_rewards=rewards)
    a = BatchedTrafficEnv(s, agent_actions=True, **kw)
    b = BatchedTrafficEnv(s, **kw)
    return a, b


def _same_step(ra, rb, t):
    import torch

    oa, rwa, tea, tra, ia = ra
    ob, rwb, teb, trb, ib = rb
    assert torch.equal(oa, ob), t
    assert np.array_equal(_bits(rwa), _bits(rwb)) and torch.equal(tea, teb) and torch.equal(tra, trb), t
    assert set(ia) == set(ib), t
    for k in ia:
        assert torch.equal(ia[k], ib[k]), (t, k)


@pytest.mark.parametrize("rewards", [False, True])
def test_env_agent_actions_equal_the_scattered_full_action(cuda_device, rewards):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import InvalidAction

    N, M, Q = 128, 16, 10
    s = synthetic.config2(N, M, seed=90)
    obs_np = _observer_list(np.random.default_rng(91), N, M, Q)
    obs = torch.from_numpy(obs_np).cuda()
    ea, eb = _env_pair(s, N, M, obs, rewards)
    assert ea.action_space["shape"] == (N, Q, 2) and eb.action_space["shape"] == (N, 2)
    oa, _ = ea.reset(seed=1)
    ob, _ = eb.reset(seed=1)
    assert torch.equal(oa, ob)
    full = np.zeros((N, M, 2), np.float32)
    resets = 0
    for t in range(14):
        rows = synthetic.random_actions(900 + t, (N, Q))[..., ::-1].copy()   # (steer, accel)
        full = scatter_agent_action(full, rows, eb.world.type_id.cpu().numpy(), len(eb.world.type_table), obs_np)
        ra = ea.step(torch.from_numpy(rows).cuda())
        rb = eb.step(torch.from_numpy(full).cuda())
        _same_step(ra, rb, t)
        resets += int(ea.world.step_count.eq(0).sum())
    assert resets >= N   # max_step 6: every scenario auto-reset
    # npc_action fills the slots no agent drives
    npc = torch.full((N, M, 2), 0.25, device=cuda_device)
    rows = synthetic.random_actions(950, (N, Q))
    ea.step(torch.from_numpy(rows).cuda(), npc_action=npc)
    full = scatter_agent_action(np.full((N, M, 2), 0.25, np.float32), rows, eb.world.type_id.cpu().numpy(),
                                len(eb.world.type_table), obs_np)
    eb.step(torch.from_numpy(full).cuda())
    assert torch.equal(ea._action.cpu(), torch.from_numpy(full))
    for k in STATE:
        assert torch.equal(getattr(ea.world, k), getattr(eb.world, k)), k
    for bad in ((N, 2), (N, M, 2), (N, Q + 1, 2), (N, Q)):
        with pytest.raises(InvalidAction):
            ea.step(torch.zeros(bad, device=cuda_device))
    for e in (ea, eb):
        e.close()


@pytest.mark.parametrize("rewards", [False, True])
def test_env_with_one_row_on_slot_zero_is_the_ego_env(cuda_device, rewards):
    import torch
    from tactics2d_b200 import synthetic

    N, M = 128, 16
    s = synthetic.config2(N, M, seed=95)
    ea, eb = _env_pair(s, N, M, torch.zeros((N, 1), dtype=torch.int16, device=cuda_device), rewards)
    assert ea.action_space["shape"] == (N, 1, 2)
    oa, _ = ea.reset(seed=2)
    ob, _ = eb.reset(seed=2)
    assert torch.equal(oa, ob)
    for t in range(14):
        ego = torch.from_numpy(synthetic.random_actions(960 + t, (N, 1))[..., ::-1].copy()).cuda()
        _same_step(ea.step(ego), eb.step(ego[:, 0].contiguous()), t)
    for e in (ea, eb):
        e.close()


def test_env_without_agent_actions_keeps_its_action_space(cuda_device):
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    s = synthetic.config2(16, 8, seed=97)
    env = BatchedTrafficEnv(s, observation="agents", vector_obs=dict(k_agents=2, k_segments=2))
    assert env.action_space["shape"] == (16, 2) and not env.agent_actions
    env.close()
    with pytest.raises(ValueError):
        BatchedTrafficEnv(s, observation="vector", agent_actions=True)
