"""Route following on the device (DESIGN.md section 1 "Route following"): OffRoute and the progress term of the env
epilogue and K10 against tests/route_oracle.py at odd N and M, Q up to 128, their place in the status chain, no change
without routes, one K10 row on slot 0 = the env epilogue, K12 (t2d_route_observe) against the oracle inside guarded
buffers, the env through resets and shuffles, a replayed ego on its own logged track, and the C-level rejections."""

import ctypes as C

import numpy as np
import pytest

from oracle import scenario as O
from tests import agent_reward_oracle as R
from tests import route_oracle as RO

pytestmark = pytest.mark.gpu

THRESHOLD, WEIGHT, OFF_REWARD = 3.0, 0.25, -4.0


def _bits(t):
    return t.detach().cpu().numpy().view(np.uint8)


def _world(N, M, seed, max_step=50):
    import torch

    from tactics2d_b200 import BatchedWorld, synthetic

    s = synthetic.config2(N, M, seed=seed)
    w = BatchedWorld(N, M, s.table, max_step=max_step, steer_first=True)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    return w, s, torch.zeros((N, M, 2), dtype=torch.float32, device=w.device)


def _random_routes(s, seed, n_paths=48):
    """Routes of 2..64 vertices near the participants (some with zero-length segments, one all zero-length), and a
    route id per slot with -1 and ids the table does not hold among them."""
    rng = np.random.default_rng(seed)
    N, M = s.shape
    paths = []
    for p in range(n_paths):
        nv = int(rng.integers(2, 65))
        n, m = int(rng.integers(0, N)), int(rng.integers(0, M))
        c = np.array([s.x[n, m], s.y[n, m]], np.float64)
        pts = c + np.cumsum(rng.normal(0, 2.5, (nv, 2)), 0) - rng.normal(0, 2.0, 2)
        if p % 7 == 3:
            pts[nv // 2] = pts[max(0, nv // 2 - 1)]                    # a zero-length segment
        paths.append(pts.astype(np.float32))
    paths[5] = np.repeat(paths[5][:1], 3, 0)                          # no segment of non-zero length: no route
    rid = rng.integers(-2, n_paths + 3, (N, M)).astype(np.int16)
    # give most slots a route that passes close by: a path through their own position
    near = rng.uniform(0, 1, (N, M)) < 0.5
    for n, m in zip(*np.nonzero(near)):
        if len(paths) >= 32000:
            break
        h = float(s.heading[n, m]) + rng.normal(0, 0.3)
        off = rng.normal(0, 2.5)
        t = np.linspace(-20, 20, int(rng.integers(2, 9)))
        base = np.array([s.x[n, m] - off * np.sin(h), s.y[n, m] + off * np.cos(h)], np.float64)
        paths.append((base + t[:, None] * [np.cos(h), np.sin(h)]).astype(np.float32))
        rid[n, m] = len(paths) - 1
    return paths, rid


def _far_from_threshold(paths, rid, x, y, slots):
    for n, m in slots:
        r = int(rid[n, m])
        if 0 <= r < len(paths):
            c = RO.closest(paths[r], float(x[n, m]), float(y[n, m]))
            if c is not None:
                assert abs(c[4] - THRESHOLD) > 1e-9, "a case lies on the threshold: draw another seed"


def _np(t):
    return t.detach().cpu().numpy()


@pytest.mark.parametrize("N,M", [(4099, 64), (257, 33), (129, 128), (65, 1)])
def test_env_epilogue_against_the_oracle(cuda_device, N, M):
    w, s, act = _world(N, M, seed=N + M)
    paths, rid = _random_routes(s, seed=N)
    w.set_paths(paths)
    w.set_routes(rid, THRESHOLD, WEIGHT, OFF_REWARD)
    seen_off = seen_prog = 0
    for t in range(3):
        pre_sb = _np(w.route_s_best).copy()
        r = w.step(act)
        st, fl = _np(r.status), _np(r.flags)
        x, y = _np(w.x), _np(w.y)
        _far_from_threshold(paths, rid, x, y, [(n, 0) for n in range(N)])
        e = w.env_epilogue()
        ref = RO.env_epilogue(fl, st, _np(w.step_count), w.max_step, x, y, rid, paths, THRESHOLD, WEIGHT, OFF_REWARD, pre_sb)
        assert np.array_equal(_np(e.traffic_status), ref["traffic_status"]), t
        assert np.array_equal(_np(e.terminated), ref["terminated"]) and np.array_equal(_np(e.truncated), ref["truncated"])
        assert np.array_equal(_np(e.done), ref["done"])
        np.testing.assert_allclose(_np(w.route_s_best), ref["s_best"], rtol=1e-15, atol=0)
        np.testing.assert_allclose(_np(e.reward), ref["reward"], rtol=1e-6, atol=5e-6)
        seen_off += int((ref["traffic_status"][:, 0] == RO.OFF_ROUTE).sum())
        seen_prog += int(np.isfinite(ref["s_best"]).sum())
        w.reset(e.done, {k: w.x.new_tensor(getattr(s, k)) for k in ("x", "y", "heading", "speed")})
    assert seen_off > 0 and (M == 1 or seen_prog > 0)


def _k10_expected(w, fl, pre_tid, rid, paths, observers, pre_sb):
    x, y, h = _np(w.x), _np(w.y), _np(w.heading)
    n_types = len(w.type_table)
    base = R.agents_epilogue(fl, pre_tid, x, y, h, _np(w.step_count), w.type_table.as_oracle_table(), n_types,
                             observers=observers, max_step=w.max_step, reset_trackers=False)
    st, state, sv = RO.agent_rows(base["status"], x, y, pre_tid, n_types, rid, paths, THRESHOLD, observers)
    reward = base["reward"].astype(np.float32)
    term, trunc = base["terminated"].copy(), base["truncated"].copy()
    sb = np.array(pre_sb, np.float64)
    off = state == 2
    reward[off] = np.float32(OFF_REWARD)
    term[off], trunc[off] = False, True
    for n, q in zip(*np.nonzero((state == 1) & (base["status"] == O.NORMAL))):
        tt, sb[n, q] = RO.progress(sv[n, q], sb[n, q], WEIGHT)
        reward[n, q] = np.float32(reward[n, q] + np.float32(tt))
    done = ~(st == O.NORMAL).any(1)
    sb[done] = -np.inf
    traffic = base["traffic"].copy()
    for n, q in zip(*np.nonzero(off)):
        traffic[n, q if observers is None else observers[n, q]] = RO.OFF_ROUTE
    return dict(status=st, reward=reward, terminated=term, truncated=trunc, done=done.astype(np.uint8), traffic=traffic,
                s_best=sb)


@pytest.mark.parametrize("N,M,Q", [(1025, 64, 64), (257, 33, 33), (129, 128, 128), (65, 1, 1), (257, 64, 33)])
def test_agents_epilogue_against_the_oracle(cuda_device, N, M, Q):
    import torch

    w, s, act = _world(N, M, seed=3 * N + M)
    paths, rid = _random_routes(s, seed=N + Q)
    w.set_paths(paths)
    observers = None
    if Q != M or M == 33:   # a list with -1, M and duplicates
        rng = np.random.default_rng(Q)
        o = rng.integers(-1, M + 1, (N, Q)).astype(np.int16)
        o[:, 1 % Q] = o[:, 0]
        observers = torch.from_numpy(o).to(w.device)
    w.set_agents(observers)
    w.set_routes(rid, THRESHOLD, WEIGHT, OFF_REWARD)
    obs_np = None if observers is None else _np(observers)
    seen_off = 0
    for t in range(2):
        pre_tid, pre_sb = _np(w.type_id).copy(), _np(w.agent_route_s_best).copy()
        r = w.step(act)
        fl = _np(r.flags)
        a = w.agents_epilogue()
        ref = _k10_expected(w, fl, pre_tid, rid, paths, obs_np, pre_sb)
        for k in ("status", "terminated", "truncated", "done", "traffic"):
            assert np.array_equal(_np(getattr(a, k)).astype(ref[k].dtype), ref[k]), (t, k)
        np.testing.assert_allclose(_np(w.agent_route_s_best), ref["s_best"], rtol=1e-15, atol=0)
        np.testing.assert_allclose(_np(a.reward), ref["reward"], rtol=1e-6, atol=5e-6)
        seen_off += int((ref["traffic"] == RO.OFF_ROUTE).sum())
    assert seen_off > 0


def test_priority_against_every_other_detector(cuda_device):
    """Off route with each higher-priority detector (time, out of bound, collision) and with completion."""
    import torch

    from tactics2d_b200 import BatchedWorld, synthetic
    from tactics2d_b200.types import TypeTable

    s = synthetic.config2(8, 4, seed=2)
    w = BatchedWorld(8, 4, s.table, max_step=5, steer_first=True)
    w.set_map(None, (-1000.0, 1000.0, -1000.0, 1000.0))
    x = np.zeros((8, 4), np.float32)
    y = np.tile(np.arange(4, dtype=np.float32) * 20.0, (8, 1))
    w.set_state(x, y, np.zeros((8, 4), np.float32), np.zeros((8, 4), np.float32), type_id=np.zeros((8, 4), np.uint8))
    w.set_paths([np.array([[0.0, 500.0], [10.0, 500.0]], np.float32)])      # far from everybody: all off route
    w.set_routes(np.zeros((8, 4), np.int16), THRESHOLD, WEIGHT, OFF_REWARD)
    w.check_events()
    for st in (O.NORMAL, O.COMPLETED, O.TIME_EXCEEDED, O.OUT_BOUND, O.NO_ACTION, O.FAILED):
        w._out.status.fill_(st)
        fl = w._out.flags
        fl.zero_()
        if st == O.FAILED:
            fl[:, 0] = 2                                                   # static collision
        e = w.env_epilogue(reset_trackers_on_done=False)
        off = st in (O.NORMAL, O.COMPLETED)
        assert (_np(e.traffic_status)[:, 0] == (RO.OFF_ROUTE if off else (3 if st == O.FAILED else 1))).all(), st
        assert not _np(e.terminated).any() and _np(e.truncated).all(), st
        if off:
            assert (_np(e.reward) == np.float32(OFF_REWARD)).all()
    # K10: every row's own chain - collision and out of bound win, completion loses
    w.set_agents(None)
    w.set_routes(np.zeros((8, 4), np.int16), THRESHOLD, WEIGHT, OFF_REWARD)
    fl = w._out.flags
    fl.zero_()
    fl[:, 1] = 2
    fl[:, 2] = 4
    a = w.agents_epilogue()
    st = _np(a.status)
    assert (st[:, 0] == O.FAILED).all() and (st[:, 1] == O.FAILED).all() and (st[:, 2] == O.OUT_BOUND).all()
    assert (_np(a.traffic)[:, 0] == RO.OFF_ROUTE).all() and (_np(a.traffic)[:, 1] == 3).all()
    assert (_np(a.reward)[:, 0] == np.float32(OFF_REWARD)).all() and (_np(a.reward)[:, 1] == -5.0).all()
    # the exact threshold: d == threshold is on route
    w2 = BatchedWorld(1, 1, TypeTable.vehicles("kinematics"))
    w2.set_state(np.zeros((1, 1)), np.full((1, 1), 3.0), np.zeros((1, 1)), np.zeros((1, 1)), type_id=np.zeros((1, 1)))
    w2.set_paths([np.array([[-5.0, 0.0], [5.0, 0.0]], np.float32)])
    w2.set_routes(np.zeros((1, 1)), 3.0)
    w2.check_events()
    assert int(w2.env_epilogue().traffic_status[0, 0]) == 1
    w2.set_routes(np.zeros((1, 1)), np.nextafter(3.0, 0.0))
    assert int(w2.env_epilogue().traffic_status[0, 0]) == RO.OFF_ROUTE


def _outputs(w, agents):
    e = w.env_epilogue()
    out = [_bits(t).copy() for t in (e.reward, e.terminated, e.truncated, e.done, e.traffic_status)]
    if agents:
        a = w.agents_epilogue()
        out += [_bits(t).copy() for t in (a.reward, a.terminated, a.truncated, a.status, a.iou, a.done, a.traffic)]
    return out


def test_no_routes_no_change(cuda_device):
    import torch

    worlds = []
    for mode in ("never", "unbound", "all_minus_one", "set_none"):
        w, s, act = _world(257, 33, seed=11, max_step=4)
        w.set_goal(np.stack([s.x[:, 0] + 3, s.y[:, 0], s.heading[:, 0], np.full(257, 2.5), np.full(257, 1.2)], 1))
        w.set_agents(torch.from_numpy(np.random.default_rng(1).integers(-1, 34, (257, 40)).astype(np.int16)).to(w.device))
        w.set_paths(_random_routes(s, 5)[0])
        if mode == "all_minus_one":
            w.set_routes(np.full((257, 33), -1, np.int16), THRESHOLD)
        if mode == "set_none":
            w.set_routes(_random_routes(s, 5)[1], THRESHOLD)
            w.set_routes(None)
        worlds.append((w, act))
    ref = None
    for t in range(6):
        outs = []
        for w, act in worlds:
            w.step(act)
            outs.append(_outputs(w, True))
        for o in outs[1:]:
            assert all(np.array_equal(a, b) for a, b in zip(outs[0], o)), t


def test_one_k10_row_on_slot_zero_is_the_env_epilogue(cuda_device):
    import torch

    ws = []
    for _ in range(2):
        w, s, act = _world(513, 16, seed=4, max_step=6)
        paths, rid = _random_routes(s, 9)
        w.set_paths(paths)
        w.set_routes(rid, THRESHOLD, WEIGHT, OFF_REWARD)
        ws.append((w, act))
    ws[1][0].set_agents(torch.zeros((513, 1), dtype=torch.int16, device=ws[1][0].device))
    pool = {k: ws[0][0].x.new_tensor(getattr(s, k)) for k in ("x", "y", "heading", "speed")}
    for t in range(8):
        (we, ae), (wa, aa) = ws
        we.step(ae)
        wa.step(aa)
        e = we.env_epilogue()
        a = wa.agents_epilogue()
        assert np.array_equal(_bits(a.reward[:, 0]), _bits(e.reward)), t
        assert np.array_equal(_np(a.terminated[:, 0]), _np(e.terminated)) and np.array_equal(_np(a.truncated[:, 0]), _np(e.truncated))
        assert np.array_equal(_np(a.done), _np(e.done)), t
        assert np.array_equal(_np(wa.agent_route_s_best[:, 0]), _np(we.route_s_best)), t
        we.reset(e.done, pool)
        wa.reset(a.done, pool)


TAIL = 8


@pytest.mark.parametrize("P", [0, 1, 8, 32])
@pytest.mark.parametrize("N,M,Q", [(257, 33, 40), (65, 128, 128), (9, 1, 1)])
def test_route_observe_against_the_oracle(cuda_device, P, N, M, Q):
    import torch

    from tactics2d_b200 import _lib

    w, s, act = _world(N, M, seed=P + N)
    paths, rid = _random_routes(s, seed=P)
    paths[0] = np.array([[s.x[0, 0], s.y[0, 0]], [s.x[0, 0] + 1.0, s.y[0, 0]]], np.float32)   # shorter than the look-ahead
    rid[0, 0] = 0
    w.set_paths(paths)
    w.set_routes(rid, THRESHOLD)
    tid = _np(w.type_id).copy()
    tid[1 % N, :: 3] = 255                                                                  # empty / retired slots
    w.type_id.copy_(torch.from_numpy(tid))
    rng = np.random.default_rng(P)
    o = rng.integers(-1, M + 1, (N, Q)).astype(np.int16)
    o[:, 0] = 0
    o[:, -1] = o[:, 0]
    obs = torch.from_numpy(o).to(w.device)
    F = RO.FIELDS + 2 * P
    sentinel = np.float32(-7.5e33)
    buf = torch.full((N * Q * F + TAIL * Q * F,), float(sentinel), dtype=torch.float32, device=w.device)
    _lib.check(w.lib.t2d_route_observe(w._ctx, C.c_void_p(obs.data_ptr()), Q, P, 2.5, C.c_void_p(buf.data_ptr()), None))
    got = _np(buf)
    assert (got[N * Q * F:] == sentinel).all()
    ref = RO.observe(_np(w.x), _np(w.y), _np(w.heading), tid, len(w.type_table), rid, paths, P, 2.5, observers=o)
    got = got[:N * Q * F].reshape(N, Q, F)
    assert not (got == sentinel).any()
    assert np.array_equal(got[..., 0], ref[..., 0].astype(np.float32))
    np.testing.assert_allclose(got, ref.astype(np.float32), rtol=2e-6, atol=2e-5)
    assert (ref[..., 0] == 1).any() and (ref[..., 0] == 0).any()
    # the ego form: [N, F], row n = slot 0's
    ego = _np(w.route_observe(P, 2.5))
    assert ego.shape == (N, F) and np.array_equal(ego, got[:, 0])


def test_env_rollouts_with_routes(cuda_device):
    import torch

    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    N, M = 33, 8
    s = synthetic.config2(N, M, seed=6)
    paths, rid = _random_routes(s, seed=6)
    route = dict(paths=paths, route_id=rid, threshold=THRESHOLD, progress_weight=WEIGHT, off_route_reward=OFF_REWARD,
                 n_points=4, spacing=1.5)
    with pytest.raises(ValueError):
        BatchedTrafficEnv(s, route=dict(route, colour=1))
    env = BatchedTrafficEnv(s, max_step=5, route=route)
    obs, info = env.reset(seed=1)
    assert info["route"].shape == (N, RO.FIELDS + 8)
    pool = np.asarray(rid, np.int16)
    assert np.array_equal(_np(env.world.route_id), pool)
    act = torch.full((N, 2), 0.2, device=env.world.device)
    dones = 0
    for t in range(12):
        pre_sb = _np(env.world.route_s_best).copy()
        _, rew, term, trunc, info = env.step(act)
        done = _np(term) | _np(trunc)
        dones += int(done.sum())
        sb = _np(env.world.route_s_best)
        assert np.isneginf(sb[done]).all(), t                 # cleared on done
        assert (sb[~done] >= pre_sb[~done]).all(), t            # the best only grows within an episode
        assert np.array_equal(_np(env.world.route_id), pool)   # an auto-reset keeps every scenario's route
        off = _np(info["traffic_status"])[:, 0] == RO.OFF_ROUTE
        assert _np(trunc)[off].all() and (_np(rew)[off] == np.float32(OFF_REWARD)).all()
        ref = RO.observe(_np(env.world.x), _np(env.world.y), _np(env.world.heading), _np(env.world.type_id), len(s.table),
                         pool, paths, 4, 1.5, Q=1)[:, 0]
        np.testing.assert_allclose(_np(info["route"]), ref.astype(np.float32), rtol=2e-6, atol=2e-5)
    assert dones > 0
    env.reset(options={"shuffle": True})
    assert np.array_equal(_np(env.world.route_id), pool)       # without a log the types and routes stay per scenario
    # agents: [N, Q, F], observers without a list = every slot
    env = BatchedTrafficEnv(s, max_step=5, route=route, observation="agents", vector_obs=dict(k_agents=2, k_segments=2),
                            agent_rewards=True)
    _, info = env.reset()
    assert info["route"].shape == (N, M, RO.FIELDS + 8)
    for t in range(6):
        _, rew, term, trunc, info = env.step(act)
        assert rew.shape == (N, M)
        st = _np(info["agent_status"])
        assert np.isneginf(_np(env.world.agent_route_s_best)[(st != O.NORMAL).all(1)]).all()


def test_replayed_ego_on_its_logged_track(cuda_device, tmp_path):
    from tactics2d_b200 import BatchedWorld
    from tactics2d_b200.dataset_parser import LevelXParser, ReplayLog, build_replay_episodes
    from tests.test_levelx_parser import _write_ind

    _write_ind(tmp_path)
    log = ReplayLog.from_levelx(LevelXParser("inD"), 3, str(tmp_path))
    ep = build_replay_episodes(log, 3, [0, 80, 200], [0, 1, 0])
    paths, rid = ep.ego_routes()
    w = BatchedWorld(3, 3, ep.table, max_step=1000)
    w.set_state(ep.pool["x"], ep.pool["y"], ep.pool["heading"], ep.pool["speed"], type_id=ep.type_id)
    w.set_paths(paths)
    w.set_routes(rid, 0.01, progress_weight=1.0)
    total = np.zeros(3)
    for k in range(max(len(p) for p in paths)):
        xy = np.stack([p[min(k, len(p) - 1)] for p in paths])
        w.x[:, 0] = w.x.new_tensor(xy[:, 0])
        w.y[:, 0] = w.y.new_tensor(xy[:, 1])
        w.check_events()
        w._out.status.fill_(O.NORMAL)
        e = w.env_epilogue(reset_trackers_on_done=False)
        assert (_np(e.traffic_status)[:, 0] != RO.OFF_ROUTE).all(), k
        total += _np(e.reward).astype(np.float64) - (-np.tanh(w.step_count.cpu().numpy() / 1000) * 0.001)
    for p in range(3):
        L = RO.closest(paths[p], paths[p][-1, 0], paths[p][-1, 1])[6]
        assert _np(w.route_s_best)[p] == L
        assert abs(total[p] - L) < 1e-4 * max(1.0, L)


def test_c_level_rejections_keep_the_binding(cuda_device):
    from tactics2d_b200 import _lib

    w, s, act = _world(33, 8, seed=2)
    paths, rid = _random_routes(s, 2)
    w.set_paths(paths)
    w.set_routes(rid, THRESHOLD, WEIGHT, OFF_REWARD)
    w.step(act)
    before = [_bits(t).copy() for t in (w.env_epilogue(reset_trackers_on_done=False).reward,)]
    lib, ctx = w.lib, w._ctx
    ptr = C.c_void_p(w.route_id.data_ptr())
    for thr, wt, off in ((float("nan"), 0.1, -5.0), (-1.0, 0.1, -5.0), (float("inf"), 0.1, -5.0), (1.0, float("nan"), -5.0),
                         (1.0, 0.1, float("inf"))):
        assert lib.t2d_set_routes(ctx, ptr, thr, wt, off) == -1
    out = C.c_void_p(w.x.data_ptr())
    n0 = lib.t2d_launch_count()
    for q, p, sp in ((0, 4, 1.0), (129, 4, 1.0), (9, 4, 1.0), (4, -1, 1.0), (4, 257, 1.0), (4, 4, 0.0), (4, 4, float("nan"))):
        assert lib.t2d_route_observe(ctx, None, q, p, sp, out, None) == -1, (q, p, sp)
    assert lib.t2d_route_observe(ctx, None, 4, 4, 1.0, None, None) == -1
    assert lib.t2d_bind_route_trackers(ctx, None, C.c_void_p(w.x.data_ptr()), 0) == -1
    assert lib.t2d_launch_count() == n0
    # the binding is whole: the same routes, weights and trackers
    w.route_s_best.fill_(-np.inf)
    w.step(act)
    w2, _, act2 = _world(33, 8, seed=2)
    w2.set_paths(paths)
    w2.set_routes(rid, THRESHOLD, WEIGHT, OFF_REWARD)
    w2.step(act2)
    w2.env_epilogue(reset_trackers_on_done=False)
    w2.route_s_best.fill_(-np.inf)
    w2.step(act2)
    assert np.array_equal(_bits(w.env_epilogue().reward), _bits(w2.env_epilogue().reward))
    with pytest.raises(_lib.T2DError):
        w.set_routes(rid, float("nan"))
    assert w.route_id is not None and w._routes["threshold"] == THRESHOLD
