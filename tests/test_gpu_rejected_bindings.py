"""A rejected setter leaves every binding whole.  After each call the library refuses, a world keeps stepping bit for bit
like a twin that never saw the call: state, flags, hit indices, status, done, the goal IoU, agents_epilogue, control
with last_accel, and the BEV.  The three host steps interleaved on one world equal the device path on a twin."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, M, Q = 64, 16, 3
RING = np.array([[26, 26, 34, 26], [34, 26, 34, 34], [34, 34, 26, 34], [26, 34, 26, 26]], np.float32)


def _scene():
    from tactics2d_b200 import synthetic

    return synthetic.config2(N, M, seed=21, size=60.0)


def _tiles(s, ring=RING):
    keys = ["curbstone" if i % 2 else "roadline" for i in range(len(s.segments))]
    return [dict(segments=s.segments, bounds=s.bounds, style=keys),
            dict(segments=ring, bounds=(-10.0, 70.0, -10.0, 70.0), poly_start=[0, len(ring)], style=["keepout"] * len(ring))]


def _world(dev, table=False):
    """A world with every binding the rejected setters touch: map (or a two-tile table) with segment styles, goal, agents
    with goals, controllers with pure-pursuit paths, and an ego action."""
    import torch

    from tactics2d_b200 import BatchedWorld
    from tactics2d_b200.controller import IDMController, PurePursuitController

    s = _scene()
    w = BatchedWorld(N, M, s.table, device=dev, max_step=40)
    if table:
        w.set_map_table(_tiles(s), np.arange(N) % 2)
    else:
        w.set_map(s.segments, s.bounds, style=["curbstone"] * len(s.segments))
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    goal = np.stack([s.x[:, 0] + 3.0, s.y[:, 0], s.heading[:, 0], np.full(N, 2.5), np.full(N, 1.2)], 1)
    w.set_goal(goal.astype(np.float32), arrival_threshold=0.6, no_action_max_step=3)
    obs = torch.tensor([[0, 1, 2]] * N, dtype=torch.int16, device=dev)
    g = np.stack([s.x[:, :Q] - 2.0, s.y[:, :Q], s.heading[:, :Q], np.full((N, Q), 2.5), np.full((N, Q), 1.2)], -1)
    g[::4, 1, 0] = np.nan                                   # some rows without a goal
    w.set_agents(obs, torch.from_numpy(g.astype(np.float32)).to(dev), arrival_threshold=0.5, no_action_max_step=4)
    w.set_paths([np.array([[0, 0], [30, 10], [60, 60]], np.float32), np.array([[60, 0], [0, 60]], np.float32)])
    rng = np.random.default_rng(3)
    cid = rng.integers(0, 2, (N, M)).astype(np.uint8)
    cid[:, :Q] = 255                                        # the agents take the caller's actions
    lead = np.tile(np.arange(M, dtype=np.int16) - 1, (N, 1))
    pid = rng.integers(-1, 2, (N, M)).astype(np.int16)
    w.set_controllers([IDMController(), PurePursuitController(min_pre_aiming_distance=4.0, target_speed=6.0)], cid, lead, pid)
    w.set_ego_action(torch.from_numpy(np.random.default_rng(4).uniform(-1, 1, (N, 2)).astype(np.float32)).to(dev))
    return w


def _scribble(dev):
    """Fresh NaN blocks of the sizes the setters allocate: a block the library still reads would now hold NaNs."""
    import torch

    return [torch.full((n,), float("nan"), device=dev) for n in (N, 2 * N, 4 * N, 5 * N, N * Q, 4 * N * Q, 5 * N * Q,
                                                                  N * M, N * M // 4, N * M // 2)]


def _rollout(w, ticks=4):
    import torch

    from tactics2d_b200 import synthetic

    out = []
    for t in range(ticks):
        act = torch.from_numpy(synthetic.random_actions(50 + t, (N, M))).to(w.device)
        w.control(act)
        r = w.step(act)
        e = w.agents_epilogue()
        img = w.bev(resolution=(40, 24), perception_range=25.0, rgb=False)
        snap = dict(act=act, last_accel=w.last_accel, flags=r.flags, hit_index=r.hit_index, hit_segment=r.hit_segment,
                    status=r.status, done=r.done, iou=r.iou, type_id=w.type_id, reward=e.reward, terminated=e.terminated,
                    truncated=e.truncated, agent_status=e.status, agent_iou=e.iou, agent_done=e.done, bev=img,
                    **{k: getattr(w, k) for k in ("x", "y", "heading", "speed", "vx", "vy")})
        out.append({k: np.ascontiguousarray(v.cpu().numpy()) for k, v in snap.items()})
    return out


def _assert_twins(a, b):
    ra, rb = _rollout(a), _rollout(b)
    for t, (sa, sb) in enumerate(zip(ra, rb)):
        for k in sa:
            assert np.array_equal(sa[k].view(np.uint8), sb[k].view(np.uint8)), (t, k)
    last = ra[-1]
    assert (last["flags"] != 0).any() and (last["hit_segment"] >= 0).any() and (last["bev"] != last["bev"][0, 0, 0]).any()


def _reject_goal(w):
    w.set_goal(np.zeros((N, 5), np.float32), arrival_threshold=0.0)


def _reject_agents(w):
    import torch

    obs = torch.zeros((N, Q), dtype=torch.int16, device=w.device)
    w.set_agents(obs, torch.zeros((N, Q, 5), dtype=torch.float32, device=w.device), arrival_threshold=1.5)


def _reject_ego_action(w):
    import torch

    buf = torch.zeros(2 * N + 1, dtype=torch.float32, device=w.device)
    view = buf[1:].view(N, 2)                               # contiguous, but only 4-byte aligned
    assert view.is_contiguous() and view.data_ptr() % 8 == 4
    w.set_ego_action(view)


def _reject_controllers(w):
    from tactics2d_b200 import _lib
    from tactics2d_b200.controller import IDMController

    w.set_controllers([IDMController(), _lib.ControllerParamsC(kind=99)], np.zeros((N, M), np.uint8))


def _reject_map(w):
    seg = _scene().segments.copy()
    seg[3, 1] = np.nan
    w.set_map(seg, (0.0, 60.0, 0.0, 60.0))


def _reject_map_table(w):
    bad = RING.copy()
    bad[3, 3] = 27.0                                        # the last edge no longer returns to the ring's start
    w.set_map_table(_tiles(_scene(), bad), np.zeros(N, np.int64))


def _reject_paths(w):
    w.set_paths([np.array([[0, 0], [10, 0]], np.float32), np.array([[5, 5]], np.float32)])


@pytest.mark.parametrize("reject,table", [
    (_reject_goal, False), (_reject_agents, False), (_reject_ego_action, False), (_reject_controllers, False),
    (_reject_map, False), (_reject_map_table, True), (_reject_paths, False)],
    ids=["set_goal", "set_agents", "set_ego_action", "set_controllers", "set_map", "set_map_table", "set_paths"])
def test_rejected_setter_keeps_the_bindings(cuda_device, reject, table):
    from tactics2d_b200._lib import T2DError

    a, b = _world(cuda_device, table), _world(cuda_device, table)
    with pytest.raises((T2DError, ValueError)):
        reject(a)
    junk = _scribble(cuda_device)
    _assert_twins(a, b)
    del junk
    a.close()
    b.close()


def test_host_steps_interleaved_equal_the_device_path(cuda_device):
    """step_host_ego, step_host, step_host_agents, step_host_ego on one world share and create their staging in turn;
    each equals its device-path equivalent on a twin."""
    import torch

    from tactics2d_b200 import BatchedWorld, synthetic
    from tactics2d_b200.controller import IDMController

    s = _scene()
    worlds = []
    for _ in range(2):
        w = BatchedWorld(N, M, s.table, device=cuda_device, max_step=40)
        w.set_map(s.segments, s.bounds)
        w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
        cid = np.zeros((N, M), np.uint8)
        cid[:, 0] = 255
        w.set_controllers([IDMController()], cid, lead_index=np.tile(np.arange(M, dtype=np.int16) - 1, (N, 1)))
        w.set_agents(torch.tensor([[0, 2, 5]] * N, dtype=torch.int16, device=cuda_device))
        worlds.append(w)
    a, b = worlds
    act_a = torch.zeros((N, M, 2), device=cuda_device)
    act_b = torch.zeros((N, M, 2), device=cuda_device)

    def same_state(t):
        torch.cuda.synchronize()
        for k in ("x", "y", "heading", "speed", "type_id"):
            assert torch.equal(getattr(a, k), getattr(b, k)), (t, k)
        for k in ("flags", "hit_index", "hit_segment"):
            assert torch.equal(getattr(a.result, k), getattr(b.result, k)), (t, k)
        assert torch.equal(act_a, act_b), t

    def ego_step(t):
        ego = synthetic.random_actions(80 + t, (N, 1))[:, 0].copy()
        done, status = a.step_host_ego(ego, act_a)
        b.set_ego_action(torch.from_numpy(ego).to(cuda_device))
        b.control(act_b)
        r = b.step(act_b)
        b.set_ego_action(None)
        same_state(t)
        assert np.array_equal(done, r.done.cpu().numpy()) and np.array_equal(status, r.status.cpu().numpy()), t

    ego_step(0)
    full = synthetic.random_actions(90, (N, M))
    done, status = a.step_host(full)
    r = b.step(torch.from_numpy(full).to(cuda_device))
    same_state(1)
    assert np.array_equal(done, r.done.cpu().numpy()) and np.array_equal(status, r.status.cpu().numpy())
    rows = synthetic.random_actions(91, (N, Q))
    got = a.step_host_agents(rows, act_a)
    b.scatter_agent_action(torch.from_numpy(rows).to(cuda_device), act_b, b._agents["observers"])
    b.control(act_b)
    b.step(act_b)
    e = b.agents_epilogue()
    same_state(2)
    for h, d in zip(got, (e.reward, e.terminated, e.truncated, e.status, e.done)):
        assert np.array_equal(h, d.cpu().numpy())
    ego_step(3)
    assert (a.result.flags.cpu().numpy() != 0).any()
    a.close()
    b.close()
