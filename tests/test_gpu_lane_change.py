"""K18 (``t2d_set_lane_change``) against the float64 MOBIL decision (tests/lane_change_oracle.py), K5's lane keeping for
IDM rows, the closed-loop scenes (tests/lane_scenes.py), the host step entries, resets, graph replay, the rejections and
the env's ``info["lane_path"]``."""

import math

import numpy as np
import pytest

from oracle import scenario as O
from tests import lane_change_oracle as LC
from tests import lane_scenes as S
from tests import leader_oracle as L

pytestmark = pytest.mark.gpu

OBB, DISC, NONE = 0, 1, 2
HW, RNG = 1.8, 100.0
KW = dict(politeness=0.3, threshold=0.1, b_safe=3.0, min_gap=7.0, cooldown=12)


def _table():
    from tactics2d_b200.types import TypeParams, TypeTable

    car = TypeParams(half_len=2.4, half_wid=0.95, lf=1.3, lr=1.3, steer_lo=-0.6, steer_hi=0.6, speed_lo=0.0, speed_hi=30.0,
                     accel_lo=-6.0, accel_hi=3.0)
    ped = TypeParams(radius=0.4, model=2, shape=DISC, speed_hi=3.0)
    ghost = TypeParams(half_len=1.0, half_wid=1.0, shape=NONE)
    return TypeTable([car, ped, ghost])


def _paths(curved):
    """Four lanes 3.5 m apart (straight, or gently curved), reaching past every position, then one without a segment."""
    x = np.linspace(-80.0, 260.0, 35)
    bend = 6.0 * np.sin(x / 50.0) if curved else 0.0 * x
    lanes = [np.stack([x, 3.5 * l + bend], 1) for l in range(4)]
    return [p.astype(np.float32) for p in lanes + [np.array([[5.0, 5.0], [5.0, 5.0]])]]


def _ctrls():
    from tactics2d_b200.controller import IDMController, PIDController

    keep = PIDController(dt=0.1, kp_lat=0.03, ki_lat=0.01, kd_lat=0.08, max_steering=0.2, derivative_filter_alpha=0.5,
                         lateral_error="path_cross_track")
    head = PIDController(dt=0.1, kp_lat=0.5, ki_lat=0.0, kd_lat=0.1, lateral_error="path_heading")
    return [IDMController(desired_speed=14.0, min_spacing=10.0, max_acceleration=2.0, comfortable_deceleration=5.0,
                          lateral=keep),
            IDMController(desired_speed=9.0, time_headway=1.2, lateral=head),
            IDMController(desired_speed=12.0)]


def _rows():
    return [{k: getattr(r, k) for k, _ in r._fields_} for r in (c.params() for c in _ctrls())]


def _scene(n, m, seed, curved):
    rng = np.random.default_rng(seed)
    lane = rng.integers(0, 4, (n, m))
    x = rng.uniform(-10.0, 170.0, (n, m))
    y = 3.5 * lane + (6.0 * np.sin(x / 50.0) if curved else 0.0) + rng.normal(0.0, 0.5, (n, m))
    h = rng.normal(0.0, 0.05, (n, m))
    v = rng.uniform(2.0, 16.0, (n, m))
    tid = rng.choice([0, 0, 0, 0, 1, 2], size=(n, m)).astype(np.uint8)
    tid[rng.random((n, m)) < 0.1] = 255
    cid = rng.choice([0, 0, 0, 1, 2, 255], size=(n, m)).astype(np.uint8)
    cid[:, 0] = 255                                             # the ego is driven by the caller
    pid = np.where(rng.random((n, m)) < 0.9, lane, rng.integers(-1, 6, (n, m))).astype(np.int16)
    cool = np.where(rng.random((n, m)) < 0.2, rng.integers(1, 4, (n, m)), 0).astype(np.int16)
    left = rng.integers(-1, 5, 5)
    right = rng.integers(-1, 5, 5)
    left[left == np.arange(5)] = -1
    right[right == np.arange(5)] = -1
    left[:3], right[1:4] = [1, 2, 3], [0, 1, 2]    # the lanes' own neighbours, then random links
    return [a.astype(np.float32) for a in (x, y, h, v)] + [tid, cid, pid, cool, left.tolist(), right.tolist()]


def _world(device, n, m, seed, curved, kw=KW):
    from tactics2d_b200 import BatchedWorld

    x, y, h, v, tid, cid, pid, cool, left, right = _scene(n, m, seed, curved)
    w = BatchedWorld(n, m, _table(), device=device)
    w.set_state(x, y, h, v, type_id=tid)
    w.set_paths(_paths(curved))
    w.set_controllers(_ctrls(), cid, path_id=pid)
    w.set_leader_search(HW, RNG)
    w.set_lane_change(left, right, **kw)
    return w, (x, y, h, v, tid, cid, pid, cool, left, right)


def _oracle(w, sc, lane_path, cool, kw=KW):
    x, y, h, v, tid, cid, pid, _, left, right = sc
    st = w.state_numpy()
    return LC.decide(st["x"], st["y"], st["speed"], tid, [OBB, DISC, NONE], cid, _rows(), lane_path, cool, left, right,
                     w.paths, HW, RNG,
                     **{k: kw[k] for k in ("politeness", "threshold", "b_safe", "min_gap")}, cool_ticks=kw["cooldown"])


def _check(w, ref, min_robust=0.9):
    r = ref["robust"]
    assert r.mean() >= min_robust, r.mean()
    for got, want in ((w.lane_path, ref["lane_path"]), (w.lane_cooldown, ref["cooldown"]), (w.lane_change, ref["change"])):
        got = got.cpu().numpy()
        assert np.array_equal(got[r], want[r])


@pytest.mark.parametrize("m", [1, 2, 33, 64, 97, 128])
@pytest.mark.parametrize("curved", [False, True])
def test_k18_matches_oracle(cuda_device, m, curved):
    import torch

    n = 23
    w, sc = _world(cuda_device, n, m, seed=m + 100 * curved, curved=curved)
    lane_in = w.lane_path.cpu().numpy()
    assert np.array_equal(lane_in, sc[6])                     # the binding copied path_id
    w.lane_cooldown.copy_(torch.from_numpy(sc[7]).to(cuda_device))
    w.lane_change.fill_(99)                                   # sentinel: every slot is written
    ref = _oracle(w, sc, lane_in, sc[7])
    w.control(torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device))
    assert not (w.lane_change == 99).any()
    _check(w, ref)
    if m >= 33:
        assert ref["changer"].sum() > 0 and (ref["change"] != 0).sum() > 0


def test_idm_lane_keeping_matches_oracle(cuda_device):
    import torch

    n, m = 9, 40
    w, sc = _world(cuda_device, n, m, seed=3, curved=True)
    w.set_lane_change(None)
    x, y, h, v, tid, cid, pid, *_ = sc
    rng = np.random.default_rng(4)
    state = rng.normal(0.0, 0.2, (n, m, 6))
    w.pid_state.copy_(torch.from_numpy(state).to(cuda_device))
    table = _table().as_oracle_table()
    tid_o = np.where(tid < 3, tid, 255)
    for t in range(3):
        before = w.state_numpy()
        ps = w.pid_state.cpu().numpy()
        lead = w.find_leaders(HW, RNG)[0].cpu().numpy()
        la = w.last_accel.cpu().numpy()
        act = w.control(torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device)).cpu().numpy()
        want, want_la, want_ps = LC.control_tick(before, tid_o, table, np.zeros((n, m, 2), np.float32), cid, _rows(), lead,
                                                 pid, w.paths, la, ps)
        ctl = (cid != 255) & (tid < 3)
        np.testing.assert_allclose(act[ctl, 0], want[ctl, 0], rtol=3e-6, atol=3e-6)    # idm_law
        np.testing.assert_allclose(act[ctl, 1], want[ctl, 1], rtol=1e-6, atol=1e-6)    # the lateral channel
        np.testing.assert_allclose(w.pid_state.cpu().numpy(), want_ps, rtol=1e-9, atol=1e-9)
        assert (np.abs(act[ctl, 1]) > 0).sum() > 0
        w.step(torch.from_numpy(act).to(cuda_device))


@pytest.mark.parametrize("scene", ["highway", "rings"])
def test_closed_loop_scene_matches_oracle(cuda_device, scene):
    import torch

    from tactics2d_b200 import BatchedWorld

    st, tid, cid, pid, paths, left, right, lane0 = getattr(S, scene)()
    m = tid.shape[1]
    w = BatchedWorld(1, m, S.table(), device=cuda_device)
    w.set_state(st["x"], st["y"], st["heading"], st["speed"], type_id=tid)
    w.set_paths(paths)
    w.set_controllers(S.controllers(), cid, path_id=pid)
    w.set_leader_search(S.HALF_WIDTH, S.MAX_RANGE)
    w.set_lane_change(left, right, **S.LANE)
    table = S.table().as_oracle_table()
    hits = np.zeros(m, np.uint8)
    lefts = 0
    for t in range(150):
        before = w.state_numpy()
        lane, cool, ps, la = (a.cpu().numpy() for a in (w.lane_path, w.lane_cooldown, w.pid_state, w.last_accel))
        ref = LC.decide(before["x"], before["y"], before["speed"], tid, [OBB], cid, S.ctab(), lane, cool, left, right,
                        paths, S.HALF_WIDTH, S.MAX_RANGE, **{k: S.LANE[k] for k in ("politeness", "threshold", "b_safe",
                                                                                   "min_gap")},
                        cool_ticks=S.LANE["cooldown"])
        act = w.control(torch.zeros((1, m, 2), dtype=torch.float32, device=cuda_device)).cpu().numpy()
        _check(w, ref, min_robust=0.0)
        lefts += int((w.lane_change.cpu().numpy()[0, lane0] == 1).sum())
        lead = L.find(before["x"], before["y"], before["heading"], tid, [OBB], S.HALF_WIDTH, S.MAX_RANGE,
                      w.lane_path.cpu().numpy(), paths)
        want, _, _ = LC.control_tick(before, tid, table, np.zeros((1, m, 2), np.float32), cid, S.ctab(), lead["lead"],
                                     w.lane_path.cpu().numpy(), paths, la, ps)
        ok = lead["robust"][0]
        np.testing.assert_allclose(act[0, ok], want[0, ok], rtol=1e-5, atol=1e-5)
        r = w.step(torch.from_numpy(act).to(cuda_device))
        hits |= r.flags[0].cpu().numpy() & O.F_DYNAMIC
    assert not hits.any() and lefts > 0


def test_step_host_ego_and_agents_equal_the_device_sequence(cuda_device):
    import torch

    n, m = 11, 40
    worlds = [_world(cuda_device, n, m, seed=8, curved=False)[0] for _ in range(3)]
    w1, w2, w3 = worlds
    w3.set_agents(torch.zeros((n, 1), dtype=torch.int16, device=cuda_device))
    a1, a2, a3 = (torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device) for _ in range(3))
    rng = np.random.default_rng(5)
    for t in range(5):
        ego = rng.uniform(-0.2, 0.2, (n, 2)).astype(np.float32)
        w1.set_ego_action(torch.from_numpy(ego).to(cuda_device))
        w1.control(a1)
        w1.step(a1)
        w2.step_host_ego(ego, a2)
        w3.set_ego_action(torch.from_numpy(ego).to(cuda_device))
        w3.step_host_agents(ego[:, None, :], a3)
        torch.cuda.synchronize()
        for w in ((w2, w3) if t == 0 else (w2,)):   # K10 may retire slots of w3 after its first step
            for k in ("lane_path", "lane_cooldown", "lane_change"):
                assert torch.equal(getattr(w1, k), getattr(w, k)), (t, k)
        for k in ("x", "y", "heading", "speed"):
            assert torch.equal(getattr(w1, k), getattr(w2, k)), (t, k)


def test_reset_restores_the_starting_lanes(cuda_device):
    import torch

    n, m = 6, 16
    w, sc = _world(cuda_device, n, m, seed=2, curved=False)
    pool = {k: getattr(w, k).clone() for k in ("x", "y", "heading", "speed")}
    w.lane_path.fill_(3)
    w.lane_cooldown.fill_(5)
    w.lane_change.fill_(1)
    mask = torch.tensor([1, 0, 1, 0, 0, 1], dtype=torch.uint8, device=cuda_device)
    w.reset(mask, pool)
    torch.cuda.synchronize()
    keep = ~mask.bool()
    assert torch.equal(w.lane_path[mask.bool()], torch.from_numpy(sc[6]).to(cuda_device)[mask.bool()])
    assert (w.lane_cooldown[mask.bool()] == 0).all() and (w.lane_change[mask.bool()] == 0).all()
    assert (w.lane_path[keep] == 3).all() and (w.lane_cooldown[keep] == 5).all() and (w.lane_change[keep] == 1).all()
    w.set_reset_sampler(7, tries=2)
    w.lane_path.fill_(3)
    w.lane_cooldown.fill_(5)
    w.reset_sampled(mask, pool)
    torch.cuda.synchronize()
    assert torch.equal(w.lane_path[mask.bool()], torch.from_numpy(sc[6]).to(cuda_device)[mask.bool()])
    assert (w.lane_cooldown[mask.bool()] == 0).all() and (w.lane_path[keep] == 3).all()


def test_graph_capture_of_control(cuda_device):
    import torch

    n, m = 7, 48
    w1, _ = _world(cuda_device, n, m, seed=11, curved=True)
    w2, _ = _world(cuda_device, n, m, seed=11, curved=True)
    a1 = torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device)
    a2 = a1.clone()
    s = torch.cuda.Stream(cuda_device)
    s.wait_stream(torch.cuda.current_stream(cuda_device))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            w2.control(a2)
    torch.cuda.current_stream(cuda_device).wait_stream(s)
    for t in range(3):
        w1.control(a1)
        g.replay()
        torch.cuda.synchronize()
        for k in ("lane_path", "lane_cooldown", "lane_change", "leader"):
            assert torch.equal(getattr(w1, k), getattr(w2, k)), (t, k)
        assert torch.equal(a1, a2)


def test_rejections_keep_the_binding_and_rebinds_drop_it(cuda_device):
    import ctypes as C

    import torch

    from tactics2d_b200 import _lib

    n, m = 4, 8
    w, sc = _world(cuda_device, n, m, seed=1, curved=False)
    left, right = sc[8], sc[9]
    lp = w.lane_path
    bad = [dict(politeness=-0.1), dict(politeness=math.nan), dict(threshold=math.inf), dict(b_safe=0.0),
           dict(min_gap=0.0), dict(min_gap=RNG + 1.0), dict(cooldown=-1), dict(cooldown=40000)]
    for b in bad:
        with pytest.raises(_lib.T2DError):
            w.set_lane_change(left, right, **dict(KW, **b))
    for l2 in ([0] + left[1:], [5] + left[1:], [-2] + left[1:]):   # names itself, outside the table
        with pytest.raises(_lib.T2DError):
            w.set_lane_change(l2, right, **KW)
    assert w.lane_path is lp
    w.lane_change.fill_(99)
    w.control(torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device))
    assert not (w.lane_change == 99).any()                    # the kept binding ran
    p = _lib.LaneChangeParamsC(politeness=0.0, threshold=0.2, b_safe=2.0, min_gap=6.0, cooldown=10)
    nb = np.zeros(5, np.int16) - 1
    buf = torch.zeros(n * m + 1, dtype=torch.int16, device=cuda_device)
    odd = C.c_void_p(buf.data_ptr() + 1)
    ok = C.c_void_p(buf.data_ptr())
    lib, ctx = w.lib, w._ctx
    assert lib.t2d_set_lane_change(ctx, C.byref(p), C.c_void_p(nb.ctypes.data), C.c_void_p(nb.ctypes.data), odd, ok,
                                   None) == -1
    assert lib.t2d_set_lane_change(ctx, C.byref(p), None, C.c_void_p(nb.ctypes.data), ok, ok, None) == -1
    w.set_leader_search(None)                                 # unbinding the search drops it
    assert w.lane_path is None
    assert lib.t2d_set_lane_change(ctx, C.byref(p), C.c_void_p(nb.ctypes.data), C.c_void_p(nb.ctypes.data), ok,
                                   C.c_void_p(buf.data_ptr() + 2), None) == -4      # no search: T2D_E_STATE
    w.set_leader_search(HW, RNG)
    w.set_lane_change(left, right, **KW)
    w.set_paths(w.paths)
    assert w.lane_path is None
    w.set_lane_change(left, right, **KW)
    w.set_controllers(_ctrls(), sc[5], path_id=sc[6])
    assert w.lane_path is None
    w.set_lane_change(left, right, **KW)
    w.set_controllers(_ctrls(), sc[5])                        # no path_id
    with pytest.raises(_lib.T2DError):
        w.set_lane_change(left, right, **KW)
    # nothing bound: control launches what it did before, on path_id
    w.set_controllers(_ctrls(), sc[5], path_id=sc[6])
    w.control(torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device))


def test_env_info_lane_path_after_auto_reset(cuda_device):
    import torch

    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    n, m = 8, 12
    scene = synthetic.config2(n, m, seed=3)
    with pytest.raises(ValueError):
        BatchedTrafficEnv(scene, device=cuda_device, lane_change=dict(left=[-1], right=[-1]))
    with pytest.raises(ValueError):
        BatchedTrafficEnv(scene, device=cuda_device, leaders={}, lane_change=dict(left=[-1], right=[-1], gap=3.0))
    env = BatchedTrafficEnv(scene, device=cuda_device, max_step=3, leaders=dict(half_width=1.8, max_range=60.0),
                            lane_change=dict(left=[1, -1], right=[-1, 0], threshold=-1e9, min_gap=1e-3, cooldown=0))
    ys = np.asarray(scene.y)
    env.world.set_paths([np.array([[-500.0, 0.0], [500.0, 0.0]]), np.array([[-500.0, 3.5], [500.0, 3.5]])])
    pid = np.zeros((n, m), np.int16)
    cid = np.zeros((n, m), np.uint8)
    cid[:, 0] = 255
    env.world.set_controllers(_ctrls()[:1], cid, path_id=pid)
    _, info = env.reset(seed=0)
    assert torch.equal(info["lane_path"], torch.from_numpy(pid).to(cuda_device))
    assert (info["lane_change"] == 0).all()
    for t in range(4):
        _, _, _, _, info = env.step(torch.zeros((n, 2), dtype=torch.float32, device=cuda_device))
        if t == 2:   # every scenario ended at max_step and was reset: back on path_id with no decision
            assert torch.equal(info["lane_path"], torch.from_numpy(pid).to(cuda_device))
            assert (info["lane_change"] == 0).all()
        assert info["lane_path"].shape == (n, m) and info["lane_change"].dtype == torch.int8
    assert ys.shape == (n, m)
