"""K17 (``t2d_find_leaders`` / ``t2d_set_leader_search``) against the float64 leader search (tests/leader_oracle.py), K5
following the search's leaders, the host step entries, the rejections and the env's ``info["leader"]``."""

import math

import numpy as np
import pytest

from oracle import controllers as OC
from oracle import scenario as O
from tests import leader_oracle as L
from tests import leader_scenes as S

pytestmark = pytest.mark.gpu

OBB, DISC, NONE = 0, 1, 2


def _table():
    from tactics2d_b200.types import TypeParams, TypeTable

    car = TypeParams(half_len=2.4, half_wid=0.95, lf=1.3, lr=1.3, steer_lo=-0.6, steer_hi=0.6, speed_lo=-5.0, speed_hi=30.0,
                     accel_lo=-6.0, accel_hi=3.0)
    ped = TypeParams(radius=0.4, model=2, shape=DISC, speed_hi=3.0)
    ghost = TypeParams(half_len=1.0, half_wid=1.0, shape=NONE)
    return TypeTable([car, ped, ghost])


def _paths():
    """Three lanes with a kink and a curved one, reaching past every position so that no projection is clamped to an
    end (a clamp puts several slots at one arc length: exact ties), then a path without a segment of non-zero length."""
    lanes = [np.array([[-60.0, 3.5 * l], [60.0, 3.5 * l + 0.5], [240.0, 3.5 * l]]) for l in range(3)]
    x = np.linspace(-60.0, 240.0, 33)
    curve = np.stack([x, 10.5 + 2.0 * np.sin(x / 30.0)], 1)
    return [p.astype(np.float32) for p in lanes + [curve, np.array([[5.0, 5.0], [5.0, 5.0]])]]


def _scene(n, m, seed, nan=False):
    """Participants along four lanes, some reversed, 15 % empty slots, some retired (type 200); with ``nan`` a few NaN
    positions (only for the search alone: the tick is not asked to move them)."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(-10.0, 170.0, (n, m))
    y = 3.5 * rng.integers(0, 4, (n, m)) + rng.normal(0.0, 0.6, (n, m))
    h = rng.normal(0.0, 0.08, (n, m)) + np.where(rng.random((n, m)) < 0.1, math.pi, 0.0)
    tid = rng.choice([0, 0, 0, 1, 2], size=(n, m)).astype(np.uint8)
    tid[rng.random((n, m)) < 0.15] = 255
    tid[rng.random((n, m)) < 0.05] = 200
    if nan:
        x[rng.random((n, m)) < 0.01] = np.nan
    pid = rng.integers(-1, 6, (n, m)).astype(np.int16)          # 5: not in the table; 4: no segment of non-zero length
    return [a.astype(np.float32) for a in (x, y, h)] + [tid, pid]


def _world(device, n, m, seed, paths=True, nan=False):
    from tactics2d_b200 import BatchedWorld
    from tactics2d_b200.controller import IDMController

    x, y, h, tid, pid = _scene(n, m, seed, nan)
    w = BatchedWorld(n, m, _table(), device=device)
    w.set_state(x, y, h, np.full((n, m), 8.0, np.float32), type_id=tid)
    if paths:
        w.set_paths(_paths())
        w.set_controllers([IDMController()], np.full((n, m), 255, np.uint8), path_id=pid)
    return w, (x, y, h, tid, pid if paths else None)


def _ulp32(v):
    v = np.abs(np.asarray(v, np.float32))
    return (np.nextafter(v, np.float32(np.inf)) - v).astype(np.float64)


def _check(lead, gap, ref, min_robust=0.99):
    """Leaders exact on every robust follower; path-frame gaps bit-exact, heading-frame gaps within K8's tolerance."""
    r = ref["robust"]
    assert r.mean() >= min_robust, r.mean()
    assert np.array_equal(lead[r], ref["lead"][r])
    both = r & (ref["lead"] >= 0)
    path = both & (ref["frame"] == L.PATH)
    assert np.array_equal(gap[path], ref["gap"][path].astype(np.float32))
    head = both & (ref["frame"] == L.HEADING)
    want = ref["gap"][head]
    assert np.all(np.abs(gap[head].astype(np.float64) - want) <= _ulp32(want) + 1e-12 * (1.0 + want))
    none = r & (ref["lead"] < 0)
    assert np.all(gap[none] == np.inf)


@pytest.mark.parametrize("m", [1, 5, 33, 64, 128])
@pytest.mark.parametrize("paths", [False, True])
def test_find_leaders_matches_oracle(cuda_device, m, paths):
    n = 24
    w, (x, y, h, tid, pid) = _world(cuda_device, n, m, seed=m + 7 * paths, paths=paths, nan=True)
    lead, gap = w.find_leaders(1.8, 100.0)
    ref = L.find(x, y, h, tid, [OBB, DISC, NONE], 1.8, 100.0, pid, _paths() if paths else None)
    _check(lead.cpu().numpy(), gap.cpu().numpy(), ref)
    if m >= 33:
        assert (ref["lead"] >= 0).mean() > 0.3
        if paths:
            assert (ref["frame"] == L.PATH).sum() > 0 and (ref["frame"] == L.HEADING).sum() > 0


def _ctrl_world(device, n, m, seed):
    from tactics2d_b200.controller import AccelerationController, IDMController

    w, (x, y, h, tid, pid) = _world(device, n, m, seed)
    rng = np.random.default_rng(seed + 1)
    cid = rng.choice([255, 0, 1, 2], size=(n, m)).astype(np.uint8)
    cid[:, 0] = 255                                             # the ego is driven by the caller
    lead = rng.integers(-1, m, (n, m)).astype(np.int16)
    ctrls = [IDMController(), IDMController(desired_speed=20.0, max_acceleration=2.0), AccelerationController(target_speed=9.0)]
    la = rng.uniform(0.0, 2.0, (n, m)).astype(np.float32)
    w.set_controllers(ctrls, cid, lead_index=lead, path_id=pid, last_accel=la)
    return w, ctrls, cid, pid, la


def test_control_with_search_equals_find_then_lead_index(cuda_device):
    import torch

    n, m = 40, 64
    w1, ctrls, cid, pid, la = _ctrl_world(cuda_device, n, m, 3)
    w2, *_ = _ctrl_world(cuda_device, n, m, 3)
    ext = torch.from_numpy(np.random.default_rng(4).uniform(-1, 1, (n, m, 2)).astype(np.float32)).to(cuda_device)
    w1.set_leader_search(1.8, 100.0)
    a1 = w1.control(ext.clone())
    lead, gap = w2.find_leaders(1.8, 100.0)
    assert torch.equal(w1.leader, lead) and torch.equal(w1.leader_gap, gap)
    w2.set_controllers(ctrls, cid, lead_index=lead.clone(), path_id=pid, last_accel=la)
    a2 = w2.control(ext.clone())
    assert torch.equal(a1, a2)
    assert torch.equal(w1.last_accel, w2.last_accel)


def test_control_then_step_rollout_matches_oracle(cuda_device):
    import torch

    from tactics2d_b200 import synthetic

    n, m = 16, 48
    w, ctrls, cid, pid, _ = _ctrl_world(cuda_device, n, m, 9)
    w.set_leader_search(2.0, 60.0)
    table = _table().as_oracle_table()
    ctab = [{k: getattr(r, k) for k, _ in r._fields_} for r in (c.params() for c in ctrls)]
    x, y, h, tid, _ = _scene(n, m, 9)
    controlled = (cid != 255) & (tid < 3)
    paths64 = [p.astype(np.float64) for p in _paths()]
    la = w.last_accel.cpu().numpy()
    for t in range(6):
        ext = synthetic.random_actions(300 + t, (n, m))
        before = w.state_numpy()
        ref = L.find(before["x"], before["y"], before["heading"], tid, [OBB, DISC, NONE], 2.0, 60.0, pid, _paths())
        act = w.control(torch.from_numpy(ext).to(cuda_device)).cpu().numpy()
        got_lead = w.leader.cpu().numpy()
        _check(got_lead, w.leader_gap.cpu().numpy(), ref, min_robust=0.98)
        want_act, want_la = OC.control_tick(before, np.where(tid < 3, tid, 255), table, ext, cid, ctab, got_lead, pid,
                                            paths64, la)
        assert np.array_equal(act[~controlled], ext[~controlled])
        np.testing.assert_allclose(act[controlled], want_act[controlled], rtol=3e-6, atol=3e-6)
        la = w.last_accel.cpu().numpy()
        w.step(torch.from_numpy(act).to(cuda_device))
    assert controlled.sum() > 0


def _platoon_world(device, search):
    from tactics2d_b200 import BatchedWorld

    st, tid, cid, pid, paths = S.scene()
    w = BatchedWorld(1, tid.shape[1], S.table(), device=device)
    w.set_state(st["x"], st["y"], st["heading"], st["speed"], type_id=tid)
    w.set_paths(paths)
    w.set_controllers(S.controllers(), cid, path_id=pid)
    if search:
        w.set_leader_search(S.HALF_WIDTH, S.MAX_RANGE)
    return w


def test_platoon_and_cut_in_closed_loop_on_device(cuda_device):
    import torch

    for search in (True, False):
        w = _platoon_world(cuda_device, search)
        m = w.M
        hits = np.zeros(m, np.uint8)
        followed_cut_in = False
        for t in range(100):
            act = w.control(torch.from_numpy(S.script(t, m)).to(cuda_device))
            if search:
                followed_cut_in |= int(w.leader[0, 1]) == S.CUT_IN
            r = w.step(act)
            hits |= r.flags[0].cpu().numpy() & O.F_DYNAMIC
        if search:
            assert not hits[S.IDM_SLOTS].any() and followed_cut_in
        else:
            assert hits[S.IDM_SLOTS].any()


def test_step_host_ego_equals_the_device_sequence(cuda_device):
    import torch

    n, m = 32, 40
    w1, *_ = _ctrl_world(cuda_device, n, m, 21)
    w2, *_ = _ctrl_world(cuda_device, n, m, 21)
    for w in (w1, w2):
        w.set_leader_search(1.8, 80.0)
    a1 = torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device)
    a2 = a1.clone()
    rng = np.random.default_rng(5)
    for t in range(5):
        ego = rng.uniform(-1, 1, (n, 2)).astype(np.float32)
        w1.set_ego_action(torch.from_numpy(ego).to(cuda_device))
        w1.control(a1)
        w1.step(a1)
        w2.step_host_ego(ego, a2)
        torch.cuda.synchronize()
        assert torch.equal(w1.leader, w2.leader)
        for k in ("x", "y", "heading", "speed"):
            assert torch.equal(getattr(w1, k), getattr(w2, k)), (t, k)
        assert torch.equal(w1.last_accel, w2.last_accel)


def test_rejections_keep_the_binding(cuda_device):
    import ctypes as C

    import torch

    from tactics2d_b200 import _lib

    w, *_ = _ctrl_world(cuda_device, 4, 8, 1)
    w.set_leader_search(1.8, 100.0)
    lead, gap = w.leader, w.leader_gap
    for hw, rng in ((0.0, 100.0), (100.5, 100.0), (math.nan, 100.0), (1.8, 0.0), (1.8, 1.0e5 + 1.0), (1.8, math.inf)):
        with pytest.raises(_lib.T2DError):
            w.set_leader_search(hw, rng)
        with pytest.raises(_lib.T2DError):
            w.find_leaders(hw, rng)
    assert w.leader is lead
    lead.fill_(99)
    w.control(torch.zeros((4, 8, 2), dtype=torch.float32, device=cuda_device))
    assert torch.equal(lead, w.find_leaders(1.8, 100.0)[0])   # the kept binding is what control wrote
    ctx, s = w._ctx, w._stream()
    buf = torch.zeros(4 * 8 + 2, dtype=torch.int16, device=cuda_device)
    g = torch.zeros(4 * 8 + 1, dtype=torch.float32, device=cuda_device)
    odd = C.c_void_p(buf.data_ptr() + 1)
    assert w.lib.t2d_find_leaders(ctx, 1.8, 100.0, None, None, s) == -1
    assert w.lib.t2d_find_leaders(ctx, 1.8, 100.0, odd, None, s) == -1
    assert w.lib.t2d_find_leaders(ctx, 1.8, 100.0, C.c_void_p(buf.data_ptr()), C.c_void_p(g.data_ptr() + 2), s) == -1
    assert w.lib.t2d_set_leader_search(ctx, 1.8, 100.0, odd, None) == -1
    w.set_leader_search(None)
    assert w.leader is None
    assert w.lib.t2d_set_leader_search(ctx, 1.8, 100.0, None, None) == 0


def test_env_info_leader_after_auto_reset(cuda_device):
    import torch

    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    scene = synthetic.config2(16, 24, seed=3)
    with pytest.raises(ValueError):
        BatchedTrafficEnv(scene, device=cuda_device, leaders=dict(width=2.0))
    env = BatchedTrafficEnv(scene, device=cuda_device, max_step=4, leaders=dict(half_width=2.0, max_range=50.0))
    shapes = scene.table.as_oracle_table()["shape"]
    _, info = env.reset(seed=0)
    for t in range(6):
        if t:
            _, _, _, _, info = env.step(torch.zeros((16, 2), dtype=torch.float32, device=cuda_device))
        st = env.world.state_numpy()
        ref = L.find(st["x"], st["y"], st["heading"], env.world.type_id.cpu().numpy(), shapes, 2.0, 50.0)
        _check(info["leader"].cpu().numpy(), info["leader_gap"].cpu().numpy(), ref)
        assert info["leader"].shape == (16, 24) and info["leader_gap"].dtype == torch.float32
    assert env.world.leader is not None
