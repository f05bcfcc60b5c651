"""K19 (``t2d_find_yields`` / ``t2d_set_yielding``) against the float64 statement of DESIGN.md section 1 "Yielding at
conflict zones" (tests/yield_oracle.py), K5's yielding instance, the unbound identity, the closed loop on the
intersection and the roundabout, the highway guard of reactive replay, the rejections and the env."""

import ctypes as C

import numpy as np
import pytest

from tactics2d_b200 import synthetic as S
from tactics2d_b200.traffic.conflicts import conflict_zones
from tests import yield_oracle as Y

pytestmark = pytest.mark.gpu

HW, RANGE = 1.8, 100.0
SENT_I, SENT_F = 12345, -7.0
SCENES = {"intersection": S.intersection, "merge": S.t_junction, "roundabout": S.roundabout}


def _rows():
    """Row 0: the scenes' IDM without lane keeping (K5's acceleration alone); row 1: adaptive cruise (a partner that
    never yields)."""
    from tactics2d_b200.controller import AccelerationController, IDMController

    return [IDMController(desired_speed=10.0, time_headway=1.0, min_spacing=5.0, max_acceleration=2.0,
                          comfortable_deceleration=6.0), AccelerationController(target_speed=8.0)]


def _dicts(rows):
    return [{k: getattr(r, k) for k, _ in r._fields_} for r in (c.params() for c in rows)]


def _state(scene_fn, n, m, seed):
    """A random state of the scene's paths: every slot somewhere along a random path (up to 40 m past its zones), off it
    by N(0, 0.4) m, at 0-12 m/s; 10 % empty; 10 % adaptive cruise; 10 % external; 10 % without a path but with a route
    (partners only)."""
    base = scene_fn(1, 4, seed)
    paths = base.paths
    rng = np.random.default_rng(seed)
    L = [float(np.sum(np.hypot(*np.diff(np.asarray(p, np.float64), axis=0).T))) for p in paths]
    pid = rng.integers(0, len(paths), (n, m)).astype(np.int16)
    x, y, h = (np.zeros((n, m)) for _ in range(3))
    for p in range(len(paths)):
        sel = pid == p
        s = rng.uniform(0.0, min(L[p], 260.0), sel.sum())
        px, py, ph = S._point_at(paths[p], s)
        x[sel] = px + rng.normal(0.0, 0.4, sel.sum())
        y[sel] = py + rng.normal(0.0, 0.4, sel.sum())
        h[sel] = ph
    v = rng.uniform(0.0, 12.0, (n, m))
    tid = np.where(rng.random((n, m)) < 0.1, 255, 0).astype(np.uint8)
    cid = np.zeros((n, m), np.uint8)
    u = rng.random((n, m))
    cid[u < 0.2] = 1
    cid[u < 0.1] = 255
    route = np.full((n, m), -1, np.int16)
    r = rng.random((n, m)) < 0.1
    route[r] = pid[r]
    pid[r] = -1
    prio = rng.integers(0, 2, len(paths)).astype(np.int16)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    return paths, prio, f(x), f(y), f(h), f(v), tid, cid, pid, route


def _world(device, n, m, paths, prio, x, y, h, v, tid, cid, pid, route, yielding=True, rows=None):
    from tactics2d_b200 import BatchedWorld

    w = BatchedWorld(n, m, S.path_table(), device=device)
    w.set_state(x, y, h, v, type_id=tid)
    w.set_paths(paths)
    w.set_controllers(_rows() if rows is None else rows, cid, path_id=pid)
    w.set_routes(route, threshold=5.0)
    w.set_leader_search(HW, RANGE)
    if yielding:
        w.set_yielding(priority=prio)
    return w


def _kinds(cid):
    from tactics2d_b200.controller.controller_base import CTRL_CRUISE, CTRL_IDM

    return np.select([cid == 0, cid == 1], [CTRL_IDM, CTRL_CRUISE], -1)


def _oracle(paths, prio, x, y, v, tid, cid, pid, route, path_now=None):
    return Y.find(x, y, v, tid, [0], _kinds(cid), pid if path_now is None else path_now, paths, conflict_zones(paths),
                  prio, HW, RANGE, route_id=route)


def _find_into_sentinels(w, n, m):
    """t2d_find_yields into sentinel-filled buffers with a guard tail; returns the written [N, M] part."""
    import torch

    nm, tail = n * m, 67
    yt = torch.full((nm + tail,), SENT_I, dtype=torch.int16, device=w.device)
    sg = torch.full((nm + tail,), SENT_F, dtype=torch.float32, device=w.device)
    stream = C.c_void_p(torch.cuda.current_stream(w.device).cuda_stream)
    from tactics2d_b200 import _lib

    _lib.check(w.lib.t2d_find_yields(w._ctx, C.c_void_p(yt.data_ptr()), C.c_void_p(sg.data_ptr()), stream))
    yt, sg = yt.cpu().numpy(), sg.cpu().numpy()
    assert (yt[nm:] == SENT_I).all() and (sg[nm:] == SENT_F).all(), "the guard tail was written"
    assert not (yt[:nm] == SENT_I).any() and not (sg[:nm] == SENT_F).any(), "a slot was not written"
    return yt[:nm].reshape(n, m), sg[:nm].reshape(n, m)


def _check(yt, sg, ref, min_robust=0.97):
    r = ref["robust"]
    assert r.mean() >= min_robust, r.mean()
    assert np.array_equal(yt[r], ref["yield_to"][r]), np.argwhere((yt != ref["yield_to"]) & r)[:5]
    assert np.array_equal(sg[r], ref["stop_gap"][r].astype(np.float32))
    assert (yt[~ref["yielder"]] == -1).all() and np.isinf(sg[~ref["yielder"]]).all()


@pytest.mark.parametrize("name", sorted(SCENES))
@pytest.mark.parametrize("n,m", [(4099, 1), (257, 33), (131, 64), (67, 97), (35, 128)])
def test_find_yields_matches_the_oracle(cuda_device, name, n, m):
    st = _state(SCENES[name], n, m, seed=m + 7 * n)
    w = _world(cuda_device, n, m, *st)
    yt, sg = _find_into_sentinels(w, n, m)
    paths, prio, x, y, h, v, tid, cid, pid, route = st
    ref = _oracle(paths, prio, x, y, v, tid, cid, pid, route)
    _check(yt, sg, ref)
    if m >= 33:   # the scene makes real decisions: yields and routes partners both present
        assert (ref["yield_to"] >= 0).sum() >= 5


def test_lane_change_slots_yield_on_their_lane(cuda_device):
    """With a lane change bound, K19 reads lane_path (here a copy of path_id: no neighbours), like K17."""
    import torch

    n, m = 67, 64
    paths, prio, x, y, h, v, tid, cid, pid, route = _state(S.intersection, n, m, seed=3)
    w = _world(cuda_device, n, m, paths, prio, x, y, h, v, tid, cid, pid, route, yielding=False)
    none = np.full(len(paths), -1)
    w.set_lane_change(none, none)
    w.set_yielding(priority=prio)
    lane = w.lane_path
    moved = torch.from_numpy(np.where(pid >= 0, (pid.astype(np.int64) + 1) % len(paths), -1).astype(np.int16))
    lane.copy_(moved.to(lane.device))
    yt, sg = _find_into_sentinels(w, n, m)
    _check(yt, sg, _oracle(paths, prio, x, y, v, tid, cid, pid, route, path_now=moved.numpy()))


@pytest.mark.parametrize("name", sorted(SCENES))
def test_control_takes_the_smaller_law(cuda_device, name):
    """K5's yielding instance: an IDM row with a stop takes min(IDM on its leader, IDM on the stop point at speed 0)."""
    import torch

    n, m = 97, 64
    paths, prio, x, y, h, v, tid, cid, pid, route = _state(SCENES[name], n, m, seed=11)
    w = _world(cuda_device, n, m, paths, prio, x, y, h, v, tid, cid, pid, route)
    act = torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device)
    w.control(act)
    ref = _oracle(paths, prio, x, y, v, tid, cid, pid, route)
    yt, sg = w.yield_to.cpu().numpy(), w.stop_gap.cpu().numpy()
    _check(yt, sg, ref)
    lead = w.leader.cpu().numpy()
    got = act.cpu().numpy()[..., 0]
    row = _dicts(_rows())[0]
    xd, yd, vd = (a.astype(np.float64) for a in (x, y, v))
    checked = 0
    for i, k in zip(*np.nonzero(ref["robust"] & (cid == 0) & (tid == 0))):
        li = int(lead[i, k])
        has = li >= 0
        lj = li if has else k
        stop = (ref["stop_x"][i, k], ref["stop_y"][i, k]) if ref["yield_to"][i, k] >= 0 else None
        want = Y.idm_with_stop(vd[i, k], xd[i, k], yd[i, k], has, vd[i, lj], xd[i, lj], yd[i, lj], row, stop)
        assert abs(got[i, k] - want) <= 3e-6 * max(1.0, abs(want)), (i, k, got[i, k], want, stop)
        checked += stop is not None
    assert checked >= 20


def _run(w, ticks, act):
    """control + step for ``ticks``; the share of scenarios with a dynamic collision between path-following cars."""
    import torch

    hit = torch.zeros(w.N, dtype=torch.bool, device=w.device)
    for _ in range(ticks):
        w.control(act)
        r = w.step(act)
        hit |= ((r.flags & 1) != 0).any(1)
    return hit.cpu().numpy()


def _passed(w, scene):
    """Every car's arc length on its path is past the end of every zone of that path."""
    z = conflict_zones(scene.paths)
    x, y = w.x.cpu().numpy(), w.y.cpu().numpy()
    paths = [np.asarray(p, np.float64) for p in scene.paths]
    end = [z.s_out_p[z.zone_off[p]:z.zone_off[p + 1]].max() for p in range(len(paths))]
    from tests import route_oracle as R

    ok = np.ones(scene.shape, bool)
    for i, k in zip(*np.nonzero(scene.path_id >= 0)):
        p = int(scene.path_id[i, k])
        ok[i, k] = R.closest(paths[p], x[i, k], y[i, k])[5] > end[p]
    return ok


def _closed_loop(device, scene, ticks, yielding):
    import torch

    from tactics2d_b200 import BatchedWorld

    n, m = scene.shape
    w = BatchedWorld(n, m, scene.table, device=device, interval=100)
    w.set_state(scene.x, scene.y, scene.heading, scene.speed, type_id=scene.type_id)
    w.set_paths(scene.paths)
    w.set_controllers([S.path_controller()], scene.ctrl_id, path_id=scene.path_id)
    w.set_leader_search(HW, RANGE)
    if yielding:
        w.set_yielding(priority=scene.priority)
    act = torch.zeros((n, m, 2), dtype=torch.float32, device=device)
    return w, _run(w, ticks, act)


# without yielding, 91.7 % of the intersection's scenarios and all of the roundabout's have a collision (H100, these seeds)
@pytest.mark.parametrize("name,m,ticks,min_crash", [("intersection", 8, 450, 0.85), ("roundabout", 11, 450, 0.95)])
def test_closed_loop_yields_without_collision_or_deadlock(cuda_device, name, m, ticks, min_crash):
    """1024 scenarios for 45 s: with yielding no dynamic collision and every car past every zone of its path (no deadlock);
    the same scenes without yielding collide in at least ``min_crash`` of the scenarios, so they discriminate."""
    scene = SCENES[name](1024, m, seed=5)
    _, crash_free = _closed_loop(cuda_device, scene, ticks, yielding=False)
    w, crash = _closed_loop(cuda_device, scene, ticks, yielding=True)
    passed = _passed(w, scene)
    print(f"{name}: collisions without yielding in {crash_free.mean():.3f} of 1024 scenarios, with yielding in "
          f"{crash.mean():.3f}; cars past their zones {passed[scene.path_id >= 0].mean():.4f}")
    assert crash_free.mean() >= min_crash, "the scene must make crossing cars meet when nobody yields"
    assert not crash.any(), np.flatnonzero(crash)[:10]
    assert passed[scene.path_id >= 0].all(), np.argwhere(~passed & (scene.path_id >= 0))[:10]


def _reactive_env(device, yielding):
    from tactics2d_b200.envs.batched_env import BatchedTrafficEnv
    from tests import reactive_scenes as RS

    eps, _ = RS.stopped_ego()
    kw = {} if not yielding else dict(yielding=dict(critical_gap=3.0))
    return BatchedTrafficEnv(None, replay=eps, device=device, max_step=400, leaders=dict(half_width=RS.HALF_WIDTH),
                             reactive=dict(controller=RS.controller()), **kw)


def test_highway_reactive_replay_is_unchanged_by_yielding(cuda_device):
    import torch

    plain, yl = _reactive_env(cuda_device, False), _reactive_env(cuda_device, True)
    plain.reset()
    _, info = yl.reset()
    assert (info["yield_to"] == -1).all() and torch.isinf(info["stop_gap"]).all()
    act = torch.zeros((1, 2), dtype=torch.float32, device=cuda_device)
    for _ in range(150):
        plain.step(act)
        _, _, _, _, info = yl.step(act)
        assert (info["yield_to"] == -1).all()
        for k in ("x", "y", "heading", "speed"):
            assert torch.equal(getattr(plain.world, k), getattr(yl.world, k)), k
    assert torch.equal(plain.world.last_accel, yl.world.last_accel)


def test_unbound_control_and_step_are_bit_identical(cuda_device):
    import torch

    n, m = 131, 64
    st = _state(S.intersection, n, m, seed=21)
    rows = [S.path_controller(), _rows()[1]]   # lane keeping: K5's PID instance
    ref = _world(cuda_device, n, m, *st, yielding=False, rows=rows)
    unb = _world(cuda_device, n, m, *st, rows=rows)
    unb.unset_yielding()
    assert unb.yield_to is None
    acts = [torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device) for _ in range(2)]
    for _ in range(30):
        for w, a in zip((ref, unb), acts):
            w.control(a)
            w.step(a)
        assert torch.equal(acts[0], acts[1])
        for k in ("x", "y", "heading", "speed"):
            assert torch.equal(getattr(ref, k), getattr(unb, k)), k
        assert torch.equal(ref.result.flags, unb.result.flags)


def test_host_steps_launch_k19(cuda_device):
    """t2d_step_host_ego runs the same K18 / K17 / K19 / K5 chain as control + step."""
    import torch

    n, m = 64, 16
    scene = S.intersection(n, m, seed=2)
    ws = []
    for _ in range(2):
        w, _ = _closed_loop(cuda_device, scene, 0, yielding=True)
        ws.append(w)
    ego = np.zeros((n, 2), np.float32)
    act = torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device)
    for _ in range(40):
        ws[0].control(act)
        ws[0].step(act)
        ws[1].step_host_ego(ego)
    for k in ("x", "y", "speed"):
        assert torch.equal(getattr(ws[0], k), getattr(ws[1], k)), k
    assert torch.equal(ws[0].yield_to, ws[1].yield_to)
    assert (ws[0].yield_to >= 0).any()


def test_rejections_keep_the_binding(cuda_device):
    import torch

    from tactics2d_b200 import _lib
    from tactics2d_b200._lib import T2DError

    n, m = 8, 8
    st = _state(S.intersection, n, m, seed=1)
    w = _world(cuda_device, n, m, *st)
    lib, ctx = w.lib, w._ctx
    z = conflict_zones(st[0])
    P = len(st[0])
    good_rows = np.zeros(len(z), _lib.ZONE_DTYPE)
    for k in ("q", "s_in_p", "s_out_p", "s_in_q", "s_out_q"):
        good_rows[k] = getattr(z, k)

    out = (w.yield_to, w.stop_gap)   # kept alive past the unbinding below

    def call(p=None, rows=good_rows, off=z.zone_off, yt=None, sg=None):
        off = np.ascontiguousarray(off, np.int32)
        p = _lib.YieldParamsC(3.0, 3.0, 0.5) if p is None else p
        yt = out[0].data_ptr() if yt is None else yt
        sg = out[1].data_ptr() if sg is None else sg
        return lib.t2d_set_yielding(ctx, C.byref(p), C.c_void_p(rows.ctypes.data), C.c_void_p(off.ctypes.data), None,
                                    C.c_void_p(yt), C.c_void_p(sg))

    assert call() == 0
    good = w.find_yields()[0].clone()
    q_out = good_rows.copy(); q_out["q"][0] = P
    q_self = good_rows.copy(); q_self["q"][0] = z.p[0]
    unsorted = good_rows.copy(); unsorted["s_in_p"][0] = unsorted["s_in_p"][1] + 1.0; unsorted["s_out_p"][0] += 100.0
    nan = good_rows.copy(); nan["s_in_q"][0] = np.nan
    for rows in (q_out, q_self, unsorted, nan):
        assert call(rows=rows) == -1
    for p in (_lib.YieldParamsC(0.0, 3.0, 0.5), _lib.YieldParamsC(3.0, -1.0, 0.5), _lib.YieldParamsC(3.0, 3.0, np.nan)):
        assert call(p=p) == -1
    dec = z.zone_off.copy(); dec[1] = dec[2] + 1
    assert call(off=dec) == -1
    assert call(yt=out[0].data_ptr() + 1) == -1
    assert call(sg=out[1].data_ptr() + 2) == -1
    # the previous binding is whole: control still yields as before
    assert torch.equal(w.find_yields()[0], good)
    w.set_leader_search(None)   # drops it
    assert w.yield_to is None
    with pytest.raises(T2DError):
        w.find_yields()
    assert call() == -4   # no search: T2D_E_STATE
    w.set_leader_search(HW, RANGE)
    w.set_yielding()
    w.set_paths(st[0])
    assert w.yield_to is None
    with pytest.raises(T2DError):
        w.find_yields()
    from tactics2d_b200 import BatchedWorld

    bare = BatchedWorld(n, m, S.path_table(), device=cuda_device)
    bare.set_paths(st[0])
    with pytest.raises(T2DError, match="controllers not set"):
        bare.set_yielding()


def test_env_info_and_auto_reset(cuda_device):
    """info carries the yields of the state after the auto-reset; a setter that drops the binding is followed by a
    new one at the next reset; yielding needs leaders."""
    import torch

    from tactics2d_b200.envs.batched_env import BatchedTrafficEnv

    with pytest.raises(ValueError):
        BatchedTrafficEnv(None, replay=None, yielding=dict(), device=cuda_device)
    env = _reactive_env_crossing(cuda_device)
    obs, info = env.reset()
    w = env.world
    assert info["yield_to"].shape == (1, w.M) and info["stop_gap"].dtype == torch.float32
    act = torch.zeros((1, 2), dtype=torch.float32, device=cuda_device)
    seen, reset_seen = 0, False
    for _ in range(300):
        obs, r, term, trunc, info = env.step(act)
        yt, sg = w.find_yields()
        assert torch.equal(info["yield_to"], yt) and torch.equal(info["stop_gap"], sg)
        seen += int((info["yield_to"] >= 0).sum())
        reset_seen |= bool(trunc[0] | term[0])
    assert seen > 0 and reset_seen
    w.set_controllers([S.path_controller()], np.zeros((1, w.M), np.uint8))   # drops the yielding
    assert w.yield_to is None
    env.reset()
    assert w.yield_to is not None


def _reactive_env_crossing(device):
    """Reactive replay of the two-stream crossing log, the ego parked far off, with yielding."""
    from tactics2d_b200.dataset_parser.replay import build_replay_episodes
    from tactics2d_b200.envs.batched_env import BatchedTrafficEnv
    from tests import reactive_scenes as RS

    log = S.crossing_log(duration_ms=60000, seed=3)
    log, ego = RS._with_parked(log, -300.0, -300.0)
    eps = build_replay_episodes(log, 16, [2000], [ego], RS.table(), horizon_ms=25000, reuse_slots=True)
    return BatchedTrafficEnv(None, replay=eps, device=device, max_step=250, leaders=dict(half_width=HW),
                             reactive=dict(controller=S.path_controller()), yielding=dict(critical_gap=3.0))
