"""Reactive replay on the device (``t2d_set_log_reactive``: K7's reactive instance and K5's per-slot desired speed)
against tests/reactive_replay_oracle.py: the handover at resets and in ticks bit for bit with every output starting as a
sentinel, row_track and slot schedules at several M, the closed loop of tests/reactive_scenes.py, the host step entries,
graph replay, the env, the rejections and drops, and plain replay unchanged with nothing bound."""

import ctypes as C

import numpy as np
import pytest

from oracle import scenario as O
from tests import reactive_replay_oracle as RO
from tests import reactive_scenes as RS

pytestmark = pytest.mark.gpu

KEYS = ("x", "y", "heading", "speed", "vx", "vy")


def _episodes(kind, m, seed=0):
    from tactics2d_b200 import synthetic
    from tactics2d_b200.dataset_parser.replay import build_replay_episodes

    if kind == "schedule":   # slots reused mid-episode, 40 ms records sampled every 100 ms
        log = synthetic.highway_log(60000, seed, rate_per_s=3.0, length_m=300.0, period_ms=40)
        rng = np.random.default_rng(seed)
        ego = rng.choice(np.nonzero(log.first_ms < 20000)[0], 3)
        t0 = log.first_ms[ego] + 40 * rng.integers(0, 5, 3)
        return build_replay_episodes(log, m, t0.tolist(), log.ids[ego].tolist(), RS.table(), horizon_ms=20000,
                                     reuse_slots=True)
    return synthetic.replay_episodes(3, m, 3 * m, seed=seed, table=RS.table(), duration_ms=8000, max_frames=80)


def _drive_rows(eps):
    rows = eps.table.rows
    return np.array([next(i for i, q in enumerate(rows) if q.model != 4 and q.name == rows[r].name
                          and q.half_len == rows[r].half_len and q.half_wid == rows[r].half_wid)
                     for r in eps.log.type_row], np.uint8)


def _world(device, eps, reactive=True):
    import torch

    from tactics2d_b200 import BatchedWorld

    P, M = eps.type_id.shape
    w = BatchedWorld(P, M, eps.table, device=device)
    w.set_log(eps.log, eps.t0, **eps.binding())
    paths, tp, ds = eps.log.track_paths()
    w.set_paths(paths)
    ctrl = np.zeros((P, M), np.uint8)
    ctrl[:, 0] = 255
    w.set_controllers([RS.controller()], ctrl)
    w.set_leader_search(RS.HALF_WIDTH, RS.MAX_RANGE)
    if reactive:
        w.set_reactive_replay(tp, desired_speed=ds)
    pool = {k: torch.from_numpy(np.ascontiguousarray(eps.pool[k], np.float32)).to(device) for k in KEYS}
    return w, pool, (paths, tp, ds)


def _snapshot(w):
    s = {k: getattr(w, k).cpu().numpy() for k in KEYS}
    s["type_id"] = w.type_id.cpu().numpy()
    s["drive_path"] = w.drive_path.cpu().numpy()
    s["slot_desired_speed"] = w.slot_desired_speed.cpu().numpy()
    s["pid_state"] = w._ctrl["pid_state"].cpu().numpy().reshape(w.N, w.M, 6)
    s["last_accel"] = w.last_accel.cpu().numpy()
    return s


def _sentinels(w):
    for k in KEYS:
        getattr(w, k).fill_(7.0)
    w.type_id.fill_(200)
    w.drive_path.fill_(99)
    w.slot_desired_speed.fill_(3.0)
    w._ctrl["pid_state"].fill_(5.0)
    w.last_accel.fill_(2.0)


def _reset_all(w, eps, pool):
    import torch

    P = eps.type_id.shape[0]
    w.type_id.copy_(torch.from_numpy(eps.type_id).to(w.device))
    w.reset(torch.ones(P, dtype=torch.uint8, device=w.device), pool)


def _same(got, want, keys, exact=True):
    for k in keys:
        if exact:
            assert np.array_equal(got[k], want[k], equal_nan=True), k
        else:
            err = np.abs(got[k].astype(np.float64) - want[k]) / np.maximum(np.abs(want[k]), 1.0)
            assert err.max() <= 1e-5, (k, err.max())


@pytest.mark.parametrize("kind", ["row_track", "schedule"])
@pytest.mark.parametrize("m", [1, 2, 33, 64, 97, 128])
def test_k7_reactive_matches_oracle(cuda_device, kind, m):
    """K7 in reset mode over sentinels, then in tick mode (the ticks' K1 moves only the simulated slots, which the oracle
    keeps at their previous state, so every slot K1 leaves alone is compared bit for bit)."""
    import torch

    eps = _episodes(kind, m, seed=m)
    w, pool, (paths, tp, ds) = _world(cuda_device, eps)
    dr = _drive_rows(eps)
    bind = dict(row_track=eps.row_track, schedule=eps.schedule)
    P = eps.type_id.shape[0]
    _sentinels(w)
    before = _snapshot(w)
    w.type_id.copy_(torch.from_numpy(eps.type_id).to(cuda_device))
    before["type_id"] = eps.type_id.copy()
    w.reset(torch.tensor([1, 0, 1], dtype=torch.uint8, device=cuda_device)[:P], pool)
    torch.cuda.synchronize()
    # K2 rewrote the masked scenarios from the pool (and zeroed their controller memory): the oracle's K7 starts there
    got = _snapshot(w)
    mask = np.array([1, 0, 1], bool)[:P]
    start = {k: np.where(mask[:, None], np.asarray(eps.pool[k], np.float32), before[k]) for k in KEYS}
    start.update(type_id=before["type_id"], drive_path=before["drive_path"], slot_desired_speed=before["slot_desired_speed"],
                 pid_state=np.where(mask[:, None, None], 0.0, before["pid_state"]),
                 last_accel=np.where(mask[:, None], np.float32(0.0), before["last_accel"]))
    want = RO.apply(start, eps.log, eps.t0, np.arange(P), np.zeros(P, np.int64), 100, tp, dr, ds, 0, mask, **bind)
    _same(got, want, KEYS + ("type_id", "drive_path", "slot_desired_speed", "pid_state", "last_accel"))
    assert (got["drive_path"][~mask] == 99).all() and (got["slot_desired_speed"][~mask] == 3.0).all()
    _reset_all(w, eps, pool)
    act = torch.zeros((P, m, 2), dtype=torch.float32, device=cuda_device)
    for t in range(12):
        prev = _snapshot(w)
        w.step(act)                                         # no control: K1 gets zero actions
        torch.cuda.synchronize()
        got = _snapshot(w)
        want = RO.apply(prev, eps.log, eps.t0, np.arange(P), np.full(P, t, np.int64), 100, tp, dr, ds, 1, **bind)
        _same(got, want, ("type_id", "drive_path", "slot_desired_speed", "pid_state", "last_accel"))
        moved = want["simulated"].copy()
        moved[:, 0] = True                                  # the ego (never replayed) is integrated as well
        for k in KEYS:
            assert np.array_equal(got[k][~moved], want[k][~moved]), (t, k)
        st = O.physics_tick(want, want["type_id"], np.zeros((P, m, 2), np.float32), eps.table.as_oracle_table())
        _same({k: got[k][moved] for k in ("x", "y", "speed")}, {k: st[k][moved] for k in ("x", "y", "speed")},
              ("x", "y", "speed"), exact=False)


def _closed_loop(cuda_device, scene, reactive, ticks, host=None):
    import torch

    eps = scene[0]
    w, pool, (paths, tp, ds) = _world(cuda_device, eps, reactive)
    if not reactive:
        w.set_controllers(None, None)
    if host == "agents":
        w.set_agents(torch.zeros((eps.type_id.shape[0], 1), dtype=torch.int16, device=cuda_device))
    _reset_all(w, eps, pool)
    P, M = eps.type_id.shape
    act = torch.zeros((P, M, 2), dtype=torch.float32, device=cuda_device)
    ego = np.zeros((P, 2), np.float32)
    w.set_ego_action(torch.zeros((P, 2), dtype=torch.float32, device=cuda_device))
    states, flags = [], []
    for _ in range(ticks):
        if host == "ego":
            w.step_host_ego(ego, act)
        elif host == "agents":
            w.step_host_agents(ego[:, None, :], act)
        else:
            if reactive:
                w.control(act)
            r = w.step(act)
        torch.cuda.synchronize()
        states.append({k: getattr(w, k).cpu().numpy() for k in ("x", "y", "heading", "speed")})
        states[-1]["type_id"] = w.type_id.cpu().numpy()
        flags.append(w.result.flags.cpu().numpy() if host is None else None)
    return w, states, flags


def test_closed_loop_matches_oracle_and_stops_behind_the_ego(cuda_device):
    eps, ego_x = scene = RS.stopped_ego()
    ticks = 120
    w, states, flags = _closed_loop(cuda_device, scene, True, ticks)
    paths, tp, ds = eps.log.track_paths()
    ref = RO.rollout(eps, eps.table, RS.ctab(), paths, tp, _drive_rows(eps), ds, ticks, RS.HALF_WIDTH, RS.MAX_RANGE)
    tab = eps.table.as_oracle_table()
    for t in range(ticks):
        assert np.array_equal(states[t]["type_id"], ref["type_id"][t]), t
        _same(states[t], ref["states"][t], ("x", "y", "heading", "speed"), exact=False)
        fl = O.events(states[t]["x"], states[t]["y"], states[t]["heading"], states[t]["type_id"], tab)[0]
        assert np.array_equal(fl, flags[t]), t
    assert not any((f & O.F_DYNAMIC).any() for f in flags)
    _, plain, pflags = _closed_loop(cuda_device, scene, False, 300)
    assert any((f[:, 0] & O.F_DYNAMIC).any() for f in pflags)


def test_host_step_entries_equal_the_device_sequence(cuda_device):
    scene = RS.stopped_ego()
    _, dev, _ = _closed_loop(cuda_device, scene, True, 30)
    for host, ticks in (("ego", 30), ("agents", 1)):   # K10 may retire the agent slot after its first step
        _, got, _ = _closed_loop(cuda_device, scene, True, ticks, host)
        for a, b in zip(dev, got):
            for k in a:
                assert np.array_equal(a[k], b[k]), (host, k)


def test_graph_replay_of_control_and_step(cuda_device):
    import torch

    scene = RS.stopped_ego()
    eps = scene[0]
    w1, pool1, _ = _world(cuda_device, eps)
    w2, pool2, _ = _world(cuda_device, eps)
    _reset_all(w1, eps, pool1)
    _reset_all(w2, eps, pool2)
    P, M = eps.type_id.shape
    a1 = torch.zeros((P, M, 2), dtype=torch.float32, device=cuda_device)
    a2 = a1.clone()
    w2.control(a2)   # warm both paths
    w2.step(a2)
    w1.control(a1)
    w1.step(a1)
    torch.cuda.synchronize()
    s = torch.cuda.Stream(cuda_device)
    s.wait_stream(torch.cuda.current_stream(cuda_device))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            w2.control(a2)
            w2.step(a2)
    torch.cuda.current_stream(cuda_device).wait_stream(s)
    for t in range(20):
        w1.control(a1)
        w1.step(a1)
        g.replay()
        torch.cuda.synchronize()
        for k in ("x", "y", "heading", "speed", "type_id", "drive_path", "slot_desired_speed"):
            assert torch.equal(getattr(w1, k), getattr(w2, k)), (t, k)


def test_env_binds_at_reset_and_hands_over_on_auto_reset(cuda_device):
    import torch

    from tactics2d_b200.envs.batched_env import BatchedTrafficEnv

    eps, _ = RS.stopped_ego()
    env = BatchedTrafficEnv(None, replay=eps, device=cuda_device, max_step=40, leaders=dict(half_width=RS.HALF_WIDTH),
                            reactive=dict(controller=RS.controller()))
    obs, info = env.reset()
    w = env.world
    assert info["reactive"].any() and torch.equal(info["reactive"], w.drive_path >= 0)
    act = torch.zeros((1, 2), dtype=torch.float32, device=cuda_device)
    start = w.x.clone()
    for t in range(45):
        obs, r, term, trunc, info = env.step(act)
        if bool(trunc[0]):   # the auto-reset hands the present tracks over again, from the log at t0
            assert torch.equal(w.x, start) and torch.equal(info["reactive"], w.drive_path >= 0)
            assert (w.slot_desired_speed[w.drive_path >= 0] > 0).all()
            break
    else:
        pytest.fail("no truncation")
    w.set_controllers([RS.controller()], np.zeros((1, w.M), np.uint8))   # drops the binding; the next reset binds again
    assert w.drive_path is None
    env.reset()
    assert w.drive_path is not None


def test_nothing_bound_is_plain_replay(cuda_device):
    import torch

    for kind in ("row_track", "schedule"):
        eps = _episodes(kind, 33, seed=3)
        w1, p1, (paths, tp, ds) = _world(cuda_device, eps, reactive=False)
        w2, p2, _ = _world(cuda_device, eps, reactive=True)
        w2.set_reactive_replay(None)
        _reset_all(w1, eps, p1)
        _reset_all(w2, eps, p2)
        P, M = eps.type_id.shape
        a1 = torch.zeros((P, M, 2), dtype=torch.float32, device=cuda_device)
        a2 = a1.clone()
        for _ in range(10):
            w1.control(a1)
            w1.step(a1)
            w2.control(a2)
            w2.step(a2)
        torch.cuda.synchronize()
        for k in KEYS + ("type_id",):
            assert torch.equal(getattr(w1, k), getattr(w2, k)), k
        assert torch.equal(a1, a2)


def test_rejections_keep_the_binding_and_rebinds_drop_it(cuda_device):
    import torch

    from tactics2d_b200 import _lib

    eps = _episodes("row_track", 8, seed=1)
    w, pool, (paths, tp, ds) = _world(cuda_device, eps)
    K = len(eps.log)
    dr = _drive_rows(eps)
    lib, ctx = w.lib, w._ctx
    dp0 = w.drive_path
    buf = torch.zeros(w.N * w.M * 2 + 2, dtype=torch.float32, device=cuda_device)
    ok16, ok32 = C.c_void_p(buf.data_ptr()), C.c_void_p(buf.data_ptr() + 4 * (w.N * w.M + 1))
    keep = []

    def call(track_path=tp, drive_row=dr, speed=ds, n=K, drive_path=ok16, sds=ok32):
        a = [np.ascontiguousarray(track_path, np.int16), np.ascontiguousarray(drive_row, np.uint8),
             np.ascontiguousarray(speed, np.float32)]
        keep.append(a)
        c = _lib.ReactiveReplayC(n, C.c_void_p(a[0].ctypes.data), C.c_void_p(a[1].ctypes.data),
                                 C.c_void_p(a[2].ctypes.data), drive_path, sds)
        return lib.t2d_set_log_reactive(ctx, C.byref(c))

    INVALID, STATE = -1, -4
    r = tp.copy()
    r[0] = len(paths)
    assert call(track_path=r) == INVALID
    r[0] = -2
    assert call(track_path=r) == INVALID
    k = int(np.nonzero(tp >= 0)[0][0])
    for row in (eps.log.type_row[k], len(eps.table)):                   # static, outside the table
        d = dr.copy()
        d[k] = row
        assert call(drive_row=d) == INVALID
    other = next(i for i, q in enumerate(eps.table.rows) if q.model != 4 and q.half_len != eps.table.rows[dr[k]].half_len)
    d = dr.copy()
    d[k] = other
    assert call(drive_row=d) == INVALID                                 # another shape's extents
    for v in (0.0, -1.0, np.nan, np.inf):
        s = ds.copy()
        s[k] = v
        assert call(speed=s) == INVALID
    assert call(n=K + 1) == INVALID
    assert call(drive_path=C.c_void_p(buf.data_ptr() + 1)) == INVALID
    assert call(sds=C.c_void_p(buf.data_ptr() + 2)) == INVALID
    assert call(drive_path=None) == INVALID
    assert w.drive_path is dp0
    _sentinels(w)
    _reset_all(w, eps, pool)
    assert not (w.drive_path == 99).any()                               # the kept binding ran
    for drop in (lambda: w.set_paths(w.paths), lambda: w.set_controllers([RS.controller()], np.zeros((w.N, w.M), np.uint8)),
                 lambda: w.set_type_table(w.type_table), lambda: w.set_leader_search(None),
                 lambda: w.set_log(eps.log, eps.t0, **eps.binding())):
        w.set_leader_search(RS.HALF_WIDTH, RS.MAX_RANGE)
        w.set_reactive_replay(tp, desired_speed=ds)
        drop()
        assert w.drive_path is None
    w.set_leader_search(None)
    assert call() == STATE                                              # no search
    w.set_leader_search(RS.HALF_WIDTH, RS.MAX_RANGE)
    w.set_controllers([RS.controller()], np.zeros((w.N, w.M), np.uint8), path_id=np.full((w.N, w.M), -1, np.int16))
    w.set_lane_change([-1] * len(paths), [-1] * len(paths))
    assert call() == STATE                                              # a lane change bound
    w.set_lane_change(None)
    w.set_reactive_replay(tp, desired_speed=ds)
    with pytest.raises(_lib.T2DError):
        w.set_lane_change([-1] * len(paths), [-1] * len(paths))
    w.set_paths([])
    assert call() == STATE                                              # no paths
    w.set_paths(paths)
    w.set_controllers(None, None)
    assert call() == STATE                                              # no controllers
    w.set_controllers([RS.controller()], np.zeros((w.N, w.M), np.uint8))
    w.set_log(None)
    assert call() == STATE                                              # no log
