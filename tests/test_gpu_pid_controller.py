"""PID controller rows of t2d_control (T2D_CTRL_PID) on the device: the reference's sequences, the PIDController facade,
control -> step rollouts against the float64 restatement, reset / retirement of the per-slot state, the host-step path,
the rejections, and the sign of the path-derived error in closed loop."""

import numpy as np
import pytest

from . import pid_oracle as OC
from .pid_cases import CONFIGS, quirk, row_c, sequence

pytestmark = pytest.mark.gpu


def _ulp_close(got, want, n_ulp=2):
    want32 = np.asarray(want, np.float64)
    tol = n_ulp * np.spacing(np.abs(want32).astype(np.float32)).astype(np.float64)
    assert np.all(np.abs(np.asarray(got, np.float64) - want32) <= tol), (got, want)


def test_golden_sequences_through_t2d_control(cuda_device):
    """Every reference sequence in its own scenario of one batch: the fp64 state after every step within 1e-12, the
    outputs within 2 fp32 ulp (wheel_base and the accel limits are fp32 in the row)."""
    import torch

    from tactics2d_b200 import BatchedWorld
    from tactics2d_b200.types import TypeParams, TypeTable

    n = len(CONFIGS)
    w = BatchedWorld(n, 1, TypeTable([TypeParams()]), device=cuda_device, steer_first=True)
    seqs = [sequence(c) for c in CONFIGS]
    T = len(seqs[0][0])
    target = torch.zeros((n, 1, 2), dtype=torch.float32, device=cuda_device)
    w.set_controllers([row_c(c) for c in CONFIGS], ctrl_id=np.arange(n, dtype=np.uint8).reshape(n, 1), pid_target=target)
    assert w.pid_target.data_ptr() == target.data_ptr() and w.pid_state.dtype == torch.float64
    for t in range(T):
        inp = np.stack([s[0][t] for s in seqs])
        w.set_state(inp[:, None, 0], inp[:, None, 1], inp[:, None, 2], inp[:, None, 3], type_id=np.zeros((n, 1), np.uint8))
        target.copy_(torch.from_numpy(inp[:, None, 4:6].astype(np.float32)))
        act = w.control(torch.zeros((n, 1, 2), dtype=torch.float32, device=cuda_device)).cpu().numpy()[:, 0]
        state = w.pid_state.cpu().numpy()[:, 0]
        for k, (cfg, (_, out, st)) in enumerate(zip(CONFIGS, seqs)):
            np.testing.assert_allclose(state[k], st[t], rtol=1e-12, atol=1e-12, err_msg=f"{cfg['name']} step {t}")
            _ulp_close(act[k, 1], out[t, 1])
            if not quirk(cfg):
                _ulp_close(act[k, 0], out[t, 0])


def test_facade_matches_reference_sequences(cuda_device):
    """PIDController.step / reset / _lat_integral: the reference's step, mode and reset tests, and its sequences."""
    from tactics2d_b200.controller import PIDController
    from tactics2d_b200.participant.trajectory import State

    ego = State(frame=0, x=0, y=0, heading=0, speed=5.0)
    c = PIDController(control_mode="combined")
    s, a = c.step(ego, target_heading=0.1, target_speed=10.0)
    assert -c.max_steering <= s <= c.max_steering and c.min_accel <= a <= c.max_accel
    s, a = c.step(ego, cross_track_error=0.5, target_speed=10.0, wheel_base=2.5)
    assert -c.max_steering <= s <= c.max_steering and c.min_accel <= a <= c.max_accel
    s, a = PIDController(control_mode="lateral").step(ego, target_heading=0.2)
    assert a == 0.0 and abs(s) <= 0.5
    s, a = PIDController(control_mode="longitudinal").step(ego, target_speed=10.0)
    assert s == 0.0 and -5.0 <= a <= 3.0
    for _ in range(5):
        c.step(ego, target_heading=0.1, target_speed=10.0)
    assert c._lat_integral != 0.0 and c._lon_prev_error == 5.0
    c.reset()
    assert (c._lat_integral, c._lat_prev_error, c._lat_prev_derivative, c._lon_integral, c._lon_prev_error,
            c._lon_prev_derivative) == (0.0,) * 6
    with pytest.raises(ValueError, match="Lateral control requires"):
        PIDController(control_mode="lateral").step(ego)
    with pytest.raises(TypeError, match="target_speed must be numeric"):
        PIDController(control_mode="longitudinal").step(ego, target_speed="fast")
    lat = PIDController(control_mode="lateral")
    with pytest.raises(ValueError, match="wheel_base must be positive"):
        lat.step(ego, cross_track_error=0.5, wheel_base=0.0)
    assert lat._lat_prev_error == 0.5                   # the state advanced before the reference raised
    for cfg in CONFIGS:
        inp, out, st = sequence(cfg)
        kw = {k: cfg[k] for k in ("dt", "kp_lat", "ki_lat", "kd_lat", "max_steering", "kp_lon", "ki_lon", "kd_lon",
                                  "max_accel", "min_accel", "derivative_filter_alpha", "control_mode")}
        c = PIDController(**kw)
        for t in range(len(inp)):
            x, y, h, v, ts, lt = (float(q) for q in inp[t])
            kwargs = {}
            if cfg["lateral"] == "heading":
                kwargs["target_heading"] = lt
            elif cfg["lateral"] == "cross":
                kwargs["cross_track_error"] = lt
            if cfg["wheel_base"] is not None:
                kwargs["wheel_base"] = cfg["wheel_base"]
            if cfg["target_speed"]:
                kwargs["target_speed"] = ts
            s, a = c.step(State(frame=0, x=x, y=y, heading=h, speed=v), **kwargs)
            got = [c._lat_integral, c._lat_prev_error, c._lat_prev_derivative, c._lon_integral, c._lon_prev_error,
                   c._lon_prev_derivative]
            np.testing.assert_allclose(got, st[t], rtol=1e-12, atol=1e-12, err_msg=f"{cfg['name']} step {t}")
            _ulp_close(s, out[t, 0])
            _ulp_close(a, out[t, 1])
    # a heading error with a cross-track keyword as well takes the cross-track scaling (pid_controller.py:355-362)
    c = PIDController()
    s, _ = c.step(ego, target_heading=0.0625, cross_track_error=9.0, wheel_base=4.0)
    _, _, want = OC.pid_step(dict(OC.PID_DEFAULTS, pid_lateral=OC.PID_LAT_HEADING, pid_longitudinal=0), 0, 0, 0, 5, 0,
                             0.0625, np.zeros(6))
    assert s == pytest.approx((1.5 * want[1] + 0.5 * want[2] + 0.2 * want[0]) * (2.0 / 4.0), rel=1e-12)


SHAPES = [(48, 32), (9, 100), (5, 3), (33, 128), (7, 1)]


def _pid_rows():
    from tactics2d_b200.controller import IDMController, PIDController, PurePursuitController, AccelerationController

    rows = [IDMController(), AccelerationController(target_speed=9.0), PurePursuitController(min_pre_aiming_distance=5.0)]
    for lat_err, mode in (("target_heading", "combined"), ("cross_track_error", "combined"), ("path_heading", "lateral"),
                          ("path_cross_track", "combined"), ("path_cross_track", "longitudinal")):
        c = PIDController(control_mode=mode, lateral_error=lat_err, dt=0.1, kp_lat=0.9, ki_lat=0.3, kd_lat=0.4)
        rows.append(c)
    rows[-2].update_driving_style(0.4)
    return [r.params() for r in rows]


def _rollout_world(cuda_device, n, m, seed):
    from tactics2d_b200 import BatchedWorld, synthetic

    scene = synthetic.with_inactive(synthetic.config4(n, m, seed=seed), 0.15, seed=seed + 1) if m > 3 else synthetic.config4(n, m, seed=seed)
    w = BatchedWorld(n, m, scene.table, device=cuda_device, steer_first=bool(seed % 2))
    w.set_map(scene.segments, scene.bounds)
    w.set_state(scene.x, scene.y, scene.heading, scene.speed, vx=scene.vx, vy=scene.vy, type_id=scene.type_id)
    paths = [np.array([[0, 0], [50, 10], [50, 10], [120, 10]], np.float32),
             np.array([[10, -40], [10, 90], [-60, 160]], np.float32),
             np.array([[5, 5], [5, 5]], np.float32)]                           # only a zero-length segment
    w.set_paths(paths)
    return w, scene, paths


@pytest.mark.parametrize("n,m", SHAPES)
def test_control_then_step_rollout_matches_restatement(cuda_device, n, m):
    import torch

    from tactics2d_b200 import synthetic

    w, scene, paths = _rollout_world(cuda_device, n, m, seed=n + m)
    rng = np.random.default_rng(n * 1000 + m)
    rows = _pid_rows()
    ctrl_id = rng.choice([255, 0, 1, 2, 3, 4, 5, 6, 7], size=(n, m)).astype(np.uint8)
    lead = rng.integers(-1, m, size=(n, m)).astype(np.int16)
    pid = rng.integers(-1, len(paths) + 1, size=(n, m)).astype(np.int16)    # -1 and one past the end included
    target = np.stack([rng.uniform(0, 15, (n, m)), rng.uniform(-4, 4, (n, m))], 2).astype(np.float32)
    w.set_controllers(rows, ctrl_id, lead, pid, pid_target=target)
    sentinel = rng.uniform(-3, 3, (n, m, 6))
    w.pid_state.copy_(torch.from_numpy(sentinel))
    table = scene.table.as_oracle_table()
    ctab = [{k: getattr(r, k) for k, _ in r._fields_} for r in rows]
    la = np.zeros((n, m), np.float32)
    st = sentinel.copy()
    is_pid = (ctrl_id >= 3) & (ctrl_id != 255)
    controlled = (ctrl_id != 255) & (scene.type_id != 255)
    for t in range(6):
        ext = synthetic.random_actions(700 + t, (n, m))
        before = w.state_numpy()
        want_act, want_la, want_st = OC.control_tick(before, scene.type_id, table, ext, ctrl_id, ctab, lead, pid,
                                                     [p.astype(np.float64) for p in paths], la, bool(w.flags_cfg & 2),
                                                     pid_target=target, pid_state=st)
        act = w.control(torch.from_numpy(ext).to(cuda_device)).cpu().numpy()
        got_st = w.pid_state.cpu().numpy()
        assert np.array_equal(act[~controlled], ext[~controlled])
        np.testing.assert_allclose(act[controlled], want_act[controlled], rtol=3e-6, atol=3e-6)
        got_la = w.last_accel.cpu().numpy()
        np.testing.assert_allclose(got_la, want_la, rtol=3e-6, atol=3e-6)
        np.testing.assert_allclose(got_st, want_st, rtol=1e-12, atol=1e-12)
        assert np.array_equal(got_st[~(is_pid & (scene.type_id != 255))], sentinel[~(is_pid & (scene.type_id != 255))])
        la, st = got_la, got_st
        w.step(torch.from_numpy(act).to(cuda_device))
    assert (is_pid & (scene.type_id != 255)).sum() > 0


def test_masked_reset_zeroes_exactly_the_reset_scenarios(cuda_device):
    import torch

    n, m = 12, 40
    w, scene, paths = _rollout_world(cuda_device, n, m, seed=3)
    ctrl_id = np.full((n, m), 5, np.uint8)
    w.set_controllers(_pid_rows(), ctrl_id, pid_target=np.ones((n, m, 2), np.float32))
    w.pid_state.fill_(2.5)
    mask = torch.zeros(n, dtype=torch.uint8, device=cuda_device)
    mask[[1, 4, 11]] = 1
    pool = {k: torch.from_numpy(np.asarray(getattr(scene, k), np.float32)).to(cuda_device) for k in ("x", "y", "heading", "speed")}
    w.reset(mask, pool)
    st = w.pid_state.cpu().numpy()
    reset = mask.cpu().numpy().astype(bool)
    assert np.all(st[reset] == 0.0) and np.all(st[~reset] == 2.5)


def test_host_step_equals_device_path(cuda_device):
    import torch

    n, m = 16, 24
    runs = []
    for host in (False, True):
        w, scene, paths = _rollout_world(cuda_device, n, m, seed=8)
        rng = np.random.default_rng(4)
        ctrl_id = rng.choice([0, 3, 4, 6], size=(n, m)).astype(np.uint8)
        ctrl_id[:, 0] = 255
        w.set_controllers(_pid_rows(), ctrl_id, path_id=rng.integers(0, 2, (n, m)).astype(np.int16),
                          pid_target=np.stack([rng.uniform(2, 9, (n, m)), rng.uniform(-1, 1, (n, m))], 2).astype(np.float32))
        action = torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device)
        for t in range(5):
            ego = np.tile(np.array([[0.5, 0.1]], np.float32), (n, 1))
            if host:
                w.step_host_ego(ego, action)
            else:
                action[:, 0] = torch.from_numpy(ego).to(cuda_device)
                w.control(action)
                w.step(action)
        runs.append((w.pid_state.cpu().numpy(), w.state_numpy()))
    assert np.array_equal(runs[0][0], runs[1][0])
    for k in ("x", "y", "heading", "speed"):
        assert np.array_equal(runs[0][1][k], runs[1][1][k])


def test_rejections_keep_the_previous_binding(cuda_device):
    import torch

    from tactics2d_b200 import _lib
    from tactics2d_b200.controller import PIDController

    n, m = 4, 3
    w, scene, paths = _rollout_world(cuda_device, n, m, seed=2)
    ctrl_id = np.full((n, m), 0, np.uint8)
    good = PIDController().params()
    w.set_controllers([good], ctrl_id, pid_target=np.ones((n, m, 2), np.float32))
    bound = (w.pid_target, w.pid_state)
    lib, ctx = w.lib, w._ctx

    def bad(**kw):
        r = PIDController().params()
        for k, v in kw.items():
            setattr(r, k, v)
        return r
    for r in (bad(dt=0.0), bad(max_steering=0.0), bad(max_accel=0.0), bad(min_accel=0.0), bad(max_accel=1.0, min_accel=2.0),
              bad(derivative_filter_alpha=0.0), bad(derivative_filter_alpha=1.5), bad(pid_lateral=7),
              bad(pid_longitudinal=2), bad(pid_lateral=2, wheel_base=0.0), bad(pid_lateral=4, wheel_base=-1.0)):
        with pytest.raises(_lib.T2DError):
            w.set_controllers([r], ctrl_id, pid_target=np.ones((n, m, 2), np.float32))
        assert (w.pid_target, w.pid_state) == bound
    act = torch.full((n, m, 2), 7.0, device=cuda_device)
    w.control(act)
    assert w.pid_state.abs().sum() > 0                               # the previous binding still runs
    snap = (act.clone(), w.last_accel.clone(), w.pid_state.clone())
    from tactics2d_b200.world import _ptr
    assert lib.t2d_set_pid(ctx, _ptr(w.pid_target), _ptr(None)) != 0       # a target without a state
    _lib.check(lib.t2d_set_pid(ctx, _ptr(None), _ptr(None)))
    for before in (lambda: None, lambda: _lib.check(lib.t2d_set_pid(ctx, _ptr(None), _ptr(snap[2])))):
        before()
        launches = _lib.load().t2d_launch_count()
        assert lib.t2d_control(ctx, _ptr(act), w._stream()) != 0      # no state / no target: refused
        assert _lib.load().t2d_launch_count() == launches
        torch.cuda.synchronize()
        assert torch.equal(act, snap[0]) and torch.equal(w.last_accel, snap[1])
    # a PATH-only table needs no target
    row = bad(pid_lateral=4, pid_longitudinal=0)
    w.set_controllers([row], ctrl_id, path_id=np.zeros((n, m), np.int16))
    w.control(act)


def test_closed_loop_sign_and_convergence(cuda_device):
    """A PID NPC 2 m right of a straight path, heading along it, steers left at once and closes 90 % of the offset in
    200 ticks (gains and speed rehearsed with tests/pid_oracle.py + oracle.physics)."""
    import torch

    from tactics2d_b200 import BatchedWorld
    from tactics2d_b200.controller import PIDController
    from tactics2d_b200.types import TypeParams, TypeTable

    w = BatchedWorld(1, 2, TypeTable([TypeParams()]), device=cuda_device)
    w.set_state(np.array([[0.0, 0.0]]), np.array([[-2.0, 0.0]]), np.zeros((1, 2)), np.array([[5.0, 0.0]]),
                type_id=np.array([[0, 255]], np.uint8))
    w.set_paths([np.array([[-10.0, 0.0], [400.0, 0.0]])])
    c = PIDController(lateral_error="path_cross_track", dt=0.1, kp_lat=0.4, ki_lat=0.02, kd_lat=0.6)
    row = c.params()
    row.wheel_base = 2.0
    w.set_controllers([row], np.array([[0, 255]], np.uint8), path_id=np.zeros((1, 2), np.int16),
                      pid_target=np.array([[[5.0, 0.0], [0.0, 0.0]]], np.float32))
    action = torch.zeros((1, 2, 2), dtype=torch.float32, device=cuda_device)
    for t in range(200):
        w.control(action)
        if t == 0:
            assert float(action[0, 0, 1]) > 0.0                          # (accel, steer): a left turn
        w.step(action)
    assert abs(float(w.y[0, 0])) < 0.2
