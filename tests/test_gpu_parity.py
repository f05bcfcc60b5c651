"""GPU parity tests proper: the CUDA path (through the C ABI) against the float64 oracle.

Protocol (SURVEY.md section 7 "hard parts"): teacher-forced per step -
  1. physics: the oracle steps the SAME fp32 state the GPU read, in float64; GPU state must be
     within 1e-5 relative (heading modulo 2 pi);
  2. events: the oracle evaluates collisions / out-of-bound on the poses the GPU WROTE (cast to
     float64); flags, first-hit participant and first-hit segment indices must be bit-exact;
  3. status / done: bit-exact from those flags and the step counter.
plus short free-running rollouts with an error-growth budget.
"""

import numpy as np
import pytest

from oracle import scenario as O
from tests.util import assert_state_close, heading_err, rel_err

pytestmark = pytest.mark.gpu


def _world(scene, device, **kw):
    import torch  # noqa: F401

    from tactics2d_b200 import BatchedWorld

    n, m = scene.shape
    w = BatchedWorld(n, m, scene.table, device=device, **kw)
    w.set_map(scene.segments, scene.bounds)
    w.set_state(scene.x, scene.y, scene.heading, scene.speed, vx=scene.vx, vy=scene.vy, type_id=scene.type_id)
    return w


class _CompiledOracle:
    """The float64 oracle in C + OpenMP (oracle/c/oracle_tick.c; held to the NumPy oracle at 1e-12 by
    tests/test_oracle_c.py): the same two entry points as oracle.scenario, fast enough for full BASELINE sizes."""

    @staticmethod
    def physics_tick(state, type_id, action, table, interval=100, delta_t=5, steer_first=False):
        from oracle import c_oracle as CO

        return CO.physics(state, type_id, action, table, interval, delta_t, steer_first)

    @staticmethod
    def events(x, y, heading, type_id, table, segments=None, bounds=None):
        from oracle import c_oracle as CO

        return CO.events(x, y, heading, type_id, table, segments, bounds)


def _teacher_forced(scene, device, steps, seed=0, interval=100, delta_t=5, max_step=0, any_participant=False,
                    steer_first=False, action_fn=None, rtol=1e-5, compiled=False):
    import torch

    from tactics2d_b200 import synthetic

    P = _CompiledOracle if compiled else O   # who restates the physics and the events

    n, m = scene.shape
    w = _world(scene, device, interval=interval, delta_t=delta_t, max_step=max_step, any_participant=any_participant,
               steer_first=steer_first)
    table = scene.table.as_oracle_table()
    stats = dict(dyn=0, static=0, oob=0, done=0, worst={})
    cnt = np.zeros(n, np.int32)
    for t in range(steps):
        before = w.state_numpy()
        act = action_fn(t) if action_fn else synthetic.random_actions(seed * 1000 + t, (n, m))
        ref = P.physics_tick(before, scene.type_id, act, table, interval, delta_t, steer_first)
        r = w.step(torch.from_numpy(act).to(device))
        torch.cuda.synchronize()
        got = w.state_numpy()
        active = scene.type_id != 255
        worst = assert_state_close(got, ref, mask=active, rtol=rtol, what=f"step {t}")
        for k, v in worst.items():
            stats["worst"][k] = max(stats["worst"].get(k, 0.0), v)
        # inactive slots pass through untouched
        for k in ("x", "y", "heading", "speed", "vx", "vy"):
            assert np.array_equal(got[k][~active], before[k][~active])
        fl, hi, hs = P.events(got["x"], got["y"], got["heading"], scene.type_id, table, scene.segments, scene.bounds)
        gfl, ghi, ghs = r.flags.cpu().numpy(), r.hit_index.cpu().numpy(), r.hit_segment.cpu().numpy()
        assert np.array_equal(gfl, fl), f"flags differ at step {t}: {np.argwhere(gfl != fl)[:5]}"
        assert np.array_equal(ghi, hi), f"hit_index differs at step {t}: {np.argwhere(ghi != hi)[:5]}"
        assert np.array_equal(ghs, hs), f"hit_segment differs at step {t}: {np.argwhere(ghs != hs)[:5]}"
        cnt += 1
        st, done = O.status(fl, scene.type_id, cnt, max_step, ego_only=not any_participant)
        assert np.array_equal(r.status.cpu().numpy(), st)
        assert np.array_equal(r.done.cpu().numpy(), done)
        assert np.array_equal(w.step_count.cpu().numpy(), cnt)
        stats["dyn"] += int((fl & 1).astype(bool).sum())
        stats["static"] += int((fl & 2).astype(bool).sum())
        stats["oob"] += int((fl & 4).astype(bool).sum())
        stats["done"] += int(done.sum())
    w.close()
    return stats


def test_config1_parity_gate(cuda_device):
    """BASELINE.json configs[0]: 1 scenario x 8 participants, SingleTrackKinematics, empty map:
    200 teacher-forced steps, then 50 free-running steps against the float64 free-running oracle."""
    import torch

    from tactics2d_b200 import synthetic

    scene = synthetic.config1(0)
    stats = _teacher_forced(scene, cuda_device, 200, seed=1)
    assert stats["dyn"] > 0, "config 1 must exercise colliding pairs"
    # free run
    w = _world(scene, cuda_device)
    table = scene.table.as_oracle_table()
    ref = {k: v.astype(np.float64) for k, v in scene.state().items()}
    for t in range(50):
        act = synthetic.random_actions(5000 + t, scene.shape)
        ref = O.physics_tick(ref, scene.type_id, act, table)
        w.step(torch.from_numpy(act).to(cuda_device))
    got = w.state_numpy()
    assert rel_err(got["x"], ref["x"]).max() < 5e-4 and rel_err(got["y"], ref["y"]).max() < 5e-4
    assert heading_err(got["heading"], ref["heading"]).max() < 5e-4
    w.close()


@pytest.mark.parametrize("n,m", [(64, 64), (33, 64), (16, 128), (40, 32), (7, 8), (5, 4)])
def test_config2_kinematics_obb_gridmap(cuda_device, n, m):
    from tactics2d_b200 import synthetic

    scene = synthetic.config2(n, m, seed=11 + n, size=200.0 if m >= 64 else 80.0)
    stats = _teacher_forced(scene, cuda_device, 6, seed=2, max_step=4)
    assert stats["static"] > 0 and stats["done"] > 0


def test_dense_arena_many_collisions(cuda_device):
    """64 vehicles in a 60 m arena: most participants collide; first-hit indices must still be exact."""
    from tactics2d_b200 import synthetic

    scene = synthetic.config2(48, 64, seed=5, size=60.0)
    stats = _teacher_forced(scene, cuda_device, 4, seed=3, any_participant=True)
    assert stats["dyn"] > 48 * 64 * 0.3 * 4


@pytest.mark.parametrize("m", [1, 3, 5, 7, 13, 30, 63, 100])
def test_ragged_participant_counts(cuda_device, m):
    """M not a multiple of 4 (scalar load path, padded lanes) and inactive slots."""
    from tactics2d_b200 import synthetic

    scene = synthetic.with_inactive(synthetic.config2(21, m, seed=m, size=max(30.0, 6.0 * m ** 0.5)), 0.2, seed=m)
    _teacher_forced(scene, cuda_device, 4, seed=4, any_participant=True)


def test_mixed_models_and_shapes(cuda_device):
    """Config-4 style: vehicles + cyclists (kinematics) + pedestrians (PointMass newton, discs),
    with 10 % inactive slots, walls and bounds."""
    from tactics2d_b200 import synthetic

    scene = synthetic.config4(96, 32, seed=9, size=70.0, segments=synthetic.grid_wall_segments(70.0, 35.0, 12.0))
    scene = synthetic.with_inactive(scene, 0.1, seed=1)
    act = lambda t: synthetic.random_actions(700 + t, scene.shape, accel=(-3, 3), steer=(-1.2, 1.2))
    stats = _teacher_forced(scene, cuda_device, 8, action_fn=act, any_participant=True)
    assert stats["dyn"] > 0 and stats["static"] > 0


def test_pointmass_euler_and_static_types(cuda_device):
    from tactics2d_b200 import TypeParams, TypeTable, synthetic

    rows = [TypeParams.pedestrian("adult_male", "euler"), TypeParams.pedestrian("children_six_year_old", "newton"),
            TypeParams.obstacle(6.0, 3.0), TypeParams.vehicle("large_car")]
    table = TypeTable(rows)
    base = synthetic.config2(32, 16, seed=21, size=30.0)
    rng = np.random.default_rng(3)
    tid = rng.integers(0, 4, base.shape).astype(np.uint8)
    speed = np.where(tid <= 1, rng.uniform(0, 3, base.shape), base.speed).astype(np.float32)
    speed = np.where(tid == 2, 0.0, speed).astype(np.float32)
    scene = synthetic._finish(table, base.x, base.y, base.heading, speed, tid, base.segments, base.bounds, "pm")
    act = lambda t: synthetic.random_actions(900 + t, scene.shape, accel=(-4, 4), steer=(-4, 4))
    _teacher_forced(scene, cuda_device, 6, action_fn=act, any_participant=True, interval=50, delta_t=3)


def test_config3_dynamics(cuda_device):
    """SingleTrackDynamics at highway speeds (20-40 m/s) with straight road-edge polylines."""
    from tactics2d_b200 import synthetic

    segs = np.array([[0, -30, 668, -30], [0, 2, 668, 2], [0, -14, 668, -14]], dtype=np.float32)
    scene = synthetic.config3(64, 64, seed=3, segments=segs)
    act = lambda t: synthetic.random_actions(300 + t, scene.shape, accel=(-6, 3), steer=(-0.05, 0.05))
    stats = _teacher_forced(scene, cuda_device, 6, action_fn=act, any_participant=True)
    assert stats["worst"]["x"] < 1e-5


def test_dynamics_low_speed_region(cuda_device):
    """Low speeds.  The reference's explicit Euler of the yaw-rate equation multiplies any perturbation
    by |1 - 1.34/v| per 5 ms sub-step (medium car): unstable below v = 0.67 m/s, x1e10 per step at
    v = 0.3.  The device runs this model in fp64, so parity holds wherever the amplification stays
    below ~1e9: |v| >= 0.45 here, and the (non-stiff) |v| < 0.1 fallback branch.  Between 0.1 and
    ~0.35 m/s no implementation that differs from the reference by a single rounding can reproduce
    its output; that band is excluded (DESIGN.md "numerics")."""
    from tactics2d_b200 import synthetic

    scene = synthetic.config3(32, 16, seed=8)
    rng = np.random.default_rng(4)
    v = rng.uniform(0.45, 1.0, scene.shape).astype(np.float32)
    v[:, :4] = rng.uniform(0.0, 0.09, (scene.shape[0], 4))   # low-speed kinematic fallback branch
    scene = synthetic._finish(scene.table, scene.x, scene.y, scene.heading, v, scene.type_id, None, None, "dyn-low")
    act = lambda t: synthetic.random_actions(40 + t, scene.shape, accel=(0.0, 0.0), steer=(-0.5, 0.5))
    _teacher_forced(scene, cuda_device, 1, action_fn=act)


@pytest.mark.parametrize("interval,delta_t", [(9, 5), (50, 3), (33, 10), (100, 1)])
def test_intervals_and_remainder(cuda_device, interval, delta_t):
    from tactics2d_b200 import synthetic

    scene = synthetic.config4(16, 32, seed=2, size=60.0)
    _teacher_forced(scene, cuda_device, 3, seed=6, interval=interval, delta_t=delta_t)


def test_steer_first_action_order(cuda_device):
    """Env action order is (steering, accel) (envs/parking.py:239)."""
    from tactics2d_b200 import synthetic

    scene = synthetic.config4(8, 32, seed=12, size=60.0)
    _teacher_forced(scene, cuda_device, 3, seed=8, steer_first=True)


def test_full_size_config2_one_step(cuda_device):
    """BASELINE.json configs[1] at full size (4096 x 64): one teacher-forced step, every flag and
    index compared (the NumPy oracle needs a few seconds per step at this size)."""
    from tactics2d_b200 import synthetic

    scene = synthetic.config2(4096, 64, seed=1)
    stats = _teacher_forced(scene, cuda_device, 1, seed=9)
    assert stats["dyn"] > 1000 and stats["static"] > 5000


def test_check_events_matches_step_and_is_idempotent(cuda_device):
    import torch

    from tactics2d_b200 import synthetic

    scene = synthetic.config2(32, 64, seed=3, size=90.0)
    w = _world(scene, cuda_device)
    r = w.step(torch.from_numpy(synthetic.random_actions(1, scene.shape)).to(cuda_device))
    fl, hi, hs = r.flags.clone(), r.hit_index.clone(), r.hit_segment.clone()
    state = w.state_numpy()
    for _ in range(2):
        r2 = w.check_events()
        torch.cuda.synchronize()
        assert torch.equal(r2.flags, fl) and torch.equal(r2.hit_index, hi) and torch.equal(r2.hit_segment, hs)
    after = w.state_numpy()
    for k in state:
        assert np.array_equal(state[k], after[k])
    assert int(w.step_count.max()) == 1
    w.close()


def test_collision_symmetry_property(cuda_device):
    """Size-independent property at full size: i hits j <=> j hits i, so hit_index[n, hit_index[n, i]] <= i."""
    import torch

    from tactics2d_b200 import synthetic

    scene = synthetic.config2(4096, 64, seed=33, size=120.0)
    w = _world(scene, cuda_device)
    r = w.step(torch.from_numpy(synthetic.random_actions(2, scene.shape)).to(cuda_device))
    hi = r.hit_index.cpu().numpy().astype(np.int64)
    n_idx, i_idx = np.nonzero(hi >= 0)
    j = hi[n_idx, i_idx]
    back = hi[n_idx, j]
    assert (back >= 0).all() and (back <= i_idx).all()
    assert ((r.flags.cpu().numpy() & 1) == (hi >= 0)).all()
    w.close()


def test_touching_counts_and_containment(cuda_device):
    """Closed-set semantics on exactly representable poses: touching boxes intersect, a wall wholly
    inside a box intersects, a box wholly inside a box intersects, corner on the boundary is inside."""
    import torch

    from tactics2d_b200 import BatchedWorld, TypeParams, TypeTable

    table = TypeTable([TypeParams.obstacle(4.0, 2.0), TypeParams.obstacle(1.0, 0.5), TypeParams.pedestrian("adult_male")])
    x = np.array([[0.0, 4.0, 20.0, 20.25, 40.0, 42.25, 60.0, 70.0]], np.float32)
    y = np.array([[0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 9.0, 0.0]], np.float32)
    h = np.zeros((1, 8), np.float32)
    tid = np.array([[0, 0, 0, 1, 0, 2, 0, 0]], np.uint8)   # 0-1 touch; 3 inside 2; disc 5 (r=.2) misses box 4 by .05
    w = BatchedWorld(1, 8, table, device=cuda_device, any_participant=True)
    segs = np.array([[59.5, 9.0, 60.5, 9.0], [100.0, 0.0, 101.0, 0.0]], np.float32)   # seg 0 wholly inside box 6
    w.set_map(segs, (-10.0, 72.0, -10.0, 10.0))    # box 6 top edge touches ymax=10 -> inside; box 7 right edge touches xmax -> inside
    w.set_state(x, y, h, np.zeros((1, 8), np.float32), type_id=tid)
    r = w.check_events()
    torch.cuda.synchronize()
    hi = r.hit_index.cpu().numpy()[0]
    hs = r.hit_segment.cpu().numpy()[0]
    fl = r.flags.cpu().numpy()[0]
    assert list(hi) == [1, 0, 3, 2, -1, -1, -1, -1]
    assert list(hs) == [-1, -1, -1, -1, -1, -1, 0, -1]
    assert not (fl & 4).any()
    ofl, ohi, ohs = O.events(x, y, h, tid, table.as_oracle_table(), segs, (-10.0, 72.0, -10.0, 10.0))
    assert np.array_equal(ofl[0], fl) and np.array_equal(ohi[0], hi) and np.array_equal(ohs[0], hs)
    w.close()


def test_reset_pool(cuda_device):
    import torch

    from tactics2d_b200 import synthetic

    scene = synthetic.config2(64, 64, seed=4)
    w = _world(scene, cuda_device, max_step=2)
    init = {k: torch.from_numpy(v).to(cuda_device) for k, v in scene.state().items()}
    for t in range(3):
        r = w.step(torch.from_numpy(synthetic.random_actions(t, scene.shape)).to(cuda_device))
    assert int(r.done.sum()) == 64  # time exceeded everywhere
    mask = torch.zeros(64, dtype=torch.uint8, device=cuda_device)
    mask[::2] = 1
    idx = torch.arange(63, -1, -1, dtype=torch.int32, device=cuda_device)
    before = w.state_numpy()
    w.reset(mask, init, idx)
    torch.cuda.synchronize()
    after = w.state_numpy()
    cnt = w.step_count.cpu().numpy()
    for n in range(64):
        if n % 2 == 0:
            assert np.array_equal(after["x"][n], scene.x[63 - n]) and np.array_equal(after["vy"][n], scene.vy[63 - n])
            assert cnt[n] == 0
        else:
            assert np.array_equal(after["x"][n], before["x"][n]) and cnt[n] == 3
    w.close()


# ---------------------------------------------------------------------------- the reference's own map files
def test_config3_dynamics_on_highD_tile(cuda_device):
    """BASELINE.json configs[2]: SingleTrackDynamics + map-polyline collision on the highD_1 tile (compiled from
    data/highD_map/highD_1.osm of the reference checkout by tactics2d_b200.map; solid lane markings = road edges)."""
    from tactics2d_b200 import synthetic
    from tactics2d_b200.map import load_collidable_segments

    seg, bounds = load_collidable_segments("highD_1")
    scene = synthetic.config3(64, 64, seed=13, segments=seg, bounds=bounds)
    act = lambda t: synthetic.random_actions(1300 + t, scene.shape, accel=(-6, 3), steer=(-0.05, 0.05))
    stats = _teacher_forced(scene, cuda_device, 5, action_fn=act, any_participant=True)
    assert stats["static"] > 0


def test_config4_mixed_on_inD_tile(cuda_device):
    """configs[3] (one shard): vehicles / cyclists / pedestrians on the inD_1 intersection (211 collidable segments)."""
    from tactics2d_b200 import synthetic
    from tactics2d_b200.map import load_collidable_segments

    seg, bounds = load_collidable_segments("inD_1")
    scene = synthetic.with_inactive(synthetic.config4(128, 32, seed=14, segments=seg, bounds=bounds, size=150.0), 0.05, seed=2)
    act = lambda t: synthetic.random_actions(1400 + t, scene.shape, accel=(-3, 3), steer=(-0.8, 0.8))
    stats = _teacher_forced(scene, cuda_device, 5, action_fn=act, any_participant=True)
    assert stats["static"] > 0 and stats["dyn"] > 0


def test_config5_m128_on_rounD_tile(cuda_device):
    """configs[4] (one shard): 128 participants per scenario (a whole warp per scenario) on rounD_0 (411 segments)."""
    from tactics2d_b200 import synthetic
    from tactics2d_b200.map import load_collidable_segments

    seg, bounds = load_collidable_segments("rounD_0")
    scene = synthetic.config5(24, 128, seed=15, segments=seg, bounds=bounds, size=200.0)
    stats = _teacher_forced(scene, cuda_device, 4, seed=15, any_participant=True)
    assert stats["static"] > 0 and stats["dyn"] > 0


def test_map_too_large_for_shared_memory_uses_global_path(cuda_device):
    """A map blob above the shared-memory staging limit is read from global memory (same results)."""
    from tactics2d_b200 import synthetic

    rng = np.random.default_rng(0)
    # ~9000 short random segments over a 400 m square: blob > 120 KB
    p = rng.uniform(0, 400, (9000, 2))
    d = rng.uniform(-6, 6, (9000, 2))
    seg = np.concatenate([p, p + d], 1).astype(np.float32)
    scene = synthetic.config2(12, 64, seed=16, size=400.0)
    scene.segments = seg
    stats = _teacher_forced(scene, cuda_device, 2, seed=16, any_participant=True)
    assert stats["static"] > 0


@pytest.mark.parametrize("n,m,chunks", [(256, 64, 0), (100, 7, 3), (50, 128, 2), (4096, 64, 0)])
def test_step_host_equals_step(cuda_device, monkeypatch, n, m, chunks):
    """t2d_step_host (host action in, host done / status out, chunked copy under the kernel) is the same tick as
    t2d_step on device buffers: state, flags, hit indices, status and done bit-identical over a rollout that
    carries collisions and time-outs, for chunk splits that do and do not divide N."""
    import torch

    from tactics2d_b200 import synthetic

    monkeypatch.setenv("T2D_HOST_CHUNKS", str(chunks))
    scene = synthetic.config2(n, m, seed=77)
    a = _world(scene, cuda_device, max_step=4)
    b = _world(scene, cuda_device, max_step=4)
    seen_done = 0
    for t in range(6):
        act = synthetic.random_actions(4200 + t, (n, m))
        ra = a.step(torch.from_numpy(act).to(cuda_device))
        host = torch.from_numpy(act).pin_memory() if t % 2 == 0 else act          # pinned and pageable callers
        done, status = b.step_host(host)
        torch.cuda.synchronize()
        sa, sb = a.state_numpy(), b.state_numpy()
        for k in sa:
            assert np.array_equal(sa[k], sb[k], equal_nan=True), (t, k)
        assert np.array_equal(ra.flags.cpu().numpy(), b.result.flags.cpu().numpy())
        assert np.array_equal(ra.hit_index.cpu().numpy(), b.result.hit_index.cpu().numpy())
        assert np.array_equal(ra.hit_segment.cpu().numpy(), b.result.hit_segment.cpu().numpy())
        assert np.array_equal(ra.status.cpu().numpy(), status)
        assert np.array_equal(ra.done.cpu().numpy(), done)
        seen_done += int(done.sum())
    assert seen_done > 0


# ---------------------------------------------------------------------------- every BASELINE configuration at full size
# (checker: the compiled float64 oracle; >= 3 teacher-forced steps each; every state within 1e-5, every flag / index /
#  status / done bit-exact)
def test_full_size_config2_three_steps_compiled_oracle(cuda_device):
    from tactics2d_b200 import synthetic

    scene = synthetic.config2(4096, 64, seed=1)
    stats = _teacher_forced(scene, cuda_device, 3, seed=19, compiled=True)
    assert stats["dyn"] > 3000 and stats["static"] > 15000


def test_full_size_config3_dynamics_on_highD(cuda_device):
    """configs[2]: 4096 x 64 SingleTrackDynamics on the highD_1 tile."""
    from tactics2d_b200 import synthetic
    from tactics2d_b200.map import load_collidable_segments

    seg, bounds = load_collidable_segments("highD_1")
    scene = synthetic.config3(4096, 64, seed=23, segments=seg, bounds=bounds)
    act = lambda t: synthetic.random_actions(2300 + t, scene.shape, accel=(-6, 3), steer=(-0.05, 0.05))
    stats = _teacher_forced(scene, cuda_device, 3, action_fn=act, any_participant=True, compiled=True)
    assert stats["static"] > 0 and stats["dyn"] > 0


def test_full_size_config4_mixed_on_inD(cuda_device):
    """configs[3]: 16384 x 32 vehicles / cyclists / pedestrians on the inD_1 intersection."""
    from tactics2d_b200 import synthetic
    from tactics2d_b200.map import load_collidable_segments

    seg, bounds = load_collidable_segments("inD_1")
    scene = synthetic.config4(16384, 32, seed=24, segments=seg, bounds=bounds)
    act = lambda t: synthetic.random_actions(2400 + t, scene.shape, accel=(-3, 3), steer=(-0.8, 0.8))
    stats = _teacher_forced(scene, cuda_device, 3, action_fn=act, any_participant=True, compiled=True)
    assert stats["static"] > 1000 and stats["dyn"] > 1000


def test_large_config5_m128_on_rounD(cuda_device):
    """configs[4] at one GPU's share of the 8-GPU job: 8192 x 128 kinematic vehicles on rounD_0 (more warp tiles than
    the GPU holds at once: the persistent CTAs loop)."""
    from tactics2d_b200 import synthetic
    from tactics2d_b200.map import load_collidable_segments

    seg, bounds = load_collidable_segments("rounD_0")
    scene = synthetic.config5(8192, 128, seed=25, segments=seg, bounds=bounds)
    stats = _teacher_forced(scene, cuda_device, 3, seed=25, any_participant=True, compiled=True)
    assert stats["static"] > 1000 and stats["dyn"] > 1000


def _free_rollout(scene, device, steps, action_fn, budget, **kw):
    """GPU and float64 oracle both run FREE from the same initial state (the oracle never sees the GPU's states): the
    trajectories may drift apart by rounding only - position / speed error within `budget` (relative to max(|ref|, 1))
    after `steps` ticks; participants that touch anything are excluded from then on (a flag flips one ulp apart)."""
    import torch

    n, m = scene.shape
    w = _world(scene, device, **kw)
    table = scene.table.as_oracle_table()
    ref = {k: v.astype(np.float64) for k, v in scene.state().items()}
    worst = 0.0
    for t in range(steps):
        act = action_fn(t)
        ref = _CompiledOracle.physics_tick({k: v.astype(np.float32) for k, v in ref.items()}, scene.type_id, act, table)
        w.step(torch.from_numpy(act).to(device))
    torch.cuda.synchronize()
    got = w.state_numpy()
    active = scene.type_id != 255
    for k in ("x", "y", "speed"):
        worst = max(worst, float(np.max(rel_err(got[k], ref[k])[active])))
    worst = max(worst, float(np.max(heading_err(got["heading"], ref["heading"])[active])))
    w.close()
    assert worst <= budget, worst
    return worst


def test_free_rollout_50_steps_config2(cuda_device):
    """50 free-running ticks at C2 (1024 x 64): fp32 state against the float64 oracle fed its own fp32-rounded states.
    Budget 5e-4: ~1e-5 per tick at most, errors do not compound beyond linear growth over 50 ticks."""
    from tactics2d_b200 import synthetic

    scene = synthetic.config2(1024, 64, seed=31)
    act = lambda t: synthetic.random_actions(3100 + t, scene.shape)
    _free_rollout(scene, cuda_device, 50, act, 5e-4)


def test_free_rollout_50_steps_config4(cuda_device):
    from tactics2d_b200 import synthetic
    from tactics2d_b200.map import load_collidable_segments

    seg, bounds = load_collidable_segments("inD_1")
    scene = synthetic.config4(1024, 32, seed=34, segments=seg, bounds=bounds)
    act = lambda t: synthetic.random_actions(3400 + t, scene.shape, accel=(-3, 3), steer=(-0.8, 0.8))
    _free_rollout(scene, cuda_device, 50, act, 5e-4)
