"""Sampled resets on the device (K13 -> K2 -> K14, ``BatchedWorld.set_reset_sampler`` / ``reset_sampled``) against the
restatement in tests/reset_sampler_oracle.py: the drawn rows and episode counters, the placed start states and their
tries bit for bit, the check_events invariant, the row-owned columns, and the rejected calls."""

import numpy as np
import pytest
import torch

from tactics2d_b200 import BatchedWorld, TypeParams, TypeTable
from tests import env_chain_oracle as EC
from tests import reset_sampler_oracle as R
from tests.util import RTOL, rel_err

pytestmark = pytest.mark.gpu
STATE = ("x", "y", "heading", "speed", "vx", "vy")


def _scene(rng, P, M, size, table, types):
    f = lambda a: a.astype(np.float32)
    return dict(x=f(rng.uniform(-size, size, (P, M))), y=f(rng.uniform(-size, size, (P, M))),
                heading=f(rng.uniform(-np.pi, np.pi, (P, M))), speed=f(rng.uniform(0, 5, (P, M))),
                type_id=rng.choice(types, (P, M)).astype(np.uint8))


def _pool(sc, dev):
    return {k: torch.from_numpy(np.ascontiguousarray(sc[k])).to(dev) for k in ("x", "y", "heading", "speed")}


def _np_pool(pool):
    """The pool as the oracle's K2 takes it: vx, vy as K2 derives them for a pool without velocities."""
    p = {k: v.cpu().numpy() for k, v in pool.items()}
    h = p["heading"].astype(np.float64)
    p["vx"] = (p["speed"] * np.cos(h)).astype(np.float32)
    p["vy"] = (p["speed"] * np.sin(h)).astype(np.float32)
    return p


def _snap(w):
    s = w.state_numpy()
    s["type_id"] = w.type_id.cpu().numpy()
    s["step_count"] = w.step_count.cpu().numpy()
    return s


def _ctx(table):
    t = table.as_oracle_table()
    return dict(table=t, n_types=len(table), model=t["model"], wheel_radius=t["wheel_radius"].astype(np.float32))


@pytest.mark.parametrize("N", [1, 7, 4099])
@pytest.mark.parametrize("P_of", ["1", "2", "7", "N"])
def test_rows_and_episode_counters(N, P_of, cuda_device):
    P = N if P_of == "N" else int(P_of)
    M = 3
    table = TypeTable([TypeParams.vehicle("medium_car")])
    rng = np.random.default_rng(N * 10 + P)
    sc = _scene(rng, max(P, N), M, 100.0, table, [0])
    w = BatchedWorld(N, M, table, device=cuda_device)
    w.set_state(sc["x"][:N], sc["y"][:N], sc["heading"][:N], sc["speed"][:N], type_id=sc["type_id"][:N])
    pool = {k: v[:P] for k, v in _pool(sc, cuda_device).items()}
    seed = 0x1234_5678_9ABC_DEF0 + N
    w.set_reset_sampler(seed)
    ep = np.zeros(N, np.uint32)
    pr = np.arange(N, dtype=np.int32)
    for _ in range(3):
        mask = rng.random(N) < 0.5
        before = {k: getattr(w, k).cpu().numpy().copy() for k in STATE + ("type_id", "step_count", "reset_try")}
        w.step_count.fill_(3)
        before["step_count"][:] = 3
        w.reset_sampled(torch.from_numpy(mask.astype(np.uint8)), pool)
        torch.cuda.synchronize()
        rows = R.pool_rows(mask, ep, seed, P)
        for k in ("type_id", "step_count", "reset_try"):
            assert np.array_equal(getattr(w, k).cpu().numpy()[~mask], before[k][~mask]), k
        pr[mask] = rows[mask]
        ep[mask] += 1
        assert np.array_equal(w.pool_row.cpu().numpy(), pr)
        assert np.array_equal(w.episode_count.cpu().numpy().view(np.uint32), ep)
        for k in STATE:
            got = getattr(w, k).cpu().numpy()
            assert np.array_equal(got[~mask].view(np.uint32), before[k][~mask].view(np.uint32)), k
            if k in ("x", "y", "heading", "speed"):
                assert np.array_equal(got[mask], pool[k].cpu().numpy()[pr[mask]]), k
    assert np.array_equal(w.reset_try.cpu().numpy(), np.full((N, M), -1, np.int8))
    w.close()


def _tables():
    cars = [TypeParams.vehicle("medium_car"), TypeParams.vehicle("small_car"), TypeParams.pedestrian()]
    return {"mixed": (TypeTable(cars), [0, 1, 2]),
            "drift": (TypeTable([TypeParams.vehicle("medium_car", "drift"), TypeParams.pedestrian()]), [0, 1])}


def _check_placement(w, table, before, prev_try, mask, pool, seed, ep, jit, tries, scene_of, sample_rows=True):
    ctx = _ctx(table)
    snap = dict(before)
    pr = R.pool_rows(mask, ep, seed, pool["x"].shape[0], sample_rows)
    s = EC.reset(snap, mask, _np_pool(pool), pr, ctx)
    ref, rt, ep2 = R.place(s, mask, ep, seed, jit, tries, ctx["table"], ctx["n_types"], scene_of, reset_try=prev_try)
    got = _snap(w)
    for k in ("x", "y", "heading", "speed"):
        assert np.array_equal(got[k].view(np.uint32), ref[k].view(np.uint32)), k
    vs = np.maximum(np.abs(ref["speed"]).astype(np.float64), 1.0)
    for k in ("vx", "vy"):
        assert rel_err(got[k], ref[k], vs).max() <= RTOL, k
    assert np.array_equal(w.reset_try.cpu().numpy(), rt)
    assert np.array_equal(w.episode_count.cpu().numpy().view(np.uint32), ep2)
    if "omega_wf" in ref:
        assert np.array_equal(got["omega_wf"], ref["omega_wf"]) and np.array_equal(got["omega_wr"], ref["omega_wr"])
    # the invariant: a placed slot shows no event
    fl = w.check_events().flags.cpu().numpy()
    placed = w.reset_try.cpu().numpy() >= 0
    assert (fl[placed] == 0).all()
    return rt, ep2


@pytest.mark.parametrize("M,T,kind", [(1, 1, "mixed"), (33, 8, "mixed"), (64, 32, "mixed"), (128, 8, "mixed"),
                                      (128, 32, "mixed"), (2, 32, "drift"), (33, 1, "drift"), (64, 8, "drift")])
def test_placement_matches_the_oracle(M, T, kind, cuda_device):
    table, types = _tables()[kind]
    N, P = 3, 7
    rng = np.random.default_rng(M * 100 + T)
    size = 3.0 * np.sqrt(M) + 6.0   # dense: a slot's jitter finds most tries blocked
    sc = _scene(rng, P, M, size, table, types)
    walls = np.asarray([(-size - 2, -size - 2, size + 2, -size - 2), (size + 2, -size - 2, size + 2, size + 2),
                        (-size / 2, 0.0, size / 2, 0.0), (0.0, -size / 2, 0.0, size / 2)], np.float32)
    bounds = (-size - 3, size + 3, -size - 3, size + 3)
    w = BatchedWorld(N, M, table, device=cuda_device)
    w.set_map(walls, bounds)
    w.set_state(sc["x"][:N], sc["y"][:N], sc["heading"][:N], sc["speed"][:N], type_id=sc["type_id"][:N])
    jit = np.tile(np.array([[-2.0, 2.0], [-2.0, 2.0], [-0.5, 0.5], [-1.0, 1.0]], np.float32), (M, 1, 1))
    jit[M // 2] = 0.0   # one slot without jitter
    seed = 77 + M
    w.set_reset_sampler(seed, jitter=jit, tries=T)
    pool = _pool(sc, cuda_device)
    ep = np.zeros(N, np.uint32)
    for r in range(2):
        mask = np.ones(N, bool) if r == 0 else rng.random(N) < 0.6
        before, prev_try = _snap(w), w.reset_try.cpu().numpy()
        w.reset_sampled(torch.from_numpy(mask.astype(np.uint8)), pool)
        torch.cuda.synchronize()
        rt, ep = _check_placement(w, table, before, prev_try, mask, pool, seed, ep, jit, T,
                                  lambda n: (walls, bounds, None))
    moved = jit.reshape(M, 8).any(1)
    assert (rt >= 0).any() or M == 1
    if M >= 64:   # dense enough that some jittered slot finds every try blocked and keeps its pool state
        assert (rt[:, moved] == -1).any()


def test_area_tiles_follow_the_row_and_block_placement(cuda_device):
    """A map table whose tile follows the drawn row (an Area frame with a hole, and an open lot), with the type, target
    and route pools: the row-owned columns take the row's values and the placement sees the row's tile."""
    ped, car = TypeParams.pedestrian(), TypeParams.vehicle("medium_car")
    table = TypeTable([car, ped])
    N, M, P = 6, 4, 5
    ring = lambda x0, x1, y0, y1: [(x0, y0, x1, y0), (x1, y0, x1, y1), (x1, y1, x0, y1), (x0, y1, x0, y0)]
    frame = ring(-30, -4, -30, 30) + ring(4, 30, -30, 30) + ring(-4, 4, 4, 30) + ring(-4, 4, -30, -4)
    tiles = [dict(segments=np.asarray(frame, np.float32), bounds=(-40, 40, -40, 40), poly_start=[0, 4, 8, 12, 16]),
             dict(segments=np.asarray(ring(-1, 1, 10, 12), np.float32), bounds=(-20, 20, -20, 20), poly_start=[0, 4])]
    w = BatchedWorld(N, M, table, device=cuda_device)
    w.set_map_table(tiles, np.zeros(N, np.int64))
    rng = np.random.default_rng(5)
    sc = _scene(rng, P, M, 2.0, table, [1])
    sc["x"][:, 1:] += 40.0   # the other slots far away (outside the box: not jittered below)
    w.set_state(*(np.resize(sc[k], (N, M)) for k in ("x", "y", "heading", "speed")), type_id=np.ones((N, M), np.uint8))
    target = rng.uniform(-5, 5, (N, 5)).astype(np.float32)
    target[:, 3:] = 1.0
    w.set_goal(target)
    w.set_paths([np.array([[0, 0], [10, 0]], np.float32), np.array([[0, 0], [0, 10]], np.float32)])
    w.set_routes(np.full((N, M), -1, np.int16), threshold=5.0)
    pool_type = rng.choice([0, 1, 255], (P, M)).astype(np.uint8)
    pool_type[:, 0] = 1
    pool_target = rng.uniform(-5, 5, (P, 5)).astype(np.float32)
    pool_tile = rng.integers(0, 2, P).astype(np.int16)
    pool_route = rng.integers(-1, 2, (P, M)).astype(np.int16)
    jit = np.zeros((M, 4, 2), np.float32)
    jit[0] = [[-2.0, 2.0], [-2.0, 2.0], [0.0, 0.0], [0.0, 0.0]]
    seed = 99
    w.set_reset_sampler(seed, jitter=jit, tries=8, type_id=pool_type, target=pool_target, tile_id=pool_tile,
                        route_id=pool_route)
    pool = _pool(sc, cuda_device)
    mask = np.array([1, 1, 0, 1, 1, 1], bool)
    before = _snap(w)
    old_target = w._goal["target"].cpu().numpy().copy()
    w.reset_sampled(torch.from_numpy(mask.astype(np.uint8)), pool)
    torch.cuda.synchronize()
    rows = R.pool_rows(mask, np.zeros(N, np.uint32), seed, P)
    tid = w.type_id.cpu().numpy()
    assert np.array_equal(tid[mask], pool_type[rows[mask]]) and np.array_equal(tid[~mask], before["type_id"][~mask])
    tg = w._goal["target"].cpu().numpy()
    assert np.array_equal(tg[mask], pool_target[rows[mask]]) and np.array_equal(tg[~mask], old_target[~mask])
    assert np.array_equal(w.tile_id.cpu().numpy()[mask], pool_tile[rows[mask]])
    assert np.array_equal(w.route_id.cpu().numpy()[mask], pool_route[rows[mask]])
    # the placement on each scenario's own tile
    ctx = _ctx(table)
    s = dict(before)
    s["type_id"] = tid.copy()
    s = EC.reset(s, mask, _np_pool(pool), rows, ctx)
    s["type_id"] = tid
    tile_of = w.tile_id.cpu().numpy()
    scene_of = lambda n: (tiles[tile_of[n]]["segments"], tiles[tile_of[n]]["bounds"], tiles[tile_of[n]]["poly_start"])
    ref, rt, _ = R.place(s, mask, np.zeros(N, np.uint32), seed, jit, 8, ctx["table"], ctx["n_types"], scene_of)
    got = _snap(w)
    for k in ("x", "y", "heading", "speed"):
        assert np.array_equal(got[k].view(np.uint32), ref[k].view(np.uint32)), k
    assert np.array_equal(w.reset_try.cpu().numpy(), rt)
    fl = w.check_events().flags.cpu().numpy()
    assert (fl[w.reset_try.cpu().numpy() >= 0] == 0).all()
    w.close()


def test_rejected_calls_keep_the_bound_sampler(cuda_device):
    table = TypeTable([TypeParams.vehicle("medium_car")])
    N, M = 3, 2
    w = BatchedWorld(N, M, table, device=cuda_device)
    w.set_state(np.zeros((N, M)), np.zeros((N, M)), np.zeros((N, M)), np.zeros((N, M)), type_id=np.zeros((N, M)))
    pool = {k: torch.zeros((N, M), dtype=torch.float32, device=cuda_device) for k in ("x", "y", "heading", "speed")}
    mask = torch.ones(N, dtype=torch.uint8)
    with pytest.raises(RuntimeError):
        w.reset_sampled(mask, pool)
    w.set_reset_sampler(5, sample_rows=False)
    bound = w._sampler
    jit = np.zeros((M, 4, 2), np.float32)
    bad = [dict(tries=0), dict(tries=33), dict(jitter=np.zeros((M + 1, 4, 2))),
           dict(jitter=np.where(np.arange(8).reshape(1, 4, 2) % 2 == 0, 1.0, 0.0) + jit),
           dict(jitter=jit + np.nan), dict(target=np.zeros((2, 5))), dict(tile_id=np.zeros(2)),
           dict(route_id=np.zeros((2, M))), dict(type_id=np.full((2, M), 7))]
    for kw in bad:
        with pytest.raises(ValueError):
            w.set_reset_sampler(5, **kw)
        assert w._sampler is bound
    w.set_reset_sampler(5, type_id=np.zeros((2, M)), sample_rows=False)
    with pytest.raises(ValueError):   # the pool must have the row pools' rows
        w.reset_sampled(mask, pool)
    w.set_reset_sampler(5, sample_rows=False)
    with pytest.raises(ValueError):   # without row draws: one row per scenario
        w.reset_sampled(mask, {k: v[:2] for k, v in pool.items()})
    n0 = w.episode_count.clone()
    w.reset_sampled(mask, pool)
    torch.cuda.synchronize()
    assert (w.episode_count == n0 + 1).all()
    w.set_reset_sampler(None)
    assert w.pool_row is None
    with pytest.raises(RuntimeError):
        w.reset_sampled(mask, pool)
    w.close()


def test_unmasked_scenarios_keep_every_buffer_and_a_wheel_pool_is_kept(cuda_device):
    """Unmasked scenarios keep every world buffer the sampled reset writes (state, wheels, types, step counts, the tries);
    a moved drift slot keeps the wheel speeds a reset wheel pool gave it."""
    table, types = _tables()["drift"]
    N, M = 7, 9
    rng = np.random.default_rng(3)
    sc = _scene(rng, N, M, 12.0, table, types)
    w = BatchedWorld(N, M, table, device=cuda_device)
    w.set_state(sc["x"], sc["y"], sc["heading"], sc["speed"], type_id=sc["type_id"])
    w.step_count.fill_(5)
    jit = np.tile(np.array([[-1.0, 1.0], [-1.0, 1.0], [-0.2, 0.2], [0.0, 1.0]], np.float32), (M, 1, 1))
    w.set_reset_sampler(4, jitter=jit, tries=8, sample_rows=False)
    pool = _pool(sc, cuda_device)
    pool["omega_wf"] = torch.full((N, M), 3.5, device=cuda_device)
    pool["omega_wr"] = torch.full((N, M), 2.5, device=cuda_device)
    w.reset_sampled(torch.ones(N, dtype=torch.uint8), pool)
    w.step_count.fill_(5)
    mask = np.array([1, 0, 1, 0, 0, 1, 0], bool)
    keys = ("x", "y", "heading", "speed", "vx", "vy", "omega_front", "omega_rear", "type_id", "step_count", "reset_try")
    before = {k: getattr(w, k).cpu().numpy().copy() for k in keys}
    w.reset_sampled(torch.from_numpy(mask.astype(np.uint8)), pool)
    torch.cuda.synchronize()
    for k in keys:
        got = getattr(w, k).cpu().numpy()
        assert np.array_equal(got[~mask].view(np.uint8), before[k][~mask].view(np.uint8)), k
    rt = w.reset_try.cpu().numpy()
    moved = mask[:, None] & (rt >= 0)
    assert moved.any()
    assert (w.omega_front.cpu().numpy()[mask] == 3.5).all() and (w.omega_rear.cpu().numpy()[mask] == 2.5).all()
    assert (w.step_count.cpu().numpy()[mask] == 0).all()
    w.close()


def test_agents_retired_types_give_way_to_the_type_pool(cuda_device):
    table = TypeTable([TypeParams.vehicle("medium_car"), TypeParams.pedestrian()])
    N, M, P = 5, 4, 3
    w = BatchedWorld(N, M, table, device=cuda_device)
    w.set_state(np.zeros((N, M)), np.arange(N * M, dtype=np.float32).reshape(N, M) * 10, np.zeros((N, M)),
                np.zeros((N, M)), type_id=np.zeros((N, M), np.uint8))
    w.set_agents()
    w.retired_type[:, 1] = 0          # slot 1 of every scenario retired as a car ...
    w.type_id[:, 1] = 255
    pool_type = np.ones((P, M), np.uint8)   # ... while every pool row makes it a pedestrian
    w.set_reset_sampler(8, type_id=pool_type)
    pool = {k: torch.zeros((P, M), dtype=torch.float32, device=cuda_device) for k in ("x", "y", "heading", "speed")}
    mask = np.array([1, 0, 1, 1, 0], bool)
    w.reset_sampled(torch.from_numpy(mask.astype(np.uint8)), pool)
    torch.cuda.synchronize()
    tid, ret = w.type_id.cpu().numpy(), w.retired_type.cpu().numpy()
    assert (tid[mask] == 1).all() and (ret[mask] == 255).all()
    assert (tid[~mask, 1] == 255).all() and (ret[~mask, 1] == 0).all()
    w.close()


def test_a_log_replays_the_drawn_row_and_the_ego_avoids_its_traffic(cuda_device):
    from tactics2d_b200 import synthetic

    P, M, N = 9, 12, 6
    rep = synthetic.replay_episodes(P, M, 60, seed=13, size=60.0)
    sc = rep.scene()
    table = sc.table
    w = BatchedWorld(N, M, table, device=cuda_device)
    w.set_state(sc.x[:N], sc.y[:N], sc.heading[:N], sc.speed[:N], type_id=sc.type_id[:N])
    w.set_log(rep.log, rep.t0, **rep.binding())
    jit = np.zeros((M, 4, 2), np.float32)
    jit[0] = [[-6.0, 6.0], [-6.0, 6.0], [-0.5, 0.5], [0.0, 0.0]]
    seed = 21
    w.set_reset_sampler(seed, jitter=jit, tries=32)
    pool = {k: torch.from_numpy(np.ascontiguousarray(getattr(sc, k))).to(cuda_device) for k in ("x", "y", "heading", "speed")}
    mask = np.ones(N, bool)
    w.reset_sampled(torch.from_numpy(mask.astype(np.uint8)), pool)
    torch.cuda.synchronize()
    rows = R.pool_rows(mask, np.zeros(N, np.uint32), seed, P)
    assert np.array_equal(w.log_row.cpu().numpy(), rows) and np.array_equal(w.pool_row.cpu().numpy(), rows)
    # slot 0 from its pool row, the replayed slots as K7 left them: the oracle places the ego among them
    s = _snap(w)
    for k, v in (("x", sc.x), ("y", sc.y), ("heading", sc.heading), ("speed", sc.speed)):
        s[k][:, 0] = v[rows, 0]
    ctx = _ctx(table)
    ref, rt, _ = R.place(s, mask, np.zeros(N, np.uint32), seed, jit, 32, ctx["table"], ctx["n_types"],
                         lambda n: (None, None, None))
    for k in ("x", "y", "heading", "speed"):
        assert np.array_equal(_snap(w)[k].view(np.uint32), ref[k].view(np.uint32)), k
    assert np.array_equal(w.reset_try.cpu().numpy(), rt)
    fl = w.check_events().flags.cpu().numpy()
    assert (rt[:, 0] >= 0).all() and (fl[:, 0] == 0).all()
    w.close()


def _env(sc, seed, auto_reset=True, **kw):
    from tactics2d_b200.envs import BatchedTrafficEnv

    M = sc.shape[1]
    jit = np.tile(np.array([[-1.5, 1.5], [-1.5, 1.5], [-0.3, 0.3], [0.0, 0.5]], np.float32), (M, 1, 1))
    return BatchedTrafficEnv(sc, max_step=5, auto_reset=auto_reset, sampler=dict(seed=seed, jitter=jit, tries=8), **kw), jit


def test_env_rollouts_draw_every_episode(cuda_device):
    """Every reset and auto-reset of the env is the oracle's sampled reset of the state the tick left; the same seed
    reproduces every bit, another seed differs, and an unseeded reset keeps drawing."""
    from tactics2d_b200 import synthetic

    N, M = 33, 9
    sc = synthetic.config4(N, M, seed=17)
    (A, jit), (B, _), (C, _), (D, _) = _env(sc, 0), _env(sc, 0, auto_reset=False), _env(sc, 0), _env(sc, 1)
    ctx = _ctx(sc.table)
    pool = {k: np.ascontiguousarray(v) for k, v in sc.state().items()}
    scene_of = lambda n: (A.world.segments, A.world.bounds, None)
    keys = ("x", "y", "heading", "speed", "vx", "vy", "type_id", "step_count", "pool_row", "episode_count", "reset_try")
    grab = lambda e: {k: getattr(e.world, k).cpu().numpy().copy() for k in keys}

    def same(a, b, what):
        for k in keys:
            assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), f"{what}: {k}"

    for e in (A, B, C):
        e.reset(seed=0)
    D.reset(seed=1)
    same(grab(A), grab(B), "reset")
    same(grab(A), grab(C), "reset")
    assert not np.array_equal(grab(A)["x"], grab(D)["x"]), "another seed draws the same episodes"
    rng = np.random.default_rng(0)
    episodes = np.zeros(N, np.int64)
    for t in range(24):
        act = torch.from_numpy(rng.uniform(-1, 1, (N, 2)).astype(np.float32)).to(cuda_device)
        ra, rb, rc = A.step(act.clone()), B.step(act.clone()), C.step(act.clone())
        for i in (1, 2, 3):
            assert np.array_equal(ra[i].cpu().numpy(), rb[i].cpu().numpy()), f"step {t}: output {i}"
        assert np.array_equal(ra[4]["pool_row"].cpu().numpy(), A.world.pool_row.cpu().numpy())
        done = B.scenario_manager.env_result.done.cpu().numpy().astype(bool)
        post = _snap(B.world)
        pre_try = B.world.reset_try.cpu().numpy()
        ep = B.world.episode_count.cpu().numpy().view(np.uint32)
        want, pr, rt, ep2 = R.reset_sampled(post, done, pool, ctx, 0, ep, B.world.pool_row.cpu().numpy(), jitter=jit,
                                            tries=8, row_pools={"type_id": sc.type_id}, scene_of=scene_of)
        rt[~done] = pre_try[~done]
        got = grab(A)
        for k in ("x", "y", "heading", "speed", "type_id", "step_count"):
            assert np.array_equal(got[k].view(np.uint8), want[k].view(np.uint8)), f"step {t}: {k}"
        assert np.array_equal(got["pool_row"], pr) and np.array_equal(got["reset_try"], rt)
        assert np.array_equal(got["episode_count"].view(np.uint32), ep2)
        B.scenario_manager.reset(mask=B.scenario_manager.env_result.done, sample=True)
        same(got, grab(B), f"step {t}")
        same(got, grab(C), f"step {t} (same seed)")
        episodes += done
    assert episodes.min() >= 3
    ep = A.world.episode_count.cpu().numpy().view(np.uint32).copy()
    A.reset()
    assert np.array_equal(A.world.episode_count.cpu().numpy().view(np.uint32), ep + 1)
    assert np.array_equal(A.world.pool_row.cpu().numpy(), R.pool_rows(np.ones(N, bool), ep, 0, N))
    A.reset(seed=0)
    assert (A.world.episode_count.cpu().numpy() == 1).all()
    with pytest.raises(ValueError):
        A.reset(options={"shuffle": True})
    for e in (A, B, C, D):
        e.close()


def test_env_sampler_misuse_is_rejected(cuda_device):
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    sc = synthetic.config4(5, 4, seed=2)
    with pytest.raises(ValueError):
        BatchedTrafficEnv(sc, sampler=dict(seed=0, colour=1))
    rep = synthetic.replay_episodes(5, 4, 20, seed=1)
    jit = np.zeros((4, 4, 2), np.float32)
    jit[1] = [[-1, 1], [0, 0], [0, 0], [0, 0]]
    with pytest.raises(ValueError):
        BatchedTrafficEnv(None, replay=rep, sampler=dict(seed=0, jitter=jit))
    goals = torch.zeros((5, 1, 5), device=cuda_device)
    with pytest.raises(ValueError):
        BatchedTrafficEnv(sc, observation="agents", agent_rewards=True,
                          vector_obs=dict(observers=torch.zeros((5, 1), dtype=torch.int16, device=cuda_device), goals=goals),
                          sampler=dict(seed=0))


def test_rejected_tile_pool_after_a_smaller_map(cuda_device):
    table = TypeTable([TypeParams.vehicle("medium_car")])
    N, M = 3, 2
    w = BatchedWorld(N, M, table, device=cuda_device)
    w.set_state(np.zeros((N, M)), np.zeros((N, M)), np.zeros((N, M)), np.zeros((N, M)), type_id=np.zeros((N, M)))
    tile = lambda b: dict(segments=None, bounds=(-b, b, -b, b))
    w.set_map_table([tile(10), tile(20), tile(30)], np.zeros(N, np.int64))
    w.set_reset_sampler(1, tile_id=np.array([0, 2], np.int16))
    w.set_map_table([tile(10), tile(20)], np.zeros(N, np.int64))
    pool = {k: torch.zeros((2, M), dtype=torch.float32, device=cuda_device) for k in ("x", "y", "heading", "speed")}
    with pytest.raises(ValueError):
        w.reset_sampled(torch.ones(N, dtype=torch.uint8), pool)
    w.close()
