"""The C2-shaped tick's x sort starts from the slot order each scenario had after its previous tick (the world's [N][64]
order hint), repairs it with two odd-even transposition passes and keeps it only if it is strictly ascending in every
scenario of the warp; otherwise the warp runs the sort network.  Either way the sorted list is the same, so every case
ticks a world that takes the C2-shaped instance next to one kept on the generic instance (T2D_TICK_GENERIC=1 at its
creation) and compares state and outputs bit for bit after every tick.  `t2d_tick_order_fallback_count` (warp tiles
that took the network) shows which path each case drove: a fresh world's identity hint, the bench's restore every 8
ticks, shuffled slots, empty and non-solid slots, a scene too fast for two passes, a hint overwritten with duplicates or
garbage, a world switching between the instances, odd batch sizes and a persistent launch."""

import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

STATE = ("x", "y", "heading", "speed", "vx", "vy")
OUTPUTS = ("flags", "hit_index", "hit_segment", "status", "done")


def _world(sc, device, monkeypatch, generic, interval=100):
    from tactics2d_b200 import BatchedWorld

    n, m = sc.shape
    with monkeypatch.context() as mp:
        if generic:
            mp.setenv("T2D_TICK_GENERIC", "1")
        w = BatchedWorld(n, m, sc.table, device=device, interval=interval, max_step=7)
    w.set_map(sc.segments, sc.bounds)
    w.set_state(sc.x, sc.y, sc.heading, sc.speed, type_id=sc.type_id)
    return w


def _hint(w, write=None):
    """The world's order hint as [N, 64] uint8; `write` ([N, 64] uint8) replaces it after the read."""
    from tactics2d_b200 import _lib

    got = np.zeros((w.N, 64), np.uint8)
    src = None if write is None else np.ascontiguousarray(write, np.uint8)
    _lib.check(w.lib.t2d_order_hint(w._ctx, got.ctypes.data, None if src is None else src.ctypes.data))
    return got


def _sorted_slots(w, solid):
    """The slots of every scenario in the order of the tick's sort keys: f2ord(x) with the low 7 bits replaced by the
    slot, non-solid slots last."""
    x = w.state_numpy()["x"].astype(np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    o = np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000)
    slot = np.arange(x.shape[1], dtype=np.uint64)[None, :]
    key = np.where(solid & ~np.isnan(x), o & ~np.uint64(127), np.uint64(0xFFFFFF80)) | slot
    return np.argsort(key, axis=1).astype(np.uint8)


class Pair:
    """A C2-shaped world `a` and a generic world `b` on the same scene; `tick` steps both and compares them."""

    def __init__(self, sc, device, monkeypatch, **kw):
        from tactics2d_b200 import _lib

        self.lib = _lib.load()
        self.sc = sc
        self.a = _world(sc, device, monkeypatch, False, **kw)
        self.b = _world(sc, device, monkeypatch, True, **kw)
        self.device = device
        self.tiles = (sc.shape[0] + 1) // 2
        self.fixed = 0

    def tick(self, seed, scale=1.0):
        """One tick of both worlds; returns the warp tiles of `a`'s tick that fell back to the network."""
        import torch

        from tactics2d_b200 import synthetic

        act = torch.from_numpy(synthetic.random_actions(seed, self.sc.shape) * np.float32(scale)).to(self.device)
        torch.cuda.synchronize()
        f0, c0 = self.lib.t2d_tick_order_fallback_count(), self.lib.t2d_tick_fixed_count()
        ra = self.a.step(act)
        torch.cuda.synchronize()
        fell = self.lib.t2d_tick_order_fallback_count() - f0
        self.fixed += self.lib.t2d_tick_fixed_count() - c0
        rb = self.b.step(act)
        torch.cuda.synchronize()
        sa, sb = self.a.state_numpy(), self.b.state_numpy()
        for k in STATE:
            assert np.array_equal(sa[k].view(np.uint32), sb[k].view(np.uint32)), (seed, k)
        for k in OUTPUTS:
            assert np.array_equal(getattr(ra, k).cpu().numpy(), getattr(rb, k).cpu().numpy()), (seed, k)
        assert 0 <= fell <= self.tiles
        return fell

    def close(self):
        self.a.close()
        self.b.close()


@pytest.fixture
def pair(cuda_device, monkeypatch):
    made = []

    def make(sc, **kw):
        p = Pair(sc, cuda_device, monkeypatch, **kw)
        made.append(p)
        return p

    yield make
    for p in made:
        p.close()


def _c2(n, seed=31, **kw):
    from tactics2d_b200 import synthetic

    return synthetic.config2(n, 64, seed=seed, **kw)


def test_fresh_world_falls_back_then_repairs(pair):
    """t2d_create fills the hint with the identity, which the C2 scene's x order is not: the first tick falls back in
    every warp, and from then on nearly every warp keeps the repaired order.  After each tick the hint holds every
    scenario's slots in sort-key order."""
    p = pair(_c2(1024))
    solid = np.ones(p.sc.shape, bool)
    assert (_hint(p.a) == np.arange(64, dtype=np.uint8)[None, :]).all()
    fell = [p.tick(100 + t) for t in range(10)]
    assert fell[0] == p.tiles, fell
    assert sum(fell[1:]) < 0.05 * 9 * p.tiles, fell
    assert np.array_equal(_hint(p.a), _sorted_slots(p.a, solid))
    assert p.fixed == 10


def test_bench_pattern_restore_every_eight_ticks(pair):
    """8 ticks, a restore of the configured state (the hint stays as the 8th tick left it), 8 ticks: the order after
    the restore is 8 ticks stale and most warps fall back once, then repair again."""
    import torch

    sc = _c2(4096, seed=1)
    p = pair(sc)
    pools = [{k: getattr(w, k).clone() for k in ("x", "y", "heading", "speed", "vx", "vy")} for w in (p.a, p.b)]
    ones = torch.ones(sc.shape[0], dtype=torch.uint8, device=p.device)
    fell = []
    for rnd in range(2):
        for w, pool in zip((p.a, p.b), pools):
            w.reset(ones, pool)
        fell.append([p.tick(9000 + t) for t in range(8)])
    assert fell[0][0] == p.tiles                   # identity hint
    assert fell[1][0] > p.tiles // 2, fell         # 8 ticks stale
    assert sum(fell[0][1:]) + sum(fell[1][1:]) < 0.05 * 14 * p.tiles, fell
    assert p.fixed == 16


def test_shuffled_slots_and_shuffled_hint(pair):
    """Every scenario's slots in a random order, then a hint that is a random permutation of each scenario's slots:
    both make the next tick fall back in (nearly) every warp, and the tick after it repairs."""
    sc = _c2(512, seed=32)
    perm = np.argsort(np.random.default_rng(32).random(sc.shape), axis=1)
    take = lambda v: np.ascontiguousarray(np.take_along_axis(v, perm, axis=1))
    sc = dataclasses.replace(sc, x=take(sc.x), y=take(sc.y), heading=take(sc.heading), speed=take(sc.speed),
                             vx=take(sc.vx), vy=take(sc.vy), type_id=take(sc.type_id))
    p = pair(sc)
    assert p.tick(200) == p.tiles
    assert p.tick(201) < 0.05 * p.tiles
    _hint(p.a, np.argsort(np.random.default_rng(33).random((512, 64)), axis=1))
    assert p.tick(202) >= 0.95 * p.tiles
    assert p.tick(203) < 0.05 * p.tiles
    for t in range(204, 210):
        p.tick(t)


def test_empty_and_non_solid_slots(pair):
    """A quarter of the slots inactive and a fifth of the rest of a type without a collision shape: their keys sort
    last, in slot order, on both paths.  The scene is dense (about 3.4 m between vehicles), so the x order changes more
    than at C2 and a larger share of the warps falls back, but most keep the repaired order."""
    from tactics2d_b200 import synthetic
    from tactics2d_b200.types import SHAPE_NONE, TypeTable

    sc = synthetic.with_inactive(_c2(600, seed=34, size=3.4 * 8.0), 0.25, seed=34)
    rows = list(sc.table.rows)
    table = TypeTable(rows + [dataclasses.replace(rows[0], shape=SHAPE_NONE, name="ghost")])
    tid = sc.type_id.copy()
    ghost = (np.random.default_rng(35).random(tid.shape) < 0.2) & (tid != 255)
    tid[ghost] = len(rows)
    sc = dataclasses.replace(sc, table=table, type_id=tid)
    p = pair(sc)
    fell = [p.tick(300 + t) for t in range(10)]
    assert fell[0] == p.tiles
    assert sum(fell[1:]) < 0.6 * 9 * p.tiles, fell
    assert np.array_equal(_hint(p.a), _sorted_slots(p.a, (tid != 255) & ~ghost))


def test_fast_scene_outruns_two_passes(pair):
    """64 participants on a 32 m square at up to 40 m/s in every direction, over 1 s ticks: the x order changes too
    much for two passes, and most warps take the network on every tick."""
    sc = _c2(256, seed=36, size=32.0)
    rng = np.random.default_rng(36)
    sc = dataclasses.replace(sc, speed=rng.uniform(0.0, 40.0, sc.shape).astype(np.float32),
                             heading=rng.uniform(-np.pi, np.pi, sc.shape).astype(np.float32))
    p = pair(sc, interval=1000)
    fell = [p.tick(400 + t, scale=3.0) for t in range(10)]
    assert min(fell[1:4]) > 0.5 * p.tiles, fell


@pytest.mark.parametrize("garbage", ["duplicates", "random_bytes"])
def test_corrupt_hint(pair, garbage):
    """A hint that names one slot twice (and so misses another), or arbitrary bytes: the strict-ascent check rejects
    it in every scenario that holds it, and those warps fall back."""
    p = pair(_c2(1000, seed=37))
    for t in range(3):
        p.tick(500 + t)
    h = _hint(p.a)
    rng = np.random.default_rng(38)
    if garbage == "duplicates":
        bad = h.copy()
        bad[:, 1] = bad[:, 0]               # slot bad[:, 0] twice, the old bad[:, 1] never
        bad[1::2] = h[1::2]                 # odd scenarios keep theirs: only the even ones fail
        _hint(p.a, bad)
        assert p.tick(503) == p.tiles       # every warp holds an even scenario
    else:
        _hint(p.a, rng.integers(0, 256, h.shape, dtype=np.uint8))
        assert p.tick(503) == p.tiles
    assert p.tick(504) < 0.05 * p.tiles
    assert np.array_equal(_hint(p.a), _sorted_slots(p.a, np.ones(p.sc.shape, bool)))


def test_switching_between_instances(pair):
    """Binding an ego action puts the world on the generic instance, which leaves the hint alone; unbinding it
    returns to the C2-shaped instance, whose sort starts from the hint left before the switch."""
    import torch

    p = pair(_c2(800, seed=39))
    n = p.sc.shape[0]
    for t in range(3):
        p.tick(600 + t)
    before = _hint(p.a)
    ego = torch.zeros(n, 2, dtype=torch.float32, device=p.device)
    for w in (p.a, p.b):
        w.set_ego_action(ego)
    c0 = p.fixed
    for t in range(3):
        assert p.tick(603 + t) == 0
    assert p.fixed == c0
    assert np.array_equal(_hint(p.a), before)
    for w in (p.a, p.b):
        w.set_ego_action(None)
    fell = [p.tick(606 + t) for t in range(4)]
    assert p.fixed == c0 + 4
    assert sum(fell[1:]) < 0.05 * 3 * p.tiles, fell


@pytest.mark.parametrize("n", [1, 3, 4097])
def test_odd_batch_sizes(pair, n):
    """A last warp tile with one scenario and an empty group (whose keys are the identity's, all non-solid)."""
    p = pair(_c2(n, seed=40))
    fell = [p.tick(700 + t) for t in range(10)]
    assert fell[0] == p.tiles
    assert min(fell[1:]) < p.tiles, fell             # the repaired order was kept
    assert n < 4 or sum(fell[1:]) < 0.05 * 9 * p.tiles, fell
    assert p.fixed == 10


def test_persistent_launch(pair, monkeypatch):
    """T2D_GRID_LIMIT=1: one CTA per SM, so every warp takes several tiles, each with its own hint."""
    monkeypatch.setenv("T2D_GRID_LIMIT", "1")
    p = pair(_c2(4097, seed=41))
    monkeypatch.delenv("T2D_GRID_LIMIT")
    fell = [p.tick(800 + t) for t in range(10)]
    assert fell[0] == p.tiles
    assert sum(fell[1:]) < 0.05 * 9 * p.tiles, fell
    assert p.fixed == 10
