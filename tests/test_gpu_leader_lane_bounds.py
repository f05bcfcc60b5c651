"""K17 (the leader search) and K18 (MOBIL lane changes) held to exact answers where the random tests' robust filters look
away, and at the shapes and path tables the random tests never reach.

* The exact scenes of tests/exact_lane_scenes.py (every bound, tie, clamped projection and kinked corner; hand answers the
  CPU file tests/test_oracle_lane_bounds.py pins on the oracles): K17 through ``t2d_find_leaders`` and through a bound
  search inside ``control``, K18 inside ``control``, each against the hand answer and the oracle with no robustness mask.
* Every slot a warp lane owns (M up to 128) and a partial last CTA (N = 1, 2, 3 mod 4), with caller buffers that carry a
  guard tail and a sentinel: every slot of [N, M] is written and nothing past it (K18's lane_path is its input too, so
  there only the tail and the robust slots' values are observed).
* One distinct path per slot (up to 128 path walks per warp, more than 128 paths in the table), hairpins and quarter
  circles whose chord is short and whose arc is long.
* ``idm_law``'s exponent branches (delta = 2, its general pow()) and its ``dist == 0`` branch, in K5 and in K18."""

import ctypes as C
import math

import numpy as np
import pytest

from oracle import controllers as OC
from tests import exact_lane_scenes as E
from tests import lane_change_oracle as LC
from tests import leader_oracle as L

pytestmark = pytest.mark.gpu

HW, RNG = E.HW, E.RNG
TAIL = 64
LEAD_SENTINEL, GAP_SENTINEL = 0x7EAD, float("nan")   # no lead the kernel writes; gap is finite or +inf
I16_SENTINEL, I8_SENTINEL = 0x5A5A, 0x5A
SHAPES = [(1, 1), (5, 2), (7, 31), (13, 32), (1, 33), (5, 63), (7, 64), (13, 65), (2, 96), (3, 97), (6, 127), (7, 128)]


def _table():
    from tactics2d_b200.types import TypeParams, TypeTable

    car = TypeParams(half_len=2.4, half_wid=0.95, lf=1.3, lr=1.3, steer_lo=-0.6, steer_hi=0.6, speed_lo=0.0, speed_hi=40.0,
                     accel_lo=-8.0, accel_hi=4.0)
    ped = TypeParams(radius=0.4, model=2, shape=1, speed_hi=3.0)
    ghost = TypeParams(half_len=1.0, half_wid=1.0, shape=2)
    return TypeTable([car, ped, ghost])


SHAPE_IDS = [0, 1, 2]   # OBB, DISC, NONE


def _world(device, x, y, h, v, tid):
    from tactics2d_b200 import BatchedWorld

    n, m = x.shape
    w = BatchedWorld(n, m, _table(), device=device)
    w.set_state(x, y, h, v, type_id=tid)
    return w


def _np(t):
    return t.cpu().numpy()


# ================================================================================================ exact K17 cases
def test_exact_leader_cases(cuda_device):
    """Every case in its own scenario (N = 25: the last CTA holds one warp), M = 128; lead and gap bit for bit."""
    import torch

    cases = E.leader_cases()
    x, y, h, tid, pid = E.leader_batch(cases)
    n = len(cases)
    assert n % 4 == 1
    w = _world(cuda_device, x, y, h, np.full_like(x, 5.0), tid)
    w.set_paths(E.paths())
    w.set_controllers(E.controllers(), np.full(x.shape, 255, np.uint8), path_id=pid)
    ref = L.find(x, y, h, tid, [E.OBB], HW, RNG, pid, E.paths())
    lead, gap = (_np(t).copy() for t in w.find_leaders(HW, RNG))
    w.set_leader_search(HW, RNG)
    w.control(torch.zeros((n, E.M, 2), dtype=torch.float32, device=cuda_device))
    for got_lead, got_gap, how in ((lead, gap, "find_leaders"), (_np(w.leader), _np(w.leader_gap), "control")):
        wrong = [c["name"] for i, c in enumerate(cases)
                 if not (np.array_equal(got_lead[i], ref["lead"][i])
                         and np.array_equal(got_gap[i], ref["gap"][i].astype(np.float32))
                         and all((got_lead[i, s], got_gap[i, s]) == (l, np.float32(g)) for s, (l, g) in c["want"].items()))]
        assert not wrong, (how, wrong)
    # heading 0: the heading frame's gap is dx bit for bit (sincos_angle(0) is exactly (0, 1))
    i = [c["name"] for c in cases].index("heading_range_closed")
    assert gap[i, 0].view(np.uint32) == np.float32(RNG).view(np.uint32)


# ================================================================================================ exact K18 cases
def _lane_world(device, x, y, v, tid, cid, lane, cool, left, right, kw, paths, ctrls, hw=HW, rng=RNG):
    import torch

    w = _world(device, x, y, np.zeros_like(x), v, tid)
    w.set_paths(paths)
    w.set_controllers(ctrls, cid, path_id=lane)
    w.set_leader_search(hw, rng)
    w.set_lane_change(left, right, **kw)
    w.lane_cooldown.copy_(torch.from_numpy(np.asarray(cool, np.int16)).to(device))
    return w


def _decide(x, y, v, tid, cid, ctab, lane, cool, left, right, kw, paths, hw=HW, rng=RNG):
    return LC.decide(x, y, v, tid, SHAPE_IDS, cid, ctab, lane, cool, left, right, paths, hw, rng,
                     **{k: kw[k] for k in ("politeness", "threshold", "b_safe", "min_gap")}, cool_ticks=kw["cooldown"])


LANE_CASES = E.lane_cases()


@pytest.mark.parametrize("case", LANE_CASES, ids=[c["name"] for c in LANE_CASES])
def test_exact_lane_case(cuda_device, case):
    import torch

    x, y, v, tid, cid, lane, cool = E.lane_arrays(case)
    left, right = E.neighbours(case)
    w = _lane_world(cuda_device, x, y, v, tid, cid, lane, cool, left, right, case["kw"], E.paths(), E.controllers())
    w.lane_change.fill_(99)
    before = w.state_numpy()
    la = _np(w.last_accel)
    ps = _np(w.pid_state)
    act = _np(w.control(torch.zeros((1, E.M, 2), dtype=torch.float32, device=cuda_device)))
    ref = _decide(x, y, v, tid, cid, E.ctab(), lane, cool, left, right, case["kw"], E.paths())
    got = (_np(w.lane_path), _np(w.lane_cooldown), _np(w.lane_change))
    for g, k in zip(got, ("lane_path", "cooldown", "change")):
        assert np.array_equal(g, ref[k]), k
    for slot, want in case["want"].items():
        assert tuple(int(g[0, slot]) for g in got) == want, slot
    # K18 -> K17 -> K5 in the same call: the leaders are the search's on the lanes K18 just wrote, and K5 follows them
    lead = L.find(x, y, np.zeros_like(x), tid, [E.OBB], HW, RNG, got[0], E.paths())
    assert np.array_equal(_np(w.leader), lead["lead"])
    assert np.array_equal(_np(w.leader_gap), lead["gap"].astype(np.float32))
    tab = _table().as_oracle_table()
    want_act, _, _ = LC.control_tick(before, tid, tab, np.zeros((1, E.M, 2), np.float32), cid, E.ctab(), lead["lead"],
                                     got[0], E.paths(), la, ps)
    ctl = cid != 255
    np.testing.assert_allclose(act[ctl], want_act[ctl], rtol=3e-6, atol=3e-6)
    if case["name"] == "same_call_order":
        assert lead["lead"][0, 0] == 2 and lead["gap"][0, 0] == 40.0   # the car ahead on lane 1, not the one on lane 0


# ================================================================================================ shapes and guard tails
def _short_lanes():
    """Four lanes 3.5 m apart, -16 .. 144 m (segments of 32 and 64 m), a little shorter than the spread of the cars: some
    projections are clamped at either end; then a curved lane and one without a segment of non-zero length."""
    lanes = [np.array([[-16.0, 3.5 * l], [16.0, 3.5 * l], [48.0, 3.5 * l], [112.0, 3.5 * l], [144.0, 3.5 * l]])
             for l in range(4)]
    xs = np.linspace(-20.0, 150.0, 24)
    curve = np.stack([xs, 3.5 + 3.0 * np.sin(xs / 25.0)], 1)
    return [p.astype(np.float32) for p in lanes + [curve, np.array([[5.0, 5.0], [5.0, 5.0]])]]


def _shape_scene(n, m, seed):
    rng = np.random.default_rng(seed)
    lane = rng.integers(0, 4, (n, m))
    x = rng.uniform(-20.0, 150.0, (n, m))
    y = 3.5 * lane + rng.normal(0.0, 0.6, (n, m))
    h = rng.normal(0.0, 0.08, (n, m)) + np.where(rng.random((n, m)) < 0.1, math.pi, 0.0)
    v = rng.uniform(2.0, 16.0, (n, m))
    tid = rng.choice([0, 0, 0, 1, 2], size=(n, m)).astype(np.uint8)
    tid[rng.random((n, m)) < 0.1] = 255
    pid = np.where(rng.random((n, m)) < 0.8, lane, rng.integers(-1, 7, (n, m))).astype(np.int16)   # 5: no segment; 6: none
    cid = rng.choice([0, 0, 1, 2, 255], size=(n, m)).astype(np.uint8)
    cool = np.where(rng.random((n, m)) < 0.2, rng.integers(1, 4, (n, m)), 0).astype(np.int16)
    return [a.astype(np.float32) for a in (x, y, h, v)] + [tid, pid, cid, cool]


def _shape_ctrls():
    from tactics2d_b200.controller import IDMController, PIDController

    keep = PIDController(dt=0.1, kp_lat=0.03, ki_lat=0.0, kd_lat=0.08, max_steering=0.2, derivative_filter_alpha=1.0,
                         lateral_error="path_cross_track")
    return [IDMController(desired_speed=14.0, min_spacing=10.0, max_acceleration=2.0, comfortable_deceleration=5.0,
                          lateral=keep),
            IDMController(desired_speed=9.0, time_headway=1.2, lateral=keep, delta=2.0),
            IDMController(desired_speed=12.0)]


def _rows(ctrls):
    return [{k: getattr(r, k) for k, _ in r._fields_} for r in (c.params() for c in ctrls)]


def _guarded(n, m, dtype, fill, device):
    """A caller buffer of [N, M] and a guard tail, every element the sentinel."""
    import torch

    return torch.full((n * m + TAIL,), fill, dtype=dtype, device=device)


def _check_leaders(lead, gap, ref, min_robust):
    r = ref["robust"]
    assert r.mean() >= min_robust, r.mean()
    assert np.array_equal(lead[r], ref["lead"][r])
    path = r & (ref["lead"] >= 0) & (ref["frame"] == L.PATH)
    assert np.array_equal(gap[path], ref["gap"][path].astype(np.float32))
    head = r & (ref["lead"] >= 0) & (ref["frame"] == L.HEADING)
    want = ref["gap"][head]
    ulp = (np.nextafter(np.abs(want).astype(np.float32), np.float32(np.inf)) - np.abs(want).astype(np.float32))
    assert np.all(np.abs(gap[head].astype(np.float64) - want) <= ulp.astype(np.float64) + 1e-12 * (1.0 + want))
    assert np.all(gap[r & (ref["lead"] < 0)] == np.inf)


@pytest.mark.parametrize("n,m", SHAPES, ids=[f"n{n}-m{m}" for n, m in SHAPES])
def test_leaders_at_every_shape_write_every_slot_and_nothing_past(cuda_device, n, m):
    import torch

    x, y, h, v, tid, pid, cid, _ = _shape_scene(n, m, seed=1000 + 7 * m + n)
    w = _world(cuda_device, x, y, h, v, tid)
    w.set_paths(_short_lanes())
    w.set_controllers(_shape_ctrls(), cid, path_id=pid)
    lead = _guarded(n, m, torch.int16, LEAD_SENTINEL, cuda_device)
    gap = _guarded(n, m, torch.float32, GAP_SENTINEL, cuda_device)
    assert w.lib.t2d_find_leaders(w._ctx, HW, RNG, C.c_void_p(lead.data_ptr()), C.c_void_p(gap.data_ptr()),
                                  w._stream()) == 0
    torch.cuda.synchronize()
    lead, gap = _np(lead), _np(gap)
    assert (lead[n * m:] == LEAD_SENTINEL).all() and np.isnan(gap[n * m:]).all()
    lead, gap = lead[:n * m].reshape(n, m), gap[:n * m].reshape(n, m)
    assert not (lead == LEAD_SENTINEL).any() and not np.isnan(gap).any()
    ref = L.find(x, y, h, tid, SHAPE_IDS, HW, RNG, pid, _short_lanes())
    _check_leaders(lead, gap, ref, min_robust=0.9)
    # the bound search inside control writes the same
    w.set_leader_search(HW, RNG)
    w.control(torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device))
    assert np.array_equal(_np(w.leader), lead) and np.array_equal(_np(w.leader_gap), gap)
    if m >= 32:
        assert (ref["lead"] >= 0).mean() > 0.2


@pytest.mark.parametrize("n,m", SHAPES, ids=[f"n{n}-m{m}" for n, m in SHAPES])
def test_lane_changes_at_every_shape_write_every_slot_and_nothing_past(cuda_device, n, m):
    import torch

    from tactics2d_b200 import _lib

    x, y, h, v, tid, pid, cid, cool = _shape_scene(n, m, seed=2000 + 7 * m + n)
    kw = dict(politeness=0.3, threshold=0.1, b_safe=3.0, min_gap=7.0, cooldown=12)
    left, right = [1, 2, 3, -1, 2, -1], [-1, 0, 1, 2, 0, -1]
    w = _world(cuda_device, x, y, h, v, tid)
    w.set_paths(_short_lanes())
    ctrls = _shape_ctrls()
    w.set_controllers(ctrls, cid, path_id=pid)
    w.set_leader_search(HW, RNG)
    p = _lib.LaneChangeParamsC(**kw)
    nb = [np.ascontiguousarray(np.asarray(a, np.int16)) for a in (left, right)]
    lane_path = _guarded(n, m, torch.int16, I16_SENTINEL, cuda_device)
    cooldown = _guarded(n, m, torch.int16, I16_SENTINEL, cuda_device)
    change = _guarded(n, m, torch.int8, I8_SENTINEL, cuda_device)
    ptr = lambda t: C.c_void_p(t.data_ptr())
    try:
        assert w.lib.t2d_set_lane_change(w._ctx, C.byref(p), C.c_void_p(nb[0].ctypes.data), C.c_void_p(nb[1].ctypes.data),
                                         ptr(lane_path), ptr(cooldown), ptr(change)) == 0
        torch.cuda.synchronize()
        assert np.array_equal(_np(lane_path[:n * m]).reshape(n, m), pid)   # the binding copied path_id
        cooldown[:n * m].copy_(torch.from_numpy(cool.reshape(-1)).to(cuda_device))
        change[:n * m].fill_(99)
        ref = _decide(x, y, v, tid, cid, _rows(ctrls), pid, cool, left, right, kw, _short_lanes())
        w.control(torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device))
        torch.cuda.synchronize()
        out = [_np(t) for t in (lane_path, cooldown, change)]
        # lane_path is also K18's input, so an unchanged lane written back cannot be told from one left alone; a second
        # call with the cooldown sentinel in every slot has no changer, and must count every slot's cooldown down
        cooldown[:n * m].fill_(I16_SENTINEL)
        change[:n * m].fill_(99)
        w.control(torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device))
        torch.cuda.synchronize()
        again = [_np(t) for t in (lane_path, cooldown, change)]
    finally:
        w.lib.t2d_set_lane_change(w._ctx, None, None, None, None, None, None)
    for o, s in zip(out, (np.int16(I16_SENTINEL), np.int16(I16_SENTINEL), np.int8(I8_SENTINEL))):
        assert (o[n * m:] == s).all()
    got = [o[:n * m].reshape(n, m) for o in out]
    assert not (got[2] == 99).any()
    r = ref["robust"]
    assert r.mean() >= 0.9, r.mean()
    for g, k in zip(got, ("lane_path", "cooldown", "change")):
        assert np.array_equal(g[r], ref[k][r]), k
    if m >= 32:
        assert ref["changer"].sum() > 0
    assert np.array_equal(again[0], out[0])
    assert (again[1][:n * m] == I16_SENTINEL - 1).all() and (again[1][n * m:] == np.int16(I16_SENTINEL)).all()
    assert (again[2][:n * m] == 0).all() and (again[2][n * m:] == np.int8(I8_SENTINEL)).all()


# ================================================================================================ many distinct paths
FAMILIES = 3


def _hairpin(y0):
    """Out along y0 to x = 100, a half turn of radius 4 and back along y0 + 8: 20 vertices."""
    a = np.linspace(-math.pi / 2, math.pi / 2, 16)
    turn = np.stack([100.0 + 4.0 * np.cos(a), y0 + 4.0 + 4.0 * np.sin(a)], 1)
    return np.concatenate([[[-40.0, y0]], turn, [[60.0, y0 + 8.0], [20.0, y0 + 8.0], [-40.0, y0 + 8.0]]], 0)


def _quarter(y0, radius=46.0):
    """A quarter circle that leaves y0 along +x at x = 0 and turns left: 24 vertices, chord ~ 0.91 arc over 66 m."""
    a = np.linspace(0.0, math.pi / 2, 23)
    arc = np.stack([radius * np.sin(a), y0 + radius * (1.0 - np.cos(a))], 1)
    return np.concatenate([[[-40.0, y0]], arc], 0)


def _many_paths(seed, count=160):
    """``count`` distinct paths of 16 - 32 vertices in three lane families (y = 0, 3.5, 7): jittered lanes, a hairpin
    every 20 paths and a quarter circle every 20, and each path's left / right neighbour in the other two families."""
    rng = np.random.default_rng(seed)
    out, fam = [], []
    for k in range(count):
        f = k % FAMILIES
        y0 = 3.5 * f
        if k % 20 == 7:
            p = _hairpin(y0)
        elif k % 20 == 13:
            p = _quarter(y0)
        else:
            nv = 16 + (k * 7) % 17
            xs = np.sort(np.concatenate([[-40.0, 200.0], rng.uniform(-40.0, 200.0, nv - 2)]))
            p = np.stack([xs, y0 + rng.normal(0.0, 0.25, nv)], 1)
        assert 16 <= len(p) <= 32
        out.append(p.astype(np.float32))
        fam.append(f)
    fam = np.array(fam)
    left = [int(rng.choice(np.nonzero(fam == (f + 1) % FAMILIES)[0])) for f in fam]
    right = [int(rng.choice(np.nonzero(fam == (f + 2) % FAMILIES)[0])) for f in fam]
    return out, fam, left, right


def _point_on(path, rng):
    """A point near a random spot of the path (within about a metre of it)."""
    i = rng.integers(0, len(path) - 1)
    t = rng.random()
    p = path[i] + t * (path[i + 1] - path[i])
    return p + rng.normal(0.0, 0.5, 2)


def _many_scene(n, m, seed, paths, fam):
    """Every slot of a scenario on its own path (128 distinct ids of the table, another set per scenario)."""
    rng = np.random.default_rng(seed)
    P = len(paths)
    x, y, h, v = (np.zeros((n, m)) for _ in range(4))
    pid = np.zeros((n, m), np.int16)
    for i in range(n):
        ids = rng.permutation(P)[:m]
        pid[i] = ids
        for j in range(m):
            x[i, j], y[i, j] = _point_on(paths[ids[j]].astype(np.float64), rng)
    h[:] = rng.normal(0.0, 0.05, (n, m))
    v[:] = rng.uniform(2.0, 16.0, (n, m))
    tid = rng.choice([0, 0, 0, 0, 1, 2], size=(n, m)).astype(np.uint8)
    tid[rng.random((n, m)) < 0.05] = 255
    cid = rng.choice([0, 0, 0, 1, 2], size=(n, m)).astype(np.uint8)
    cool = np.where(rng.random((n, m)) < 0.1, 2, 0).astype(np.int16)
    return [a.astype(np.float32) for a in (x, y, h, v)] + [tid, pid, cid, cool]


def test_leaders_with_a_distinct_path_per_slot(cuda_device):
    import torch

    paths, fam, _, _ = _many_paths(5)
    n, m = 5, 128
    x, y, h, v, tid, pid, cid, _ = _many_scene(n, m, 6, paths, fam)
    assert all(len(set(pid[i].tolist())) == m for i in range(n)) and len(paths) > 128
    w = _world(cuda_device, x, y, h, v, tid)
    w.set_paths(paths)
    w.set_controllers(_shape_ctrls(), cid, path_id=pid)
    lead, gap = (_np(t).copy() for t in w.find_leaders(HW, RNG))
    ref = L.find(x, y, h, tid, SHAPE_IDS, HW, RNG, pid, paths)
    _check_leaders(lead, gap, ref, min_robust=0.98)
    assert (ref["frame"][tid < 3] == L.PATH).all()
    assert (ref["lead"] >= 0).mean() > 0.3
    w.set_leader_search(HW, RNG)
    w.control(torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device))
    assert np.array_equal(_np(w.leader), lead) and np.array_equal(_np(w.leader_gap), gap)


def _arc_case(path, s_follower, s_cand):
    """Positions on ``path`` at two arc lengths (the first vertex's offset subtracted by the caller)."""
    path = np.asarray(path, np.float64)
    seg = np.hypot(*(path[1:] - path[:-1]).T)
    cum = np.concatenate([[0.0], np.cumsum(seg)])

    def at(s):
        i = min(np.searchsorted(cum, s, side="right") - 1, len(seg) - 1)
        return path[i] + (s - cum[i]) / seg[i] * (path[i + 1] - path[i])

    return at(s_follower), at(s_cand)


def test_chord_inside_range_arc_beyond_it(cuda_device):
    """On a hairpin and a quarter circle a candidate closer than max_range in a straight line but farther along the path
    is not the leader; one just inside max_range along the path is."""
    hair, quarter = _hairpin(0.0).astype(np.float32), _quarter(0.0).astype(np.float32)
    pts, pid = [], []
    for k, path in enumerate((hair, quarter)):
        for s_cand in (RNG + 2.0, RNG - 2.0):
            f, c = _arc_case(path, 40.0 if k == 1 else 120.0, (40.0 if k == 1 else 120.0) + s_cand)
            assert np.hypot(*(c - f)) < RNG
            pts.append((f, c))
            pid.append(k)
    n, m = len(pts), 2
    x = np.array([[p[0][0], p[1][0]] for p in pts], np.float32)
    y = np.array([[p[0][1], p[1][1]] for p in pts], np.float32)
    path_id = np.array([[p, -1] for p in pid], np.int16)
    tid = np.zeros((n, m), np.uint8)
    w = _world(cuda_device, x, y, np.zeros_like(x), np.full_like(x, 5.0), tid)
    w.set_paths([hair, quarter])
    w.set_controllers(_shape_ctrls(), np.full((n, m), 255, np.uint8), path_id=path_id)
    lead, gap = (_np(t) for t in w.find_leaders(HW, RNG))
    ref = L.find(x, y, np.zeros_like(x), tid, SHAPE_IDS, HW, RNG, path_id, [hair, quarter])
    assert ref["robust"][:, 0].all()
    assert ref["lead"][:, 0].tolist() == [-1, 1, -1, 1]
    assert np.array_equal(lead[:, 0], ref["lead"][:, 0])
    assert np.array_equal(gap[:, 0], ref["gap"][:, 0].astype(np.float32))


def test_lane_changes_with_three_distinct_paths_per_changer(cuda_device):
    import torch

    paths, fam, left, right = _many_paths(7)
    n, m = 3, 128
    x, y, h, v, tid, pid, cid, cool = _many_scene(n, m, 8, paths, fam)
    assert all(len({int(p), left[p], right[p]}) == 3 for p in range(len(paths)))
    kw = dict(politeness=0.3, threshold=0.1, b_safe=3.0, min_gap=7.0, cooldown=12)
    ctrls = _shape_ctrls()
    w = _lane_world(cuda_device, x, y, v, tid, cid, pid, cool, left, right, kw, paths, ctrls)
    w.lane_change.fill_(99)
    ref = _decide(x, y, v, tid, cid, _rows(ctrls), pid, cool, left, right, kw, paths)
    w.control(torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device))
    r = ref["robust"]
    assert r.mean() >= 0.98, r.mean()
    for t, k in ((w.lane_path, "lane_path"), (w.lane_cooldown, "cooldown"), (w.lane_change, "change")):
        assert np.array_equal(_np(t)[r], ref[k][r]), k
    assert ref["changer"].sum() > 50 and (ref["change"] != 0).sum() > 0


# ================================================================================================ idm_law's exponents
def _idm_ctrls(lateral=False):
    from tactics2d_b200.controller import IDMController, PIDController

    keep = PIDController(dt=0.1, kp_lat=0.03, ki_lat=0.0, kd_lat=0.08, max_steering=0.2, derivative_filter_alpha=1.0,
                         lateral_error="path_cross_track") if lateral else None
    return [IDMController(desired_speed=11.0, min_spacing=6.0, max_acceleration=2.0, comfortable_deceleration=5.0,
                          delta=2.0, lateral=keep),
            IDMController(desired_speed=9.0, time_headway=1.2, comfortable_deceleration=4.0, delta=3.0, lateral=keep),
            IDMController(desired_speed=13.0, min_spacing=8.0, max_acceleration=1.5, delta=4.5, lateral=keep),
            IDMController(desired_speed=10.0, min_spacing=0.0, comfortable_deceleration=3.5, delta=2.0, lateral=keep)]


@pytest.mark.parametrize("search", [False, True], ids=["lead_index", "search"])
def test_idm_exponents_match_the_oracle(cuda_device, search):
    """K5 with delta = 2 (the fast path) and 3, 4.5 (pow), free and following; through lead_index, a leader at the
    follower's exact position gives -b.  Slots 0, 2, 4 reach -b through the clip as well (s* / 0 = inf); slot 6 (row 3:
    min_spacing 0, standing still, so s* = 0) gets NaN from 0 / 0 unless the dist == 0 branch returns -b."""
    import torch

    n, m = 9, 64
    x, y, h, v, tid, pid, _, _ = _shape_scene(n, m, seed=77)
    rng = np.random.default_rng(78)
    cid = rng.choice([0, 1, 2, 255], size=(n, m)).astype(np.uint8)
    v = (v * rng.uniform(0.5, 1.6, (n, m))).astype(np.float32)   # free flow both below and above the desired speed
    tid[:, :8] = 0
    cid[:, :8] = [0, 255, 1, 255, 2, 255, 3, 1]
    v[:, 6] = 0.0
    lead = np.where(rng.random((n, m)) < 0.3, -1, rng.integers(0, m, (n, m))).astype(np.int16)
    for j in (0, 2, 4, 6):   # slots 0, 2, 4, 6 follow slots 1, 3, 5, 7 at exactly their position
        x[:, j + 1], y[:, j + 1] = x[:, j], y[:, j]
        lead[:, j] = j + 1
    ctrls = _idm_ctrls()
    rows = _rows(ctrls)
    w = _world(cuda_device, x, y, h, v, tid)
    w.set_paths(_short_lanes())
    w.set_controllers(ctrls, cid, lead_index=lead, path_id=pid)
    if search:
        w.set_leader_search(HW, RNG)
    act = _np(w.control(torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device)))
    used = _np(w.leader) if search else lead
    tid_o = np.where(tid < 3, tid, 255)
    want, _ = OC.control_tick(w.state_numpy(), tid_o, _table().as_oracle_table(), np.zeros((n, m, 2), np.float32), cid,
                              rows, used, pid, [p.astype(np.float64) for p in _short_lanes()], np.zeros((n, m)))
    ctl = (cid != 255) & (tid < 3)
    np.testing.assert_allclose(act[ctl, 0], want[ctl, 0], rtol=3e-6, atol=3e-6)
    for d in (2.0, 3.0, 4.5):   # every exponent ran, free and following
        rows_d = np.isin(cid, [i for i, r in enumerate(rows) if r["delta"] == d]) & ctl
        assert (rows_d & (used >= 0)).sum() > 0 and (rows_d & (used < 0)).sum() > 0, d
    if search:   # the search's leaders, exact on every robust follower
        ref = L.find(x, y, h, tid, SHAPE_IDS, HW, RNG, pid, _short_lanes())
        assert np.array_equal(used[ref["robust"]], ref["lead"][ref["robust"]])
    else:
        for j in (0, 2, 4, 6):
            b = rows[int(cid[0, j])]["comfortable_deceleration"]
            assert (act[:, j, 0] == np.float32(-b)).all(), j


def test_lane_changes_with_idm_exponents(cuda_device):
    """K18's predicted accelerations with delta = 2, 3 and 4.5 rows against the oracle's."""
    import torch

    n, m = 7, 96
    x, y, h, v, tid, pid, _, cool = _shape_scene(n, m, seed=91)
    cid = np.random.default_rng(92).choice([0, 1, 2, 255], size=(n, m)).astype(np.uint8)
    kw = dict(politeness=0.5, threshold=0.05, b_safe=3.0, min_gap=6.0, cooldown=7)
    left, right = [1, 2, 3, -1, 2, -1], [-1, 0, 1, 2, 0, -1]
    ctrls = _idm_ctrls(lateral=True)
    w = _lane_world(cuda_device, x, y, v, tid, cid, pid, cool, left, right, kw, _short_lanes(), ctrls)
    w.lane_change.fill_(99)
    ref = _decide(x, y, v, tid, cid, _rows(ctrls), pid, cool, left, right, kw, _short_lanes())
    w.control(torch.zeros((n, m, 2), dtype=torch.float32, device=cuda_device))
    r = ref["robust"]
    assert r.mean() >= 0.9, r.mean()
    for t, k in ((w.lane_path, "lane_path"), (w.lane_cooldown, "cooldown"), (w.lane_change, "change")):
        assert np.array_equal(_np(t)[r], ref[k][r]), k
    moved = {int(cid[d["n"], d["slot"]]) for d in ref["decisions"]}
    assert ref["changer"].sum() > 0 and len(moved) >= 2
