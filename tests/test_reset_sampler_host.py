"""The sampled-reset arithmetic without a GPU: Philox4x32-10 and the row / jitter draws of t2d_math.cuh (g++ build of
tests/samplersim) against the Python restatement, the known-answer vectors, the row histogram, and the placement of
tests/reset_sampler_oracle.py on hand-built scenes."""

import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
from scipy import stats

from tactics2d_b200 import TypeParams, TypeTable
from tests import reset_sampler_oracle as R

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def sim():
    """g++ build of tests/samplersim (into a temporary directory: the tree may be read-only)."""
    out = os.path.join(tempfile.mkdtemp(prefix="samplersim"), "samplersim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", out,
                           os.path.join(HERE, "samplersim", "samplersim.cpp")])
    return C.CDLL(out)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


# Random123's kat_vectors for philox4x32_10: (counter, key, output)
KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_known_answers(ctr, key, want, sim):
    assert tuple(int(v) for v in R.philox(*ctr, *key)) == want
    # the header: counter (d, n, e, 0) only reaches c3 = 0; the zero vector is the seed-0 draw 0 of scenario 0, episode 0
    if ctr[3] == 0:
        seed = key[0] | (key[1] << 32)
        out = np.zeros(4, np.uint32)
        sim.ss_draw(1, C.c_uint64(seed), _p(np.array([ctr[0]], np.uint32)), _p(np.array([ctr[1]], np.uint32)),
                    _p(np.array([ctr[2]], np.uint32)), _p(out))
        assert tuple(int(v) for v in out) == want


def test_header_philox_equals_the_restatement(sim):
    rng = np.random.default_rng(0)
    n = 100_000
    d, s, e = (rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32) for _ in range(3))
    for seed in (0, 1, 0xDEADBEEFCAFEF00D):
        out = np.zeros((n, 4), np.uint32)
        sim.ss_draw(n, C.c_uint64(seed), _p(d), _p(s), _p(e), _p(out))
        ref = np.stack(R.draw(seed, d, s, e), 1)
        assert np.array_equal(out, ref)


def test_row_draw_and_ranges_are_exact(sim):
    rng = np.random.default_rng(1)
    n = 100_000
    u = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    u[:2] = (0, 0xFFFFFFFF)
    for P in (1, 2, 7, 4099, 2 ** 31 - 1):
        out = np.zeros(n, np.int32)
        sim.ss_row(n, _p(u), P, _p(out))
        ref = ((u.astype(np.uint64) * np.uint64(P)) >> np.uint64(32)).astype(np.int64)
        assert np.array_equal(out, ref) and out.min() >= 0 and out.max() < P
    assert R.unit(np.uint32(0)) == 0.0 and R.unit(np.uint32(0xFFFFFFFF)) == np.float32(1 - 2.0 ** -24)
    lo = rng.uniform(-50, 50, n).astype(np.float32)
    hi = (lo + rng.uniform(0, 10, n)).astype(np.float32)
    got = np.zeros(n, np.float32)
    sim.ss_range(n, _p(u), _p(lo), _p(hi), _p(got))
    ref = R.draw_range(u, lo, hi)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    assert ((got >= lo) & (got <= hi)).all()
    assert got[0] == lo[0]
    # the upper bound is reached where the last step rounds up
    assert R.draw_range(np.uint32(0xFFFFFFFF), np.float32(1000.0), np.float32(1001.0)) == np.float32(1001.0)


def test_candidates_equal_the_restatement(sim):
    rng = np.random.default_rng(2)
    n = 20_000
    st = np.stack([rng.uniform(-300, 300, n), rng.uniform(-300, 300, n), rng.uniform(-20, 20, n),
                   rng.uniform(-5, 20, n)], 1).astype(np.float32)
    st[:50, 2] = rng.uniform(-1e4, 1e4, 50)   # wrap far from [0, 2 pi)
    u = rng.integers(0, 2 ** 32, (n, 4), dtype=np.uint64).astype(np.uint32)
    lo = rng.uniform(-3, 0, (n, 4)).astype(np.float32)
    jit = np.stack([lo, (lo + rng.uniform(0, 6, (n, 4))).astype(np.float32)], 2).reshape(n, 8)
    got = np.zeros((n, 4), np.float32)
    sim.ss_candidate(n, _p(st), _p(u), _p(jit), _p(got))
    f32 = np.float32
    ref = np.stack([(st[:, 0] + R.draw_range(u[:, 0], jit[:, 0], jit[:, 1])).astype(f32),
                    (st[:, 1] + R.draw_range(u[:, 1], jit[:, 2], jit[:, 3])).astype(f32),
                    R.wrap_two_pi((st[:, 2] + R.draw_range(u[:, 2], jit[:, 4], jit[:, 5])).astype(f32)),
                    (st[:, 3] + R.draw_range(u[:, 3], jit[:, 6], jit[:, 7])).astype(f32)], 1)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    assert ((got[:, 2] >= 0) & (got[:, 2] < np.float32(2 * np.pi) + 1e-6)).all()


def test_row_histogram_is_uniform():
    P, n = 97, 1_000_000
    rows = R.row_draw(12345, np.arange(n) % 4099, np.arange(n) // 4099, P)
    chi2, p = stats.chisquare(np.bincount(rows, minlength=P))
    assert p > 1e-4, (chi2, p)


# ---------------------------------------------------------------- placement on hand-built scenes (the oracle itself)
CAR = TypeParams.vehicle("medium_car")
PED = TypeParams.pedestrian()


def _world(xs, ys, types):
    f = lambda a: np.asarray(a, np.float32)[None]
    return dict(x=f(xs), y=f(ys), heading=f(np.zeros(len(xs))), speed=f(np.zeros(len(xs))), vx=f(np.zeros(len(xs))),
                vy=f(np.zeros(len(xs))), type_id=np.asarray(types, np.uint8)[None])


def _place(snap, table, jit, tries, segs=None, bounds=None, ps=None, target=None, avoid=False, seed=3):
    M = snap["x"].shape[1]
    j = np.zeros((M, 4, 2), np.float32)
    j[0] = jit
    return R.place(snap, np.ones(1, bool), np.zeros(1, np.uint32), seed, j, tries, table.as_oracle_table(), len(table),
                   lambda n: (segs, bounds, ps), None if target is None else np.asarray([target], np.float32), avoid)


JIT = [[-2.0, 2.0], [-2.0, 2.0], [-0.3, 0.3], [0.0, 1.0]]


def test_walled_in_slot_falls_back():
    table = TypeTable([CAR])
    snap = _world([0.0, 4.8, -4.8, 0.0, 0.0], [0.0, 0.0, 0.0, 2.2, -2.2], [0] * 5)
    out, rt, ep = _place(snap, table, JIT, 32)
    assert rt[0, 0] == -1 and (rt[0, 1:] == -1).all() and ep[0] == 1
    for k in ("x", "y", "heading", "speed"):
        assert np.array_equal(out[k], snap[k])


def test_the_one_free_try_is_taken():
    table = TypeTable([CAR])
    snap = _world([0.0], [0.0], [0])
    cx, cy, ch, cv = R.candidate(3, 0, 0, 0, 8, np.asarray(JIT, np.float32).reshape(8), 0.0, 0.0, 0.0, 0.0)
    # bounds 1 mm around try 5's box: no other try's box fits them
    k = 5
    c, s = abs(np.cos(np.float64(ch[k]))), abs(np.sin(np.float64(ch[k])))
    ex, ey = c * CAR.half_len + s * CAR.half_wid + 1e-3, s * CAR.half_len + c * CAR.half_wid + 1e-3
    bounds = (float(cx[k]) - ex, float(cx[k]) + ex, float(cy[k]) - ey, float(cy[k]) + ey)
    out, rt, _ = _place(snap, table, JIT, 8, bounds=bounds)
    assert rt[0, 0] == k
    assert out["x"][0, 0] == cx[k] and out["heading"][0, 0] == ch[k]


def test_a_pedestrian_disc_is_placed():
    table = TypeTable([CAR, PED])
    snap = _world([0.0, 3.0], [0.0, 0.0], [1, 0])
    out, rt, _ = _place(snap, table, [[-0.5, 0.5], [-0.5, 0.5], [-1.0, 1.0], [0.0, 0.5]], 8)
    assert rt[0, 0] == 0
    assert out["x"][0, 0] != snap["x"][0, 0]


def _ring(x0, x1, y0, y1):
    pts = [(x0, y0), (x1, y0), (x1, y1), (x0, y1)]
    return [(*pts[i], *pts[(i + 1) % 4]) for i in range(4)]


def test_a_pose_inside_an_area_hole_is_accepted():
    table = TypeTable([PED])
    jit = [[-1.0, 1.0], [-1.0, 1.0], [0.0, 0.0], [0.0, 0.0]]
    snap = _world([0.0], [0.0], [0])
    # a square Area frame of four rings around a 6 m hole: a pose in the hole lies inside no ring and touches no edge
    frame = _ring(-20, -3, -20, 20) + _ring(3, 20, -20, 20) + _ring(-3, 3, 3, 20) + _ring(-3, 3, -20, -3)
    out, rt, _ = _place(snap, table, jit, 8, segs=np.asarray(frame, np.float32), ps=[0, 4, 8, 12, 16])
    assert rt[0, 0] == 0
    # the same place covered by one filled Area: every try lies inside it
    _, rt, _ = _place(snap, table, jit, 8, segs=np.asarray(_ring(-20, 20, -20, 20), np.float32), ps=[0, 4])
    assert rt[0, 0] == -1


def test_avoid_target_rejects_a_pose_on_the_target():
    table = TypeTable([CAR])
    snap = _world([0.0], [0.0], [0])
    tgt = (0.0, 0.0, 0.0, 5.0, 5.0)
    _, rt, _ = _place(snap, table, JIT, 8, target=tgt, avoid=False)
    assert rt[0, 0] == 0
    _, rt, _ = _place(snap, table, JIT, 8, target=tgt, avoid=True)
    assert rt[0, 0] == -1


def test_bench_reset_help_without_a_device():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench_reset.py"), "--help"], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "usage:" in r.stdout, r.stderr[-2000:]
