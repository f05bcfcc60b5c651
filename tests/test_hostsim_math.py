"""The device arithmetic (tactics2d_b200/csrc/t2d_math.cuh) against the float64 oracle and the reference's golden vectors.

Every test runs twice through the same C entry points: here on the g++ build of tests/hostsim (no GPU needed), and in
tests/test_devsim_math.py on tests/devsim, the header compiled with the library's own nvcc flags and run on the GPU - FMA
contraction, ``rsqrtf``, ``__fdividef``, CUDA's ``sincosf`` and the warp vote of the fast kinematics loop are what the sm_90a
kernels execute, so the device run is the one that speaks for the shipped code.  (Both harnesses are test infrastructure;
the product has no CPU path.)"""

import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import geometry as G
from oracle import physics as P
from tactics2d_b200 import TypeParams, TypeTable
from tests.util import heading_err, rel_err

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
DEVSIM_SRC = os.path.join(HERE, "devsim", "devsim.cu")
DEVSIM_OUT = os.path.join(HERE, "devsim", "_devsim.so")
MATH_HDR = os.path.join(os.path.dirname(HERE), "tactics2d_b200", "csrc", "t2d_math.cuh")
RNG = dict(steer_lo=-0.524, steer_hi=0.524, speed_lo=-16.67, speed_hi=69.44, accel_lo=-11.0, accel_hi=3.121)
MEDIUM = dict(lf=4.284 / 2 - 0.880, lr=4.284 / 2 - 0.767)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


def build_devsim():
    """nvcc build of tests/devsim with the library's NVCC_FLAGS (taken from __graft_entry__, so they cannot drift apart);
    rebuilt when the source, the math header or the flags changed."""
    import __graft_entry__ as entry

    deps = [DEVSIM_SRC, MATH_HDR, os.path.abspath(entry.__file__)]
    if not os.path.exists(DEVSIM_OUT) or os.path.getmtime(DEVSIM_OUT) < max(os.path.getmtime(d) for d in deps):
        tmp = DEVSIM_OUT + f".{os.getpid()}.tmp"
        subprocess.check_call([_nvcc()] + entry.NVCC_FLAGS + ["-o", tmp, DEVSIM_SRC])
        os.replace(tmp, DEVSIM_OUT)
    return DEVSIM_OUT


@pytest.fixture(scope="session")
def devsim():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return C.CDLL(build_devsim())


@pytest.fixture(scope="module")
def sim(hostsim):
    """The harness under test: here the g++ build; tests/test_devsim_math.py runs this module's tests on the sm_90a build."""
    return hostsim


def _exported(path):
    out = subprocess.run(["nm", "-D", "--defined-only", path], check=True, capture_output=True, text=True).stdout
    return {f[2] for f in (line.split() for line in out.splitlines()) if len(f) == 3 and f[1] == "T" and f[2].startswith("hs_")}


def test_devsim_builds_and_exports_the_hostsim_entry_points(hostsim):
    """The device twin compiles for sm_90a without a GPU and offers exactly the host harness's entry points, so every
    battery below can run on either."""
    if _nvcc() is None or shutil.which("nm") is None:
        pytest.skip("needs nvcc and nm")
    dev = _exported(build_devsim())
    host = _exported(hostsim._name)
    assert len(host) >= 9 and dev == host, (sorted(dev ^ host))


def run_physics(hs, table, tid, x, y, h, v, vx, vy, act, interval=100, delta_t=5):
    arrs = [np.ascontiguousarray(a, dtype=np.float32).copy() for a in (x, y, h, v, vx, vy)]
    act = np.ascontiguousarray(act, dtype=np.float32)
    app = np.zeros_like(act)
    tid = np.ascontiguousarray(tid, dtype=np.int32)
    hs.hs_physics(C.c_int(len(tid)), table.to_c_array(), _p(tid), C.c_int(interval // delta_t), C.c_double(delta_t / 1000),
                  C.c_double((interval % delta_t) / 1000), C.c_double(interval / 1000), *[_p(a) for a in arrs], _p(act), _p(app))
    return [a.astype(np.float64) for a in arrs], app.astype(np.float64)


def _check(got, app, ref, sel=None):
    sel = slice(None) if sel is None else sel
    x, y, h, v, vx, vy = got
    vs = np.maximum(np.abs(ref[:, 3]), 1.0)
    errs = dict(x=rel_err(x, ref[:, 0])[sel].max(), y=rel_err(y, ref[:, 1])[sel].max(), h=heading_err(h, ref[:, 2])[sel].max(),
                v=rel_err(v, ref[:, 3])[sel].max(), vx=rel_err(vx, ref[:, 4], vs)[sel].max(), vy=rel_err(vy, ref[:, 5], vs)[sel].max(),
                a=rel_err(app[:, 0], ref[:, 6])[sel].max(), d=rel_err(app[:, 1], ref[:, 7])[sel].max())
    return errs


def test_bicycles_vs_reference_golden(sim):
    g = np.load(os.path.join(GOLD, "physics_bicycle.npz"))
    st, ac = g["states"], g["actions"]
    worst = {}
    for key in g.files:
        if not (key.startswith("kin_") or key.startswith("dyn_")):
            continue
        tag, name, interval, dt = key.split("_")
        interval = int(interval)
        dt = P.effective_delta_t(None if dt == "None" else int(dt), interval)
        kw = dict(MEDIUM, **(RNG if name == "con" else {}))
        if tag == "dyn":
            kw.update(mass=float(g["mass"]), mass_height=float(g["mass_height"]), model=1)
        table = TypeTable([TypeParams(**kw)])
        got, app = run_physics(sim, table, np.zeros(len(st)), st[:, 0], st[:, 1], st[:, 2], st[:, 3], 0 * st[:, 0], 0 * st[:, 0], ac,
                               interval, dt)
        sel = None
        if tag == "dyn":   # outside the band where the reference's explicit Euler is unstable (see DESIGN.md section 4)
            v_end = st[:, 3] + np.clip(ac[:, 0], kw.get("accel_lo", -np.inf), kw.get("accel_hi", np.inf)) * interval / 1000
            # forward >= 0.7 m/s, or reversing faster than 3 m/s (in reverse the slip-angle equation grows by
            # (1 + 0.72/|v|) per sub-step, which amplifies the fp32 rounding of the golden float64 inputs)
            sel = ((st[:, 3] >= 0.7) & (v_end >= 0.7)) | ((st[:, 3] <= -3.0) & (v_end <= -3.0))
        e = _check(got, app, g[key], sel)
        for k, v in e.items():
            worst[k] = max(worst.get(k, 0), v)
        assert max(e.values()) <= 1e-5, (key, e)
    assert worst["x"] < 5e-6


def test_kinematics_4wide_equals_1wide_and_oracle(sim):
    rng = np.random.default_rng(0)
    n = 4096
    p = TypeParams(**MEDIUM, **RNG)
    table = TypeTable([p])
    x, y = rng.uniform(-1000, 1000, n), rng.uniform(-1000, 1000, n)
    h, v = rng.uniform(0, 2 * np.pi, n), rng.uniform(-16, 69, n)
    act = np.stack([rng.uniform(-14, 6, n), rng.uniform(-0.8, 0.8, n)], 1)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    x, y, h, v, act = f32(x), f32(y), f32(h), f32(v), f32(act)
    (x1, y1, h1, v1, vx1, vy1), _ = run_physics(sim, table, np.zeros(n), x, y, h, v, 0 * x, 0 * x, act)
    arrs = [a.copy() for a in (x, y, h, v, 0 * x, 0 * x)]
    c = p.to_c()
    sim.hs_kinematics4(C.c_int(n), C.byref(c), C.c_int(20), C.c_double(0.005), C.c_double(0.0), *[_p(a) for a in arrs], _p(act))
    # the ILP-4 path is the same arithmetic; a group takes the bound-free fast loop only when none of its members touches a
    # speed bound, so members of mixed groups may differ from their solo run in the last bits.  The group is four
    # participants on the host, but a whole warp on the device (32 solo participants, 128 four-wide ones), where the two
    # runs therefore pick different loops far more often: a heading apart by 5e-7 rad, each within 8e-7 of float64.  There
    # a velocity component is compared on the scale of the speed it is part of (DESIGN.md section 4), not on its own,
    # which near vx = 0 would ask for the heading to agree to 1e-9 rad.
    device = sim._name.endswith("_devsim.so")
    same = 0
    for k, (a, b) in enumerate(zip(arrs, (x1, y1, h1, v1, vx1, vy1))):
        scale = np.maximum(1.0, np.abs(v1) if device and k >= 4 else np.abs(b))
        assert np.max(np.abs(a.astype(np.float64) - b) / scale) < 2e-6
        same += int(np.mean(a.astype(np.float64) == b) > 0.8)
    assert same == 6
    t = table.as_oracle_table()
    o = P.step_kinematics(x, y, h, v, act[:, 0], act[:, 1], t["lf"][0], t["lr"][0], (t["steer_lo"][0], t["steer_hi"][0]),
                          (t["speed_lo"][0], t["speed_hi"][0]), (t["accel_lo"][0], t["accel_hi"][0]))
    assert rel_err(x1, o["x"]).max() < 5e-6 and rel_err(y1, o["y"]).max() < 5e-6 and heading_err(h1, o["heading"]).max() < 3e-6
    assert rel_err(v1, o["speed"]).max() < 1e-6
    x4, y4, h4, v4 = (a.astype(np.float64) for a in arrs[:4])
    assert rel_err(x4, o["x"]).max() < 5e-6 and rel_err(y4, o["y"]).max() < 5e-6 and heading_err(h4, o["heading"]).max() < 3e-6
    assert rel_err(v4, o["speed"]).max() < 1e-6


def test_kinematics_large_rotation_fallback(sim):
    """Unconstrained speeds: per-sub-step rotation beyond the polynomial's range takes the exact-trig path."""
    rng = np.random.default_rng(1)
    n = 512
    table = TypeTable([TypeParams(**MEDIUM)])
    x = np.zeros(n, np.float32)
    v = rng.uniform(150, 400, n).astype(np.float32)
    h = rng.uniform(0, 6.28, n).astype(np.float32)
    act = np.stack([rng.uniform(-5, 5, n), rng.uniform(-0.7, 0.7, n)], 1).astype(np.float32)
    (x1, y1, h1, v1, _, _), _ = run_physics(sim, table, np.zeros(n), x, x, h, v, x, x, act)
    o = P.step_kinematics(x, x, h, v, act[:, 0], act[:, 1], table.as_oracle_table()["lf"][0], table.as_oracle_table()["lr"][0],
                          (-np.inf, np.inf), (-np.inf, np.inf), (-np.inf, np.inf))
    assert np.abs(x1 - o["x"]).max() < 2e-4 and np.abs(y1 - o["y"]).max() < 2e-4 and heading_err(h1, o["heading"]).max() < 2e-5


def test_pointmass_vs_reference_golden(sim):
    g = np.load(os.path.join(GOLD, "physics_pointmass.npz"))
    st, ac = g["states"], g["actions"]
    ranges = {"ped": (-7.0, 7.0), "band": (1.0, 3.0), "flt": 4.0, "unc": None}
    for key in g.files:
        if not key.startswith("pm_"):
            continue
        _, name, backend, interval, dt = key.split("_")
        lo, hi = P.normalize_range_pointmass(ranges[name])
        table = TypeTable([TypeParams(speed_lo=lo, speed_hi=hi, model=3 if backend == "euler" else 2, shape=1)])
        h0 = np.arctan2(st[:, 3], st[:, 2])
        (x, y, h, v, vx, vy), _ = run_physics(sim, table, np.zeros(len(st)), st[:, 0], st[:, 1], h0, 0 * h0, st[:, 2], st[:, 3], ac,
                                              int(interval), int(dt))
        ref = g[key]
        moving = ref[:, 5] > 1e-3
        vs = np.maximum(ref[:, 5], 1.0)
        assert rel_err(x, ref[:, 0]).max() <= 1e-5 and rel_err(y, ref[:, 1]).max() <= 1e-5, key
        assert heading_err(h[moving], ref[moving, 2]).max() <= 2e-5, key
        assert rel_err(vx, ref[:, 3], vs).max() <= 1e-5 and rel_err(vy, ref[:, 4], vs).max() <= 1e-5, key
        assert rel_err(v, ref[:, 5]).max() <= 1e-5, key


def test_wrap_two_pi(sim):
    sim.hs_wrap.restype = C.c_float
    for phi in [0.0, -1e-7, 6.2831853, 6.283186, 12.6, -3.0, 100.0, -100.0, 6.2831855]:
        r = sim.hs_wrap(C.c_float(phi))
        assert 0.0 <= r < 2 * np.pi
        assert heading_err(r, np.mod(np.float64(np.float32(phi)), 2 * np.pi)) < 2e-5 * max(1, abs(phi))


def _poses(rng, n, near):
    """Random pose pairs, a fraction of them within ~1e-5 m of contact, fp32 rounded."""
    a = np.zeros((n, 5), np.float32)
    b = np.zeros((n, 5), np.float32)
    for arr in (a, b):
        arr[:, 0:2] = rng.uniform(-500, 500, (n, 2))
        arr[:, 2] = rng.uniform(0, 2 * np.pi, n)
        arr[:, 3] = rng.uniform(0.1, 3.0, n)
        arr[:, 4] = np.where(rng.uniform(0, 1, n) < 0.3, -1.0, rng.uniform(0.1, 1.2, n))
    b[:, 0:2] = a[:, 0:2] + rng.uniform(-6, 6, (n, 2)).astype(np.float32)
    return a, b


def _oracle_pairs(a, b):
    a, b = a.astype(np.float64), b.astype(np.float64)
    ca, sa, cb, sb = np.cos(a[:, 2]), np.sin(a[:, 2]), np.cos(b[:, 2]), np.sin(b[:, 2])
    ka, kb = a[:, 4] < 0, b[:, 4] < 0
    oo = G.obb_obb(a[:, 0], a[:, 1], ca, sa, a[:, 3], a[:, 4], b[:, 0], b[:, 1], cb, sb, b[:, 3], b[:, 4])
    oc = G.obb_circle(a[:, 0], a[:, 1], ca, sa, a[:, 3], a[:, 4], b[:, 0], b[:, 1], b[:, 3])
    co = G.obb_circle(b[:, 0], b[:, 1], cb, sb, b[:, 3], b[:, 4], a[:, 0], a[:, 1], a[:, 3])
    cc = G.circle_circle(a[:, 0], a[:, 1], a[:, 3], b[:, 0], b[:, 1], b[:, 3])
    return np.where(ka, np.where(kb, cc, co), np.where(kb, oc, oo))


def test_filtered_pair_predicates_are_exact(sim):
    """The fp32 filter never contradicts the float64 predicate: a definite verdict equals the oracle, and
    the exact twin always equals the oracle; the undecided band is narrow."""
    rng = np.random.default_rng(5)
    n = 400000
    a, b = _poses(rng, n, 0.0)
    f32 = np.zeros(n, np.int32)
    ex = np.zeros(n, np.int32)
    sim.hs_pairs(C.c_int(n), _p(a), _p(b), _p(f32), _p(ex))
    ref = _oracle_pairs(a, b)
    assert np.array_equal(ex.astype(bool), ref)
    decided = f32 >= 0
    assert np.array_equal(f32[decided].astype(bool), ref[decided])
    assert 0.05 < ref.mean() < 0.6 and (~decided).mean() < 2e-4


def test_filtered_pair_predicates_near_contact(sim):
    """Pairs pushed to within +-2e-5 m of contact along the centre line: the filter must hand them to fp64."""
    rng = np.random.default_rng(6)
    n = 20000
    a = np.zeros((n, 5), np.float32)
    b = np.zeros((n, 5), np.float32)
    a[:, 3], a[:, 4], b[:, 3], b[:, 4] = 2.142, 0.8995, 2.142, 0.8995
    a[:, 0:2] = rng.uniform(-300, 300, (n, 2))
    gap = rng.uniform(-2e-5, 2e-5, n)
    b[:, 0] = a[:, 0] + np.float32(2 * 2.142) + gap.astype(np.float32)   # bumper to bumper, heading 0
    b[:, 1] = a[:, 1] + rng.uniform(-1.5, 1.5, n).astype(np.float32)
    f32 = np.zeros(n, np.int32)
    ex = np.zeros(n, np.int32)
    sim.hs_pairs(C.c_int(n), _p(a), _p(b), _p(f32), _p(ex))
    ref = _oracle_pairs(a, b)
    assert np.array_equal(ex.astype(bool), ref) and 0.2 < ref.mean() < 0.8
    decided = f32 >= 0
    assert np.array_equal(f32[decided].astype(bool), ref[decided])
    assert (~decided).mean() > 0.5   # most of this band is (rightly) undecided in fp32


def test_filtered_segment_and_outbound_predicates(sim):
    rng = np.random.default_rng(7)
    n = 300000
    a, _ = _poses(rng, n, 0.0)
    seg = np.zeros((n, 4), np.float32)
    seg[:, 0:2] = a[:, 0:2] + rng.uniform(-8, 8, (n, 2)).astype(np.float32)
    seg[:, 2:4] = seg[:, 0:2] + rng.uniform(-20, 20, (n, 2)).astype(np.float32)
    seg[:100, 2:4] = seg[:100, 0:2]   # degenerate segments
    f32 = np.zeros(n, np.int32)
    ex = np.zeros(n, np.int32)
    sim.hs_segments(C.c_int(n), _p(a), _p(seg), _p(f32), _p(ex))
    A, S = a.astype(np.float64), seg.astype(np.float64)
    c, s = np.cos(A[:, 2]), np.sin(A[:, 2])
    ref = np.where(A[:, 4] < 0, G.circle_segment(A[:, 0], A[:, 1], A[:, 3], S[:, 0], S[:, 1], S[:, 2], S[:, 3]),
                   G.obb_segment(A[:, 0], A[:, 1], c, s, A[:, 3], A[:, 4], S[:, 0], S[:, 1], S[:, 2], S[:, 3]))
    assert np.array_equal(ex.astype(bool), ref)
    d = f32 >= 0
    assert np.array_equal(f32[d].astype(bool), ref[d]) and (~d).mean() < 1e-3 and 0.05 < ref.mean() < 0.7
    # out of bound
    bounds = np.array([-400.0, 400.0, -300.0, 350.0], np.float32)
    a[: n // 2, 0] = np.where(rng.uniform(0, 1, n // 2) < 0.5, -400, 400) + rng.uniform(-4, 4, n // 2)
    sim.hs_outbound(C.c_int(n), _p(a), _p(bounds), _p(f32), _p(ex))
    A = a.astype(np.float64)
    c, s = np.cos(A[:, 2]), np.sin(A[:, 2])
    circ = A[:, 4] < 0
    exx, eyy = G.extents(c, s, A[:, 3], A[:, 4])
    ref = G.out_of_bound(A[:, 0], A[:, 1], np.where(circ, A[:, 3], exx), np.where(circ, A[:, 3], eyy), bounds.astype(np.float64))
    assert np.array_equal(ex.astype(bool), ref)
    d = f32 >= 0
    assert np.array_equal(f32[d].astype(bool), ref[d]) and 0.1 < ref.mean() < 0.9


def test_rect_iou_matches_oracle_and_monte_carlo(sim):
    rng = np.random.default_rng(11)
    n = 1500
    a = np.zeros((n, 5), np.float32)
    b = np.zeros((n, 5), np.float32)
    a[:, :2] = rng.uniform(-5, 5, (n, 2)); a[:, 2] = rng.uniform(0, 6.28, n); a[:, 3] = rng.uniform(.5, 3, n); a[:, 4] = rng.uniform(.3, 1.5, n)
    b[:, :2] = a[:, :2] + rng.uniform(-2, 2, (n, 2)); b[:, 2] = rng.uniform(0, 6.28, n); b[:, 3] = rng.uniform(.5, 3, n); b[:, 4] = rng.uniform(.3, 1.5, n)
    b[:40] = a[:40]
    out = np.zeros(n)
    sim.hs_rect_iou(C.c_int(n), _p(a), _p(b), _p(out))
    ref = np.array([G.rect_iou(*map(float, a[i]), *map(float, b[i])) for i in range(n)])
    assert np.abs(out - ref).max() < 1e-13 and np.allclose(out[:40], 1.0) and 0.1 < ref.mean() < 0.6
    # independent check: Monte-Carlo area ratio on a few pairs
    pts = rng.uniform(-12, 12, (600000, 2))

    def inside(r):
        c, s = np.cos(r[2]), np.sin(r[2])
        dx, dy = pts[:, 0] - r[0], pts[:, 1] - r[1]
        return (np.abs(dx * c + dy * s) <= r[3]) & (np.abs(dy * c - dx * s) <= r[4])

    for i in (100, 200, 300):
        ia, ib = inside(a[i].astype(float)), inside(b[i].astype(float))
        mc = (ia & ib).sum() / max((ia | ib).sum(), 1)
        assert abs(mc - ref[i]) < 0.02


@pytest.mark.parametrize("name", ["con", "unc"])
@pytest.mark.parametrize("interval,delta_t", [(100, 5), (9, 5), (50, 3)])
def test_drift_vs_reference_golden(sim, name, interval, delta_t):
    """SingleTrackDrift device arithmetic against the unmodified reference: first step from the golden inputs, second
    step from the reference's own first-step output rounded to fp32 (what the device state would hold)."""
    g = np.load(os.path.join(GOLD, "physics_drift.npz"))
    kw = dict(MEDIUM, mass=float(g["mass"]), mass_height=float(g["mass_height"]), model=5, **(RNG if name == "con" else {}))
    c = TypeParams(**kw).to_c()
    want = g[f"drift_{name}_{interval}_{delta_t}"]
    st, om = g["states"], g["omega"]
    n = len(st)

    def run(x, y, h, v, wf, wr, act):
        arrs = [np.ascontiguousarray(a, dtype=np.float32).copy() for a in (x, y, h, v, wf, wr)]
        act = np.ascontiguousarray(act, dtype=np.float32)
        app = np.zeros_like(act)
        sim.hs_drift(C.c_int(n), C.byref(c), C.c_int(interval // delta_t), C.c_double(delta_t / 1000),
                         C.c_double((interval % delta_t) / 1000), *[_p(a) for a in arrs], _p(act), _p(app))
        return [a.astype(np.float64) for a in arrs], app.astype(np.float64)

    def check(got, app, ref):
        x, y, h, v, wf, wr = got
        assert rel_err(x, ref[:, 0]).max() < 1e-5 and rel_err(y, ref[:, 1]).max() < 1e-5
        assert heading_err(h, ref[:, 2]).max() < 1e-5
        assert rel_err(v, ref[:, 3]).max() < 1e-5
        assert rel_err(wf, ref[:, 4]).max() < 1e-5 and rel_err(wr, ref[:, 5]).max() < 1e-5
        assert rel_err(app[:, 0], ref[:, 6]).max() < 1e-6 and rel_err(app[:, 1], ref[:, 7]).max() < 1e-6

    inf = (-np.inf, np.inf)
    rng = {k: (tuple(g[k]) if name == "con" else inf) for k in ("steer_range", "speed_range", "accel_range")}
    rng32 = {k: tuple(np.float32(v).astype(np.float64)) for k, v in rng.items()}
    f32 = lambda v: np.float64(np.float32(v))

    def oracle(s6, act):
        r = P.step_drift(s6[:, 0], s6[:, 1], s6[:, 2], s6[:, 3], s6[:, 4], s6[:, 5], act[:, 0], act[:, 1], f32(kw["lf"]), f32(kw["lr"]),
                         f32(kw["mass"]), f32(0.344), f32(0.76), 1.0, 1500.0, f32(1.7), rng32["steer_range"], rng32["speed_range"],
                         rng32["accel_range"], interval, delta_t)
        return np.stack([r[f] for f in ("x", "y", "heading", "speed", "omega_wf", "omega_wr", "accel", "delta")], 1)

    s0 = np.concatenate([st, om], 1)
    got, app = run(*s0.T, g["actions"])
    # The reference's own numbers (float64 parameters) on the rows where parameter rounding is harmless.  With explicit
    # Euler at 5 ms the wheel-spin equation of this model is stiff (d omega / dt ~ R F_x / I_yw ~ 2000 rad/s^2 per unit
    # slip), so on many rows the 6e-8 rounding of (lf, lr, mass, R, I_yw) to fp32 alone moves the float64 result by
    # 1e-4 .. 1e-3; those rows are held to the restatement with the SAME fp32 parameters below instead.
    ref64 = g[f"drift_{name}_{interval}_{delta_t}"][:, 0]
    ref32 = oracle(s0, g["actions"])
    calm = (np.abs(ref64 - ref32) / np.maximum(1.0, np.abs(ref64))).max(1) < 2e-7
    assert calm.sum() >= 20
    check([a[calm] for a in got], app[calm], want[calm, 0])
    # ... and every row against the float64 restatement holding the fp32-rounded parameters
    check(got, app, ref32)
    # second step: teacher-forced from the reference's first-step output rounded to fp32
    w0 = want[:, 0, :6].astype(np.float32).astype(np.float64)
    got, app = run(*w0.T, g["actions2"])
    check(got, app, oracle(w0, g["actions2"]))


@pytest.mark.parametrize("n_beams", [37, 360, 1100, 3600])
def test_lidar_beam_window_is_conservative(sim, n_beams):
    """Every beam that survives the reference's own filters (sensor/lidar.py:188-213) on an edge lies inside the beam window
    the kernel computes for that edge (so culling the other beams cannot change a scan); windows are also small on average."""
    rng = np.random.default_rng(n_beams)
    n = 6000
    R = 20.0
    c = rng.uniform(-R, R, (n, 2))
    half = rng.uniform(0.01, 6.0, n)[:, None] * np.stack([np.cos(a := rng.uniform(0, 2 * np.pi, n)), np.sin(a)], 1)
    e = np.concatenate([c - half, c + half], 1)
    e[:300, :2] = rng.uniform(-0.02, 0.02, (300, 2))            # edges starting at / next to the sensor
    e[300:600] = np.concatenate([-half[300:600] * 3, half[300:600] * 3], 1) + rng.uniform(-1e-3, 1e-3, (300, 4))   # through the origin
    e[600:900, 1] = 0.0
    e[600:900, 3] = 0.0                                         # on the x axis (the beam-0 / wrap-around direction)
    e[900:1200, 0] = e[900:1200, 2]                             # vertical edges
    x1, y1, x2, y2 = e.T
    dx, dy = x2 - x1, y2 - y1
    dd = dx * dx + dy * dy
    t = np.clip(-(x1 * dx + y1 * dy) / np.where(dd > 0, dd, 1.0), 0, 1)
    dist2 = (x1 + t * dx) ** 2 + (y1 + t * dy) ** 2
    out = np.zeros((n, 2), np.int32)
    sim.hs_beam_window(C.c_int(n), _p(np.ascontiguousarray(e)), _p(np.ascontiguousarray(dist2)), C.c_int(n_beams), _p(out))
    # the reference's per-pair arithmetic, one edge at a time
    theta = np.linspace(0, 2 * np.pi, n_beams, endpoint=False)
    a, b = np.sin(theta), -np.cos(theta)
    lx, ly = np.cos(theta) * R, np.sin(theta) * R
    tz = 1e-8
    total = 0
    for i in range(n):
        d, ee, f = y2[i] - y1[i], x1[i] - x2[i], y1[i] * x2[i] - x1[i] * y2[i]
        det = a * ee - b * d
        par = det == 0
        det = np.where(par, 1.0, det)
        rx, ry = (b * f) / det, (-a * f) / det
        ok = ~par
        ok &= ~(rx > np.maximum(tz, lx) + tz) & ~(rx < np.minimum(-tz, lx) - tz) & ~(ry > np.maximum(tz, ly) + tz) & ~(ry < np.minimum(-tz, ly) - tz)
        ok &= ~(rx > max(x1[i], x2[i]) + tz) & ~(rx < min(x1[i], x2[i]) - tz) & ~(ry > max(y1[i], y2[i]) + tz) & ~(ry < min(y1[i], y2[i]) - tz)
        first, cnt = out[i]
        assert 0 <= first < n_beams and 1 <= cnt <= n_beams
        inside = ((np.arange(n_beams) - first) % n_beams) < cnt
        assert not np.any(ok & ~inside), (i, e[i], np.nonzero(ok & ~inside)[0][:5], first, cnt)
        total += cnt
    assert total / n < 0.45 * n_beams + 8     # (this sample is dominated by long edges close to the sensor)


@pytest.mark.parametrize("interval,delta_t", [(100, 5), (100, 2), (100, 1), (200, 5), (50, 3)])
def test_kinematics_error_budget_near_the_origin(sim, interval, delta_t):
    """The 1e-5 contract as an ABSOLUTE bound (|x|, |y| <= 1, where the relative scale is 1) over the full speed range of the
    medium car, for short and long sub-step counts: the carried-rotation fast loop (<= 24 sub-steps) and the general loop."""
    rng = np.random.default_rng(interval * 10 + delta_t)
    n = 50000
    p = TypeParams(**MEDIUM, **RNG)
    table = TypeTable([p])
    t = table.as_oracle_table()
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    x, y, h = f32(rng.uniform(-1, 1, n)), f32(rng.uniform(-1, 1, n)), f32(rng.uniform(0, 2 * np.pi, n))
    v, act = f32(rng.uniform(-16, 69, n)), f32(np.stack([rng.uniform(-12, 6, n), rng.uniform(-0.8, 0.8, n)], 1))
    (x1, y1, h1, v1, _, _), _ = run_physics(sim, table, np.zeros(n), x, y, h, v, 0 * x, 0 * x, act, interval, delta_t)
    o = P.step_kinematics(x, y, h, v, act[:, 0], act[:, 1], t["lf"][0], t["lr"][0], (t["steer_lo"][0], t["steer_hi"][0]),
                          (t["speed_lo"][0], t["speed_hi"][0]), (t["accel_lo"][0], t["accel_hi"][0]), interval, delta_t)
    assert rel_err(x1, o["x"]).max() < 1e-5 and rel_err(y1, o["y"]).max() < 1e-5
    assert heading_err(h1, o["heading"]).max() < 5e-6 and rel_err(v1, o["speed"]).max() < 1e-6


# ------------------------------------------------------------------------------------------------ near-contact batteries
# Every predicate kind pushed into its own fp32 filter band.  Three claims are checked on each: the exact twin equals the
# float64 oracle everywhere, a decided fp32 verdict equals the oracle, and more than half of the inner band comes back
# undecided (which shows that the battery really sat inside the band instead of beside it).
EPS = 2e-6     # EPS_LIN of t2d_math.cuh


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _rot(h, x, y):
    c, s = np.cos(h), np.sin(h)
    return c * x - s * y, s * x + c * y


def _oracle_segments(a, seg):
    A, S = a.astype(np.float64), seg.astype(np.float64)
    c, s = np.cos(A[:, 2]), np.sin(A[:, 2])
    return np.where(A[:, 4] < 0, G.circle_segment(A[:, 0], A[:, 1], A[:, 3], S[:, 0], S[:, 1], S[:, 2], S[:, 3]),
                    G.obb_segment(A[:, 0], A[:, 1], c, s, A[:, 3], A[:, 4], S[:, 0], S[:, 1], S[:, 2], S[:, 3]))


def _oracle_outbound(a, bounds):
    A = a.astype(np.float64)
    c, s = np.cos(A[:, 2]), np.sin(A[:, 2])
    circ = A[:, 4] < 0
    exx, eyy = G.extents(c, s, A[:, 3], A[:, 4])
    return G.out_of_bound(A[:, 0], A[:, 1], np.where(circ, A[:, 3], exx), np.where(circ, A[:, 3], eyy), bounds.astype(np.float64))


def _call(fn, a, b):
    n = len(a)
    f32 = np.zeros(n, np.int32)
    ex = np.zeros(n, np.int32)
    fn(C.c_int(n), _p(_f32(a)), _p(_f32(b)), _p(f32), _p(ex))
    return f32, ex


def _assert_band(f32, ex, ref, inner, what):
    assert np.array_equal(ex.astype(bool), ref), (what, np.nonzero(ex.astype(bool) != ref)[0][:8])
    d = f32 >= 0
    assert np.array_equal(f32[d].astype(bool), ref[d]), (what, np.nonzero(d & (f32.astype(bool) != ref))[0][:8])
    assert inner.sum() >= 50 and (~d[inner]).mean() > 0.5, (what, inner.sum(), (~d[inner]).mean())
    assert 0.2 < ref.mean() < 0.8, (what, ref.mean())


def _box_pairs(rng, n, corner_to_corner):
    """Box pairs in contact along A's edge (corner of a rotated B against it) or corner to corner (B a scaled copy of A on
    A's diagonal, so their bounding circles are tangent as well); returns the poses, the designed gap and its band."""
    ha = rng.uniform(0, 2 * np.pi, n)
    la, wa = rng.uniform(0.8, 2.5, n), rng.uniform(0.4, 1.2, n)
    xa, ya = rng.uniform(-40, 40, n), rng.uniform(-40, 40, n)
    if corner_to_corner:
        s = rng.uniform(0.5, 1.5, n)
        lb, wb = s * la, s * wa
        ra = np.hypot(la, wa)
        sx, sy = rng.choice([-1.0, 1.0], n), rng.choice([-1.0, 1.0], n)
        hb = ha + rng.choice([0.0, np.pi], n)
        dist = ra * (1 + s)
        scale = np.maximum(la, wa) / ra                       # the SAT margin is gap * scale
        band = EPS * (dist + la + wa + lb + wb) / scale
        gap = rng.uniform(-3, 3, n) * band
        ox, oy = _rot(ha, sx * la / ra * (dist + gap), sy * wa / ra * (dist + gap))
    else:
        lb, wb = rng.uniform(0.8, 2.5, n), rng.uniform(0.4, 1.2, n)
        k = rng.integers(0, 4, n)                              # which edge of A: the frame of edge k is A's turned by k pi/2
        hk = ha + k * (np.pi / 2)
        lk, wk = np.where(k % 2 == 1, wa, la), np.where(k % 2 == 1, la, wa)
        phi = rng.uniform(0.2, 1.37, n) * rng.choice([-1.0, 1.0], n)
        hb = hk + phi
        sp, cp = np.sin(phi), np.cos(phi)
        ext = lb * np.abs(sp) + wb * cp                        # B's half extent across the edge
        cx = -np.sign(sp) * lb * cp + wb * sp                  # along-edge offset of B's corner nearest the edge
        band = EPS * (2 * (wk + ext) + la + wa + lb + wb)
        gap = rng.uniform(-3, 3, n) * band
        ox, oy = _rot(hk, rng.uniform(-0.8, 0.8, n) * lk - cx, wk + ext + gap)
    a = np.stack([xa, ya, np.mod(ha, 2 * np.pi), la, wa], 1)
    b = np.stack([xa + ox, ya + oy, np.mod(hb, 2 * np.pi), lb, wb], 1)
    swap = rng.uniform(0, 1, n) < 0.5                          # B's axes separate as often as A's
    a[swap], b[swap] = b[swap].copy(), a[swap].copy()
    return _f32(a), _f32(b), gap, band


@pytest.mark.parametrize("corner_to_corner", [False, True], ids=["corner_to_edge", "corner_to_corner"])
def test_near_contact_rotated_boxes(sim, corner_to_corner):
    a, b, gap, band = _box_pairs(np.random.default_rng(31 + corner_to_corner), 40000, corner_to_corner)
    f32, ex = _call(sim.hs_pairs, a, b)
    _assert_band(f32, ex, _oracle_pairs(a, b), np.abs(gap) < 0.5 * band, "box-box")


def test_near_contact_discs_tangent_to_the_ulp(sim):
    """Disc pairs exactly tangent (centres on a 3-4-5 triangle or an axis, every coordinate exact in fp32), then B moved by
    -100 .. 100 ulp along x: the closed predicate holds exactly for k <= 0."""
    rng = np.random.default_rng(33)
    radii = np.array([(1.25, 1.25), (0.5, 2.0), (1.0, 1.5)])
    offs = np.array([(2.5, 0.0), (1.5, 2.0), (2.0, 1.5)])
    n0 = 60
    ks = np.arange(-100, 101)
    base = np.stack([rng.integers(64, 3840, n0) / 64.0, rng.integers(-3840, 3840, n0) / 64.0], 1)
    r = radii[rng.integers(0, 3, n0)]
    o = offs[rng.integers(0, 3, n0)] * np.stack([np.ones(n0), rng.choice([-1.0, 1.0], n0)], 1)
    a = np.zeros((n0, len(ks), 5), np.float32)
    b = np.zeros_like(a)
    a[..., 0], a[..., 1], a[..., 3], a[..., 4] = base[:, None, 0], base[:, None, 1], r[:, None, 0], -1.0
    xb = (base[:, 0] + o[:, 0]).astype(np.float32)
    b[..., 0] = (xb.view(np.int32)[:, None] + ks[None]).astype(np.int32).view(np.float32)   # xb > 0: +k ulp moves away
    b[..., 1], b[..., 3], b[..., 4] = (base[:, 1] + o[:, 1])[:, None], r[:, None, 1], -1.0
    a, b = a.reshape(-1, 5), b.reshape(-1, 5)
    k = np.broadcast_to(ks, (n0, len(ks))).reshape(-1)
    f32, ex = _call(sim.hs_pairs, a, b)
    ref = _oracle_pairs(a, b)
    assert np.array_equal(ref, k <= 0)
    _assert_band(f32, ex, ref, np.abs(k) <= 1, "disc-disc")


def test_near_contact_disc_box(sim):
    """A disc against a rotated box, at a face or at a corner, gaps over +-3 bands."""
    rng = np.random.default_rng(34)
    n = 40000
    h = rng.uniform(0, 2 * np.pi, n)
    la, wa, r = rng.uniform(0.8, 2.5, n), rng.uniform(0.4, 1.2, n), rng.uniform(0.2, 1.5, n)
    xa, ya = rng.uniform(-40, 40, n), rng.uniform(-40, 40, n)
    face = rng.uniform(0, 1, n) < 0.5
    beta = rng.uniform(0.15, np.pi / 2 - 0.15, n)
    sx, sy = rng.choice([-1.0, 1.0], n), rng.choice([-1.0, 1.0], n)
    band = 2 * (2 * EPS) * (la + wa + r + la + wa + r)         # in metres of gap: 2 e1, e1 from the centre offset's size
    gap = rng.uniform(-3, 3, n) * band
    lx = np.where(face, sx * (la + r + gap), sx * (la + (r + gap) * np.cos(beta)))
    ly = np.where(face, rng.uniform(-0.9, 0.9, n) * wa, sy * (wa + (r + gap) * np.sin(beta)))
    ox, oy = _rot(h, lx, ly)
    box = np.stack([xa, ya, h, la, wa], 1)
    disc = np.stack([xa + ox, ya + oy, np.zeros(n), r, -np.ones(n)], 1)
    swap = rng.uniform(0, 1, n) < 0.5
    a, b = np.where(swap[:, None], disc, box), np.where(swap[:, None], box, disc)
    a, b = _f32(a), _f32(b)
    f32, ex = _call(sim.hs_pairs, a, b)
    _assert_band(f32, ex, _oracle_pairs(a, b), np.abs(gap) < 0.25 * band, "disc-box")


def test_near_contact_box_and_disc_segments(sim):
    """Segments parallel to a box edge, perpendicular to it (an endpoint approaching the edge) and oblique, and segments
    passing a disc or ending next to it, at gaps over +-3 bands."""
    rng = np.random.default_rng(35)
    n = 40000
    h = rng.uniform(0, 2 * np.pi, n)
    la, wa = rng.uniform(0.8, 2.5, n), rng.uniform(0.4, 1.2, n)
    xa, ya = rng.uniform(-40, 40, n), rng.uniform(-40, 40, n)
    disc = rng.uniform(0, 1, n) < 0.4
    la = np.where(disc, rng.uniform(0.2, 1.5, n), la)
    kind = rng.integers(0, 3, n)                               # 0 parallel, 1 perpendicular (endpoint), 2 oblique
    k = rng.integers(0, 4, n)
    hk = h + k * (np.pi / 2)
    lk = np.where(disc, la, np.where(k % 2 == 1, wa, la))
    wk = np.where(disc, la, np.where(k % 2 == 1, la, wa))
    length = rng.uniform(1.0, 6.0, n)
    ang = np.where(kind == 0, 0.0, np.where(kind == 1, np.pi / 2, rng.uniform(0.3, 1.2, n)))
    # box: e1 = EPS (|u| + |v| + l + w); disc: e1 = 2 EPS (|u| + |d| + r) and the gap band is 2 e1
    size = 2 * (lk + wk + length) + la + wa
    band = np.where(disc, 4 * 2 * EPS * (lk + 2 * length + la), EPS * size)
    gap = rng.uniform(-3, 3, n) * band
    t0 = np.where(disc, 0.0, rng.uniform(-0.8, 0.8, n) * lk)
    # start point on the line at distance wk + gap from the centre, across the edge (the disc: its surface)
    p1x, p1y = t0, wk + gap
    ux, uy = np.cos(ang), np.sin(ang)                          # parallel: along the edge; else leaving the edge
    para = kind == 0
    p1x = np.where(para, t0 - 0.5 * length, p1x)
    p2x, p2y = p1x + length * ux, p1y + length * uy
    x1, y1 = _rot(hk, p1x, p1y)
    x2, y2 = _rot(hk, p2x, p2y)
    a = _f32(np.stack([xa, ya, np.mod(h, 2 * np.pi), la, np.where(disc, -1.0, wa)], 1))
    seg = _f32(np.stack([xa + x1, ya + y1, xa + x2, ya + y2], 1))
    f32, ex = _call(sim.hs_segments, a, seg)
    ref = _oracle_segments(a, seg)
    inner = np.abs(gap) < 0.25 * band
    for what, sel in (("box-segment", ~disc), ("disc-segment", disc)):
        _assert_band(f32[sel], ex[sel], ref[sel], inner[sel], what)


def test_segment_endpoint_exactly_on_a_box_edge(sim):
    """Heading 0, box edges and segment endpoints on exactly representable coordinates: an endpoint ON the edge touches
    (closed sets), one ulp outside does not, one ulp inside does."""
    rng = np.random.default_rng(36)
    n = 6000
    la = rng.choice([2.25, 1.5, 2.0], n)
    wa = rng.choice([1.0, 0.75], n)
    xa, ya = rng.integers(1, 40, n).astype(np.float64), rng.integers(-40, 40, n).astype(np.float64)
    t = rng.integers(-6, 7, n) / 8.0 * wa
    beta = rng.uniform(-1.4, 1.4, n)
    ks = rng.integers(-3, 4, n)
    ex1 = (xa + la).astype(np.float32)                         # the right edge, x > 0: +k ulp is outward
    ex1 = (ex1.view(np.int32) + ks).astype(np.int32).view(np.float32).astype(np.float64)
    seg = _f32(np.stack([ex1, ya + t, ex1 + 3 * np.cos(beta), ya + t + 3 * np.sin(beta)], 1))
    a = _f32(np.stack([xa, ya, np.zeros(n), la, wa], 1))
    f32, ex = _call(sim.hs_segments, a, seg)
    ref = _oracle_segments(a, seg)
    assert np.array_equal(ref, ks <= 0)
    _assert_band(f32, ex, ref, ks == 0, "endpoint-on-edge")


def test_pose_extent_exactly_on_the_bound(sim):
    """OutBound is strict: a heading-0 box or a disc whose extent ends exactly on a limit is inside, one ulp further out
    is out.  Then rotated boxes at gaps over +-3 bands from every limit."""
    rng = np.random.default_rng(37)
    bounds = np.array([-64.0, 64.0, -48.0, 48.0], np.float32)
    n = 8000
    disc = rng.uniform(0, 1, n) < 0.3
    l = np.where(disc, rng.choice([0.25, 0.5], n), rng.choice([2.25, 1.5], n))
    w = np.where(disc, -1.0, rng.choice([1.0, 0.75], n))
    side = rng.integers(0, 4, n)
    ks = rng.integers(-3, 4, n)
    ext = np.where(side < 2, l, np.where(disc, l, w))          # half extent across the limit at heading 0
    lim = bounds[side].astype(np.float64)
    sgn = np.where(side % 2 == 1, 1.0, -1.0)                   # +: the max limits
    c = (lim - sgn * ext).astype(np.float32)                   # exact: extent ends on the limit
    c = (c.view(np.int32) + (ks * sgn * np.sign(c)).astype(np.int32)).view(np.float32)   # +k ulp outward
    other = rng.uniform(-20, 20, n).astype(np.float32)
    a = _f32(np.stack([np.where(side < 2, c, other), np.where(side < 2, other, c), np.zeros(n), l, w], 1))
    out32 = np.zeros(n, np.int32)
    out_ex = np.zeros(n, np.int32)
    sim.hs_outbound(C.c_int(n), _p(a), _p(bounds), _p(out32), _p(out_ex))
    ref = _oracle_outbound(a, bounds)
    assert np.array_equal(ref, ks > 0)
    _assert_band(out32, out_ex, ref, ks == 0, "extent-on-limit")
    # rotated boxes near every limit
    h = rng.uniform(0, 2 * np.pi, n)
    la, wa = rng.uniform(0.8, 2.5, n), rng.uniform(0.4, 1.2, n)
    exx, eyy = la * np.abs(np.cos(h)) + wa * np.abs(np.sin(h)), la * np.abs(np.sin(h)) + wa * np.abs(np.cos(h))
    e_side = np.where(side < 2, exx, eyy)
    band = EPS * (128.0 + la + wa)
    gap = rng.uniform(-3, 3, n) * band
    cc = lim - sgn * (e_side - gap)                            # gap > 0: out by gap
    a = _f32(np.stack([np.where(side < 2, cc, other), np.where(side < 2, other, cc), h, la, wa], 1))
    sim.hs_outbound(C.c_int(n), _p(a), _p(bounds), _p(out32), _p(out_ex))
    _assert_band(out32, out_ex, _oracle_outbound(a, bounds), np.abs(gap) < 0.5 * band, "rotated-extent")


# ------------------------------------------------------------------------------------------------ kinematics
@pytest.mark.parametrize("interval", [5, 10, 100, 120, 125, 200])
def test_kinematics4_absolute_budget_near_the_origin(sim, interval):
    """hs_kinematics4 (four participants per lane: on the device 128 per warp, K1's layout) at 1, 2, 20, 24, 25 and 40
    sub-steps of 5 ms from |x|, |y| <= 1, held to 1e-5 max(|ref|, 1): an ABSOLUTE 1e-5 wherever the result is within 1 m
    of the origin (thousands of participants here).  Every other block of 128 carries one participant that runs into a
    speed bound, so on the device half the warps vote for the general loop and half may take the fast one."""
    rng = np.random.default_rng(interval)
    n = 128 * 256
    p = TypeParams(**MEDIUM, **RNG)
    t = TypeTable([p]).as_oracle_table()
    x, y, h = _f32(rng.uniform(-1, 1, n)), _f32(rng.uniform(-1, 1, n)), _f32(rng.uniform(0, 2 * np.pi, n))
    v = rng.uniform(-10, 60, n)
    act = np.stack([rng.uniform(-3, 2, n), rng.uniform(-0.8, 0.8, n)], 1)
    plant = np.arange(0, n // 128, 2) * 128 + rng.integers(0, 128, n // 256)
    v[plant] = RNG["speed_hi"] - 0.01                          # 3 m/s^2 reaches the bound within one 5 ms sub-step
    act[plant, 0] = 3.0
    v, act = _f32(v), _f32(act)
    arrs = [a.copy() for a in (x, y, h, v, 0 * x, 0 * x)]
    c = p.to_c()
    sim.hs_kinematics4(C.c_int(n), C.byref(c), C.c_int(interval // 5), C.c_double(0.005), C.c_double(0.0), *[_p(a) for a in arrs],
                       _p(act))
    o = P.step_kinematics(x, y, h, v, act[:, 0], act[:, 1], t["lf"][0], t["lr"][0], (t["steer_lo"][0], t["steer_hi"][0]),
                          (t["speed_lo"][0], t["speed_hi"][0]), (t["accel_lo"][0], t["accel_hi"][0]), interval, 5)
    x1, y1, h1, v1 = (a.astype(np.float64) for a in arrs[:4])
    assert rel_err(x1, o["x"]).max() < 1e-5 and rel_err(y1, o["y"]).max() < 1e-5
    assert (np.abs(o["x"]) <= 1).sum() > 2000 and (np.abs(o["y"]) <= 1).sum() > 2000
    assert heading_err(h1, o["heading"]).max() < 5e-6 and rel_err(v1, o["speed"]).max() < 1e-6
    assert (o["speed"][plant] == np.float32(RNG["speed_hi"])).all()   # the planted participants did reach the bound


def test_kinematics_rare_trigonometry(sim):
    """The arguments the branch-free trigonometry cannot take and re-does afterwards: a steering range of +-1.2 rad (beyond
    0.78) and headings of 513 .. 1e4 rad in the input state, through the 1-wide and the 4-wide kinematics, against
    oracle.physics.  The new heading is a sum at the input's magnitude, so its error may reach half an fp32 ulp of it."""
    rng = np.random.default_rng(38)
    n = 128 * 64
    wide = dict(RNG, steer_lo=-1.2, steer_hi=1.2)
    p = TypeParams(**MEDIUM, **wide)
    table = TypeTable([p])
    t = table.as_oracle_table()
    x, y = _f32(rng.uniform(-1, 1, n)), _f32(rng.uniform(-1, 1, n))
    big = rng.uniform(0, 1, n) < 0.5
    h = _f32(np.where(big, rng.uniform(513, 1e4, n) * rng.choice([-1.0, 1.0], n), rng.uniform(0, 2 * np.pi, n)))
    v = _f32(rng.uniform(-10, 40, n))
    act = _f32(np.stack([rng.uniform(-3, 2, n), rng.uniform(-1.5, 1.5, n)], 1))
    o = P.step_kinematics(x, y, h, v, act[:, 0], act[:, 1], t["lf"][0], t["lr"][0], (t["steer_lo"][0], t["steer_hi"][0]),
                          (t["speed_lo"][0], t["speed_hi"][0]), (t["accel_lo"][0], t["accel_hi"][0]))
    h_tol = 1e-5 + np.spacing(np.abs(h) + 8.0).astype(np.float64)
    (x1, y1, h1, v1, _, _), app = run_physics(sim, table, np.zeros(n), x, y, h, v, 0 * x, 0 * x, act)
    assert np.abs(app[:, 1] - np.clip(act[:, 1], -1.2, 1.2)).max() == 0 and (np.abs(app[:, 1]) > 0.78).mean() > 0.3
    arrs = [a.copy() for a in (x, y, h, v, 0 * x, 0 * x)]
    c = p.to_c()
    sim.hs_kinematics4(C.c_int(n), C.byref(c), C.c_int(20), C.c_double(0.005), C.c_double(0.0), *[_p(a) for a in arrs], _p(act))
    for got in ((x1, y1, h1, v1), tuple(a.astype(np.float64) for a in arrs[:4])):
        gx, gy, gh, gv = got
        assert np.abs(gx - o["x"]).max() < 1e-5 and np.abs(gy - o["y"]).max() < 1e-5
        assert (heading_err(gh, o["heading"]) <= h_tol).all() and heading_err(gh[~big], o["heading"][~big]).max() < 5e-6
        assert rel_err(gv, o["speed"]).max() < 1e-6
