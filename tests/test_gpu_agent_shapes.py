"""The multi-agent kernels at every row and slot a lane owns: K11 (t2d_scatter_agent_action), K10 (t2d_agents_epilogue),
K4's observer rows (t2d_lidar_scan_agents) and K9 (t2d_observe_agents), at M and Q up to 128 (k = 0 .. 3 of lane l's rows and
slots l + 32 k) and at odd N (a partial last CTA), against the float64 oracles with each kernel's own test file's criterion.
The scene, list and K10 input builders are tests/agent_shape_scenes.py.

Every output buffer a C entry takes is allocated with a guard tail of eight scenarios' rows (one CTA of K10 / K11, two of
K4 / K9) and filled with a sentinel bit pattern before every call: a row the kernel skipped keeps the sentinel instead of
an earlier call's value, and a write past the rows changes the tail.  Also: a multi-agent step chain and the host step at
M = Q = 128, and the env with agent actions, rewards and lidar at that shape against the same world-level sequence."""

import ctypes as C

import numpy as np
import pytest

from oracle import lidar as OL
from oracle import scenario as O
from tests import agent_lidar_oracle as AL
from tests import agent_obs_oracle as A
from tests import agent_reward_oracle as R
from tests import agent_shape_scenes as S
from tests import vector_obs_oracle as V
from tests.agent_action_oracle import owner_rows, scatter_agent_action

CASES = S.cases()
IDS = [S.case_id(c) for c in CASES]
TAIL = 8   # scenarios (K10, K11) or rows (K4, K9) of guard tail
SENTINEL = {"float32": 0x7FBADBAD, "uint8": 0xA5, "int16": 0x5A5A}   # a NaN payload no kernel writes, 165, 23130
SEL_ROWS = (0, 31, 32, 63, 64, 95, 96, 126, 127)


# ------------------------------------------------------------------ CPU: what the builders claim
def test_builders_cover_what_they_claim():
    ns, ms, qs = ({c[i] for c in S.SHAPES} for i in range(3))
    assert ms >= {1, 2, 33, 65, 96, 97, 127, 128}
    for q in (1, 32, 33, 64, 65, 96, 97, 127, 128):
        assert any(c[2] == q and c[3] for c in CASES) and any(c[2] == q and not c[3] for c in CASES), q
    assert ns >= {1, 3, 5, 9, 13} and all(n % 4 for n in ns) and max(ns) > 4096
    # known types: slot 126 empty (the scene's M - 2) and slot 50 empty
    types = np.zeros((3, 128), np.uint8)
    types[:, [50, 126]] = O.INACTIVE
    obs = S.observer_list(np.random.default_rng(0), types, 128).astype(np.int64)
    assert (obs[:, 5] == obs[:, 97]).all() and (obs[:, 70] == obs[:, 100]).all() and (obs[:, 2] == obs[:, 37]).all()
    assert (obs[:, [5, 70]] >= 96).all() and (obs[:, 127] == 127).all()
    assert (obs[:, 65] == -1).all() and (obs[:, 66] == 128).all() and (obs[:, 98] == -1).all() and (obs[:, 99] == 128).all()
    assert (np.take_along_axis(types, obs[:, [67, 101]], 1) == O.INACTIVE).all()
    assert (obs[:, 96:] >= 96).sum(1).min() >= 25
    cov = S.list_coverage(obs, types)
    assert all(cov[k] for k in S.require_list_coverage(cov, 128, 128))
    # a list whose duplicates stay in one lane (q = 1 and 33, q = 95 and 127), and which never names slot M - 1, fails
    bad = np.tile(np.arange(128), (3, 1))
    bad[:, 33] = 1
    bad[:, 127] = 95
    cov = S.list_coverage(bad, types)
    assert not cov["cross_duplicates"] and not cov["last_slot"] and not cov["minus_one_k2"]
    with pytest.raises(AssertionError):
        S.require_list_coverage(cov, 128, 128)
    # (5, 97) alone: a cross-lane duplicate, but no k = 3 row loses to a k = 2 row
    one = np.tile(np.arange(128), (3, 1))
    one[:, 97] = one[:, 5] = 100
    cov = S.list_coverage(one, np.zeros((3, 128), np.uint8))
    assert cov["cross_duplicates"] and cov["k3_loses_to_k0"] and not cov["k3_loses_to_k2"]
    # the K10 flags: every kind on slots >= 96 at the first call, nothing after the third
    rng = np.random.default_rng(1)
    assert all(S.flag_coverage(S.k10_flags(rng, 4, 128, 0)).values())
    assert not any(S.flag_coverage(S.k10_flags(rng, 4, 128, 3)).values())
    # the goals: NaN on q % 4 == 0, the slot's own pose on q % 4 == 1
    x = rng.uniform(0, 9, (2, 8)).astype(np.float32)
    table = dict(half_len=np.float32([2.0, 2.5]), half_wid=np.float32([1.0, 0.9]))
    t = np.zeros((2, 8), np.uint8)
    t[:, 3] = 1
    g = S.k10_goals(rng, x, x, x, t, table, None)
    assert np.isnan(g[:, 0::4, 0]).all() and not np.isnan(g[:, 1::4, 0]).any()
    assert np.array_equal(g[:, 1, :3], np.stack([x[:, 1]] * 3, -1)) and (g[:, 3, 3] == 2.5).all()


# ------------------------------------------------------------------ helpers
class Guarded:
    """A flat device buffer: ``shape`` elements, then a guard tail of ``tail`` elements, every element a sentinel."""

    def __init__(self, shape, tail, dtype):
        import torch

        self.shape, self.n = tuple(shape), int(np.prod(shape))
        self.dtype = dtype
        self.t = torch.empty(self.n + tail, dtype=getattr(torch, dtype), device="cuda")
        self.fill()

    def bits(self):
        import torch

        return self.t.view(torch.int32) if self.dtype == "float32" else self.t

    def fill(self):
        self.bits().fill_(SENTINEL[self.dtype])

    @property
    def body(self):
        return self.t[:self.n].view(self.shape)

    @property
    def ptr(self):
        return C.c_void_p(self.t.data_ptr())

    def check(self, name):
        """Every element of the body written, the tail untouched."""
        b = self.bits()
        assert bool((b[self.n:] == SENTINEL[self.dtype]).all()), f"{name}: a write past the buffer's rows"
        left = int((b[:self.n] == SENTINEL[self.dtype]).sum())
        assert left == 0, f"{name}: {left} elements never written"


def _bits(a):
    a = a.cpu().numpy() if hasattr(a, "cpu") else a
    return np.ascontiguousarray(a).view(np.uint32)


def _random_bits(rng, shape):
    b = rng.integers(0, 2**32, shape, dtype=np.uint64).astype(np.uint32)
    special = np.asarray([0x80000000, 0x7FC00001, 0xFFBADBAD, 0x00000001], np.uint32)[:b.size]
    b.reshape(-1)[:special.size] = special
    return b.view(np.float32)


def _world(s, max_step=0, **kw):
    """The scene's world, state and types from a masked reset of every scenario (so that later resets restore them)."""
    import torch
    from tactics2d_b200 import BatchedWorld

    n, m = s.shape
    w = BatchedWorld(n, m, s.table, max_step=max_step, **kw)
    w.set_map(s.segments, s.bounds)
    pool = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in s.state().items()}
    w.type_id.copy_(torch.from_numpy(s.type_id).cuda())
    w.reset(torch.ones(n, dtype=torch.uint8, device="cuda"), pool)
    return w, pool


def _list(case, s, seed):
    """(observers int16 [N, Q] numpy or None, the device tensor or None)."""
    import torch

    n, m, q, listed = case
    if not listed:
        return None, None
    obs = S.observer_list(np.random.default_rng(seed), s.type_id, q)
    return obs, torch.from_numpy(obs).cuda()


def _p(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _rows_of(observers, n, Q):
    """The observer list, or without one the list "row q is slot q" of Q rows (the oracles read None as Q = M)."""
    return np.tile(np.arange(Q, dtype=np.int16), (n, 1)) if observers is None else observers


def _bind_agents(w, obs_t, Q, goals_t, no_action_max):
    """``set_agents`` for Q rows.  Without a list ``set_agents`` binds Q = M; rows 0 .. Q - 1 on slots 0 .. Q - 1 with
    Q < M only exist at the C level, so they are bound there, with row state arrays of Q rows in ``w._agents``."""
    import torch

    if obs_t is not None or Q == w.M:
        w.set_agents(obs_t, goals_t, 0.95, no_action_max)
        return
    f32, dev = torch.float32, w.device
    a = dict(observers=None, goals=goals_t, Q=Q, last_pose=torch.zeros((w.N, Q, 4), dtype=f32, device=dev),
             noact_count=torch.zeros((w.N, Q), dtype=torch.int32, device=dev),
             retired_type=torch.full((w.N, w.M), O.INACTIVE, dtype=torch.uint8, device=dev),
             max_iou=torch.full((w.N, Q), -float("inf"), dtype=f32, device=dev),
             min_dist=torch.full((w.N, Q), float("inf"), dtype=f32, device=dev))
    assert w.lib.t2d_set_agents(w._ctx, None, Q, _p(goals_t), 0.95, no_action_max, _p(a["last_pose"]),
                                _p(a["noact_count"]), _p(a["retired_type"])) == 0
    w._agents = a


def _sel(n):
    """The scenarios held to an oracle: the first and the last (in the last, partial CTA) and one between."""
    return np.unique([0, n // 2, n - 1])


# ------------------------------------------------------------------ K11
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_k11_scatter_bit_for_bit(cuda_device, case):
    import torch

    N, M, Q, listed = case
    s = S.scene(N, M, 10)
    w, _ = _world(s)
    obs, obs_t = _list(case, s, 11)
    rng = np.random.default_rng(12)
    base = _random_bits(rng, (N, M, 2))
    rows = _random_bits(rng, (N, Q, 2))
    act = Guarded((N, M, 2), TAIL * M * 2, "float32")
    act.body.copy_(torch.from_numpy(base).view(torch.float32))
    rows_t = torch.from_numpy(rows).cuda()
    assert w.lib.t2d_scatter_agent_action(w._ctx, _p(obs_t), Q, _p(rows_t), act.ptr, w._stream()) == 0
    torch.cuda.synchronize()
    types = w.type_id.cpu().numpy()
    ref = scatter_agent_action(base, rows, types, len(w.type_table), obs)
    assert np.array_equal(_bits(act.body), _bits(ref))   # the owned slots take their row, every other slot keeps its bits
    tail = act.bits()[act.n:]
    assert bool((tail == SENTINEL["float32"]).all())
    written = (owner_rows(types, Q, obs) < Q) & (types < len(w.type_table))
    assert written.any()
    if M > 96 and Q > 96:
        assert written[:, 96:].any()   # slots a lane owns at k = 3
    w.close()


# ------------------------------------------------------------------ K10
class K10Out:
    def __init__(self, N, M, Q):
        self.reward = Guarded((N, Q), TAIL * Q, "float32")
        self.terminated = Guarded((N, Q), TAIL * Q, "uint8")
        self.truncated = Guarded((N, Q), TAIL * Q, "uint8")
        self.status = Guarded((N, Q), TAIL * Q, "uint8")
        self.iou = Guarded((N, Q), TAIL * Q, "float32")
        self.done = Guarded((N,), TAIL, "uint8")
        self.traffic = Guarded((N, M), TAIL * M, "uint8")
        self.all = dict(reward=self.reward, terminated=self.terminated, truncated=self.truncated, status=self.status,
                        iou=self.iou, done=self.done, traffic=self.traffic)

    def call(self, w, flags):
        import torch

        a = w._agents
        assert a["max_iou"].shape == self.reward.shape and w.M == self.traffic.shape[1]   # K10 writes the bound N·Q rows
        for g in self.all.values():
            g.fill()
        rc = w.lib.t2d_agents_epilogue(w._ctx, _p(flags), self.reward.ptr, self.terminated.ptr, self.truncated.ptr,
                                       self.status.ptr, self.iou.ptr, self.done.ptr, _p(a["max_iou"]), _p(a["min_dist"]),
                                       self.traffic.ptr, 1, w._stream())
        assert rc == 0
        torch.cuda.synchronize()
        for k, g in self.all.items():
            g.check(k)


def _k10_parity(w, out, flags_np, sel, observers, goals, no_action_max):
    """One K10 call, teacher-forced: the oracle starts from the device's type ids and row state before the call."""
    import torch

    a_ = w._agents
    pre = {k: a_[k].cpu().numpy()[sel] for k in ("last_pose", "noact_count", "max_iou", "min_dist", "retired_type")}
    pre_type = w.type_id.cpu().numpy()[sel]
    out.call(w, torch.from_numpy(flags_np).cuda())
    st = w.state_numpy()
    ref = R.agents_epilogue(flags_np[sel], pre_type, st["x"][sel], st["y"][sel], st["heading"][sel],
                            w.step_count.cpu().numpy()[sel], w.type_table.as_oracle_table(), len(w.type_table),
                            observers=_rows_of(observers, w.N, goals.shape[1])[sel], goals=goals[sel],
                            last_pose=pre["last_pose"], noact_count=pre["noact_count"], max_iou=pre["max_iou"],
                            min_dist=pre["min_dist"], retired=pre["retired_type"], max_step=w.max_step, threshold=0.95,
                            no_action_max=no_action_max)
    got = lambda g: g.body.cpu().numpy()[sel]
    assert np.abs(got(out.iou) - ref["iou"]).max() <= 2e-6
    ok = ~(np.abs(ref["iou"] - 0.95) <= 1e-6).any(1)   # scenarios no IoU puts at the threshold
    assert ok.any()
    for k in ("status", "terminated", "truncated"):
        assert np.array_equal(got(getattr(out, k))[ok], ref[k][ok]), k
    assert np.array_equal(got(out.done)[ok], ref["done"][ok])
    assert np.array_equal(w.type_id.cpu().numpy()[sel][ok], ref["type_id"][ok])
    assert np.array_equal(a_["retired_type"].cpu().numpy()[sel][ok], ref["retired"][ok])
    rw = got(out.reward)[ok]
    assert np.allclose(rw, ref["reward"][ok], rtol=1e-6, atol=5e-6), np.abs(rw - ref["reward"][ok]).max()
    mi, md = a_["max_iou"].cpu().numpy()[sel][ok], a_["min_dist"].cpu().numpy()[sel][ok]
    assert np.allclose(mi, ref["max_iou"][ok], rtol=0, atol=2e-6, equal_nan=False)
    assert np.allclose(md, ref["min_dist"][ok], rtol=1e-6, atol=1e-6)
    assert np.array_equal(got(out.traffic), ref["traffic"])
    return ref, got(out.status)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_k10_crafted_flags_retirement_and_restore(cuda_device, case):
    """Five K10 calls on crafted flags (no tick): flags of every kind on slots >= 96, goals at the slot's pose (COMPLETED),
    still rows with no_action_max = 2 (NO_ACTION from the fourth call), a scenario past max_step; then a masked reset
    that restores the retired slots, and one more call."""
    import torch

    N, M, Q, listed = case
    s = S.scene(N, M, 20)
    w, pool = _world(s, max_step=4)
    obs, obs_t = _list(case, s, 21)
    rng = np.random.default_rng(22)
    st = w.state_numpy()
    goals = S.k10_goals(rng, st["x"], st["y"], st["heading"], w.type_id.cpu().numpy(), w.type_table.as_oracle_table(), obs,
                        Q)
    goals_t = torch.from_numpy(goals).cuda()
    _bind_agents(w, obs_t, Q, goals_t, 2)
    assert w._agents["max_iou"].shape == (N, Q)   # the outputs below are sized for the bound Q
    out = K10Out(N, M, Q)
    sel = _sel(N)
    types0 = w.type_id.cpu().numpy()
    seen = {}   # status -> rows q at which it was seen
    for t in range(5):
        if t >= 1:
            w.x[:, 1::2] += 0.7   # odd slots move, even slots stand still
        if t == 4:
            w.step_count[N - 1] = 5   # past max_step: TIME_EXCEEDED for every present row of the last scenario
        flags = S.k10_flags(rng, N, M, t)
        if t == 0 and M >= 100:
            assert all(S.flag_coverage(flags).values())
        _, status = _k10_parity(w, out, flags, sel, obs, goals, 2)
        full = out.status.body.cpu().numpy()
        for v in np.unique(full):
            seen.setdefault(int(v), set()).update(np.nonzero((full == v).any(0))[0].tolist())
    retired = w.type_id.cpu().numpy() == O.INACTIVE
    gone = retired & (types0 != O.INACTIVE)
    assert gone.any()
    if not listed and Q >= 100:
        assert max(seen[O.NO_ACTION]) >= 64 and max(seen[O.COMPLETED]) >= 64, seen
        assert max(seen[O.FAILED]) >= 96 and max(seen[O.OUT_BOUND]) >= 96 and O.TIME_EXCEEDED in seen, seen
        assert gone[:, 96:].any(1).all()
    # the masked reset restores the retired slots of the even scenarios
    a_ = w._agents
    mask = (np.arange(N) % 2 == 0).astype(np.uint8)
    ref = R.reset(mask, w.type_id.cpu().numpy(), a_["retired_type"].cpu().numpy(), a_["last_pose"].cpu().numpy(),
                  a_["noact_count"].cpu().numpy())
    w.reset(torch.from_numpy(mask).cuda(), pool)
    torch.cuda.synchronize()
    assert np.array_equal(w.type_id.cpu().numpy(), ref[0]) and np.array_equal(a_["retired_type"].cpu().numpy(), ref[1])
    assert np.array_equal(a_["last_pose"].cpu().numpy()[..., 3], ref[2][..., 3])
    assert np.array_equal(a_["noact_count"].cpu().numpy(), ref[3])
    assert np.array_equal(ref[0][mask == 1], types0[mask == 1])
    if M > 96 and (listed or Q > 96):   # (without a list, Q = 1 is slot 0 alone)
        back = gone & (mask[:, None] == 1)
        assert back[:, 96:].any()   # slots >= 96 retired, then restored
    _k10_parity(w, out, np.zeros((N, M), np.uint8), sel, obs, goals, 2)
    w.close()


@pytest.mark.gpu
def test_k10_done_mask_waits_for_row_127(cuda_device):
    """M = Q = 128, every slot a row: even scenarios have every row settled but q = 127 (lane 31, k = 3), odd ones every
    row.  done is 0 and 1."""
    N, M = 13, 128
    s = S.scene(N, M, 30)
    w, _ = _world(s)
    w.set_agents()
    flags = np.full((N, M), O.F_STATIC, np.uint8)
    flags[0::2, 127] = 0
    out = K10Out(N, M, M)
    goals = np.full((N, M, 5), np.nan, np.float32)
    ref, status = _k10_parity(w, out, flags, np.arange(N), None, goals, 100)
    done = out.done.body.cpu().numpy()
    assert np.array_equal(done, (np.arange(N) % 2).astype(np.uint8))
    assert (status[0::2, 127] == O.NORMAL).all() and (status[1::2, 127] == O.FAILED).all()
    assert ((status[:, :127] == O.FAILED) | (status[:, :127] == 0)).all()
    w.close()


# ------------------------------------------------------------------ K4
def _beams(n_beams):
    import torch

    theta = np.linspace(0, 2 * np.pi, n_beams, endpoint=False)
    return torch.from_numpy(np.stack([np.cos(theta), np.sin(theta)], 1)).cuda().contiguous()


def _state_world(s):
    from tactics2d_b200 import BatchedWorld

    n, m = s.shape
    w = BatchedWorld(n, m, s.table)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    return w


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_k4_observer_rows(cuda_device, case):
    import torch

    N, M, Q, listed = case
    s = S.scene(N, M, 40)
    w = _state_world(s)
    obs, obs_t = _list(case, s, 41)
    nb, rng_m = 360, S.lidar_range(M)
    scan = Guarded((N, Q, nb), TAIL * nb, "float32")
    assert w.lib.t2d_lidar_scan_agents(w._ctx, _p(obs_t), Q, nb, rng_m, _p(_beams(nb)), scan.ptr, w._stream()) == 0
    torch.cuda.synchronize()
    scan.check("scan")
    sel = _sel(N)
    rng = np.random.default_rng(42)
    rows = np.unique([q for q in SEL_ROWS if q < Q] + rng.integers(0, Q, 4).tolist() + [Q - 1])
    slots = np.broadcast_to(rows, (N, len(rows))) if obs is None else obs[:, rows]
    st = w.state_numpy()
    f64 = lambda k: st[k][sel].astype(np.float64)
    ref = AL.scan_agents(f64("x"), f64("y"), f64("heading"), s.type_id[sel], w.type_table.as_oracle_table(), nb, rng_m,
                         observers=slots[sel], segments=s.segments)
    AL.compare(scan.body.cpu().numpy()[sel][:, rows], ref, rng_m)
    assert np.isfinite(ref).any()
    if M == 128:   # most of the other 127 boxes lie within reach of the rows held to the oracle
        x, y = st["x"][sel].astype(np.float64), st["y"][sel].astype(np.float64)
        j = np.clip(slots[sel].astype(np.int64), 0, M - 1)
        d = np.hypot(x[:, None, :] - np.take_along_axis(x, j, 1)[..., None],
                     y[:, None, :] - np.take_along_axis(y, j, 1)[..., None])
        assert ((d <= rng_m).sum(-1) - 1).mean() > 100
    w.close()


@pytest.mark.gpu
def test_k4_ego_scan_at_m128_and_ragged_n(cuda_device):
    import torch

    N, M = 4099, 128
    s = S.scene(N, M, 45)
    w = _state_world(s)
    nb, rng_m = 360, S.lidar_range(M)
    scan = Guarded((N, nb), TAIL * nb, "float32")
    assert w.lib.t2d_lidar_scan(w._ctx, nb, rng_m, _p(_beams(nb)), scan.ptr, w._stream()) == 0
    torch.cuda.synchronize()
    scan.check("scan")
    sel = np.asarray([0, 1, 2049, N - 3, N - 2, N - 1])
    st = w.state_numpy()
    f64 = lambda k: st[k][sel].astype(np.float64)
    ref = OL.scan_world(f64("x"), f64("y"), f64("heading"), s.type_id[sel], w.type_table.as_oracle_table(), s.segments, nb,
                        rng_m)
    AL.compare(scan.body.cpu().numpy()[sel], ref, rng_m)
    # the per-agent entry with one row on slot 0 is the same scan
    again = Guarded((N, 1, nb), TAIL * nb, "float32")
    assert w.lib.t2d_lidar_scan_agents(w._ctx, None, 1, nb, rng_m, _p(_beams(nb)), again.ptr, w._stream()) == 0
    torch.cuda.synchronize()
    again.check("scan")
    assert torch.equal(again.body[:, 0], scan.body)
    w.close()


# ------------------------------------------------------------------ K9
K9_CASES = [c for c in CASES if c[2] in (33, 97, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", K9_CASES, ids=[S.case_id(c) for c in K9_CASES])
def test_k9_observer_rows(cuda_device, case):
    import torch
    from tactics2d_b200 import _lib

    N, M, Q, listed = case
    s = S.scene(N, M, 50)
    w = _state_world(s)
    obs, obs_t = _list(case, s, 51)
    rng = np.random.default_rng(52)
    st = w.state_numpy()
    goals = S.k10_goals(rng, st["x"], st["y"], st["heading"], s.type_id, w.type_table.as_oracle_table(), obs, Q)
    goals_t = torch.from_numpy(goals).cuda()
    assert goals.shape == (N, Q, 5)
    K, Sg, ra, rs = 16, 32, 50.0, 30.0
    F = V.width(K, Sg)
    out = Guarded((N, Q, F), TAIL * F, "float32")
    ai = Guarded((N, Q, K), TAIL * K, "int16")
    si = Guarded((N, Q, Sg), TAIL * Sg, "int16")
    cfg = _lib.ObsConfigC(K, Sg, ra, rs)
    assert w.lib.t2d_observe_agents(w._ctx, C.byref(cfg), _p(obs_t), Q, _p(goals_t), out.ptr, ai.ptr, si.ptr,
                                    w._stream()) == 0
    torch.cuda.synchronize()
    for name, g in (("out", out), ("agent_index", ai), ("segment_index", si)):
        g.check(name)
    sel = _sel(N)
    ref, rai, rsi = A.observe_agents({k: v[sel] for k, v in st.items()}, s.type_id[sel], V.table_of(w.type_table), K, Sg,
                                     ra, rs, observers=_rows_of(obs, N, Q)[sel],
                                     step_count=w.step_count.cpu().numpy()[sel], max_step=w.max_step, goals=goals[sel],
                                     tiles=[dict(segments=s.segments, poly_start=None)])
    assert np.array_equal(ai.body.cpu().numpy()[sel], rai) and np.array_equal(si.body.cpu().numpy()[sel], rsi)
    V.compare(out.body.cpu().numpy()[sel].reshape(-1, F), ref.reshape(-1, F), K, Sg)
    assert (rai >= 0).any() and (rsi >= 0).any()
    w.close()


# ------------------------------------------------------------------ the multi-agent step at M = Q = 128
def _idm(w, observers, seed):
    """IDM on every slot no row names, each following a random slot that a row names."""
    from tactics2d_b200.controller import IDMController

    rng = np.random.default_rng(seed)
    named = owner_rows(w.type_id.cpu().numpy(), observers.shape[1], observers) < observers.shape[1]
    cid = np.where(named, 255, 0).astype(np.uint8)
    lead = np.full((w.N, w.M), -1, np.int16)
    for n in range(w.N):
        agents = np.nonzero(named[n])[0]
        if len(agents):
            lead[n] = rng.choice(agents, w.M)
    w.set_controllers([IDMController()], cid, lead_index=lead)
    return named


@pytest.mark.gpu
def test_step_chain_at_m128_q128_against_the_oracles(cuda_device):
    """scatter -> control (IDM followers of agents) -> tick -> K10 -> reset -> K9 and K4, each held to its oracle."""
    import torch
    from tactics2d_b200 import synthetic

    N, M, Q = 13, 128, 128
    s = S.scene(N, M, 60)
    w, pool = _world(s, max_step=5)
    obs = S.observer_list(np.random.default_rng(61), s.type_id, Q)
    obs_t = torch.from_numpy(obs).cuda()
    rng = np.random.default_rng(62)
    st = w.state_numpy()
    goals = S.k10_goals(rng, st["x"], st["y"], st["heading"], s.type_id, w.type_table.as_oracle_table(), obs)
    w.set_agents(obs_t, torch.from_numpy(goals).cuda(), 0.95, 100)
    named = _idm(w, obs, 63)
    assert (~named).any()
    table, n_types = w.type_table.as_oracle_table(), len(w.type_table)
    act = torch.zeros((N, M, 2), device=cuda_device)
    sel = _sel(N)
    rows_sel = np.asarray([0, 5, 64, 97, 100, 126, 127])
    settled = resets = 0
    for t in range(7):
        rows = synthetic.random_actions(640 + t, (N, Q))
        before = act.cpu().numpy()
        types = w.type_id.cpu().numpy()
        w.scatter_agent_action(torch.from_numpy(rows).cuda(), act, obs_t)
        torch.cuda.synchronize()
        assert np.array_equal(_bits(act), _bits(scatter_agent_action(before, rows, types, n_types, obs))), t
        w.control(act)
        w.step(act)
        a_ = w._agents
        pre = {k: a_[k].cpu().numpy()[sel] for k in ("last_pose", "noact_count", "max_iou", "min_dist", "retired_type")}
        pre_type = w.type_id.cpu().numpy()[sel]
        a = w.agents_epilogue()
        torch.cuda.synchronize()
        st = w.state_numpy()
        ref = R.agents_epilogue(w.result.flags.cpu().numpy()[sel], pre_type, st["x"][sel], st["y"][sel], st["heading"][sel],
                                w.step_count.cpu().numpy()[sel], table, n_types, observers=obs[sel], goals=goals[sel],
                                last_pose=pre["last_pose"], noact_count=pre["noact_count"], max_iou=pre["max_iou"],
                                min_dist=pre["min_dist"], retired=pre["retired_type"], max_step=w.max_step)
        ok = ~(np.abs(ref["iou"] - 0.95) <= 1e-6).any(1)
        for k in ("status", "terminated", "truncated"):
            assert np.array_equal(getattr(a, k).cpu().numpy()[sel][ok], ref[k][ok]), (t, k)
        assert np.array_equal(a.done.cpu().numpy()[sel][ok], ref["done"][ok]), t
        assert np.array_equal(w.type_id.cpu().numpy()[sel][ok], ref["type_id"][ok]), t
        assert np.allclose(a.reward.cpu().numpy()[sel][ok], ref["reward"][ok], rtol=1e-6, atol=5e-6), t
        settled += int(((ref["status"] != O.NORMAL) & (ref["status"] != 0)).sum())
        resets += int(a.done.sum())
        w.reset(a.done, pool)
        # the observation and the lidar of the next step, from the post-reset world
        st = w.state_numpy()
        types = w.type_id.cpu().numpy()
        o = w.observe_agents(16, 32, 50.0, 30.0, observers=obs_t)
        torch.cuda.synchronize()
        ref_o, rai, rsi = A.observe_agents({k: v[sel] for k, v in st.items()}, types[sel], V.table_of(w.type_table), 16, 32,
                                           50.0, 30.0, observers=obs[sel], step_count=w.step_count.cpu().numpy()[sel],
                                           max_step=w.max_step, tiles=[dict(segments=s.segments, poly_start=None)])
        assert np.array_equal(o.agent_index.cpu().numpy()[sel], rai) and np.array_equal(o.segment_index.cpu().numpy()[sel], rsi)
        V.compare(o.flat.cpu().numpy()[sel].reshape(-1, o.flat.shape[2]), ref_o.reshape(-1, o.flat.shape[2]), 16, 32)
        scan = w.lidar_scan_agents(90, 150.0, observers=obs_t)
        torch.cuda.synchronize()
        f64 = lambda k: st[k][sel].astype(np.float64)
        ref_l = AL.scan_agents(f64("x"), f64("y"), f64("heading"), types[sel], table, 90, 150.0,
                               observers=obs[sel][:, rows_sel], segments=s.segments)
        AL.compare(scan.cpu().numpy()[sel][:, rows_sel], ref_l, 150.0)
    assert settled > 50 and resets > 0
    assert (w.last_accel.cpu().numpy()[~named] != 0).any()
    w.close()


@pytest.mark.gpu
@pytest.mark.parametrize("Q", [128, 97])
def test_step_host_agents_equals_the_device_path_at_m128(cuda_device, Q):
    """The packed read-back (7·N·Q + N bytes) at Q = 128 and at an odd Q, odd N, controllers set."""
    import torch
    from tactics2d_b200 import synthetic

    N, M = 13, 128
    s = S.scene(N, M, 70)
    obs = S.observer_list(np.random.default_rng(71), s.type_id, Q)
    obs_t = torch.from_numpy(obs).cuda()
    (wa, pa), (wb, pb) = _world(s, max_step=4), _world(s, max_step=4)
    st = wa.state_numpy()
    goals = torch.from_numpy(S.k10_goals(np.random.default_rng(72), st["x"], st["y"], st["heading"], s.type_id,
                                         wa.type_table.as_oracle_table(), obs)).cuda()
    for w in (wa, wb):
        w.set_agents(obs_t, goals, 0.95, 3)
        _idm(w, obs, 73)
    act_a, act_b = (torch.zeros((N, M, 2), device=cuda_device) for _ in range(2))
    resets = 0
    for t in range(8):
        rows = synthetic.random_actions(740 + t, (N, Q))
        reward, term, trunc, status, done = wa.step_host_agents(rows, act_a)
        wb.scatter_agent_action(torch.from_numpy(rows).cuda(), act_b, obs_t)
        wb.control(act_b)
        wb.step(act_b)
        e = wb.agents_epilogue()
        torch.cuda.synchronize()
        assert reward.shape == (N, Q) and done.shape == (N,)
        assert np.array_equal(_bits(reward), _bits(e.reward)), t
        assert np.array_equal(term, e.terminated.cpu().numpy()) and np.array_equal(trunc, e.truncated.cpu().numpy()), t
        assert np.array_equal(status, e.status.cpu().numpy()) and np.array_equal(done, e.done.cpu().numpy()), t
        for k in ("x", "y", "heading", "speed", "type_id", "step_count"):
            assert torch.equal(getattr(wa, k), getattr(wb, k)), (t, k)
        for k in ("max_iou", "min_dist", "retired_type", "last_pose", "noact_count"):
            assert torch.equal(wa._agents[k], wb._agents[k]), (t, k)
        assert torch.equal(act_a, act_b), t
        resets += int(done.sum())
        mask = torch.from_numpy(done.copy()).cuda()
        for w, pool in ((wa, pa), (wb, pb)):
            w.reset(mask, pool)
    assert resets >= N
    for w in (wa, wb):
        w.close()


@pytest.mark.gpu
def test_env_at_m128_q128_equals_the_world_sequence(cuda_device):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    N, M, Q = 5, 128, 128
    s = S.scene(N, M, 80)
    obs = S.observer_list(np.random.default_rng(81), s.type_id, Q)
    obs_t = torch.from_numpy(obs).cuda()
    goals = torch.from_numpy(S.k10_goals(np.random.default_rng(82), s.x, s.y, s.heading, s.type_id,
                                         s.table.as_oracle_table(), obs)).cuda()
    vo = dict(k_agents=16, k_segments=32, observers=obs_t, goals=goals)
    lidar = dict(n_beams=90, max_range=150.0)
    env = BatchedTrafficEnv(s, max_step=4, observation="agents", vector_obs=vo, agent_rewards=True, agent_actions=True,
                            lidar=lidar)
    # the same sequence on a world of its own
    w = BatchedWorld(N, M, s.table, max_step=4, steer_first=True)
    w.set_map(s.segments, s.bounds)
    pool = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in s.state().items()}
    w.set_agents(obs_t, goals, 0.95, 100)
    w.type_id.copy_(torch.from_numpy(s.type_id).cuda())
    w.reset(torch.ones(N, dtype=torch.uint8, device="cuda"), pool)
    act = torch.zeros((N, M, 2), device=cuda_device)
    o_env, info = env.reset()
    assert torch.equal(o_env, w.observe_agents(**vo).flat)
    assert torch.equal(info["lidar"], w.lidar_scan_agents(**lidar, observers=obs_t))
    resets = 0
    for t in range(9):
        rows = torch.from_numpy(synthetic.random_actions(840 + t, (N, Q))[..., ::-1].copy()).cuda()   # (steer, accel)
        o_env, r_env, te_env, tr_env, info = env.step(rows)
        w.scatter_agent_action(rows, act, obs_t)
        w.step(act)
        a = w.agents_epilogue()
        assert np.array_equal(_bits(r_env), _bits(a.reward)), t
        assert torch.equal(te_env, a.terminated) and torch.equal(tr_env, a.truncated), t
        assert torch.equal(info["agent_status"], a.status) and torch.equal(info["agent_iou"], a.iou), t
        assert torch.equal(info["traffic_status"], a.traffic), t
        resets += int(a.done.sum())
        w.reset(a.done, pool)
        assert torch.equal(o_env, w.observe_agents(**vo).flat), t
        assert torch.equal(info["lidar"], w.lidar_scan_agents(**lidar, observers=obs_t)), t
        for k in ("x", "y", "heading", "speed", "type_id", "step_count"):
            assert torch.equal(getattr(env.world, k), getattr(w, k)), (t, k)
    assert resets >= N
    env.close()
    w.close()
