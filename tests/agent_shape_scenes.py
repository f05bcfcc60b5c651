"""Shapes, scenes, observer lists and crafted K10 inputs for tests/test_gpu_agent_shapes.py (TEST INFRASTRUCTURE ONLY).

The multi-agent kernels give one warp a scenario (K10, K11) or an observer row (K4, K9), and lane l owns the rows and slots
l, l + 32, l + 64 and l + 96 (k = 0 .. 3).  The shapes below reach every k, the lists put their duplicates, absent rows and
the last slot into the upper lanes, and every N is odd, so that the last CTA of every launch is partial.  Each builder
asserts what it claims to cover (``list_coverage`` / ``require_list_coverage``, ``flag_coverage``); the CPU test of the
test file checks those claims on known inputs.  Everything is NumPy on the host, seeded."""

from __future__ import annotations

import numpy as np

from oracle import scenario as O

# (N, M, Q): every M of {1, 2, 33, 65, 96, 97, 127, 128}, every Q of {1, 32, 33, 64, 65, 96, 97, 127, 128} with a list and,
# where Q <= M, without one; N never a multiple of 4 (nor of 8: K10 and K11 run 8 scenarios per CTA, K4 and K9 4 rows).
SHAPES = [
    (1, 1, 1),
    (3, 2, 33),
    (5, 33, 32),
    (9, 33, 33),
    (13, 65, 64),
    (3, 65, 65),
    (5, 96, 96),
    (9, 97, 97),
    (13, 127, 127),
    (1, 128, 128),
    (4099, 128, 97),
    (5, 128, 1),
]


def cases():
    """(N, M, Q, listed) for every shape: with an observer list, and without one where Q <= M."""
    out = []
    for n, m, q in SHAPES:
        if q <= m:
            out.append((n, m, q, False))
        out.append((n, m, q, True))
    return out


def case_id(c):
    n, m, q, listed = c
    return f"N{n}-M{m}-Q{q}-{'list' if listed else 'slots'}"


def scene(n, m, seed):
    """A scene whose slots 0 and M - 1 are active boxes, with empty slots (type 255) at M - 2 (M >= 4) and at about 4 % of
    the slots 1 .. M - 3.  M = 128: ``synthetic.config5`` on the rounD_0 tile in a 140 m arena (most of the other 127 boxes
    within a 150 m lidar's reach of every slot); otherwise ``synthetic.config2`` in an arena scaled to M."""
    from tactics2d_b200 import synthetic

    if m == 128:
        from tactics2d_b200.map import load_collidable_segments

        seg, bounds = load_collidable_segments("rounD_0")
        s = synthetic.config5(n, m, seed=seed, segments=seg, bounds=bounds, size=140.0)
    else:
        s = synthetic.config2(n, m, seed=seed, size=max(30.0, 16.0 * np.ceil(np.sqrt(m))))
    tid = s.type_id.copy()
    rng = np.random.default_rng(seed + 1)
    if m >= 4:
        tid[:, m - 2] = O.INACTIVE
        inner = np.zeros((n, m), bool)
        inner[:, 1:m - 2] = rng.random((n, m - 3)) < 0.04
        tid[inner] = O.INACTIVE
    s.type_id = np.ascontiguousarray(tid)
    assert (tid[:, 0] != O.INACTIVE).all() and (tid[:, m - 1] != O.INACTIVE).all()
    return s


def lidar_range(m):
    """The lidar range the tests use on ``scene(., m, .)``."""
    return 150.0 if m == 128 else max(30.0, 16.0 * np.ceil(np.sqrt(m))) * 0.75


# rows of the duplicate pairs (winner, loser): winner and loser in different lanes and different k
PAIRS_LOW = ((2, 37),)                # k 0 / lane 2 against k 1 / lane 5 (Q >= 38)
PAIRS_HIGH = ((5, 97), (70, 100))     # k 0 / lane 5 against k 3 / lane 1, k 2 / lane 6 against k 3 / lane 4 (Q >= 104)
ABSENT_K2 = (65, 66, 67)              # -1, M, an empty slot (Q >= 69)
ABSENT_K3 = (98, 99, 101)             # the same in k = 3 (Q >= 104)


def observer_list(rng, types, Q):
    """int16 [N, Q] observer list over ``types`` (uint8 [N, M], 255 = empty) that reaches the upper lanes:

    * row Q - 1 observes slot M - 1 (slot 0 is active, so that row sees slot 0);
    * Q >= 97 and M >= 97: rows 96 .. Q - 1 observe active slots >= 96;
    * duplicate pairs whose lowest row is in another lane and another k than the losing row: (2, 37) when Q >= 38, and
      (5, 97), (70, 100) on slots >= 96 (M >= 100) when Q >= 104; no other row names a pair's slot;
    * -1, M and an empty slot at rows 65, 66, 67 (Q >= 69) and 98, 99, 101 (Q >= 104), else at the highest free rows;
    * every other row a random active slot.
    The list's coverage is asserted before it is returned."""
    types = np.asarray(types)
    N, M = types.shape
    obs = np.zeros((N, Q), np.int64)
    pairs = [p for p in PAIRS_LOW if Q >= 38] + [p for p in PAIRS_HIGH if Q >= 104]
    used = {Q - 1} | {q for p in pairs for q in p}
    if Q >= 69:
        absent = list(ABSENT_K2) + (list(ABSENT_K3) if Q >= 104 else [])
    else:
        absent = [q for q in range(Q - 2, -1, -1) if q not in used][:3]
    kinds = [-1, M, "empty"] * 2
    for n in range(N):
        act = np.nonzero(types[n] != O.INACTIVE)[0]
        empty = np.nonzero(types[n] == O.INACTIVE)[0]
        mid = act[(act != 0) & (act != M - 1)]
        high = mid[mid >= 96]
        pair_slots = []
        for i, _ in enumerate(pairs):
            pool = high if (i > 0 and len(high) > len(pairs)) else mid
            pool = np.setdiff1d(pool, pair_slots)
            pair_slots.append(int(rng.choice(pool)) if len(pool) else None)
        free = np.setdiff1d(act, [s for s in pair_slots if s is not None])
        obs[n] = rng.choice(free, Q)
        if Q >= 97 and M >= 97:
            up = np.setdiff1d(free[free >= 96], [])
            obs[n, 96:] = rng.choice(up, Q - 96)
        for (qa, qb), s in zip(pairs, pair_slots):
            if s is not None:
                obs[n, qa] = obs[n, qb] = s
        for q, kind in zip(absent, kinds):
            if kind == "empty":
                if len(empty):
                    obs[n, q] = rng.choice(empty)
            else:
                obs[n, q] = kind
        obs[n, Q - 1] = M - 1
    obs = obs.astype(np.int16)
    require_list_coverage(list_coverage(obs, types), M, Q)
    return obs


def list_coverage(observers, types, n_types=None):
    """What an observer list exercises, each fact holding in EVERY scenario: dict of bool."""
    obs = np.asarray(observers, np.int64)
    types = np.asarray(types)
    N, M = types.shape
    Q = obs.shape[1]
    n_types = O.INACTIVE if n_types is None else n_types
    active = types < n_types
    rows = np.arange(N)[:, None]
    q = np.broadcast_to(np.arange(Q), (N, Q))
    inr = (obs >= 0) & (obs < M)
    sl = np.where(inr, obs, 0)
    on_active = inr & active[rows, sl]
    owner = np.full((N, M), Q, np.int64)
    nn, qq = np.nonzero(inr)
    np.minimum.at(owner, (nn, obs[nn, qq]), qq)
    win = owner[rows, sl]
    cross = inr & (win < q) & (win % 32 != q % 32) & (win // 32 != q // 32)
    k = q // 32
    every = lambda a: bool(a.any(1).all())
    return dict(
        last_slot=every(on_active & (obs == M - 1)) and bool(active[:, 0].all()),
        upper_rows_on_upper_slots=every(on_active & (q >= 96) & (obs >= 96)),
        cross_duplicates=every(cross),
        k3_loses_to_k0=every(cross & (k == 3) & (win // 32 == 0) & (obs >= 96)),
        k3_loses_to_k2=every(cross & (k == 3) & (win // 32 == 2) & (obs >= 96)),
        minus_one_k2=every((obs == -1) & (k == 2)), m_k2=every((obs == M) & (k == 2)),
        empty_k2=every(inr & ~active[rows, sl] & (k == 2)),
        minus_one_k3=every((obs == -1) & (k == 3)), m_k3=every((obs == M) & (k == 3)),
        empty_k3=every(inr & ~active[rows, sl] & (k == 3)),
        minus_one=every(obs == -1), m=every(obs == M), empty=every(inr & ~active[rows, sl]))


def require_list_coverage(cov, M, Q):
    """Asserts the facts ``observer_list`` promises for an [N, Q] list over M slots."""
    need = ["last_slot"]
    if Q >= 97 and M >= 97:
        need.append("upper_rows_on_upper_slots")
    if Q >= 38:
        need.append("cross_duplicates")
    if Q >= 104 and M >= 100:
        need += ["k3_loses_to_k0", "k3_loses_to_k2"]
    if Q >= 5:
        need += ["minus_one", "m"] + (["empty"] if M >= 4 else [])
    if Q >= 69:
        need += ["minus_one_k2", "m_k2"] + (["empty_k2"] if M >= 4 else [])
    if Q >= 104:
        need += ["minus_one_k3", "m_k3"] + (["empty_k3"] if M >= 4 else [])
    missing = [k for k in need if not cov[k]]
    assert not missing, f"observer list (M={M}, Q={Q}) does not cover {missing}"
    return need


# ------------------------------------------------------------------ K10 inputs
FLAG_KINDS = (O.F_DYNAMIC, O.F_STATIC, O.F_OUTBOUND, O.F_STATIC | O.F_DYNAMIC, O.F_DYNAMIC | O.F_OUTBOUND)
UPPER_FLAGS = {96: O.F_STATIC, 97: O.F_DYNAMIC, 98: O.F_OUTBOUND, 99: O.F_STATIC | O.F_DYNAMIC | O.F_OUTBOUND}


def k10_flags(rng, n, m, call):
    """uint8 [N, M] event bytes for K10 call ``call``: calls 0, 1, 2 flag the slots m with m % 6 == call (a random kind
    each), call 0 also slots 96 .. 99 with static, dynamic, out-of-bound and all three; later calls flag nothing."""
    f = np.zeros((n, m), np.uint8)
    if call < 3:
        sel = np.arange(m) % 6 == call
        f[:, sel] = np.asarray(FLAG_KINDS, np.uint8)[rng.integers(0, len(FLAG_KINDS), (n, int(sel.sum())))]
    if call == 0:
        for s, v in UPPER_FLAGS.items():
            if s < m:
                f[:, s] = v
    return f


def flag_coverage(flags):
    """Which flag bits appear on slots >= 96 in every scenario."""
    up = np.asarray(flags)[:, 96:]
    return {b: bool(((up & b) != 0).any(1).all()) for b in (O.F_STATIC, O.F_DYNAMIC, O.F_OUTBOUND)}


def k10_goals(rng, x, y, h, types, table, observers, Q=None):
    """fp32 [N, Q, 5] goals (Q: the list's, else ``Q`` or M rows on slots 0 .. Q - 1): rows with q % 4 == 0 none (NaN
    cx), q % 4 == 1 their slot's own pose and extents (IoU 1: the row completes), the others 0.5 - 3 m off their slot."""
    types = np.asarray(types)
    N, M = types.shape
    Q = observers.shape[1] if observers is not None else (M if Q is None else Q)
    slot = np.broadcast_to(np.arange(Q), (N, Q)) if observers is None else np.clip(np.asarray(observers, np.int64), 0, M - 1)
    t = np.take_along_axis(types, slot, 1).astype(np.int64)
    hl_t, hw_t = np.asarray(table["half_len"], np.float32), np.asarray(table["half_wid"], np.float32)
    ok = t < len(hl_t)
    hl = np.where(ok, hl_t[np.where(ok, t, 0)], np.float32(2.4))
    hw = np.where(ok, hw_t[np.where(ok, t, 0)], np.float32(1.0))
    gx, gy, gh = (np.take_along_axis(np.asarray(a, np.float32), slot, 1) for a in (x, y, h))
    off = rng.uniform(0.5, 3.0, (N, Q)) * rng.choice([-1.0, 1.0], (N, Q))
    mode = np.arange(Q) % 4
    g = np.stack([np.where(mode == 1, gx, gx + off), np.where(mode == 1, gy, gy - 0.5 * off), gh, hl, hw], -1)
    g = g.astype(np.float32)
    g[:, mode == 0, 0] = np.nan
    return np.ascontiguousarray(g)
