"""Restatement of the sampled reset (K13 -> K2 / K7 -> K14; DESIGN.md section 1 "Sampled resets"), TEST INFRASTRUCTURE ONLY.

* ``philox``: Philox4x32-10 in Python integers (NumPy uint64 lanes), key (seed low, seed high), counter (d, n, e, 0);
* ``row_draw``: the multiply-high row of draw 0;
* ``draw_range`` / ``wrap_two_pi`` / ``candidate``: the float32 jitter arithmetic, one rounding per operation;
* ``place``: the sequential placement, each try decided by ``oracle.scenario.events`` (the slot's flags at the candidate,
  the other slots at their current state) and, for the ego with ``avoid_target``, the target box of ``oracle.geometry``;
* ``reset_sampled``: the whole masked chain on an env snapshot: the draw, ``tests.env_chain_oracle.reset``, the placement.
"""

from __future__ import annotations

import numpy as np

from oracle import geometry as G
from oracle import scenario as O
from tests import env_chain_oracle as EC

M32 = np.uint64(0xFFFFFFFF)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)


def philox(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 of the counters (c0, c1, c2, c3) under the key (k0, k1); every argument broadcasts.  Returns the
    four output words as uint32 arrays."""
    c = [np.asarray(v, dtype=np.uint64) & M32 for v in (c0, c1, c2, c3)]
    k0, k1 = np.asarray(k0, dtype=np.uint64) & M32, np.asarray(k1, dtype=np.uint64) & M32
    for _ in range(10):
        p0, p1 = _M0 * c[0], _M1 * c[2]   # < 2^64: exact in uint64
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & M32, p1 & M32, ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & M32, p0 & M32]
        k0, k1 = (k0 + _W0) & M32, (k1 + _W1) & M32
    return tuple(v.astype(np.uint32) for v in c)


def draw(seed: int, d, n, e):
    """The four words of draw d of scenario n in its episode e."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return philox(d, n, e, 0, seed & 0xFFFFFFFF, seed >> 32)


def row_draw(seed: int, n, e, P: int):
    """Pool row of scenario n in episode e over P rows: (u0 P) >> 32."""
    u0 = draw(seed, 0, n, e)[0].astype(np.uint64)
    return ((u0 * np.uint64(P)) >> np.uint64(32)).astype(np.int64)


def unit(u):
    """(u >> 8) 2^-24 in float32."""
    return (np.asarray(u, np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)


def draw_range(u, lo, hi):
    lo, hi = np.float32(lo), np.float32(hi)
    return (lo + unit(u) * (hi - lo)).astype(np.float32)


def fma32(a, b, c):
    """fmaf: a b + c rounded once to float32.  a b is exact in float64; the float64 sum's rounding error is recovered
    (TwoSum) and decides the one case the second rounding could get wrong, a float64 sum exactly halfway between two
    float32 numbers."""
    a, b, c = (np.asarray(v, dtype=np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bv = s - p
    err = (p - (s - bv)) + (c - bv)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    other = np.nextafter(r, np.where(s > r64, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    tie = (s != r64) & (s == (r64 + other.astype(np.float64)) / 2.0) & (err != 0.0)
    toward_other = np.sign(err) == np.sign(other.astype(np.float64) - r64)
    return np.where(tie & toward_other, other, r).astype(np.float32)


TWO_PI_HI = np.float32(6.2831854820251465)
TWO_PI_LO = np.float32(-1.7484555e-7)
INV_TWO_PI = np.float32(0.15915494309189535)
RINT_MAGIC = np.float32(12582912.0)


def wrap_two_pi(phi):
    """t2d_math.cuh's wrap_two_pi in float32."""
    phi = np.asarray(phi, dtype=np.float32)
    q = ((fma32(phi, INV_TWO_PI, np.float32(-0.5)) + RINT_MAGIC) - RINT_MAGIC).astype(np.float32)
    r = fma32(-q, TWO_PI_HI, phi)
    r = fma32(-q, TWO_PI_LO, r)
    r = np.where(r < 0, (r + TWO_PI_HI).astype(np.float32), r)
    r = np.where(r >= TWO_PI_HI, (r - TWO_PI_HI).astype(np.float32), r)
    return np.where(r < 0, np.float32(0.0), r).astype(np.float32)


def candidate(seed, n, e, m, tries, jit, x, y, h, v):
    """The candidates of tries 0 .. tries-1 of slot m: float32 arrays (x, y, heading, speed) [tries]."""
    u = draw(seed, 1 + 32 * m + np.arange(tries), n, e)
    j = np.asarray(jit, dtype=np.float32).reshape(8)
    f32 = np.float32
    cx = (f32(x) + draw_range(u[0], j[0], j[1])).astype(f32)
    cy = (f32(y) + draw_range(u[1], j[2], j[3])).astype(f32)
    ch = wrap_two_pi((f32(h) + draw_range(u[2], j[4], j[5])).astype(f32))
    cv = (f32(v) + draw_range(u[3], j[6], j[7])).astype(f32)
    return cx, cy, ch, cv


def blocked(x, y, h, type_id, m, table, segments=None, bounds=None, poly_start=None, target=None):
    """[T] bool: would check_events flag slot m in each row of the [T, M] poses (slot m at its candidate, the others at
    their current state)?  ``target`` (cx, cy, heading, half_len, half_wid): slot m must not meet that box either."""
    tid = np.asarray(type_id)
    dyn = O.events(x, y, h, tid, table)[0][:, m] != 0
    one = lambda a: np.ascontiguousarray(a[:, m:m + 1])
    st = O.events(one(x), one(y), one(h), one(tid), table, segments, bounds, poly_start=poly_start)[0][:, 0] != 0
    out = dyn | st
    if target is not None:
        row = int(tid[0, m])
        xs, ys, hs = (np.asarray(a[:, m], np.float64) for a in (x, y, h))
        c, s = np.cos(hs), np.sin(hs)
        tx, ty, th, tl, tw = (float(np.float32(v)) for v in target)
        tc, ts = np.cos(th), np.sin(th)
        if table["shape"][row] == O.CIRCLE:
            hit = G.obb_circle(tx, ty, tc, ts, tl, tw, xs, ys, table["radius"][row])
        else:
            hit = G.obb_obb(xs, ys, c, s, table["half_len"][row], table["half_wid"][row], tx, ty, tc, ts, tl, tw)
        out = out | (np.asarray(hit) & (table["shape"][row] != O.NOSHAPE))
    return out


def place(snap, mask, episode, seed, jitter, tries, table, n_types, scene_of, target=None, avoid_target=False,
          reset_try=None, pool_wheels=False):
    """K14 on a snapshot after K2 (and K7): returns (snapshot', reset_try [N, M] int8, episode' [N] uint32).
    ``scene_of(n)`` -> (segments, bounds, poly_start) of scenario n's tile; ``target`` [N, 5] or None; ``reset_try``: the
    tries of the previous reset, which the unmasked scenarios keep (default all -1); ``pool_wheels``: the reset took wheel
    speeds from a pool, which a moved slot keeps (else a moved drift slot rolls freely at its new speed)."""
    out = {k: np.array(v, copy=True) for k, v in snap.items()}
    N, M = out["x"].shape
    rt = np.full((N, M), -1, np.int8) if reset_try is None else np.array(reset_try, np.int8, copy=True)
    ep = np.array(episode, dtype=np.uint32, copy=True)
    jit = None if jitter is None else np.asarray(jitter, np.float32).reshape(M, 8)
    for n in np.nonzero(np.asarray(mask).astype(bool))[0]:
        e = int(ep[n])
        rt[n] = -1
        if jit is not None:
            segs, bounds, ps = scene_of(n)
            for m in range(M):
                t = int(out["type_id"][n, m])
                if t >= n_types or not jit[m].any():
                    continue
                cx, cy, ch, cv = candidate(seed, n, e, m, tries, jit[m], out["x"][n, m], out["y"][n, m],
                                           out["heading"][n, m], out["speed"][n, m])
                if table["shape"][t] == O.NOSHAPE:
                    ok = np.ones(tries, bool)
                else:
                    rows = lambda k: np.repeat(out[k][n][None], tries, 0).astype(np.float32)
                    X, Y, H = rows("x"), rows("y"), rows("heading")
                    X[:, m], Y[:, m], H[:, m] = cx, cy, ch
                    tid = np.repeat(out["type_id"][n][None], tries, 0)
                    tg = target[n] if (avoid_target and m == 0 and target is not None) else None
                    ok = ~blocked(X, Y, H, tid, m, table, segs, bounds, ps, tg)
                if not ok.any():
                    continue
                w = int(np.argmax(ok))
                rt[n, m] = w
                out["x"][n, m], out["y"][n, m], out["heading"][n, m], out["speed"][n, m] = cx[w], cy[w], ch[w], cv[w]
                out["vx"][n, m] = np.float32(cv[w] * np.cos(np.float64(ch[w])))
                out["vy"][n, m] = np.float32(cv[w] * np.sin(np.float64(ch[w])))
                if "omega_wf" in out and not pool_wheels and table["model"][t] == O.DRIFT:
                    wv = np.float32(cv[w] / np.float32(table["wheel_radius"][t]))
                    out["omega_wf"][n, m] = out["omega_wr"][n, m] = wv
        ep[n] = np.uint32(e + 1)
    return out, rt, ep


def pool_rows(mask, episode, seed, P, sample_rows=True):
    """K13's row of every scenario ([N] int64; only the masked entries are meaningful)."""
    N = len(mask)
    if not sample_rows:
        return np.minimum(np.arange(N), P - 1)
    return row_draw(seed, np.arange(N), np.asarray(episode, np.uint32), P)


def reset_sampled(snap, mask, pool, ctx, seed, episode, pool_row, jitter=None, tries=8, sample_rows=True,
                  avoid_target=False, row_pools=None, scene_of=None):
    """The masked chain on an env snapshot: K13 (the row and the row-owned columns ``row_pools`` = dict of
    ``type_id`` [P, M], ``target`` [P, 5], ``tile_id`` [P], ``route_id`` [P, M], each optional; their snapshot keys are
    ``type_id``, ``target``, ``tile_id``, ``route_id``), K2 via ``tests.env_chain_oracle.reset``, then K14.  Returns
    (snapshot', pool_row', reset_try, episode')."""
    m = np.asarray(mask).astype(bool)
    P = pool["x"].shape[0]
    rows = pool_rows(m, episode, seed, P, sample_rows)
    pr = np.array(pool_row, dtype=np.int32, copy=True)
    pr[m] = rows[m]
    s = {k: np.array(v, copy=True) for k, v in snap.items()}
    for k, src in (row_pools or {}).items():
        if src is not None:
            s[k][m] = np.asarray(src)[rows[m]]
    if row_pools and row_pools.get("type_id") is not None and "retired" in s:
        s["retired"][m] = 255
    s = EC.reset(s, m, pool, pr, ctx)
    tgt = s.get("target", ctx.get("target"))
    out, rt, ep = place(s, m, episode, seed, jitter, tries, ctx["table"], ctx["n_types"], scene_of, tgt, avoid_target)
    return out, pr, rt, ep
