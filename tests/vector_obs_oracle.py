"""Float64 NumPy statement of the vector observation (DESIGN.md section 1 "Vector observation"; K8, ``t2d_observe``).

Vectorised over scenarios.  Every value is an elementwise float64 operation (one rounding each, NumPy never contracts to
FMA) in the order the contract writes it, then rounded once to float32, so the selection, order, indices, valid, dist,
extents, speed, t_frac and in_ring are what the kernel must produce bit for bit; the rotated values go through libm's
sin / cos and may differ from the device's in the last bits (``rotated_tolerance``).
"""

from __future__ import annotations

import numpy as np

SHAPE_OBB, SHAPE_CIRCLE, SHAPE_NONE = 0, 1, 2
EGO_F, GOAL_F, AGENT_F, SEG_F = 8, 8, 11, 9

# columns that go through the ego's (or a heading difference's) sin / cos: checked within rotated_tolerance
EGO_ROTATED = (2, 3)
GOAL_ROTATED = (1, 2, 3, 4)
AGENT_ROTATED = (1, 2, 3, 4, 5, 6)
SEG_ROTATED = (1, 2, 3, 4, 5, 6)


def width(k_agents, k_segments):
    return EGO_F + GOAL_F + AGENT_F * k_agents + SEG_F * k_segments


def table_of(type_table):
    """The rows ``observe`` needs from a ``tactics2d_b200.types.TypeTable``."""
    return [dict(shape=r.shape, half_len=r.half_len, half_wid=r.half_wid, radius=r.radius) for r in type_table.rows]


def _extents(table, t):
    """(half_len, half_wid, is_disc) per type id (any shape array; ids >= len(table) give zeros)."""
    n = len(table)
    hl = np.zeros(n + 1, np.float32); hw = np.zeros(n + 1, np.float32); disc = np.zeros(n + 1, np.float32)
    shape = np.full(n + 1, SHAPE_NONE, np.int64)
    for i, r in enumerate(table):
        shape[i] = r["shape"]
        if r["shape"] == SHAPE_CIRCLE:
            hl[i] = hw[i] = np.float32(r["radius"]); disc[i] = 1.0
        elif r["shape"] == SHAPE_OBB:
            hl[i] = np.float32(r["half_len"]); hw[i] = np.float32(r["half_wid"])
    ti = np.minimum(np.asarray(t, np.int64), n)
    return hl[ti], hw[ti], disc[ti], shape[ti]


def _rot(c, s, dx, dy):
    return c * dx + s * dy, -s * dx + c * dy


def _seg_closest(x1, y1, x2, y2, x0, y0):
    ax, ay = x1 - x0, y1 - y0
    ux, uy = x2 - x1, y2 - y1
    uu = ux * ux + uy * uy
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(uu > 0, np.clip(-(ax * ux + ay * uy) / np.where(uu > 0, uu, 1.0), 0.0, 1.0), 0.0)
    px, py = ax + t * ux, ay + t * uy
    return px, py, px * px + py * py, ax, ay


def observe(state, type_id, table, k_agents, k_segments, agent_range, segment_range, step_count=None, max_step=0,
            target=None, tiles=(), tile_id=None):
    """state: dict of [N, M] arrays x, y, heading, speed, vx, vy (fp32 values); type_id [N, M]; table: list of dicts with
    shape, half_len, half_wid, radius (one per type row); tiles: list of dicts with segments [S, 4] (fp32) and poly_start
    ([P + 1] or None); tile_id [N] (None: tile 0).  Returns (flat float32 [N, F], agent_index int16 [N, K], segment_index
    int16 [N, S])."""
    f64 = lambda a: np.asarray(a, np.float32).astype(np.float64)
    x, y, h = f64(state["x"]), f64(state["y"]), f64(state["heading"])
    vx, vy, v = f64(state["vx"]), f64(state["vy"]), np.asarray(state["speed"], np.float32)
    tid = np.asarray(type_id, np.int64)
    N, M = tid.shape
    K, S = int(k_agents), int(k_segments)
    n_types = len(table)
    out = np.zeros((N, width(K, S)), np.float32)
    aidx = np.full((N, K), -1, np.int16)
    sidx = np.full((N, S), -1, np.int16)
    ego = tid[:, 0] < n_types
    x0, y0, h0 = x[:, :1], y[:, :1], h[:, :1]
    c, s = np.cos(h0), np.sin(h0)
    # ---- ego
    hl, hw, disc, _ = _extents(table, tid[:, 0])
    vl, vt = _rot(c[:, 0], s[:, 0], vx[:, 0], vy[:, 0])
    steps = np.zeros(N) if step_count is None else np.asarray(step_count, np.float64)
    tf = steps / float(max_step) if max_step > 0 else np.zeros(N)
    out[:, 0] = 1.0; out[:, 1] = v[:, 0]; out[:, 2] = vl; out[:, 3] = vt
    out[:, 4] = hl; out[:, 5] = hw; out[:, 6] = disc; out[:, 7] = tf
    # ---- goal
    if target is not None:
        g = np.asarray(target, np.float32).reshape(N, 5).astype(np.float64)
        dx, dy = g[:, 0] - x0[:, 0], g[:, 1] - y0[:, 0]
        ex, ey = _rot(c[:, 0], s[:, 0], dx, dy)
        dh = g[:, 2] - h0[:, 0]
        out[:, 8] = 1.0; out[:, 9] = ex; out[:, 10] = ey; out[:, 11] = np.cos(dh); out[:, 12] = np.sin(dh)
        out[:, 13] = g[:, 3]; out[:, 14] = g[:, 4]; out[:, 15] = np.sqrt(dx * dx + dy * dy)
    # ---- agents
    if K > 0:
        _, _, _, shape = _extents(table, tid)
        cand = (tid < n_types) & (shape != SHAPE_NONE)
        cand[:, 0] = False
        dx, dy = x - x0, y - y0
        with np.errstate(invalid="ignore"):
            d2 = dx * dx + dy * dy
            r = np.float64(np.float32(agent_range))
            inr = cand & (d2 <= r * r)
        key = np.where(inr, d2, np.inf)
        slot = np.broadcast_to(np.arange(M), (N, M))
        order = np.lexsort((slot, key), axis=-1)[:, :K]
        rows = np.arange(N)[:, None]
        keep = inr[rows, order]
        j = np.where(keep, order, 0)
        ahl, ahw, adisc, _ = _extents(table, tid[rows, j])
        ddx, ddy = dx[rows, j], dy[rows, j]
        ex, ey = _rot(c, s, ddx, ddy)
        wx, wy = _rot(c, s, vx[rows, j], vy[rows, j])
        dh = h[rows, j] - h0
        blk = np.stack([np.ones_like(ddx), ex, ey, np.cos(dh), np.sin(dh), wx, wy, ahl, ahw, adisc,
                        np.sqrt(ddx * ddx + ddy * ddy)], -1)
        blk = np.where(keep[..., None], blk, 0.0).astype(np.float32)
        pad = np.zeros((N, K, AGENT_F), np.float32)
        pad[:, :blk.shape[1]] = blk
        out[:, EGO_F + GOAL_F:EGO_F + GOAL_F + AGENT_F * K] = pad.reshape(N, -1)
        ai = np.where(keep, order, -1).astype(np.int16)
        aidx[:, :ai.shape[1]] = ai
    # ---- segments, one tile at a time
    if S > 0 and len(tiles) > 0:
        tids = np.zeros(N, np.int64) if tile_id is None else np.asarray(tile_id, np.int64)
        s0 = EGO_F + GOAL_F + AGENT_F * K
        for t, tile in enumerate(tiles):
            seg = tile.get("segments")
            if seg is None or len(seg) == 0:
                continue
            sel = np.nonzero(tids == t)[0]
            if sel.size == 0:
                continue
            seg = np.asarray(seg, np.float32).reshape(-1, 4).astype(np.float64)
            ns = seg.shape[0]
            ps = tile.get("poly_start")
            ring = np.zeros(ns, bool)
            if ps is not None and len(ps) >= 2:
                ring[int(ps[0]):int(ps[-1])] = True
            X0, Y0, C, Sn = x0[sel], y0[sel], c[sel], s[sel]
            x1, y1, x2, y2 = (seg[None, :, k] for k in range(4))
            px, py, d2, ax, ay = _seg_closest(x1, y1, x2, y2, X0, Y0)
            r = np.float64(np.float32(segment_range))
            with np.errstate(invalid="ignore"):
                inr = d2 <= r * r
            key = np.where(inr, d2, np.inf)
            index = np.broadcast_to(np.arange(ns), key.shape)
            order = np.lexsort((index, key), axis=-1)[:, :S]
            rows = np.arange(sel.size)[:, None]
            keep = inr[rows, order]
            e1x, e1y = _rot(C, Sn, ax[rows, order], ay[rows, order])
            bx, by = seg[order, 2] - X0, seg[order, 3] - Y0
            e2x, e2y = _rot(C, Sn, bx, by)
            ecx, ecy = _rot(C, Sn, px[rows, order], py[rows, order])
            blk = np.stack([np.ones_like(e1x), e1x, e1y, e2x, e2y, ecx, ecy, np.sqrt(d2[rows, order]),
                            ring[order].astype(np.float64)], -1)
            blk = np.where(keep[..., None], blk, 0.0).astype(np.float32)
            pad = np.zeros((sel.size, S, SEG_F), np.float32)
            pad[:, :blk.shape[1]] = blk
            out[sel, s0:] = pad.reshape(sel.size, -1)
            si = np.where(keep, order, -1).astype(np.int16)
            sidx[sel, :si.shape[1]] = si
    # ---- no ego: zeros, indices -1
    out[~ego] = 0.0
    aidx[~ego] = -1
    sidx[~ego] = -1
    return out, aidx, sidx


def split(flat, k_agents, k_segments):
    """(ego [N, 8], goal [N, 8], agents [N, K, 11], segments [N, S, 9]) views of a flat row array."""
    N = flat.shape[0]
    a0 = EGO_F + GOAL_F
    s0 = a0 + AGENT_F * k_agents
    return (flat[:, :EGO_F], flat[:, EGO_F:a0], flat[:, a0:s0].reshape(N, k_agents, AGENT_F),
            flat[:, s0:].reshape(N, k_segments, SEG_F))


def rotated_tolerance(ref, dist):
    """|got - ref| allowed for a value that went through sin / cos: one float32 ulp of the reference plus 1e-12 (1 + dist)."""
    ref = np.asarray(ref, np.float32)
    return np.abs(np.spacing(np.abs(ref))).astype(np.float64) + 1e-12 * (1.0 + np.asarray(dist, np.float64))


def compare(got, ref, k_agents, k_segments):
    """Asserts the contract's exactness: every column bit-exact except the rotated ones, which are held to
    ``rotated_tolerance`` with the row's dist (the ego's speed for its velocity).  Returns the largest rotated error."""
    g = split(np.asarray(got), k_agents, k_segments)
    r = split(np.asarray(ref), k_agents, k_segments)
    worst = 0.0
    for blk, (gb, rb, rot) in enumerate(zip(g, r, (EGO_ROTATED, GOAL_ROTATED, AGENT_ROTATED, SEG_ROTATED))):
        nf = gb.shape[-1]
        exact = [k for k in range(nf) if k not in rot]
        ge, re_ = gb[..., exact], rb[..., exact]
        bad = ge.view(np.uint32) != re_.view(np.uint32)
        assert not bad.any(), (blk, np.argwhere(bad)[:5], ge[bad][:5], re_[bad][:5])
        if blk == 0:
            dist = np.abs(rb[..., 1])
        else:
            dist = rb[..., 7] if blk in (1, 3) else rb[..., 10]
        for k in rot:
            err = np.abs(gb[..., k].astype(np.float64) - rb[..., k].astype(np.float64))
            tol = rotated_tolerance(rb[..., k], dist)
            assert (err <= tol).all(), (blk, k, np.argwhere(err > tol)[:5], err.max())
            if err.size:
                worst = max(worst, float(err.max()))
    return worst
