"""Float64 NumPy statement of the per-agent vector observation (DESIGN.md section 1 "Per-agent vector observation"; K9,
``t2d_observe_agents``): the vector observation of ``vector_obs_oracle`` with the observer a parameter.

Vectorised over scenarios and observers (in blocks of scenarios, to bound the memory of the [N, Q, M] and [N, Q, segments]
distance arrays).  Every value is the same elementwise float64 operation, in the same order, as ``vector_obs_oracle.observe``,
so a row observed by slot 0 without per-row goals is that oracle's row bit for bit; the exactness and the tolerance of the
rotated values are that oracle's (``vector_obs_oracle.compare``).
"""

from __future__ import annotations

import numpy as np

from tests.vector_obs_oracle import AGENT_F, EGO_F, GOAL_F, SEG_F, SHAPE_NONE, _extents, _rot, _seg_closest, width


def observe_agents(state, type_id, table, k_agents, k_segments, agent_range, segment_range, observers=None, step_count=None,
                   max_step=0, target=None, goals=None, tiles=(), tile_id=None, block=None):
    """As ``vector_obs_oracle.observe``, plus: observers int [N, Q] (None: every slot, Q = M); goals [N, Q, 5] (None: the
    rows observed by slot 0 take ``target``, the others none; a NaN cx: none).  Returns (flat float32 [N, Q, F], agent_index
    int16 [N, Q, K], segment_index int16 [N, Q, S])."""
    tid = np.asarray(type_id, np.int64)
    N, M = tid.shape
    obs = np.broadcast_to(np.arange(M), (N, M)) if observers is None else np.asarray(observers, np.int64).reshape(N, -1)
    Q = obs.shape[1]
    K, S = int(k_agents), int(k_segments)
    out = np.zeros((N, Q, width(K, S)), np.float32)
    aidx = np.full((N, Q, K), -1, np.int16)
    sidx = np.full((N, Q, S), -1, np.int16)
    n_seg = max([0] + [len(t["segments"]) for t in tiles if t.get("segments") is not None])
    if block is None:
        block = max(1, 2_000_000 // (Q * max(M, n_seg, 1)))
    steps = np.zeros(N) if step_count is None else np.asarray(step_count, np.float64).reshape(N)
    tids = np.zeros(N, np.int64) if tile_id is None else np.asarray(tile_id, np.int64).reshape(N)
    tgt = None if target is None else np.asarray(target, np.float32).reshape(N, 5)
    gls = None if goals is None else np.asarray(goals, np.float32).reshape(N, Q, 5)
    for b0 in range(0, N, block):
        b = slice(b0, min(N, b0 + block))
        _block({k: np.asarray(v)[b] for k, v in state.items()}, tid[b], table, K, S, agent_range, segment_range, obs[b],
               steps[b], max_step, None if tgt is None else tgt[b], None if gls is None else gls[b], tiles, tids[b],
               out[b], aidx[b], sidx[b])
    return out, aidx, sidx


def _block(state, tid, table, K, S, agent_range, segment_range, obs, steps, max_step, target, goals, tiles, tids, out, aidx,
           sidx):
    f64 = lambda a: np.asarray(a, np.float32).astype(np.float64)
    x, y, h = f64(state["x"]), f64(state["y"]), f64(state["heading"])
    vx, vy, v = f64(state["vx"]), f64(state["vy"]), np.asarray(state["speed"], np.float32)
    N, M = tid.shape
    Q = obs.shape[1]
    n_types = len(table)
    rows = np.arange(N)[:, None]
    valid = (obs >= 0) & (obs < M)
    j = np.where(valid, obs, 0)
    tj = tid[rows, j]
    ego = valid & (tj < n_types)
    x0, y0, h0 = x[rows, j], y[rows, j], h[rows, j]   # [N, Q]
    c, s = np.cos(h0), np.sin(h0)
    # ---- ego (the observer)
    hl, hw, disc, _ = _extents(table, tj)
    vl, vt = _rot(c, s, vx[rows, j], vy[rows, j])
    tf = steps / float(max_step) if max_step > 0 else np.zeros(N)
    out[..., 0] = 1.0; out[..., 1] = v[rows, j]; out[..., 2] = vl; out[..., 3] = vt
    out[..., 4] = hl; out[..., 5] = hw; out[..., 6] = disc; out[..., 7] = tf[:, None]
    # ---- goal
    if goals is not None:
        g = goals.astype(np.float64)
        has = ~np.isnan(g[..., 0])
    elif target is not None:
        g = np.broadcast_to(target.astype(np.float64)[:, None, :], (N, Q, 5))
        has = valid & (obs == 0)
    else:
        g, has = None, None
    if g is not None:
        with np.errstate(invalid="ignore"):
            dx, dy = g[..., 0] - x0, g[..., 1] - y0
            ex, ey = _rot(c, s, dx, dy)
            dh = g[..., 2] - h0
            blk = np.stack([np.ones_like(dx), ex, ey, np.cos(dh), np.sin(dh), g[..., 3], g[..., 4],
                            np.sqrt(dx * dx + dy * dy)], -1)
        out[..., EGO_F:EGO_F + GOAL_F] = np.where(has[..., None], blk, 0.0).astype(np.float32)
    # ---- agents: every other active slot with a shape, slot 0 included
    if K > 0:
        _, _, _, shape = _extents(table, tid)
        slot = np.arange(M)
        cand = ((tid < n_types) & (shape != SHAPE_NONE))[:, None, :] & (slot[None, None, :] != j[..., None])
        dx, dy = x[:, None, :] - x0[..., None], y[:, None, :] - y0[..., None]   # [N, Q, M]
        with np.errstate(invalid="ignore"):
            d2 = dx * dx + dy * dy
            r = np.float64(np.float32(agent_range))
            inr = cand & (d2 <= r * r)
        key = np.where(inr, d2, np.inf)
        order = np.lexsort((np.broadcast_to(slot, key.shape), key), axis=-1)[..., :K]
        keep = np.take_along_axis(inr, order, -1)
        jj = np.where(keep, order, 0)
        r3 = np.arange(N)[:, None, None]
        ahl, ahw, adisc, _ = _extents(table, tid[r3, jj])
        ddx, ddy = np.take_along_axis(dx, jj, -1), np.take_along_axis(dy, jj, -1)
        C, Sn = c[..., None], s[..., None]
        ex, ey = _rot(C, Sn, ddx, ddy)
        wx, wy = _rot(C, Sn, vx[r3, jj], vy[r3, jj])
        dh = h[r3, jj] - h0[..., None]
        blk = np.stack([np.ones_like(ddx), ex, ey, np.cos(dh), np.sin(dh), wx, wy, ahl, ahw, adisc,
                        np.sqrt(ddx * ddx + ddy * ddy)], -1)
        blk = np.where(keep[..., None], blk, 0.0).astype(np.float32)
        kk = blk.shape[2]
        a0 = EGO_F + GOAL_F
        out[..., a0:a0 + AGENT_F * kk] = blk.reshape(N, Q, -1)
        aidx[..., :kk] = np.where(keep, order, -1)
    # ---- segments of each scenario's tile, from the observer's centre
    if S > 0:
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
            X0, Y0, C, Sn = (a[sel][..., None] for a in (x0, y0, c, s))   # [n, Q, 1]
            x1, y1, x2, y2 = (seg[None, None, :, k] for k in range(4))
            px, py, d2, ax, ay = _seg_closest(x1, y1, x2, y2, X0, Y0)
            r = np.float64(np.float32(segment_range))
            with np.errstate(invalid="ignore"):
                inr = d2 <= r * r
            key = np.where(inr, d2, np.inf)
            order = np.lexsort((np.broadcast_to(np.arange(ns), key.shape), key), axis=-1)[..., :S]
            tk = lambda a: np.take_along_axis(a, order, -1)
            keep = tk(inr)
            e1x, e1y = _rot(C, Sn, tk(ax), tk(ay))
            bx, by = seg[order, 2] - X0, seg[order, 3] - Y0
            e2x, e2y = _rot(C, Sn, bx, by)
            ecx, ecy = _rot(C, Sn, tk(px), tk(py))
            blk = np.stack([np.ones_like(e1x), e1x, e1y, e2x, e2y, ecx, ecy, np.sqrt(tk(d2)),
                            ring[order].astype(np.float64)], -1)
            blk = np.where(keep[..., None], blk, 0.0).astype(np.float32)
            kk = blk.shape[2]
            out[sel, :, s0:s0 + SEG_F * kk] = blk.reshape(sel.size, Q, -1)
            sidx[sel, :, :kk] = np.where(keep, order, -1)
    # ---- no observer: zeros, indices -1
    out[~ego] = 0.0
    aidx[~ego] = -1
    sidx[~ego] = -1


def split(flat, k_agents, k_segments):
    """(ego [..., 8], goal [..., 8], agents [..., K, 11], segments [..., S, 9]) views of rows of any leading shape."""
    lead = flat.shape[:-1]
    a0 = EGO_F + GOAL_F
    s0 = a0 + AGENT_F * k_agents
    return (flat[..., :EGO_F], flat[..., EGO_F:a0], flat[..., a0:s0].reshape(*lead, k_agents, AGENT_F),
            flat[..., s0:].reshape(*lead, k_segments, SEG_F))
