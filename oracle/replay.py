"""Float64 NumPy restatement of log replay (K7, ``t2d_set_log``; DESIGN.md section 1 "Log replay").

A track k holds ``n_frames[k]`` fp32 records (x, y, heading, vx, vy) every ``period_ms[k]`` from ``first_ms[k]`` on.  Scenario
n runs episode row ``row = clip(log_row[n], 0, n_rows - 1)`` and samples it at

    t = t0[row] + (step_count[n] + offset) * interval_ms          (offset 1 before a tick, 0 at a reset)

For a slot bound to track k (``row_track[row, m] = k >= 0``), with ``j, r = divmod(t - first_k, period_k)``:

* t outside [first_k, first_k + (n_frames_k - 1) period_k]: the track is absent, ``type_id = 255``, the state is untouched;
* r == 0: record j, bit for bit; ``type_id = type_row[k]``;
* else, in float64, one rounding per operation in this order, w = r / period:
  x, y, vx, vy = a + w * (b - a)  (records j, j + 1);
  heading: d = hb - ha, d -= 2 pi if d > pi, else d += 2 pi if d < -pi; h = ha + w * d; h += 2 pi if h < 0, else h -= 2 pi
  if h >= 2 pi; then fp32, and an fp32 result equal to fp32(2 pi) becomes 0;
* speed = fp32(sqrt(vx * vx + vy * vy)) of the fp32 vx, vy (``State.speed``).
"""

from __future__ import annotations

import numpy as np

TYPE_INACTIVE = 255
TWO_PI_F32 = np.float32(2 * np.pi)


def sample(log, t0, row_track, log_row, step_count, interval_ms: int, offset: int = 1):
    """The replay of every (scenario, slot).  ``log``: any object with ``first_ms, n_frames, period_ms, type_row`` [K] and
    ``records`` [F, 5].  Returns ``(replayed, present, state, type_id)``: bool [N, M] (bound to a track / bound and present),
    dict of fp32 [N, M] ``x, y, heading, speed, vx, vy`` (valid where present) and uint8 [N, M] (valid where replayed)."""
    first = np.asarray(log.first_ms, np.int64)
    period = np.asarray(log.period_ms, np.int64)
    nfr = np.asarray(log.n_frames, np.int64)
    rec = np.asarray(log.records, np.float32).reshape(-1, 5)
    off = np.concatenate([[0], np.cumsum(nfr)[:-1]]).astype(np.int64)
    t0 = np.asarray(t0, np.int64)
    rt = np.asarray(row_track, np.int64)
    row = np.clip(np.asarray(log_row, np.int64), 0, len(t0) - 1)
    k = rt[row]                                                         # [N, M]
    replayed = k >= 0
    kk = np.where(replayed, k, 0)
    t = t0[row][:, None] + (np.asarray(step_count, np.int64)[:, None] + offset) * int(interval_ms)
    d = t - first[kk]
    present = replayed & (d >= 0) & (d <= (nfr[kk] - 1) * period[kk])
    dd = np.where(present, d, 0)
    j, r = dd // period[kk], dd % period[kk]
    a = rec[off[kk] + j].astype(np.float64)                            # [N, M, 5]
    nxt = np.minimum(off[kk] + j + 1, len(rec) - 1)
    b = np.where((r > 0)[..., None], rec[nxt].astype(np.float64), a)
    w = r.astype(np.float64) / period[kk].astype(np.float64)

    def lerp(c):
        return (a[..., c] + w * (b[..., c] - a[..., c])).astype(np.float32)

    x, y, vx, vy = lerp(0), lerp(1), lerp(3), lerp(4)
    ha = a[..., 2]
    dh = b[..., 2] - ha
    dh = np.where(dh > np.pi, dh - 2 * np.pi, np.where(dh < -np.pi, dh + 2 * np.pi, dh))
    hh = ha + w * dh
    hh = np.where(hh < 0.0, hh + 2 * np.pi, np.where(hh >= 2 * np.pi, hh - 2 * np.pi, hh))
    h = hh.astype(np.float32)
    h = np.where(h == TWO_PI_F32, np.float32(0.0), h)
    on = r == 0                                                          # exact frames: the record's bits
    x = np.where(on, rec[off[kk] + j][..., 0], x)
    y = np.where(on, rec[off[kk] + j][..., 1], y)
    h = np.where(on, rec[off[kk] + j][..., 2], h)
    vx = np.where(on, rec[off[kk] + j][..., 3], vx)
    vy = np.where(on, rec[off[kk] + j][..., 4], vy)
    v64x, v64y = vx.astype(np.float64), vy.astype(np.float64)
    speed = np.sqrt(v64x * v64x + v64y * v64y).astype(np.float32)
    tid = np.where(present, np.asarray(log.type_row, np.uint8)[kk], np.uint8(TYPE_INACTIVE)).astype(np.uint8)
    state = dict(x=x, y=y, heading=h, speed=speed, vx=vx, vy=vy)
    return replayed, present, state, tid


def apply(state: dict, type_id, log, t0, row_track, log_row, step_count, interval_ms: int, offset: int = 1, mask=None):
    """``state`` / ``type_id`` after K7: copies with the replayed slots (of the scenarios in ``mask``, default all) rewritten."""
    replayed, present, s, tid = sample(log, t0, row_track, log_row, step_count, interval_ms, offset)
    if mask is not None:
        sel = np.asarray(mask, bool)[:, None]
        replayed, present = replayed & sel, present & sel
    out = {k: np.array(v, copy=True) for k, v in state.items()}
    for key in ("x", "y", "heading", "speed", "vx", "vy"):
        out[key] = np.where(present, s[key], out[key]).astype(np.float32)
    t = np.where(replayed, tid, np.asarray(type_id, np.uint8)).astype(np.uint8)
    return out, t
