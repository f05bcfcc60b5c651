"""Float64 statement of log replay with slot schedules (``t2d_set_log_schedule``; DESIGN.md section 1 "Log replay", "Slot
schedules").

Slot m of row p holds the entries ``slot_track[slot_off[p * M + m] : slot_off[p * M + m + 1]]``.  At the sample time t of
``oracle/replay.py`` the slot's track is the entry with ``first_k <= t <= last_k``, found here by a plain scan; that track is
then sampled by ``oracle.replay.sample`` itself, so state and type follow the single-track statement bit for bit.  A slot
with entries but none present at t gets ``type_id = 255`` and keeps its state; a slot without entries is not replayed.
"""

from __future__ import annotations

import numpy as np

from oracle import replay as R


def active_track(log, t0, slot_off, slot_track, log_row, step_count, interval_ms: int, offset: int = 1):
    """``(scheduled, track)``: bool [N, M] (the slot has entries) and int64 [N, M] (the entry present at t, -1 for none)."""
    first = np.asarray(log.first_ms, np.int64)
    last = first + (np.asarray(log.n_frames, np.int64) - 1) * np.asarray(log.period_ms, np.int64)
    t0 = np.asarray(t0, np.int64)
    off = np.asarray(slot_off, np.int64)
    trk = np.asarray(slot_track, np.int64)
    row = np.clip(np.asarray(log_row, np.int64), 0, len(t0) - 1)
    N = len(row)
    M = (len(off) - 1) // len(t0)
    t = t0[row] + (np.asarray(step_count, np.int64) + offset) * int(interval_ms)
    length = off[1:] - off[:-1]                                          # [P * M]
    L = max(int(length.max()), 1)
    # every slot's entries side by side (padded with -1), scanned all at once: [P * M, L]
    e = off[:-1, None] + np.arange(L)[None]
    pad = np.where(np.arange(L)[None] < length[:, None], trk[np.minimum(e, max(len(trk) - 1, 0))] if len(trk) else -1, -1)
    s = (row[:, None] * M + np.arange(M)[None])                          # [N, M]
    k = pad[s]                                                           # [N, M, L]
    kk = np.maximum(k, 0)
    tt = t[:, None, None]
    hit = (k >= 0) & (first[kk] <= tt) & (tt <= last[kk])
    track = np.where(hit.any(-1), np.take_along_axis(k, hit.argmax(-1)[..., None], -1)[..., 0], -1)
    return length[s] > 0, track


def sample(log, t0, slot_off, slot_track, log_row, step_count, interval_ms: int, offset: int = 1):
    """As ``oracle.replay.sample`` over a schedule: ``(replayed, present, state, type_id, track)``; ``replayed`` = the slot
    has entries, ``track`` = the active track or -1."""
    scheduled, track = active_track(log, t0, slot_off, slot_track, log_row, step_count, interval_ms, offset)
    row = np.clip(np.asarray(log_row, np.int64), 0, len(t0) - 1)
    n = len(row)
    # every scenario as its own row of a one-track-per-slot binding: the active track, sampled by the single-track statement
    _, present, state, tid = R.sample(log, np.asarray(t0, np.int64)[row], track, np.arange(n), step_count, interval_ms, offset)
    tid = np.where(scheduled & ~present, np.uint8(R.TYPE_INACTIVE), tid).astype(np.uint8)
    return scheduled, present, state, tid, track


def apply(state: dict, type_id, log, t0, slot_off, slot_track, log_row, step_count, interval_ms: int, offset: int = 1,
          mask=None):
    """``state`` / ``type_id`` after K7 with a schedule bound (``mask``: the scenarios replayed, default all)."""
    replayed, present, s, tid, _ = sample(log, t0, slot_off, slot_track, log_row, step_count, interval_ms, offset)
    if mask is not None:
        sel = np.asarray(mask, bool)[:, None]
        replayed, present = replayed & sel, present & sel
    out = {k: np.array(v, copy=True) for k, v in state.items()}
    for key in ("x", "y", "heading", "speed", "vx", "vy"):
        out[key] = np.where(present, s[key], out[key]).astype(np.float32)
    t = np.where(replayed, tid, np.asarray(type_id, np.uint8)).astype(np.uint8)
    return out, t
