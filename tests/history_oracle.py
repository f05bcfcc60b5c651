"""Float64 NumPy statement of the trajectory history (DESIGN.md section 1 "Trajectory history"; K15 / K16,
``t2d_set_history`` / ``t2d_observe_history``).

``Ring`` restates the ring: ``append`` after every tick, ``restart`` of the masked scenarios after a reset, ``view`` the
entries that count for each slot's current occupant, lag 0 (the newest) first.  ``observe`` restates K16: each entry's
recorded pose and velocity in the observer's current frame with the elementwise float64 operations of
``vector_obs_oracle``'s agent rows, in their order, so a lag-0 block of the current state is that oracle's agent row
fields 1..6 bit for bit; the rotated values carry ``vector_obs_oracle.rotated_tolerance`` against the device.
"""

from __future__ import annotations

import numpy as np

from tests.vector_obs_oracle import _rot, rotated_tolerance

FIELDS = ("x", "y", "heading", "speed", "vx", "vy")
HIST_F = 7
ROTATED = (1, 2, 3, 4, 5, 6)


class Ring:
    """The ring of an N x M world of length H: ``f[k]`` fp32 [N, H, M] per field of ``FIELDS``, ``type_id`` uint8
    [N, H, M], ``track`` int32 [N, H, M] (recorded only when a track array is passed), ``count`` int64 [N]."""

    def __init__(self, N, M, H):
        if not 1 <= H <= 64:
            raise ValueError("H must be in 1..64")
        self.N, self.M, self.H = N, M, H
        self.f = {k: np.zeros((N, H, M), np.float32) for k in FIELDS}
        self.type_id = np.full((N, H, M), 255, np.uint8)
        self.track = np.full((N, H, M), -1, np.int32)
        self.count = np.zeros(N, np.int64)

    def _write(self, sel, e, state, type_id, track):
        idx = e % self.H
        for k in FIELDS:
            self.f[k][sel, idx] = np.asarray(state[k], np.float32)[sel]
        self.type_id[sel, idx] = np.asarray(type_id, np.uint8)[sel]
        if track is not None:
            self.track[sel, idx] = np.asarray(track, np.int32)[sel]
        self.count[sel] = e + 1

    def append(self, state, type_id, track=None):
        """Trajectory.add_state of every slot: entry count[n] of every scenario is the state after the tick."""
        sel = np.arange(self.N)
        self._write(sel, self.count.copy(), state, type_id, track)

    def restart(self, mask, state, type_id, track=None):
        """Trajectory.reset(state) of every slot of the masked scenarios: entry 0 is the state, count 1."""
        sel = np.nonzero(np.asarray(mask) != 0)[0]
        self._write(sel, np.zeros(sel.size, np.int64), state, type_id, track)

    def lag_index(self):
        """(ring index [N, H] of every lag, recent [N, H]: the lag is one of the last min(count, H) entries)."""
        lag = np.arange(self.H)
        return (self.count[:, None] - 1 - lag[None, :]) % self.H, lag[None, :] < np.minimum(self.count, self.H)[:, None]

    def view(self, type_id_now, n_types, track_now=None):
        """``BatchedWorld.history()``: every field [N, M, H] lag 0 first, zeros (type 255) where not valid, and valid."""
        idx, recent = self.lag_index()
        pick = lambda a: np.take_along_axis(a, idx[:, :, None], 1).transpose(0, 2, 1)
        tid = pick(self.type_id)
        now = np.asarray(type_id_now, np.int64)[:, :, None]
        valid = recent[:, None, :] & (tid.astype(np.int64) == now) & (tid.astype(np.int64) < n_types)
        if track_now is not None:
            valid &= pick(self.track) == np.asarray(track_now, np.int32)[:, :, None]
        out = {k: np.where(valid, pick(self.f[k]), np.float32(0)) for k in FIELDS}
        out["type_id"] = np.where(valid, tid, np.uint8(255))
        out["valid"] = valid
        out["count"] = self.count.copy()
        return out


def observe(ring, state, type_id, n_types, agent_index=None, observers=None, Q=0, track_now=None):
    """K16.  state / type_id: the current [N, M] world; Q = 0: one row per scenario observed by slot 0, agent_index [N, K];
    Q > 0: rows observers [N, Q] (None: row q is slot q), agent_index [N, Q, K].  Returns (out float32 [rows, 1 + K, H, 7],
    dist float64 [rows, 1 + K, H]: the distance of every entry from the observer, for the rotated tolerance)."""
    N, M, H = ring.N, ring.M, ring.H
    tid = np.asarray(type_id, np.int64)
    rows_q = max(Q, 1)
    if Q == 0:
        jo = np.zeros((N, 1), np.int64)
    elif observers is None:
        jo = np.broadcast_to(np.arange(Q), (N, Q)).astype(np.int64)
    else:
        jo = np.asarray(observers, np.int64).reshape(N, Q)
    K = 0 if agent_index is None else np.asarray(agent_index).shape[-1]
    ai = np.zeros((N, rows_q, K), np.int64) if agent_index is None else np.asarray(agent_index, np.int64).reshape(N, rows_q, K)
    slots = np.concatenate([jo[:, :, None], ai], -1)                       # [N, Q, 1 + K]
    f64 = lambda a: np.asarray(a, np.float32).astype(np.float64)
    x, y, h = f64(state["x"]), f64(state["y"]), f64(state["heading"])
    r = np.arange(N)[:, None]
    obs_ok = (jo >= 0) & (jo < M)
    j0 = np.where(obs_ok, jo, 0)
    obs_ok &= tid[r, j0] < n_types
    x0, y0, h0 = x[r, j0], y[r, j0], h[r, j0]                               # [N, Q]
    c, s = np.cos(h0), np.sin(h0)
    idx, recent = ring.lag_index()                                         # [N, H]
    slot_ok = (slots >= 0) & (slots < M)
    j = np.where(slot_ok, slots, 0)                                        # [N, Q, 1 + K]
    t_now = tid[r[:, :, None], j]
    slot_ok &= (t_now < n_types) & obs_ok[:, :, None]
    r4, i4, j4 = np.arange(N)[:, None, None, None], idx[:, None, None, :], j[..., None]   # -> [N, Q, 1 + K, H]
    rec = lambda a: a[r4, i4, j4]
    valid = slot_ok[..., None] & recent[:, None, None, :] & (rec(ring.type_id).astype(np.int64) == t_now[..., None])
    if track_now is not None:
        k_now = np.asarray(track_now, np.int32)[r[:, :, None], j]
        valid &= rec(ring.track) == k_now[..., None]
    C, S = c[:, :, None, None], s[:, :, None, None]
    dx = rec(ring.f["x"]).astype(np.float64) - x0[:, :, None, None]
    dy = rec(ring.f["y"]).astype(np.float64) - y0[:, :, None, None]
    ex, ey = _rot(C, S, dx, dy)
    wx, wy = _rot(C, S, rec(ring.f["vx"]).astype(np.float64), rec(ring.f["vy"]).astype(np.float64))
    dh = rec(ring.f["heading"]).astype(np.float64) - h0[:, :, None, None]
    blk = np.stack([np.ones_like(dx), ex, ey, np.cos(dh), np.sin(dh), wx, wy], -1)
    out = np.where(valid[..., None], blk, 0.0).astype(np.float32).reshape(N * rows_q, 1 + K, H, HIST_F)
    dist = np.where(valid, np.sqrt(dx * dx + dy * dy), 0.0).reshape(N * rows_q, 1 + K, H)
    return out, dist


def compare(got, ref, dist):
    """valid bit-exact, every rotated value within ``rotated_tolerance`` of the entry's distance; returns the worst error."""
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    bad = got[..., 0].view(np.uint32) != ref[..., 0].view(np.uint32)
    assert not bad.any(), np.argwhere(bad)[:5]
    zero = ref[..., 0] == 0
    assert (got[zero] == 0).all(), "an invalid entry is not zero"
    worst = 0.0
    for k in ROTATED:
        err = np.abs(got[..., k].astype(np.float64) - ref[..., k].astype(np.float64))
        tol = rotated_tolerance(ref[..., k], dist)
        assert (err <= tol).all(), (k, np.argwhere(err > tol)[:5], err.max())
        if err.size:
            worst = max(worst, float(err.max()))
    return worst
