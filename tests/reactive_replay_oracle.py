"""Float64 statement of reactive replay (``t2d_set_log_reactive``; DESIGN.md section 1 "Reactive replay") (TEST
INFRASTRUCTURE ONLY), composed from the oracles of the parts it joins.

K7 (``apply``): the slot's track at sample time t comes from ``oracle/replay.py`` (``row_track``) or
``tests/schedule_oracle.py`` (a schedule).  A present track k with ``track_path[k] >= 0`` is reactive:

* handover - reset mode (``mask`` given), or ``t - interval_ms < first_k`` in tick mode: the plain replay's state and
  ``type_row[k]``, bit for bit; ``drive_path = track_path[k]``, ``slot_desired_speed = desired_speed[k]``,
  ``pid_state[..., 0:3] = 0`` and ``last_accel = 0``;
* simulated - every later sample: the state is kept, ``type_id = drive_row[k]``, ``drive_path`` and
  ``slot_desired_speed`` as at the handover.

Every other slot of the replayed scenarios gets ``drive_path = -1`` and the plain replay.

K5 (``control_tick``): ``tests/lane_change_oracle.control_tick`` (``oracle.controllers`` with the lateral law of
``tests/pid_oracle.py``) on ``drive_path``, then the IDM acceleration of every slot with ``drive_path >= 0`` again with
``desired_speed = slot_desired_speed``.  ``rollout`` chains ``tests/leader_oracle.find``, that pass, K7 and
``oracle.scenario.physics_tick`` / ``events`` in the device's order."""

from __future__ import annotations

import numpy as np

from oracle import controllers as OC
from oracle import replay as R
from tests import lane_change_oracle as LC
from tests import leader_oracle as L
from tests import schedule_oracle as S


def sample(log, t0, log_row, step_count, interval_ms, offset, row_track=None, schedule=None):
    """``(replayed, present, state, type_id, track, t)`` of plain replay: bool [N, M] (the slot has a track), bool [N, M]
    (one is present at t), the sampled fp32 state, the plain type ids, the present track (-1: none) and t [N]."""
    if schedule is not None:
        replayed, present, st, tid, track = S.sample(log, t0, schedule[0], schedule[1], log_row, step_count, interval_ms,
                                                     offset)
    else:
        replayed, present, st, tid = R.sample(log, t0, row_track, log_row, step_count, interval_ms, offset)
        row = np.clip(np.asarray(log_row, np.int64), 0, len(t0) - 1)
        track = np.where(present, np.asarray(row_track, np.int64)[row], -1)
    row = np.clip(np.asarray(log_row, np.int64), 0, len(t0) - 1)
    t = np.asarray(t0, np.int64)[row] + (np.asarray(step_count, np.int64) + offset) * int(interval_ms)
    return replayed, present, st, tid, track, t


def apply(world: dict, log, t0, log_row, step_count, interval_ms, track_path, drive_row, desired_speed, offset=1,
          mask=None, row_track=None, schedule=None):
    """K7 with a reactive replay bound.  ``world``: dict of ``x, y, heading, speed, vx, vy`` (fp32 [N, M]), ``type_id``,
    ``drive_path``, ``slot_desired_speed``, ``pid_state`` [N, M, 6], ``last_accel``; returns a new dict with what the
    launch writes, plus ``handover`` and ``simulated`` (bool [N, M]).  ``mask``: reset mode over those scenarios."""
    replayed, present, st, tid, track, t = sample(log, t0, log_row, step_count, interval_ms, offset, row_track, schedule)
    N, M = tid.shape
    sel = np.ones(N, bool) if mask is None else np.asarray(mask, bool)
    sel = sel[:, None] & np.ones((1, M), bool)
    tp = np.asarray(track_path, np.int64)
    k = np.maximum(track, 0)
    reactive = sel & present & (tp[k] >= 0)
    first = np.asarray(log.first_ms, np.int64)[k]
    hand = reactive & ((mask is not None) | (t[:, None] - first < int(interval_ms)))
    sim = reactive & ~hand
    out = {key: np.array(v, copy=True) for key, v in world.items()}
    posed = sel & present & ~sim
    for key in ("x", "y", "heading", "speed", "vx", "vy"):
        out[key] = np.where(posed, st[key], out[key]).astype(np.float32)
    ty = np.where(sel & replayed, tid, out["type_id"])
    out["type_id"] = np.where(sim, np.asarray(drive_row, np.uint8)[k], ty).astype(np.uint8)
    out["drive_path"] = np.where(sel, np.where(reactive, tp[k], -1), out["drive_path"]).astype(np.int16)
    out["slot_desired_speed"] = np.where(reactive, np.asarray(desired_speed, np.float32)[k],
                                         out["slot_desired_speed"]).astype(np.float32)
    out["pid_state"][..., 0:3] = np.where(hand[..., None], 0.0, out["pid_state"][..., 0:3])
    out["last_accel"] = np.where(hand, np.float32(0.0), out["last_accel"]).astype(np.float32)
    out["handover"], out["simulated"] = hand, sim
    return out


def control_tick(state, type_id, table, action, ctrl_id, ctab, lead, drive_path, paths, last_accel, pid_state,
                 slot_desired_speed, steer_first=False):
    """K5's reactive instance: ``(action', last_accel', pid_state')``."""
    out, _, st = LC.control_tick(state, type_id, table, action, ctrl_id, ctab, lead, drive_path, paths, last_accel,
                                 pid_state, steer_first)
    x, y, v = (np.asarray(state[key], np.float64) for key in ("x", "y", "speed"))
    N, M = x.shape
    ai = 1 if steer_first else 0
    for n in range(N):
        for m in range(M):
            cid = int(ctrl_id[n, m])
            if drive_path[n, m] < 0 or cid == 255 or int(type_id[n, m]) == 255 or int(ctab[cid]["kind"]) != OC.IDM:
                continue
            li = int(lead[n, m])
            has = 0 <= li < M and int(type_id[n, li]) != 255 and li != m
            row = dict(ctab[cid], desired_speed=float(np.float32(slot_desired_speed[n, m])))
            xl, yl, vl = (x[n, li], y[n, li], v[n, li]) if has else (0.0, 0.0, 0.0)
            out[n, m, ai] = np.float32(OC.idm(v[n, m], x[n, m], y[n, m], has, vl, xl, yl, row))
    return out, OC.applied_accel_magnitude(out, type_id, table, steer_first).astype(np.float32), st


def reset_world(pool: dict, type_id, M: int) -> dict:
    """The world right after K2 from a one-row-per-scenario pool, before K7: pool state, zero controller memory,
    ``drive_path`` -1 and ``slot_desired_speed`` 0 (what the binding sets)."""
    N = type_id.shape[0]
    w = {key: np.asarray(pool[key], np.float32).copy() for key in ("x", "y", "heading", "speed", "vx", "vy")}
    w.update(type_id=np.asarray(type_id, np.uint8).copy(), drive_path=np.full((N, M), -1, np.int16),
             slot_desired_speed=np.zeros((N, M), np.float32), pid_state=np.zeros((N, M, 6)),
             last_accel=np.zeros((N, M), np.float32))
    return w


def rollout(episodes, table, ctab, paths, track_path, drive_row, desired_speed, ticks, half_width, max_range,
            reactive=True, interval_ms=100, delta_t=5):
    """The env's loop in float64 on every row of ``episodes`` (one scenario per row, the ego held at zero action, the
    other slots on controller row 0): reset (K2, then K7 in reset mode), then per tick K17 + K5 (reactive only), K7 and
    the physics.  Without ``reactive`` every track is plain replay and nothing is controlled.  Returns ``dict(states,
    type_id, hits, ego_hits, world)``: the state after every tick, the type ids, the dynamic-collision flags OR-ed over
    the rollout and the ego's per tick."""
    from oracle import scenario as O

    tab = table.as_oracle_table()
    P, M = episodes.type_id.shape
    tp = np.asarray(track_path) if reactive else np.full(len(episodes.log), -1, np.int16)
    bind = dict(row_track=episodes.row_track, schedule=episodes.schedule)
    w = reset_world(episodes.pool, episodes.type_id, M)
    step = np.zeros(P, np.int64)
    rows = np.arange(P)
    w = apply(w, episodes.log, episodes.t0, rows, step, interval_ms, tp, drive_row, desired_speed, 0, np.ones(P, bool), **bind)
    shapes = np.asarray(tab["shape"])
    ctrl = np.zeros((P, M), np.uint8)
    ctrl[:, 0] = 255
    hits = np.zeros((P, M), np.uint8)
    out = dict(states=[], type_id=[], ego_hits=[])
    for _ in range(ticks):
        act = np.zeros((P, M, 2), np.float32)
        if reactive:
            lead = L.find(w["x"], w["y"], w["heading"], w["type_id"], shapes, half_width, max_range, w["drive_path"],
                          paths)["lead"]
            act, w["last_accel"], w["pid_state"] = control_tick(w, w["type_id"], tab, act, ctrl, ctab, lead, w["drive_path"],
                                                                paths, w["last_accel"], w["pid_state"],
                                                                w["slot_desired_speed"])
        w = apply(w, episodes.log, episodes.t0, rows, step, interval_ms, tp, drive_row, desired_speed, 1, **bind)
        st = O.physics_tick(w, w["type_id"], act, tab, interval_ms, delta_t)
        for key in ("x", "y", "heading", "speed", "vx", "vy"):
            w[key] = np.asarray(st[key], np.float32)
        step += 1
        fl = O.events(w["x"], w["y"], w["heading"], w["type_id"], tab)[0] & O.F_DYNAMIC
        hits |= fl
        out["ego_hits"].append(fl[:, 0].copy())
        out["states"].append({key: w[key].copy() for key in ("x", "y", "heading", "speed")})
        out["type_id"].append(w["type_id"].copy())
    out["hits"], out["world"] = hits, w
    return out
