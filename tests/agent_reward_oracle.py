"""Float64 restatement of DESIGN.md section 1 "Per-agent status and reward" (K10, ``t2d_agents_epilogue``) and of the
matching part of the masked reset (TEST INFRASTRUCTURE ONLY).

Row (n, q) is the agent observed by slot ``observers[n, q]`` (slot q without a list).  The detectors, the status chain
and the reward chain are the ego's, from ``oracle.scenario`` (``goal_events``, ``status_with_goal``, ``env_epilogue``),
applied to every row as if the row were a one-participant scenario of its own; this module only gathers the rows, masks
the absent ones, retires the settled slots and reduces the done mask over each scenario's rows."""

from __future__ import annotations

import numpy as np

from oracle import scenario as O

ABSENT = 0


def _rows(N, M, Q, observers):
    """(slot [N, Q] int64, in_range [N, Q] bool) of an observer list (None: row q is slot q)."""
    slot = np.broadcast_to(np.arange(Q, dtype=np.int64), (N, Q)) if observers is None else np.asarray(observers, np.int64)
    return slot, (slot >= 0) & (slot < M)


def agents_epilogue(flags, type_id, x, y, heading, step_count, table, n_types, observers=None, goals=None,
                    last_pose=None, noact_count=None, max_iou=None, min_dist=None, retired=None, max_step=0,
                    threshold=0.95, no_action_max=100, reset_trackers=True):
    """One K10 launch on the post-tick state.  ``flags`` / ``type_id`` / ``x`` / ``y`` / ``heading``: [N, M];
    ``step_count`` [N] (after the tick); ``table``: ``TypeTable.as_oracle_table()``; ``observers`` [N, Q] or None;
    ``goals`` [N, Q, 5] or None; the row state ``last_pose`` [N, Q, 4], ``noact_count`` [N, Q], ``max_iou`` /
    ``min_dist`` [N, Q] and ``retired`` [N, M] (defaults: fresh).  Returns a dict of the outputs (status, reward,
    terminated, truncated, iou, done, traffic) and of the updated state (last_pose, noact_count, max_iou, min_dist,
    type_id, retired)."""
    flags = np.asarray(flags)
    type_id = np.asarray(type_id)
    N, M = flags.shape
    Q = M if observers is None else np.asarray(observers).shape[1]
    slot, in_range = _rows(N, M, Q, observers)
    sl = np.where(in_range, slot, 0)
    take = lambda a: np.take_along_axis(np.asarray(a), sl, 1)
    t_row = np.where(in_range, take(type_id), O.INACTIVE)
    active = t_row < n_types
    f_row = np.where(active, take(flags), 0).astype(np.uint8)
    xr, yr, hr = (take(np.asarray(a, np.float64)) for a in (x, y, heading))
    g = np.full((N, Q, 5), np.nan) if goals is None else np.asarray(goals, np.float64)
    has_goal = active & ~np.isnan(g[..., 0])
    last_pose = np.zeros((N, Q, 4)) if last_pose is None else np.array(last_pose, np.float64)
    noact_count = np.zeros((N, Q), np.int64) if noact_count is None else np.array(noact_count, np.int64)
    max_iou = np.full((N, Q), -np.inf) if max_iou is None else np.array(max_iou, np.float64)
    min_dist = np.full((N, Q), np.inf) if min_dist is None else np.array(min_dist, np.float64)
    retired = np.full((N, M), O.INACTIVE, np.uint8) if retired is None else np.array(retired, np.uint8)

    # every row as the ego (participant 0) of a one-slot scenario: flat [N·Q, 1]
    R = N * Q
    col = lambda a: a.reshape(R, 1)
    det_type = np.where(has_goal, t_row, O.INACTIVE).astype(np.uint8)   # rows without a goal have no detectors
    arrived, noact, iou, lp, cnt = O.goal_events(col(xr), col(yr), col(hr), col(det_type), table,
                                                 np.nan_to_num(g.reshape(R, 5)), last_pose.reshape(R, 4),
                                                 noact_count.reshape(R), threshold, no_action_max)
    cnt_row = np.repeat(np.asarray(step_count, np.int64), Q)
    st, _ = O.status_with_goal(col(f_row), col(t_row.astype(np.uint8)), cnt_row, arrived, noact, max_step)
    st = np.where(active.reshape(R), st, ABSENT).astype(np.uint8)

    reward = np.zeros(R)
    term = np.zeros(R, bool)
    trunc = np.zeros(R, bool)
    mi, md = max_iou.reshape(R).copy(), min_dist.reshape(R).copy()
    for sel, goal in ((has_goal.reshape(R), True), ((active & ~has_goal).reshape(R), False)):
        if not sel.any():
            continue
        e = O.env_epilogue(col(f_row)[sel], st[sel], cnt_row[sel], max_step,
                           iou=iou[sel] if goal else None, ego_xy=np.stack([xr.reshape(R), yr.reshape(R)], 1)[sel],
                           target=g.reshape(R, 5)[sel] if goal else None, max_iou=mi[sel] if goal else None,
                           min_dist=md[sel] if goal else None, reset_trackers=False)
        reward[sel], term[sel], trunc[sel] = e["reward"], e["terminated"], e["truncated"]
        if goal:
            mi[sel], md[sel] = e["max_iou"], e["min_dist"]
    iou = np.where(has_goal.reshape(R), iou, 0.0)

    st2 = st.reshape(N, Q)
    done = ~(st2 == O.NORMAL).any(1)
    if reset_trackers:
        mi = np.where(np.repeat(done, Q), -np.inf, mi)
        md = np.where(np.repeat(done, Q), np.inf, md)
    # retirement: every slot one of whose active rows settled
    settle = active & (st2 != O.NORMAL)
    new_type = type_id.copy()
    nn, qq = np.nonzero(settle)
    retired[nn, slot[nn, qq]] = t_row[nn, qq]
    new_type[nn, slot[nn, qq]] = O.INACTIVE
    traffic = np.where(flags & O.F_STATIC, 3, np.where(flags & O.F_DYNAMIC, 4, 1)).astype(np.uint8)
    return dict(status=st2, reward=reward.reshape(N, Q), terminated=term.reshape(N, Q), truncated=trunc.reshape(N, Q),
                iou=iou.reshape(N, Q), done=done.astype(np.uint8), traffic=traffic,
                last_pose=np.where(has_goal[..., None], lp.reshape(N, Q, 4), last_pose),
                noact_count=np.where(has_goal, cnt.reshape(N, Q), noact_count),
                max_iou=mi.reshape(N, Q), min_dist=md.reshape(N, Q), type_id=new_type, retired=retired)


def reset(mask, type_id, retired, last_pose, noact_count):
    """The agents' part of a masked reset (K2): the masked scenarios' retired slots take their types back, their retired
    marks clear and their rows' NoAction state starts fresh.  Returns (type_id, retired, last_pose, noact_count)."""
    m = np.asarray(mask, bool)
    type_id, retired = np.array(type_id), np.array(retired)
    last_pose, noact_count = np.array(last_pose, np.float64), np.array(noact_count)
    back = m[:, None] & (retired != O.INACTIVE)
    type_id = np.where(back, retired, type_id).astype(np.uint8)
    retired = np.where(m[:, None], O.INACTIVE, retired).astype(np.uint8)
    last_pose[m, :, 3] = 0.0
    noact_count[m] = 0
    return type_id, retired, last_pose, noact_count
