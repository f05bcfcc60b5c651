"""The float64 chain of one ``BatchedTrafficEnv.step`` and of its masked reset (TEST INFRASTRUCTURE ONLY).

``step`` runs K11 (agent action scatter) -> K5 (controllers) -> the drift pre-pass and K1 (the tick) -> the env epilogue or
K10 (per-agent epilogue) -> K2 (+ K7) on the done mask.  Each stage here is the existing restatement of its kernel, fed
with what the device read before the stage (teacher forcing): the helpers only put the env's bindings into the shape the
restatements take.  A ``snapshot`` is a dict of host arrays of every per-scenario quantity the env keeps (see
``tests/test_gpu_env_episodes.py``)."""

from __future__ import annotations

import numpy as np

from oracle import c_oracle as CO
from oracle import scenario as O
from tests import agent_action_oracle as A
from tests import agent_reward_oracle as R
from tests import pid_oracle as P

STATE = ("x", "y", "heading", "speed", "vx", "vy")


def controls(pre, ctx, action):
    """K5 on the pre-step snapshot: ``(action', last_accel', pid_state')``.  ``action`` [N, M, 2] is the buffer K5
    reads (after K11 and the ego's row); retired and inactive slots carry type 255 in ``pre["type_id"]``."""
    c = ctx["ctrl"]
    return P.control_tick(pre, pre["type_id"], ctx["table"], action, c["ctrl_id"], c["rows"], c["lead_index"], c["path_id"],
                          c["paths"], pre["last_accel"], True, c["pid_target"], pre.get("pid_state"))


def scatter(action, agent_action, pre, ctx):
    """K11: the agents' rows scattered into ``action``."""
    return A.scatter_agent_action(action, agent_action, pre["type_id"], ctx["n_types"], ctx["observers"])


def physics(pre, action, ctx):
    """K1's (and the drift pre-pass') state update of the action the device applied, in float64."""
    st = {k: pre[k] for k in STATE + ("omega_wf", "omega_wr") if k in pre}
    return O.physics_tick(st, pre["type_id"], action, ctx["table"], ctx["interval"], ctx["delta_t"], steer_first=True)


def events(post, type_id, ctx):
    """Flags, first-hit participant and segment on the poses the device wrote."""
    return CO.events(post["x"], post["y"], post["heading"], type_id, ctx["table"], ctx["segments"], ctx["bounds"])


def ego_status(pre, post, flags, ctx):
    """K1's scenario status with the ego's goal detectors (``set_goal``), or without them: ``(status, goal)`` where
    ``goal`` is None or (iou, last_pose', count')."""
    cnt = pre["step_count"].astype(np.int64) + 1
    if ctx.get("target") is None:
        return O.status(flags, pre["type_id"], cnt, ctx["max_step"])[0], None
    arrived, noact, iou, lp, count = O.goal_events(post["x"], post["y"], post["heading"], pre["type_id"], ctx["table"],
                                                   ctx["target"], pre["goal_last_pose"], pre["goal_count"],
                                                   ctx["threshold"], ctx["no_action_max"])
    st, _ = O.status_with_goal(flags, pre["type_id"], cnt, arrived, noact, ctx["max_step"])
    return st, (iou, lp, count)


def env_epilogue(pre, post, flags, status, iou, ctx):
    """The env epilogue on the tick's outputs; ``pre`` holds the extrema before it."""
    tgt = ctx.get("target")
    N = flags.shape[0]
    xy = np.stack([post["x"][:, 0], post["y"][:, 0]], 1).astype(np.float64)
    mi = pre.get("max_iou", np.full(N, -np.inf))   # (the env allocates the extrema at its first epilogue)
    md = pre.get("min_dist", np.full(N, np.inf))
    return O.env_epilogue(flags, status, post["step_count"], ctx["max_step"], iou=iou, ego_xy=xy, target=tgt,
                          max_iou=None if tgt is None else mi, min_dist=None if tgt is None else md)


def agents_epilogue(pre, post, flags, ctx):
    """K10 on the tick's outputs; ``pre`` holds the row state and the retired types before it."""
    return R.agents_epilogue(flags, pre["type_id"], post["x"], post["y"], post["heading"], post["step_count"], ctx["table"],
                             ctx["n_types"], observers=ctx["observers"], goals=ctx["goals"],
                             last_pose=pre["agent_last_pose"], noact_count=pre["agent_count"], max_iou=pre["max_iou"],
                             min_dist=pre["min_dist"], retired=pre["retired"], max_step=ctx["max_step"],
                             threshold=ctx["threshold"], no_action_max=ctx["no_action_max"])


def reset(snap, mask, pool, pool_index, ctx):
    """K2 on a snapshot: the masked scenarios take pool row ``pool_index[n]`` (n without one) and start every piece of
    per-slot and per-scenario state afresh; everything else keeps its bits.  Replayed slots (K7) are not restated."""
    out = {k: np.array(v, copy=True) for k, v in snap.items()}
    m = np.asarray(mask).astype(bool)
    N = m.shape[0]
    n_pool = pool["x"].shape[0]
    r = np.clip(np.arange(N) if pool_index is None else np.asarray(pool_index, np.int64), 0, n_pool - 1)[m]
    for k in STATE:
        out[k][m] = pool[k][r]
    out["step_count"][m] = 0
    for k in ("last_accel", "pid_state"):
        if k in out:
            out[k][m] = 0
    if "goal_last_pose" in out:
        out["goal_last_pose"][m, 3] = 0.0
        out["goal_count"][m] = 0
    if "retired" in out:
        out["type_id"], out["retired"], lp, cnt = R.reset(m, out["type_id"], out["retired"], out["agent_last_pose"],
                                                          out["agent_count"])
        out["agent_last_pose"], out["agent_count"] = lp.astype(np.float32), cnt.astype(snap["agent_count"].dtype)
    if "omega_wf" in out:
        if pool.get("omega_wf") is not None:
            for k in ("omega_wf", "omega_wr"):
                out[k][m] = pool[k][r]
        else:   # free rolling: fp32 speed / wheel radius of the (restored) type, 0 for every other slot
            tid = out["type_id"][m].astype(np.int64)
            drift = (tid < ctx["n_types"]) & (ctx["model"][np.minimum(tid, ctx["n_types"] - 1)] == O.DRIFT)
            rad = ctx["wheel_radius"][np.minimum(tid, ctx["n_types"] - 1)]
            w = np.where(drift, pool["speed"][r].astype(np.float32) / rad, np.float32(0.0)).astype(np.float32)
            out["omega_wf"][m] = w
            out["omega_wr"][m] = w
    return out
