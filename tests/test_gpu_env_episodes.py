"""BatchedTrafficEnv across episodes: every auto-reset must start a scenario exactly like its first episode, and every step
of the chain K11 -> K5 -> (drift pre-pass) -> K1 -> env epilogue / K10 -> K2 (+ K7) must match its float64 restatement
through the resets.

Every case runs two envs built alike side by side on the same inputs:

* A (``auto_reset=True``) is driven by tables indexed by each scenario's step within its episode (``world.step_count``
  read back before the step), so every episode of a scenario receives the same inputs and must reproduce the first one
  after the most recent ``env.reset`` bit for bit: state, wheel speeds, types, the action buffer after K5, the controllers'
  memory, the detector state, the extrema, every returned tensor and the observation.  On the step where a scenario
  auto-resets its observation and lidar equal its row of what ``env.reset`` returned.
* B (``auto_reset=False``) runs the env's own reset line by hand after every step, so that each stage can be held to
  ``tests/env_chain_oracle.py`` before the next one reads it (teacher forcing), and after the reset it must equal A bit
  for bit.

A leak of any per-slot or per-scenario state from one episode into the next, a controller that reads a retired leader or
a PID slot that integrates while retired shows here even where every per-kernel test passes."""

import dataclasses
from typing import Callable, Optional

import numpy as np
import pytest

from oracle import scenario as O
from tests import env_chain_oracle as EC
from tests.util import assert_state_close, rel_err

pytestmark = pytest.mark.gpu

THRESHOLD, NO_ACTION_MAX = 0.95, 3
MIN_EPISODES = 3
OMEGA = ("omega_wf", "omega_wr")


def _np(t):
    return None if t is None else t.detach().cpu().numpy().copy()


def _bits(a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.float32:
        return a.view(np.uint32)
    if a.dtype == np.float64:
        return a.view(np.uint64)
    return a.view(np.uint8) if a.dtype == np.bool_ else a


def _same(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def _snap(env, full):
    """Every per-scenario quantity the env keeps, as host arrays with a leading N axis."""
    w = env.world
    s = w.state_numpy()
    keep = dict(type_id=w.type_id, step_count=w.step_count, last_accel=w.last_accel, pid_state=w.pid_state, action=full,
                retired=w.retired_type, log_row=w.log_row, track=w.replay_track)
    if w._goal is not None:
        keep.update(goal_last_pose=w._goal["last_pose"], goal_count=w._goal["count"])
    if w._agents is not None:
        a = w._agents
        keep.update(agent_last_pose=a["last_pose"], agent_count=a["noact_count"], max_iou=a["max_iou"], min_dist=a["min_dist"])
    elif w._env is not None:
        keep.update(max_iou=w._env["max_iou"], min_dist=w._env["min_dist"])
    s.update({k: _np(v) for k, v in keep.items() if v is not None})
    return s


def _outputs(ret):
    import torch

    obs, reward, term, trunc, info = ret
    out = dict(reward=reward, terminated=term, truncated=trunc)
    if torch.is_tensor(obs):   # ("state" observations are the state tensors themselves)
        out["obs"] = obs
    for k in ("scenario_status", "traffic_status", "flags", "hit_index", "hit_segment", "track", "iou", "agent_status",
              "agent_iou", "lidar"):
        if k in info:
            out[k] = info[k]
    return {k: _np(v) for k, v in out.items()}


def _done(env):
    return env.world._agents["done"] if env.agent_rewards else env.scenario_manager.env_result.done


def _full(env, kw):
    """The action buffer K5 fills: the caller's [N, M, 2] tensor, or the env's own."""
    a = kw["action"]
    return a if a.dim() == 3 and not env.agent_actions else env._action


@dataclasses.dataclass
class Case:
    make: Callable          # auto_reset -> env with its controllers bound, not yet reset
    act: Callable           # k [N] (each scenario's step within its episode) -> env.step keyword arguments, fresh tensors
    steps: int
    shuffle_at: Optional[int] = None
    oracle: bool = True     # hold B to tests/env_chain_oracle.py


class _FirstEpisodes:
    """Per (episode step k, scenario n): the bits of the first episode since the last env.reset; later ones must match."""

    def __init__(self, N, K):
        self.N, self.K = N, K
        self.ref = {}
        self.have = np.zeros((K, N), bool)

    def restart(self, reset_out):
        self.have[:] = False
        self.reset_out = reset_out
        self.episodes = np.zeros(self.N, np.int64)

    def check(self, k, rec, done, t):
        rows = np.arange(self.N)
        new = ~self.have[k, rows]
        old = ~new
        for f, a in rec.items():
            b = _bits(a)
            if f not in self.ref:
                self.ref[f] = np.zeros((self.K,) + b.shape, b.dtype)
            self.ref[f][k[new], rows[new]] = b[new]
            if not old.any():
                continue
            diff = (self.ref[f][k[old], rows[old]] != b[old]).reshape(int(old.sum()), -1).any(1)
            assert not diff.any(), (f"step {t}: {f} of scenarios {rows[old][diff][:8]} at episode step {k[old][diff][:8]} "
                                    "differs from their first episode")
        self.have[k, rows] = True
        d = done.astype(bool)
        for f, a in self.reset_out.items():   # the auto-reset shows what env.reset showed
            assert _same(rec[f][d], a[d]), f"step {t}: {f} after the auto-reset differs from env.reset's"
        self.episodes += d


def _ctx(env):
    """The env's bindings as the restatements take them."""
    w = env.world
    tt = w.type_table
    c = w._ctrl
    ctx = dict(table=tt.as_oracle_table(), n_types=len(tt), model=np.array([r.model for r in tt.rows]),
               wheel_radius=np.array([r.wheel_radius for r in tt.rows], np.float32), interval=w.interval,
               delta_t=w.delta_t, max_step=w.max_step, segments=w.segments, bounds=w.bounds,
               pool={k: _np(v) for k, v in env._pool.items()}, observers=_np(env.vector_obs.get("observers")),
               goals=_np(env.vector_obs.get("goals")), target=None if w._goal is None else _np(w._goal["target"]),
               threshold=THRESHOLD, no_action_max=NO_ACTION_MAX, ctrl=None)
    if c is not None:
        ctx["ctrl"] = dict(rows=[{k: getattr(r, k) for k, _ in r._fields_} for r in c["rows"]], ctrl_id=_np(c["ctrl_id"]),
                           lead_index=_np(c["lead_index"]), path_id=_np(c["path_id"]),
                           paths=[p.astype(np.float64) for p in (w.paths or [])], pid_target=_np(c["pid_target"]))
    return ctx


def _check_step(env, kw, pre, post, out, ctx, seen, t):
    """B's step, stage by stage, against the restatements; returns nothing, records what happened in ``seen``."""
    nt = ctx["n_types"]
    active = pre["type_id"] < nt
    # K11 and the ego's row: the buffer K5 reads
    ext = pre["action"].copy()
    if env.agent_actions:
        ext = EC.scatter(ext, _np(kw["action"]), pre, ctx)
    elif kw["action"].dim() == 2:
        ext[:, 0] = np.where(active[:, :1], _np(kw["action"]), ext[:, 0])
    got = post["action"]
    c = ctx["ctrl"]
    if c is None:
        assert _same(got, ext), f"step {t}: action buffer"
    else:
        want, la, st = EC.controls(pre, ctx, ext)
        ctl = (c["ctrl_id"] != 255) & active
        assert _same(got[~ctl], want[~ctl]), f"step {t}: K5 touched a row it does not drive"
        np.testing.assert_allclose(got[ctl], want[ctl], rtol=3e-6, atol=3e-6, err_msg=f"step {t}: K5 actions")
        np.testing.assert_allclose(post["last_accel"], la, rtol=3e-6, atol=3e-6, err_msg=f"step {t}: last_accel")
        if "pid_state" in post:
            np.testing.assert_allclose(post["pid_state"], st, rtol=1e-12, atol=1e-12, err_msg=f"step {t}: pid_state")
        lead = c["lead_index"].astype(np.int64)
        ok = (lead >= 0) & (lead < lead.shape[1])
        lt = np.take_along_axis(pre["type_id"], np.where(ok, lead, 0), 1)
        if "retired" in pre:
            lr = np.take_along_axis(pre["retired"], np.where(ok, lead, 0), 1)
            seen["retired_lead"] += int((ctl & ok & (lt >= nt) & (lr < nt)).sum())
        seen["absent_lead"] += int((ctl & ok & (lt >= nt)).sum())
    # the tick, with the actions the device applied
    ref = EC.physics(pre, got, ctx)
    assert_state_close(post, ref, mask=active, rtol=1e-5, what=f"step {t}")
    for k in EC.STATE + tuple(k for k in OMEGA if k in pre):
        assert _same(post[k][~active], pre[k][~active]), f"step {t}: {k} of an inactive or retired slot moved"
    if "omega_wf" in pre:
        drift = active & (ctx["model"][np.minimum(pre["type_id"], nt - 1)] == O.DRIFT)
        for k in OMEGA:
            assert rel_err(post[k], ref[k])[drift].max(initial=0.0) < 1e-5, f"step {t}: {k}"
            assert _same(post[k][~drift], pre[k][~drift]), f"step {t}: {k} of a slot without wheels"
        seen["drift"] += int(drift.sum())
    fl, hi, hs = EC.events(post, pre["type_id"], ctx)
    for k, v in (("flags", fl), ("hit_index", hi), ("hit_segment", hs)):
        assert _same(out[k], v), f"step {t}: {k} at {np.argwhere(out[k] != v)[:5].tolist()}"
    assert _same(post["step_count"], pre["step_count"] + 1), f"step {t}: step_count"
    if env.agent_rewards:
        assert _same(out["scenario_status"], EC.ego_status(pre, post, fl, ctx)[0]), f"step {t}: K1 status"
        e = EC.agents_epilogue(pre, post, fl, ctx)
        assert np.abs(out["agent_iou"] - e["iou"]).max() <= 2e-6, f"step {t}: agent IoU"
        ok = ~(np.abs(e["iou"] - THRESHOLD) <= 1e-6).any(1)   # no row at the arrival threshold
        for k, g in (("status", out["agent_status"]), ("terminated", out["terminated"]), ("truncated", out["truncated"]),
                     ("done", _np(env.world._agents["done"])), ("type_id", post["type_id"]), ("retired", post["retired"]),
                     ("noact_count", post["agent_count"])):
            assert np.array_equal(g[ok], e[k][ok].astype(g.dtype)), f"step {t}: K10 {k}"
        np.testing.assert_allclose(out["reward"][ok], e["reward"][ok], rtol=1e-5, atol=2e-6, err_msg=f"step {t}: reward")
        status = out["agent_status"]
        seen["agent_status"] |= set(np.unique(status[ok]).tolist())
    else:
        st, goal = EC.ego_status(pre, post, fl, ctx)
        ok = np.ones(st.shape, bool)
        iou = None
        if goal is not None:
            g_iou, lp, cnt = goal
            box = active[:, 0] & (ctx["table"]["shape"][np.minimum(pre["type_id"][:, 0], nt - 1)] == O.OBB)
            assert np.abs(out["iou"][box] - g_iou[box]).max(initial=0.0) <= 2e-6, f"step {t}: ego IoU"
            ok = ~(np.abs(g_iou - THRESHOLD) <= 1e-6)
            assert _same(post["goal_count"][ok], cnt[ok].astype(np.int32)), f"step {t}: NoAction count"
            assert _same(post["goal_last_pose"][box], lp[box].astype(np.float32)), f"step {t}: NoAction pose"
            iou = out["iou"]
        assert _same(out["scenario_status"][ok], st[ok]), f"step {t}: status"
        e = EC.env_epilogue(pre, post, fl, out["scenario_status"], iou, ctx)
        for k in ("terminated", "truncated"):
            assert np.array_equal(out[k], e[k]), f"step {t}: {k}"
        assert np.array_equal(_np(env.scenario_manager.env_result.done), e["done"]), f"step {t}: done"
        np.testing.assert_allclose(out["reward"], e["reward"], rtol=1e-5, atol=2e-6, err_msg=f"step {t}: reward")
        status = out["scenario_status"]
    assert _same(out["traffic_status"], e.get("traffic_status", e.get("traffic"))), f"step {t}: TrafficStatus"
    if e.get("max_iou") is not None:
        for k in ("max_iou", "min_dist"):
            np.testing.assert_allclose(post[k], e[k], rtol=1e-6, atol=1e-6, err_msg=f"step {t}: {k}")
    seen["status"] |= set(np.unique(status).tolist())


def _run(case, device):
    import torch

    A, B = case.make(True), case.make(False)
    N = A.num_envs
    ctx = _ctx(B) if case.oracle else None
    first = _FirstEpisodes(N, A.max_step + 2)
    seen = dict(status=set(), agent_status=set(), retired_lead=0, absent_lead=0, drift=0, pid_restored=0,
                drift_restored=0, shuffled=0)

    def shown(ret):
        obs, info = ret
        out = {"obs": _np(obs)} if torch.is_tensor(obs) else {}
        if "lidar" in info:
            out["lidar"] = _np(info["lidar"])
        return out

    def reset(**kw):
        sa, sb = shown(A.reset(**kw)), shown(B.reset(**kw))
        for f, v in sa.items():
            assert _same(v, sb[f]), f"env.reset: {f} of A and B differ"
        first.restart(sa)

    reset(seed=0)
    for t in range(case.steps):
        if t == case.shuffle_at:
            row = _np(A.world.log_row)
            reset(options={"shuffle": True})
            seen["shuffled"] = int((_np(A.world.log_row) != row).sum())
        k =np.minimum(_np(A.world.step_count).astype(np.int64), first.K - 1)
        kw_a, kw_b = case.act(k), case.act(k)
        rec = _outputs(A.step(**kw_a))
        rec.update(_snap(A, _full(A, kw_a)))
        pre = _snap(B, _full(B, kw_b))
        out = _outputs(B.step(**kw_b))
        post = _snap(B, _full(B, kw_b))
        if case.oracle:
            _check_step(B, kw_b, pre, post, out, ctx, seen, t)
        done = _done(B)
        d = _np(done).astype(bool)
        # the env's own auto-reset line, by hand
        B.scenario_manager.reset(mask=done, pool_index=B.world.log_row)
        after = _snap(B, _full(B, kw_b))
        if case.oracle:
            want = EC.reset(post, d, ctx["pool"], None if post.get("log_row") is None else post["log_row"], ctx)
            for f, v in want.items():
                assert _same(after[f], v), f"step {t}: K2 left {f} at {np.argwhere(_bits(after[f]) != _bits(v))[:5].tolist()}"
            if "retired" in post:
                back = d[:, None] & (post["retired"] < ctx["n_types"])
                if ctx["ctrl"] is not None:
                    pid_row = np.array([r["kind"] == 4 for r in ctx["ctrl"]["rows"]] + [False])
                    cid = ctx["ctrl"]["ctrl_id"].astype(np.int64)
                    seen["pid_restored"] += int((back & pid_row[np.minimum(cid, len(pid_row) - 1)]).sum())
                drift = ctx["model"][np.minimum(post["retired"], ctx["n_types"] - 1)] == O.DRIFT
                seen["drift_restored"] += int((back & drift).sum())
        # B, reset by hand, is A
        out.update(after)
        if "obs" in out:
            out["obs"] = _np(B._obs())
        if "lidar" in out:
            out["lidar"] = _np(B._add_lidar({})["lidar"])
        for f, v in rec.items():
            assert _same(v, out[f]), f"step {t}: {f} of the env's auto-reset differs from the reset by hand"
        assert _same(_np(_done(A)), d)
        first.check(k, rec, d, t)
    assert first.episodes.min() >= MIN_EPISODES, f"a scenario finished only {first.episodes.min()} episodes"
    A.close()
    B.close()
    return seen


# ---------------------------------------------------------------------------------------------------------------- scenes

def _with(sc, **kw):
    """``sc`` with some arrays replaced; vx / vy follow a new speed."""
    sc = dataclasses.replace(sc, **kw)
    if "speed" in kw:
        v, h = sc.speed.astype(np.float64), sc.heading.astype(np.float64)
        sc = dataclasses.replace(sc, vx=(v * np.cos(h)).astype(np.float32), vy=(v * np.sin(h)).astype(np.float32))
    return sc


PATHS = [np.array([[0, 0], [20, 5], [40, 5], [40, 5], [60, 20], [80, 20], [100, 40], [120, 60], [140, 60], [150, 80]],
                  np.float32),                                                   # a zero-length segment in the middle
         np.array([[10, -40], [10, 90], [-60, 160]], np.float32),
         np.array([[5, 5], [5, 5]], np.float32)]                                 # only a zero-length segment


def _controllers(rng, sc, choices, lead=None):
    """Controller bindings over ``tests/test_gpu_pid_controller._pid_rows`` (IDM, cruise, pure pursuit, five PID sources):
    ``(rows, ctrl_id, lead_index, path_id, pid_target)``; the ego (slot 0) stays the policy's."""
    from tests.test_gpu_pid_controller import _pid_rows

    N, M = sc.shape
    ctrl_id = rng.choice(choices, size=(N, M)).astype(np.uint8)
    ctrl_id[:, 0] = 255
    if lead is None:
        lead = rng.integers(-1, M, size=(N, M))
        lead[::3, 2] = 2                                                         # itself
        inactive = sc.type_id == 255
        for n in np.nonzero(inactive.any(1))[0]:
            lead[n, 1] = np.nonzero(inactive[n])[0][0]                           # an inactive slot
    path_id = rng.integers(-1, len(PATHS) + 1, size=(N, M)).astype(np.int16)     # -1 and one past the end included
    target = np.stack([rng.uniform(0, 12, (N, M)), rng.uniform(-3, 3, (N, M))], 2).astype(np.float32)
    return _pid_rows(), ctrl_id, lead.astype(np.int16), path_id, target


def _bind(env, ctrl):
    rows, ctrl_id, lead, path_id, target = ctrl
    env.world.set_paths(PATHS)
    env.world.set_controllers(rows, ctrl_id, lead, path_id, pid_target=target)
    return env


def _table_action(device, table):
    import torch

    n = np.arange(table.shape[1])
    return lambda k: {"action": torch.from_numpy(np.ascontiguousarray(table[k, n])).to(device)}


def _e1(device, max_step=7):
    """Egos with targets (parked on it, standing still, driving) among controlled NPCs; vector observation and lidar."""
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    N, M = 129, 33
    sc = synthetic.with_inactive(synthetic.config4(N, M, seed=41), 0.15, seed=42)
    rng = np.random.default_rng(43)
    tid = sc.type_id.copy()
    tid[:, 0] = rng.integers(0, 9, N)                                            # every ego a car (a box the detectors score)
    n = np.arange(N)
    parked, still = n % 4 == 0, n % 4 == 1
    speed = sc.speed.copy()
    speed[parked | still, 0] = 0.0
    sc = _with(sc, type_id=tid, speed=speed)
    hl = np.array([r.half_len for r in sc.table.rows], np.float32)[tid[:, 0]]
    hw = np.array([r.half_wid for r in sc.table.rows], np.float32)[tid[:, 0]]
    off = np.where(parked[:, None], 0.0, np.where(still[:, None], 30.0, rng.normal(0, 3, (N, 2))))
    target = np.stack([sc.x[:, 0] + off[:, 0], sc.y[:, 0] + off[:, 1], sc.heading[:, 0], hl, hw], 1).astype(np.float32)
    ego = np.stack([rng.uniform(-0.5, 0.5, (max_step + 2, N)), rng.uniform(-3, 3, (max_step + 2, N))], 2).astype(np.float32)
    ego[:, parked | still] = 0.0
    ctrl = _controllers(rng, sc, [255, 0, 1, 2, 3, 4, 5, 6, 7])

    def make(auto_reset):
        return _bind(BatchedTrafficEnv(sc, device=device, max_step=max_step, auto_reset=auto_reset, target=target,
                                       arrival_threshold=THRESHOLD, no_action_max_step=NO_ACTION_MAX, observation="vector",
                                       vector_obs=dict(k_agents=4, k_segments=4), lidar=dict(n_beams=32, max_range=20.0)),
                     ctrl)
    return Case(make, _table_action(device, ego), steps=3 * (max_step + 1) + 2)


def test_e1_egos_with_targets_among_controlled_npcs(cuda_device):
    seen = _run(_e1(cuda_device), cuda_device)
    assert {O.COMPLETED, O.NO_ACTION, O.TIME_EXCEEDED} <= seen["status"], seen["status"]
    assert seen["absent_lead"] > 0


def test_e2_c2_shaped_tick_inside_the_env(cuda_device):
    """config2 at M = 64, kinematics only, no ego action bound and no goal: the env's ticks take the C2-shaped instance."""
    from tactics2d_b200 import _lib, synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    N, M, max_step = 257, 64, 7
    sc = synthetic.config2(N, M, seed=51)
    rng = np.random.default_rng(52)
    ctrl = _controllers(rng, sc, [255, 0, 1, 2, 3, 4, 5, 6, 7])
    table = np.stack([rng.uniform(-0.6, 0.6, (max_step + 2, N, M)), rng.uniform(-4, 3, (max_step + 2, N, M))],
                     3).astype(np.float32)

    def make(auto_reset):
        return _bind(BatchedTrafficEnv(sc, device=cuda_device, max_step=max_step, auto_reset=auto_reset), ctrl)
    lib = _lib.load()
    c0 = lib.t2d_tick_fixed_count()
    steps = 3 * (max_step + 1) + 1
    seen = _run(Case(make, _table_action(cuda_device, table), steps=steps), cuda_device)
    assert lib.t2d_tick_fixed_count() - c0 == 2 * steps
    assert {O.TIME_EXCEEDED, O.FAILED} <= seen["status"], seen["status"]


def test_e3_agents_retire_and_come_back(cuda_device):
    """Per-agent rewards and actions over an observer list with duplicates, -1 and M; PID-driven agents retire; NPCs
    follow agents that retire."""
    import torch

    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    N, M, Q, max_step = 67, 128, 40, 7
    sc = synthetic.with_inactive(synthetic.config4(N, M, seed=61), 0.15, seed=62)
    rng = np.random.default_rng(63)
    obs = rng.integers(0, M, (N, Q))
    obs[:, 1] = obs[:, 0]                                                        # a duplicate
    obs[:, 2] = -1
    obs[:, 3] = M
    sl = np.clip(obs, 0, M - 1)
    x, y, h = (np.take_along_axis(a, sl, 1) for a in (sc.x, sc.y, sc.heading))
    goals = np.stack([x + rng.normal(0, 2, x.shape), y + rng.normal(0, 2, x.shape), h, np.full(x.shape, 2.4),
                      np.full(x.shape, 1.0)], -1).astype(np.float32)
    goals[:, ::3, 0] = np.nan
    agent = np.zeros((N, M), bool)
    np.put_along_axis(agent, sl[:, 4:], True, 1)
    lead = np.where(agent, -1, np.take_along_axis(obs, rng.integers(4, Q, (N, M)), 1))   # NPCs follow agents
    rows, ctrl_id, lead, path_id, target = _controllers(rng, sc, [255, 0, 1, 2], lead=lead)
    ctrl_id[:, 0] = 255
    pid_agents = obs[:, 4:14]                                                    # ten agents per scenario are PID-driven
    np.put_along_axis(ctrl_id, pid_agents, (3 + np.arange(10) % 5).astype(np.uint8)[None].repeat(N, 0), 1)
    table = np.stack([rng.uniform(-0.6, 0.6, (max_step + 2, N, Q)), rng.uniform(-4, 3, (max_step + 2, N, Q))],
                     3).astype(np.float32)

    def make(auto_reset):
        vo = dict(k_agents=4, k_segments=4, observers=torch.from_numpy(obs.astype(np.int16)).to(cuda_device),
                  goals=torch.from_numpy(goals).to(cuda_device))
        return _bind(BatchedTrafficEnv(sc, device=cuda_device, max_step=max_step, auto_reset=auto_reset,
                                       arrival_threshold=THRESHOLD, no_action_max_step=NO_ACTION_MAX, observation="agents",
                                       vector_obs=vo, agent_rewards=True, agent_actions=True,
                                       lidar=dict(n_beams=16, max_range=15.0)),
                     (rows, ctrl_id, lead, path_id, target))
    seen = _run(Case(make, _table_action(cuda_device, table), steps=3 * (max_step + 1) + 2), cuda_device)
    assert {O.FAILED, O.TIME_EXCEEDED} <= seen["agent_status"], seen["agent_status"]
    assert seen["pid_restored"] > 0 and seen["retired_lead"] > 0, seen


@pytest.mark.parametrize("pool_wheels", [False, True])
def test_e4_drift_wheels_through_retirement_and_reset(cuda_device, pool_wheels):
    """A table mixing SingleTrackDrift rows with a kinematic one; every slot is an agent, so drift slots retire and K2
    restores them before it sets their wheel speeds (free rolling, or the pool's columns)."""
    import torch

    from tactics2d_b200 import TypeParams, TypeTable, synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    N, M, max_step = 65, 16, 5
    sc = synthetic.config2(N, M, seed=71, size=50.0)
    rng = np.random.default_rng(72)
    table = TypeTable([TypeParams.vehicle("medium_car"), TypeParams.vehicle("medium_car", model="drift"),
                       TypeParams.vehicle("large_car", model="drift")])
    tid = rng.integers(0, 3, (N, M)).astype(np.uint8)
    tid[rng.random((N, M)) < 0.1] = 255
    sc = _with(sc, table=table, type_id=tid, speed=rng.uniform(3.0, 12.0, (N, M)).astype(np.float32))
    act = np.stack([rng.uniform(-0.3, 0.3, (max_step + 2, N, M)), rng.uniform(-1, 1.5, (max_step + 2, N, M))],
                   3).astype(np.float32)

    # initial wheel speeds off free rolling by up to 10 %, so that a reset that ignores the columns shows
    wheels = (sc.speed / np.float32(0.344) * rng.uniform(0.9, 1.1, (2, N, M))).astype(np.float32)

    def make(auto_reset):
        env = BatchedTrafficEnv(sc, device=cuda_device, max_step=max_step, auto_reset=auto_reset, observation="agents",
                                vector_obs=dict(k_agents=4, k_segments=4), agent_rewards=True, agent_actions=True)
        if pool_wheels:   # (the scenario manager resets from this dict)
            for k, v in zip(OMEGA, wheels):
                env._pool[k] = torch.from_numpy(np.ascontiguousarray(v)).to(cuda_device)
        return env
    seen =_run(Case(make, _table_action(cuda_device, act), steps=3 * (max_step + 1) + 2), cuda_device)
    assert seen["drift"] > 0 and seen["drift_restored"] > 0, seen


def test_e5_replay_with_a_shuffle_in_the_middle(cuda_device):
    """Scheduled log replay with a BEV observation; one shuffled env.reset mid-run deals new rows, and the auto-resets
    after it restart each scenario's new row (``log_row``)."""
    from tactics2d_b200.envs import BatchedTrafficEnv
    from tests.test_gpu_replay_schedule import _walk_episodes

    N, M, max_step = 65, 24, 7
    ep = _walk_episodes(N, M, seed=81)
    rng = np.random.default_rng(82)
    ego = np.stack([rng.uniform(-0.5, 0.5, (max_step + 2, N)), rng.uniform(-3, 3, (max_step + 2, N))], 2).astype(np.float32)

    def make(auto_reset):
        return BatchedTrafficEnv(None, replay=ep, device=cuda_device, max_step=max_step, auto_reset=auto_reset,
                                 observation="bev", bev_resolution=(24, 16), bev_range=15.0)
    steps = 2 * (max_step + 1) + 3 * (max_step + 1) + 1
    seen = _run(Case(make, _table_action(cuda_device, ego), steps=steps, shuffle_at=2 * (max_step + 1), oracle=False),
                cuda_device)
    assert seen["shuffled"] > N // 2   # scenarios the shuffle dealt another row
