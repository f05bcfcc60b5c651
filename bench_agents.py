"""Time the per-agent epilogue (K10, ``BatchedWorld.agents_epilogue``) and ``BatchedTrafficEnv.step`` with
``agent_rewards=True``; one JSON line per measurement.

Scenes: C2 (4096 scenarios x 64 vehicles on the synthetic grid map) and C4 (16384 x 32 mixed traffic on the inD_1 tile),
as ``bench.py`` builds them, every slot an agent (Q = M) and every row with a goal 1 m off its slot's pose: the worst case,
every box row runs both detector IoUs.

(a) K10 alone: CUDA events around CUDA-graph replays of 20 launches each, for at least ``--seconds`` after warm-up.  The
launches read an all-zero event byte array, no time limit is set and the NoAction limit is out of reach, so that no row
settles and every launch does the same work.  The line holds the bytes the launch must move (computed from the shapes:
per row the type gather, pose, flag, goal, detector state and extrema read and written, and the outputs; per slot the
flag and the TrafficStatus) and their share of the H100 SXM data sheet's 3.35 TB/s.

(b) ``BatchedTrafficEnv.step`` with ``observation="agents"`` (every slot observing, K = 16, S = 32) with and without
``agent_rewards``, alternating for ``--rounds`` rounds, in wall-clock microseconds per step ending in a synchronise.

The GPU name and power limit are read in the same run and printed on every line.

``--actions`` measures the per-agent action instead (K11, ``BatchedWorld.scatter_agent_action``):

(a) K11 alone at C2 and C4 with Q = M, once without an observer list and once with a list in which every scenario names
some slots twice (and so leaves others unnamed), timed like K10 above.  Bytes from the shapes: the agent actions and the
observers read, one type byte per slot, and at most one action per slot written.

(b) ``BatchedTrafficEnv.step`` with ``observation="agents"``, ``agent_rewards`` and ``agent_actions`` (an [N, Q, 2] action)
against the same env fed the pre-scattered [N, M, 2] action, alternating for ``--rounds`` rounds.

(c) ``BatchedWorld.step_host_agents`` (every slot an agent, Q = M) against ``step_host`` at C2, which uploads the same
2 MiB of actions per step, alternating, in wall-clock microseconds per step (both end in a synchronise).
"""

from __future__ import annotations

import argparse
import json

import numpy as np

from benchlib import PEAK_BYTES_PER_S, alternate, gpu_info, require_cuda, scene, time_graph


def _goals(s, device):
    """A goal 1 m ahead of every slot's initial pose, [N, M, 5]."""
    import torch

    g = np.stack([s.x + np.cos(s.heading), s.y + np.sin(s.heading), s.heading, np.full(s.x.shape, 2.4),
                  np.full(s.x.shape, 1.0)], -1).astype(np.float32)
    return torch.from_numpy(g).to(device)


def k10_bytes(n, m, q, observers=False, goals=True):
    """Bytes one K10 launch must read and write, from the shapes (each byte once)."""
    row_read = (2 if observers else 0) + 1 + 12 + 1 + 8   # observer, type, x y heading, flag, max_iou + min_dist
    row_write = 4 + 1 + 1 + 1 + 4 + 8                      # reward, terminated, truncated, status, iou, extrema
    if goals:
        row_read += 20 + 16 + 4                             # goal, last pose, NoAction count
        row_write += 16 + 4
    return n * q * (row_read + row_write) + n * m * (1 + 1) + n * (4 + 1)   # + flag / TrafficStatus per slot, steps / done


def time_k10(name, seconds):
    import ctypes as C

    import torch
    from tactics2d_b200 import BatchedWorld

    s = scene(name)
    n, m = s.shape
    w = BatchedWorld(n, m, s.table)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    w.set_agents(None, _goals(s, w.device), 0.95, 2**30)
    a = w._agents
    zero_flags = torch.zeros((n, m), dtype=torch.uint8, device=w.device)
    p = lambda t: C.c_void_p(t.data_ptr())
    args = [p(a[k]) for k in ("reward", "terminated", "truncated", "status", "iou", "done", "max_iou", "min_dist", "traffic")]

    def launch():
        w.lib.t2d_agents_epilogue(w._ctx, p(zero_flags), *args, 1, w._stream())

    us, _ = time_graph(launch, seconds, per_graph=20)
    assert int((a["status"] == 1).sum()) == int((w.type_id < len(w.type_table)).sum()), "a row settled"
    b = k10_bytes(n, m, m)
    w.close()
    return dict(us_per_call=round(us, 3), bytes=b, hbm_bound_us=round(b / PEAK_BYTES_PER_S * 1e6, 3),
                share_of_hbm_peak=round(b / PEAK_BYTES_PER_S * 1e6 / us, 3), n=n, m=m, q=m)


def _envs(s, **variants):
    """{label: a reset ``BatchedTrafficEnv`` with every slot observing (K = 16, S = 32), the goals of ``_goals`` and the
    keyword arguments of ``variants[label]``}."""
    from tactics2d_b200.envs import BatchedTrafficEnv

    envs = {}
    for label, kw in variants.items():
        cfg = dict(k_agents=16, k_segments=32, goals=_goals(s, "cuda:0"))
        envs[label] = BatchedTrafficEnv(s, max_step=200, observation="agents", vector_obs=cfg, **kw)
        envs[label].reset(seed=0)
    return envs


def time_env(name, rounds, steps):
    import torch

    s = scene(name)
    n, m = s.shape
    envs = _envs(s, ego_only=dict(agent_rewards=False), agent_rewards=dict(agent_rewards=True))
    act = torch.full((n, 2), 0.05, device="cuda:0")
    times = alternate({k: (lambda env=env: env.step(act)) for k, env in envs.items()}, rounds, steps)
    for env in envs.values():
        env.close()
    return dict(us_per_step_ego_only=[round(v, 1) for v in times["ego_only"]],
                us_per_step_agent_rewards=[round(v, 1) for v in times["agent_rewards"]], n=n, m=m, q=m)


def k11_bytes(n, m, q, observers):
    """Bytes one K11 launch moves at most, from the shapes: agent actions, observers and types read, every slot written."""
    return n * q * 8 + (n * q * 2 if observers else 0) + n * m + n * m * 8


def _duplicate_list(n, m, seed=0):
    """int16 [n, m]: every row a slot of its scenario, about a third of them naming a slot an earlier row names."""
    rng = np.random.default_rng(seed)
    obs = np.broadcast_to(np.arange(m, dtype=np.int16), (n, m)).copy()
    dup = rng.uniform(0, 1, (n, m)) < 1 / 3
    obs[dup] = rng.integers(0, m, int(dup.sum()))
    return obs


def time_k11(name, seconds, with_list):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    s = scene(name)
    n, m = s.shape
    w = BatchedWorld(n, m, s.table)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    obs = torch.from_numpy(_duplicate_list(n, m)).to(w.device) if with_list else None
    rows = torch.from_numpy(synthetic.random_actions(1, (n, m))).to(w.device)
    act = torch.zeros((n, m, 2), dtype=torch.float32, device=w.device)
    us, _ = time_graph(lambda: w.scatter_agent_action(rows, act, obs), seconds, per_graph=20)
    b = k11_bytes(n, m, m, with_list)
    w.close()
    return dict(us_per_call=round(us, 3), bytes_at_most=b, hbm_bound_us=round(b / PEAK_BYTES_PER_S * 1e6, 3),
                share_of_hbm_peak=round(b / PEAK_BYTES_PER_S * 1e6 / us, 3), n=n, m=m, q=m,
                observers="duplicates" if with_list else "none")


def time_env_actions(name, rounds, steps):
    import torch
    from tactics2d_b200 import synthetic

    s = scene(name)
    n, m = s.shape
    envs = _envs(s, prescattered=dict(agent_rewards=True, agent_actions=False),
                 agent_actions=dict(agent_rewards=True, agent_actions=True))
    rows = torch.from_numpy(synthetic.random_actions(2, (n, m), accel=(-0.1, 0.1), steer=(-0.05, 0.05))).cuda()
    act = {"agent_actions": rows, "prescattered": rows.clone()}   # Q = M without a list: the pre-scattered action is the same
    times = alternate({k: (lambda env=env, a=act[k]: env.step(a)) for k, env in envs.items()}, rounds, steps)
    for env in envs.values():
        env.close()
    return dict(us_per_step_prescattered=[round(v, 1) for v in times["prescattered"]],
                us_per_step_agent_actions=[round(v, 1) for v in times["agent_actions"]], n=n, m=m, q=m)


def time_host_step(rounds, steps):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    s = scene("c2")
    n, m = s.shape
    worlds = {}
    for agents in (False, True):
        w = BatchedWorld(n, m, s.table)
        w.set_map(s.segments, s.bounds)
        w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
        if agents:
            w.set_agents()
        worlds[agents] = w
    host = torch.from_numpy(synthetic.random_actions(3, (n, m), accel=(-0.1, 0.1), steer=(-0.05, 0.05))).pin_memory()
    # the warm-up also makes the staging allocations
    times = alternate({False: lambda: worlds[False].step_host(host), True: lambda: worlds[True].step_host_agents(host)},
                      rounds, steps)
    for w in worlds.values():
        w.close()
    return dict(us_per_step_step_host=[round(v, 1) for v in times[False]],
                us_per_step_step_host_agents=[round(v, 1) for v in times[True]], n=n, m=m, q=m,
                upload_bytes=n * m * 8, download_bytes_step_host=2 * n, download_bytes_step_host_agents=7 * n * m + n)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--scenes", default="c2,c4")
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--actions", action="store_true", help="measure the per-agent action (K11) and the host step instead")
    args = ap.parse_args()
    require_cuda("bench_agents.py")
    name, power, _ = gpu_info()
    if args.actions:
        for key in args.scenes.split(","):
            for with_list in (False, True):
                print(json.dumps(dict(what="k11", scene=key, gpu=name, power_limit=power,
                                      **time_k11(key, args.seconds, with_list))), flush=True)
            print(json.dumps(dict(what="env_step_actions", scene=key, gpu=name, power_limit=power,
                                  **time_env_actions(key, args.rounds, args.steps))), flush=True)
        print(json.dumps(dict(what="host_step", scene="c2", gpu=name, power_limit=power,
                              **time_host_step(args.rounds, args.steps))), flush=True)
        return
    for key in args.scenes.split(","):
        print(json.dumps(dict(what="k10", scene=key, gpu=name, power_limit=power, **time_k10(key, args.seconds))), flush=True)
        print(json.dumps(dict(what="env_step", scene=key, gpu=name, power_limit=power,
                              **time_env(key, args.rounds, args.steps))), flush=True)


if __name__ == "__main__":
    main()
