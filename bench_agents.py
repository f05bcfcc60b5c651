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
import time

import numpy as np

PEAK_BYTES_PER_S = 3.35e12


def _gpu_info():
    import subprocess

    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (v.strip() for v in out.split(","))
        return name, power
    except Exception:
        import torch

        return torch.cuda.get_device_name(0), "unknown"


def _scene(name):
    from tactics2d_b200 import synthetic
    from tactics2d_b200.map import load_collidable_segments

    if name == "c2":
        return synthetic.config2(4096, 64, seed=1)
    seg, b = load_collidable_segments("inD_1")
    return synthetic.config4(16384, 32, seed=4, segments=seg, bounds=b)


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


def time_k10(name, seconds, reps=20):
    import ctypes as C

    import torch
    from tactics2d_b200 import BatchedWorld

    s = _scene(name)
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

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            launch()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            launch()
    for _ in range(5):
        g.replay()
    torch.cuda.synchronize()
    assert int((a["status"] == 1).sum()) == int((w.type_id < len(w.type_table)).sum()), "a row settled"
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    calls, ms = 0, 0.0
    t_end = time.perf_counter() + seconds
    while time.perf_counter() < t_end:
        e0.record()
        for _ in range(10):
            g.replay()
        e1.record()
        e1.synchronize()
        ms += e0.elapsed_time(e1)
        calls += 10 * reps
    us = ms * 1e3 / calls
    b = k10_bytes(n, m, m)
    w.close()
    return dict(us_per_call=round(us, 3), bytes=b, hbm_bound_us=round(b / PEAK_BYTES_PER_S * 1e6, 3),
                share_of_hbm_peak=round(b / PEAK_BYTES_PER_S * 1e6 / us, 3), n=n, m=m, q=m)


def time_env(name, rounds, steps):
    import torch
    from tactics2d_b200.envs import BatchedTrafficEnv

    s = _scene(name)
    n, m = s.shape
    envs = {}
    for rewards in (False, True):
        cfg = dict(k_agents=16, k_segments=32, goals=_goals(s, "cuda:0"))
        envs[rewards] = BatchedTrafficEnv(s, max_step=200, observation="agents", vector_obs=cfg, agent_rewards=rewards)
        envs[rewards].reset(seed=0)
    act = torch.full((n, 2), 0.05, device="cuda:0")
    for env in envs.values():   # warm-up
        for _ in range(3):
            env.step(act)
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for _ in range(rounds):
        for rewards, env in envs.items():
            t0 = time.perf_counter()
            for _ in range(steps):
                env.step(act)
            torch.cuda.synchronize()
            times[rewards].append((time.perf_counter() - t0) * 1e6 / steps)
    for env in envs.values():
        env.close()
    return dict(us_per_step_ego_only=[round(v, 1) for v in times[False]],
                us_per_step_agent_rewards=[round(v, 1) for v in times[True]], n=n, m=m, q=m)


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


def time_k11(name, seconds, with_list, reps=20):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    s = _scene(name)
    n, m = s.shape
    w = BatchedWorld(n, m, s.table)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    obs = torch.from_numpy(_duplicate_list(n, m)).to(w.device) if with_list else None
    rows = torch.from_numpy(synthetic.random_actions(1, (n, m))).to(w.device)
    act = torch.zeros((n, m, 2), dtype=torch.float32, device=w.device)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            w.scatter_agent_action(rows, act, obs)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            w.scatter_agent_action(rows, act, obs)
    for _ in range(5):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    calls, ms = 0, 0.0
    t_end = time.perf_counter() + seconds
    while time.perf_counter() < t_end:
        e0.record()
        for _ in range(10):
            g.replay()
        e1.record()
        e1.synchronize()
        ms += e0.elapsed_time(e1)
        calls += 10 * reps
    us = ms * 1e3 / calls
    b = k11_bytes(n, m, m, with_list)
    w.close()
    return dict(us_per_call=round(us, 3), bytes_at_most=b, hbm_bound_us=round(b / PEAK_BYTES_PER_S * 1e6, 3),
                share_of_hbm_peak=round(b / PEAK_BYTES_PER_S * 1e6 / us, 3), n=n, m=m, q=m,
                observers="duplicates" if with_list else "none")


def time_env_actions(name, rounds, steps):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    s = _scene(name)
    n, m = s.shape
    envs = {}
    for scatter in (False, True):
        cfg = dict(k_agents=16, k_segments=32, goals=_goals(s, "cuda:0"))
        envs[scatter] = BatchedTrafficEnv(s, max_step=200, observation="agents", vector_obs=cfg, agent_rewards=True,
                                          agent_actions=scatter)
        envs[scatter].reset(seed=0)
    rows = torch.from_numpy(synthetic.random_actions(2, (n, m), accel=(-0.1, 0.1), steer=(-0.05, 0.05))).cuda()
    act = {True: rows, False: rows.clone()}   # Q = M without a list: the pre-scattered action is the same array
    for scatter, env in envs.items():   # warm-up
        for _ in range(3):
            env.step(act[scatter])
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for _ in range(rounds):
        for scatter, env in envs.items():
            t0 = time.perf_counter()
            for _ in range(steps):
                env.step(act[scatter])
            torch.cuda.synchronize()
            times[scatter].append((time.perf_counter() - t0) * 1e6 / steps)
    for env in envs.values():
        env.close()
    return dict(us_per_step_prescattered=[round(v, 1) for v in times[False]],
                us_per_step_agent_actions=[round(v, 1) for v in times[True]], n=n, m=m, q=m)


def time_host_step(rounds, steps):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    s = _scene("c2")
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
    run = {False: lambda: worlds[False].step_host(host), True: lambda: worlds[True].step_host_agents(host)}
    for f in run.values():   # warm-up (and the staging allocations)
        for _ in range(3):
            f()
    times = {False: [], True: []}
    for _ in range(rounds):
        for agents, f in run.items():
            t0 = time.perf_counter()
            for _ in range(steps):
                f()
            times[agents].append((time.perf_counter() - t0) * 1e6 / steps)
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
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_agents.py measures on a CUDA device; none is visible")
    name, power = _gpu_info()
    if args.actions:
        for scene in args.scenes.split(","):
            for with_list in (False, True):
                print(json.dumps(dict(what="k11", scene=scene, gpu=name, power_limit=power,
                                      **time_k11(scene, args.seconds, with_list))), flush=True)
            print(json.dumps(dict(what="env_step_actions", scene=scene, gpu=name, power_limit=power,
                                  **time_env_actions(scene, args.rounds, args.steps))), flush=True)
        print(json.dumps(dict(what="host_step", scene="c2", gpu=name, power_limit=power,
                              **time_host_step(args.rounds, args.steps))), flush=True)
        return
    for scene in args.scenes.split(","):
        print(json.dumps(dict(what="k10", scene=scene, gpu=name, power_limit=power, **time_k10(scene, args.seconds))), flush=True)
        print(json.dumps(dict(what="env_step", scene=scene, gpu=name, power_limit=power,
                              **time_env(scene, args.rounds, args.steps))), flush=True)


if __name__ == "__main__":
    main()
