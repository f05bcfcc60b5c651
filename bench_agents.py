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


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--scenes", default="c2,c4")
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=40)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_agents.py measures on a CUDA device; none is visible")
    name, power = _gpu_info()
    for scene in args.scenes.split(","):
        print(json.dumps(dict(what="k10", scene=scene, gpu=name, power_limit=power, **time_k10(scene, args.seconds))), flush=True)
        print(json.dumps(dict(what="env_step", scene=scene, gpu=name, power_limit=power,
                              **time_env(scene, args.rounds, args.steps))), flush=True)


if __name__ == "__main__":
    main()
