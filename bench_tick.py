#!/usr/bin/env python
"""bench_tick.py - the fused tick (K1, `t2d_step_kernel`) alone, per scene, in microseconds per tick.

    python bench_tick.py [--scenes c2,c2_shuffled,c4,c5] [--steps K] [--reps R] [--c5-scenarios N]

Scenes: C2 (4096 x 64, bench.py's default), C2 with the slot order of every scenario shuffled (one random permutation per
scenario, applied to the state, the type ids and the actions alike: the same world with its slots renumbered), C4
(16384 x 32 mixed, inD_1) and C5 (rounD_0, M = 128; 16384 scenarios by default instead of 65536 to keep a run short).

Timing as in bench.py: the steps rotate over world replicas whose bytes exceed 2.5 x the L2, in chunks of 8 ticks per
replica that each start from the restored replicas; a chunk is one CUDA-graph replay timed with CUDA events, and the
restore stays outside the events.  Each scene is timed --reps times; one JSON line per scene, plus one naming the GPU and
its power limit.  `T2D_B200_LIB` selects another build of the library (A/B comparisons).  Nothing is written.
"""

from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import BYTES_PER_PARTICIPANT, BYTES_PER_SCENARIO, TICKS_PER_CHUNK, make_scene  # noqa: E402
from benchlib import gpu_info  # noqa: E402


def shuffled(scene, seed):
    """The scene with every scenario's slots in a random order; returns (scene, permutation [N, M])."""
    import dataclasses

    n, m = scene.shape
    perm = np.argsort(np.random.default_rng(seed).random((n, m)), axis=1)
    take = lambda a: np.ascontiguousarray(np.take_along_axis(a, perm, axis=1))
    return dataclasses.replace(scene, x=take(scene.x), y=take(scene.y), heading=take(scene.heading), speed=take(scene.speed),
                               vx=take(scene.vx), vy=take(scene.vy), type_id=take(scene.type_id),
                               name=scene.name + ", slots shuffled"), perm


def time_scene(key, args, device):
    import torch

    from tactics2d_b200 import BatchedWorld, synthetic

    config = "c2" if key.startswith("c2") else key
    n_cfg = args.c5_scenarios if key == "c5" else None
    scene0 = make_scene(config, seed=1, n=n_cfg)
    n, m = scene0.shape
    bytes_per_launch = n * m * BYTES_PER_PARTICIPANT + n * BYTES_PER_SCENARIO
    l2_bytes = torch.cuda.get_device_properties(device).L2_cache_size
    R = max(4, int(np.ceil(2.5 * l2_bytes / bytes_per_launch)))

    worlds, actions, pools = [], [], []
    for r in range(R):
        sc = scene0 if r == 0 else make_scene(config, seed=1 + r, n=n_cfg)
        act = synthetic.random_actions(9000 + r, (n, m))
        if key == "c2_shuffled":
            sc, perm = shuffled(sc, 500 + r)
            act = np.ascontiguousarray(np.take_along_axis(act, perm[..., None], axis=1))
        w = BatchedWorld(n, m, sc.table, device=device, max_step=0)
        w.set_map(sc.segments, sc.bounds)
        w.set_state(sc.x, sc.y, sc.heading, sc.speed, vx=sc.vx, vy=sc.vy, type_id=sc.type_id)
        worlds.append(w)
        actions.append(torch.from_numpy(act).to(device))
        pools.append({k: getattr(w, k).clone() for k in ("x", "y", "heading", "speed", "vx", "vy")})
    ones = torch.ones(n, dtype=torch.uint8, device=device)

    def restore():
        for w, p in zip(worlds, pools):
            w.reset(ones, p)

    C = TICKS_PER_CHUNK * R
    for i in range(3):
        worlds[i % R].step(actions[i % R])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(C):
            worlds[i % R].step(actions[i % R])
    n_chunks = max(1, args.steps // C)

    def timed():
        total = 0.0
        for _ in range(n_chunks):
            restore()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            total += e0.elapsed_time(e1)
        return total * 1e3 / (n_chunks * C)

    timed()   # warm-up of the exact timed path
    us = [timed() for _ in range(args.reps)]
    for w in worlds:
        w.close()
    return {"scene": key, "workload": scene0.name + (", slots shuffled" if key == "c2_shuffled" else ""), "N": n, "M": m,
            "replicas": R, "ticks_per_rep": n_chunks * C, "us_per_tick": us, "median_us": float(np.median(us))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="c2,c2_shuffled,c4,c5")
    ap.add_argument("--steps", type=int, default=8000, help="ticks per repetition (rounded down to whole chunks, at least one)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--c5-scenarios", type=int, default=16384)
    args = ap.parse_args()

    import torch

    import __graft_entry__ as entry

    entry.build()
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    print(json.dumps({"gpu": torch.cuda.get_device_name(device), "nvidia_smi": gpu_info().nvidia_smi,
                      "lib": os.environ.get("T2D_B200_LIB", "in-tree")}), flush=True)
    for key in args.scenes.split(","):
        if key not in ("c2", "c2_shuffled", "c4", "c5"):
            raise SystemExit(f"unknown scene {key}")
        print(json.dumps(time_scene(key, args, device)), flush=True)


if __name__ == "__main__":
    main()
