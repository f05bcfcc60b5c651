"""Time the sampled resets (DESIGN.md section 1 "Sampled resets") at the C2 shape, 4096 scenarios x 64 participants, every
scenario reset; one JSON line per measurement, each a CUDA graph of the call (``benchlib.time_graph``):

* ``reset``: ``BatchedWorld.reset`` (K2) from a pool of one row per scenario;
* ``sampled_rows``: ``reset_sampled`` with row draws and no jitter (K13, K2, K14 counting the episode);
* ``sampled_jitter``: the same with every slot jittered by up to 0.5 m, 0.1 rad and 0.5 m/s, at 8 and 32 tries (K14 checks
  every try of a slot against the bench scene's walls and every other slot);
* ``env_step``: ``BatchedTrafficEnv.step`` with such a sampler (T = 8) and without one, alternated in one run
  (``benchlib.alternate``), at a 1/200 done rate: ``max_step`` 200 and the step counters staggered over 0..199, so that
  about 20 scenarios auto-reset at every step.

Resets are off the tick's path; the numbers say what a reset of the whole batch costs next to a tick.  The GPU name and
power limit are read in the same run and printed on every line.
"""

from __future__ import annotations

import argparse
import json

import numpy as np

from benchlib import alternate, gpu_info, require_cuda, scene, time_graph


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5, help="length of one timed CUDA-graph window")
    ap.add_argument("--steps", type=int, default=400, help="env steps per alternation round")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    require_cuda("bench_reset.py")
    import torch

    from tactics2d_b200 import BatchedWorld

    name, power, _ = gpu_info()
    s = scene("c2")
    N, M = s.shape
    out = lambda **kw: print(json.dumps(dict(kw, N=N, M=M, gpu=name, power_limit=power)), flush=True)

    w = BatchedWorld(N, M, s.table, device="cuda:0")
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    dev = torch.device("cuda:0")
    pool = {k: torch.from_numpy(np.ascontiguousarray(getattr(s, k), dtype=np.float32)).to(dev)
            for k in ("x", "y", "heading", "speed")}
    mask = torch.ones(N, dtype=torch.uint8, device=dev)

    us, calls = time_graph(lambda: w.reset(mask, pool), args.seconds)
    out(what="reset", us=us, calls=calls)
    w.set_reset_sampler(seed=1)
    us, calls = time_graph(lambda: w.reset_sampled(mask, pool), args.seconds)
    out(what="sampled_rows", us=us, calls=calls)
    jit = np.tile(np.array([[-0.5, 0.5], [-0.5, 0.5], [-0.1, 0.1], [-0.5, 0.5]], np.float32), (M, 1, 1))
    for tries in (8, 32):
        w.set_reset_sampler(seed=1, jitter=jit, tries=tries)
        us, calls = time_graph(lambda: w.reset_sampled(mask, pool), args.seconds)
        torch.cuda.synchronize()
        placed = float((w.reset_try >= 0).float().mean())
        out(what="sampled_jitter", tries=tries, us=us, calls=calls, placed_fraction=placed)
    w.close()

    from tactics2d_b200.envs import BatchedTrafficEnv

    envs = {"no_sampler": BatchedTrafficEnv(s, max_step=200),
            "sampler": BatchedTrafficEnv(s, max_step=200, sampler=dict(seed=1, jitter=jit, tries=8))}
    act = torch.zeros((N, 2), dtype=torch.float32, device=dev)
    stagger = torch.from_numpy(np.random.default_rng(0).integers(0, 200, N).astype(np.int32)).to(dev)
    for e in envs.values():
        e.reset(seed=0)
        e.world.step_count.copy_(stagger)
    times = alternate({k: (lambda e=e: e.step(act)) for k, e in envs.items()}, args.rounds, args.steps)
    for k, v in times.items():
        out(what="env_step", env=k, us_per_step=sorted(v)[len(v) // 2], rounds=v, done_rate=1 / 200)
    for e in envs.values():
        e.close()


if __name__ == "__main__":
    main()
