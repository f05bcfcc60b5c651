"""Time yielding at conflict zones (K19, ``BatchedWorld.set_yielding``) at the C2 shape, 4096 scenarios x 64 participants
on the four-arm intersection of ``synthetic.intersection`` (16 IDM cars with lane keeping per arm); one JSON line per
measurement.

(a) ``search``: ``control`` + ``step`` with a bound leader search (K17, K5, K1).
(b) ``search_yield``: the same with bound yielding (K17, K19, then K5's yielding instance, K1).
(c) ``find_yields``: ``find_yields`` alone (one K19 launch) on the scene's start state.

(a) and (b) start every round from the scene's start state, so that every round times the same 10 s of traffic at the
default ``--reps`` (100 ms ticks).  CUDA events around ``--reps`` calls after ``--warmup`` ones, repeated ``--rounds``
times; the line holds the median microseconds per call.  The GPU name and power limit are read in the same run and
printed on every line.
"""

from __future__ import annotations

import argparse
import json

import numpy as np

from benchlib import gpu_info, require_cuda

N, M = 4096, 64


def _time(fn, args, before=None):
    import torch

    if before:
        before()
    for _ in range(args.warmup):
        fn()
    times = []
    for _ in range(args.rounds):
        if before:
            before()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.reps):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / args.reps)
    return float(np.median(times)), [round(min(times), 2), round(max(times), 2)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    require_cuda("bench_yield.py")
    import torch

    from tactics2d_b200 import BatchedWorld, synthetic

    name, power, _ = gpu_info()
    sc = synthetic.intersection(N, M, seed=19)
    w = BatchedWorld(N, M, sc.table, interval=100)
    w.set_paths(sc.paths)
    w.set_controllers([synthetic.path_controller()], sc.ctrl_id, path_id=sc.path_id)
    w.set_leader_search(1.8, 100.0)
    action = torch.zeros((N, M, 2), dtype=torch.float32, device=w.device)

    def start():
        w.set_state(sc.x, sc.y, sc.heading, sc.speed, type_id=sc.type_id)
        w.pid_state.zero_()

    def tick():
        w.control(action)
        w.step(action)

    def line(case, us, spread, **extra):
        print(json.dumps(dict(what="yield", case=case, N=N, M=M, us_per_call=round(us, 2), us_spread=spread, gpu=name,
                              power_limit=power, **extra)), flush=True)

    line("search", *_time(tick, args, start))
    w.set_yielding(priority=sc.priority)
    line("search_yield", *_time(tick, args, start), zones=len(w.conflict_zones))
    start()
    yields = int((w.find_yields()[0] >= 0).sum())
    line("find_yields", *_time(w.find_yields, args), yielding_slots_at_start=yields)


if __name__ == "__main__":
    main()
