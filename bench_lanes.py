"""Time the lane change (K18, ``BatchedWorld.set_lane_change``) at the C2 shape, 4096 scenarios x 64 participants on four
straight 8-vertex lanes with neighbour links; one JSON line per measurement.

(a) ``control_search``: ``BatchedWorld.control`` with every NPC on an IDM row with lane keeping and a bound leader search.
(b) ``control_lanes``: the same with a bound lane change (K18, then K17, then K5).
(c) ``k18``: K18 alone, its kernel time inside (b) from ``torch.profiler``.

CUDA events around ``--reps`` launches after ``--warmup`` ones, repeated ``--rounds`` times; the line holds the median
microseconds per call.  The GPU name and power limit are read in the same run and printed on every line.
"""

from __future__ import annotations

import argparse
import json

import numpy as np

from benchlib import gpu_info, require_cuda

N, M = 4096, 64
LANES, LANE_W = 4, 3.5


def _time(fn, args):
    import torch

    for _ in range(args.warmup):
        fn()
    times = []
    for _ in range(args.rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.reps):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / args.reps)
    return float(np.median(times)), [round(min(times), 2), round(max(times), 2)]


def _kernel_time(fn, args, name):
    """Median over rounds of the mean device time of the kernels whose name holds ``name``, per call of ``fn``."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    for _ in range(args.warmup):
        fn()
    times = []
    for _ in range(args.rounds):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                fn()
            torch.cuda.synchronize()
        total = sum(e.device_time_total for e in prof.key_averages() if name in e.key)
        times.append(total / args.reps)
    return float(np.median(times)), [round(min(times), 2), round(max(times), 2)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    require_cuda("bench_lanes.py")
    import torch

    from tactics2d_b200 import BatchedWorld
    from tactics2d_b200.controller import IDMController, PIDController
    from tactics2d_b200.types import TypeParams, TypeTable

    name, power, _ = gpu_info()
    rng = np.random.default_rng(18)
    lane = rng.integers(0, LANES, (N, M))
    x = rng.uniform(0.0, 300.0, (N, M)).astype(np.float32)
    y = (LANE_W * lane + rng.normal(0.0, 0.3, (N, M))).astype(np.float32)
    h = rng.normal(0.0, 0.05, (N, M)).astype(np.float32)
    v = rng.uniform(6.0, 16.0, (N, M)).astype(np.float32)
    table = TypeTable([TypeParams(half_len=2.4, half_wid=0.95, lf=1.3, lr=1.3, accel_lo=-6.0, accel_hi=3.0)])
    w = BatchedWorld(N, M, table)
    w.set_state(x, y, h, v, type_id=np.zeros((N, M), np.uint8))

    def line(case, us, spread):
        print(json.dumps(dict(what="lanes", case=case, N=N, M=M, us_per_call=round(us, 2), us_spread=spread, gpu=name,
                              power_limit=power)), flush=True)

    ids = np.zeros((N, M), np.uint8)
    ids[:, 0] = 255
    xs = np.linspace(-20.0, 320.0, 8)
    w.set_paths([np.stack([xs, np.full(8, LANE_W * k)], 1).astype(np.float32) for k in range(LANES)])
    keep = PIDController(dt=0.1, kp_lat=0.03, kd_lat=0.08, max_steering=0.2, lateral_error="path_cross_track")
    w.set_controllers([IDMController(desired_speed=14.0, lateral=keep)], ids, path_id=lane.astype(np.int16))
    w.set_leader_search(1.8, 100.0)
    action = torch.zeros((N, M, 2), dtype=torch.float32, device=w.device)
    control = lambda: w.control(action)
    line("control_search", *_time(control, args))
    left = [k + 1 if k + 1 < LANES else -1 for k in range(LANES)]
    right = [k - 1 for k in range(LANES)]
    # a cooldown of 0 and a low threshold keep every car deciding every call, whatever the previous calls changed
    w.set_lane_change(left, right, politeness=0.2, threshold=0.1, b_safe=3.0, min_gap=6.0, cooldown=0)
    line("control_lanes", *_time(control, args))
    line("k18", *_kernel_time(control, args, "lane_change_kernel"))


if __name__ == "__main__":
    main()
