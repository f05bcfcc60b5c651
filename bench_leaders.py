"""Time the leader search (K17, ``BatchedWorld.find_leaders``) and the controller launch with and without a bound search at
the C2 shape, 4096 scenarios x 64 participants; one JSON line per measurement.

(a) ``heading``: no paths, every follower in the heading frame.
(b) ``path_lanes``: four straight 8-vertex lane paths, every slot on the path of its lane (four distinct paths per scenario).
(c) ``path_worst``: every slot on a 32-vertex path of its own (64 distinct paths per scenario, each projected once).
(d) ``control`` / ``control_search``: ``BatchedWorld.control`` with every NPC on an IDM row on the lane scene, without and
    with ``set_leader_search``.

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


def _lanes(rng):
    """Participants spread along four lanes of a 300 m road, a little off their lane's centre line."""
    lane = rng.integers(0, LANES, (N, M))
    x = rng.uniform(0.0, 300.0, (N, M))
    y = LANE_W * lane + rng.normal(0.0, 0.3, (N, M))
    h = rng.normal(0.0, 0.05, (N, M))
    return [a.astype(np.float32) for a in (x, y, h)] + [lane]


def _path(y0, n_vert, wiggle):
    x = np.linspace(-20.0, 320.0, n_vert)
    return np.stack([x, y0 + wiggle * np.sin(x / 40.0)], 1).astype(np.float32)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    require_cuda("bench_leaders.py")
    import torch

    from tactics2d_b200 import BatchedWorld
    from tactics2d_b200.controller import IDMController
    from tactics2d_b200.types import TypeParams, TypeTable

    name, power, _ = gpu_info()
    rng = np.random.default_rng(17)
    x, y, h, lane = _lanes(rng)
    table = TypeTable([TypeParams(half_len=2.4, half_wid=0.95, lf=1.3, lr=1.3, accel_lo=-6.0, accel_hi=3.0)])
    w = BatchedWorld(N, M, table)
    w.set_state(x, y, h, np.full((N, M), 12.0, np.float32), type_id=np.zeros((N, M), np.uint8))

    def line(case, us, spread):
        print(json.dumps(dict(what="leaders", case=case, N=N, M=M, us_per_call=round(us, 2), us_spread=spread, gpu=name,
                              power_limit=power)), flush=True)

    find = lambda: w.find_leaders(1.8, 100.0)
    line("heading", *_time(find, args))
    ids = np.full((N, M), 255, np.uint8)
    w.set_paths([_path(LANE_W * k, 8, 0.0) for k in range(LANES)])
    w.set_controllers([IDMController()], ids, path_id=lane.astype(np.int16))
    line("path_lanes", *_time(find, args))
    w.set_paths([_path(LANE_W * (k % LANES), 32, 0.5) for k in range(M)])
    w.set_controllers([IDMController()], ids, path_id=np.tile(np.arange(M, dtype=np.int16), (N, 1)))
    line("path_worst", *_time(find, args))

    ids = np.zeros((N, M), np.uint8)
    ids[:, 0] = 255
    w.set_paths([_path(LANE_W * k, 8, 0.0) for k in range(LANES)])
    w.set_controllers([IDMController()], ids, path_id=lane.astype(np.int16))
    action = torch.zeros((N, M, 2), dtype=torch.float32, device=w.device)
    control = lambda: w.control(action)
    line("control", *_time(control, args))
    w.set_leader_search(1.8, 100.0)
    line("control_search", *_time(control, args))


if __name__ == "__main__":
    main()
