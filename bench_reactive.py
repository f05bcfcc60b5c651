"""Time reactive replay (``BatchedWorld.set_reactive_replay``: K7's reactive instance, K17 on every track's own path and
K5's per-slot desired speed) against plain replay of the same log; one JSON line per measurement.

The scene is the car-following three-lane highway of ``synthetic.idm_highway_log`` (60 s, 100 ms records) with every
scenario on one episode row of 64 slots reused along the recording, 4096 scenarios.  Both variants bind the same paths,
controllers (an IDM row with a PID cross-track channel on every replayed slot) and leader search, so they differ only in
what reactive replay adds: every reactive slot follows its own path (K17's per-path projections), and the tick
integrates the handed-over slots.  Each line holds the median microseconds of one ``control`` + ``step`` over
``--rounds`` CUDA-event windows of ``--reps`` calls after ``--warmup`` ones, and the GPU name and power limit read in
the same run.
"""

from __future__ import annotations

import argparse
import json

import numpy as np

from benchlib import gpu_info, require_cuda

N, M = 4096, 64


def _world(eps, reactive):
    import torch

    from tactics2d_b200 import BatchedWorld
    from tactics2d_b200.controller import IDMController, PIDController

    row = np.zeros(N, np.int64)                          # every scenario runs row 0 of the episodes
    w = BatchedWorld(N, M, eps.table, device="cuda:0")
    w.set_log(eps.log, eps.t0, **eps.binding())
    paths, tp, ds = eps.log.track_paths()
    w.set_paths(paths)
    ctrl = np.zeros((N, M), np.uint8)
    ctrl[:, 0] = 255
    keep = PIDController(dt=0.1, kp_lat=0.03, ki_lat=0.0, kd_lat=0.08, max_steering=0.2, derivative_filter_alpha=1.0,
                         lateral_error="path_cross_track")
    w.set_controllers([IDMController(desired_speed=15.0, min_spacing=30.0, max_acceleration=8.0,
                                     comfortable_deceleration=9.0, lateral=keep)], ctrl)
    w.set_leader_search(1.8, 100.0)
    if reactive:
        w.set_reactive_replay(tp, desired_speed=ds)
    pool = {k: torch.from_numpy(np.ascontiguousarray(eps.pool[k], np.float32)).cuda()
            for k in ("x", "y", "heading", "speed", "vx", "vy")}
    w.type_id.copy_(torch.from_numpy(eps.type_id[row]).cuda())
    w.reset(torch.ones(N, dtype=torch.uint8, device="cuda:0"), pool,
            pool_index=torch.zeros(N, dtype=torch.int32, device="cuda:0"))
    return w, paths


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    require_cuda("bench_reactive.py")
    import torch

    from tactics2d_b200.dataset_parser.replay import build_replay_episodes
    from tactics2d_b200.synthetic import idm_highway_log
    from tactics2d_b200.types import TypeTable

    log = idm_highway_log(60000, 0, desired=(12.0, 14.0, 16.0), headway_s=5.0)
    k = int(np.argmax(log.n_frames))
    eps = build_replay_episodes(log, M, [int(log.first_ms[k])], [int(log.ids[k])], TypeTable.from_templates("kinematics"),
                                reuse_slots=True)
    name, power, _ = gpu_info()
    for reactive in (False, True):
        w, paths = _world(eps, reactive)
        act = torch.zeros((N, M, 2), dtype=torch.float32, device="cuda:0")

        def call():
            w.control(act)
            w.step(act)

        for _ in range(args.warmup):
            call()
        times = []
        for _ in range(args.rounds):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.reps):
                call()
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b) * 1e3 / args.reps)
        n_vert = [len(p) for p in paths]
        print(json.dumps(dict(bench="reactive_replay", variant="reactive" if reactive else "plain", N=N, M=M,
                              us_per_control_step=round(float(np.median(times)), 2),
                              spread=[round(min(times), 2), round(max(times), 2)],
                              reactive_slots=int((w.drive_path >= 0).sum()) if reactive else 0,
                              path_vertices=[min(n_vert), max(n_vert)], gpu=name, power_limit=power)))
        w.close()


if __name__ == "__main__":
    main()
