"""Time the NPC controller launch (K5, ``BatchedWorld.control``) at the C2 shape, 4096 scenarios x 64 participants; one
JSON line per measurement.

(a) ``idm``: every participant but the ego on an IDM row - the controller ``bench.py``'s end-to-end line runs.
(b) ``pid_path8`` / ``pid_path32``: every NPC on a PID row with the PATH_CROSS_TRACK lateral error and a speed target, on
    paths of 8 and 32 vertices.
(c) ``mixed``: the NPCs spread over IDM, cruise, pure pursuit and PID rows.

CUDA events around ``--reps`` launches after ``--warmup`` ones, repeated ``--rounds`` times; the line holds the median
microseconds per call and the algorithmic bytes of one call (action in and out, last_accel in and out, the PID state
read and written and the PID target read, the ctrl_id / type_id bytes and the fp32 state each law reads; paths, which
stay in L2, excluded) as a share of the H100 SXM data sheet's 3.35 TB/s.  The GPU name and power limit are read in the
same run and printed on every line.
"""

from __future__ import annotations

import argparse
import json

import numpy as np

from benchlib import PEAK_BYTES_PER_S, gpu_info, require_cuda

N, M = 4096, 64


def _path(n_vert, k):
    x = np.linspace(-100.0, 100.0, n_vert)
    return np.stack([x, 20.0 * np.sin(x / 30.0 + k)], 1).astype(np.float32)


def _bytes(ctrl_id, kinds, is_pid):
    """Bytes one call must move: per slot the type and ctrl ids (2 B), last_accel read + written (8 B); per controlled
    slot the action written (8 B) and x, y, speed, heading (16 B); per PID slot its state read + written (96 B) and its
    target (8 B); the action of the uncontrolled slots is read (8 B)."""
    controlled = ctrl_id != 255
    n_pid = int(is_pid.sum())
    return (N * M * (2 + 8) + int(controlled.sum()) * (8 + 16) + int((~controlled).sum()) * 8 + n_pid * (96 + 8))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    require_cuda("bench_control.py")
    import torch

    from tactics2d_b200 import BatchedWorld, synthetic
    from tactics2d_b200.controller import AccelerationController, IDMController, PIDController, PurePursuitController

    name, power, _ = gpu_info()
    scene = synthetic.config4(N, M, seed=4)
    w = BatchedWorld(N, M, scene.table)
    w.set_state(scene.x, scene.y, scene.heading, scene.speed, vx=scene.vx, vy=scene.vy, type_id=scene.type_id)
    rng = np.random.default_rng(1)
    pid = PIDController(lateral_error="path_cross_track", dt=0.1)
    pp = PurePursuitController()
    cases = []
    ids = np.zeros((N, M), np.uint8)
    ids[:, 0] = 255
    cases.append(("idm", [IDMController()], ids, None))
    for nv in (8, 32):
        cases.append((f"pid_path{nv}", [pid], ids.copy(), nv))
    mixed = rng.integers(0, 4, (N, M)).astype(np.uint8)
    mixed[:, 0] = 255
    cases.append(("mixed", [IDMController(), AccelerationController(), pp, pid], mixed, 32))
    target = np.stack([rng.uniform(0, 15, (N, M)), np.zeros((N, M))], 2).astype(np.float32)
    action = torch.zeros((N, M, 2), dtype=torch.float32, device=w.device)
    for case, ctrls, cid, nv in cases:
        if nv is not None:
            w.set_paths([_path(nv, k) for k in range(16)])
        path_id = rng.integers(0, 16, (N, M)).astype(np.int16)
        rows = [c.params() for c in ctrls]
        w.set_controllers(rows, cid, path_id=path_id, pid_target=target)
        is_pid = np.isin(cid, [i for i, r in enumerate(rows) if r.kind == 4])
        for _ in range(args.warmup):
            w.control(action)
        times = []
        for _ in range(args.rounds):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.reps):
                w.control(action)
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b) * 1e3 / args.reps)
        us = float(np.median(times))
        nbytes = _bytes(cid, rows, is_pid)
        print(json.dumps(dict(what="control", case=case, N=N, M=M, us_per_call=round(us, 2),
                              us_spread=[round(min(times), 2), round(max(times), 2)], algorithmic_bytes=nbytes,
                              hbm_share=round(nbytes / (us * 1e-6) / PEAK_BYTES_PER_S, 4), gpu=name, power_limit=power)),
              flush=True)


if __name__ == "__main__":
    main()
