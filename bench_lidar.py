"""Time the single-line lidar (K4): the ego scan (``BatchedWorld.lidar_scan``) and the per-agent scan
(``BatchedWorld.lidar_scan_agents``), and ``BatchedTrafficEnv.step`` with and without ``lidar=``; one JSON line per
measurement.

Scenes: C2 (4096 scenarios x 64 vehicles on the synthetic grid map) and C4 (16384 x 32 mixed traffic on the inD_1 tile), as
``bench.py`` builds them, at (360 beams, 20 m: ``ParkingEnv``'s lidar) and (500 beams, 12 m: the reference's defaults).

(a) The kernel alone: CUDA events around CUDA-graph replays of 20 launches each, for at least ``--seconds`` after warm-up,
for the ego scan, Q = 8 (an explicit list of slots 0..7) and Q = M (every slot, no list).  The line holds the bytes the
launch must move (computed from the shapes: the fp32 output N·Q·B·4, the observer list, the observers' and the other
slots' pose and type, the beam table) and their share of the H100 SXM data sheet's 3.35 TB/s.  On a tree without
``lidar_scan_agents`` only the ego scan is timed, so the same script measures a tree before the per-agent scan.

(b) ``BatchedTrafficEnv.step`` with ``observation="agents"`` (every slot observing, K = 16, S = 32) with and without
``lidar=dict(n_beams=360, max_range=20.0)``, alternating for ``--rounds`` rounds, in wall-clock microseconds per step
ending in a synchronise.

The GPU name and power limit are read in the same run and printed on every line.
"""

from __future__ import annotations

import argparse
import json

import numpy as np

from benchlib import PEAK_BYTES_PER_S, alternate, gpu_info, require_cuda, scene, time_graph

SETTINGS = ((360, 20.0), (500, 12.0))


def lidar_bytes(n, m, q, n_beams, observers):
    """Bytes one launch must move, from the shapes (each byte once): the output, the list, every slot's pose and type
    (the observers' and the obstacles'), the beam table."""
    return n * q * n_beams * 4 + (n * q * 2 if observers else 0) + n * m * (12 + 1) + n_beams * 16


def time_kernel(name, seconds, ego_only=False):
    """One dict per (setting, variant)."""
    import torch
    from tactics2d_b200 import BatchedWorld

    s = scene(name)
    n, m = s.shape
    w = BatchedWorld(n, m, s.table)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    agents = hasattr(w, "lidar_scan_agents") and not ego_only
    first8 = torch.from_numpy(np.broadcast_to(np.arange(8, dtype=np.int16), (n, 8)).copy()).to(w.device)
    out = []
    for n_beams, max_range in SETTINGS:
        variants = [("ego", 1, False, lambda: w.lidar_scan(n_beams, max_range))]
        if agents:
            variants += [("agents", 8, True, lambda: w.lidar_scan_agents(n_beams, max_range, observers=first8)),
                         ("agents", m, False, lambda: w.lidar_scan_agents(n_beams, max_range))]
        for call, q, with_list, launch in variants:
            us, _ = time_graph(launch, seconds, per_graph=20)
            b = lidar_bytes(n, m, q, n_beams, with_list)
            out.append(dict(call=call, n_beams=n_beams, max_range=max_range, us_per_call=round(us, 2), bytes=b,
                            hbm_bound_us=round(b / PEAK_BYTES_PER_S * 1e6, 2),
                            share_of_hbm_peak=round(b / PEAK_BYTES_PER_S * 1e6 / us, 3), n=n, m=m, q=q,
                            observers="slots 0..7" if with_list else "none"))
    w.__dict__.pop("_agent_lidar", None)
    w.close()
    return out


def time_env(name, rounds, steps):
    import torch
    from tactics2d_b200.envs import BatchedTrafficEnv

    s = scene(name)
    n, m = s.shape
    envs = {}
    for lidar in (False, True):
        envs[lidar] = BatchedTrafficEnv(s, max_step=200, observation="agents", vector_obs=dict(k_agents=16, k_segments=32),
                                        lidar=dict(n_beams=360, max_range=20.0) if lidar else None)
        envs[lidar].reset(seed=0)
    act = torch.full((n, 2), 0.05, device="cuda:0")
    times = alternate({lidar: (lambda env=env: env.step(act)) for lidar, env in envs.items()}, rounds, steps)
    for env in envs.values():
        env.close()
    return dict(us_per_step_without_lidar=[round(v, 1) for v in times[False]],
                us_per_step_with_lidar=[round(v, 1) for v in times[True]], n=n, m=m, q=m, n_beams=360, max_range=20.0)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--scenes", default="c2,c4")
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--ego-only", action="store_true", help="time the ego scan alone (no per-agent scan, no env step)")
    args = ap.parse_args()
    require_cuda("bench_lidar.py")
    from tactics2d_b200 import BatchedWorld

    name, power, _ = gpu_info()
    for key in args.scenes.split(","):
        for r in time_kernel(key, args.seconds, args.ego_only):
            print(json.dumps(dict(what="lidar", scene=key, gpu=name, power_limit=power, **r)), flush=True)
    if hasattr(BatchedWorld, "lidar_scan_agents") and not args.ego_only:
        for key in args.scenes.split(","):
            print(json.dumps(dict(what="env_step_lidar", scene=key, gpu=name, power_limit=power,
                                  **time_env(key, args.rounds, args.steps))), flush=True)


if __name__ == "__main__":
    main()
