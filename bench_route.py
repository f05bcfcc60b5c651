"""Time route following (DESIGN.md section 1 "Route following") at the C2 shape, 4096 scenarios x 64 participants; one
JSON line per measurement.

(a) ``env_step``: ``BatchedTrafficEnv.step`` without routes and with a route of 8 and of 64 vertices per ego (a straight
    line from the ego's start along its heading, so that the egos stay on it), the three envs alternated in one run
    (``benchlib.alternate``): the OffRoute probe and progress term in the env epilogue, and K12 at P = 8 into
    ``info["route"]`` after the auto-reset.
(b) ``agent_rewards``: K10 (``BatchedWorld.agents_epilogue``) at Q = 64, every row's slot on one of 16 shared routes of
    64 vertices across the scene, and the same launch without routes, each in a CUDA graph (``benchlib.time_graph``).
    Every row runs the whole closest-point walk whether it ends on or off its route, so the shared routes cost what
    routes of the rows' own would.
(c) ``route_observe``: K12 alone at Q = 64 rows per scenario and P = 8 and 32 look-ahead points, in a CUDA graph.

The algorithmic bytes of (b) and (c) are those the launch must move from and to HBM (the route vertices, which stay in
L2, excluded), printed beside the time with their share of the H100 SXM data sheet's 3.35 TB/s.  The GPU name and power
limit are read in the same run and printed on every line.
"""

from __future__ import annotations

import argparse
import json

import numpy as np

from benchlib import PEAK_BYTES_PER_S, alternate, gpu_info, require_cuda, scene, time_graph


def _routes(s, n_vert, slots):
    """One straight route of ``n_vert`` vertices per (scenario, slot) of ``slots``, 100 m long from the slot's start along
    its heading: (paths, route_id [N, M])."""
    N, M = s.shape
    paths, rid = [], np.full((N, M), -1, np.int16)
    t = np.linspace(-10.0, 90.0, n_vert)
    for m in slots:
        x, y, h = s.x[:, m].astype(np.float64), s.y[:, m].astype(np.float64), s.heading[:, m].astype(np.float64)
        for n in range(N):
            rid[n, m] = len(paths)
            paths.append(np.stack([x[n] + t * np.cos(h[n]), y[n] + t * np.sin(h[n])], 1).astype(np.float32))
    return paths, rid


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50, help="env steps per alternation round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=0.5, help="length of one timed CUDA-graph window")
    args = ap.parse_args()
    require_cuda("bench_route.py")
    import torch

    from tactics2d_b200 import BatchedWorld
    from tactics2d_b200.envs import BatchedTrafficEnv

    name, power, _ = gpu_info()
    s = scene("c2")
    N, M = s.shape
    out = lambda **kw: print(json.dumps(dict(kw, N=N, M=M, gpu=name, power_limit=power)), flush=True)

    # (a) the env step with and without routes
    envs = {"none": BatchedTrafficEnv(s, max_step=200)}
    for nv in (8, 64):
        paths, rid = _routes(s, nv, [0])
        envs[f"route{nv}"] = BatchedTrafficEnv(s, max_step=200, route=dict(paths=paths, route_id=rid[:, 0], threshold=5.0))
    for env in envs.values():
        env.reset(seed=0)
    act = torch.zeros((N, 2), dtype=torch.float32, device="cuda")
    times = alternate({k: (lambda env=env: env.step(act)) for k, env in envs.items()}, args.rounds, args.steps)
    for k, t in times.items():
        out(what="env_step", case=k, us_per_step=round(float(np.median(t)), 2), us_spread=[round(min(t), 2), round(max(t), 2)])

    # (b) K10 at Q = 64 with a route on every row, and without routes
    w = BatchedWorld(N, M, s.table)
    w.set_state(s.x, s.y, s.heading, s.speed, vx=s.vx, vy=s.vy, type_id=s.type_id)
    w.check_events()
    w.set_agents(None)
    type_id0 = w.type_id.clone()
    lo, hi = np.array([s.x.min(), s.y.min()]), np.array([s.x.max(), s.y.max()])
    rng = np.random.default_rng(0)
    w.set_paths([(lo + (hi - lo) * rng.uniform(0, 1, (64, 2))).astype(np.float32) for _ in range(16)])
    rid = rng.integers(0, 16, (N, M)).astype(np.int16)
    for case, bound in (("no_routes", False), ("route64", True)):
        w.set_routes(rid if bound else None, 5.0)

        def launch():
            w.type_id.copy_(type_id0)   # retired slots come back: every launch scores every row
            w.agents_epilogue()
        us, _ = time_graph(launch, args.seconds, per_graph=20)
        # flags, type ids (read, and the copy back) and the state x, y per slot; per row reward, status, terminated,
        # truncated, iou, max_iou / min_dist read + written; with routes route_id per slot and s_best read + written
        nbytes = N * M * (1 + 3 + 8) + N * M * (4 + 3 + 4 + 16) + N + (N * M * (2 + 16) if bound else 0)
        out(what="agent_rewards", case=case, Q=M, us_per_call=round(us, 2), algorithmic_bytes=nbytes,
            hbm_share=round(nbytes / (us * 1e-6) / PEAK_BYTES_PER_S, 4), note="includes a type_id copy of N*M bytes")

    # (c) K12 alone
    obs = torch.arange(M, dtype=torch.int16, device=w.device).expand(N, M).contiguous()
    for P in (8, 32):
        us, _ = time_graph(lambda: w.route_observe(P, 2.0, obs), args.seconds, per_graph=20)
        F = 5 + 2 * P
        nbytes = N * M * (2 + 1 + 2 + 12 + 4 * F)   # observer, type, route id, x / y / heading in; the row out
        out(what="route_observe", P=P, Q=M, us_per_call=round(us, 2), algorithmic_bytes=nbytes,
            hbm_share=round(nbytes / (us * 1e-6) / PEAK_BYTES_PER_S, 4))


if __name__ == "__main__":
    main()
