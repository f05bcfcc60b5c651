"""Time the trajectory history (DESIGN.md section 1 "Trajectory history") at the C2 shape, 4096 scenarios x 64
participants; one JSON line per measurement.

(a) ``tick``: ``BatchedWorld.step`` without a history and with H = 8, 16 and 32 (the tick, then K15's append), the four
    worlds alternated in one run (``benchlib.alternate``); they start from the same scene and take the same actions, so
    they stay in step with each other.
(b) ``reset``: ``BatchedWorld.reset`` of every scenario without a history and with H = 16 (K2, then K15's restart), each
    in a CUDA graph (``benchlib.time_graph``).
(c) ``observe_history``: K16 alone in a CUDA graph, for the egos (K = 16 agents, H = 16) and for agents (Q = 64 rows per
    scenario, K = 8, H = 8), after H ticks so that every entry is valid.
(d) ``env_step``: ``BatchedTrafficEnv.step`` with ``observation="vector"`` without and with ``history=dict(length=16)``,
    alternated.

The algorithmic bytes are those a launch must move from and to HBM (``_bytes``), printed beside the time with their share
of the H100 SXM data sheet's 3.35 TB/s.  The GPU name and power limit are read in the same run and printed on every line.
"""

from __future__ import annotations

import argparse
import json

import numpy as np

from benchlib import PEAK_BYTES_PER_S, alternate, gpu_info, require_cuda, scene, time_graph


def _bytes(what, N, M, H=0, Q=0, K=0):
    """The HBM bytes of one launch: K15 reads the 25 B state of every slot and writes it into the ring, plus the count;
    K16 reads per row the observer's slot, K agent indices, per block the slot's type and H ring entries of 21 B (type
    and five fp32 values; speed is not read), and writes (1 + K) H 7 fp32."""
    if what == "append":
        return 2 * 25 * N * M + 16 * N
    if what == "observe":
        rows = N * max(Q, 1)
        return rows * (2 * (1 if Q else 0) + 13 + 2 * K + (1 + K) * (1 + 8 + H * 21) + (1 + K) * H * 7 * 4) + 8 * N
    raise ValueError(what)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="steps per alternation round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=0.5, help="length of one timed CUDA-graph window")
    args = ap.parse_args()
    require_cuda("bench_history.py")
    import torch

    from tactics2d_b200 import BatchedWorld
    from tactics2d_b200.envs import BatchedTrafficEnv

    name, power, _ = gpu_info()
    s = scene("c2")
    N, M = s.shape
    dev = torch.device("cuda:0")
    out = lambda **kw: print(json.dumps(dict(kw, N=N, M=M, gpu=name, power_limit=power)), flush=True)

    def world(H):
        w = BatchedWorld(N, M, s.table, device=dev)
        w.set_map(s.segments, s.bounds)
        w.set_state(s.x, s.y, s.heading, s.speed, vx=s.vx, vy=s.vy, type_id=s.type_id)
        if H:
            w.set_history(H)
        return w

    # (a) tick vs tick + append
    worlds = {H: world(H) for H in (0, 8, 16, 32)}
    act = torch.from_numpy(np.random.default_rng(0).uniform(-0.5, 0.5, (N, M, 2)).astype(np.float32)).to(dev)
    times = alternate({H: (lambda w=w: w.step(act)) for H, w in worlds.items()}, args.rounds, args.steps)
    base = float(np.median(times[0]))
    for H, t in times.items():
        med = float(np.median(t))
        out(what="tick", H=H, us_per_step=round(med, 2), us_spread=[round(min(t), 2), round(max(t), 2)],
            append_us=round(med - base, 2) if H else None, append_bytes=_bytes("append", N, M) if H else 0)

    # (b) the restart inside an all-scenario reset
    pool = {k: torch.from_numpy(np.ascontiguousarray(getattr(s, k), dtype=np.float32)).to(dev)
            for k in ("x", "y", "heading", "speed")}
    mask = torch.ones(N, dtype=torch.uint8, device=dev)
    for H in (0, 16):
        w = worlds[H]
        us, calls = time_graph(lambda w=w: w.reset(mask, pool), args.seconds)
        out(what="reset", H=H, us=round(us, 2), calls=calls)

    # (c) K16 for the egos and for agents, every entry valid
    for Q, K, H in ((0, 16, 16), (64, 8, 8)):
        w = worlds[16] if H == 16 else worlds[8]
        w.reset(mask, pool)
        for _ in range(H):
            w.step(act)
        if Q:
            obs = torch.arange(M, dtype=torch.int16, device=dev).expand(N, Q).contiguous()
            idx = w.observe_agents(K, 0, observers=obs).agent_index
            call = lambda w=w, idx=idx, obs=obs: w.observe_history(idx, obs)
        else:
            idx = w.observe(K, 0).agent_index
            call = lambda w=w, idx=idx: w.observe_history(idx)
        us, calls = time_graph(call, args.seconds, per_graph=20)
        nbytes = _bytes("observe", N, M, H, Q, K)
        valid = float(call()[..., 0].mean())
        out(what="observe_history", Q=Q, K=K, H=H, us_per_call=round(us, 2), algorithmic_bytes=nbytes,
            hbm_share=round(nbytes / (us * 1e-6) / PEAK_BYTES_PER_S, 4), valid_fraction=round(valid, 4))
    for w in worlds.values():
        w.close()

    # (d) the env step with and without a history
    vo = dict(k_agents=16, k_segments=0)
    envs = {"no_history": BatchedTrafficEnv(s, max_step=200, observation="vector", vector_obs=vo),
            "history16": BatchedTrafficEnv(s, max_step=200, observation="vector", vector_obs=vo, history=dict(length=16))}
    ego = torch.zeros((N, 2), dtype=torch.float32, device=dev)
    for e in envs.values():
        e.reset(seed=0)
    times = alternate({k: (lambda e=e: e.step(ego)) for k, e in envs.items()}, args.rounds, args.steps)
    for k, t in times.items():
        out(what="env_step", env=k, us_per_step=round(float(np.median(t)), 2), us_spread=[round(min(t), 2), round(max(t), 2)])
    for e in envs.values():
        e.close()


if __name__ == "__main__":
    main()
