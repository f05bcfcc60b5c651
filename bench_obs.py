"""Time the vector observation kernel (K8, ``BatchedWorld.observe``) and ``BatchedTrafficEnv.step`` with it; one JSON line
per measurement.

Scenes: C2 (4096 scenarios x 64 participants on the synthetic grid map), C4 (16384 x 32 mixed traffic on the inD_1 tile,
set through ``set_map_table``) and 8192 x 128 vehicles on rounD_0 (the C5 scene), all as ``bench.py`` builds them; 16
agent rows and 32 segment rows within 50 m / 30 m.  A call is timed with CUDA events over CUDA-graph replays of one observe each, for at least
``--seconds`` after warm-up.  Each line holds the GPU name and power limit, microseconds per call, the call's algorithmic
bytes (the state of every slot, the tile ids, the segments of each scenario's tile, the row and indices written) and their
share of the H100 SXM data sheet's 3.35 TB/s.  Then ``BatchedTrafficEnv.step`` at C2 with ``observation="state"`` and
``"vector"``, alternating, in wall-clock microseconds per step (the env's step ends in host work, not in a graph).

``--agents`` times the per-agent observation instead (K9, ``BatchedWorld.observe_agents``) on the same three scenes: every
slot observing (Q = M) and the ego alone (Q = 1, observer 0), each alternated with K8's ``observe`` on the same world for
``--rounds`` rounds; its bytes add the rows and indices of every observer (the state, tile ids and segments are counted once
per scenario, as for K8).
"""

from __future__ import annotations

import argparse
import json

import numpy as np

from benchlib import PEAK_BYTES_PER_S, alternate, gpu_info, require_cuda, scene, time_graph

K_AGENTS, K_SEGMENTS, AGENT_RANGE, SEGMENT_RANGE = 16, 32, 50.0, 30.0
OBS_ARGS = (K_AGENTS, K_SEGMENTS, AGENT_RANGE, SEGMENT_RANGE)


def _world(key):
    """(world, segments per scenario's tile, map table in use): C2 and C4 as ``bench.py`` builds them, C4's tile set through
    ``set_map_table``, and the C5 scene of ``bench.py`` at 8192 scenarios."""
    from tactics2d_b200 import BatchedWorld

    s = scene("c5", n=8192) if key == "round" else scene(key)
    n, m = s.shape
    w = BatchedWorld(n, m, s.table)
    if key == "c4":
        w.set_map_table([dict(segments=s.segments, bounds=s.bounds)], np.zeros(n, np.int64))
    else:
        w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    return w, len(s.segments), key == "c4"


def _bytes(w, n_seg, map_table):
    """Algorithmic bytes of one call: x, y, heading, speed, vx, vy + type of every slot (21 B), the step counter, the tile
    id, the tile's segments (16 B each) for every scenario, and the row + the two index arrays written."""
    F = 16 + 11 * K_AGENTS + 9 * K_SEGMENTS
    read = w.N * (w.M * 21 + 4 + (2 if map_table else 0) + 16 * n_seg)
    write = w.N * (4 * F + 2 * (K_AGENTS + K_SEGMENTS))
    return read, write


def _agents(a, gpu, power):
    """K9 with every slot and with observer 0 alone, each alternated with K8 on the same world."""
    import torch

    for key in a.scenes.split(","):
        w, n_seg, map_table = _world(key)
        ego = torch.zeros((w.N, 1), dtype=torch.int16, device=w.device)
        k8_rd, k8_wr = _bytes(w, n_seg, map_table)
        k8 = lambda: w.observe(*OBS_ARGS)
        for r in range(a.rounds):
            for kernel, q, call in (("k9", w.M, lambda: w.observe_agents(*OBS_ARGS)), ("k8", 1, k8),
                                    ("k9", 1, lambda: w.observe_agents(*OBS_ARGS, observers=ego)), ("k8", 1, k8)):
                us, reps = time_graph(call, a.seconds)
                rd = k8_rd + (2 * w.N * q if kernel == "k9" and q == 1 else 0)   # the observer list
                wr = k8_wr * q
                print(json.dumps(dict(metric="observe_agents" if kernel == "k9" else "observe", kernel=kernel, scene=key,
                                      round=r, n=w.N, m=w.M, q=q, segments_per_tile=n_seg, k_agents=K_AGENTS,
                                      k_segments=K_SEGMENTS, agent_range=AGENT_RANGE, segment_range=SEGMENT_RANGE, gpu=gpu,
                                      power_limit=power, us_per_call=round(us, 2), replays=reps, bytes_read=rd,
                                      bytes_written=wr, achieved_gb_s=round((rd + wr) / (us * 1e-6) / 1e9, 1),
                                      share_of_hbm=round((rd + wr) / (us * 1e-6) / PEAK_BYTES_PER_S, 3))), flush=True)
        w.close()


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--scenes", default="c2,c4,round")
    ap.add_argument("--env-steps", type=int, default=2000)
    ap.add_argument("--env-rounds", type=int, default=3)
    ap.add_argument("--agents", action="store_true", help="time observe_agents (K9) against observe (K8) instead")
    ap.add_argument("--rounds", type=int, default=3, help="with --agents: alternating rounds per scene")
    a = ap.parse_args(argv)
    require_cuda("bench_obs.py")
    gpu, power, _ = gpu_info()
    if a.agents:
        _agents(a, gpu, power)
        return
    for key in a.scenes.split(","):
        w, n_seg, map_table = _world(key)
        us, reps = time_graph(lambda: w.observe(*OBS_ARGS), a.seconds)
        rd, wr = _bytes(w, n_seg, map_table)
        o = w.observe(*OBS_ARGS)
        rows_a = float((o.agent_index >= 0).sum(1).float().mean())
        rows_s = float((o.segment_index >= 0).sum(1).float().mean())
        print(json.dumps(dict(metric="observe", scene=key, n=w.N, m=w.M, segments_per_tile=n_seg, k_agents=K_AGENTS,
                              k_segments=K_SEGMENTS, agent_range=AGENT_RANGE, segment_range=SEGMENT_RANGE, gpu=gpu,
                              power_limit=power, us_per_call=round(us, 2), replays=reps, bytes_read=rd, bytes_written=wr,
                              achieved_gb_s=round((rd + wr) / (us * 1e-6) / 1e9, 1),
                              share_of_hbm=round((rd + wr) / (us * 1e-6) / PEAK_BYTES_PER_S, 3),
                              mean_agent_rows=round(rows_a, 2), mean_segment_rows=round(rows_s, 2))), flush=True)
        w.close()
    if a.env_rounds == 0:
        return
    import torch
    from tactics2d_b200.envs import BatchedTrafficEnv

    s = scene("c2")
    envs = {observation: BatchedTrafficEnv(s, max_step=200, observation=observation) for observation in ("state", "vector")}
    for env in envs.values():
        env.reset()
    act = torch.zeros((s.shape[0], 2), device="cuda:0")
    times = alternate({k: (lambda env=env: env.step(act)) for k, env in envs.items()}, a.env_rounds, a.env_steps, warmup=50)
    for env in envs.values():
        env.close()
    for r in range(a.env_rounds):
        for observation, us in times.items():
            print(json.dumps(dict(metric="env_step", scene="c2", observation=observation, round=r, gpu=gpu, power_limit=power,
                                  steps=a.env_steps, us_per_step=round(us[r], 2))), flush=True)


if __name__ == "__main__":
    main()
