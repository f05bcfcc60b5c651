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
import sys
import time

import numpy as np

PEAK_BYTES_PER_S = 3.35e12
K_AGENTS, K_SEGMENTS, AGENT_RANGE, SEGMENT_RANGE = 16, 32, 50.0, 30.0


def _gpu_info():
    import subprocess

    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (v.strip() for v in out.split(","))
        return name, power
    except Exception:
        import torch

        return torch.cuda.get_device_name(0), "unknown"


def _world(scene):
    """(world, segments per scenario's tile, map table in use): C2 and C4 as ``bench.py`` builds them, C4's tile set through
    ``set_map_table``, and the C5 scene of ``bench.py`` at 8192 scenarios."""
    from tactics2d_b200 import BatchedWorld, synthetic
    from tactics2d_b200.map import load_collidable_segments

    if scene == "c2":
        s = synthetic.config2(4096, 64, seed=1)
    elif scene == "c4":
        seg, b = load_collidable_segments("inD_1")
        s = synthetic.config4(16384, 32, seed=4, segments=seg, bounds=b)
    else:
        seg, b = load_collidable_segments("rounD_0")
        s = synthetic.config5(8192, 128, seed=5, segments=seg, bounds=b)
    n, m = s.shape
    w = BatchedWorld(n, m, s.table)
    if scene == "c4":
        w.set_map_table([dict(segments=s.segments, bounds=s.bounds)], np.zeros(n, np.int64))
    else:
        w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    return w, len(s.segments), scene == "c4"


def _time_observe(w, seconds, call=None):
    import torch

    args = (K_AGENTS, K_SEGMENTS, AGENT_RANGE, SEGMENT_RANGE)
    if call is None:
        call = lambda: w.observe(*args)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for _ in range(3):
            call()
    torch.cuda.current_stream().wait_stream(st)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call()
    for _ in range(20):
        g.replay()
    torch.cuda.synchronize()
    b, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    b.record()
    for _ in range(50):
        g.replay()
    e.record()
    e.synchronize()
    reps = max(100, int(seconds / max(b.elapsed_time(e) / 50 / 1e3, 1e-7)))
    b.record()
    for _ in range(reps):
        g.replay()
    e.record()
    e.synchronize()
    return b.elapsed_time(e) / reps * 1e3, reps


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

    args = (K_AGENTS, K_SEGMENTS, AGENT_RANGE, SEGMENT_RANGE)
    for scene in a.scenes.split(","):
        w, n_seg, map_table = _world(scene)
        ego = torch.zeros((w.N, 1), dtype=torch.int16, device=w.device)
        k8_rd, k8_wr = _bytes(w, n_seg, map_table)
        for r in range(a.rounds):
            for kernel, q, call in (("k9", w.M, lambda: w.observe_agents(*args)), ("k8", 1, None),
                                    ("k9", 1, lambda: w.observe_agents(*args, observers=ego)), ("k8", 1, None)):
                us, reps = _time_observe(w, a.seconds, call)
                rd = k8_rd + (2 * w.N * q if call is not None and q == 1 else 0)   # the observer list
                wr = k8_wr * q
                print(json.dumps(dict(metric="observe_agents" if kernel == "k9" else "observe", kernel=kernel, scene=scene,
                                      round=r, n=w.N, m=w.M, q=q, segments_per_tile=n_seg, k_agents=K_AGENTS,
                                      k_segments=K_SEGMENTS, agent_range=AGENT_RANGE, segment_range=SEGMENT_RANGE, gpu=gpu,
                                      power_limit=power, us_per_call=round(us, 2), replays=reps, bytes_read=rd,
                                      bytes_written=wr, achieved_gb_s=round((rd + wr) / (us * 1e-6) / 1e9, 1),
                                      share_of_hbm=round((rd + wr) / (us * 1e-6) / PEAK_BYTES_PER_S, 3))), flush=True)
        w.close()


def _time_env(observation, steps, warmup):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    s = synthetic.config2(4096, 64, seed=1)
    env = BatchedTrafficEnv(s, max_step=200, observation=observation)
    env.reset()
    act = torch.zeros((4096, 2), device=env.world.device)
    for _ in range(warmup):
        env.step(act)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(steps):
        env.step(act)
    torch.cuda.synchronize()
    us = (time.perf_counter() - t) / steps * 1e6
    env.close()
    return us


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--scenes", default="c2,c4,round")
    ap.add_argument("--env-steps", type=int, default=2000)
    ap.add_argument("--env-rounds", type=int, default=3)
    ap.add_argument("--agents", action="store_true", help="time observe_agents (K9) against observe (K8) instead")
    ap.add_argument("--rounds", type=int, default=3, help="with --agents: alternating rounds per scene")
    a = ap.parse_args(argv)
    import torch

    if not torch.cuda.is_available():
        sys.exit("bench_obs.py needs a CUDA device")
    gpu, power = _gpu_info()
    if a.agents:
        _agents(a, gpu, power)
        return
    for scene in a.scenes.split(","):
        w, n_seg, map_table = _world(scene)
        us, reps = _time_observe(w, a.seconds)
        rd, wr = _bytes(w, n_seg, map_table)
        o = w.observe(K_AGENTS, K_SEGMENTS, AGENT_RANGE, SEGMENT_RANGE)
        rows_a = float((o.agent_index >= 0).sum(1).float().mean())
        rows_s = float((o.segment_index >= 0).sum(1).float().mean())
        print(json.dumps(dict(metric="observe", scene=scene, n=w.N, m=w.M, segments_per_tile=n_seg, k_agents=K_AGENTS,
                              k_segments=K_SEGMENTS, agent_range=AGENT_RANGE, segment_range=SEGMENT_RANGE, gpu=gpu,
                              power_limit=power, us_per_call=round(us, 2), replays=reps, bytes_read=rd, bytes_written=wr,
                              achieved_gb_s=round((rd + wr) / (us * 1e-6) / 1e9, 1),
                              share_of_hbm=round((rd + wr) / (us * 1e-6) / PEAK_BYTES_PER_S, 3),
                              mean_agent_rows=round(rows_a, 2), mean_segment_rows=round(rows_s, 2))), flush=True)
        w.close()
    for r in range(a.env_rounds):
        for observation in ("state", "vector"):
            us = _time_env(observation, a.env_steps, 50)
            print(json.dumps(dict(metric="env_step", scene="c2", observation=observation, round=r, gpu=gpu, power_limit=power,
                                  steps=a.env_steps, us_per_step=round(us, 2))), flush=True)


if __name__ == "__main__":
    main()
