"""Time log replay (K7, ``BatchedWorld.set_log``) in the tick and print one JSON line.

World: C2-shaped, 4096 scenarios x 64 participants on the synthetic grid map (``synthetic.config2``'s map), slot 0 a
kinematic ego, slots 1..63 replaying a seeded synthetic recording (``synthetic.replay_episodes``: 20000 vehicle tracks of
40 ms frames, ticks of 100 ms, so every other tick interpolates).  Against it: the same world with those 63 slots as plain
static rows and no log bound (the state and types the replay gave them at t0: the tracks present then as static rows of their
class, the others empty).  A tick is timed with CUDA events over CUDA-graph replays for at least ``--seconds`` (the
two worlds alternate, twice each).  One graph replay is ``--ticks`` ticks followed by zeroing ``step_count`` (in both
worlds), so that every tick samples the first ``--ticks`` intervals of its episode and the recording stays in view however
long the timing runs.  K7's own duration comes from a separate ``torch.profiler`` run; its algorithmic bytes (per replayed
slot: row_track entry, track entry, the one or two frame records read, state + type written; absent tracks: the type
only) over that duration are set against the H100 SXM data sheet's 3.35 TB/s.
"""

from __future__ import annotations

import argparse
import json
import sys

import numpy as np

PEAK_BYTES_PER_S = 3.35e12


def _worlds(n, m, n_tracks, seed):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    ep = synthetic.replay_episodes(n, m, n_tracks, seed=seed)
    c2 = synthetic.config2(8, 8, seed=1)   # only its map
    pool = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in ep.pool.items()}
    out = []
    for replay in (True, False):
        w = BatchedWorld(n, m, ep.table, interval=100)
        w.set_map(c2.segments, c2.bounds)
        w.type_id.copy_(torch.from_numpy(ep.type_id).cuda())
        if replay:
            w.set_log(ep.log, ep.t0, ep.row_track)
        w.reset(torch.ones(n, dtype=torch.uint8, device="cuda"), pool)
        out.append(w)
    rep, plain = out
    torch.cuda.synchronize()
    # the comparison world: the replayed world's state and types at reset (the tracks present at t0 as static rows of their
    # class, the others empty slots), no log
    st = rep.state_numpy()
    plain.set_state(st["x"], st["y"], st["heading"], st["speed"], st["vx"], st["vy"], type_id=rep.type_id)
    return ep, rep, plain


def _graph(w, action, ticks):
    import torch

    def body():
        for _ in range(ticks):
            w.step(action)
        w.step_count.zero_()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            body()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        body()
    return g


def _time(g, ticks, seconds):
    import torch

    for _ in range(10):
        g.replay()
    b, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    b.record()
    for _ in range(20):
        g.replay()
    e.record()
    e.synchronize()
    per = b.elapsed_time(e) / 20 / 1e3
    reps = max(20, int(seconds / max(per, 1e-7)))
    b.record()
    for _ in range(reps):
        g.replay()
    e.record()
    e.synchronize()
    return b.elapsed_time(e) / reps / ticks * 1e3, reps * ticks


def _k7_bytes(ep, n, ticks, interval):
    """Algorithmic bytes of one K7 launch, averaged over the ``ticks`` sampling offsets a graph replay covers."""
    from oracle import replay as R

    rows = np.arange(n)
    bound = ep.row_track[rows] >= 0
    first = ep.log.first_ms.astype(np.int64)
    total = 0.0
    for step in range(ticks):
        _, pres, _, _ = R.sample(ep.log, ep.t0, ep.row_track, rows, np.full(n, step), interval, 1)
        k = np.maximum(ep.row_track[rows], 0)
        t = ep.t0[rows].astype(np.int64)[:, None] + (step + 1) * interval
        on_frame = ((t - first[k]) % ep.log.period_ms[k].astype(np.int64)) == 0
        rec = np.where(on_frame, 20, 40)
        per = np.where(pres, 4 + 16 + rec + 24 + 1 + 1, np.where(bound, 4 + 16 + 1, 0))   # (+1: the track's type row)
        total += float(per.sum())
    return total / ticks, int(bound.sum())


def _profile_k7(w, action, ticks):
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(4):
            for _ in range(ticks):
                w.step(action)
            w.step_count.zero_()
        torch.cuda.synchronize()
    durs = [e for e in prof.key_averages() if "t2d_replay_kernel" in e.key]
    if not durs:
        return None, 0
    e = durs[0]
    tot = getattr(e, "device_time_total", None)
    if tot is None:
        tot = e.cuda_time_total
    return tot / e.count, e.count   # microseconds per launch


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--m", type=int, default=64)
    ap.add_argument("--tracks", type=int, default=20000)
    ap.add_argument("--ticks", type=int, default=10)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args(argv)
    import torch
    from bench_bev import _gpu_info

    if not torch.cuda.is_available():
        sys.exit("bench_replay.py needs a CUDA device")
    gpu, power = _gpu_info()
    ep, rep, plain = _worlds(a.n, a.m, a.tracks, a.seed)
    from tactics2d_b200 import synthetic

    action = torch.from_numpy(synthetic.random_actions(0, (a.n, a.m))).cuda()
    graphs = {"replay": _graph(rep, action, a.ticks), "static": _graph(plain, action, a.ticks)}
    us = {"replay": [], "static": []}
    for _ in range(2):
        for name in ("replay", "static"):
            t, _ = _time(graphs[name], a.ticks, a.seconds)
            us[name].append(round(t, 3))
    k7_us, k7_launches = _profile_k7(rep, action, a.ticks)
    nbytes, n_bound = _k7_bytes(ep, a.n, a.ticks, 100)
    rate = None if not k7_us else nbytes / (k7_us * 1e-6)
    print(json.dumps(dict(
        metric="log_replay_tick", n=a.n, m=a.m, tracks=a.tracks, records=int(len(ep.log.records)), replayed_slots=n_bound,
        gpu=gpu, power_limit=power, ticks_per_graph=a.ticks, us_per_tick_replay=us["replay"], us_per_tick_static=us["static"],
        replay_overhead_us=round(min(us["replay"]) - min(us["static"]), 3),
        k7_us=None if k7_us is None else round(k7_us, 3), k7_profiled_launches=k7_launches,
        k7_bytes_per_launch=int(nbytes), k7_bytes_per_replayed_slot=round(nbytes / max(n_bound, 1), 1),
        k7_achieved_gb_s=None if rate is None else round(rate / 1e9, 1),
        k7_share_of_hbm_peak=None if rate is None else round(rate / PEAK_BYTES_PER_S, 3))), flush=True)
    rep.close(); plain.close()


if __name__ == "__main__":
    main()
