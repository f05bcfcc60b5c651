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

``--schedule`` times slot schedules instead (``BatchedWorld.set_log(..., schedule=...)``, metric ``log_replay_schedule_tick``):
the same 4096 x 64 shape on ``synthetic.highway_episodes`` (a highway-like recording, 100 s episode windows, every slot
replaying the tracks of its schedule one after the other), 100 ms ticks, and each scenario's ``step_count`` held at its own
random point of the episode (a graph replay restores those counts instead of zeroing them), so that slots switch tracks
inside the timed window.  K7's bytes then also count the slot's offset, ceil(log2 L) 8-byte probes of its L entries, the
entry taken and the ``replay_track`` store.
"""

from __future__ import annotations

import argparse
import json

import numpy as np

from benchlib import PEAK_BYTES_PER_S, gpu_info, require_cuda, scene, time_graph


def _worlds(n, m, n_tracks, seed):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    ep = synthetic.replay_episodes(n, m, n_tracks, seed=seed)
    c2 = scene("c2", n=8, m=8)   # only its map
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


def _ticks(w, action, ticks, start=None):
    """``ticks`` ticks, then every scenario back to its first step (``start`` None) or to ``start``: one graph replay."""
    for _ in range(ticks):
        w.step(action)
    if start is None:
        w.step_count.zero_()
    else:
        w.step_count.copy_(start)


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


def _profile_k7(w, action, ticks, start=None):
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(4):
            _ticks(w, action, ticks, start)
        torch.cuda.synchronize()
    durs = [e for e in prof.key_averages() if "t2d_replay_kernel" in e.key]
    if not durs:
        return None, 0
    e = durs[0]
    tot = getattr(e, "device_time_total", None)
    if tot is None:
        tot = e.cuda_time_total
    return tot / e.count, e.count   # microseconds per launch


def _schedule_worlds(n, m, seed):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    ep = synthetic.highway_episodes(n, m, seed=seed, duration_ms=200000, horizon_ms=100000)
    pool = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in ep.pool.items()}
    start = torch.from_numpy(np.random.default_rng(seed).integers(0, 990, n).astype(np.int32)).cuda()
    out = []
    for replay in (True, False):
        w = BatchedWorld(n, m, ep.table, interval=100)
        w.set_map(*_highway_map())
        w.type_id.copy_(torch.from_numpy(ep.type_id).cuda())
        if replay:
            w.set_log(ep.log, ep.t0, schedule=ep.schedule)
        w.reset(torch.ones(n, dtype=torch.uint8, device="cuda"), pool)
        out.append(w)
    rep, plain = out
    for _ in range(2):   # the replayed slots at each scenario's starting point
        rep.step_count.copy_(start)
        rep.step(torch.zeros((n, m, 2), device="cuda"))
    rep.step_count.copy_(start)
    plain.step_count.copy_(start)
    torch.cuda.synchronize()
    st = rep.state_numpy()
    plain.set_state(st["x"], st["y"], st["heading"], st["speed"], st["vx"], st["vy"], type_id=rep.type_id)
    return ep, rep, plain, start


def _highway_map():
    """The two carriageways' outer edges of ``synthetic.highway_log`` (3 lanes of 3.75 m each side) over its 420 m."""
    seg = np.asarray([[0.0, -11.25, 420.0, -11.25], [0.0, 11.25, 420.0, 11.25]], np.float32)
    return seg, (-20.0, 440.0, -20.0, 20.0)


def _k7_schedule_bytes(ep, start, ticks, interval):
    """Algorithmic bytes of one scheduled K7 launch, averaged over the ``ticks`` launches a graph replay makes, and the
    (scenario, slot) track switches within those ticks."""
    from tests import schedule_oracle as S

    n, m = ep.type_id.shape
    rows = np.arange(n)
    off, _ = ep.schedule
    L = np.diff(off.astype(np.int64)).reshape(n, m)
    probes = np.where(L > 1, np.ceil(np.log2(np.maximum(L, 1))), 0)
    first = ep.log.first_ms.astype(np.int64)
    total, prev, switches = 0.0, None, 0
    for step in range(ticks):
        _, pres, _, _, trk = S.sample(ep.log, ep.t0, *ep.schedule, rows, start + step, interval, 1)
        k = np.maximum(trk, 0)
        t = ep.t0.astype(np.int64)[:, None] + (start[:, None] + step + 1) * interval
        rec = np.where(((t - first[k]) % ep.log.period_ms[k].astype(np.int64)) == 0, 20, 40)
        sched = L > 0
        per = 4 + 4 + np.where(sched, 8 * probes + 8 + 16, 0) + np.where(pres, 1 + rec + 24 + 1, np.where(sched, 1, 0))
        total += float(per.sum())
        if prev is not None:
            switches += int(((trk >= 0) & (prev >= 0) & (trk != prev)).sum())
        prev = trk
    return total / ticks, int((L > 0).sum()), switches, float(L[L > 0].mean()), int(L.max())


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--m", type=int, default=64)
    ap.add_argument("--tracks", type=int, default=20000)
    ap.add_argument("--ticks", type=int, default=10)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--schedule", action="store_true", help="time slot schedules on a highway-like recording instead")
    a = ap.parse_args(argv)
    require_cuda("bench_replay.py")
    import torch
    from tactics2d_b200 import synthetic

    gpu, power, _ = gpu_info()
    if a.schedule:
        ep, rep, plain, start = _schedule_worlds(a.n, a.m, a.seed)
    else:
        (ep, rep, plain), start = _worlds(a.n, a.m, a.tracks, a.seed), None
    action = torch.from_numpy(synthetic.random_actions(0, (a.n, a.m))).cuda()
    us = {"replay": [], "static": []}
    for _ in range(2):
        for name, w in (("replay", rep), ("static", plain)):
            t, _ = time_graph(lambda: _ticks(w, action, a.ticks, start), a.seconds)
            us[name].append(round(t / a.ticks, 3))
    k7_us, k7_launches = _profile_k7(rep, action, a.ticks, start)
    if a.schedule:
        nbytes, n_rows, switches, mean_l, max_l = _k7_schedule_bytes(ep, start.cpu().numpy().astype(np.int64), a.ticks, 100)
        head = dict(metric="log_replay_schedule_tick", n=a.n, m=a.m, tracks=int(len(ep.log)), records=int(len(ep.log.records)),
                    scheduled_slots=n_rows, entries=int(len(ep.schedule[1])), mean_entries_per_slot=round(mean_l, 2),
                    max_entries_per_slot=max_l, dropped=int(ep.dropped.sum()), switches_per_graph=switches)
        per_slot = "k7_bytes_per_scheduled_slot"
    else:
        nbytes, n_rows = _k7_bytes(ep, a.n, a.ticks, 100)
        head = dict(metric="log_replay_tick", n=a.n, m=a.m, tracks=a.tracks, records=int(len(ep.log.records)),
                    replayed_slots=n_rows)
        per_slot = "k7_bytes_per_replayed_slot"
    rate = None if not k7_us else nbytes / (k7_us * 1e-6)
    print(json.dumps(dict(
        **head, gpu=gpu, power_limit=power, ticks_per_graph=a.ticks, us_per_tick_replay=us["replay"],
        us_per_tick_static=us["static"], replay_overhead_us=round(min(us["replay"]) - min(us["static"]), 3),
        k7_us=None if k7_us is None else round(k7_us, 3), k7_profiled_launches=k7_launches,
        k7_bytes_per_launch=int(nbytes), **{per_slot: round(nbytes / max(n_rows, 1), 1)},
        k7_achieved_gb_s=None if rate is None else round(rate / 1e9, 1),
        k7_share_of_hbm_peak=None if rate is None else round(rate / PEAK_BYTES_PER_S, 3))), flush=True)
    rep.close(); plain.close()


if __name__ == "__main__":
    main()
