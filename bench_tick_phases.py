#!/usr/bin/env python
"""bench_tick_phases.py - where one tick's time goes, phase by phase, at C2 (4096 x 64, kinematics, grid map).

    python bench_tick_phases.py [--ticks K] [--warmup W] [--lib PATH] [--cohorts C] [--restore-every R]

Compiles `t2d_kernels.cu` with -DT2D_TICK_TIMELINE into a temporary directory (or takes a library built that way from
--lib) and loads it in place of the in-tree build.  In that build lane 0 of every warp of the tick records %globaltimer
and %clock64 at nine points of its first tile: entry, after griddepcontrol.wait, loads consumed, physics done, sort
done, sweep done, drain done, static done, exit.  Two worlds hold the same C2 scene: one runs the tick's C2-shaped
instance, the other is kept on the generic instance (T2D_TICK_GENERIC=1 at its creation).  They tick in alternation,
each tick on its own with the L2 flushed before it, and after each tick the timeline is read back.  Before every R-th
tick both worlds are restored to the configured scene, as bench.py restores its replicas every 8 ticks: the C2-shaped
instance starts its x sort from the order the previous tick left (the order hint), so after a restore that order is
stale and most warps fall back to the sort network.

Printed, one JSON line per instance: per phase the median and p99 over all warps and ticks of its duration in SM
cycles and in ns (cycles converted at the clock measured over the warps' lifetimes), the spread of the warps' entry,
post-wait and loads-consumed times relative to the first warp of the tick, the median warp lifetime and the median
tick span (first entry to last exit).  Then the same once per cohort: the warps of every CTA split into C equal groups
by their index in the CTA (default 2: the C2-shaped instance's cohorts A and B, which issue their first loads one after
the other), with times still taken from the tick's first entry.  Last, the C2-shaped instance once per sort path: its
ticks where most warps kept the repaired order ("hint") and those where most fell back ("network"), by
t2d_tick_order_fallback_count, each also per cohort.  The timeline build is a measurement build: the
recording itself costs time, so its spans are longer than the shipped tick's.  Nothing is written to the tree.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from benchlib import gpu_info  # noqa: E402

POINTS = ["entry", "wait", "loads", "physics", "sort", "sweep", "drain", "static", "exit"]
TL_MAX_WARPS = 4096   # t2d_tick.cuh: TL_MAX_WARPS, TL_POINTS
WPC = 8               # warps per CTA of the tick at C2 (2048 warp tiles: pick_wpc's largest CTA); a warp's slot is its tile


def build_timeline_lib(out_dir):
    import __graft_entry__ as entry

    src = os.path.join(ROOT, "tactics2d_b200", "csrc", "t2d_kernels.cu")
    out = os.path.join(out_dir, "libt2d_b200_timeline.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc] + entry.NVCC_FLAGS + ["-DT2D_TICK_TIMELINE", "-o", out, src])
    return out


def summarise(records, sel=None):
    """records: list of [warps, points, 2] arrays (globaltimer ns, clock64) of one tick each; sel: a boolean mask over
    the warp slots to summarise (None: all).  Times relative to the tick's start are taken from all its warps."""
    durs, starts, waits, loads, life_ns, spans = [], [], [], [], [], []
    cyc_total = ns_total = 0
    for r in records:
        ok = (r[:, :, 0] != 0).all(axis=1)
        t0 = r[ok, 0, 0].astype(np.int64).min()
        if sel is not None:
            ok &= sel
        g = r[ok, :, 0].astype(np.int64)
        c = r[ok, :, 1].astype(np.int64)
        durs.append(np.diff(c, axis=1))
        starts.append(g[:, 0] - t0)
        waits.append(g[:, 1] - t0)
        loads.append(g[:, 2] - t0)
        life_ns.append(g[:, -1] - g[:, 0])
        spans.append(int(g[:, -1].max() - t0))
        cyc_total += int((c[:, -1] - c[:, 0]).sum())
        ns_total += int((g[:, -1] - g[:, 0]).sum())
    d = np.concatenate(durs)
    ghz = cyc_total / ns_total
    phases = {}
    for k in range(len(POINTS) - 1):
        col = d[:, k]
        phases[f"{POINTS[k]}->{POINTS[k + 1]}"] = {
            "median_cycles": float(np.median(col)), "p99_cycles": float(np.percentile(col, 99)),
            "median_ns": float(np.median(col) / ghz), "p99_ns": float(np.percentile(col, 99) / ghz)}
    dist = lambda a: {"median": float(np.median(a)), "p99": float(np.percentile(a, 99)), "max": float(a.max())}
    return {"warps_per_tick": int(d.shape[0] // len(records)), "ticks": len(records), "sm_clock_ghz": round(ghz, 4),
            "phases": phases,
            "entry_spread_ns": dist(np.concatenate(starts)),
            "wait_done_ns": dist(np.concatenate(waits)),
            "loads_done_ns": dist(np.concatenate(loads)),
            "warp_life_ns_median": float(np.median(np.concatenate(life_ns))),
            "tick_span_ns_median": float(np.median(spans))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=50, help="timed ticks per instance")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--lib", default=None, help="a library built with -DT2D_TICK_TIMELINE (default: build one in a temp dir)")
    ap.add_argument("--cohorts", type=int, default=2, help="also summarise the warps of each CTA in this many equal groups")
    ap.add_argument("--restore-every", type=int, default=8, help="restore the configured scene before every R-th tick (0: never)")
    args = ap.parse_args()

    tmp = tempfile.mkdtemp(prefix="t2d_timeline_")
    os.environ["T2D_B200_LIB"] = args.lib or build_timeline_lib(tmp)   # before the package binds the library

    import torch

    from bench import make_scene
    from tactics2d_b200 import BatchedWorld, _lib, synthetic

    lib = _lib.load()
    if not hasattr(lib, "t2d_tick_timeline"):
        raise SystemExit(f"{_lib.LIB_PATH} was not built with -DT2D_TICK_TIMELINE")
    read = lib.t2d_tick_timeline
    read.restype, read.argtypes = C.c_int, [C.c_void_p, C.c_int64, C.c_int]
    buf = np.zeros((TL_MAX_WARPS, len(POINTS), 2), dtype=np.uint64)

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    scene = make_scene("c2", seed=1)
    n, m = scene.shape
    worlds = {}
    for name, generic in (("fixed", False), ("generic", True)):
        if generic:
            os.environ["T2D_TICK_GENERIC"] = "1"
        try:
            w = BatchedWorld(n, m, scene.table, device=device, max_step=0)
        finally:
            os.environ.pop("T2D_TICK_GENERIC", None)
        w.set_map(scene.segments, scene.bounds)
        w.set_state(scene.x, scene.y, scene.heading, scene.speed, vx=scene.vx, vy=scene.vy, type_id=scene.type_id)
        worlds[name] = w
    flush = torch.empty(2 * torch.cuda.get_device_properties(device).L2_cache_size // 4, dtype=torch.float32, device=device)

    pools = {name: {k: getattr(w, k).clone() for k in ("x", "y", "heading", "speed", "vx", "vy")} for name, w in worlds.items()}
    ones = torch.ones(n, dtype=torch.uint8, device=device)
    records = {k: [] for k in worlds}
    network = []   # per timed tick of the C2-shaped instance: did most of its warps fall back to the sort network?
    fixed0 = lib.t2d_tick_fixed_count()
    _lib.check(read(buf.ctypes.data, buf.nbytes, 1))
    for t in range(args.warmup + args.ticks):
        if args.restore_every and t % args.restore_every == 0:
            for name, w in worlds.items():
                w.reset(ones, pools[name])
        act = torch.from_numpy(synthetic.random_actions(7000 + t, (n, m))).to(device)
        for name, w in worlds.items():
            flush.zero_()
            torch.cuda.synchronize()
            f0 = lib.t2d_tick_order_fallback_count()
            w.step(act)
            torch.cuda.synchronize()
            fell = lib.t2d_tick_order_fallback_count() - f0
            _lib.check(read(buf.ctypes.data, buf.nbytes, 1))
            if t >= args.warmup:
                records[name].append(buf.copy())
                if name == "fixed":
                    network.append(2 * fell > (n + 1) // 2)
    n_fixed = lib.t2d_tick_fixed_count() - fixed0
    if n_fixed != args.warmup + args.ticks:
        raise SystemExit(f"the C2-shaped instance ran {n_fixed} times, expected {args.warmup + args.ticks}")

    print(json.dumps({"gpu": torch.cuda.get_device_properties(device).name, "nvidia_smi": gpu_info().nvidia_smi,
                      "scene": scene.name, "N": n, "M": m}), flush=True)
    slot = np.arange(TL_MAX_WARPS) % WPC
    for name in worlds:
        print(json.dumps({"instance": name, **summarise(records[name])}), flush=True)
        for k in range(args.cohorts):
            sel = slot * args.cohorts // WPC == k
            print(json.dumps({"instance": name, "cohort": k, "warps": f"{k * WPC // args.cohorts}-{(k + 1) * WPC // args.cohorts - 1}",
                              **summarise(records[name], sel)}), flush=True)
    for path, sel_ticks in (("hint", [not f for f in network]), ("network", network)):
        recs = [r for r, keep in zip(records["fixed"], sel_ticks) if keep]
        if not recs:
            continue
        print(json.dumps({"instance": "fixed", "sort_path": path, **summarise(recs)}), flush=True)
        for k in range(args.cohorts):
            sel = slot * args.cohorts // WPC == k
            print(json.dumps({"instance": "fixed", "sort_path": path, "cohort": k,
                              "warps": f"{k * WPC // args.cohorts}-{(k + 1) * WPC // args.cohorts - 1}", **summarise(recs, sel)}), flush=True)
    for w in worlds.values():
        w.close()


if __name__ == "__main__":
    main()
