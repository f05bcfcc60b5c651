"""Time the BEV observation kernel (K6, ``BatchedWorld.bev``) and print one JSON line per configuration.

Scenes: C2 (4096 scenarios x 64 participants on the synthetic grid map, ``synthetic.config2``) and the same
participants moved onto the inD_1 map through ``set_map_table`` (its Areas and road border, per-segment styles).  Each
renders 200 x 200 images, as RGB (the reference's observation) and as style indices.  A call is timed with CUDA events
over CUDA-graph replays of one render each, for at least ``--seconds`` after warm-up; the output holds the GPU name and
power limit, microseconds per call, bytes written per call, the achieved store rate and its share of the H100 SXM data
sheet's 3.35 TB/s HBM3 bandwidth (the kernel reads little: its lower bound is the image stores).
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys

import numpy as np

PEAK_BYTES_PER_S = 3.35e12


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (v.strip() for v in out.split(","))
        return name, power
    except Exception:
        import torch

        return torch.cuda.get_device_name(0), "unknown"


def _world(scene_name, n, m):
    from tactics2d_b200 import BatchedWorld, synthetic

    s = synthetic.config2(n, m, seed=1)
    w = BatchedWorld(n, m, s.table)
    x, y = s.x, s.y
    if scene_name == "c2":
        w.set_map(s.segments, s.bounds)
    else:
        from tactics2d_b200.map import load_areas, polygons_to_segments, segment_style_keys

        areas = load_areas("inD_1")
        xy = np.concatenate([a.outer for a in areas])
        b = (float(xy[:, 0].min()), float(xy[:, 0].max()), float(xy[:, 1].min()), float(xy[:, 1].max()))
        seg, ps = polygons_to_segments(areas)
        w.set_map_table([dict(segments=seg, poly_start=ps, bounds=b, style=segment_style_keys(areas))], np.zeros(n, np.int64))
        # the C2 arena (200 m square) scaled onto the map's box
        x = (b[0] + (x - x.min()) / max(np.ptp(x), 1e-6) * (b[1] - b[0])).astype(np.float32)
        y = (b[2] + (y - y.min()) / max(np.ptp(y), 1e-6) * (b[3] - b[2])).astype(np.float32)
    w.set_state(x, y, s.heading, s.speed, type_id=s.type_id)
    return w


def _time(w, res, rgb, seconds):
    import torch

    out = w.bev(res, rgb=rgb)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            w.bev(res, rgb=rgb)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        w.bev(res, rgb=rgb)
    for _ in range(10):
        g.replay()
    torch.cuda.synchronize()
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
    return b.elapsed_time(e) / reps * 1e3, reps, out.numel()


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--m", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--scenes", default="c2,inD_1")
    a = ap.parse_args(argv)
    import torch

    if not torch.cuda.is_available():
        sys.exit("bench_bev.py needs a CUDA device")
    gpu, power = _gpu_info()
    for scene in a.scenes.split(","):
        w = _world(scene, a.n, a.m)
        for rgb in (True, False):
            us, reps, nbytes = _time(w, (200, 200), rgb, a.seconds)
            rate = nbytes / (us * 1e-6)
            print(json.dumps(dict(metric="bev_render", scene=scene, n=a.n, m=a.m, resolution=[200, 200],
                                  output="rgb" if rgb else "class", gpu=gpu, power_limit=power, us_per_call=round(us, 2),
                                  replays=reps, bytes_per_call=nbytes, achieved_gb_s=round(rate / 1e9, 1),
                                  share_of_store_bound=round(rate / PEAK_BYTES_PER_S, 3))), flush=True)
        w.close()


if __name__ == "__main__":
    main()
