"""Time the BEV observation kernel (K6, ``BatchedWorld.bev``) and print one JSON line per configuration.

Scenes: C2 (4096 scenarios x 64 participants on the synthetic grid map, ``synthetic.config2``) and the same
participants moved onto the inD_1 map through ``set_map_table`` (its Areas and road border, per-segment styles).  Each
renders 200 x 200 images, as RGB (the reference's observation) and as style indices.  A call is timed with CUDA events
over CUDA-graph replays of one render each, for at least ``--seconds`` after warm-up; the output holds the GPU name and
power limit, microseconds per call, bytes written per call, the achieved store rate and its share of the H100 SXM data
sheet's 3.35 TB/s HBM3 bandwidth (the kernel reads little: its lower bound is the image stores).

``--agents`` times the per-agent view (``BatchedWorld.bev_agents``) instead, on the same scenes: ``--q`` observer rows per
scenario, slots 0 .. q-1, one 200 x 200 image each.
"""

from __future__ import annotations

import argparse
import json

import numpy as np

from benchlib import PEAK_BYTES_PER_S, gpu_info, require_cuda, scene, time_graph


def _world(scene_name, n, m):
    from tactics2d_b200 import BatchedWorld

    s = scene("c2", n=n, m=m)
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


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--m", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--scenes", default="c2,inD_1")
    ap.add_argument("--agents", action="store_true", help="time bev_agents (one image per observer row) instead of bev")
    ap.add_argument("--q", type=int, default=8, help="observer rows per scenario with --agents")
    a = ap.parse_args(argv)
    require_cuda("bench_bev.py")
    gpu, power, _ = gpu_info()
    for key in a.scenes.split(","):
        w = _world(key, a.n, a.m)
        if a.agents:
            _bench_agents(w, key, a, gpu, power)
            w.close()
            continue
        for rgb in (True, False):
            nbytes = w.bev((200, 200), rgb=rgb).numel()
            us, reps = time_graph(lambda: w.bev((200, 200), rgb=rgb), a.seconds)
            rate = nbytes / (us * 1e-6)
            print(json.dumps(dict(metric="bev_render", scene=key, n=a.n, m=a.m, resolution=[200, 200],
                                  output="rgb" if rgb else "class", gpu=gpu, power_limit=power, us_per_call=round(us, 2),
                                  replays=reps, bytes_per_call=nbytes, achieved_gb_s=round(rate / 1e9, 1),
                                  share_of_store_bound=round(rate / PEAK_BYTES_PER_S, 3))), flush=True)
        w.close()


def _bench_agents(w, key, a, gpu, power):
    import torch

    obs = torch.arange(a.q, dtype=torch.int16, device=w.device).expand(a.n, a.q).contiguous()
    for rgb in (True, False):
        nbytes = w.bev_agents((200, 200), 20.0, rgb=rgb, observers=obs).numel()
        us, reps = time_graph(lambda: w.bev_agents((200, 200), 20.0, rgb=rgb, observers=obs), a.seconds)
        rate = nbytes / (us * 1e-6)
        print(json.dumps(dict(metric="bev_render_agents", scene=key, n=a.n, m=a.m, q=a.q, resolution=[200, 200],
                              output="rgb" if rgb else "class", gpu=gpu, power_limit=power, us_per_call=round(us, 2),
                              us_per_row=round(us / a.q, 2), replays=reps, bytes_per_call=nbytes,
                              achieved_gb_s=round(rate / 1e9, 1), share_of_store_bound=round(rate / PEAK_BYTES_PER_S, 3))),
              flush=True)
        w._agent_bev.clear()   # the next output's buffer is allocated afresh


if __name__ == "__main__":
    main()
