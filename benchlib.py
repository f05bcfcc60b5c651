"""What the side benchmarks (``bench_*.py``) share: the card a number was measured on, the scenes, a CUDA-graph kernel timer
and an alternating wall-clock step loop.

Nothing here imports torch or the package at import time: ``bench_tick_phases.py`` points ``T2D_B200_LIB`` at another build
before the package binds the library.  Nothing here calls a library API either, so an A/B run against an older tree can copy
this file next to the scripts.
"""

from __future__ import annotations

import collections
import math
import subprocess
import time

PEAK_BYTES_PER_S = 3.35e12   # H100 SXM data sheet, HBM3
SCENE_SEEDS = {"c2": 1, "c4": 4, "c5": 5}
GpuInfo = collections.namedtuple("GpuInfo", "name power_limit nvidia_smi")


def gpu_info():
    """``GpuInfo`` of the first GPU: its name, power limit and the raw nvidia-smi line, which also holds the max SM clock.
    An absolute number is only worth something with the card it was measured on.  Without nvidia-smi: torch's device
    name, "unknown" and None."""
    try:
        raw = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, _ = (v.strip() for v in raw.split(","))
        return GpuInfo(name, power, raw)
    except Exception:
        import torch

        return GpuInfo(torch.cuda.get_device_name(0), "unknown", None)


def require_cuda(script):
    """Exit with a message when no CUDA device is visible: the side benchmarks measure on the GPU and nowhere else."""
    import torch

    if not torch.cuda.is_available():
        raise SystemExit(f"{script} measures on a CUDA device; none is visible")


def scene(name, n=None, m=None):
    """``bench.make_scene``'s scene ``name`` ("c2", "c4" or "c5") at the seed the side benchmarks use for it."""
    from bench import make_scene

    return make_scene(name, seed=SCENE_SEEDS[name], n=n, m=m)


def time_graph(call, seconds, per_graph=1):
    """(microseconds per ``call``, calls timed).  ``call`` is warmed up on a side stream, ``per_graph`` calls are captured in
    one CUDA graph, and the graph is replayed back to back between two CUDA events until one such window lasts at least
    ``seconds``; a shorter window only sizes the next.  The host waits on the device only between windows."""
    import torch

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            call()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(per_graph):
            call()
    for _ in range(5):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    replays = 5
    while True:
        e0.record()
        for _ in range(replays):
            g.replay()
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= seconds * 1e3:
            return ms * 1e3 / (replays * per_graph), replays * per_graph
        replays = math.ceil(replays * 1.1 * seconds * 1e3 / max(ms, 1e-3))   # 10 % over the estimate: one more window


def alternate(runs, rounds, steps, warmup=3):
    """{label: wall-clock microseconds per step, one entry per round} for ``runs``, a dict of label -> zero-argument step.
    Every step is warmed up ``warmup`` times; then each round runs ``steps`` steps of every label in turn, so that drift on
    a shared host hits all labels alike.  Each window ends in a synchronise: it holds the device's work, not its launch."""
    import torch

    for step in runs.values():
        for _ in range(warmup):
            step()
    torch.cuda.synchronize()
    times = {label: [] for label in runs}
    for _ in range(rounds):
        for label, step in runs.items():
            t0 = time.perf_counter()
            for _ in range(steps):
                step()
            torch.cuda.synchronize()
            times[label].append((time.perf_counter() - t0) * 1e6 / steps)
    return times
