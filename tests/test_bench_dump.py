"""bench.py --dump-outputs: the host side of the dump (size bound, seeded sample of whole scenarios) on stand-in CPU tensors."""

import os
import sys
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402

STATE = ("x", "y", "heading", "speed", "vx", "vy")
RESULT = ("flags", "hit_index", "hit_segment", "status", "done")


def _stand_in(n, m):
    """World + StepResult shaped like BatchedWorld's, every value naming its scenario (no memory per element: expanded views)."""
    import torch

    scn = torch.arange(n, dtype=torch.float32)
    world = SimpleNamespace(N=n, M=m, **{k: scn[:, None].expand(n, m) for k in STATE})
    result = SimpleNamespace(flags=(scn % 7).to(torch.uint8)[:, None].expand(n, m),
                             hit_index=(scn % 1000).to(torch.int16)[:, None].expand(n, m),
                             hit_segment=(scn % 999).to(torch.int16)[:, None].expand(n, m),
                             status=(scn % 5).to(torch.uint8), done=(scn % 2).to(torch.uint8))
    return world, result


def _files(d):
    return {f: np.load(os.path.join(d, f)) for f in sorted(os.listdir(d))}


def test_small_output_is_written_whole(tmp_path):
    world, result = _stand_in(64, 8)
    bench.dump_outputs(str(tmp_path), world, result)
    got = _files(tmp_path)
    assert sorted(got) == sorted(k + ".npy" for k in STATE + RESULT)
    assert all(a.dtype == np.float32 for a in got.values())
    assert np.array_equal(got["x.npy"][:, 0], np.arange(64)) and got["x.npy"].shape == (64, 8)
    assert np.array_equal(got["hit_index.npy"][:, 3], np.arange(64) % 1000)


def test_c5_sized_output_is_a_seeded_sample_within_64_mib(tmp_path):
    n, m = 65536, 128
    world, result = _stand_in(n, m)
    a, b = tmp_path / "a", tmp_path / "b"
    bench.dump_outputs(str(a), world, result)
    bench.dump_outputs(str(b), world, result)
    assert sum(os.path.getsize(a / f) for f in os.listdir(a)) <= 64 << 20
    ga, gb = _files(a), _files(b)
    idx = ga["sampled_scenarios.npy"]
    assert np.array_equal(idx, gb["sampled_scenarios.npy"])                     # same sample on every run
    assert 0 < len(idx) < n and np.all(np.diff(idx) > 0) and idx.max() < n      # sorted, distinct, in range
    for k in STATE:
        assert ga[k + ".npy"].shape == (len(idx), m)
        assert np.array_equal(ga[k + ".npy"][:, 0], idx)                          # the rows are the sampled scenarios
    assert np.array_equal(ga["status.npy"], idx % 5) and np.array_equal(ga["done.npy"], idx % 2)
    for f in ga:
        assert np.array_equal(ga[f], gb[f])


def test_extra_arrays_are_written_whole_and_counted(tmp_path):
    import torch

    world, result = _stand_in(128, 4)
    done_all = torch.arange(8 * 128, dtype=torch.uint8).view(8, 128) % 2
    bench.dump_outputs(str(tmp_path), world, result, extra={"done_all": done_all})
    got = _files(tmp_path)
    assert got["done_all.npy"].shape == (8, 128) and np.array_equal(got["done_all.npy"], done_all.numpy())
