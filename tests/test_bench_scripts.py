"""The side benchmarks parse their arguments without a device, and their shared helper module imports neither torch nor the
package: ``bench_tick_phases.py`` imports it before it points the package at another build of the library."""

import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = ["bench_agents.py", "bench_bev.py", "bench_control.py", "bench_lidar.py", "bench_obs.py", "bench_replay.py",
           "bench_tick.py", "bench_tick_phases.py"]


def _run(args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    return subprocess.run([sys.executable, *args], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)


@pytest.mark.parametrize("script", SCRIPTS)
def test_help_without_a_device(script):
    r = _run([os.path.join(ROOT, script), "--help"])
    assert r.returncode == 0, r.stderr[-2000:]
    assert "usage:" in r.stdout


def test_benchlib_imports_neither_torch_nor_the_package():
    # a fresh interpreter: other test modules import torch during collection
    r = _run(["-c", "import sys, benchlib; print(sorted({'torch', 'tactics2d_b200'} & set(sys.modules)))"])
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.strip() == "[]"
