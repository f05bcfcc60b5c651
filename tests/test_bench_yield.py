"""``bench_yield.py`` parses its arguments without a device, like the other side benchmarks."""

import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_help_without_a_device():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench_yield.py"), "--help"], cwd=ROOT,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "usage:" in r.stdout
