"""tests/test_gpu_cell_pipeline_median_routes.py under the host emulation (tests/host/run_emulated.py), in both resume
orders of a block's threads: the histogram of the per-cell median is filled by shared-memory atomics inside the smoothing
output loops and read behind the barrier that ends them, so a result that depended on the order would mean a missing
barrier.  Test infrastructure only; says nothing about performance."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None and not os.path.exists("/usr/bin/g++"), reason="no host compiler")
@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_median_routes_under_the_host_emulation(order):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "host", "run_emulated.py"),
                        os.path.join(ROOT, "tests", "test_gpu_cell_pipeline_median_routes.py"), "-k", "test_median_route"],
                       capture_output=True, text=True, timeout=1500, env=dict(os.environ, EMU_ORDER=order))
    tail = "\n".join(r.stdout.splitlines()[-25:]) + r.stderr[-2000:]
    assert r.returncode == 0, tail
    assert "10 passed" in r.stdout and "failed" not in r.stdout, tail
