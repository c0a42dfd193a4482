"""CPU checks of the running mean and the random-trees null: the GPU tests of tests/test_gpu_random_trees.py run against
the kernels' own source (icnv_random_trees.cu with icnv_dist.cu, icnv_hclust.cu and the cell pipeline) under the host
emulation of tests/host/ (built by tests/host/build_emu_random_trees.py; both resume orders of the block's threads; the
emulation reports 4 SMs, so waves of at most 4 members), and the R closures / shim that bind them are checked the way
tests/test_r_shim_compiles.py checks the rest of the R layer (no R here)."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# what tests/host/run_emulated.py does (point the ctypes loader at an emulated build first), for this one test file
EMULATE = """
import sys
sys.path[:0] = [{root!r}]
import pytest
from infercnv_b200 import _lib
_lib.LIB_PATH = {lib!r}
sys.exit(pytest.main([{test!r}, "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"]))
"""


@pytest.fixture(scope="module")
def emulated_lib(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tests", "host"))
    import build_emu_random_trees
    return build_emu_random_trees.build(str(tmp_path_factory.mktemp("emu_random_trees")))


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_gpu_random_trees_tests_under_the_host_emulation(order, emulated_lib):
    env = dict(os.environ, EMU_ORDER=order)
    code = EMULATE.format(root=ROOT, lib=emulated_lib, test=os.path.join(ROOT, "tests", "test_gpu_random_trees.py"))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert re.search(r"\d+ passed", r.stdout), r.stdout[-2000:]


def test_r_closures_are_installed():
    src = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnv_b200.R")).read()
    assert "b200_smooth_by_chromosome_runmeans <- function(infercnv_obj, window_length)" in src
    assert ("b200_.parameterize_random_cluster_heights_smoothed_trees <- function(expr_matrix, hclust_method, window_size,"
            " plot = FALSE)") in src
    assert '.Call("icnvR_runmean"' in src and '.Call("icnvR_random_tree_heights"' in src
    assert '"smooth_by_chromosome_runmeans"' in src and '".parameterize_random_cluster_heights_smoothed_trees"' in src
    shim = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")).read()
    assert '{"icnvR_runmean", (DL_FUNC)&icnvR_runmean, 4}' in shim
    assert '{"icnvR_random_tree_heights", (DL_FUNC)&icnvR_random_tree_heights, 5}' in shim


def test_r_shim_with_random_trees_compiles_against_the_mock_headers():
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    r = subprocess.run([gcc, "-fsyntax-only", "-Wall", "-Werror=implicit-function-declaration",
                        "-Werror=incompatible-pointer-types", "-Werror=int-conversion",
                        "-I", os.path.join(ROOT, "infercnv_b200", "r", "mock"), "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
