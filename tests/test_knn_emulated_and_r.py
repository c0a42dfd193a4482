"""CPU checks of the nn2() path: the GPU tests of tests/test_gpu_knn.py run against the kernel's own source (icnv_dist.cu)
under the host emulation of tests/host/ (both resume orders of the block's threads; the emulation reports 4 SMs, so its
launches split the candidate range differently from the H100's), and the R closure / shim that bind it are checked the way
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
    import build_emu_hclust     # the emulated sources, icnv_dist.cu among them, built into a directory of our choosing
    return build_emu_hclust.build(str(tmp_path_factory.mktemp("emu_knn")))


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_gpu_knn_tests_under_the_host_emulation(order, emulated_lib):
    env = dict(os.environ, EMU_ORDER=order)
    code = EMULATE.format(root=ROOT, lib=emulated_lib, test=os.path.join(ROOT, "tests", "test_gpu_knn.py"))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert re.search(r"\d+ passed", r.stdout), r.stdout[-2000:]


def test_r_closure_is_bound_as_the_nn2_import():
    src = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnv_b200.R")).read()
    assert ('b200_nn2 <- function(data, query = data, k = min(10, nrow(data)), treetype = c("kd", "bd"),\n'
            '                     searchtype = c("standard", "priority", "radius"), radius = 0, eps = 0)') in src
    assert 'assign("nn2", b200_nn2, envir = imp)' in src
    assert 'assign("nn2", .icnv_env$orig_nn2, envir = imp)' in src
    assert '.Call("icnvR_knn", data, as.integer(k))' in src
    assert 'list(nn.idx = res[[1]], nn.dists = res[[2]])' in src
    shim = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")).read()
    assert '{"icnvR_knn", (DL_FUNC)&icnvR_knn, 2}' in shim


def test_r_shim_with_knn_compiles_against_the_mock_headers():
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    r = subprocess.run([gcc, "-fsyntax-only", "-Wall", "-Werror=implicit-function-declaration",
                        "-Werror=incompatible-pointer-types", "-Werror=int-conversion",
                        "-I", os.path.join(ROOT, "infercnv_b200", "r", "mock"), "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
