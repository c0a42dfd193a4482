"""CPU checks of the Leiden PCA-route graph: the GPU tests of tests/test_gpu_seurat_snn.py run against the kernels' own
source (icnv_snn.cu, with icnv_dist.cu's kNN) under the host emulation of tests/host/ (both resume orders of the block's
threads; the FP64 tensor-core product runs as the stand-in of tests/host/build_emu_snn.py), and the R closure / shim that
bind it are checked the way tests/test_r_shim_compiles.py checks the rest of the R layer (no R here)."""
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
    import build_emu_snn
    return build_emu_snn.build(str(tmp_path_factory.mktemp("emu_snn")))


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_gpu_seurat_snn_tests_under_the_host_emulation(order, emulated_lib):
    env = dict(os.environ, EMU_ORDER=order)
    code = EMULATE.format(root=ROOT, lib=emulated_lib, test=os.path.join(ROOT, "tests", "test_gpu_seurat_snn.py"))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert re.search(r"\d+ passed", r.stdout), r.stdout[-2000:]


def test_r_closure_replaces_the_leiden_preprocess_routine():
    src = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnv_b200.R")).read()
    assert ("b200_.leiden_seurat_preprocess_routine <- function(expr_data, k_nn, resolution_parameter, "
            "objective_function) {") in src
    assert '".parameterize_random_cluster_heights_smoothed_trees", ".leiden_seurat_preprocess_routine")' in src
    assert '.Call("icnvR_seurat_snn", expr_data, as.integer(k_nn))' in src
    body = src[src.index("b200_.leiden_seurat_preprocess_routine <- function"):]
    body = body[:body.index("\n}\n")]
    # the RNG is seeded before the graph reaches igraph, and igraph is called as the original calls it
    assert body.index("set.seed(42)") < body.index("graph_from_adjacency_matrix(snn, mode = \"min\", weighted = TRUE)")
    assert ("cluster_leiden(graph_obj, resolution_parameter = resolution_parameter,\n"
            "                                                    objective_function = objective_function)") in body
    assert "orig(expr_data, k_nn, resolution_parameter, objective_function)" in body
    assert "k_nn <= 64" in body and "res[[4]] == 0L" in body
    shim = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")).read()
    assert '{"icnvR_seurat_snn", (DL_FUNC)&icnvR_seurat_snn, 2}' in shim


def test_r_shim_with_seurat_snn_compiles_against_the_mock_headers():
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    r = subprocess.run([gcc, "-fsyntax-only", "-Wall", "-Werror=implicit-function-declaration",
                        "-Werror=incompatible-pointer-types", "-Werror=int-conversion",
                        "-I", os.path.join(ROOT, "infercnv_b200", "r", "mock"), "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
