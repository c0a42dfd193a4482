"""CPU checks of the subclustering trees: the GPU tests of tests/test_gpu_subclusters.py run against the kernels' own source
(icnv_subclusters.cu with icnv_dist.cu, icnv_hclust.cu and the column statistics) under the host emulation of tests/host/
(built by tests/host/build_emu_subclusters.py; both resume orders of the block's threads; the emulation reports 4 SMs, so
several waves), and the R closure / shim entries that bind them are checked the way tests/test_r_shim_compiles.py checks the
rest of the R layer (no R here)."""
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
    import build_emu_subclusters
    return build_emu_subclusters.build(str(tmp_path_factory.mktemp("emu_subclusters")))


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_gpu_subcluster_tests_under_the_host_emulation(order, emulated_lib):
    env = dict(os.environ, EMU_ORDER=order)
    code = EMULATE.format(root=ROOT, lib=emulated_lib, test=os.path.join(ROOT, "tests", "test_gpu_subclusters.py"))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert re.search(r"\d+ passed", r.stdout), r.stdout[-2000:]


def test_r_closure_is_installed():
    src = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnv_b200.R")).read()
    assert "b200_define_signif_tumor_subclusters <- function(infercnv_obj, p_val = 0.1, k_nn = 20," in src
    assert '.Call("icnvR_zscore_outlier_genes"' in src and '.Call("icnvR_cluster_groups"' in src
    assert '"define_signif_tumor_subclusters",' in src
    assert "infercnv:::.leiden_seurat_preprocess_routine" in src and "infercnv:::.leiden_simple_snn" in src
    assert "infercnv:::.whole_dataset_leiden_subclustering_per_chr" in src
    shim = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")).read()
    assert '{"icnvR_zscore_outlier_genes", (DL_FUNC)&icnvR_zscore_outlier_genes, 2}' in shim
    assert '{"icnvR_cluster_groups", (DL_FUNC)&icnvR_cluster_groups, 4}' in shim


def test_r_shim_with_subclusters_compiles_against_the_mock_headers():
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    r = subprocess.run([gcc, "-fsyntax-only", "-Wall", "-Werror=implicit-function-declaration",
                        "-Werror=incompatible-pointer-types", "-Werror=int-conversion",
                        "-I", os.path.join(ROOT, "infercnv_b200", "r", "mock"), "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
