"""CPU checks of the non-DE mask: the GPU tests of tests/test_gpu_de_mask.py run against the kernels' own source
(icnv_de.cu) under the host emulation of tests/host/ (built by tests/host/build_emu_de.py; both resume orders of the
block's threads), and the R closure / shim that bind it are checked the way tests/test_r_shim_compiles.py checks the rest
of the R layer (no R here)."""
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
    import build_emu_de
    return build_emu_de.build(str(tmp_path_factory.mktemp("emu_de")))


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_gpu_de_mask_tests_under_the_host_emulation(order, emulated_lib):
    env = dict(os.environ, EMU_ORDER=order)
    code = EMULATE.format(root=ROOT, lib=emulated_lib, test=os.path.join(ROOT, "tests", "test_gpu_de_mask.py"))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert re.search(r"\d+ passed", r.stdout), r.stdout[-2000:]


def test_r_closure_is_installed():
    src = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnv_b200.R")).read()
    assert ('b200_mask_non_DE_genes_basic <- function(infercnv_obj, p_val_thresh = 0.05, test.use = "wilcoxon",\n'
            '                                         center_val = mean(infercnv_obj@expr.data), require_DE_all_normals = "any")'
            ) in src
    assert '"mask_non_DE_genes_basic"' in src and '.Call("icnvR_mask_non_de"' in src
    assert 'sprintf("Finding DE genes between %s and %s"' in src and 'sprintf("Found %d genes / %d total as DE"' in src
    shim = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")).read()
    assert '{"icnvR_mask_non_de", (DL_FUNC)&icnvR_mask_non_de, 8}' in shim


def test_r_shim_with_the_mask_compiles_against_the_mock_headers():
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    r = subprocess.run([gcc, "-fsyntax-only", "-Wall", "-Werror=implicit-function-declaration",
                        "-Werror=incompatible-pointer-types", "-Werror=int-conversion",
                        "-I", os.path.join(ROOT, "infercnv_b200", "r", "mock"), "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
