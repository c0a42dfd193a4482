"""CPU checks of the hclust() path: the GPU tests of tests/test_gpu_hclust.py run against the kernel's own source under the
host emulation of tests/host/ (both resume orders of the block's threads), and the R closure / shim that bind it are checked the way
tests/test_r_shim_compiles.py checks the rest of the R layer (no R here)."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# what tests/host/run_emulated.py does (point the ctypes loader at an emulated build first), for this one test file and
# with the emulated build that includes the linkage kernel (tests/host/build_emu_hclust.py)
EMULATE = """
import sys
sys.path[:0] = [{root!r}]
import pytest
from infercnv_b200 import _lib
_lib.LIB_PATH = {lib!r}
sys.exit(pytest.main([{test!r}, "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider", "-k", "not full_size and not 20000"]))
"""


@pytest.fixture(scope="module")
def emulated_lib(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tests", "host"))
    import build_emu_hclust
    return build_emu_hclust.build(str(tmp_path_factory.mktemp("emu_hclust")))


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_gpu_hclust_tests_under_the_host_emulation(order, emulated_lib):
    env = dict(os.environ, EMU_ORDER=order)
    code = EMULATE.format(root=ROOT, lib=emulated_lib, test=os.path.join(ROOT, "tests", "test_gpu_hclust.py"))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert re.search(r"\d+ passed", r.stdout), r.stdout[-2000:]


def test_r_closure_is_bound_as_the_hclust_import():
    src = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnv_b200.R")).read()
    assert 'b200_hclust <- function(d, method = "complete", members = NULL)' in src
    assert 'assign("hclust", b200_hclust, envir = imp)' in src
    assert 'assign("hclust", .icnv_env$orig_hclust, envir = imp)' in src
    assert '.Call("icnvR_hclust", d, code)' in src
    shim = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")).read()
    assert '{"icnvR_hclust", (DL_FUNC)&icnvR_hclust, 2}' in shim


def test_r_shim_with_hclust_compiles_against_the_mock_headers():
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    r = subprocess.run([gcc, "-fsyntax-only", "-Wall", "-Werror=implicit-function-declaration",
                        "-Werror=incompatible-pointer-types", "-Werror=int-conversion",
                        "-I", os.path.join(ROOT, "infercnv_b200", "r", "mock"), "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
