"""CPU checks of the packed-triangle linkage (K19): the GPU tests of tests/test_gpu_hclust_tri.py run against the kernel's own
source under the host emulation of tests/host/ (both resume orders of the block's threads, sizes up to 40 observations), and
the R closures / shim routines that bind it are checked the way tests/test_r_shim_compiles.py checks the rest of the R layer
(no R here)."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# what tests/host/run_emulated.py does (point the ctypes loader at an emulated build first), for this one test file and
# with the emulated build that includes the packed-triangle linkage (tests/host/build_emu_hclust_tri.py)
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
    import build_emu_hclust_tri
    return build_emu_hclust_tri.build(str(tmp_path_factory.mktemp("emu_hclust_tri")))


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_gpu_hclust_tri_tests_under_the_host_emulation(order, emulated_lib):
    env = dict(os.environ, EMU_ORDER=order)
    code = EMULATE.format(root=ROOT, lib=emulated_lib, test=os.path.join(ROOT, "tests", "test_gpu_hclust_tri.py"))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert re.search(r"\d+ passed", r.stdout), r.stdout[-2000:]


def test_r_closures_route_past_65536_to_the_packed_triangle():
    src = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnv_b200.R")).read()
    assert '.icnv_try(.Call("icnvR_hclust_tri", d, code), "hclust (packed triangle)")' in src
    assert 'if (n <= 65536) .icnv_try(.Call("icnvR_hclust", d, code), "hclust") else' in src
    assert '.Call("icnvR_cluster_cells", m, kp, as.integer(lists[[i]]), codes[[hclust_method]])' in src
    assert "big <- lengths(lists) > 65536" in src
    assert "nrow(x) <= 65535 * 128" in src
    shim = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")).read()
    assert '{"icnvR_hclust_tri", (DL_FUNC)&icnvR_hclust_tri, 2}' in shim
    assert '{"icnvR_cluster_cells", (DL_FUNC)&icnvR_cluster_cells, 4}' in shim


def test_r_shim_with_the_packed_triangle_compiles_against_the_mock_headers():
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    r = subprocess.run([gcc, "-fsyntax-only", "-Wall", "-Werror=implicit-function-declaration",
                        "-Werror=incompatible-pointer-types", "-Werror=int-conversion",
                        "-I", os.path.join(ROOT, "infercnv_b200", "r", "mock"), "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
