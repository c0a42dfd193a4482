"""CPU checks of the coordinate smoother: the GPU tests of tests/test_gpu_smooth_coordinates.py run against the kernel's
own source (icnv_smooth_coords.cu) under the host emulation of tests/host/ (built by tests/host/build_emu_smooth_coords.py;
both resume orders of the block's threads), and the R closure / shim that bind it are checked the way
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
    import build_emu_smooth_coords
    return build_emu_smooth_coords.build(str(tmp_path_factory.mktemp("emu_smooth_coords")))


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_gpu_smooth_coordinates_tests_under_the_host_emulation(order, emulated_lib):
    env = dict(os.environ, EMU_ORDER=order)
    code = EMULATE.format(root=ROOT, lib=emulated_lib, test=os.path.join(ROOT, "tests", "test_gpu_smooth_coordinates.py"))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert re.search(r"\d+ passed", r.stdout), r.stdout[-2000:]


def test_r_closure_is_installed():
    src = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnv_b200.R")).read()
    assert "b200_smooth_by_chromosome_coordinates <- function(infercnv_obj, window_length)" in src
    assert '.Call("icnvR_smooth_coordinates"' in src
    assert '"smooth_by_chromosome_coordinates"' in src
    assert 'flog.info(paste0("smooth_by_chromosome: chr: ", chr))' in src
    assert "b200_smooth_by_chromosome_coordinates(infercnv_obj@.hspike, window_length = 51)" in src
    shim = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")).read()
    assert '{"icnvR_smooth_coordinates", (DL_FUNC)&icnvR_smooth_coordinates, 6}' in shim


def test_r_shim_with_coordinate_smoothing_compiles_against_the_mock_headers():
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    r = subprocess.run([gcc, "-fsyntax-only", "-Wall", "-Werror=implicit-function-declaration",
                        "-Werror=incompatible-pointer-types", "-Werror=int-conversion",
                        "-I", os.path.join(ROOT, "infercnv_b200", "r", "mock"), "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
