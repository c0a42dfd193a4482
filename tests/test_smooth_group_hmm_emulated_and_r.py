"""CPU checks of the fused group-mode calls: the GPU tests of tests/test_gpu_smooth_group_hmm.py run against the library's
own source under the host emulation of tests/host/ (built by tests/host/build_emu_smooth_coords.py, whose library holds
icnv_api.cu, icnv_smooth.cu and icnv_viterbi.cu; both resume orders of the block's threads), and the R closure / shim
routines that bind them are checked the way tests/test_r_shim_compiles.py checks the rest of the R layer (no R here)."""
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
sys.exit(pytest.main([{test!r}, "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider", "-k", {sel!r}]))
"""
# the cases small enough for the emulation: list order, chunks across slabs, overlaps, errors and the drivers' lists
SELECT = "errors or sizes or overlapping or (odd_layouts and thirty) or mirror"


@pytest.fixture(scope="module")
def emulated_lib(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tests", "host"))
    import build_emu_smooth_coords
    return build_emu_smooth_coords.build(str(tmp_path_factory.mktemp("emu_group_hmm")))


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_gpu_smooth_group_hmm_tests_under_the_host_emulation(order, emulated_lib):
    env = dict(os.environ, EMU_ORDER=order)
    code = EMULATE.format(root=ROOT, lib=emulated_lib, test=os.path.join(ROOT, "tests", "test_gpu_smooth_group_hmm.py"),
                          sel=SELECT)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert re.search(r"\d+ passed", r.stdout), r.stdout[-2000:]


def test_r_closure_is_installed():
    src = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnv_b200.R")).read()
    assert ('median_filter_window=NULL, analysis_mode="cells", cluster_by_groups=TRUE,\n'
            '                                          tumor_subcluster_partition_method="random_trees") {') in src
    assert '.Call("icnvR_smooth_hmm_groups"' in src and '.Call("icnvR_smooth_i3_hmm_groups"' in src
    # the i6 sds: the smoothed hspike's fit, in the order the reference's drivers evaluate it
    body = src[src.index(".icnv_smooth_block_groups <- function"):]
    steps = ["infercnvb200_run_smooth_block(infercnv_obj@.hspike", "infercnv:::get_spike_dists(", "infercnv:::.get_HMM(",
             "infercnv:::get_hspike_cnv_mean_sd_trend_by_num_cells_fit(", "infercnv:::.get_state_emission_params(",
             '.Call("icnvR_smooth_hmm_groups"']
    at = [body.index(s) for s in steps]
    assert at == sorted(at)
    assert 'unlist(infercnv_obj@tumor_subclusters[["subclusters"]], recursive=FALSE)' in src
    shim = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")).read()
    assert '{"icnvR_smooth_hmm_groups", (DL_FUNC)&icnvR_smooth_hmm_groups, 12}' in shim
    assert '{"icnvR_smooth_i3_hmm_groups", (DL_FUNC)&icnvR_smooth_i3_hmm_groups, 10}' in shim
    for name, n in (("icnvR_smooth_hmm_groups", 12), ("icnvR_smooth_i3_hmm_groups", 10)):
        sig = re.search(r"SEXP " + name + r"\(([^)]*)\)", shim).group(1)
        assert sig.count("SEXP") == n, name
        call = re.search(r'\.Call\("' + name + r'",(.*?)"smooth_', src, re.S).group(1)
        depth, args = 0, 1   # the arguments after the routine's name: commas inside .Call( ... ) at its own depth, plus one
        for ch in call:
            depth += {"(": 1, ")": -1}.get(ch, 0)
            args += ch == "," and depth == 0
        assert args == n, (name, args)


def test_r_shim_with_group_calls_compiles_against_the_mock_headers():
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    r = subprocess.run([gcc, "-fsyntax-only", "-Wall", "-Werror=implicit-function-declaration",
                        "-Werror=incompatible-pointer-types", "-Werror=int-conversion",
                        "-I", os.path.join(ROOT, "infercnv_b200", "r", "mock"), "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
