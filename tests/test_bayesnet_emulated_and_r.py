"""CPU checks of the Bayesian network filter: the GPU tests of tests/test_gpu_bayesnet.py run against the kernels' own source
(icnv_bayes.cu) under the host emulation of tests/host/ (built by tests/host/build_emu_bayesnet.py) in both resume orders of
the block's threads, whose draws must be bit-identical; and the R closure / shim that bind it are checked the way
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

# one small sampling run, its outputs printed as a digest
DIGEST = """
import hashlib, sys
sys.path[:0] = [{root!r}]
import numpy as np
from infercnv_b200 import _lib
_lib.LIB_PATH = {lib!r}
from infercnv_b200 import api
rng = np.random.default_rng(3)
X = np.asfortranarray(rng.normal(1.0, 0.3, size=(40, 300)))
res = api.bayesnet(X, [np.arange(10), np.arange(10, 40), np.array([5])], [np.arange(300), np.arange(0, 300, 7), np.arange(9)],
                   [0.4, 0.7, 1.0, 1.3, 1.6, 1.9], [30.0, 40.0, 60.0, 40.0, 30.0, 20.0], 6, n_burn=5, n_keep=10, seed=9,
                   pooled=[False, False, True], want_loglik=True)
h = hashlib.sha256()
for k in ("theta", "state_counts", "loglik"):
    for a in res[k]:
        h.update(np.ascontiguousarray(a).tobytes())
print("DIGEST", h.hexdigest())
"""


@pytest.fixture(scope="module")
def emulated_lib(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tests", "host"))
    import build_emu_bayesnet
    return build_emu_bayesnet.build(str(tmp_path_factory.mktemp("emu_bayesnet")))


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_gpu_bayesnet_tests_under_the_host_emulation(order, emulated_lib):
    env = dict(os.environ, EMU_ORDER=order)
    code = EMULATE.format(root=ROOT, lib=emulated_lib, test=os.path.join(ROOT, "tests", "test_gpu_bayesnet.py"))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert re.search(r"\d+ passed", r.stdout), r.stdout[-2000:]


def test_both_thread_orders_draw_the_same_bits(emulated_lib):
    out = []
    for order in ("forward", "reverse"):
        r = subprocess.run([sys.executable, "-c", DIGEST.format(root=ROOT, lib=emulated_lib)], cwd=ROOT,
                           env=dict(os.environ, EMU_ORDER=order), capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        out.append(re.search(r"DIGEST (\w+)", r.stdout).group(1))
    assert out[0] == out[1]


def test_r_closure_is_installed():
    src = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnv_b200.R")).read()
    assert ("b200_inferCNVBayesNet <- function( file_dir,\n"
            "                              infercnv_obj,\n"
            "                              HMM_states,\n"
            "                              out_dir,\n"
            "                              resume_file_token,\n"
            "                              model_file        = NULL,\n"
            "                              CORES             = 1,\n"
            "                              postMcmcMethod    = NULL,\n"
            "                              plotingProbs      = TRUE,\n"
            "                              quietly           = TRUE,\n"
            "                              diagnostics       = FALSE,\n"
            "                              HMM_type          = HMM_type,\n"
            "                              k_obs_groups      = k_obs_groups,\n"
            "                              cluster_by_groups = cluster_by_groups,\n"
            "                              reassignCNVs      = TRUE,\n"
            "                              no_plot           = no_plot,\n"
            "                              useRaster) {") in src
    assert '"mask_non_DE_genes_basic", "inferCNVBayesNet"' in src and '.Call("icnvR_bayesnet"' in src
    assert '"Gibbs sampling time: "' in src and "saveRDS(" in src and "postProbNormal(" in src
    assert "sample.int(2^31 - 1, 1), sample.int(2^31 - 1, 1)" in src
    shim = open(os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")).read()
    assert '{"icnvR_bayesnet", (DL_FUNC)&icnvR_bayesnet, 10}' in shim


def test_r_shim_with_the_bayesnet_compiles_against_the_mock_headers():
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    r = subprocess.run([gcc, "-fsyntax-only", "-Wall", "-Werror=implicit-function-declaration",
                        "-Werror=incompatible-pointer-types", "-Werror=int-conversion",
                        "-I", os.path.join(ROOT, "infercnv_b200", "r", "mock"), "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "infercnv_b200", "r", "infercnvb200_shim.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
