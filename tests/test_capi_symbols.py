"""The C-ABI shared library loads without a GPU and exports every symbol include/infercnv_b200.h
declares; compute entries fail loudly (no CPU fallback) when no CUDA device is present."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    hdr = open(os.path.join(ROOT, "include", "infercnv_b200.h")).read()
    return sorted(set(re.findall(r"ICNV_API\s+[\w\s\*]+?\b(icnv_\w+)\s*\(", hdr)))


def test_header_symbols_are_exported_and_bound():
    from infercnv_b200 import _lib
    lib = _lib.load()
    names = _declared()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), f"{n} declared in the header but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes prototype"
    assert lib.icnv_version().startswith(b"infercnv_b200")


def test_no_cpu_fallback_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from infercnv_b200 import api
    from infercnv_b200._lib import InfercnvB200Error
    with pytest.raises(InfercnvB200Error) as e:
        api.center(np.ones((4, 3)))
    assert e.value.code == -1
    with pytest.raises(InfercnvB200Error):
        api.smooth_block(np.ones((6, 3)), [0], [6], [[0]])
    with pytest.raises(InfercnvB200Error) as e:
        api.last_cell_kernel()
    assert e.value.code == -1


def test_cell_kernel_query_is_declared_and_bound():
    """icnv_debug_cell_kernel reports which fused cell-pipeline instantiation ran (tests/test_gpu_cell_pipeline_variants.py
    asserts it per case): declared in the header, exported, six ints out."""
    from infercnv_b200 import _lib
    assert "icnv_debug_cell_kernel" in _declared()
    assert _lib.SIGNATURES["icnv_debug_cell_kernel"] == (_lib.c_int, [_lib._P])
    assert hasattr(_lib.load(), "icnv_debug_cell_kernel")


def test_hmm_mode_other_than_0_or_1_is_refused():
    """icnv_set_hmm_mode takes 0 (reference-order arithmetic) and 1 (certified FP64 pass); any other mode, 2 included, is
    ICNV_E_BAD_ARG.  The mode is host state: no device is needed."""
    from infercnv_b200 import _lib
    lib = _lib.load()
    assert lib.icnv_set_hmm_mode(2) == -3 and b"hmm mode" in lib.icnv_last_error()
    assert lib.icnv_set_hmm_mode(1) == 0


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "infercnv_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".c", ".h", ".R")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                assert "oracle" not in src.replace("oracle/", "").lower() or f == "build.py" or "test infrastructure" in src.lower() \
                    or all("import" not in line and "include" not in line for line in src.splitlines() if "oracle" in line.lower()), \
                    f"{f} refers to the oracle"
