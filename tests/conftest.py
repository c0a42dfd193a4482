import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _split(idx, off):
    return [np.asarray(idx[off[i]:off[i + 1]], dtype=np.int32) for i in range(len(off) - 1)]


@pytest.fixture(scope="session")
def example_object():
    """data/infercnv_object_example.rda of the reference (see tests/golden/make_golden.py)."""
    d = np.load(os.path.join(GOLDEN, "example_object.npz"))
    return {
        "counts": np.asfortranarray(d["counts"].astype(np.float64)),
        "expr": np.asfortranarray(d["expr"]),
        "chr_codes": d["chr_codes"],
        "ref_groups": [g - 1 for g in _split(d["ref_idx"], d["ref_off"])],
        "obs_groups": [g - 1 for g in _split(d["obs_idx"], d["obs_off"])],
        "subclusters": [g - 1 for g in _split(d["sub_idx"], d["sub_off"])],
        "sub_names": list(d["sub_names"]),
    }


@pytest.fixture(scope="session")
def oligo():
    """inst/extdata oligodendroglioma example after the reference's ingest filters (8508 x 184)."""
    d = np.load(os.path.join(GOLDEN, "oligodendroglioma.npz"))
    return {
        "counts": np.asfortranarray(d["counts"].astype(np.float64)),
        "chr_codes": d["chr_codes"],
        "ref_groups": [g - 1 for g in _split(d["ref_idx"], d["ref_off"])],
        "obs_groups": [g - 1 for g in _split(d["obs_idx"], d["obs_off"])],
    }


@pytest.fixture(scope="session")
def hmm_fixture():
    d = np.load(os.path.join(GOLDEN, "hmm_fixture.npz"))
    return {"mean": d["mu"], "sd": d["sd"], "hmm_states": d["hmm_states"]}
