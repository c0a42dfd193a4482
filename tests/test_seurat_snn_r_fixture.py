"""Consumes tools/make_seurat_snn_fixture.R's output when a box with R and Seurat 5 has produced it
(ICNV_SEURAT_FIXTURE_DIR): K18's variable features and SNN graph against Seurat's own on the same matrix.  Skipped when the
fixture is absent (producing it needs R with Seurat 5); tests/test_gpu_seurat_snn.py pins the same computation against
the NumPy restatement meanwhile.

The bounds are the deviations K18 states: vst's loess is interpolated in R and direct on the device, so features may differ
only where the standardised variance lies within LOESS_REL of the cut; irlba's tolerance (1e-5) can move near-ties of the
neighbour lists, so at least 99 % of the graph's rows must have Seurat's columns."""
import os

import numpy as np
import pytest

DIR = os.environ.get("ICNV_SEURAT_FIXTURE_DIR", os.path.join(os.path.dirname(__file__), "golden", "seurat_fixture"))
pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not os.path.exists(os.path.join(DIR, "snn_x.bin")),
                                 reason="no Seurat-generated fixture (run tools/make_seurat_snn_fixture.R on a box with R)")]
LOESS_REL = 1e-3


def _load():
    meta = dict(line.split("=") for line in open(os.path.join(DIR, "meta.txt")).read().split())
    G, C, k = int(meta["G"]), int(meta["C"]), int(meta["k"])
    X = np.fromfile(os.path.join(DIR, "x.bin"), dtype="<f8").reshape(C, G).T
    feats = np.array([int(v) - 1 for v in open(os.path.join(DIR, "features.txt")).read().split()])
    i = np.fromfile(os.path.join(DIR, "snn_i.bin"), dtype="<i4")
    j = np.fromfile(os.path.join(DIR, "snn_j.bin"), dtype="<i4")
    x = np.fromfile(os.path.join(DIR, "snn_x.bin"), dtype="<f8")
    return np.asfortranarray(X), feats, (i, j, x), k


def test_variable_features_and_graph_match_seurat():
    import scipy.sparse as sp
    from infercnv_b200 import api
    from tests import seurat_snn_reference as sr
    api.init(0)
    X, feats, (i, j, x), k = _load()
    C = X.shape[1]
    r = api.seurat_snn(X, k=k)
    _, sv, _ = sr.variable_features(X)
    cut = np.sort(sv)[::-1][len(feats) - 1]
    differ = np.setxor1d(r.features, feats)
    assert np.all(np.abs(sv[differ] - cut) <= LOESS_REL * cut), differ
    want = sp.csr_matrix((x, (i, j)), shape=(C, C))
    want.sort_indices()
    same = [np.array_equal(r.indices[r.indptr[a]:r.indptr[a + 1]], want.indices[want.indptr[a]:want.indptr[a + 1]])
            for a in range(C)]
    assert np.mean(same) >= 0.99
