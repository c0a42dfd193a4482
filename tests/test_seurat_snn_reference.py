"""Hand-checked cases of tests/seurat_snn_reference.py, the NumPy restatement K18's GPU tests compare against."""
import numpy as np

from tests import seurat_snn_reference as sr


def test_k3_graph_by_hand():
    """Five points on a line at 0, 1, 2, 10, 11 with k = 3 (self included; point 1's tie between 0 and 2 goes to position 0):
    N(0) = {0, 1, 2}, N(1) = {1, 0, 2}, N(2) = {2, 1, 0}, N(3) = {3, 4, 2}, N(4) = {4, 3, 2}.  s = 3 gives 3 / 3 = 1,
    s = 1 gives 1 / (3 + 2) = 0.2, and no pair shares exactly 2."""
    E = np.array([[0.0], [1.0], [2.0], [10.0], [11.0]])
    idx = sr.knn(E, 3)
    assert idx.tolist() == [[0, 1, 2], [1, 0, 2], [2, 1, 0], [3, 4, 2], [4, 3, 2]]
    g = sr.snn(idx, 5, 3).toarray()
    want = np.array([[1.0, 1.0, 1.0, 0.2, 0.2],
                     [1.0, 1.0, 1.0, 0.2, 0.2],
                     [1.0, 1.0, 1.0, 0.2, 0.2],
                     [0.2, 0.2, 0.2, 1.0, 1.0],
                     [0.2, 0.2, 0.2, 1.0, 1.0]])
    assert np.array_equal(g, want)


def test_prune_edge_k24_s3_is_kept():
    """k = 24: s = 3 gives 3 / (24 + 21) = 1/15 exactly in double, which is not < 1/15, so the pair is kept; s = 2 gives
    2 / 46 < 1/15 and is dropped."""
    k, n = 24, 100
    assert 3 / (k + (k - 3)) == 1.0 / 15.0
    idx = np.array([[i] + [(i + 1 + j) % n for j in range(k - 1)] for i in range(n)], dtype=np.int32)
    idx[0] = [0, 1, 2] + list(range(3, 24))
    idx[1] = [1, 0, 2] + list(range(24, 45))
    idx[2] = [2, 0] + list(range(45, 67))
    g = sr.snn(idx, n, k).toarray()
    assert g[0, 1] == 1.0 / 15.0 and g[1, 0] == 1.0 / 15.0
    assert g[0, 2] == 0.0


def test_tied_standardised_variances_resolved_by_index():
    """Genes 2 and 5 are the same values: equal standardised variances, and the lower index ranks first."""
    rng = np.random.default_rng(3)
    X = rng.gamma(4.0, 1.0, size=(40, 200)) + 1.0
    X[5] = X[2]
    feats, sv, _ = sr.variable_features(X, 40)
    assert sv[2] == sv[5]
    r = {g: i for i, g in enumerate(feats)}
    assert r[2] + 1 == r[5]


def test_constant_gene_scores_zero_and_is_left_out_of_pca():
    rng = np.random.default_rng(4)
    X = rng.gamma(4.0, 1.0, size=(30, 100)) + 1.0
    X[7] = 2.5
    feats, sv, _ = sr.variable_features(X, 30)
    assert sv[7] == 0.0 and feats[-1] == 7
    use, lam, V, E = sr.pca(X, feats, 5)
    assert 7 not in use and len(use) == 29
    assert np.all(np.diff(lam[:6]) <= 0)
    for j in range(5):
        f = np.argmax(np.abs(V[:, j]))
        assert V[f, j] > 0


def test_loess_reproduces_a_quadratic():
    """Degree-2 local regression is exact on a quadratic, whatever the weights."""
    x = np.linspace(-1.0, 2.0, 50)
    y = 0.3 - 0.7 * x + 0.25 * x * x
    fit, sing = sr.loess_direct(x, y)
    assert np.allclose(fit, y, atol=1e-12) and not sing.any()
