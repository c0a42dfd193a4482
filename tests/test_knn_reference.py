"""tests/knn_reference.py, the expected values of the k-nearest-neighbour kernel, pinned on the CPU: against scipy's exact
kd-tree (cKDTree.query, eps = 0 - what RANN's ANN search computes) on tie-free data, and against hand-made ties, where the
rule (squared distance, then position) decides."""
import numpy as np
import pytest
from scipy.spatial import cKDTree
from scipy.spatial.distance import pdist

from tests import knn_reference as kr


@pytest.mark.parametrize("n,G,k", [(1, 3, 1), (2, 1, 2), (50, 3, 7), (300, 17, 20), (257, 64, 64)])
def test_brute_force_equals_cKDTree_on_tie_free_data(n, G, k):
    x = np.random.default_rng(n + G).normal(size=(n, G))
    idx, dist = kr.knn_brute(x, k)
    td, ti = cKDTree(x).query(x, k=k, eps=0)
    td, ti = td.reshape(n, k), ti.reshape(n, k)
    assert np.array_equal(idx, ti)
    np.testing.assert_allclose(dist, td, rtol=1e-13, atol=1e-15)
    assert np.array_equal(idx[:, 0], np.arange(n))        # self first


@pytest.mark.parametrize("n,k", [(2, 1), (130, 20), (300, 64)])
def test_from_the_dist_vector_equals_brute_force(n, k):
    x = np.random.default_rng(n).normal(size=(n, 9))
    idx, dist = kr.knn_from_dist(pdist(x), n, k, block=37)
    bi, bd = kr.knn_brute(x, k)
    assert np.array_equal(idx, bi)
    np.testing.assert_allclose(dist, bd, rtol=1e-13, atol=1e-15)


def test_duplicates_order_by_position():
    rng = np.random.default_rng(1)
    base = rng.normal(size=(20, 5))
    x = base[rng.integers(0, 20, size=120)]
    k = 12
    idx, dist = kr.knn_brute(x, k)
    for i in range(len(x)):
        same = np.flatnonzero(np.all(x == x[i], axis=1))
        m = min(len(same), k)
        assert np.array_equal(idx[i, :m], same[:m])         # the copies of cell i, lowest positions first
        assert np.all(dist[i, :m] == 0.0)
        # ties further out: equal distances appear in ascending position
        for a in range(k - 1):
            if dist[i, a] == dist[i, a + 1]:
                assert idx[i, a] < idx[i, a + 1]
    # cKDTree finds the same distances (its order among ties is its own)
    td, _ = cKDTree(x).query(x, k=k, eps=0)
    np.testing.assert_allclose(dist, td, rtol=1e-13, atol=1e-15)


def test_all_equal_rows_and_no_genes():
    n, k = 40, 9
    for x in (np.full((n, 6), 2.5), np.zeros((n, 0))):
        idx, dist = kr.knn_brute(x, k)
        assert np.array_equal(idx, np.tile(np.arange(k, dtype=np.int32), (n, 1)))
        assert np.all(dist == 0.0)
        idx2, dist2 = kr.knn_from_dist(pdist(x) if x.shape[1] else np.zeros(n * (n - 1) // 2), n, k)
        assert np.array_equal(idx2, idx) and np.all(dist2 == 0.0)


def test_k_equal_to_n_lists_every_position():
    x = np.random.default_rng(4).normal(size=(33, 4))
    idx, _ = kr.knn_brute(x, 33)
    assert np.array_equal(np.sort(idx, axis=1), np.tile(np.arange(33), (33, 1)))
