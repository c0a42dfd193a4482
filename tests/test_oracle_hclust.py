"""The reference restatement of the linkage kernel (tests/hclust_reference.py) pinned by things that are not itself: scipy's
linkage on tie-free data, a literal closest-pair transcription, R's hcass2 loop, and the two ward.D2 trees the reference
stores in its example object (`@tumor_subclusters$hc`).  CPU only."""
import os

import numpy as np
import pytest
from scipy.cluster.hierarchy import linkage
from scipy.spatial.distance import pdist

from tests import hclust_reference as hr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
SCIPY = {"single": "single", "complete": "complete", "average": "average", "mcquitty": "weighted", "ward.D2": "ward"}


def scipy_to_r(Z, n):
    """scipy's linkage matrix -> R's merge (scipy numbers the cluster of step s as n + s, 0-based; R as +s, 1-based)."""
    m = np.zeros((n - 1, 2), dtype=np.int32)
    for s, (a, b) in enumerate(Z[:, :2].astype(int)):
        lo, hi = sorted((a, b))
        m[s] = [-(lo + 1) if lo < n else lo - n + 1, -(hi + 1) if hi < n else hi - n + 1]
    return m


def tie_free(n, seed):
    x = np.random.default_rng(seed).normal(size=(n, 7))
    return pdist(x)


@pytest.mark.parametrize("n", [2, 3, 10, 257, 1000])
@pytest.mark.parametrize("method", sorted(SCIPY))
def test_nn_chain_matches_scipy_on_tie_free_data(n, method):
    d = tie_free(n, n)
    merge, height, order = hr.nn_chain(d, n, hr.METHODS[method])
    Z = linkage(d, SCIPY[method])
    assert np.array_equal(merge, scipy_to_r(Z, n))
    np.testing.assert_allclose(height, Z[:, 2], rtol=1e-13, atol=0)
    hr.check_tree(d, n, hr.METHODS[method], merge, height, order)


@pytest.mark.parametrize("n", [2, 3, 10, 257])
@pytest.mark.parametrize("method", sorted(hr.METHODS))
def test_nn_chain_matches_the_literal_closest_pair_transcription(n, method):
    d = tie_free(n, 100 + n)
    code = hr.METHODS[method]
    m1, h1, o1 = hr.nn_chain(d, n, code)
    m2, h2, o2 = hr.closest_pair(d, n, code)
    assert np.array_equal(m1, m2) and np.array_equal(o1, o2)
    np.testing.assert_allclose(h1, h2, rtol=1e-13, atol=0)


def test_nn_chain_matches_the_closest_pair_transcription_at_1000_for_ward_d():
    """ward.D has no scipy counterpart: the literal transcription pins it at the largest size too."""
    d = tie_free(1000, 7)
    m1, h1, _ = hr.nn_chain(d, 1000, 4)
    m2, h2, _ = hr.closest_pair(d, 1000, 4)
    assert np.array_equal(m1, m2)
    np.testing.assert_allclose(h1, h2, rtol=1e-13, atol=0)


def tie_laden(kind, n, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "duplicates":         # duplicated cells: zero distances
        x = rng.normal(size=(max(n // 3, 1), 4))
        return pdist(x[rng.integers(0, len(x), size=n)])
    if kind == "integers":
        return rng.integers(1, 6, size=n * (n - 1) // 2).astype(np.float64)
    return np.full(n * (n - 1) // 2, 2.5)    # all equal


@pytest.mark.parametrize("kind", ["duplicates", "integers", "equal"])
@pytest.mark.parametrize("n", [2, 3, 31, 200])
@pytest.mark.parametrize("method", sorted(hr.METHODS))
def test_tie_laden_inputs_give_valid_trees(kind, n, method):
    d = tie_laden(kind, n)
    merge, height, order = hr.nn_chain(d, n, hr.METHODS[method])
    hr.check_tree(d, n, hr.METHODS[method], merge, height, order)


def test_reference_trees_from_the_example_object():
    """`@tumor_subclusters$hc$tumor` / `$normal` of data/infercnv_object_example.rda: ward.D2 on the euclidean distances
    of the pre-denoise smooth block, the group's cells in list order."""
    from oracle import oracle as orc
    z = np.load(os.path.join(GOLD, "example_object.npz"))
    h = np.load(os.path.join(GOLD, "example_hclust.npz"))
    counts = z["counts"].astype(np.float64)
    cs, cl = orc.chr_ranges(z["chr_codes"])
    refs = [z["ref_idx"][z["ref_off"][k]:z["ref_off"][k + 1]] - 1 for k in range(len(z["ref_off"]) - 1)]
    X = orc.smooth_block(orc.normalize_by_seq_depth(counts), cs, cl, refs)
    for name, idx in (("tumor", z["obs_idx"] - 1), ("normal", z["ref_idx"] - 1)):
        assert np.array_equal(h[f"{name}_cols"], idx)
        d = pdist(X[:, idx].T)
        merge, height, order = hr.nn_chain(d, len(idx), 7)
        assert np.array_equal(merge, h[f"{name}_merge"]), name
        assert np.array_equal(order, h[f"{name}_order"]), name
        np.testing.assert_allclose(height, h[f"{name}_height"], rtol=1e-13, atol=0)
    # the merge the reference stores, in R's convention
    assert h["tumor_merge"].tolist() == [[-6, -10], [-1, -3], [-2, -4], [-5, 3], [-9, 4], [1, 5], [-8, 2], [-7, 6], [7, 8]]
    assert h["tumor_order"].tolist() == [8, 1, 3, 7, 6, 10, 9, 5, 2, 4]


@pytest.mark.parametrize("n", [2, 3, 10, 500])
def test_host_order_matches_hcass2(n):
    """icnv_hclust_order (host code of the library, no GPU) against R's hcass2 loop."""
    from infercnv_b200 import api
    for method in (0, 7):
        merge, _, _ = hr.nn_chain(tie_free(n, 3 * n), n, method)
        assert np.array_equal(api.hclust_order(merge), hr.hcass2_order(merge, n))


def test_host_order_rejects_a_merge_that_is_not_a_tree():
    from infercnv_b200 import api
    from infercnv_b200._lib import InfercnvB200Error
    with pytest.raises(InfercnvB200Error):
        api.hclust_order(np.array([[-1, -2], [1, 1]], dtype=np.int32))
