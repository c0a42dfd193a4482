"""CPU checks of the restatements behind the subclustering trees (tests/subclusters_reference.py): R's row mean of the
z-score filter in exact rationals against the long-double two-pass mean, at the 0.8 threshold and on its two quirks, and
cutree / the subcluster assembly against the trees and lists stored in the reference's example object."""
import os
from fractions import Fraction

import numpy as np
import pytest

from tests import hclust_reference as hr
from tests import subclusters_reference as sr

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_exact_and_long_double_row_means_agree():
    rng = np.random.default_rng(0)
    Z = np.abs(rng.normal(size=(200, 37)) * rng.uniform(0.1, 3, size=(200, 1)))
    exact = sr.row_mean_exact(Z)
    assert np.array_equal(exact, [float(sum(Fraction(float(v)) for v in r) / len(r)) for r in Z])
    if sr.HAS_EXTENDED:
        assert np.array_equal(sr.row_mean_r(Z), exact)
    else:
        np.testing.assert_allclose(sr.row_mean_r(Z), exact, rtol=4e-16)


def test_rows_a_few_ulp_from_the_threshold():
    """Constant rows at 0.8 and its neighbours, and pairs whose exact mean is the midpoint between two neighbours (rounded
    to even): the mask flips exactly where the correctly rounded mean reaches 0.8."""
    v = [0.8]
    for _ in range(3):
        v = [np.nextafter(v[0], 0.0)] + v + [np.nextafter(v[-1], 1.0)]
    rows = [np.full(9, x) for x in v] + [np.array([a, b]) for a, b in zip(v[:-1], v[1:])]
    rows += [np.array([a, b, b]) for a, b in zip(v[:-1], v[1:])]
    for r in rows:
        Z = r[None, :]
        m = sr.row_mean_exact(Z)[0]
        assert abs(m - 0.8) <= 4 * np.spacing(0.8)
        want = Fraction(m) >= Fraction(0.8)
        assert sr.outlier_mask(Z, np.arange(Z.shape[1]), 0.0, 1.0)[0] == want
        if sr.HAS_EXTENDED:
            assert sr.row_mean_r(Z)[0] == m
    mid = sr.row_mean_exact(np.array([[0.8, np.nextafter(0.8, 0.0)]]))[0]
    assert mid in (0.8, np.nextafter(0.8, 0.0))


def test_constant_reference_makes_every_mean_nan():
    X = np.full((5, 4), 2.5)
    Z = sr.zscores(X, np.arange(4), 2.5, 0.0)
    assert np.isnan(Z).all() and np.isnan(sr.row_mean_exact(Z)).all()
    assert not sr.outlier_mask(X, np.arange(4), 2.5, 0.0).any()
    # x != mu with sigma = 0: +Inf passes, as R's mean(c(Inf, ...)) >= 0.8 does
    X[2, 1] = 3.0
    assert sr.outlier_mask(X, np.arange(4), 2.5, 0.0).tolist() == [False, False, False, False, False]
    Z = sr.zscores(X, [1], 2.5, 0.0)
    assert sr.outlier_mask(X, [1], 2.5, 0.0).tolist() == [False, False, True, False, False] and np.isinf(Z[2, 0])


def test_no_outlier_keeps_no_gene():
    """which() returns integer(0), and expr.data[-integer(0), ] has no rows: the mirror's gene list is then empty."""
    from mirror import ops  # noqa: F401  (the mirror is importable without a GPU)
    mask = np.zeros(7, dtype=bool)
    out = np.flatnonzero(mask)
    kept = np.delete(np.arange(7), out) if out.size else np.arange(7)[:0]
    assert kept.size == 0


def _example_groups():
    z = np.load(os.path.join(GOLD, "example_object.npz"))
    return {"tumor": z["obs_idx"], "normal": z["ref_idx"]}   # 1-based, list order


def test_assembly_reproduces_the_stored_subclusters():
    """partition_method = "none", z_score_filter = 0 (the stored trees were built without the filter): cutree(k = 1) and the
    naming loop over each stored ward.D2 tree give the stored tumor_s1 / normal_s1 lists."""
    from mirror import ops
    h = np.load(os.path.join(GOLD, "example_hclust.npz"))
    s = np.load(os.path.join(GOLD, "example_subclusters.npz"))
    for g, idx in _example_groups().items():
        assert np.array_equal(h[f"{g}_cols"], idx - 1)
        merge, height, order = h[f"{g}_merge"], h[f"{g}_height"], h[f"{g}_order"]
        grps = sr.cutree(merge, height, k=1)
        assert grps.tolist() == [1] * len(idx)
        subs = sr.assemble(g, idx, order, grps)
        assert list(subs) == s[f"{g}_names"].tolist() == [f"{g}_s1"]
        assert np.array_equal(subs[f"{g}_s1"], s[f"{g}_idx"])
        mine = ops._assemble_subclusters(g, idx, order, ops.cutree(merge, height, k=1))
        assert list(mine) == list(subs) and np.array_equal(mine[f"{g}_s1"], subs[f"{g}_s1"])


def test_cutree_by_height_on_a_small_tree():
    # observations 1..5; merges: (1,2) at 1, (4,5) at 2, (3, m1) at 3, (m2, m3) at 4
    merge = np.array([[-1, -2], [-4, -5], [-3, 1], [2, 3]])
    height = np.array([1.0, 2.0, 3.0, 4.0])
    for cut in (sr.cutree, __import__("mirror.ops", fromlist=["cutree"]).cutree):
        assert cut(merge, height, h=0.5).tolist() == [1, 2, 3, 4, 5]
        assert cut(merge, height, h=1.0).tolist() == [1, 1, 2, 3, 4]      # a merge AT h is applied
        assert cut(merge, height, h=2.5).tolist() == [1, 1, 2, 3, 3]
        assert cut(merge, height, h=3.0).tolist() == [1, 1, 1, 2, 2]
        assert cut(merge, height, h=10.0).tolist() == [1] * 5
        assert cut(merge, height, k=2).tolist() == [1, 1, 1, 2, 2]
    with pytest.raises(ValueError):
        sr.cutree(merge, height, k=6)


@pytest.mark.parametrize("n", [3, 10, 64])
def test_mirror_cutree_equals_the_restatement(n):
    from mirror import ops
    rng = np.random.default_rng(n)
    x = rng.normal(size=(n, 4))
    d = np.array([np.linalg.norm(x[a] - x[b]) for a in range(n) for b in range(a + 1, n)])
    merge, height, order = hr.nn_chain(d, n, 7)
    for k in range(1, n + 1):
        assert np.array_equal(ops.cutree(merge, height, k=k), sr.cutree(merge, height, k=k))
    for h in np.concatenate([height, (height[:-1] + height[1:]) / 2, [0.0, height[-1] * 2]]):
        grps = sr.cutree(merge, height, h=h)
        assert np.array_equal(ops.cutree(merge, height, h=h), grps)
        subs = sr.assemble("g", np.arange(n), order, grps)
        assert np.array_equal(np.concatenate(list(subs.values())), order - 1)
        mine = ops._assemble_subclusters("g", np.arange(n), order, grps)
        assert list(mine) == list(subs)
