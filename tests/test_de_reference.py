"""CPU pins of tests/de_reference.py, the expected values of the non-DE mask (tests/test_gpu_de_mask.py): R's Wilcoxon,
Welch and BH rules against scipy, the exact null against enumeration, the mask rules on hand cases, and the generator."""
import numpy as np
import pytest
from scipy import stats

from tests import de_reference as dr


def rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


@pytest.mark.parametrize("nx,ny", [(1, 1), (1, 7), (3, 5), (12, 9), (49, 49), (49, 50), (50, 49), (51, 51), (200, 30)])
@pytest.mark.parametrize("ties", [False, True])
def test_wilcoxon_matches_mannwhitneyu(nx, ny, ties):
    rng = np.random.default_rng(nx * 100 + ny + ties)
    x, y = rng.normal(size=nx) + 0.3, rng.normal(size=ny)
    if ties:
        x, y = np.round(x * 2) / 2, np.round(y * 2) / 2
    exact = nx < 50 and ny < 50 and len(np.unique(np.concatenate([x, y]))) == nx + ny
    want = stats.mannwhitneyu(x, y, alternative="two-sided", use_continuity=True,
                              method="exact" if exact else "asymptotic").pvalue
    assert rel(dr.wilcox_p(x, y), want) < 1e-12


def test_exact_null_against_enumeration():
    for m in range(1, 7):
        for n in range(1, 7):
            assert dr.rank_sum_counts(m, n) == dr.brute_force_counts(m, n)


def test_all_tied_wilcoxon_is_nan():
    assert np.isnan(dr.wilcox_p(np.ones(60), np.ones(70)))


@pytest.mark.parametrize("nx,ny", [(2, 2), (5, 40), (300, 17)])
def test_welch_matches_ttest_ind(nx, ny):
    rng = np.random.default_rng(nx + ny)
    x, y = rng.normal(size=nx) * 2 + 0.5, rng.normal(size=ny)
    want = stats.ttest_ind(x, y, equal_var=False).pvalue
    assert rel(dr.welch_p(x, y), want) < 1e-12


def test_welch_na_cases():
    assert np.isnan(dr.welch_p([1.0], [1.0, 2.0, 3.0]))                 # n_x < 2
    assert np.isnan(dr.welch_p([1.0, 2.0, 3.0], [2.0]))                 # n_y < 2
    assert np.isnan(dr.welch_p([5.0, 5.0, 5.0], [5.0, 5.0]))            # essentially constant
    assert np.isnan(dr.welch_p([5.0, 5.0, 5.0], [4.0, 4.0]))
    assert not np.isnan(dr.welch_p([5.0, 5.0, 5.0], [4.0, 4.1]))


def test_bh_matches_false_discovery_control_and_keeps_na():
    rng = np.random.default_rng(3)
    p = rng.uniform(size=500) ** 3
    p[::7] = p[3]                                                          # ties
    assert np.allclose(dr.bh(p), stats.false_discovery_control(p), rtol=1e-15, atol=0)
    q = p.copy()
    q[[5, 9, 100]] = np.nan
    got = dr.bh(q)
    assert np.isnan(got[[5, 9, 100]]).all()
    ok = ~np.isnan(q)
    assert np.allclose(got[ok], stats.false_discovery_control(q[ok]), rtol=1e-15, atol=0)   # n = the non-NA count


def test_de_counts_include_na():
    A = np.array([[0.01, np.nan], [np.nan, 0.2], [0.04, 0.01]])
    assert dr.de_counts(A, 0.05) == [(3, 3), (2, 3)]


def _mask(n_ref, subs, pde, rule, C=12):
    """Hand case: genes 0 .. 2, reference groups of columns [0], [1], [2] (first n_ref of them), DE pattern pde[s][j]."""
    G = 3
    X = np.arange(G * C, dtype=np.float64).reshape(G, C, order="F") + 1
    refs = [[0], [1], [2]][:n_ref]
    A = np.full((G, len(subs) * n_ref), 0.5)
    for s in range(len(subs)):
        for j in range(n_ref):
            A[:, s * n_ref + j] = np.where(np.asarray(pde[s][j]), 0.01, 0.5)
    return X, dr.mask_from_padj(X, refs, subs, A, 0.05, rule, -1.0)


def test_mask_rules_by_hand():
    big = list(range(3, 9))               # six cells
    small = [9, 10]                       # two cells: untested -> n_ref
    # one reference group
    X, Y = _mask(1, [big, small], [[[1, 0, 0]], [[0, 0, 0]]], "any")
    assert (Y[:, [0] + small] == X[:, [0] + small]).all()       # references and small subclusters are kept
    assert (Y[0, big] == X[0, big]).all() and (Y[1:, big] == -1).all()
    assert (Y[:, 11] == -1).all() and (Y[:, [1, 2]] == -1).all()  # cells outside every list (and non-reference 1, 2)
    # two and three reference groups
    for n_ref, rule, pattern, keep in [
        (2, "any", [[1, 0, 0], [0, 1, 0]], [True, True, False]),
        (2, "all", [[1, 1, 0], [1, 0, 0]], [True, False, False]),
        (2, "most", [[1, 0, 0], [0, 0, 0]], [True, False, False]),
        (3, "most", [[1, 1, 0], [1, 0, 0], [0, 1, 0]], [True, True, False]),
        (3, "all", [[1, 1, 1], [1, 1, 0], [1, 1, 1]], [True, True, False]),
        (3, "any", [[0, 0, 0], [0, 0, 1], [0, 0, 0]], [False, False, True]),
    ]:
        X, Y = _mask(n_ref, [big], [pattern], rule)
        for g in range(3):
            assert (Y[g, big] == X[g, big]).all() == keep[g], (n_ref, rule, g)
            assert ((Y[g, big] == -1).all()) == (not keep[g])
        assert (Y[:, :n_ref] == X[:, :n_ref]).all()


@pytest.mark.parametrize("size", [1, 2, 3, 4])
def test_small_subclusters_are_kept_whatever_the_tests(size):
    sub = list(range(3, 3 + size))
    X, Y = _mask(2, [sub], [[[0, 0, 0], [0, 0, 0]]], "all")
    assert (Y[:, sub] == X[:, sub]).all()


def test_unnamed_subcluster_list_is_not_tested():
    subs = {"a": {"a_s1": [3, 4, 5], "a_s2": [6, 7]}, "b": [8, 9, 10]}
    got = dr.tested_subclusters(["a", "b"], subs)
    assert [n for n, _ in got] == ["a_s1", "a_s2"]


def test_generator_uniforms_and_law():
    u0, u1 = dr.uniforms(7, 3, 11, np.arange(1000))
    assert (u0 > 0).all() and (u0 <= 1).all() and (u1 > 0).all() and (u1 <= 1).all()
    z = np.concatenate([dr.normals(2024, a, g, 10000) for a in range(10) for g in range(10)])
    assert z.size == 10 ** 6
    assert stats.kstest(z, "norm").pvalue > 1e-3
    j = np.concatenate([dr.jittered(np.zeros(10000), 5, a, 0, 1e-4, 1e-4) for a in range(10)])
    assert stats.kstest(j, stats.norm(loc=1e-4, scale=1e-4).cdf).pvalue > 1e-3
    # no correlation across keys: groups, genes, positions, the reference / subcluster sides
    a = dr.normals(1, 0, 0, 100000)
    for b in (dr.normals(1, 1, 0, 100000), dr.normals(1, 0, 1, 100000), dr.normals(1, dr.SUB_KEY, 0, 100000),
              dr.normals(2, 0, 0, 100000), np.roll(a, 1)):
        assert abs(np.corrcoef(a, b)[0, 1]) < 0.015


def test_sd_zero_keeps_every_tie():
    x = np.array([1.0, 1.0, 2.0])
    assert np.array_equal(dr.jittered(x, 1, 0, 0, 1e-4, 0.0), x + 1e-4)
