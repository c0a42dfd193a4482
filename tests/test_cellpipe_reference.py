"""The checker of tests/test_gpu_cell_pipeline_variants.py, tested on the CPU: the extended-precision reference of the fused cell
pipeline (tests/cellpipe_reference.py) accepts an FP64 prefix-sum implementation of the kernel's arithmetic within its derived
bound, and rejects it once the reference itself is perturbed by one step - a narrower window, one edge denominator, the
adjacent order statistic as the median."""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import cellpipe_reference as cref

pytestmark = pytest.mark.skipif(not cref.HAS_EXTENDED, reason="np.longdouble is not an extended-precision type here")

LENS = np.array([300, 1, 2, 40, 150, 103, 404], dtype=np.int32)   # one / two genes, shorter than the window, long ones
CS = np.concatenate([[0], np.cumsum(LENS)[:-1]]).astype(np.int32)


def _data(seed=3):
    rng = np.random.default_rng(seed)
    G = int(LENS.sum())
    X = rng.gamma(2.0, 1.5, size=(4, G))
    X[rng.random(X.shape) < 0.3] = 0.0
    L = np.log2(X + 1.0)
    lo = np.quantile(L, 0.4, axis=0) - 0.05
    hi = lo + rng.uniform(0.0, 0.3, size=G)
    return X, lo, hi


def _pass2(lo, hi, window=101):
    return dict(apply_log=True, lo1=lo, hi1=hi, threshold=3.0, window=window, center=1, lo2=lo - 1.0, hi2=hi - 1.0,
                apply_exp2=True)


def test_prefix_sum_model_is_inside_the_bound_and_matches_the_oracle():
    X, lo, hi = _data()
    L = int(LENS.max())   # the model sums each chromosome sequentially: one slice per chromosome
    for opts in (_pass2(lo, hi), _pass2(lo, hi, 3), dict(window=51, center=2), dict(apply_log=True, mid1=lo, threshold=2.0,
                                                                                      window=15, center=0, mid2=hi)):
        got = cref.prefix_sum_model(X, CS, LENS, **opts)
        want, bound = cref.cell_pipeline(X, CS, LENS, L=L, NW=1, **opts)
        r = cref.error_ratio(got, want, bound)
        assert r < 0.5, (opts.keys(), r)   # single-gene chromosomes: only stage A / D roundings, the bound is tight there
    # the reference is the oracle's smoothing (the C restatement of the R loops) in other words
    sm, _ = cref.cell_pipeline(X, CS, LENS, window=101)
    np.testing.assert_allclose(sm.astype(np.float64), orc.smooth_by_chromosome(np.asfortranarray(X.T), CS, LENS, 101).T,
                               rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize("perturb", [dict(window_shrink=1), dict(edge_denominator_shift=True), dict(median_shift=1)],
                         ids=["window_one_step_narrower", "edge_denominator_off_by_one", "adjacent_order_statistic"])
def test_the_checker_rejects_a_perturbed_reference(perturb):
    X, lo, hi = _data()
    L = int(LENS.max())
    for window in (101, 3):
        opts = _pass2(lo, hi, window)
        got = cref.prefix_sum_model(X, CS, LENS, **opts)
        want, bound = cref.cell_pipeline(X, CS, LENS, L=L, NW=1, **opts)
        assert cref.error_ratio(got, want, bound) < 0.5
        bad, _ = cref.cell_pipeline(X, CS, LENS, L=L, NW=1, **opts, **perturb)
        assert cref.error_ratio(got, bad, bound) > 1e3, (window, perturb)


def test_zero_bound_means_exact():
    want = np.array([[1.0, 2.0]], dtype=np.longdouble)
    assert cref.error_ratio(np.array([[1.0, 2.0]]), want, np.zeros((1, 2))) == 0.0
    assert cref.error_ratio(np.array([[1.0, np.nextafter(2.0, 3.0)]]), want, np.zeros((1, 2))) == float("inf")
    assert cref.error_ratio(np.array([[1.0, np.nan]]), want, np.ones((1, 2))) == float("inf")
