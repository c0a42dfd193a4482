"""The two routes to the per-cell median of the fused cell pipeline, each taken on purpose.

The histogram of the smoothed column is counted while stage B stores it, in bins placed from the mean and the standard
deviation of the stage-A output x' (infercnv_b200/csrc/icnv_smooth.cu, hist_geometry).  That placement is an estimate: the
bracketing selection takes over whenever it fails.  The columns here make it fail in each possible way, next to columns for
which it holds, and the route every cell took is read back from the library's counters (icnv_debug_stats), so a case that
stops reaching its route fails instead of passing for the wrong reason:
  * the middle ranks outside the span: more than half of the column is an exact 0 and the rest lies far above it;
  * more than CAND_MAX = 64 values in the middle bin: a few huge outliers widen the bins until one holds the column, or more
    than half of the column is one tied value (whole chromosomes of zeros, which the prefix sums smooth to exact zeros);
  * no variance: a constant column;
  * even and odd gene counts (bulk copy / element-wise load, the +inf pad of the odd column).
Every variant of the kernel must stay within the error bound of tests/cellpipe_reference.py and bit-identical to the variants
that share its slice partition (the sweep of tests/test_gpu_cell_pipeline_variants.py).  Runs on an H100 (-m gpu) and under
the host emulation.
"""
import ctypes as ct

import numpy as np
import pytest

from infercnv_b200 import _lib
from tests import cellpipe_reference as cref
from tests import test_gpu_cell_pipeline_variants as var

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not cref.HAS_EXTENDED, reason="np.longdouble is not an extended type here")]

api = var.api   # the module-scoped fixture that initialises the library

LENS = {"even": [700, 1, 640, 501, 202, 900, 98], "odd": [700, 1, 640, 501, 202, 900, 99]}
RAW = dict(window=101, center=1)   # no log, no dead band: the column itself is x'


def _stats():
    """(medians, by the histogram, by the bracketing selection: split exit, gather exit); the counters are reset"""
    out = (ct.c_ulonglong * 16)()
    fn = _lib.load().icnv_debug_stats
    fn.restype, fn.argtypes = ct.c_int, [ct.c_void_p, ct.c_int]
    assert fn(out, 1) == 0
    return int(out[1]), int(out[10]), int(out[2]), int(out[3])


def _columns(rng, cl, kind, C=3):
    G = int(cl.sum())
    cs = np.concatenate([[0], np.cumsum(cl)[:-1]])
    X = rng.normal(0.0, 1.0, size=(C, G))
    if kind == "one_sided":      # chromosomes 0 .. 3 (six genes in ten) are 0, the rest lies around 10
        X = 10.0 + 3.0 * X
        X[:, :cs[4]] = 0.0
    elif kind == "outliers":     # sd(x') ~ 1e7: every smoothed value of the bulk falls into one bin
        X[:, rng.choice(G, size=5, replace=False)] = 1e9
    elif kind == "ties":         # the same zeros inside noise that straddles them: the median is one of > G / 2 equal values
        X[:, :cs[4]] = 0.0
    elif kind == "constant":
        X[:] = 0.375
    else:
        assert kind == "plain"
    return X


@pytest.mark.parametrize("parity", sorted(LENS))
@pytest.mark.parametrize("kind", ["plain", "one_sided", "outliers", "ties", "constant"])
def test_median_route(api, monkeypatch, kind, parity):
    rng = np.random.default_rng({"even": 21, "odd": 22}[parity])
    cs, cl = var._layout(LENS[parity])
    X = _columns(rng, cl, kind)
    assert X.shape[1] % 2 == (parity == "odd")
    case = var.Case(f"{kind} {parity}", cs, cl, X, RAW)
    try:
        for env in ({}, {"ICNV_CELL_KERNEL": "4"}):   # the two-buffer and the single-buffer kernel
            var._configure(api, monkeypatch, env)
            _stats()
            rc, _, flag, sel = case.run()
            medians, by_hist, split, gather = _stats()
            assert rc == 0 and flag == 0 and sel[0] == (4 if env else 3) and medians == X.shape[0], (rc, flag, sel, medians)
            assert split + gather == medians - by_hist, (medians, by_hist, split, gather)
            assert by_hist == (medians if kind == "plain" else 0), f"{case.name} {sel}: {by_hist} of {medians} medians by the histogram"
    finally:
        var._configure(api, monkeypatch, {})
    # the same columns through the whole pipeline's stages as well (log, dead band, clamp, second dead band, 2^x): whichever
    # route a cell takes there, every variant agrees with the reference
    Xp = np.abs(X)
    sweep = [case, var.Case(f"{kind} {parity} pass2", cs, cl, Xp, var._opts(rng, Xp))]
    var.sweep(api, monkeypatch, sweep)
