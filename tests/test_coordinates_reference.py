"""CPU pins of tests/coordinates_reference.py: the vectorised R-arithmetic restatement of smooth_by_chromosome_coordinates
against the literal transcription of the R helper in exact rationals, on hand-built gene layouts (each one checked to
contain the case it is named for) and on the bundled example's gene coordinates."""
import os

import numpy as np
import pytest

from tests import coordinates_reference as cr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def layout(case):
    """(gene_start, gene_stop, chr_start, chr_len, W) for a named case."""
    if case == "empty_window":          # genes longer than 2 W: no gene in its own window
        st, sp, W = [0, 50, 120, 300], [100, 200, 130, 900], 10.0
    elif case == "hole_non_multiple":   # gene 2 reaches past pos + W for gene 1: around = {0, 1, 3, 4}, L = 5, Lw = 4
        st, sp, W = [0, 10, 20, 30, 40], [5, 15, 1000, 35, 45], 50.0
    elif case == "hole_multiple":       # row 0: around = {0, 3}, lo = 0, hi = 3: L = 4, Lw = 2
        st, sp, W = [0, 3, 4, 6], [2, 500, 600, 8], 20.0
    elif case == "w_below_2":
        st, sp, W = [0, 10, 20, 30], [5, 15, 25, 35], 1.5
    elif case == "one_gene_chromosome":
        st, sp, W = [0, 10, 20, 30, 40, 50], [5, 15, 25, 35, 45, 55], 12.0
        return np.array(st, float), np.array(sp, float), [0, 1, 5], [1, 4, 1], W
    elif case == "window_wider_than_chromosome":
        st, sp, W = list(range(0, 90, 10)), list(range(4, 94, 10)), 1e9
    elif case == "non_integer_window":
        st, sp, W = list(range(0, 120, 10)), list(range(6, 126, 10)), 23.7
    elif case == "unsorted_starts":
        rng = np.random.default_rng(5)
        st = rng.permutation(np.arange(0, 200, 10)).tolist()
        sp = [s + int(rng.integers(1, 40)) for s in st]
        W = 30.0
    else:
        raise KeyError(case)
    n = len(st)
    return np.array(st, float), np.array(sp, float), [0], [n], W


def features(st, sp, cs, cl, W):
    """Which of the cases the layout's stencil exhibits."""
    f = set()
    for s0, n in zip(cs, cl):
        if n < 2:
            f.add("one_gene_chromosome")
            continue
        if W < 2:
            f.add("w_below_2")
            continue
        s, e = st[s0:s0 + n], sp[s0:s0 + n]
        for i in range(n):
            pos = (s[i] + e[i]) / 2
            a = np.flatnonzero((s > pos - W) & (e < pos + W))
            if a.size == 0:
                f.add("empty_window")
                continue
            _, L, wv = cr.stencil_row(s, e, W, i)
            if L > len(wv):
                f.add("hole_multiple" if L % len(wv) == 0 else "hole_non_multiple")
            if a.size == n:
                f.add("window_wider_than_chromosome")
        if np.any(np.diff(s) < 0):
            f.add("unsorted_starts")
    if W != np.floor(W):
        f.add("non_integer_window")
    return f


def assert_pinned(X, cs, cl, st, sp, W, exact_rows=None):
    """smooth_ld within 8 u (sum |x| + Lw |y|) / den + 4 u |y| of the exact rationals (the weights are rounded doubles in
    R: at most 2 u off each), and the same bands; exact_rows: the global rows to transcribe (default all)."""
    Y, _, _, den, L = cr.smooth_ld(X, cs, cl, st, sp, W)
    rows = cr.stencil(X.shape[0], cs, cl, st, sp, W)
    for s0, n in zip(cs, cl):
        if n < 2 or W < 2:
            assert np.array_equal(Y[s0:s0 + n], X[s0:s0 + n])
            continue
        pick = range(n) if exact_rows is None else [i for i in range(n) if s0 + i in exact_rows]
        for c in range(X.shape[1]):
            col, shape = cr.helper_exact(X[s0:s0 + n, c], st[s0:s0 + n], sp[s0:s0 + n], W, pick)
            for i in pick:
                y_ex, sh = col[i], shape[i]
                lo, Lr, wv = rows[s0 + i]
                assert (lo - s0, Lr, len(wv)) == sh
                ye = float(y_ex)
                xs = np.abs(X[lo:lo + Lr, c]).sum()
                tol = 8 * cr.U * (xs + len(wv) * abs(ye)) / den[s0 + i] + 4 * cr.U * abs(ye) + 2.0 ** -1074
                assert abs(Y[s0 + i, c] - ye) <= tol, (s0 + i, c, Y[s0 + i, c], ye)


CASES = ["empty_window", "hole_non_multiple", "hole_multiple", "w_below_2", "one_gene_chromosome",
         "window_wider_than_chromosome", "non_integer_window", "unsorted_starts"]


@pytest.mark.parametrize("case", CASES)
def test_restatement_matches_the_exact_transcription(case):
    st, sp, cs, cl, W = layout(case)
    assert case in features(st, sp, cs, cl, W)
    rng = np.random.default_rng(len(case))
    X = rng.normal(size=(len(st), 4)) * np.array([1.0, 1e3, 1e-3, 1.0]) + np.array([0.0, 0.0, 0.0, 5.0])
    assert_pinned(X, cs, cl, st, sp, W)


def test_exact_transcription_recycles_like_r():
    """hole_non_multiple by hand: row 1 has around = {0, 1, 3, 4}, so x[0..4] meets the weights w0 w1 w3 w4 w0."""
    from fractions import Fraction as F
    st, sp, _, _, W = layout("hole_non_multiple")
    x = [1.0, 2.0, 4.0, 8.0, 16.0]
    col, shape = cr.helper_exact(x, st, sp, W)
    pos = F(25, 2)
    w = [1 - abs((F(sp[j]) + F(st[j])) / 2 - pos) / F(W) for j in (0, 1, 3, 4)]
    assert shape[1] == (0, 5, 4)
    assert col[1] == (1 * w[0] + 2 * w[1] + 4 * w[2] + 8 * w[3] + 16 * w[0]) / sum(w)


def fixture():
    z = np.load(os.path.join(GOLDEN, "cnv_regions_fixture.npz"), allow_pickle=True)
    e = np.load(os.path.join(GOLDEN, "example_object.npz"), allow_pickle=True)
    assert np.array_equal(z["chr_codes"], e["chr_codes"])
    X = np.log2(np.asarray(e["expr"], np.float64) + 1)
    X = X - X.mean(axis=1, keepdims=True)             # signed values, as at step 10
    st, sp = z["gene_start"].astype(np.float64), z["gene_stop"].astype(np.float64)
    assert X.shape[0] == len(st) == len(sp) == 4613
    codes = np.asarray(z["chr_codes"])
    change = np.flatnonzero(codes[1:] != codes[:-1]) + 1
    cs = np.concatenate([[0], change])
    cl = np.diff(np.concatenate([cs, [len(codes)]]))
    return X, st, sp, cs.tolist(), cl.tolist()


# rows with holes and empty windows of the example's gene order, counted independently of the restatement
FIXTURE_COUNTS = {1e7: (14, 0), 1e6: (None, None), 1e5: (17, 285), 2e4: (None, 1986)}


@pytest.mark.parametrize("W", [1e7, 1e6, 1e5, 2e4])
def test_restatement_on_the_example_coordinates(W):
    X, st, sp, cs, cl = fixture()
    holes = empty = 0
    rows = set(range(0, len(st), 97))   # a sample of rows plus every row with a hole goes through the exact helper
    for s0, n in zip(cs, cl):
        if n < 2:
            continue
        s, e = st[s0:s0 + n], sp[s0:s0 + n]
        for i in range(n):
            pos = (s[i] + e[i]) / 2
            empty += not np.any((s > pos - W) & (e < pos + W))
            _, L, wv = cr.stencil_row(s, e, W, i)
            if L > len(wv):
                holes += 1
                rows.add(s0 + i)
    want_holes, want_empty = FIXTURE_COUNTS[W]
    assert want_holes is None or holes == want_holes
    assert want_empty is None or empty == want_empty
    assert_pinned(X[:, :3], cs, cl, st, sp, W, exact_rows=rows)
