"""TEST INFRASTRUCTURE: smooth_by_chromosome_coordinates (R/inferCNV_ops.R:2534-2622) restated for the tests of K16.

* helper_exact: a literal transcription of .smooth_helper_by_coordinates for one chromosome and one cell in exact rationals
  (R's 0.1 is the double 0.1), with R's recycling of the weights where `around` has holes.  Small cases only.
* stencil / smooth_ld: the same rule vectorised with R's arithmetic - weights and products in float64, the numerator and
  sum(w) as sequential long-double sums (np.cumsum; np.sum would be pairwise), rounded to double, then one double division.
  On x86-64 NumPy's longdouble is R's LDOUBLE, so smooth_ld is R's result bit for bit.
* check_coordinates: enforces the bound of include/infercnv_b200.h on a result against smooth_ld and returns the share of
  outputs bit-identical to it.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

U = 2.0 ** -53     # double
ULD = 2.0 ** -64   # x87 long double


def gamma(n, u):
    n = np.asarray(n, dtype=np.float64)
    return n * u / (1.0 - n * u)


def helper_exact(obs, start, stop, W, rows=None):
    """.smooth_helper_by_coordinates(obs, W, genes) line by line (0-based), every value a Fraction.  Returns the smoothed
    column and, per gene, (lo, L, Lw): the band's first gene, its length and the number of weights before recycling.
    rows: compute only these genes (the others stay copies with shape None)."""
    F = Fraction
    n = len(obs)
    s, e, Wf, x = [F(v) for v in start], [F(v) for v in stop], F(W), [F(v) for v in obs]
    out, shape = list(x), [None] * n
    for i in range(n) if rows is None else rows:
        pos = (s[i] + e[i]) / 2
        around = [j for j in range(n) if s[j] > pos - Wf and e[j] < pos + Wf]
        if len(around) == 0:
            around = [i]
        w = [1 - abs((e[j] + s[j]) / 2 - pos) / Wf for j in around]
        to_add = len(around) // 2                       # floor(length(around - 10) / 2)
        lo, hi = max(0, min(around) - to_add), min(n - 1, max(around) + to_add)
        w = [F(0.1)] * (min(around) - lo) + w + [F(0.1)] * (hi - max(around))
        idx = range(lo, hi + 1)
        out[i] = sum(x[k] * w[(k - lo) % len(w)] for k in idx) / sum(w)   # R's `*` recycles w
        shape[i] = (lo, hi - lo + 1, len(w))
    return out, shape


def stencil_row(s, e, W, i):
    """Row i of one chromosome (coordinates s, e as float64) in R's double arithmetic: (lo, L, wv)."""
    n = len(s)
    pos = (s[i] + e[i]) / 2
    a = np.flatnonzero((s > pos - W) & (e < pos + W))
    if a.size == 0:
        a = np.array([i])
    w = 1 - np.abs((e[a] + s[a]) / 2 - pos) / W
    to_add = len(a) // 2
    lo, hi = max(0, int(a[0]) - to_add), min(n - 1, int(a[-1]) + to_add)
    wv = np.concatenate([np.full(int(a[0]) - lo, 0.1), w, np.full(hi - int(a[-1]), 0.1)])
    return lo, hi - lo + 1, wv


def stencil(G, chr_start, chr_len, gene_start, gene_stop, W):
    """Per row of [0, G): (lo, L, wv) with lo global; a copied row is (i, 1, [1.0])."""
    rows = [(i, 1, np.ones(1)) for i in range(G)]
    s_all, e_all = np.asarray(gene_start, np.float64), np.asarray(gene_stop, np.float64)
    for s0, n in zip(chr_start, chr_len):
        if n < 2 or W < 2:
            continue
        s, e = s_all[s0:s0 + n], e_all[s0:s0 + n]
        for i in range(n):
            lo, L, wv = stencil_row(s, e, W, i)
            rows[s0 + i] = (s0 + lo, L, wv)
    return rows


def smooth_ld(X, chr_start, chr_len, gene_start, gene_stop, W, rows=None):
    """R's arithmetic on the genes x cells matrix X: Y (float64) and, per output, the long-double numerator S, the
    long-double sum A of |products|, den and the band length L (all (G, C) but den / L, which are (G,))."""
    X = np.asarray(X, dtype=np.float64)
    G, C = X.shape
    if rows is None:
        rows = stencil(G, chr_start, chr_len, gene_start, gene_stop, W)
    S = np.empty((G, C), np.longdouble)
    A = np.empty((G, C), np.longdouble)
    den = np.empty(G)
    L = np.empty(G, np.int64)
    for i, (lo, n, wv) in enumerate(rows):
        t = X[lo:lo + n] * np.resize(wv, n)[:, None]                 # R's `*`, recycling wv
        S[i] = np.cumsum(t.astype(np.longdouble), axis=0)[-1]
        A[i] = np.cumsum(np.abs(t).astype(np.longdouble), axis=0)[-1]
        den[i] = np.float64(np.cumsum(wv.astype(np.longdouble))[-1])
        L[i] = n
    Y = S.astype(np.float64) / den[:, None]
    return Y, S, A, den, L


def synthetic_coordinates(G, seed, golden_dir):
    """G genes over the example's chromosomes in its proportions, each chromosome over the example's genomic span with
    sorted uniform starts and lengths drawn from the example's gene lengths: (gene_start, gene_stop, chr_start, chr_len)."""
    import os
    z = np.load(os.path.join(golden_dir, "cnv_regions_fixture.npz"), allow_pickle=True)
    codes, st, sp = np.asarray(z["chr_codes"]), z["gene_start"].astype(np.float64), z["gene_stop"].astype(np.float64)
    change = np.flatnonzero(codes[1:] != codes[:-1]) + 1
    fs = np.concatenate([[0], change])
    fl = np.diff(np.concatenate([fs, [len(codes)]]))
    want = fl / fl.sum() * G
    cl = np.floor(want).astype(np.int64)
    cl[np.argsort(cl - want)[: G - cl.sum()]] += 1             # largest remainders
    rng = np.random.default_rng(seed)
    lengths = sp - st
    starts, stops = [], []
    for s0, n0, n in zip(fs, fl, cl):
        lo, hi = st[s0:s0 + n0].min(), sp[s0:s0 + n0].max()
        s = np.sort(np.floor(rng.uniform(lo, hi, n)))
        starts.append(s)
        stops.append(s + rng.choice(lengths, n))
    cs = np.concatenate([[0], np.cumsum(cl)[:-1]])
    return np.concatenate(starts), np.concatenate(stops), cs.astype(np.int32), cl.astype(np.int32)


def check_coordinates(Y, X, chr_start, chr_len, gene_start, gene_stop, W, ref=None) -> float:
    """|Y - Y_R| within the sum of the header's two bounds (GPU and R against S / den), with |S| bounded from the
    long-double S; returns the share of outputs bit-identical to Y_R."""
    Y_R, S, A, den, L = ref if ref is not None else smooth_ld(X, chr_start, chr_len, gene_start, gene_stop, W)
    Y = np.asarray(Y, dtype=np.float64)
    assert Y.shape == Y_R.shape
    n1 = np.maximum(L - 1, 0)[:, None]
    g2, gl = gamma(n1, U) ** 2, gamma(n1, ULD)
    A64 = A.astype(np.float64)
    S_up = np.abs(S.astype(np.float64)) * (1 + 2 * U) + gl * A64 * 1.01   # >= |S|: S_ld is within gl A of it
    tol = (2 * (2 * U + U * U) * S_up + ((1 + U) * g2 + (1 + U) ** 2 * gl) * A64) / den[:, None]
    tol = tol * (1 + 1e-9) + 2.0 ** -1074
    err = np.abs(Y - Y_R)
    bad = ~(err <= tol)
    assert not bad.any(), (f"{int(bad.sum())} outputs outside the bound; worst at {np.unravel_index(np.argmax(err - tol), err.shape)}: "
                           f"|dY| = {err.max():.3e}")
    return float(np.mean(Y == Y_R))
