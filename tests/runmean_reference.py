"""TEST INFRASTRUCTURE: restatements of the running mean and of the random-trees permutations (icnv_random_trees.cu).

* runmean_ld: caTools::runmean(x, k) (endrule "mean", align "center") per column range, window sums in long double, with
  the error bound the kernel promises widened by this restatement's own error; check_runmean enforces it.
* catools_transcription: caTools' running-sum algorithm written out literally - sum of the first window, the left edge
  growing, the running sum, the right edge shrinking - in exact rational arithmetic, for small pinning cases.
* hash3 / permutations: the splitmix generator of the kernels (icnv_common.cuh; oracle/infercnv_oracle.c's syn_hash3) in
  NumPy uint64 arithmetic, the permutation of every gene it defines, and the permuted clade matrix of a member.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

U = 2.0 ** -53
U_LD = float(np.finfo(np.longdouble).eps) / 2


def window(p: int, L: int, k: int) -> tuple[int, int]:
    """Inclusive window [a, b] of position p in a range of L genes."""
    kk = min(k, L)
    k2 = kk // 2
    k1 = kk - 1 - k2
    return max(0, p - k1), min(L - 1, p + k2)


def _ranges(G, chr_start, chr_len):
    if chr_start is None:
        return [(0, G)]
    return [(int(s), int(l)) for s, l in zip(chr_start, chr_len)]


def runmean_ld(X, k, chr_start=None, chr_len=None):
    """(mean, bound): the long-double window means of every column range and the kernel's error bound around them,
    widened by this restatement's own error.  Copied genes have a zero bound."""
    X = np.asarray(X, dtype=np.float64)
    if X.ndim == 1:
        X = X[:, None]
    G, C = X.shape
    out = X.astype(np.longdouble).copy()
    tol = np.zeros((G, C))
    for s, L in _ranges(G, chr_start, chr_len):
        if k <= 1 or L < 2:
            continue
        x = X[s:s + L].astype(np.longdouble)
        ax = np.abs(x)
        kk = min(k, L)
        k2 = kk // 2
        k1 = kk - 1 - k2
        pad = np.zeros((L + kk - 1, C), dtype=np.longdouble)
        pad[k1:k1 + L] = x
        apad = np.zeros_like(pad)
        apad[k1:k1 + L] = ax
        win = np.lib.stride_tricks.sliding_window_view(pad, kk, axis=0)   # (L, C, kk): window of p = pad[p .. p + kk)
        awin = np.lib.stride_tricks.sliding_window_view(apad, kk, axis=0)
        sums = win.sum(axis=-1)
        asums = awin.sum(axis=-1)
        cnt = np.array([window(p, L, k)[1] - window(p, L, k)[0] + 1 for p in range(L)], dtype=np.float64)[:, None]
        mean = sums / cnt
        out[s:s + L] = mean
        T = ax.sum(axis=0).astype(np.float64)[None, :]
        kernel = 2 * U * np.abs(mean.astype(np.float64)) + 8 * L * U * U * T / cnt
        own = (kk + 2) * U_LD * asums.astype(np.float64) / cnt      # long-double summation and division
        tol[s:s + L] = kernel + own + np.finfo(np.float64).tiny
    return out, tol


def check_runmean(Y, X, k, chr_start=None, chr_len=None):
    """Assert the kernel's output Y is within the bound of the restatement; return the worst error / bound ratio."""
    ref, tol = runmean_ld(X, k, chr_start, chr_len)
    Y = np.asarray(Y, dtype=np.float64).reshape(ref.shape)
    err = np.abs(Y.astype(np.longdouble) - ref).astype(np.float64)
    bad = err > tol
    assert not bad.any(), f"{int(bad.sum())} values outside the bound, worst {float((err / tol).max()):.3g} x the bound"
    return float(np.max(np.divide(err, tol, out=np.zeros_like(err), where=tol > 0))) if err.size else 0.0


def catools_transcription(x, k):
    """caTools' running mean (endrule "mean", align "center") as its four steps, in exact rationals."""
    x = [Fraction(float(v)) for v in x]
    n = len(x)
    if k <= 1 or n < 2:
        return [float(v) for v in x]
    k = min(k, n)
    k2 = k // 2
    k1 = k - 1 - k2
    y = [Fraction(0)] * n
    s = sum(x[:k2 + 1], Fraction(0))          # 1. the first window, [0, k2]
    cnt = k2 + 1
    p = 0
    y[0] = s / cnt
    while p + 1 <= k1 and p + 1 < n:           # 2. left edge: the window grows to the right
        p += 1
        if p + k2 < n:
            s += x[p + k2]
            cnt += 1
        y[p] = s / cnt
    while p + 1 < n and p + 1 + k2 < n:        # 3. running sum: one value in, one out
        p += 1
        s += x[p + k2] - x[p - k1 - 1]
        y[p] = s / cnt
    while p + 1 < n:                           # 4. right edge: the window shrinks from the left
        p += 1
        s -= x[p - k1 - 1]
        cnt -= 1
        y[p] = s / cnt
    return [float(v) for v in y]


# ---- the generator ---------------------------------------------------------------------------------------------------
def mix64(z):
    with np.errstate(over="ignore"):
        z = np.asarray(z, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def hash3(seed, a, b, c):
    with np.errstate(over="ignore"):
        s = mix64(np.uint64(seed) ^ np.uint64(0x243F6A8885A308D3))
        h = mix64(s + np.asarray(a, dtype=np.uint64)) * np.uint64(0x9FB21C651E98DF25) + np.asarray(b, dtype=np.uint64)
        return mix64(h) ^ mix64(np.asarray(c, dtype=np.uint64) + np.uint64(0x13198A2E03707344))


def perm_key(seed, p, g, i):
    """key(p, g, i) = mix64(hash3(seed, p, g, i)).  hash3's last argument enters through an XOR only, so its raw values
    order the positions of one (p, g) in just a few ways (8 of the 24 orders of 4); the final mix64 spreads them."""
    return mix64(hash3(seed, p, g, i))


def permutations(seed, p, G, n):
    """pi[g] (G x n): the stable ascending argsort of key(p, g, i) over the list positions i."""
    g = np.arange(G, dtype=np.uint64)[:, None]
    i = np.arange(n, dtype=np.uint64)[None, :]
    keys = perm_key(seed, np.uint64(p), g, i)
    return np.argsort(keys, axis=1, kind="stable")


def permuted(Xc, seed, p):
    """The clade matrix (genes x n, columns in list order) of permutation p: X_p[g, i] = Xc[g, pi_{p,g}(i)]."""
    G, n = Xc.shape
    pi = permutations(seed, p, G, n)
    return np.take_along_axis(Xc, pi, axis=1)
