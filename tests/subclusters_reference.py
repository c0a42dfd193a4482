"""TEST INFRASTRUCTURE: reference restatements for the subclustering trees of define_signif_tumor_subclusters
(R/inferCNV_tumor_subclusters.R:2-260) and their kernels (icnv_subclusters.cu).

* ``zscores`` is the filter's element-wise step, |(x - mu) / sigma|, one IEEE rounding per operation as R evaluates it.
* ``row_mean_exact`` is the mean of each row in exact rationals, rounded once to double: what the kernel returns.
* ``row_mean_r`` is R's mean() as summary.c computes it: a long-double sum divided by n, then s += sum(x - s) / n, rounded to
  double.  On x86-64 NumPy's longdouble is R's LDOUBLE, so this is R's result bit for bit.
* ``outlier_mask`` is the filter, `apply(abs(z), 1, mean) >= 0.8`, with R's non-finite rules (a NaN mean fails, +Inf passes).
* ``cutree`` restates stats::cutree(tree, k = , h = ): merges with height <= h are applied (k = n - their number), and groups
  are numbered by first appearance in observation order.
* ``assemble`` restates .single_tumor_subclustering's naming loop: tumor_group_idx[hc$order] cut into consecutive runs whose
  lengths are the group sizes of split(grps, grps) in group-id order, named "<group>_s<id>".
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

LD = np.longdouble
HAS_EXTENDED = float(np.finfo(np.longdouble).eps) <= 1e-18


def zscores(X, cells, mu: float, sigma: float) -> np.ndarray:
    ref = np.asarray(X, dtype=np.float64)[:, np.asarray(cells)]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.abs((ref - mu) / sigma)


def _special(row):
    """(NaN in the row, +Inf in the row)"""
    return bool(np.isnan(row).any()), bool(np.isposinf(row).any())


def row_mean_exact(Z) -> np.ndarray:
    out = np.empty(Z.shape[0])
    for g, row in enumerate(Z):
        nan, inf = _special(row)
        if nan or inf:
            out[g] = np.nan if nan else np.inf
            continue
        s = sum((Fraction(float(v)) for v in row), Fraction(0))
        out[g] = float(s / len(row))   # Fraction -> float rounds to nearest, ties to even
    return out


def row_mean_r(Z) -> np.ndarray:
    out = np.empty(Z.shape[0])
    for g, row in enumerate(Z):
        x = row.astype(LD)
        s = np.cumsum(x)[-1] / LD(len(row))          # sequential long-double sum (np.sum would be pairwise)
        if np.isfinite(s):
            s = s + np.cumsum(x - s)[-1] / LD(len(row))
        out[g] = np.float64(s)
    return out


def outlier_mask(X, cells, mu: float, sigma: float, mean=row_mean_exact) -> np.ndarray:
    m = mean(zscores(X, cells, mu, sigma))
    with np.errstate(invalid="ignore"):
        return m >= 0.8


def cutree(merge, height, k=None, h=None) -> np.ndarray:
    """stats::cutree for one of k / h: the 1-based group of every observation."""
    merge = np.asarray(merge)
    n = merge.shape[0] + 1
    if h is not None:
        above = np.flatnonzero(np.append(np.asarray(height, dtype=np.float64), np.inf) > h)
        k = n + 1 - (int(above[0]) + 1)                 # which.max(c(height, Inf) > h)
    if k is None or not 1 <= k <= n:
        raise ValueError("cutree: k out of range")
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    node = {}                                          # cluster number s -> a member observation
    for s in range(n - k):
        a, b = (int(v) for v in merge[s])
        x = -a - 1 if a < 0 else node[a]
        y = -b - 1 if b < 0 else node[b]
        parent[find(x)] = find(y)
        node[s + 1] = y
    label, out = {}, np.empty(n, dtype=np.int64)
    for i in range(n):
        r = find(i)
        if r not in label:
            label[r] = len(label) + 1
        out[i] = label[r]
    return out


def assemble(tumor_name: str, tumor_group_idx, order, grps) -> dict:
    idx = np.asarray(tumor_group_idx)
    ordered = idx[np.asarray(order) - 1]
    ids, counts = np.unique(np.asarray(grps), return_counts=True)   # split(grps, grps): levels in increasing order
    out, start = {}, 0
    for g, c in zip(ids.tolist(), counts.tolist()):
        out[f"{tumor_name}_s{g}"] = ordered[start:start + c]
        start += c
    return out


def r_mean(x) -> float:
    return float(row_mean_r(np.asarray(x, dtype=np.float64)[None, :])[0])


def r_sd(x) -> float:
    """sd(x): R's var() (cov.c) - the long-double mean with its refinement, then the long-double sum of squared deviations
    over n - 1."""
    x = np.asarray(x, dtype=np.float64).astype(LD)
    n = len(x)
    m = np.cumsum(x)[-1] / LD(n)
    m = m + np.cumsum(x - m)[-1] / LD(n)
    d = x - m
    return float(np.sqrt(np.float64(np.cumsum(d * d)[-1] / LD(n - 1))))


def cut_height(height, partition_method: str, p_val: float):
    """The cut of .single_tumor_subclustering for pheight / qnorm (None for "none", cutree(k = 1))."""
    from scipy.stats import norm
    height = np.asarray(height, dtype=np.float64)
    if partition_method == "pheight":
        return p_val * float(height.max())
    if partition_method == "qnorm":
        return float(norm.ppf(1 - p_val, loc=r_mean(height), scale=r_sd(height)))
    if partition_method == "none":
        return None
    raise ValueError(partition_method)
