"""Expected values of K12, the exact k-nearest-neighbour kernel (icnv_dist.cu; RANN::nn2 with the query set = the data set),
in NumPy.

The rule: row i of the result lists the k nearest list positions of position i, itself included, ordered by squared
distance and then by position - `np.lexsort((positions, squared distances))`, first k.  The helper takes full distance
rows, either from K10's "dist" vector (the GPU's own sums, rooted: the kernel reports those very bits) or from NumPy.  A
root orders as its squared sum does, except where two different sums share a root, which random and integer-valued
inputs do not produce; so K10's roots serve as the key directly.
"""
from __future__ import annotations

import numpy as np


def knn_of_rows(rows: np.ndarray, k: int, first: int = 0):
    """rows: (b, n) distances (or squared distances) of positions first .. first + b - 1 to every position.  Returns
    (idx (b, k) int32, key (b, k)): the first k of each row under (key, position)."""
    rows = np.asarray(rows)
    b, n = rows.shape
    idx = np.empty((b, k), dtype=np.int32)
    key = np.empty((b, k), dtype=rows.dtype)
    if b == 0 or k == 0:
        return idx, key
    # only entries not after the k-th key can be among the first k (ties at the k-th place included)
    kth = np.partition(rows, k - 1, axis=1)[:, k - 1]
    pos = np.arange(n)
    for r in range(b):
        cand = np.flatnonzero(rows[r] <= kth[r])
        order = cand[np.lexsort((pos[cand], rows[r, cand]))][:k]
        idx[r] = order
        key[r] = rows[r, order]
    return idx, key


def dist_rows(d: np.ndarray, n: int, i0: int, i1: int) -> np.ndarray:
    """Full rows i0 .. i1 - 1 of the n x n distance matrix from R's "dist" vector d (strict lower triangle by columns,
    K10's output), with 0 on the diagonal."""
    i = np.arange(i0, i1, dtype=np.int64)[:, None]
    j = np.arange(n, dtype=np.int64)[None, :]
    a, b = np.minimum(i, j), np.maximum(i, j)
    at = n * a - a * (a + 1) // 2 + (b - a - 1)
    out = d[np.clip(at, 0, max(len(d) - 1, 0))] if len(d) else np.zeros(at.shape)
    return np.where(i == j, 0.0, out)


def knn_from_dist(d: np.ndarray, n: int, k: int, block: int = 512):
    """(idx (n, k) int32, dist (n, k)) from K10's "dist" vector of n positions."""
    idx = np.empty((n, k), dtype=np.int32)
    dist = np.empty((n, k), dtype=np.float64)
    for i0 in range(0, n, block):
        i1 = min(n, i0 + block)
        idx[i0:i1], dist[i0:i1] = knn_of_rows(dist_rows(d, n, i0, i1), k)
    return idx, dist


def squared_rows(x: np.ndarray, i0: int, i1: int) -> np.ndarray:
    """Squared distances of observations i0 .. i1 - 1 of x (observations x variables) to all, in the difference form."""
    diff = x[i0:i1, None, :] - x[None, :, :]
    return np.einsum("ijg,ijg->ij", diff, diff)


def knn_brute(x: np.ndarray, k: int, block: int = 64):
    """(idx, dist) by brute force in NumPy: squared distances, ordered by (squared distance, position), rooted."""
    x = np.asarray(x, dtype=np.float64)
    n = x.shape[0]
    idx = np.empty((n, k), dtype=np.int32)
    dist = np.empty((n, k), dtype=np.float64)
    for i0 in range(0, n, block):
        i1 = min(n, i0 + block)
        ii, sq = knn_of_rows(squared_rows(x, i0, i1), k)
        idx[i0:i1], dist[i0:i1] = ii, np.sqrt(sq)
    return idx, dist
