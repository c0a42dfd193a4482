"""TEST INFRASTRUCTURE: reference restatements of hclust() for the tests of the linkage kernel (icnv_hclust.cu).

* ``nn_chain`` restates the kernel's nearest-neighbour chain - the same tie rules, the same Lance-Williams formulas in the
  same operation order, the same stable sort and conversion to R's merge matrix - in NumPy.  NumPy evaluates every
  element-wise product, sum and quotient as one correctly rounded IEEE operation (no contraction), so on the same input it
  must equal the GPU bit for bit.
* ``closest_pair`` is a literal O(n^3) transcription of agglomerative clustering: merge the globally closest pair, update
  by Lance-Williams, repeat.  It shares no control flow with the chain; on tie-free data both give the same tree.
* ``hcass2_order`` is R's hcass2 loop for `order`, written as the loop it is.
* ``check_tree`` checks that a result is a valid agglomeration of the input, whatever the ties.

Method codes as fastcluster orders them: 0 single, 1 complete, 2 average, 3 mcquitty, 4 ward.D, 7 ward.D2.
"""
from __future__ import annotations

import numpy as np

METHODS = {"single": 0, "complete": 1, "average": 2, "mcquitty": 3, "ward.D": 4, "ward.D2": 7}


def square(d, n: int) -> np.ndarray:
    """R's "dist" vector (strict lower triangle by columns) -> symmetric n x n matrix, zero diagonal."""
    d = np.asarray(d, dtype=np.float64)
    M = np.zeros((n, n))
    iu = np.triu_indices(n, 1)      # row-major over a < b: the order of the condensed vector
    M[iu] = d
    M.T[iu] = d
    return M


def lance_williams(method: int, dki, dkj, dij, ni, nj, nk):
    if method == 0:
        return np.minimum(dki, dkj)
    if method == 1:
        return np.maximum(dki, dkj)
    if method == 2:
        return (ni * dki + nj * dkj) / (ni + nj)
    if method == 3:
        return (dki + dkj) / 2.0
    return ((ni + nk) * dki + (nj + nk) * dkj - nk * dij) / ((ni + nj) + nk)


def to_r(raw_i, raw_j, raw_h, n: int, method: int):
    """Stable sort by height, then union-find over the slots in sorted order -> R's merge (n-1 x 2) and height."""
    raw_h = np.asarray(raw_h, dtype=np.float64)
    order = np.argsort(raw_h, kind="stable")
    uf = list(range(n))
    node = list(range(n))

    def find(x):
        while uf[x] != x:
            uf[x] = uf[uf[x]]
            x = uf[x]
        return x

    merge = np.zeros((n - 1, 2), dtype=np.int32)
    for s, t in enumerate(order):
        x, y = find(raw_i[t]), find(raw_j[t])
        lo, hi = sorted((node[x], node[y]))
        merge[s] = [-(lo + 1) if lo < n else lo - n + 1, -(hi + 1) if hi < n else hi - n + 1]
        uf[x] = y
        node[y] = n + s
    h = raw_h[order]
    return merge, (np.sqrt(h) if method == 7 else h)


def nn_chain(d, n: int, method: int):
    """The kernel's algorithm.  Returns (merge, height, order)."""
    M = square(d, n)
    if method == 7:
        M = M * M
    inf = np.inf
    np.fill_diagonal(M, inf)
    active = np.ones(n, dtype=bool)
    size = np.ones(n, dtype=np.float64)
    chain: list[int] = []
    raw_i, raw_j, raw_h = [], [], []
    while len(raw_h) < n - 1:
        if not chain:
            chain = [int(np.flatnonzero(active)[0])]
        a = chain[-1]
        p = chain[-2] if len(chain) >= 2 else -1
        row = np.where(active, M[a], inf)
        row[a] = inf
        b = int(np.argmin(row))          # the first of equal minima: the smallest index
        if p >= 0 and M[a, p] == row[b]:
            b = p                        # the element before the tip wins a tie
        if b != p:
            if len(chain) == n:
                chain = []
            chain.append(b)
            continue
        i, j = min(a, b), max(a, b)
        dij = M[a, b]
        raw_i.append(i), raw_j.append(j), raw_h.append(dij)
        k = np.flatnonzero(active)
        k = k[(k != i) & (k != j)]
        w = lance_williams(method, M[i, k], M[j, k], dij, size[i], size[j], size[k])
        M[j, k] = w
        M[k, j] = w
        size[j] += size[i]
        active[i] = False
        chain = chain[:-2]
    merge, height = to_r(raw_i, raw_j, raw_h, n, method)
    return merge, height, hcass2_order(merge, n)


def closest_pair(d, n: int, method: int):
    """Literal O(n^3) agglomeration: repeatedly merge the closest pair of active clusters (the smaller index pair first
    on ties), Lance-Williams update into the larger slot.  Returns (merge, height, order) in R's convention."""
    M = square(d, n)
    if method == 7:
        M = M * M
    active = list(range(n))
    size = [1.0] * n
    raw_i, raw_j, raw_h = [], [], []
    for _ in range(n - 1):
        idx = np.array(active)
        sub = M[np.ix_(idx, idx)].copy()
        np.fill_diagonal(sub, np.inf)
        f = int(np.argmin(sub))
        i, j = int(idx[f // len(idx)]), int(idx[f % len(idx)])
        i, j = min(i, j), max(i, j)
        dij = M[i, j]
        raw_i.append(i), raw_j.append(j), raw_h.append(dij)
        for k in active:
            if k in (i, j):
                continue
            w = lance_williams(method, M[i, k], M[j, k], dij, size[i], size[j], size[k])
            M[j, k] = M[k, j] = w
        size[j] += size[i]
        active.remove(i)
    merge, height = to_r(raw_i, raw_j, raw_h, n, method)
    return merge, height, hcass2_order(merge, n)


def hcass2_order(merge, n: int) -> np.ndarray:
    """R's hcass2 (src/library/stats/src/hclust-utils.c, Fortran HCASS2): iorder starts as the two members of the last
    merge; going down from merge n-2, every cluster number in iorder is replaced by its two members in place."""
    merge = np.asarray(merge)
    if n == 1:
        return np.array([1], dtype=np.int32)
    iorder = [int(merge[n - 2, 0]), int(merge[n - 2, 1])]
    for i in range(n - 2, 0, -1):         # cluster number i (1-based)
        for loc in range(len(iorder)):
            if iorder[loc] == i:
                iorder[loc:loc + 1] = [int(merge[i - 1, 0]), int(merge[i - 1, 1])]
                break
    return np.array([-v for v in iorder], dtype=np.int32)


def check_tree(d, n: int, method: int, merge, height, order, rtol: float = 1e-12) -> None:
    """A valid agglomeration of d whatever the ties: replaying the merges from the input by Lance-Williams, every merge
    joins two existing clusters that are reciprocal nearest neighbours at its height, the heights do not decrease, and
    `order` is the permutation hcass2 makes of merge."""
    merge = np.asarray(merge)
    height = np.asarray(height, dtype=np.float64)
    assert merge.shape == (n - 1, 2) and height.shape == (n - 1,)
    assert np.all(np.diff(height) >= 0), "heights decrease"
    assert np.array_equal(np.sort(order), np.arange(1, n + 1)), "order is not a permutation"
    assert np.array_equal(order, hcass2_order(merge, n)), "order does not follow merge"
    M = square(d, n)
    if method == 7:
        M = M * M
    slot = {}                             # R node -> slot in M
    active = np.ones(n, dtype=bool)
    size = np.ones(n)
    for s in range(n - 1):
        x, y = (int(v) for v in merge[s])
        assert (x < 0 or x < s + 1) and (y < 0 or y < s + 1), f"merge {s + 1} uses a cluster made later"
        if x < 0 and y < 0:
            assert -x < -y, f"merge {s + 1}: singletons out of order"
        elif x > 0 and y > 0:
            assert x < y, f"merge {s + 1}: clusters out of order"
        else:
            assert x < 0, f"merge {s + 1}: the singleton comes first"
        a = -x - 1 if x < 0 else slot.pop(x)
        b = -y - 1 if y < 0 else slot.pop(y)
        assert active[a] and active[b] and a != b
        dab = M[a, b]
        h = np.sqrt(dab) if method == 7 else dab
        assert abs(h - height[s]) <= rtol * max(abs(h), 1e-300) + 1e-300, f"merge {s + 1}: height {height[s]} vs {h}"
        for u, v in ((a, b), (b, a)):       # reciprocal nearest neighbours, up to rounding
            others = active.copy()
            others[u] = False
            assert dab <= M[u, others].min() * (1 + rtol) + 1e-300, f"merge {s + 1}: not a nearest neighbour"
        i, j = min(a, b), max(a, b)
        k = np.flatnonzero(active)
        k = k[(k != i) & (k != j)]
        w = lance_williams(method, M[i, k], M[j, k], dab, size[i], size[j], size[k])
        M[j, k] = w
        M[k, j] = w
        size[j] += size[i]
        active[i] = False
        slot[s + 1] = j
