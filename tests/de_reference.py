"""NumPy restatement of mask_non_DE_genes_basic (R/inferCNV_mask_non_DE.R:28-259) and of the library's jitter generator -
the expected values of tests/test_gpu_de_mask.py, pinned by tests/test_de_reference.py against scipy.

R's rules restated here:
- wilcox.test(x, y) (two-sided, correct = TRUE, exact = NULL): W = sum of the average ranks of x in x u y - n_x (n_x + 1) / 2;
  exact when n_x < 50, n_y < 50 and no ties, p = min(1, 2 P(W' <= min(W, n_x n_y - W))); otherwise
  z = (W - n_x n_y / 2 - sign(.) / 2) / sigma, sigma^2 = n_x n_y / 12 ((n + 1) - sum(t^3 - t) / (n (n - 1))),
  p = 2 pnorm(-|z|) (NaN when every value is tied).
- t.test(x, y) (Welch): NaN where R's try() catches an error (n < 2, stderr < 10 eps max(|m_x|, |m_y|)), else
  p = 2 pt(-|t|, df), df Welch-Satterthwaite.
- p.adjust(p, "BH"): pmin(1, cummin(n / i * p[o]))[order(o)], o the decreasing order, over the non-NA values (n their count).
- .mask_DE_genes as R writes it (the count matrix, then the rule).
"""
from __future__ import annotations

import functools
import math
from itertools import combinations

import numpy as np
from scipy import special

from tests.runmean_reference import hash3, mix64

EXACT_N = 50
SUB_KEY = 1 << 32
EPS = float(np.finfo(np.float64).eps)


# ---- generator -------------------------------------------------------------------------------------------------------
def uniforms(seed, a, g, i):
    """(u0, u1) in (0, 1]: ((mix64(hash3(seed, a, g, 2 i + k)) >> 11) + 1) 2^-53 - bit-exact with the device."""
    i = np.asarray(i, dtype=np.uint64)
    out = []
    for k in (0, 1):
        h = mix64(hash3(seed, a, g, i * np.uint64(2) + np.uint64(k)))
        out.append(((h >> np.uint64(11)) + np.uint64(1)).astype(np.float64) * 2.0 ** -53)
    return out[0], out[1]


def normals(seed, a, g, n):
    """z of list positions 0 .. n - 1 of group key a, gene g (Box-Muller; the device's log / cospi may differ in the last
    bits)."""
    u0, u1 = uniforms(seed, a, g, np.arange(n))
    return np.sqrt(-2.0 * np.log(u0)) * np.cos(2.0 * np.pi * u1)


def jittered(vals, seed, a, g, jm, js):
    return vals + (jm + js * normals(seed, a, g, len(vals)))


# ---- tests -----------------------------------------------------------------------------------------------------------
def rank_sum_counts(m, n):
    """Exact counts of U = 0 .. m n under the null (Python integers): the Gaussian binomial [m + n choose m]_q."""
    c = [0] * (m * n + 1)
    c[0] = 1
    deg = 0
    for k in range(1, m + 1):
        sh = n + k
        deg += n
        for u in range(deg, sh - 1, -1):
            c[u] -= c[u - sh]
        for u in range(k, deg + 1):
            c[u] += c[u - k]
    return c


@functools.lru_cache(maxsize=None)
def rank_sum_cdf(m, n):
    c = rank_sum_counts(m, n)
    total = sum(c)
    cum = np.cumsum(np.array(c, dtype=object))
    return np.array([float(v) / float(total) for v in cum])


def brute_force_counts(m, n):
    """The same counts by enumerating every choice of x's ranks."""
    c = [0] * (m * n + 1)
    for pos in combinations(range(1, m + n + 1), m):
        c[sum(pos) - m * (m + 1) // 2] += 1
    return c


def wilcox_stats(x, y):
    """(2 W, sum(t^3 - t)) in exact integers."""
    allv = np.concatenate([x, y])
    _, inv, counts = np.unique(allv, return_inverse=True, return_counts=True)
    cum = np.cumsum(counts)
    avg2 = (2 * (cum - counts) + counts + 1)            # twice the average rank of each distinct value
    nx = len(x)
    w2 = int(avg2[inv[:nx]].sum()) - nx * (nx + 1)
    ties = int(sum(int(t) ** 3 - int(t) for t in counts))
    return w2, ties


def wilcox_p(x, y):
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    nx, ny = len(x), len(y)
    w2, ties = wilcox_stats(x, y)
    if nx < EXACT_N and ny < EXACT_N and ties == 0:
        w = w2 // 2
        mn = nx * ny
        return min(1.0, 2.0 * rank_sum_cdf(nx, ny)[min(w, mn - w)])
    nxd, nyd = float(nx), float(ny)
    z = w2 / 2.0 - nxd * nyd / 2
    N = nxd + nyd
    sigma = math.sqrt((nxd * nyd / 12) * ((N + 1) - ties / (N * (N - 1))))
    corr = 0.5 * np.sign(z)
    with np.errstate(invalid="ignore", divide="ignore"):
        z = (z - corr) / np.float64(sigma)
    return float(2.0 * special.ndtr(-abs(z)))


def _mean(x):
    return math.fsum(x) / len(x)


def welch_p(x, y):
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    nx, ny = len(x), len(y)
    if nx < 2 or ny < 2:
        return float("nan")
    mx, my = _mean(x), _mean(y)
    vx = math.fsum((x - mx) ** 2) / (nx - 1)
    vy = math.fsum((y - my) ** 2) / (ny - 1)
    sx, sy = math.sqrt(vx / nx), math.sqrt(vy / ny)
    se = math.sqrt(sx * sx + sy * sy)
    if se < 10 * EPS * max(abs(mx), abs(my)) or se == 0.0:
        return float("nan")
    df = se ** 4 / (sx ** 4 / (nx - 1) + sy ** 4 / (ny - 1))
    t = (mx - my) / se
    return float(2.0 * special.stdtr(df, -abs(t)))


def bh(p):
    """p.adjust(p, "BH") in R's operation order; NaN stays NaN and n counts the others."""
    p = np.asarray(p, dtype=np.float64)
    out = np.full(p.shape, np.nan)
    ok = ~np.isnan(p)
    q = p[ok]
    n = len(q)
    if n == 0:
        return out
    o = np.argsort(-q, kind="stable")
    i = np.arange(n, 0, -1, dtype=np.float64)
    adj = np.minimum(1.0, np.minimum.accumulate((n / i) * q[o]))
    r = np.empty(n)
    r[o] = adj
    out[ok] = r
    return out


# ---- pairs and mask --------------------------------------------------------------------------------------------------
def tested_subclusters(obs_names, subclusters):
    """R's loop of get_DE_genes_basic over observation groups: subclusters[name] is either a dict (a named list: its
    entries in order) or a plain index list (list(indices) is unnamed, so R tests nothing for that group).
    Returns [(subcluster name, indices)]."""
    out = []
    for name in obs_names:
        v = subclusters[name]
        if isinstance(v, dict):
            out.extend((k, np.asarray(idx)) for k, idx in v.items())
    return out


def de_pvals(X, ref_groups, subclusters, test="wilcoxon", jm=1e-4, js=1e-4, seed=0):
    """p_raw G x (n_sub n_ref), column s n_ref + j; jitter as the library draws it."""
    G = X.shape[0]
    n_ref = len(ref_groups)
    P = np.empty((G, len(subclusters) * n_ref))
    for s, sub in enumerate(subclusters):
        for j, ref in enumerate(ref_groups):
            col = s * n_ref + j
            for g in range(G):
                x, y = X[g, ref], X[g, sub]
                if test == "wilcoxon":
                    x = jittered(x, seed, j, g, jm, js)
                    y = jittered(y, seed, SUB_KEY + col, g, jm, js)
                    P[g, col] = wilcox_p(x, y)
                else:
                    P[g, col] = welch_p(x, y)
    return P


def mask_from_padj(X, ref_groups, subclusters, p_adj, thr, rule, center_val):
    """.mask_DE_genes (R/inferCNV_mask_non_DE.R:77-134) from the adjusted p-values, literally."""
    G, C = X.shape
    n_ref = len(ref_groups)
    M = np.zeros((G, C), dtype=np.int64)
    M[:, np.concatenate([np.asarray(r) for r in ref_groups])] = n_ref
    for sub in subclusters:
        if len(sub) < 5:
            M[:, np.asarray(sub)] = n_ref
    for s, sub in enumerate(subclusters):
        for j in range(n_ref):
            de = p_adj[:, s * n_ref + j] < thr
            if len(sub) >= 5:
                rows = np.flatnonzero(de)
                M[np.ix_(rows, np.asarray(sub))] += 1        # a repeated cell gets +1 once, as R's assignment does
    if rule == "all":
        masked = M != n_ref
    elif rule == "most":
        masked = M < n_ref / 2
    elif rule == "any":
        masked = M == 0
    else:
        raise ValueError(rule)
    Y = np.array(X, dtype=np.float64, order="F")
    Y[masked] = center_val
    return Y


def de_counts(p_adj, thr):
    """The counts of R's message "Found %d genes / %d total as DE" per pair: #(p < thr) + #NA, and G."""
    return [(int(np.sum(p_adj[:, c] < thr) + np.sum(np.isnan(p_adj[:, c]))), p_adj.shape[0]) for c in range(p_adj.shape[1])]


def mask_non_de(X, ref_groups, subclusters, test="wilcoxon", thr=0.05, rule="any", center_val=None, jm=1e-4, js=1e-4, seed=0):
    """(Y, p_raw, p_adj) of the whole step."""
    X = np.asarray(X, dtype=np.float64)
    if center_val is None:
        center_val = float(np.mean(X))
    P = de_pvals(X, ref_groups, subclusters, test, jm, js, seed)
    A = np.column_stack([bh(P[:, c]) for c in range(P.shape[1])]) if P.shape[1] else P.copy()
    return mask_from_padj(X, ref_groups, subclusters, A, thr, rule, center_val), P, A
