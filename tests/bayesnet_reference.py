"""Expected values of the Bayesian network filter (inferCNVBayesNet's Gibbs sampling, icnv_bayes.cu) in NumPy.

* `loglik` restates the library's log-likelihood pass operation for operation: L[j, k] = sum over the entries of column j,
  in list order, of hl_k - (ht_k d) d, d = x - mu_k, hl_k = 1/2 log tau_k, ht_k = 1/2 tau_k, each operation rounded on its
  own.  A pooled region (R's one-gene quirk) is one column over all its entries, cells in list order, within a cell its
  genes in list order.
* `enumerate_posterior` is the exact posterior of the mixture model for a few cells: with theta ~ Dirichlet(1, ..., 1)
  integrated out, p(eps) ∝ prod_j exp(L[j, eps_j]) prod_k Gamma(1 + n_k), which gives P(eps_j = k) and
  E[theta_k] = E[(1 + n_k) / (m + C)].
* `simplex_integral` is the same for m = 3 by brute-force quadrature over theta (the check of the enumeration).
* `gibbs` is the sampler in NumPy (its own generator, so the same posterior, not the same draws): the CPU stand-in of
  tools/bench_bayesnet.py.
* `remove_cnv` / `reassign_cnv` restate removeCNV / reassignCNV (R/inferCNV_BayesNet.R:491-629) on mean theta.
"""
from __future__ import annotations

import itertools
import math

import numpy as np


def loglik(X, genes, cells, mu, tau, pooled=False) -> np.ndarray:
    """m x C' log-likelihoods of one region of the genes x cells matrix X."""
    mu = np.asarray(mu, dtype=np.float64)
    tau = np.asarray(tau, dtype=np.float64)
    hl, ht = 0.5 * np.log(tau), 0.5 * tau
    block = np.asarray(X, dtype=np.float64)[np.ix_(np.asarray(genes), np.asarray(cells))]   # G_r x C_r
    if pooled:
        block = block.T.reshape(-1, 1)          # cells in list order, within a cell its genes
    s = np.zeros((len(mu), block.shape[1]))
    for row in block:                          # the entries of each column in list order
        d = row[None, :] - mu[:, None]
        s = s + (hl[:, None] - (ht[:, None] * d) * d)
    return s


def enumerate_posterior(L):
    """L: m x C (C <= 6).  Returns (P, E): P m x C with P[k, j] = P(eps_j = k), E[k] = E[theta_k]."""
    L = np.asarray(L, dtype=np.float64)
    m, C = L.shape
    lg = np.array([math.lgamma(1 + n) for n in range(C + 1)])
    P = np.zeros((m, C))
    E = np.zeros(m)
    logs, assigns = [], []
    for eps in itertools.product(range(m), repeat=C):
        n = np.bincount(eps, minlength=m)
        logs.append(sum(L[k, j] for j, k in enumerate(eps)) + lg[n].sum())
        assigns.append((eps, n))
    logs = np.array(logs)
    w = np.exp(logs - logs.max())
    w /= w.sum()
    for wi, (eps, n) in zip(w, assigns):
        for j, k in enumerate(eps):
            P[k, j] += wi
        E += wi * (1 + n) / (m + C)
    return P, E


def simplex_integral(L, n_grid=600):
    """m = 3 only: (P, E) by the midpoint rule over theta on the simplex, p(theta) ∝ prod_j sum_k theta_k exp(L[j, k])."""
    L = np.asarray(L, dtype=np.float64)
    m, C = L.shape
    assert m == 3
    h = 1.0 / n_grid
    a = (np.arange(n_grid) + 0.5) * h
    t1, t2 = np.meshgrid(a, a, indexing="ij")
    keep = t1 + t2 < 1.0
    th = np.stack([t1[keep], t2[keep], 1.0 - t1[keep] - t2[keep]])      # 3 x N
    eL = np.exp(L - L.max(axis=0, keepdims=True))                       # per cell, scaled
    per = th.T @ eL                                                      # N x C: sum_k theta_k e^{L[j,k]}
    logp = np.log(per).sum(axis=1)
    w = np.exp(logp - logp.max())
    w /= w.sum()
    E = th @ w
    P = np.zeros((m, C))
    for j in range(C):
        P[:, j] = (th * eL[:, j][:, None] / per[:, j][None, :]) @ w
    return P, E


def gibbs(L, n_chains, n_burn, n_keep, rng):
    """The sampler in NumPy: (theta draws (n_chains n_keep) x m, state counts m x C)."""
    L = np.asarray(L, dtype=np.float64)
    m, C = L.shape
    theta = np.empty((n_chains * n_keep, m))
    counts = np.zeros((m, C), dtype=np.int64)
    for c in range(n_chains):
        n = np.zeros(m)
        n[c % m] = C
        for s in range(n_burn + n_keep):
            g = rng.gamma(1.0 + n)
            th = g / g.sum()
            lw = np.log(th)[:, None] + L
            w = np.exp(lw - lw.max(axis=0))
            cum = np.cumsum(w, axis=0)
            u = rng.random(C) * cum[-1]
            eps = (cum < u[None, :]).sum(axis=0)
            n = np.bincount(eps, minlength=m).astype(np.float64)
            if s >= n_burn:
                theta[c * n_keep + s - n_burn] = th
                counts[eps, np.arange(C)] += 1
    return theta, counts


def remove_cnv(theta_means, normal_state, max_p_normal):
    """removeCNV's choice: 0-based indices of the regions whose mean theta of the (1-based) normal state exceeds the
    threshold."""
    tm = np.asarray(theta_means)
    return [r for r in range(tm.shape[0]) if tm[r, normal_state - 1] > max_p_normal]


def reassign_cnv(theta_means):
    """reassignCNV's new state per region: the first arg-max of mean theta, 1-based."""
    return [int(np.flatnonzero(row == row.max())[0]) + 1 for row in np.asarray(theta_means)]
