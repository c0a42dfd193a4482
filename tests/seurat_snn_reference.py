"""A NumPy restatement of what .leiden_seurat_preprocess_routine (R/inferCNV_tumor_subclusters.R:699-723) computes with
Seurat 5 - FindVariableFeatures(vst) -> ScaleData -> RunPCA(npcs) -> FindNeighbors(k.param, prune.SNN = 1/15) - in the
exact form K18 (infercnv_b200/csrc/icnv_snn.cu) computes it: the direct loess fit per gene, eigh of the Gram matrix, the
exact kNN in the (distance, position) order and the SNN graph as A A^T of the neighbour indicator.  Test-side only."""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

SPAN, SCALE_MAX, PRUNE = 0.3, 10.0, 1.0 / 15.0


def gene_stats(Xg):
    """mu and v (n - 1) of every gene of the genes x cells matrix."""
    return Xg.mean(axis=1), Xg.var(axis=1, ddof=1)


def loess_direct(x, y, span=SPAN):
    """Local quadratic fit of y on x at every x (degree 2, tricube weights on d / rho, rho the q-th smallest distance,
    q = floor(m span)).  Returns (fit, singular) with singular[i] where the weighted system is singular."""
    m = len(x)
    q = int(np.floor(m * span))
    fit = np.empty(m)
    sing = np.zeros(m, dtype=bool)
    for i in range(m):
        d = np.abs(x - x[i])
        rho = np.sort(d)[q - 1]
        if rho <= 0:
            sel = d == 0
            fit[i] = y[sel].mean()
            sing[i] = True
            continue
        u = (x - x[i]) / rho
        w = np.where(np.abs(u) < 1, (1 - np.abs(u) ** 3) ** 3, 0.0)
        A = np.stack([np.ones(m), u, u * u], axis=1)
        M = A.T @ (w[:, None] * A)
        r = A.T @ (w * y)
        ev = np.linalg.eigvalsh(M)
        if ev[0] <= 1e-12 * ev[-1]:
            fit[i] = (w * y).sum() / w.sum()
            sing[i] = True
        else:
            fit[i] = np.linalg.solve(M, r)[0]
    return fit, sing


def standardized_variance(Xg, mu, sexp):
    n = Xg.shape[1]
    out = np.zeros(len(mu))
    ok = sexp > 0
    z = np.minimum((Xg[ok] - mu[ok, None]) / sexp[ok, None], np.sqrt(n))
    out[ok] = (z * z).sum(axis=1) / (n - 1)
    return out


def variable_features(Xg, n_features=2000):
    """(ranked genes, standardised variances, singular fits): vst's ranking, ties by the lower gene index."""
    mu, v = gene_stats(Xg)
    nc = v > 0
    if np.any(mu[nc] <= 0):
        raise ValueError("a non-constant gene has mean <= 0")
    fit, sing = loess_direct(np.log10(mu[nc]), np.log10(v[nc]))
    sexp = np.zeros(len(mu))
    sexp[nc] = np.sqrt(10.0 ** fit)
    sv = standardized_variance(Xg, mu, sexp)
    order = np.lexsort((np.arange(len(sv)), -sv))
    return order[:min(n_features, len(sv))], sv, int(sing.sum())


def pca(Xg, feats, npcs=10):
    """Features (non-constant, in ascending gene order), eigenvalues, V (F x npcs, sign rule), embeddings (n x npcs)."""
    mu, v = gene_stats(Xg)
    rank = {g: r for r, g in enumerate(feats)}
    use = np.sort([g for g in feats if v[g] > 0])
    Z = np.minimum((Xg[use] - mu[use, None]) / np.sqrt(v[use])[:, None], SCALE_MAX)
    lam, U = np.linalg.eigh(Z @ Z.T)
    lam, U = lam[::-1], U[:, ::-1]
    V = U[:, :npcs].copy()
    ranks = np.array([rank[g] for g in use])
    for j in range(npcs):
        a = np.abs(V[:, j])
        best = np.flatnonzero(a == a.max())
        f = best[np.argmin(ranks[best])]
        if V[f, j] < 0:
            V[:, j] = -V[:, j]
    return use, lam, V, Z.T @ V


def knn(E, k):
    """Exact k nearest rows of E (self included), ordered by squared distance then position."""
    sq = ((E[:, None, :] - E[None, :, :]) ** 2).sum(axis=2)
    n = E.shape[0]
    return np.stack([np.lexsort((np.arange(n), sq[i]))[:k] for i in range(n)]).astype(np.int32)


def snn(idx, n, k, prune=PRUNE):
    """Seurat's ComputeSNN: s = A A^T of the neighbour indicator, w = s / (k + (k - s)), entries with w < prune dropped."""
    A = sp.csr_matrix((np.ones(idx.size), idx.ravel(), np.arange(0, idx.size + 1, k)), shape=(n, n))
    S = (A @ A.T).tocsr()
    S.sort_indices()
    s = S.data
    w = s / (k + (k - s))
    keep = ~(w < prune)
    rows = np.repeat(np.arange(n), np.diff(S.indptr))
    out = sp.csr_matrix((w[keep], (rows[keep], S.indices[keep])), shape=(n, n))
    out.sort_indices()
    return out


def seurat_snn(Xg, k=20, n_features=2000, npcs=10):
    """Everything at once: dict with features, sv, use, lam, V, emb, idx, graph."""
    feats, sv, n_sing = variable_features(Xg, n_features)
    use, lam, V, E = pca(Xg, feats, npcs)
    idx = knn(E, k)
    return {"features": feats, "sv": sv, "singular": n_sing, "use": use, "lam": lam, "V": V, "emb": E, "idx": idx,
            "graph": snn(idx, Xg.shape[1], k)}
