"""K18, the SNN graph of the Leiden PCA route (icnv_snn.cu; Seurat's vst -> ScaleData -> RunPCA -> FindNeighbors), on the GPU,
against tests/seurat_snn_reference.py.

The reference is exact arithmetic's stand-in, not the kernel's bits: the device sums in other orders (DMMA tiles, warp
trees), so every comparison carries a bound, and equality is required only where the reference's own margins exceed it -
the rank gap of the standardised variances, the eigen-gap of a component, the distance gaps of a kNN list.  Under the host
emulation (tests/test_snn_emulated_and_r.py) only the small cases run; there F is at most 39, so the 32-column subspace block
covers all or most of the feature space and converges within a few Rayleigh-Ritz checks."""
import os

import numpy as np
import pytest

from infercnv_b200 import _lib, api
from infercnv_b200._lib import InfercnvB200Error
from tests import seurat_snn_reference as sr

pytestmark = pytest.mark.gpu
EMULATED = "_emu" in os.path.basename(_lib.LIB_PATH)
SV_REL = 1e-9       # standardised variances: relative agreement expected of the two summation orders
EIG_REL = 1e-9      # eigenvectors: ||dV|| <= EIG_REL / relative eigen-gap
DIST_REL = 1e-8     # kNN: distances closer than this (relative) are near-ties


@pytest.fixture(scope="module", autouse=True)
def _init():
    api.init(0)


def planted(n, G, clones=4, seed=0, dup=0):
    """n cells x G genes (genes x cells) of `clones` planted CNV clones: per-gene base levels, clone-specific gains and
    losses over gene blocks, log-normal noise; all values positive.  dup > 0 makes the last `dup` cells copies of cell 0."""
    rng = np.random.default_rng(seed)
    base = rng.gamma(3.0, 1.0, size=G) + 0.5
    lab = rng.integers(0, clones, size=n)
    cnv = np.ones((clones, G))
    for c in range(clones):
        for _ in range(4):
            a = int(rng.integers(0, G - G // 10))
            cnv[c, a:a + G // 10] = rng.choice([0.5, 1.5, 2.0])
    X = base[:, None] * cnv[lab].T * np.exp(rng.normal(scale=0.3, size=(G, n)))
    if dup:
        X[:, n - dup:] = X[:, :1]
        lab[n - dup:] = lab[0]
    return np.asfortranarray(X), lab


def ref_knn(E, k):
    """Exact kNN of the rows of E in (squared distance, position) order, and each row's k + 1 smallest distances."""
    n = E.shape[0]
    idx = np.empty((n, k), np.int32)
    d = np.empty((n, k + 1))
    for a in range(0, n, 64):
        sq = ((E[a:a + 64, None, :] - E[None, :, :]) ** 2).sum(axis=2)
        for r in range(sq.shape[0]):
            kk = min(k + 1, n)
            kth = np.partition(sq[r], kk - 1)[kk - 1]
            cand = np.flatnonzero(sq[r] <= kth)
            o = cand[np.lexsort((cand, sq[r][cand]))]
            idx[a + r] = o[:k]
            d[a + r, :kk] = np.sqrt(sq[r][o[:kk]])
    return idx, d


def compare(X, r, k, n_features=2000, npcs=10, ref=None):
    """Check the GPU result r against the reference on X; returns the fraction of rows whose kNN lists were compared."""
    G, n = X.shape
    if ref is None:
        feats, sv, _ = sr.variable_features(X, n_features)
        use, lam, V, E = sr.pca(X, feats, npcs)
        ref = (feats, sv, use, lam, V, E)
    feats, sv, use, lam, V, E = ref
    # variable features: equal wherever the reference's rank gap exceeds the bound
    nf = min(n_features, G)
    assert r.features.shape == (nf,)
    srt = np.sort(sv)[::-1]
    tol = SV_REL * srt[0]
    gap = np.minimum(np.abs(np.diff(np.concatenate([[np.inf], srt]))), np.abs(np.diff(np.concatenate([srt, [-np.inf]]))))
    clear = gap[:nf] > tol
    assert np.array_equal(r.features[clear], feats[clear])
    np.testing.assert_allclose(sv[r.features], srt[:nf], rtol=0, atol=tol)
    st = r.stats
    assert st["F"] == len(use) and st["npcs"] == npcs and st["residual"] <= 1e-12
    # embeddings within the bound the eigen-gap allows
    assert r.embeddings.shape == (n, npcs)
    for j in range(npcs):
        g = min(lam[j] - lam[j + 1], lam[j - 1] - lam[j] if j else np.inf) / lam[0]
        if g < 1e-6:
            continue
        scale = np.abs(E[:, j]).max()
        assert np.abs(r.embeddings[:, j] - E[:, j]).max() <= EIG_REL / g * scale + 1e-12 * scale, j
    # kNN lists: equal where the reference has no near-tie among its first k + 1 distances
    idx_ref, d_ref = ref_knn(E, k)
    assert r.idx.shape == (n, k)
    dd = np.diff(d_ref[:, :min(k + 1, n)], axis=1)
    clear_rows = np.all(dd > DIST_REL * np.maximum(d_ref[:, -1:], 1e-300), axis=1)
    assert np.array_equal(r.idx[clear_rows], idx_ref[clear_rows])
    # CSR: symmetric, sorted, diagonal 1; equal to the reference graph of the GPU's own lists, and to the reference's graph
    # on every pair whose two lists are equal as sets
    g = api_csr(r, n)
    assert (g != g.T).nnz == 0
    assert np.all(g.diagonal() == 1.0)
    for i in range(n):
        row = r.indices[r.indptr[i]:r.indptr[i + 1]]
        assert np.all(np.diff(row) > 0)
    gs = sr.snn(r.idx, n, k)
    assert np.array_equal(gs.indptr, r.indptr) and np.array_equal(gs.indices, r.indices) and np.array_equal(gs.data, r.data)
    same = np.array([set(a) == set(b) for a, b in zip(r.idx.tolist(), idx_ref.tolist())])
    gr = sr.snn(idx_ref, n, k).tocsr()
    for i in np.flatnonzero(same)[:2000]:
        cols = np.union1d(g.indices[g.indptr[i]:g.indptr[i + 1]], gr.indices[gr.indptr[i]:gr.indptr[i + 1]])
        cols = cols[same[cols]]
        assert np.array_equal(g[i, cols].toarray(), gr[i, cols].toarray()), i
    return clear_rows.mean()


def api_csr(r, n):
    import scipy.sparse as sp
    return sp.csr_matrix((r.data, r.indices, r.indptr), shape=(n, n))


SHAPES = [(150, 60, 30)] if EMULATED else [(2000, 2000, 2000), (5000, 5000, 2000), (20000, 3000, 2000)]


@pytest.mark.parametrize("n,G,nf", SHAPES)
def test_planted_clones_match_the_reference(n, G, nf):
    X, lab = planted(n, G, seed=n)
    k = 10 if EMULATED else 20
    r = api.seurat_snn(X, k=k, n_features=nf)
    frac = compare(X, r, k, nf)
    assert frac > 0.9
    if not EMULATED:
        assert r.stats["iterations"] >= 8


def test_repeated_calls_and_cell_lists_give_the_same_bytes():
    n, G, nf = (150, 60, 30) if EMULATED else (3000, 2500, 2000)
    X, _ = planted(n + 40, G, seed=3)
    cells = np.random.default_rng(3).permutation(n + 40)[:n]
    a = api.seurat_snn(X, k=10, cells=cells, n_features=nf)
    b = api.seurat_snn(X, k=10, cells=cells, n_features=nf)
    c = api.seurat_snn(np.asfortranarray(X[:, cells]), k=10, n_features=nf)
    for x, y in ((a, b), (a, c)):
        for f in ("indptr", "indices", "features", "idx"):
            assert np.array_equal(getattr(x, f), getattr(y, f)), f
        for f in ("data", "embeddings"):
            assert np.array_equal(getattr(x, f).view(np.int64), getattr(y, f).view(np.int64)), f


@pytest.mark.skipif(EMULATED, reason="needs torch device tensors")
def test_engine_and_gene_range_view_equal_the_host_abi():
    """Engine.seurat_snn on a resident (C, G) tensor and on a gene-range view of it (one chromosome, the per-chromosome PCA
    route) returns the bytes of api.seurat_snn on the same values."""
    import torch
    from infercnv_b200.device import Engine
    eng = Engine(0)
    X, _ = planted(2500, 3000, seed=5)
    T = torch.as_tensor(np.ascontiguousarray(X.T), device="cuda:0")        # cells x genes
    cells = np.random.default_rng(5).permutation(2500)[:2000]
    for a, b, sel in ((0, 3000, None), (700, 1900, None), (700, 1900, cells)):
        got = eng.seurat_snn(T[:, a:b], 20, sel)
        sub = X[a:b] if sel is None else X[a:b][:, sel]
        want = api.seurat_snn(np.asfortranarray(sub), 20)
        for f in ("indptr", "indices", "features", "idx"):
            assert np.array_equal(getattr(got, f), getattr(want, f)), f
        for f in ("data", "embeddings"):
            assert np.array_equal(getattr(got, f).view(np.int64), getattr(want, f).view(np.int64)), f


def test_fewer_genes_than_n_features_a_constant_gene_and_exact_zeros():
    n, G = (150, 40) if EMULATED else (2000, 300)
    X, _ = planted(n, G, seed=11)
    X[3] = 2.0                       # constant
    X[5, ::3] = 0.0                  # exact zeros
    r = api.seurat_snn(X, k=10)
    assert len(r.features) == G and r.features[-1] == 3
    assert r.stats["sv_gap"] == np.inf and r.stats["F"] == G - 1
    compare(X, r, 10)


def test_duplicated_cells_form_a_hub_through_the_global_path():
    """The last `dup` cells copy cell 0: their embeddings are equal, each of them lists the k lowest-positioned copies, whose
    reverse lists hold every copy - more candidates than a warp's shared memory takes, so those rows take the spill path."""
    n, G, dup = (300, 60, 260) if EMULATED else (4000, 2000, 400)
    X, _ = planted(n, G, seed=13, dup=dup)
    k = 20
    r = api.seurat_snn(X, k=k, n_features=30 if EMULATED else 2000)
    assert r.stats["hub_rows"] > 0
    gs = sr.snn(r.idx, n, k)
    assert np.array_equal(gs.indptr, r.indptr) and np.array_equal(gs.indices, r.indices) and np.array_equal(gs.data, r.data)
    copies = np.r_[0, np.arange(n - dup, n)]
    assert np.all(np.isin(r.idx[n - dup:], copies))


@pytest.mark.parametrize("k", [1, 64])
def test_k_edges(k):
    n, G, nf = (150, 60, 30) if EMULATED else (2000, 1500, 2000)
    X, _ = planted(n, G, seed=k)
    r = api.seurat_snn(X, k=k, n_features=nf)
    assert r.idx.shape == (n, k)
    if k == 1:   # every cell is its own only neighbour (no duplicates): the graph is the identity
        assert np.array_equal(r.indptr, np.arange(n + 1)) and np.array_equal(r.indices, np.arange(n)) and np.all(r.data == 1)
    compare(X, r, k, nf)


def test_error_codes():
    X, _ = planted(120, 40, seed=2)
    for kw, code in (({"k": 65}, -4), ({"k": 0}, -3), ({"npcs": 17}, -4), ({"npcs": 0}, -3), ({"n_features": 0}, -3)):
        with pytest.raises(InfercnvB200Error) as e:
            api.seurat_snn(X, **kw)
        assert e.value.code == code, kw
    with pytest.raises(InfercnvB200Error) as e:
        api.seurat_snn(X[:, :30], k=40)         # k > n
    assert e.value.code == -3
    with pytest.raises(InfercnvB200Error) as e:
        api.seurat_snn(X[:, :10], k=5)          # n <= npcs
    assert e.value.code == -4
    with pytest.raises(InfercnvB200Error) as e:
        api.seurat_snn(X[:9], k=5)              # q = floor(0.3 * 9) = 2 < 3
    assert e.value.code == -4
    with pytest.raises(InfercnvB200Error) as e:
        api.seurat_snn(X[:12], k=5, n_features=10)    # q = 3, but F = 10 <= npcs
    assert e.value.code == -4
    Y = X.copy()
    Y[4, 7] = np.nan
    with pytest.raises(InfercnvB200Error) as e:
        api.seurat_snn(Y, k=5)
    assert e.value.code == -5
    api.seurat_snn(Y, k=5, cells=[0, 1, 2, 3, 4, 5, 6, 8, 9, 10, 11, 12])   # the NaN cell is not listed
    Y = X - X.mean()                            # negative means: vst's log10 is undefined there
    with pytest.raises(InfercnvB200Error) as e:
        api.seurat_snn(Y, k=5)
    assert e.value.code == -4
    with pytest.raises(InfercnvB200Error) as e:
        api.seurat_snn(X, k=5, cells=[0, 120])
    assert e.value.code == -3


@pytest.mark.skipif(EMULATED, reason="the smooth block on 184 cells: GPU only")
def test_smoothed_oligodendroglioma(oligo):
    """The oligodendroglioma fixture after the GPU smooth block, back on the linear scale (2^x, so every mean is positive
    as vst's log10 needs), all 184 cells, k = 20."""
    from oracle import oracle as orc
    cs, cl = orc.chr_ranges(oligo["chr_codes"])
    X = np.asfortranarray(np.exp2(api.smooth_block(orc.normalize_by_seq_depth(oligo["counts"]), cs, cl, oligo["ref_groups"])))
    r = api.seurat_snn(X, k=20)
    compare(X, r, 20)


@pytest.mark.skipif(EMULATED, reason="100 000 cells: GPU only")
def test_100k_cells_weight_stays_in_the_planted_clones():
    n, G = 100000, 2000
    X, lab = planted(n, G, clones=6, seed=21)
    r = api.seurat_snn(X, k=20)
    rows = np.repeat(np.arange(n), np.diff(r.indptr))
    inside = lab[rows] == lab[r.indices]
    assert r.data[inside].sum() >= 0.99 * r.data.sum()
    assert r.stats["residual"] <= 1e-12


def test_mirror_returns_the_graph_as_scipy_csr():
    from mirror import ops
    n, G = (150, 30) if EMULATED else (2000, 2500)
    X, _ = planted(n, G, seed=23)
    g = ops.leiden_seurat_preprocess_routine_graph(X, k_nn=10)
    r = api.seurat_snn(X, k=10)
    assert g.shape == (n, n) and g.format == "csr"
    assert np.array_equal(g.indptr, r.indptr) and np.array_equal(g.indices, r.indices) and np.array_equal(g.data, r.data)
