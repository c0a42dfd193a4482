"""K12, the exact k-nearest-neighbour kernel (icnv_dist.cu; RANN::nn2 with the query set = the data set), on the GPU.

The oracle is K10 itself: the kernel reports the roots of the very sums K10 roots, so `idx` and the bits of `dist` must
equal tests/knn_reference.py applied to api.pairwise_dist / pairwise_dist_rows of the same input.  Under the host
emulation (tests/test_knn_emulated_and_r.py) only the sizes up to 257 cells run; there the split rule picks one or two
splits (4 emulated SMs), while on the H100 (132 SMs) the sizes from 129 to 20 000 cells run with three to eight."""
import os

import numpy as np
import pytest

from infercnv_b200 import _lib, api
from infercnv_b200._lib import InfercnvB200Error
from tests import knn_reference as kr

pytestmark = pytest.mark.gpu
EMULATED = "_emu" in os.path.basename(_lib.LIB_PATH)
SIZES = [1, 2, 127, 128, 129, 255, 257] + ([] if EMULATED else [1000, 4097, 20000])
GENES = [0, 1, 15, 16, 17, 455] + ([] if EMULATED else [10000])


def ks(n):
    return sorted({k for k in (1, 2, 20, 64) if k <= n} | ({n} if n <= 64 else set()))


def expected(d, n, k):
    """The first k of every row from K10's vector (computed once at the largest k: the order is total, so the first k
    of the first K are the first k)."""
    return kr.knn_from_dist(d, n, k)


def assert_bitwise(got, want, k):
    gi, gd = got
    wi, wd = want
    assert gi.shape == (wi.shape[0], k) and gd.shape == (wi.shape[0], k)
    assert np.array_equal(gi, wi[:, :k]), "idx differs"
    assert np.array_equal(np.ascontiguousarray(gd).view(np.int64), np.ascontiguousarray(wd[:, :k]).view(np.int64)), \
        "dist differs"


@pytest.fixture(scope="module", autouse=True)
def _init():
    api.init(0)


@pytest.mark.parametrize("layout", ["genes_x_cells", "rows"])
@pytest.mark.parametrize("n", SIZES)
def test_equals_k10_over_sizes_and_k(n, layout):
    x = np.random.default_rng(n).normal(size=(n, 17))          # observations x variables
    if layout == "rows":
        d, run = api.pairwise_dist_rows(x), lambda k: api.knn_rows(x, k)
    else:
        X = np.asfortranarray(x.T)
        d, run = api.pairwise_dist(X), lambda k: api.knn(X, k)
    want = expected(d, n, max(ks(n)))
    for k in ks(n):
        assert_bitwise(run(k), want, k)
    assert np.array_equal(want[0][:, 0], np.arange(n))          # tie-free: self first


@pytest.mark.parametrize("layout", ["genes_x_cells", "rows"])
@pytest.mark.parametrize("G", GENES)
def test_equals_k10_over_gene_counts(G, layout):
    n = 129 if EMULATED else 1000
    x = np.random.default_rng(G).normal(size=(n, G))
    if layout == "rows":
        d, got = api.pairwise_dist_rows(x), {k: api.knn_rows(x, k) for k in (20, 64)}
    else:
        X = np.asfortranarray(x.T)
        d, got = api.pairwise_dist(X), {k: api.knn(X, k) for k in (20, 64)}
    want = expected(d, n, 64)
    for k in (20, 64):
        assert_bitwise(got[k], want, k)
    if G == 0:
        assert np.array_equal(got[64][0], np.tile(np.arange(64, dtype=np.int32), (n, 1)))
        assert np.all(got[64][1] == 0.0)


@pytest.mark.parametrize("kind", ["shuffled", "repeated"])
def test_cell_lists(kind):
    rng = np.random.default_rng(7)
    C = 300 if EMULATED else 3000
    X = np.asfortranarray(rng.normal(size=(40, C)))
    cells = rng.permutation(C)[:C - 31] if kind == "shuffled" else rng.integers(0, C, size=C // 2 + 5)
    n = len(cells)
    d = api.pairwise_dist(X, cells)
    want = expected(d, n, 64)
    for k in (1, 20, 64):
        assert_bitwise(api.knn(X, k, cells), want, k)


@pytest.mark.parametrize("kind", ["duplicates", "all_equal", "integers"])
@pytest.mark.parametrize("n", [129, 257] + ([] if EMULATED else [4097]))
def test_tie_laden_cells(kind, n):
    rng = np.random.default_rng(n)
    if kind == "duplicates":
        base = rng.normal(size=(max(n // 5, 1), 9))
        x = base[rng.integers(0, len(base), size=n)]
    elif kind == "all_equal":
        x = np.full((n, 9), -1.25)
    else:
        x = rng.integers(0, 3, size=(n, 6)).astype(np.float64)
    d = api.pairwise_dist_rows(x)
    want = expected(d, n, 64)
    for k in (2, 20, 64):
        assert_bitwise(api.knn_rows(x, k), want, k)
    if kind == "all_equal":
        assert np.array_equal(want[0], np.tile(np.arange(64, dtype=np.int32), (n, 1)))


@pytest.mark.skipif(EMULATED, reason="needs torch device tensors")
def test_engine_on_a_gene_range_view_equals_the_host_api():
    import torch
    from infercnv_b200.device import Engine
    eng = Engine(0)
    rng = np.random.default_rng(5)
    x = rng.normal(size=(3001, 600))                           # cells x genes, row-major on the device
    X = torch.as_tensor(x, device="cuda:0")
    a, b = 137, 137 + 211                                      # one "chromosome"
    cells = rng.permutation(3001)[:2500]
    for sel in (None, cells):
        gi, gd = eng.knn(X[:, a:b], 20, sel)
        torch.cuda.synchronize()
        sub = x[:, a:b] if sel is None else x[sel, a:b]
        wi, wd = api.knn_rows(np.ascontiguousarray(sub), 20)
        assert np.array_equal(gi.cpu().numpy(), wi)
        assert np.array_equal(gd.cpu().numpy().view(np.int64), np.ascontiguousarray(wd).view(np.int64))


@pytest.mark.skipif(EMULATED, reason="the smooth block on 184 cells: GPU only")
def test_smoothed_oligodendroglioma_per_chromosome(oligo):
    """The smoothed c1 matrix (the GPU smooth block on the oligodendroglioma fixture), k = 20 per chromosome over all
    cells, as the per-chromosome Leiden subclustering asks: equal to the helper on K10's distances."""
    from oracle import oracle as orc
    cs, cl = orc.chr_ranges(oligo["chr_codes"])
    X = np.asfortranarray(api.smooth_block(orc.normalize_by_seq_depth(oligo["counts"]), cs, cl, oligo["ref_groups"]))
    n = X.shape[1]
    for s, ln in zip(cs, cl):
        Xc = np.asfortranarray(X[s:s + ln])
        want = expected(api.pairwise_dist(Xc), n, 20)
        assert_bitwise(api.knn(Xc, 20), want, 20)
        assert_bitwise(api.knn_rows(np.ascontiguousarray(Xc.T), 20), want, 20)


@pytest.mark.skipif(EMULATED, reason="150 000 cells: GPU only")
def test_past_the_65536_cell_cap_planted_blobs():
    """150 000 cells x 64 genes in 8 well-separated blobs (more cells than K10 or the linkage take): every neighbour is in
    its cell's blob, and 200 sampled rows equal a NumPy brute force - the same sets wherever the k-th / (k+1)-th gap exceeds
    1e-12 relative, distances within 1e-13."""
    n, G, k, nb = 150000, 64, 20, 8
    rng = np.random.default_rng(17)
    lab = rng.integers(0, nb, size=n)
    x = rng.normal(scale=50.0, size=(nb, G))[lab] + rng.normal(size=(n, G))
    idx, dist = api.knn_rows(x, k)
    assert np.all(lab[idx] == lab[:, None])
    assert np.all(np.diff(dist, axis=1) >= 0)
    for i in rng.choice(n, size=200, replace=False):
        sq = np.sum((x - x[i]) ** 2, axis=1)
        order = np.lexsort((np.arange(n), sq))[:k + 1]
        ref = np.sqrt(sq[order])
        np.testing.assert_allclose(dist[i], ref[:k], rtol=1e-13, atol=1e-13)
        if ref[k] - ref[k - 1] > 1e-12 * ref[k]:
            assert set(idx[i].tolist()) == set(order[:k].tolist()), i


def test_error_codes_and_edges():
    x = np.random.default_rng(2).normal(size=(100, 7))
    for k in (0, -1, 101):
        with pytest.raises(InfercnvB200Error) as e:
            api.knn_rows(x, k)
        assert e.value.code == -3
    with pytest.raises(InfercnvB200Error) as e:
        api.knn_rows(x, 65)
    assert e.value.code == -4
    for bad in (np.nan, np.inf, -np.inf):
        y = x.copy()
        y[57, 3] = bad
        with pytest.raises(InfercnvB200Error) as e:
            api.knn_rows(y, 5)
        assert e.value.code == -5
        with pytest.raises(InfercnvB200Error) as e:
            api.knn(np.asfortranarray(y.T), 5)
        assert e.value.code == -5
    y = x.copy()
    y[57, 3] = np.nan
    idx, _ = api.knn(np.asfortranarray(y.T), 5, cells=[0, 1, 2, 3, 4, 5])   # the bad cell is not listed
    assert idx.shape == (6, 5)
    idx, dist = api.knn_rows(np.zeros((0, 5)), 3)                           # n = 0: nothing to write
    assert idx.size == 0 and dist.size == 0
    lib = _lib.load()
    one = np.zeros(64)
    out_i, out_d = np.zeros(64, np.int32), np.zeros(64)
    assert lib.icnv_dev_knn_f64(one.ctypes.data, 1, 1, None, 1, 2, out_i.ctypes.data, out_d.ctypes.data, None) == -3
    assert lib.icnv_knn_f64(one.ctypes.data, 1, 8, None, 8, 0, out_i.ctypes.data, out_d.ctypes.data) == -3


def test_repeated_calls_return_the_same_bytes():
    n = 257 if EMULATED else 4097
    x = np.random.default_rng(9).integers(0, 4, size=(n, 5)).astype(np.float64)
    a, b = api.knn_rows(x, 64), api.knn_rows(x, 64)
    assert np.array_equal(a[0], b[0])
    assert np.array_equal(a[1].view(np.int64), b[1].view(np.int64))
