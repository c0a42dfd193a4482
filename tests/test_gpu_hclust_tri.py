"""K19, hclust() on the packed triangle (icnv_hclust_tri.cu), on the GPU: bit-identical to the NumPy restatement
(tests/hclust_reference.py) and to K11 (icnv_hclust_f64) for the six reducible methods, on random and tie-laden input at
sizes crossing the active mask's 32-slot words, the merge's 4096-slot batches and the scan's 8192-slot batches; icnv_cluster_cells_f64
equal to icnv_pairwise_dist_f64 -> icnv_hclust_tri_f64 and to icnv_cluster_groups_f64; planted blobs recovered at
100 000 cells, past K11's limit; the error codes.  Under the host emulation (tests/test_hclust_tri_emulated.py) only the
sizes up to 40 observations run."""
import os

import numpy as np
import pytest
from scipy.spatial.distance import pdist

from infercnv_b200 import _lib, api
from infercnv_b200._lib import InfercnvB200Error
from tests import hclust_reference as hr

pytestmark = pytest.mark.gpu
EMULATED = "_emu" in os.path.basename(_lib.LIB_PATH)
gpu_only = pytest.mark.skipif(EMULATED, reason="GPU only: too large for the host emulation")
SMALL = [2, 3, 31, 32, 33, 37, 40]
LARGE = [1025, 4096, 4097, 8192, 8193]
METHODS = sorted(hr.METHODS)


@pytest.fixture(scope="module", autouse=True)
def _init():
    api.init(0)


def random_dist(n, seed):
    return pdist(np.random.default_rng(seed).normal(size=(n, 12)))


def tie_laden(kind, n, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "duplicates":
        x = rng.normal(size=(max(n // 3, 1), 4))
        return pdist(x[rng.integers(0, len(x), size=n)])
    if kind == "integers":
        return rng.integers(1, 6, size=n * (n - 1) // 2).astype(np.float64)
    return np.full(n * (n - 1) // 2, 2.5)


def assert_bitwise(got, want):
    m, h, o = got
    rm, rh, ro = want
    assert np.array_equal(m, rm), "merge differs"
    assert np.asarray(h, np.float64).tobytes() == np.asarray(rh, np.float64).tobytes(), "height differs"
    assert np.array_equal(o, ro), "order differs"


def blobs(n, k, G, seed):
    """n cells in k well-separated blobs of G genes (centres 1000 apart on average, unit spread)."""
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, k, size=n)
    centres = rng.normal(scale=200.0, size=(k, G))
    return lab, centres[lab] + rng.normal(size=(n, G))


@pytest.mark.parametrize("n", SMALL + ([] if EMULATED else LARGE))
@pytest.mark.parametrize("method", METHODS)
def test_equals_reference_on_random_data(n, method):
    d = random_dist(n, n)
    assert_bitwise(api.hclust_tri(d, method), hr.nn_chain(d, n, hr.METHODS[method]))


@pytest.mark.parametrize("kind", ["duplicates", "integers", "equal"])
@pytest.mark.parametrize("n", [33, 40] + ([] if EMULATED else [1025]))
@pytest.mark.parametrize("method", METHODS)
def test_equals_reference_on_tie_laden_data(kind, n, method):
    d = tie_laden(kind, n)
    got = api.hclust_tri(d, method)
    assert_bitwise(got, hr.nn_chain(d, n, hr.METHODS[method]))
    hr.check_tree(d, n, hr.METHODS[method], *got)


@gpu_only
@pytest.mark.parametrize("method", METHODS)
def test_equals_the_square_kernel_at_20000(method):
    """K11 equals the restatement at this size (tests/test_gpu_hclust.py); the restatement is run here for two methods."""
    n = 20000
    d = random_dist(n, 5)
    got = api.hclust_tri(d, method)
    assert_bitwise(got, api.hclust(d, method))
    if method in ("ward.D2", "single"):
        assert_bitwise(got, hr.nn_chain(d, n, hr.METHODS[method]))


def test_host_and_device_entries_agree_and_leave_the_input():
    import torch
    if EMULATED:
        pytest.skip("needs torch device tensors")
    from infercnv_b200.device import Engine
    eng = Engine(0)
    X = torch.as_tensor(np.random.default_rng(3).normal(size=(900, 64)), device="cuda:0")   # cells x genes, row-major
    D = eng.pairwise_dist(X)
    before = D.clone()
    got = eng.hclust_tri(D, 900, "ward.D2")
    assert torch.equal(D, before)
    h = D.cpu().numpy()
    assert_bitwise(got, api.hclust_tri(h, "ward.D2"))
    assert_bitwise(got, eng.hclust(D, 900, "ward.D2"))


@gpu_only
@pytest.mark.parametrize("method", ["ward.D2", "single"])
def test_equals_the_square_kernel_at_65536(method):
    """The largest n K11 takes: its tree and K19's, one after the other on the same device vector, bit for bit."""
    import torch
    from infercnv_b200.device import Engine
    n = 65536
    _, x = blobs(n, 8, 16, 11)
    x += np.random.default_rng(12).normal(scale=30.0, size=x.shape)   # blobs that touch: a tree with real work in it
    eng = Engine(0)
    D = eng.pairwise_dist(torch.as_tensor(x, device="cuda:0"))
    torch.cuda.synchronize()
    square = eng.hclust(D, n, method)
    torch.cuda.synchronize()
    tri = eng.hclust_tri(D, n, method)
    del D
    torch.cuda.empty_cache()
    assert_bitwise(tri, square)


@pytest.mark.parametrize("keep", [None, "some", "none"])
@pytest.mark.parametrize("method", ["ward.D2", "average", "single"])
def test_cluster_cells_equals_distances_then_linkage(keep, method):
    rng = np.random.default_rng(7)
    G, C, n = 70, 300, (37 if EMULATED else 257)
    X = np.asfortranarray(rng.normal(size=(G, C)))
    cells = rng.permutation(C)[:n]
    k = {None: None, "some": np.sort(rng.permutation(G)[:45])[::-1].copy(), "none": []}[keep]
    Xk = X if k is None else np.asfortranarray(X[np.asarray(k, dtype=np.int64)])
    want = api.hclust_tri(api.pairwise_dist(Xk, cells), method)
    assert_bitwise(api.cluster_cells(X, cells, method=method, keep=k), want)
    if len(cells) <= api.HCLUST_NMAX:
        assert_bitwise(api.cluster_groups(X, [cells], method=method, keep=k)[0], want)


def test_cluster_cells_without_a_cell_list_takes_every_column():
    X = np.asfortranarray(np.random.default_rng(8).normal(size=(20, 35)))
    assert_bitwise(api.cluster_cells(X, method="complete"), api.hclust_tri(api.pairwise_dist(X), "complete"))


@gpu_only
def test_engine_cluster_cells_on_a_gene_range_view():
    import torch
    from infercnv_b200.device import Engine
    rng = np.random.default_rng(9)
    X = rng.normal(size=(3000, 200))                    # cells x genes
    cells = rng.permutation(3000)[:2500]
    eng = Engine(0)
    Xd = torch.as_tensor(X, device="cuda:0")
    got = eng.cluster_cells(Xd[:, 40:130], cells, "ward.D2")
    want = api.cluster_cells(np.asfortranarray(X[:, 40:130].T), cells, method="ward.D2")
    assert_bitwise(got, want)
    keep = rng.permutation(200)[:77]
    assert_bitwise(eng.cluster_cells(Xd, cells, "average", keep=torch.as_tensor(keep, device="cuda:0")),
                   api.cluster_cells(np.asfortranarray(X.T), cells, method="average", keep=keep))


def check_blob_tree(merge, height, order, lab, x, k):
    """merge is a valid R merge matrix, order a permutation consistent with it; cutree(k) - the clusters left after the first
    n - k merges - recovers the blobs exactly; the last k - 1 heights are Ward's closed form
    sqrt(2 |A| |B| / (|A| + |B|)) |c_A - c_B| of the clusters they join."""
    n = len(lab)
    assert merge.shape == (n - 1, 2)
    seen = np.zeros(n, bool)
    for s, (a, b) in enumerate(merge.tolist()):
        for v in (a, b):
            if v < 0:
                assert not seen[-v - 1]
                seen[-v - 1] = True
            else:
                assert 1 <= v <= s
    assert seen.all()
    assert np.all(np.diff(height) >= 0)
    assert np.array_equal(np.sort(order), np.arange(1, n + 1))
    assert np.array_equal(order, api.hclust_order(merge))
    node = lambda v: -v - 1 if v < 0 else n + v - 1   # noqa: E731  (observations 0 .. n-1, merge s -> n + s)
    parent = np.arange(2 * n - 1)
    for s in range(n - k):
        parent[node(merge[s, 0])] = parent[node(merge[s, 1])] = n + s
    root = np.empty(n, np.int64)
    for i in range(n):
        r = i
        while parent[r] != r:
            r = parent[r]
        root[i] = r
        j = i
        while parent[j] != r:   # path compression
            parent[j], j = r, parent[j]
    pairs = set(zip(lab.tolist(), root.tolist()))
    assert len(pairs) == k and len({a for a, _ in pairs}) == k and len({b for _, b in pairs}) == k
    members = {r: np.flatnonzero(root == r) for r in set(root.tolist())}
    for s in range(n - k, n - 1):
        A, B = members[node(merge[s, 0])], members[node(merge[s, 1])]
        members[n + s] = np.concatenate([A, B])
        ca, cb = x[A].mean(axis=0), x[B].mean(axis=0)
        want = np.sqrt(2.0 * len(A) * len(B) / (len(A) + len(B))) * np.linalg.norm(ca - cb)
        assert abs(height[s] - want) <= 1e-12 * want, (s, height[s], want)


@gpu_only
def test_planted_blobs_at_100000_cells_through_cluster_cells():
    n, k = 100000, 6
    lab, x = blobs(n, k, 64, 21)
    merge, height, order = api.cluster_cells(np.asfortranarray(x.T), method="ward.D2")
    check_blob_tree(merge, height, order, lab, x, k)


def _host_gb():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) / 2**20
    return 0.0


@gpu_only
def test_planted_blobs_at_100000_cells_through_hclust_tri():
    n, k = 100000, 5
    if _host_gb() < 60:
        pytest.skip("the 40 GB host \"dist\" vector needs 60 GB of free host memory")
    lab, x = blobs(n, k, 64, 22)
    d = api.pairwise_dist(np.asfortranarray(x.T))
    merge, height, order = api.hclust_tri(d, "ward.D2")
    del d
    check_blob_tree(merge, height, order, lab, x, k)


def _free_bytes():
    import torch
    return torch.cuda.mem_get_info(0)[0]


def test_error_codes():
    d = random_dist(10, 1)
    for code in (5, 6):
        with pytest.raises(InfercnvB200Error) as e:
            api.hclust_tri(d, code)
        assert e.value.code == -4
    for code in (8, -1):
        with pytest.raises(InfercnvB200Error) as e:
            api.hclust_tri(d, code)
        assert e.value.code == -3
    for bad in (np.nan, np.inf, -np.inf):
        x = d.copy()
        x[17] = bad
        with pytest.raises(InfercnvB200Error) as e:
            api.hclust_tri(x, "complete")
        assert e.value.code == -5
    with pytest.raises(InfercnvB200Error) as e:       # n = 1: an empty "dist" vector
        api.hclust_tri(np.zeros(0), "complete")
    assert e.value.code == -3
    X = np.asfortranarray(np.random.default_rng(2).normal(size=(5, 8)))
    X[3, 6] = np.nan
    with pytest.raises(InfercnvB200Error) as e:
        api.cluster_cells(X, [0, 6, 2])
    assert e.value.code == -5
    assert len(api.cluster_cells(X, [0, 1, 2])[0]) == 2      # the NaN's column is not listed
    with pytest.raises(InfercnvB200Error) as e:
        api.cluster_cells(X, [0, 8])
    assert e.value.code == -3
    with pytest.raises(InfercnvB200Error) as e:
        api.cluster_cells(X, [0, 1], keep=[5])
    assert e.value.code == -3
    with pytest.raises(InfercnvB200Error) as e:
        api.cluster_cells(X, [0])
    assert e.value.code == -3


@gpu_only
def test_a_triangle_that_cannot_fit_is_refused_before_anything_is_allocated():
    """n = 200 000 needs 160 GB: ICNV_E_NOMEM from every entry point, with the free device memory unchanged (the host
    vector is never read, so a stand-in of four doubles is passed)."""
    lib = _lib.load()
    n = 200000
    one = np.zeros(4)
    m, h, o = np.zeros(4, np.int32), np.zeros(4), np.zeros(4, np.int32)
    api.hclust_tri(random_dist(10, 1), "ward.D2")       # the context and its scratch exist before the measurement
    before = _free_bytes()
    assert lib.icnv_hclust_tri_f64(one.ctypes.data, n, 7, m.ctypes.data, h.ctypes.data, o.ctypes.data) == -7
    assert lib.icnv_dev_hclust_tri_f64(one.ctypes.data, n, 7, m.ctypes.data, h.ctypes.data, None) == -7
    X = np.zeros((2, 4))
    assert lib.icnv_cluster_cells_f64(X.ctypes.data, 2, n, None, 0, None, 0, 7, m.ctypes.data, h.ctypes.data,
                                      o.ctypes.data) == -7
    assert _free_bytes() == before
    assert b"device memory" in lib.icnv_last_error()
