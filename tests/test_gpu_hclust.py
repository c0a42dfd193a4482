"""K11, the hclust() linkage kernel (icnv_hclust.cu), on the GPU: bit-identical to the NumPy restatement of its rules
(tests/hclust_reference.py, itself pinned by scipy, a literal transcription and the reference's stored trees) for the six
reducible methods, on random and tie-laden input.  Under the host emulation (tests/test_hclust_emulated_and_r.py) only the sizes
up to 33 observations run: the emulation runs a 1024-thread block as fibers, about 30 ms per row scan."""
import os

import numpy as np
import pytest
from scipy.spatial.distance import pdist

from infercnv_b200 import _lib, api
from infercnv_b200._lib import InfercnvB200Error
from tests import hclust_reference as hr

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = "_emu" in os.path.basename(_lib.LIB_PATH)
SIZES = [2, 3, 31, 32, 33] + ([] if EMULATED else [1023, 1024, 1025, 4097])
METHODS = sorted(hr.METHODS)


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
    assert np.array_equal(h.view(np.int64), rh.view(np.int64)), "height differs"
    assert np.array_equal(o, ro), "order differs"


@pytest.fixture(scope="module", autouse=True)
def _init():
    api.init(0)


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("method", METHODS)
def test_gpu_equals_reference_on_random_data(n, method):
    d = random_dist(n, n)
    assert_bitwise(api.hclust(d, method), hr.nn_chain(d, n, hr.METHODS[method]))


@pytest.mark.parametrize("kind", ["duplicates", "integers", "equal"])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("method", METHODS)
def test_gpu_equals_reference_on_tie_laden_data(kind, n, method):
    d = tie_laden(kind, n)
    got = api.hclust(d, method)
    assert_bitwise(got, hr.nn_chain(d, n, hr.METHODS[method]))
    hr.check_tree(d, n, hr.METHODS[method], *got)


@pytest.mark.skipif(EMULATED, reason="20 000 observations: GPU only")
@pytest.mark.parametrize("method", METHODS)
def test_gpu_equals_reference_at_20000(method):
    n = 20000
    d = random_dist(n, 5)
    assert_bitwise(api.hclust(d, method), hr.nn_chain(d, n, hr.METHODS[method]))


def test_reference_trees_through_the_ops_mirror():
    """`hclust(parallelDist(t(expr[, cells])), "ward.D2")` on the pre-denoise smooth block reproduces both trees stored in
    the reference's example object."""
    from mirror import ops
    from oracle import oracle as orc
    z = np.load(os.path.join(ROOT, "tests", "golden", "example_object.npz"))
    h = np.load(os.path.join(ROOT, "tests", "golden", "example_hclust.npz"))
    cs, cl = orc.chr_ranges(z["chr_codes"])
    refs = [z["ref_idx"] - 1]
    X = orc.smooth_block(orc.normalize_by_seq_depth(z["counts"].astype(np.float64)), cs, cl, refs)
    for name in ("tumor", "normal"):
        hc = ops.hclust(ops.parallelDist(X[:, h[f"{name}_cols"]].T), "ward.D2")
        assert np.array_equal(hc["merge"], h[f"{name}_merge"]), name
        assert np.array_equal(hc["order"], h[f"{name}_order"]), name
        np.testing.assert_allclose(hc["height"], h[f"{name}_height"], rtol=1e-13, atol=0)


@pytest.mark.skipif(EMULATED, reason="needs torch device tensors")
@pytest.mark.parametrize("method", ["ward.D2", "average", "single"])
def test_engine_on_a_device_vector_equals_the_host_api(method):
    import torch
    from infercnv_b200.device import Engine
    eng = Engine(0)
    X = torch.as_tensor(np.random.default_rng(3).normal(size=(700, 64)), device="cuda:0")   # cells x genes, row-major
    D = eng.pairwise_dist(X)
    torch.cuda.synchronize()
    got = eng.hclust(D, 700, method)
    assert_bitwise(got, api.hclust(D.cpu().numpy(), method))


def test_two_runs_are_bit_identical():
    n = 33 if EMULATED else 3001
    d = tie_laden("integers", n, 9)
    assert_bitwise(api.hclust(d, "ward.D2"), api.hclust(d, "ward.D2"))


def test_error_codes():
    d = random_dist(10, 1)
    for code in (5, 6):
        with pytest.raises(InfercnvB200Error) as e:
            api.hclust(d, code)
        assert e.value.code == -4
    for code in (8, -1):
        with pytest.raises(InfercnvB200Error) as e:
            api.hclust(d, code)
        assert e.value.code == -3
    for bad in (np.nan, np.inf, -np.inf):
        x = d.copy()
        x[17] = bad
        with pytest.raises(InfercnvB200Error) as e:
            api.hclust(x, "complete")
        assert e.value.code == -5
    with pytest.raises(InfercnvB200Error) as e:       # n = 1: an empty "dist" vector
        api.hclust(np.zeros(0), "complete")
    assert e.value.code == -3
    lib = _lib.load()
    one = np.zeros(4)
    m, h, o = np.zeros(4, np.int32), np.zeros(4), np.zeros(4, np.int32)
    assert lib.icnv_hclust_f64(one.ctypes.data, 65537, 7, m.ctypes.data, h.ctypes.data, o.ctypes.data) == -4
    assert lib.icnv_dev_hclust_f64(one.ctypes.data, 65537, 7, m.ctypes.data, h.ctypes.data, None) == -4
    assert lib.icnv_dev_hclust_f64(one.ctypes.data, 1, 7, m.ctypes.data, h.ctypes.data, None) == -3


@pytest.mark.skipif(EMULATED, reason="65 536 observations: GPU only")
def test_full_size_planted_blobs_are_recovered():
    """n = 65 536 (34 GB matrix) with 8 well-separated blobs: the tree is valid where it can be checked cheaply, and cutting
    it into 8 clusters recovers the blobs exactly."""
    from scipy.cluster.hierarchy import fcluster
    import torch
    from infercnv_b200.device import Engine
    n, k = 65536, 8
    rng = np.random.default_rng(11)
    lab = rng.integers(0, k, size=n)
    centres = rng.normal(scale=50.0, size=(k, 16))
    x = centres[lab] + rng.normal(size=(n, 16))
    eng = Engine(0)
    D = eng.pairwise_dist(torch.as_tensor(x, device="cuda:0"))
    merge, height, order = eng.hclust(D, n, "ward.D2")
    del D
    torch.cuda.empty_cache()
    assert np.all(np.diff(height) >= 0)
    assert np.array_equal(np.sort(order), np.arange(1, n + 1))
    assert np.array_equal(order, api.hclust_order(merge))
    Z = np.zeros((n - 1, 4))                    # R's merge -> scipy's linkage for fcluster
    to = lambda v: -v - 1 if v < 0 else n + v - 1     # noqa: E731
    Z[:, 0] = [to(v) for v in merge[:, 0]]
    Z[:, 1] = [to(v) for v in merge[:, 1]]
    Z[:, 2] = height
    cnt = np.ones(2 * n - 1)
    for s in range(n - 1):
        cnt[n + s] = cnt[int(Z[s, 0])] + cnt[int(Z[s, 1])]
    Z[:, 3] = cnt[n:]
    cut = fcluster(Z, k, criterion="maxclust")
    pairs = {(a, b) for a, b in zip(lab.tolist(), cut.tolist())}
    assert len(pairs) == k and len({a for a, _ in pairs}) == k and len({b for _, b in pairs}) == k
