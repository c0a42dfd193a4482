"""K13 on the GPU: the running mean (icnv_runmean_f64) within the bound of tests/runmean_reference.py, and the random-trees
null (icnv_random_tree_heights_f64) bit for bit equal to the composition runmean -> center -> pairwise_dist -> hclust, for
the observed tree and for every permuted member rebuilt in NumPy.  Under the host emulation
(tests/test_random_trees_emulated_and_r.py) only clades of up to 33 cells run."""
import os

import numpy as np
import pytest

from infercnv_b200 import _lib, api
from infercnv_b200._lib import InfercnvB200Error
from tests import runmean_reference as rr

pytestmark = pytest.mark.gpu
EMULATED = "_emu" in os.path.basename(_lib.LIB_PATH)
METHODS = ["single", "complete", "average", "mcquitty", "ward.D", "ward.D2"]
gpu_only = pytest.mark.skipif(EMULATED, reason="GPU only: too large for the host emulation")


@pytest.fixture(scope="module", autouse=True)
def _init():
    api.init(0)


def layout(G):
    """Ranges with short, one-gene, even-length ranges and gaps (genes outside every range)."""
    if G < 4:
        return [0], [G]
    lens = [1, 2, 40, 101, 102, 997]
    starts, pos = [], 1   # gene 0 in no range
    out_l = []
    for L in lens:
        if pos + L > G:
            break
        starts.append(pos)
        out_l.append(L)
        pos += L + 1      # one gene between ranges
    if pos < G - 1:
        starts.append(pos)
        out_l.append(G - 1 - pos)
    return starts, out_l


@pytest.mark.parametrize("k", [1, 3, 51, 101, 102])
@pytest.mark.parametrize("G", [1, 2, 100, 101, 102, 10000])
def test_runmean_within_the_bound(G, k):
    rng = np.random.default_rng(G * 7 + k)
    X = rng.normal(size=(G, 3)) * np.array([1.0, 1e6, 1e-6]) + np.array([0.0, 3e6, -1.0])
    rr.check_runmean(api.runmean(X, k), X, k)
    cs, cl = layout(G)
    Y = api.runmean(X, k, cs, cl)
    rr.check_runmean(Y, X, k, cs, cl)
    inside = np.zeros(G, bool)
    for s, L in zip(cs, cl):
        inside[s:s + L] = True
        assert np.array_equal(api.runmean(X[s:s + L], k), Y[s:s + L])   # per range == whole call, bit for bit
    assert np.array_equal(Y[~inside], X[~inside])


def test_runmean_errors():
    X = np.ones((10, 2))
    with pytest.raises(InfercnvB200Error) as e:
        api.runmean(X, 3, [0, 4], [5, 3])            # overlapping ranges
    assert e.value.code == -3
    X[3, 1] = np.nan
    with pytest.raises(InfercnvB200Error) as e:
        api.runmean(X, 3)
    assert e.value.code == -5


def composed(Xc, window, method):
    """The observed tree as separate calls: runmean -> median centring -> distances -> hclust."""
    c = api.center(api.runmean(Xc, window), "median")
    return api.hclust(api.pairwise_dist(c), method)


def clade(G, n, seed, planted=False):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(G, n))
    if planted:
        X[: G // 3, : n // 2] += 1.5
    return X


def assert_tree(got, want):
    m, h, o = got[:3]
    wm, wh, wo = want
    assert np.array_equal(m, wm), "merge differs"
    assert np.array_equal(h.view(np.int64), wh.view(np.int64)), "height differs"
    assert np.array_equal(o, wo), "order differs"


@pytest.mark.parametrize("n", [2, 3, 33] + ([] if EMULATED else [257, 2000]))
@pytest.mark.parametrize("method", METHODS)
def test_observed_tree_equals_the_composition(n, method):
    X = clade(300, n, n, planted=True)
    got = api.random_tree_heights(X, window=51, method=method, n_perm=0, seed=1)
    assert got[3].size == 0
    assert_tree(got, composed(X, 51, method))


def member_max(Xc, seed, p, window, method):
    return composed(rr.permuted(Xc, seed, p), window, method)[1].max()


@pytest.mark.parametrize("n_perm", [1, 7] + ([] if EMULATED else [150]))
def test_permuted_members_equal_the_composition(n_perm):
    n = 33 if EMULATED else 120
    X = clade(200, n, 11, planted=True)
    seed = 987654321
    merge, height, order, pm = api.random_tree_heights(X, window=101, method="ward.D2", n_perm=n_perm, seed=seed)
    assert pm.shape == (n_perm,)
    want = np.array([member_max(X, seed, p, 101, "ward.D2") for p in range(n_perm)])
    assert np.array_equal(pm.view(np.int64), want.view(np.int64))
    st = api.random_trees_stats()
    assert st["waves"] == -(-(n_perm + 1) // st["B"]) and 1 <= st["B"] <= n_perm + 1
    if n_perm == 150:
        assert st["waves"] >= 2


@pytest.mark.parametrize("method", METHODS)
def test_permuted_members_every_method(method):
    X = clade(120, 17, 5)
    _, _, _, pm = api.random_tree_heights(X, window=3, method=method, n_perm=5, seed=3)
    want = np.array([member_max(X, 3, p, 3, method) for p in range(5)])
    assert np.array_equal(pm.view(np.int64), want.view(np.int64))


def test_prefix_property_and_seeds():
    X = clade(150, 30, 2, planted=True)
    many = 12 if EMULATED else 150
    few = 5 if EMULATED else 50
    a = api.random_tree_heights(X, window=21, n_perm=many, seed=77)
    b = api.random_tree_heights(X, window=21, n_perm=few, seed=77)
    assert np.array_equal(a[3][:few].view(np.int64), b[3].view(np.int64))
    for u, v in zip(a[:3], b[:3]):
        assert np.array_equal(u, v)
    c = api.random_tree_heights(X, window=21, n_perm=many, seed=77)
    for u, v in zip(a, c):
        assert u.tobytes() == v.tobytes()
    d = api.random_tree_heights(X, window=21, n_perm=many, seed=78)
    assert not np.array_equal(a[3], d[3])
    assert np.array_equal(a[1], d[1])   # the observed tree does not depend on the seed


def test_cell_list_equals_the_dense_call():
    X = clade(100, 60, 4, planted=True)
    cells = np.random.default_rng(0).permutation(60)[:29]
    a = api.random_tree_heights(X, window=11, n_perm=6, seed=5, cells=cells)
    b = api.random_tree_heights(np.asfortranarray(X[:, cells]), window=11, n_perm=6, seed=5)
    for u, v in zip(a, b):
        assert u.tobytes() == v.tobytes()


def test_tie_heavy_input_is_repeatable():
    X = np.round(clade(80, 31, 9) * 2) / 2
    a = api.random_tree_heights(X, window=1, method="average", n_perm=6, seed=1)
    b = api.random_tree_heights(X, window=1, method="average", n_perm=6, seed=1)
    for u, v in zip(a, b):
        assert u.tobytes() == v.tobytes()
    assert_tree(a, composed(X, 1, "average"))


def test_error_codes():
    X = clade(20, 5, 0)
    for kw, code in [(dict(cells=[0]), -3), (dict(method=8), -3), (dict(n_perm=-1), -3), (dict(method="centroid"), -4),
                     (dict(method="median"), -4)]:
        kw = dict(kw)
        method = kw.pop("method", "ward.D2")
        if isinstance(method, str) and method in ("centroid", "median"):
            method = {"centroid": 5, "median": 6}[method]
        with pytest.raises(InfercnvB200Error) as e:
            api.random_tree_heights(X, method=method, **kw)
        assert e.value.code == code, kw
    with pytest.raises(InfercnvB200Error) as e:
        api.random_tree_heights(np.zeros((1, 65537)), n_perm=1)
    assert e.value.code == -4
    Y = X.copy()
    Y[3, 2] = np.inf
    with pytest.raises(InfercnvB200Error) as e:
        api.random_tree_heights(Y, n_perm=2)
    assert e.value.code == -5


@gpu_only
def test_planted_clades_beat_the_null_and_noise_does_not():
    G, half = 2000, 300
    rng = np.random.default_rng(42)
    X = rng.normal(size=(G, 2 * half))
    X[200:600, :half] += 1.0        # one whole "chromosome" offset in the first clade
    _, h, _, pm = api.random_tree_heights(X, window=101, n_perm=100, seed=2024)
    assert h.max() > pm.max()
    N = rng.normal(size=(G, 2 * half))
    _, h, _, pm = api.random_tree_heights(N, window=101, n_perm=100, seed=2024)
    assert h.max() <= pm.max()


@gpu_only
def test_engine_and_ops_mirror():
    import torch
    from infercnv_b200.device import Engine
    from mirror import ops
    X = clade(500, 90, 8, planted=True)
    cells = np.random.default_rng(1).permutation(90)[:70]
    want = api.random_tree_heights(X, window=101, n_perm=20, seed=9, cells=cells)
    eng = Engine(0)
    T = torch.as_tensor(np.ascontiguousarray(X.T), device=eng.tdev)
    got = eng.random_tree_heights(T, cells=cells, window=101, n_perm=20, seed=9)
    for u, v in zip(got, want):
        assert np.asarray(u).tobytes() == np.asarray(v).tobytes()
    r = ops.parameterize_random_cluster_heights_smoothed_trees(X[:, cells], "ward.D2", 101, n_perm=20, seed=9)
    assert np.array_equal(r["rand_max_height_dist"], want[3]) and r["max_h"] == want[1].max()
    assert np.array_equal(ops.runmean(X[:, 0], 101), api.runmean(X[:, :1], 101)[:, 0])


@gpu_only
def test_full_size_clade():
    X = clade(10000, 8000, 1, planted=True)
    merge, height, order, pm = api.random_tree_heights(X, window=101, n_perm=100, seed=1)
    assert merge.shape == (7999, 2) and np.all(np.isfinite(pm)) and pm.shape == (100,)
    assert np.array_equal(np.sort(order), np.arange(1, 8001))
