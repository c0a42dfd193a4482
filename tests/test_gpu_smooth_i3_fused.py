"""The fused i3 pass, icnv_smooth_i3_hmm_u8_f64, against the four calls it replaces.

Y must equal icnv_smooth_block_f64, the model's mu / sigma icnv_mean_sd_f64 over the reference cells of Y, the states
icnv_viterbi_u8_f64 under hmm.i3HMM_get_HMM built from the returned model, and F icnv_median_filter_f64 over the same lists -
bit for bit, over chromosome layouts, reference placements, list shapes, slab sizes and median windows.  mean_delta is
hmm.i3_mean_delta bit for bit (both are AS241).  Everything goes through the host ABI from pageable NumPy memory.
"""
import ctypes as ct

import numpy as np
import pytest

from infercnv_b200 import _lib, hmm
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

BAD_ARG = -3


@pytest.fixture(scope="module")
def api():
    from infercnv_b200 import api as a
    a.init(0)
    return a


def _layout(lens):
    lens = np.asarray(lens, dtype=np.int32)
    return np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32), lens


# the odd chromosome layouts of tests/test_gpu_cell_pipeline_variants.py
LAYOUTS = {
    "odd_ends": [301, 1, 2, 149, 77, 103, 105, 111, 0, 3, 49, 1200, 51, 99, 2, 1, 777, 0],
    "thirty": [120, 97, 88, 201, 13, 1, 64, 333, 2, 150, 101, 102, 47, 90, 500, 31, 17, 250, 3, 99, 180, 41, 60, 77, 111, 140,
               1, 200, 19, 93],
}


def _counts(rng, G, C):
    """depth-normalised-looking counts with CNV-like blocks, so that the HMM calls more than one state"""
    X = rng.gamma(2.0, 1.0, size=(G, C))
    X[G // 5: G // 3, C // 3:] *= 2.5
    X[G // 2: G // 2 + G // 8, C // 2:] *= 0.3
    return np.asfortranarray(X)


def _composition(api, X, cs, cl, refs, lists, w, p, t, window=101):
    Y = api.smooth_block(X, cs, cl, refs, window_length=window)
    mu, sigma = api.mean_sd(Y, np.concatenate(refs))
    d = hmm.i3_mean_delta(sigma, p)
    Pi, delta, mean, sd = hmm.i3HMM_get_HMM({"mu": mu, "sigma": sigma, "mean_delta": d, "KS_delta": None}, t, p)
    S = api.viterbi(Y, cs, cl, Pi, delta, mean, sd, out=np.empty(Y.shape, np.uint8, order="F"))
    F = api.median_filter(Y, cs, cl, lists, w) if lists is not None else None
    return Y, S, F, (mu, sigma, d)


def _check(api, X, cs, cl, refs, lists, w=7, p=0.05, t=1e-6, window=101):
    Y, S, F, model = api.smooth_i3_hmm(X, cs, cl, refs, i3_p_val=p, t=t, median_lists=lists, median_window=w,
                                       window_length=window)
    Y0, S0, F0, (mu, sigma, d) = _composition(api, X, cs, cl, refs, lists, w, p, t, window)
    assert np.array_equal(Y, Y0)
    assert model["mu"] == mu and model["sigma"] == sigma
    assert model["mean_delta"] == d
    assert np.array_equal(S, S0)
    if lists is None:
        assert F is None
    else:
        assert np.array_equal(F, F0)
    return S


def _subclusters(rng, cells, n_sub):
    """n_sub lists interleaved through `cells` (a real subclustering scatters a group's cells)"""
    lab = rng.integers(0, n_sub, size=len(cells))
    return [np.sort(cells[lab == k]) for k in range(n_sub) if np.any(lab == k)]


def test_bench_layout_10000_genes(api):
    import bench
    rng = np.random.default_rng(1)
    G, C = 10_000, 600
    cs, cl = bench.chr_layout(G)
    X = _counts(rng, G, C)
    refs = [np.arange(0, 36), np.arange(36, 60)]
    subs = [np.arange(a, min(a + 90, C)) for a in range(60, C, 90)]
    S = _check(api, X, cs, cl, refs, subs + refs)
    assert len(np.unique(S)) >= 2


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("w", [3, 7, 9])
def test_odd_layouts_scattered_references_interleaved_lists(api, layout, w):
    rng = np.random.default_rng(len(layout) * 10 + w)
    cs, cl = _layout(LAYOUTS[layout])
    G, C = int(cl.sum()), 260
    X = _counts(rng, G, C)
    perm = rng.permutation(C)
    refs = [np.sort(perm[:20]), np.sort(perm[20:33])]          # not the leading columns
    obs = np.sort(perm[33:])
    lists = _subclusters(rng, obs[obs < 200], 5) + refs        # cells >= 200 of the observations are in no list
    _check(api, X, cs, cl, refs, lists, w=w)


def test_no_references_proxy_group_and_no_filter(api):
    rng = np.random.default_rng(3)
    cs, cl = _layout(LAYOUTS["thirty"])
    X = _counts(rng, int(cl.sum()), 150)
    proxy = [np.arange(150)]
    _check(api, X, cs, cl, proxy, None)
    _check(api, X, cs, cl, proxy, [np.arange(0, 150, 2), np.arange(1, 150, 2)], w=7)


@pytest.mark.parametrize("p", [0.05, 0.01, 0.2, 1e-10])
def test_mean_delta_is_as241(api, p):
    from scipy.stats import norm
    rng = np.random.default_rng(4)
    cs, cl = _layout([300, 200, 500])
    X = _counts(rng, 1000, 80)
    _, _, _, model = api.smooth_i3_hmm(X, cs, cl, [np.arange(10)], i3_p_val=p)
    assert model["mean_delta"] == hmm.i3_mean_delta(model["sigma"], p)   # bitwise: both evaluate AS241 in the same order
    want = abs(norm.ppf(p, 0.0, model["sigma"]))
    assert abs(model["mean_delta"] - want) <= 1e-15 * want
    _check(api, X, cs, cl, [np.arange(10)], [np.arange(80)], p=p)


def test_lists_spanning_several_slabs(api, monkeypatch):
    """ICNV_SLAB_CELLS=64: a list spans many slabs, units hold several slabs, and runs of cells in no list are units too"""
    rng = np.random.default_rng(5)
    cs, cl = _layout(LAYOUTS["odd_ends"])
    G, C = int(cl.sum()), 700
    X = _counts(rng, G, C)
    refs = [np.arange(0, 40), np.arange(300, 330)]
    lists = [np.arange(40, 290, 3), np.arange(41, 290, 3), np.arange(400, 450), np.arange(451, 460)] + refs
    monkeypatch.setenv("ICNV_SLAB_CELLS", "64")
    api.reinit()
    try:
        _check(api, X, cs, cl, refs, lists, w=7)
        _check(api, X, cs, cl, refs, lists, w=3)
        _check(api, X, cs, cl, refs, None)
    finally:
        monkeypatch.delenv("ICNV_SLAB_CELLS")
        api.reinit()


def test_oracle_chain_on_the_bundled_example(api, oligo):
    """oracle.smooth_block -> the i3 model (oracle.i3_hmm_params) -> viterbi -> oracle.median_filter: the same states, F
    within 1e-12 relative"""
    cs, cl = orc.chr_ranges(oligo["chr_codes"])
    X = orc.normalize_by_seq_depth(oligo["counts"])
    refs = oligo["ref_groups"]
    lists = list(oligo["obs_groups"]) + list(refs)
    Y, S, F, model = api.smooth_i3_hmm(X, cs, cl, refs, median_lists=lists, median_window=7)
    Yo = orc.smooth_block(X, cs, cl, refs, nthreads=orc.max_threads())
    Pi, delta, mean, sd = orc.i3_hmm_params(Yo, np.concatenate(refs), 0.05, 1e-6)
    So = orc.viterbi_matrix(Yo, cs, cl, Pi, delta, mean, sd, nthreads=orc.max_threads())
    Fo = orc.median_filter(Yo, cs, cl, lists, 7, nthreads=orc.max_threads())
    assert np.array_equal(S.astype(np.int32), So)
    rel = np.max(np.abs(F - Fo) / np.abs(Fo))
    print(f"\n[oligodendroglioma 8508x184] i3 fused: states equal, F max rel err vs oracle {rel:.3e}")
    assert rel < 1e-12


def _raw_call(X, cs, cl, off, idx, n_grp, window, p, moff, midx, n_mf, w, Y, S, F, model):
    G, C = X.shape
    P = lambda a: None if a is None else a.ctypes.data  # noqa: E731
    return _lib.load().icnv_smooth_i3_hmm_u8_f64(P(X), P(Y), P(S), P(F), G, C, P(cs), P(cl), len(cs), P(off), P(idx), n_grp, 1,
                                                 3.0, window, 1, p, 1e-6, P(moff), P(midx), n_mf, w, P(model))


def test_errors_write_nothing(api):
    rng = np.random.default_rng(6)
    cs, cl = _layout([40, 60])
    X = _counts(rng, 100, 30)
    off, idx = np.array([0, 5], np.int32), np.arange(5, dtype=np.int32)
    moff, midx = np.array([0, 30], np.int32), np.arange(30, dtype=np.int32)
    bad_idx = midx.copy()
    bad_idx[7] = 30
    cases = [
        dict(window=100),                                   # even smoothing window
        dict(w=6), dict(w=1),                               # even / too small median window
        dict(midx=bad_idx),                                 # list index out of range
        dict(idx=np.array([0, 1, 2, 3, 31], np.int32)),     # reference index out of range
        dict(p=0.0), dict(p=1.0), dict(p=-0.5), dict(p=float("nan")),
    ]
    for case in cases:
        a = dict(window=101, w=7, p=0.05, idx=idx, midx=midx)
        a.update(case)
        Y, F = np.full((100, 30), 7.0, order="F"), np.full((100, 30), 7.0, order="F")
        S, model = np.full((100, 30), 9, np.uint8, order="F"), np.full(3, 7.0)
        rc = _raw_call(X, cs, cl, off, a["idx"], 1, a["window"], a["p"], moff, a["midx"], 1, a["w"], Y, S, F, model)
        assert rc == BAD_ARG, case
        assert np.all(Y == 7.0) and np.all(F == 7.0) and np.all(S == 9) and np.all(model == 7.0), case


def test_two_devices_match_one(api):
    if api.device_count() < 2:
        pytest.skip("needs two GPUs")
    rng = np.random.default_rng(7)
    import bench
    G, C = 10_000, 900
    cs, cl = bench.chr_layout(G)
    X = _counts(rng, G, C)
    refs = [np.arange(0, 50), np.arange(50, 90)]
    lists = _subclusters(rng, np.arange(90, 600), 4) + [np.arange(600, 900)] + refs
    one = api.smooth_i3_hmm(X, cs, cl, refs, median_lists=lists)
    try:
        assert api.init_devices([0, 1]) == 2
        two = api.smooth_i3_hmm(X, cs, cl, refs, median_lists=lists)
    finally:
        api.reinit()
    for a, b in zip(one[:3], two[:3]):
        assert np.array_equal(a, b)
    assert one[3] == two[3]


@pytest.mark.parametrize("w", [3, 7])
def test_empty_list_set_copies_y(api, w):
    """no lists: every cell is in none, so F is Y - what icnv_median_filter_f64 returns for an empty list set"""
    rng = np.random.default_rng(8)
    cs, cl = _layout(LAYOUTS["thirty"])
    X = _counts(rng, int(cl.sum()), 120)
    refs = [np.arange(0, 12), np.arange(60, 70)]
    Y, S, F, _ = api.smooth_i3_hmm(X, cs, cl, refs, median_lists=[], median_window=w)
    assert np.array_equal(F, api.median_filter(Y, cs, cl, [], w))
    assert np.array_equal(F, Y)
    _check(api, X, cs, cl, refs, [], w=w)


def test_page_locked_buffers(api):
    """page-locked input and outputs go over PCIe directly (no staging ring, F's units straight into the caller's matrix);
    the same bits as the pageable call"""
    import torch
    rng = np.random.default_rng(9)
    cs, cl = _layout(LAYOUTS["odd_ends"])
    G, C = int(cl.sum()), 3000
    X = _counts(rng, G, C)
    ref2 = np.sort(rng.choice(np.arange(150, C), 90, replace=False))   # scattered: one unit spans the whole matrix
    obs = np.setdiff1d(np.arange(150, C), ref2)
    refs = [np.arange(0, 150), ref2]
    # disjoint lists, as apply_median_filtering's subclusters and reference groups are
    lists = (_subclusters(rng, obs[obs < 1800], 6) + [obs[(obs >= 1800) & (obs < 2400)], obs[(obs >= 2500) & (obs < 2990)]]
             + refs)
    want = api.smooth_i3_hmm(X, cs, cl, refs, median_lists=lists)
    hX = torch.empty((C, G), dtype=torch.float64).pin_memory()
    hX.copy_(torch.from_numpy(X.T))
    hY = torch.empty((C, G), dtype=torch.float64).pin_memory()
    hF = torch.empty((C, G), dtype=torch.float64).pin_memory()
    hS = torch.empty((C, G), dtype=torch.uint8).pin_memory()
    off, idx = api.groups_to_csr(refs)
    moff, midx = api.groups_to_csr(lists)
    model = np.zeros(3)
    lib = _lib.load()
    _lib.check(lib.icnv_smooth_i3_hmm_u8_f64(hX.data_ptr(), hY.data_ptr(), hS.data_ptr(), hF.data_ptr(), G, C, cs.ctypes.data,
                                             cl.ctypes.data, len(cs), off.ctypes.data, idx.ctypes.data, len(refs), 1, 3.0, 101, 1,
                                             0.05, 1e-6, moff.ctypes.data, midx.ctypes.data, len(lists), 7, model.ctypes.data))
    assert np.array_equal(hY.numpy().T, want[0])
    assert np.array_equal(hS.numpy().T, want[1])
    assert np.array_equal(hF.numpy().T, want[2])
    assert (model[0], model[1], model[2]) == (want[3]["mu"], want[3]["sigma"], want[3]["mean_delta"])


def test_mirror_smooth_block_i3_hmm(api, example_object):
    """mirror.ops.smooth_block_i3_hmm: the lists apply_median_filtering builds, the states as R keeps them, the hspike
    mirrored through the plain block; without tumor_subclusters only the reference groups are filtered"""
    from mirror import ops
    ex = example_object
    cs, cl = orc.chr_ranges(ex["chr_codes"])
    X = orc.normalize_by_seq_depth(ex["counts"])
    rng = np.random.default_rng(10)
    H = rng.poisson(3.0, size=(X.shape[0], 12)).astype(float)

    def obj(subclusters):
        o = ops.Infercnv(expr_data=X, gene_order_chr=ex["chr_codes"],
                         reference_grouped_cell_indices={"normal": ex["ref_groups"][0]},
                         observation_grouped_cell_indices={"tumor": ex["obs_groups"][0]}, tumor_subclusters=subclusters)
        o.hspike = ops.Infercnv(expr_data=H, gene_order_chr=ex["chr_codes"],
                                reference_grouped_cell_indices={"simnormal": np.arange(0, 6)},
                                observation_grouped_cell_indices={"simtumor": np.arange(6, 12)})
        return o

    subs = {"subclusters": {"tumor": {"tumor_s1": ex["subclusters"][0]}}}
    refs = [np.asarray(ex["ref_groups"][0])]
    for sc, lists in ((subs, [np.asarray(ex["subclusters"][0])] + refs), (None, refs)):
        o, h, m, sd_trend = ops.smooth_block_i3_hmm(obj(sc), median_filter_window=7)
        Y, S, F, model = api.smooth_i3_hmm(X, cs, cl, refs, median_lists=lists, median_window=7)
        assert np.array_equal(o.expr_data, Y) and np.array_equal(m.expr_data, F)
        assert np.array_equal(h.expr_data, S.astype(np.float64))
        assert sd_trend == dict(model, KS_delta=None)
        assert np.array_equal(o.hspike.expr_data, api.smooth_block(H, cs, cl, [np.arange(0, 6)]))
    o, h, m, _ = ops.smooth_block_i3_hmm(obj(subs))
    assert m is None
