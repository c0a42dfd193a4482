"""The fused group-mode calls, icnv_smooth_hmm_groups_u8_f64 (i6) and icnv_smooth_i3_hmm_groups_u8_f64 (i3), against the
composition they replace: smooth_block, then viterbi(groups=...) on its output.

Y must equal icnv_smooth_block_f64, the states icnv_viterbi_u8_f64 over the same HMM lists (i3: under
hmm.i3HMM_get_HMM of the returned model, which must equal the per-cell i3 call's) - bit for bit, over chromosome layouts,
reference placements, list shapes and sizes, slab sizes and buffer kinds.  Everything goes through the host ABI.
"""
import os

import numpy as np
import pytest

from infercnv_b200 import _lib, hmm
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

BAD_ARG = -3
EMULATED = "_emu" in os.path.basename(_lib.LIB_PATH)
gpu_only = pytest.mark.skipif(EMULATED, reason="GPU only: too large for the host emulation, or needs page-locked memory")


@pytest.fixture(scope="module")
def api():
    from infercnv_b200 import api as a
    a.init(0)
    return a


def _layout(lens):
    lens = np.asarray(lens, dtype=np.int32)
    return np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32), lens


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


def _i6(groups):
    """an i6 model on the scale of the block's output (about 1) and per-group sds that shrink with the group's size, as
    .get_state_emission_params makes them"""
    Pi, delta = orc.hmm_params(6, 1e-6)
    mean = np.array([0.01, 0.5, 1.0, 1.5, 2.0, 3.0])
    base = np.array([0.05, 0.12, 0.1, 0.14, 0.2, 0.3])
    sd = np.concatenate([base * (1.0 + 3.0 / np.sqrt(len(g))) for g in groups])
    return Pi, delta, mean, sd


def _check_i6(api, X, cs, cl, refs, groups, window=101):
    Pi, delta, mean, sd = _i6(groups)
    Y, S = api.smooth_hmm(X, cs, cl, refs, Pi, delta, mean, sd, window_length=window, groups=groups)
    Y0 = api.smooth_block(X, cs, cl, refs, window_length=window)
    S0 = api.viterbi(Y0, cs, cl, Pi, delta, mean, sd, groups=groups, out=np.empty(Y0.shape, np.uint8, order="F"))
    assert np.array_equal(Y, Y0)
    assert np.array_equal(S, S0)
    return S


def _check_i3(api, X, cs, cl, refs, groups, p=0.05, t=1e-6, window=101):
    Y, S, F, model = api.smooth_i3_hmm(X, cs, cl, refs, i3_p_val=p, t=t, window_length=window, groups=groups)
    assert F is None
    Y0 = api.smooth_block(X, cs, cl, refs, window_length=window)
    mu, sigma = api.mean_sd(Y0, np.concatenate(refs))
    d = hmm.i3_mean_delta(sigma, p)
    assert (model["mu"], model["sigma"], model["mean_delta"]) == (mu, sigma, d)
    Pi, delta, mean, sd = hmm.i3HMM_get_HMM({"mu": mu, "sigma": sigma, "mean_delta": d, "KS_delta": None}, t, p)
    S0 = api.viterbi(Y0, cs, cl, Pi, delta, mean, np.tile(sd, len(groups)), groups=groups,
                     out=np.empty(Y0.shape, np.uint8, order="F"))
    assert np.array_equal(Y, Y0)
    assert np.array_equal(S, S0)
    return S, model


def _check(api, X, cs, cl, refs, groups, window=101):
    S6 = _check_i6(api, X, cs, cl, refs, groups, window)
    S3, _ = _check_i3(api, X, cs, cl, refs, groups, window=window)
    return S6, S3


def _subclusters(rng, cells, n_sub):
    """n_sub lists interleaved through `cells` (a real subclustering scatters a group's cells)"""
    lab = rng.integers(0, n_sub, size=len(cells))
    return [np.sort(cells[lab == k]) for k in range(n_sub) if np.any(lab == k)]


@gpu_only
def test_bench_layout_10000_genes_samples(api):
    import bench
    rng = np.random.default_rng(1)
    G, C = 10_000, 600
    cs, cl = bench.chr_layout(G)
    X = _counts(rng, G, C)
    refs = [np.arange(0, 36), np.arange(36, 60)]
    obs = [np.arange(a, min(a + 90, C)) for a in range(60, C, 90)]
    S6, S3 = _check(api, X, cs, cl, refs, obs + refs)
    assert len(np.unique(S6)) >= 2 and len(np.unique(S3)) >= 2
    # the per-cell i3 call fixes the same model
    _, model = _check_i3(api, X, cs, cl, refs, obs + refs)
    assert api.smooth_i3_hmm(X, cs, cl, refs)[3] == model


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("mode", ["samples", "one_cell_samples", "subclusters"])
def test_odd_layouts_scattered_references(api, layout, mode):
    rng = np.random.default_rng(len(layout) * 10 + len(mode))
    cs, cl = _layout(LAYOUTS[layout])
    G, C = int(cl.sum()), 200
    X = _counts(rng, G, C)
    perm = rng.permutation(C)
    refs = [np.sort(perm[:20]), np.sort(perm[20:33])]          # not the leading columns
    obs = np.sort(perm[33:])
    if mode == "samples":                                       # cluster_by_groups = TRUE: annotation groups, then refs
        groups = _subclusters(rng, obs, 3) + refs
    elif mode == "one_cell_samples":                            # cluster_by_groups = FALSE: every observation cell alone
        groups = [np.array([c]) for c in obs] + refs
    else:                                                       # interleaved subclusters of both kinds of cells
        groups = _subclusters(rng, obs, 7) + _subclusters(rng, np.concatenate(refs), 2)
    _check(api, X, cs, cl, refs, groups)


@pytest.mark.parametrize("slab", [None, "64"])
def test_group_sizes_around_the_chunk(api, monkeypatch, slab):
    """groups of 1, 31, 32, 33 and 1000 cells: chunks end inside, at and past a slab; with 64-cell slabs a group spans
    many slabs and a slab holds many groups"""
    rng = np.random.default_rng(2)
    cs, cl = _layout([300, 200, 500])
    G, C = 1000, 1300
    X = _counts(rng, G, C)
    perm = rng.permutation(C)
    refs = [np.sort(perm[:40])]
    sizes = [1, 31, 32, 33, 1000, 1, 1, 33, 31]
    at = np.cumsum([40] + sizes)
    groups = [perm[a:b] for a, b in zip(at[:-1], at[1:])] + refs   # in permutation order: list order is not column order
    if slab:
        monkeypatch.setenv("ICNV_SLAB_CELLS", slab)
        api.reinit()
    try:
        _check(api, X, cs, cl, refs, groups)
    finally:
        if slab:
            monkeypatch.delenv("ICNV_SLAB_CELLS")
            api.reinit()


def test_overlapping_lists_and_unlisted_cells(api, monkeypatch):
    """a cell in several lists takes the last one's trace; cells in no list get 255"""
    rng = np.random.default_rng(3)
    cs, cl = _layout(LAYOUTS["thirty"])
    G, C = int(cl.sum()), 300
    X = _counts(rng, G, C)
    refs = [np.arange(0, 25), np.arange(150, 170)]
    groups = [np.arange(25, 120), np.arange(100, 140), rng.permutation(np.arange(60, 90)), np.arange(200, 240)] + refs
    monkeypatch.setenv("ICNV_SLAB_CELLS", "64")
    api.reinit()
    try:
        S6, S3 = _check(api, X, cs, cl, refs, groups)
    finally:
        monkeypatch.delenv("ICNV_SLAB_CELLS")
        api.reinit()
    unlisted = np.setdiff1d(np.arange(C), np.concatenate(groups))
    assert len(unlisted) > 0
    assert np.all(S6[:, unlisted] == 255) and np.all(S3[:, unlisted] == 255)
    listed = np.setdiff1d(np.arange(C), unlisted)
    assert np.all(S6[:, listed] != 255)
    # cells 100..119 are in groups 0 and 1 and take group 1's trace; 60..89 are in groups 0 and 2 and take group 2's
    assert np.array_equal(S6[:, 100], S6[:, 139]) and np.array_equal(S6[:, 60], S6[:, 89])


def test_errors_write_nothing(api):
    rng = np.random.default_rng(6)
    cs, cl = _layout([40, 60])
    G, C = 100, 30
    X = _counts(rng, G, C)
    off, idx = np.array([0, 5], np.int32), np.arange(5, dtype=np.int32)
    Pi, delta = orc.hmm_params(6, 1e-6)
    mean = np.array([0.01, 0.5, 1.0, 1.5, 2.0, 3.0])
    lib = _lib.load()
    P = lambda a: None if a is None else a.ctypes.data  # noqa: E731

    def call(i3, hoff, hidx, n_hmm, sd=None, window=101, p=0.05, ridx=idx):
        Y = np.full((G, C), 7.0, order="F")
        S = np.full((G, C), 9, np.uint8, order="F")
        model = np.full(3, 7.0)
        if i3:
            rc = lib.icnv_smooth_i3_hmm_groups_u8_f64(P(X), P(Y), P(S), G, C, P(cs), P(cl), len(cs), P(off), P(ridx), 1, 1, 3.0,
                                                      window, 1, P(hoff), P(hidx), n_hmm, p, 1e-6, P(model))
        else:
            sd = np.tile(np.full(6, 0.1), max(n_hmm, 1)) if sd is None else sd
            rc = lib.icnv_smooth_hmm_groups_u8_f64(P(X), P(Y), P(S), G, C, P(cs), P(cl), len(cs), P(off), P(ridx), 1, 1, 3.0,
                                                   window, 1, P(hoff), P(hidx), n_hmm, 6, P(Pi), P(delta), P(mean), P(sd))
        assert np.all(Y == 7.0) and np.all(S == 9) and np.all(model == 7.0)
        return rc

    hoff, hidx = np.array([0, 10, 30], np.int32), np.arange(30, dtype=np.int32)
    bad_hidx = hidx.copy()
    bad_hidx[12] = 30
    for i3 in (False, True):
        assert call(i3, np.zeros(1, np.int32), np.zeros(1, np.int32), 0) == BAD_ARG          # n_hmm == 0
        assert call(i3, hoff, bad_hidx, 2) == BAD_ARG                                         # list index out of range
        assert call(i3, np.array([0, 10, 10], np.int32), hidx, 2) == BAD_ARG                  # an empty group
        assert call(i3, hoff, hidx, 2, ridx=np.array([0, 1, 2, 3, 31], np.int32)) == BAD_ARG  # reference index
    sd = np.tile(np.full(6, 0.1), 2)
    sd[6:] = 0.0
    assert call(False, hoff, hidx, 2, sd=sd) == BAD_ARG                                       # a group's median sd is 0
    for case in (dict(window=100), dict(p=0.0), dict(p=1.0), dict(p=float("nan"))):
        assert call(True, hoff, hidx, 2, **case) == BAD_ARG, case


@gpu_only
def test_page_locked_buffers(api):
    """page-locked X and Y are copied a run of consecutive columns at a time, with no staging ring: the same bits as the
    pageable call"""
    import torch
    rng = np.random.default_rng(9)
    cs, cl = _layout(LAYOUTS["odd_ends"])
    G, C = int(cl.sum()), 3000
    X = _counts(rng, G, C)
    perm = rng.permutation(C)
    refs = [np.sort(perm[:150]), np.sort(perm[150:240])]
    groups = _subclusters(rng, np.sort(perm[240:2900]), 12) + refs + [np.array([c]) for c in perm[2900:2950]]
    Pi, delta, mean, sd = _i6(groups)
    want6 = api.smooth_hmm(X, cs, cl, refs, Pi, delta, mean, sd, groups=groups)
    want3 = api.smooth_i3_hmm(X, cs, cl, refs, groups=groups)
    hX = torch.empty((C, G), dtype=torch.float64).pin_memory()
    hX.copy_(torch.from_numpy(X.T))
    hY = torch.empty((C, G), dtype=torch.float64).pin_memory()
    hS = torch.empty((C, G), dtype=torch.uint8).pin_memory()
    off, idx = api.groups_to_csr(refs)
    hoff, hidx = api.groups_to_csr(groups)
    lib = _lib.load()
    args = (hX.data_ptr(), hY.data_ptr(), hS.data_ptr(), G, C, cs.ctypes.data, cl.ctypes.data, len(cs), off.ctypes.data,
            idx.ctypes.data, len(refs), 1, 3.0, 101, 1, hoff.ctypes.data, hidx.ctypes.data, len(groups))
    _lib.check(lib.icnv_smooth_hmm_groups_u8_f64(*args, 6, Pi.ctypes.data, delta.ctypes.data, mean.ctypes.data,
                                                 sd.ctypes.data))
    assert np.array_equal(hY.numpy().T, want6[0]) and np.array_equal(hS.numpy().T, want6[1])
    model = np.zeros(3)
    _lib.check(lib.icnv_smooth_i3_hmm_groups_u8_f64(*args, 0.05, 1e-6, model.ctypes.data))
    assert np.array_equal(hY.numpy().T, want3[0]) and np.array_equal(hS.numpy().T, want3[1])
    assert (model[0], model[1], model[2]) == (want3[3]["mu"], want3[3]["sigma"], want3[3]["mean_delta"])


@gpu_only
def test_two_devices_match_one(api):
    if api.device_count() < 2:
        pytest.skip("needs two GPUs")
    import bench
    rng = np.random.default_rng(7)
    G, C = 10_000, 900
    cs, cl = bench.chr_layout(G)
    X = _counts(rng, G, C)
    refs = [np.arange(0, 50), np.arange(50, 90)]
    groups = _subclusters(rng, np.arange(90, 600), 4) + [np.array([c]) for c in range(600, 900)] + refs
    Pi, delta, mean, sd = _i6(groups)
    one = (api.smooth_hmm(X, cs, cl, refs, Pi, delta, mean, sd, groups=groups), api.smooth_i3_hmm(X, cs, cl, refs, groups=groups))
    try:
        assert api.init_devices([0, 1]) == 2
        two = (api.smooth_hmm(X, cs, cl, refs, Pi, delta, mean, sd, groups=groups),
               api.smooth_i3_hmm(X, cs, cl, refs, groups=groups))
    finally:
        api.reinit()
    for a, b in zip(one[0] + one[1][:2], two[0] + two[1][:2]):
        assert np.array_equal(a, b)
    assert one[1][3] == two[1][3]


def _example(ex, subclusters):
    from mirror import ops
    rng = np.random.default_rng(10)
    X = orc.normalize_by_seq_depth(ex["counts"])
    H = rng.poisson(3.0, size=(X.shape[0], 12)).astype(float)
    o = ops.Infercnv(expr_data=X, gene_order_chr=ex["chr_codes"],
                     reference_grouped_cell_indices={"normal": ex["ref_groups"][0]},
                     observation_grouped_cell_indices={"tumor": ex["obs_groups"][0]}, tumor_subclusters=subclusters)
    o.hspike = ops.Infercnv(expr_data=H, gene_order_chr=ex["chr_codes"],
                            reference_grouped_cell_indices={"simnormal": np.arange(0, 6)},
                            observation_grouped_cell_indices={"simtumor": np.arange(6, 12)})
    return o


@pytest.mark.parametrize("mode", [("samples", True), ("samples", False), ("subclusters", True), ("no_subclusters", True)])
def test_mirror_against_the_hmm_drivers(api, example_object, mode):
    """mirror.ops.smooth_block_hmm / smooth_block_i3_hmm(analysis_mode=...) against mirror.ops.predict_CNV_via_HMM_on_*
    applied to smooth_block: the lists the reference's drivers build, the states as R keeps them"""
    from mirror import ops
    ex = example_object
    analysis_mode, cbg = mode
    subs = {"subclusters": {"tumor": {f"tumor_s{k}": g for k, g in enumerate(ex["subclusters"])},
                            "normal": {"normal_s1": np.asarray(ex["ref_groups"][0])}}}
    obj = _example(ex, subs if analysis_mode == "subclusters" else None)
    analysis_mode = "subclusters" if analysis_mode == "no_subclusters" else analysis_mode
    levels = hmm.CNV_LEVELS
    cnv_mean_sd = {k: {"mean": m, "sd": s} for k, m, s in zip(levels, [0.01, 0.5, 1, 1.5, 2, 3], [0.05, .1, .1, .1, .2, .3])}
    fit = {k: (np.log(s), -0.4) for k, s in zip(levels, [0.2, 0.4, 0.4, 0.4, 0.6, 0.9])}
    o, h = ops.smooth_block_hmm(obj, analysis_mode, cnv_mean_sd, fit, cluster_by_groups=cbg)
    blk = ops.smooth_block(obj)
    assert np.array_equal(o.expr_data, blk.expr_data) and np.array_equal(o.hspike.expr_data, blk.hspike.expr_data)
    if analysis_mode == "samples":
        want = ops.predict_CNV_via_HMM_on_whole_tumor_samples(blk, cbg, cnv_mean_sd, fit)
    else:
        want = ops.predict_CNV_via_HMM_on_tumor_subclusters(blk, cnv_mean_sd, fit)
    assert np.array_equal(h.expr_data, want.expr_data)
    o3, h3, m3, sd_trend = ops.smooth_block_i3_hmm(obj, analysis_mode=analysis_mode, cluster_by_groups=cbg)
    assert np.array_equal(o3.expr_data, blk.expr_data) and m3 is None
    if analysis_mode == "samples":
        want3 = ops.i3HMM_predict_CNV_via_HMM_on_whole_tumor_samples(blk, cbg, sd_trend=sd_trend)
    elif obj.tumor_subclusters is not None:
        want3 = ops.i3HMM_predict_CNV_via_HMM_on_tumor_subclusters(blk, sd_trend=sd_trend)
    else:
        want3 = ops.i3HMM_predict_CNV_via_HMM_on_whole_tumor_samples(blk, True, sd_trend=sd_trend)
    assert np.array_equal(h3.expr_data, want3.expr_data)


def test_oracle_chain_on_the_bundled_example(api, oligo):
    """oracle.smooth_block -> oracle.viterbi_matrix over the samples lists (i6 and the i3 model of the block's
    reference cells): the same states"""
    cs, cl = orc.chr_ranges(oligo["chr_codes"])
    X = orc.normalize_by_seq_depth(oligo["counts"])
    refs = oligo["ref_groups"]
    groups = list(oligo["obs_groups"]) + list(refs)
    Yo = orc.smooth_block(X, cs, cl, refs, nthreads=orc.max_threads())
    Pi, delta, mean, sd = _i6(groups)
    _, S = api.smooth_hmm(X, cs, cl, refs, Pi, delta, mean, sd, groups=groups)
    So = orc.viterbi_matrix(Yo, cs, cl, Pi, delta, mean, sd, groups=groups, nthreads=orc.max_threads())
    assert np.array_equal(np.where(S == 255, -1, S.astype(np.int32)), So)
    _, S3, _, _ = api.smooth_i3_hmm(X, cs, cl, refs, groups=groups)
    Pi, delta, mean, sd = orc.i3_hmm_params(Yo, np.concatenate(refs), 0.05, 1e-6)
    So3 = orc.viterbi_matrix(Yo, cs, cl, Pi, delta, mean, sd, groups=groups, nthreads=orc.max_threads())
    assert np.array_equal(np.where(S3 == 255, -1, S3.astype(np.int32)), So3)
    print(f"\n[oligodendroglioma {X.shape[0]}x{X.shape[1]}] group-mode fused: i6 and i3 states equal the oracle's")
