"""Parity of the CUDA path (through the C ABI) against the CPU oracle and the reference's own
known answers.  Needs an H100: run with `pytest -m gpu`.

Tolerances (BASELINE.json north_star): smoothed matrix within 1e-5 relative; HMM state calls
bit-identical.  The smooth tests additionally report how far below that the kernels actually are.
"""
import os

import numpy as np
import pytest

from oracle import oracle as orc

pytestmark = pytest.mark.gpu

RTOL = 1e-5  # north_star tolerance for the smooth block


@pytest.fixture(scope="module")
def api():
    from infercnv_b200 import api as a
    a.init(0)
    return a


def _close(got, want, rtol=RTOL, atol_scale=1e-12):
    want = np.asarray(want)
    atol = atol_scale * max(1.0, float(np.max(np.abs(want))))
    np.testing.assert_allclose(got, want, rtol=rtol, atol=atol)


# ---- reference known answers (tests/testthat/test_infer_cnv.R:89-172) through the ABI ---------------
def test_subtract_ref_known_answers(api):
    from tests.test_oracle_known_answers import (matrix_averef_five, matrix_averef_five_answer, matrix_five,
                                                 matrix_three)
    for mat, groups, want in [
        (matrix_three.T, [[0, 2]], np.tile(np.arange(-1, 4, dtype=float), (3, 1))),
        (matrix_five.T, [[1, 4]], np.tile(np.arange(-3, 2) + 0.5, (5, 1))),
        (matrix_averef_five, [[1], [3, 5, 7], [9]], matrix_averef_five_answer),
    ]:
        M = api.ref_means(mat, groups)
        np.testing.assert_allclose(M, orc.ref_means(mat, groups), rtol=1e-14)
        got = api.subtract_ref(mat, M, use_bounds=True)
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
        got_nb = api.subtract_ref(mat, M, use_bounds=False)
        np.testing.assert_allclose(got_nb, orc.subtract_ref(mat, M, False), rtol=0, atol=1e-12)


def test_ref_means_inv_log(api):
    rng = np.random.default_rng(0)
    X = rng.normal(size=(300, 50))
    groups = [np.arange(0, 20), np.arange(25, 50)]
    np.testing.assert_allclose(api.ref_means(X, groups, inv_log=True), orc.ref_means(X, groups, inv_log=True),
                               rtol=1e-12)


def test_center_known_answers_and_median(api):
    m = np.arange(1, 22, dtype=float).reshape(7, 3, order="F")
    want = np.tile(np.array([-3, -2, -1, 0, 1, 2, 3], dtype=float), (3, 1)).T
    np.testing.assert_allclose(api.center(m, "mean"), want, atol=1e-12)
    rng = np.random.default_rng(1)
    for G in [1, 2, 3, 10, 11, 64, 65, 257, 1000, 2817, 4613, 5633, 8508, 10000, 11264, 11777, 20000, 23552]:
        X = rng.normal(size=(G, 7))
        X[:, 1] = 0.25                      # all equal
        X[: G // 2, 2] = 1.0                # two big tie clusters
        X[G // 2:, 2] = -1.0
        X[:, 3] = np.round(X[:, 3], 1)      # many ties
        X[:, 4] = np.exp(5 * X[:, 4])       # heavy tail
        X[:, 5] = rng.integers(0, 3, size=G)  # three values
        got = api.center(X, "median")
        want = X - np.median(X, axis=0)[None, :]
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * np.max(np.abs(X)))


def test_smooth_known_answer_w5_and_identity(api):
    from tests.test_oracle_known_answers import SMOOTH_W5, matrix_one, matrix_one_long_2
    x = np.column_stack([matrix_one_long_2, matrix_one_long_2])
    got = api.smooth(x, [0], [20], 5)
    np.testing.assert_allclose(got[:, 0], SMOOTH_W5, atol=6e-3)
    np.testing.assert_allclose(got, orc.smooth_by_chromosome(x, [0], [20], 5, literal=True), rtol=1e-13)
    for w in (0, 1):
        np.testing.assert_array_equal(api.smooth(matrix_one, [0], [5], w), matrix_one)
    got = api.smooth(matrix_one, [0], [5], 5)[:, 0]
    np.testing.assert_allclose(got, [1.67, 2.25, 3, 3.75, 4.33], atol=6e-3)


def test_smooth_lengths_and_windows_vs_literal_oracle(api):
    rng = np.random.default_rng(2)
    lens = [1, 2, 3, 4, 5, 6, 50, 51, 100, 101, 102, 150, 201, 202, 203, 500, 1, 852]
    cs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    G = int(np.sum(lens))
    X = rng.normal(size=(G, 9))
    for w in [3, 5, 51, 101, 201]:
        got = api.smooth(X, cs, lens, w)
        want = orc.smooth_by_chromosome(X, cs, lens, w, literal=True)
        err = np.max(np.abs(got - want))
        assert err < 5e-11, (w, err)   # prefix-sum formulation: ~n^1.5 ulp of cancellation, far inside 1e-5
        # single-gene chromosomes are skipped (ops.R:2417)
        np.testing.assert_array_equal(got[cs[0]], X[cs[0]])
        np.testing.assert_array_equal(got[cs[16]], X[cs[16]])


def test_smooth_rejects_even_window_and_nonfinite(api):
    from infercnv_b200._lib import InfercnvB200Error
    X = np.ones((30, 3))
    with pytest.raises(InfercnvB200Error) as e:
        api.smooth(X, [0], [30], 4)
    assert e.value.code == -3
    X[3, 1] = np.nan
    with pytest.raises(InfercnvB200Error) as e:
        api.smooth(X, [0], [30], 5)
    assert e.value.code == -5
    with pytest.raises(InfercnvB200Error):
        api.smooth(np.ones((30, 3)), [0, 10], [10, 10], 5)   # ranges do not tile [0, G)


# ---- the bundled golden of the reference: count.data -> expr.data ------------------------------------
def test_golden_example_object_smooth_block(api, example_object):
    ex = example_object
    cs, cl = orc.chr_ranges(ex["chr_codes"])
    X = orc.normalize_by_seq_depth(ex["counts"])
    got = api.smooth_block(X, cs, cl, ex["ref_groups"], apply_log=True, threshold=3.0, window_length=101)
    want = orc.smooth_block(X, cs, cl, ex["ref_groups"])
    rel = np.max(np.abs(got - want) / np.abs(want))
    print(f"\n[golden 4613x20] smooth block max rel err vs oracle: {rel:.3e}")
    assert rel < RTOL
    assert rel < 1e-11   # what the FP64 kernels actually deliver
    # against the reference's own stored output (needs the denoise step that follows the block)
    ref = np.concatenate(ex["ref_groups"])
    final = orc.clear_noise_via_ref_mean_sd(got, ref, 1.5)
    rel_ref = np.max(np.abs(final - ex["expr"]) / np.abs(ex["expr"]))
    print(f"[golden 4613x20] max rel err vs the reference's expr.data: {rel_ref:.3e}")
    assert rel_ref < RTOL


def test_oligodendroglioma_smooth_block_two_ref_groups(api, oligo):
    cs, cl = orc.chr_ranges(oligo["chr_codes"])
    X = orc.normalize_by_seq_depth(oligo["counts"])
    got = api.smooth_block(X, cs, cl, oligo["ref_groups"])
    want = orc.smooth_block(X, cs, cl, oligo["ref_groups"], nthreads=orc.max_threads())
    rel = np.max(np.abs(got - want) / np.abs(want))
    print(f"\n[oligodendroglioma 8508x184] smooth block max rel err vs oracle: {rel:.3e}")
    assert rel < RTOL and rel < 1e-11
    # no-bounds variant and no reference cells (proxy group of all observation cells, ops.R:1686-1689)
    allobs = [np.concatenate(oligo["obs_groups"])]
    got2 = api.smooth_block(X, cs, cl, allobs, use_bounds=False, window_length=51, threshold=2.0)
    want2 = orc.smooth_block(X, cs, cl, allobs, use_bounds=False, window=51, threshold=2.0, nthreads=orc.max_threads())
    assert np.max(np.abs(got2 - want2) / np.abs(want2)) < 1e-11


def test_smooth_block_slow_paths_of_the_grouped_element_wise_loops(api):
    """Stage A / D of the fused kernel evaluate log2 / 2^x four genes at a time without a per-value range branch; a value
    outside the fast path's domain re-evaluates its group.  Zeros (log2(1)), x = -1 (log2(0) = -Inf, clamped to -3 as in R,
    ops.R:2760 + 2970) and NaN / Inf inputs (error -5), each placed
    both in a four-gene group and in the per-thread remainder (G = 1300: 256 threads, groups cover genes 0..1023)."""
    from infercnv_b200._lib import InfercnvB200Error
    rng = np.random.default_rng(11)
    lens = np.array([700, 330, 270], dtype=np.int32)
    cs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32)
    G, C = int(lens.sum()), 12
    X = rng.gamma(2.0, 1.5, size=(G, C))
    X[rng.random((G, C)) < 0.4] = 0.0
    refs = [np.arange(0, 4), np.arange(4, 6)]
    X[[5, 600, 1100, 1299], 7] = -1.0          # x + 1 == 0
    got = api.smooth_block(X, cs, lens, refs, apply_log=True, threshold=3.0, window_length=101)
    want = orc.smooth_block(X, cs, lens, refs)
    assert np.all(np.isfinite(got))
    rel = np.max(np.abs(got - want) / np.abs(want))
    assert rel < 1e-11, rel
    for g in (600, 1250):
        for bad in (np.nan, np.inf):
            Xb = X.copy()
            Xb[g, 9] = bad
            with pytest.raises(InfercnvB200Error) as e:
                api.smooth_block(Xb, cs, lens, refs, apply_log=True, threshold=3.0, window_length=101)
            assert e.value.code == -5


def test_smooth_block_padded_q_layout_is_bit_identical(api, monkeypatch):
    """cell_pipeline3_kernel<NT, true> (padded Q, fixed buffer roles - the default) against <NT, false> (ping-pong buffers,
    index-selected edge loads; ICNV_CELL_PADQ=0): the same arithmetic in the same order, so identical bits.  Chromosome
    lengths cover: shorter than the window (both ends in every window), 2h+1 .. 2h+1+slice (a slice can see both ends),
    single-gene and two-gene chromosomes, long ones; windows 101, 15, 3 and none; all three thread counts."""
    rng = np.random.default_rng(5)
    for lens, C in (([300, 150, 60, 1, 201, 2, 103, 104, 115], 9), ([1500, 101, 102, 900, 77, 400], 5),
                    ([2900, 2100, 1700, 303], 3)):
        lens = np.array(lens, dtype=np.int32)
        cs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32)
        G = int(lens.sum())
        X = rng.gamma(2.0, 1.5, size=(G, C))
        X[rng.random((G, C)) < 0.3] = 0.0
        refs = [np.arange(0, 2), np.arange(2, 3)]
        for w in (101, 15, 3):
            out = {}
            for flag in ("1", "0"):
                monkeypatch.setenv("ICNV_CELL_PADQ", flag)
                api.reinit()   # tuning switches are read once, at icnv_init
                out[flag] = api.smooth_block(X, cs, lens, refs, apply_log=True, threshold=3.0, window_length=w)
            assert np.array_equal(out["1"], out["0"]), (G, w)
            want = orc.smooth_block(X, cs, lens, refs, window=w)
            assert np.max(np.abs(out["1"] - want) / np.abs(want)) < 1e-10   # prefix sums over up to 2900 genes
        for flag in ("1", "0"):
            monkeypatch.setenv("ICNV_CELL_PADQ", flag)
            api.reinit()
            out[flag] = api.smooth(np.log2(X + 1.0), cs, lens, 51)
        assert np.array_equal(out["1"], out["0"])
    monkeypatch.delenv("ICNV_CELL_PADQ")
    api.reinit()


def test_smooth_block_benchmark_layout_unrolled_slices(api, monkeypatch):
    """10 000 genes in the benchmark's 22 chromosomes: 1024 threads with slices of 11 genes, the layout for which the scan
    passes are compiled fully unrolled (cell_pipeline3_kernel<1024, true, 11>).  Same bits as the generic form
    (ICNV_CELL_LFIX=0) and as the ping-pong layout, and the oracle's values."""
    import bench
    cs, lens = bench.chr_layout(10000)
    rng = np.random.default_rng(21)
    G, C = 10000, 6
    X = rng.gamma(2.0, 1.5, size=(G, C))
    X[rng.random((G, C)) < 0.3] = 0.0
    refs = [np.arange(0, 2), np.arange(2, 3)]
    out = {}
    for name, env in (("unrolled", {}), ("generic", {"ICNV_CELL_LFIX": "0"}), ("pingpong", {"ICNV_CELL_PADQ": "0"})):
        for k in ("ICNV_CELL_LFIX", "ICNV_CELL_PADQ"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        api.reinit()   # tuning switches are read once, at icnv_init
        out[name] = api.smooth_block(X, cs, lens, refs, apply_log=True, threshold=3.0, window_length=101)
    for k in ("ICNV_CELL_LFIX", "ICNV_CELL_PADQ"):
        monkeypatch.delenv(k, raising=False)
    api.reinit()
    assert np.array_equal(out["unrolled"], out["generic"])
    assert np.array_equal(out["unrolled"], out["pingpong"])
    want = orc.smooth_block(X, cs, lens, refs)
    assert np.max(np.abs(out["unrolled"] - want) / np.abs(want)) < 1e-10


def test_smooth_block_20k_genes_single_buffer_variant(api):
    """config c5's gene count: one CTA of 1024 threads per SM (the padded column takes 178 KB of shared memory)."""
    from infercnv_b200._lib import InfercnvB200Error
    rng = np.random.default_rng(8)
    t = np.array([852, 615, 535, 288, 420, 453, 458, 297, 349, 363, 514, 472, 162, 301, 274, 397, 546, 126, 545, 239,
                  90, 212], dtype=float)
    G, C = 20000, 48
    lens = np.floor(t * G / t.sum()).astype(int)
    lens[0] += G - lens.sum()
    cs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    counts = rng.poisson(rng.lognormal(0.5, 1.0, size=(G, 1)) * rng.lognormal(0, 0.2, size=(1, C))).astype(np.float64)
    refs = [np.arange(0, 6), np.arange(6, 10)]
    got = api.smooth_block(counts, cs, lens, refs)
    want = orc.smooth_block(counts, cs, lens, refs, nthreads=orc.max_threads())
    rel = np.max(np.abs(got - want) / np.abs(want))
    print(f"\n[20000 genes] smooth block max rel err vs oracle: {rel:.3e}")
    assert rel < 1e-10
    z = api.center(np.arange(48000, dtype=np.float64).reshape(24000, 2, order="F"))   # 24 000 genes still fit without pads
    np.testing.assert_array_equal(z[:, 1], np.arange(24000, 48000) - 35999.5)
    with pytest.raises(InfercnvB200Error) as e:        # a column that does not fit shared memory: refused, the R wrapper falls back
        api.center(np.ones((40000, 2)))
    assert e.value.code == -4


# ---- HMM ------------------------------------------------------------------------------------------------------
def _hmm_input(rng, G, C, mean, sd_noise=0.08):
    lv = rng.integers(1, len(mean) - 1, size=(G // 50 + 1, C))
    X = np.repeat(np.asarray(mean)[lv], 50, axis=0)[:G] + rng.normal(scale=sd_noise, size=(G, C))
    return np.asfortranarray(X)


@pytest.mark.parametrize("m", [6, 3])
def test_viterbi_cells_bit_identical(api, hmm_fixture, m):
    rng = np.random.default_rng(10 + m)
    lens = [300, 1, 2, 90, 455, 852, 17]
    cs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    G, C = int(np.sum(lens)), 77
    if m == 6:
        mean, sd = hmm_fixture["mean"], hmm_fixture["sd"]
    else:
        mean, sd = np.array([0.9, 1.0, 1.1]), np.array([0.05] * 3)
    X = _hmm_input(rng, G, C, mean)
    Pi, delta = orc.hmm_params(m)
    want, wm = orc.viterbi_matrix(X, cs, lens, Pi, delta, mean, sd, want_margins=True, nthreads=orc.max_threads())
    got, gm = api.viterbi(X, cs, lens, Pi, delta, mean, sd, want_margins=True)
    mism = int(np.sum(got != want))
    print(f"\n[viterbi m={m}] {G}x{C}: mismatching states {mism}; min decision margin gpu {gm.min():.3e} "
          f"oracle {wm.min():.3e}")
    np.testing.assert_array_equal(got, want)
    fin = np.isfinite(wm)
    np.testing.assert_allclose(gm[fin], wm[fin], rtol=1e-6, atol=1e-9)
    assert (got[cs[1]] == 3).all()          # single-gene chromosome -> state 3 (HMM.R:1104-1107)
    got2 = api.viterbi(X, cs, lens, Pi, delta, mean, sd)   # margin-free kernel instantiation
    np.testing.assert_array_equal(got2, want)


@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_viterbi_modes_agree_with_oracle_at_scale(api, hmm_fixture, mode):
    """2e7 cell-genes of the bench's synthetic structure: the certified fast path and the
    reference-order path must both reproduce the oracle's states exactly."""
    rng = np.random.default_rng(99)
    lens = np.array([852, 615, 535, 288, 420, 453, 458, 297, 349, 363, 514, 472, 162, 301, 274, 397, 546, 126, 545,
                     239, 90, 212])
    cs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    G, C = int(lens.sum()), 1500
    mean, sd = hmm_fixture["mean"], hmm_fixture["sd"]
    base = 1.0 + 0.04 * rng.normal(size=(G, C))
    # smooth-ish CNV segments so that there are real change points with small margins
    for c in range(0, C, 3):
        k = rng.integers(0, len(lens))
        base[cs[k]:cs[k] + lens[k], c] += rng.choice([-0.25, 0.2, 0.45])
    X = np.asfortranarray(base)
    Pi, delta = orc.hmm_params(6)
    want = orc.viterbi_matrix(X, cs, lens, Pi, delta, mean, sd, nthreads=orc.max_threads())
    api.set_hmm_mode(mode)
    try:
        got = api.viterbi(X, cs, lens, Pi, delta, mean, sd)
        reruns = api.hmm_rerun_count()
    finally:
        api.set_hmm_mode("fast")
    print(f"\n[viterbi {mode}] {G}x{C}: mismatches {int(np.sum(got != want))}, sequences re-run exactly: {reruns} "
          f"of {C * len(lens)}")
    np.testing.assert_array_equal(got, want)
    if mode == "exact":
        assert reruns == 0
    else:   # the certificates must certify: a pass that sends everything to the exact kernel would also "agree"
        assert reruns < 0.02 * C * len(lens)


@pytest.mark.parametrize("m,t", [(6, 0.18), (3, 0.4), (6, 0.0)])
def test_viterbi_transition_matrices_outside_the_fast_paths_structure(api, hmm_fixture, m, t):
    """The certified fast path assumes .get_HMM's matrix with the diagonal the larger entry ("the best state stays") and
    every transition possible.  A t that makes moving cheaper than staying (t > 1/6 for i6, > 1/3 for i3), or t = 0
    (log 0 = -inf off the diagonal), must take the reference-order kernel: same states as the oracle."""
    rng = np.random.default_rng(31 + m)
    lens = [120, 45, 300]
    cs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    G, C = int(np.sum(lens)), 40
    if m == 6:
        mean, sd = hmm_fixture["mean"], hmm_fixture["sd"]
    else:
        mean, sd = np.array([0.8, 1.0, 1.2]), np.array([0.1] * 3)
    X = _hmm_input(rng, G, C, mean)
    Pi = np.full((m, m), t, order="F")
    np.fill_diagonal(Pi, 1 - 5 * t)
    delta = np.full(m, 1.0 / m)
    want = orc.viterbi_matrix(X, cs, lens, Pi, delta, mean, sd)
    got = api.viterbi(X, cs, lens, Pi, delta, mean, sd)
    np.testing.assert_array_equal(got, want)


def test_viterbi_fast_path_exact_ties_are_rerun(api):
    """Two states with identical scores at every gene (dyadic, symmetric means): the certificate
    sees a zero margin, the sequences are recomputed in reference-order arithmetic, and the
    first-index tie rule of which.max (HMM.R:1170,1173) decides as in the oracle."""
    G, C = 200, 40
    X = np.ones((G, C), order="F")
    X[50:120, ::2] = 1.25
    mean, sd = np.array([0.5, 1.5, 3.0]), np.array([0.25] * 3)
    t = 1e-6
    Pi = np.full((3, 3), t, order="F")
    np.fill_diagonal(Pi, 1 - 5 * t)
    delta = np.array([1 / 3, 1 / 3, 1 / 3])
    want = orc.viterbi_matrix(X, [0, 150], [150, 50], Pi, delta, mean, sd)
    got = api.viterbi(X, [0, 150], [150, 50], Pi, delta, mean, sd)
    reruns = api.hmm_rerun_count()
    np.testing.assert_array_equal(got, want)
    assert reruns > 0
    print(f"\n[viterbi ties] {reruns} of {2 * C} sequences re-run")


@pytest.mark.parametrize("m", [6, 3])
def test_viterbi_rerun_of_long_sequences(api, hmm_fixture, m):
    """The exact re-run works a chunk of 384 genes at a time and keeps backpointers in shared memory up to 2048 genes:
    sequences of 2500 / 700 / 385 genes whose state means sit symmetrically around the data (exact ties everywhere)
    go through both branches, for i6 and i3."""
    rng = np.random.default_rng(8)
    lens = [2500, 700, 385]
    cs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    G, C = int(np.sum(lens)), 12
    X = np.ones((G, C), order="F")
    X[:, 1::2] += 0.05 * rng.normal(size=(G, C // 2))       # half the cells: generic data
    X[100:400, ::2] = 1.25
    X[2600:2900, ::2] = 0.75
    if m == 6:
        mean, sd = np.array([0.0, 0.5, 0.75, 1.25, 1.5, 2.0]), np.array([0.2] * 6)
        Pi, delta = orc.hmm_params(6)
    else:
        mean, sd = np.array([0.5, 1.5, 3.0]), np.array([0.25] * 3)
        Pi, delta = orc.hmm_params(3, 1e-6)
    want = orc.viterbi_matrix(X, cs, lens, Pi, delta, mean, sd)
    # the FP64 pass rejects every sequence that meets a tie anywhere: all three lengths reach the exact kernel
    api.set_hmm_mode("fast")
    got = api.viterbi(X, cs, lens, Pi, delta, mean, sd)
    reruns = api.hmm_rerun_count()
    np.testing.assert_array_equal(got, want)
    assert reruns >= 3 * (C // 2)
    print(f"\n[viterbi long re-runs, m={m}] {reruns} of {3 * C} sequences re-run")


def test_viterbi_unstructured_transition_matrix_and_far_outliers(api, hmm_fixture):
    rng = np.random.default_rng(5)
    G, C = 400, 33
    mean, sd = hmm_fixture["mean"], hmm_fixture["sd"]
    X = np.asfortranarray(1.0 + 0.1 * rng.normal(size=(G, C)))
    X[10, 3] = 9.0          # |x - mean| / sd > 24: beyond the emission table
    X[200:230, 7] = 40.0
    Pi, delta = orc.hmm_params(6)
    want = orc.viterbi_matrix(X, [0], [G], Pi, delta, mean, sd)
    np.testing.assert_array_equal(api.viterbi(X, [0], [G], Pi, delta, mean, sd), want)
    Pi2 = Pi.copy()
    Pi2[0, 1] = 5e-6        # not .get_HMM's structure: generic kernel
    want2 = orc.viterbi_matrix(X, [0], [G], Pi2, delta, mean, sd)
    np.testing.assert_array_equal(api.viterbi(X, [0], [G], Pi2, delta, mean, sd), want2)


def test_viterbi_group_modes(api, hmm_fixture):
    rng = np.random.default_rng(21)
    lens = [200, 120, 1, 333]
    cs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    G, C = int(np.sum(lens)), 60
    mean, sd = hmm_fixture["mean"], hmm_fixture["sd"]
    X = _hmm_input(rng, G, C, mean, sd_noise=0.2)
    Pi, delta = orc.hmm_params(6)
    groups = [rng.permutation(np.arange(0, 25)), np.arange(30, 41), np.array([59, 45, 50])]
    sds = np.concatenate([sd * f for f in (0.5, 0.8, 1.0)])
    want = orc.viterbi_matrix(X, cs, lens, Pi, delta, mean, sds, groups=groups)
    got = api.viterbi(X, cs, lens, Pi, delta, mean, sds, groups=groups)
    np.testing.assert_array_equal(got, want)
    assert (got[:, 26] == -1).all()
    # one-byte wire format: same states, 255 where the int32 variant says -1
    got8 = api.viterbi(X, cs, lens, Pi, delta, mean, sds, groups=groups, out=np.empty((G, C), dtype=np.uint8, order="F"))
    assert got8.dtype == np.uint8
    np.testing.assert_array_equal(got8, np.where(want < 0, 255, want))


def test_viterbi_nonfinite_is_an_error(api, hmm_fixture):
    from infercnv_b200._lib import InfercnvB200Error
    X = np.ones((50, 4))
    X[7, 2] = np.inf
    Pi, delta = orc.hmm_params(6)
    with pytest.raises(InfercnvB200Error) as e:
        api.viterbi(X, [0], [50], Pi, delta, hmm_fixture["mean"], hmm_fixture["sd"])
    assert e.value.code == -5


def test_oligodendroglioma_hmm_cells_and_samples(api, oligo, hmm_fixture):
    """config c1: real matrix through the smooth block, then i6 HMM per cell and per sample,
    and i3 per cell, against the oracle (no R on the box: SURVEY section 8d 'c1 caveat')."""
    cs, cl = orc.chr_ranges(oligo["chr_codes"])
    X = orc.normalize_by_seq_depth(oligo["counts"])
    S = api.smooth_block(X, cs, cl, oligo["ref_groups"])
    mean, sd = hmm_fixture["mean"], hmm_fixture["sd"]
    Pi, delta = orc.hmm_params(6)
    nt = orc.max_threads()
    want = orc.viterbi_matrix(S, cs, cl, Pi, delta, mean, sd, nthreads=nt)
    got, gm = api.viterbi(S, cs, cl, Pi, delta, mean, sd, want_margins=True)
    print(f"\n[c1 i6 cells] mismatches {int(np.sum(got != want))} of {got.size}; min margin {gm.min():.3e}")
    np.testing.assert_array_equal(got, want)
    groups = oligo["obs_groups"]
    wantg = orc.viterbi_matrix(S, cs, cl, Pi, delta, mean, sd, groups=groups, nthreads=nt)
    gotg = api.viterbi(S, cs, cl, Pi, delta, mean, sd, groups=groups)
    np.testing.assert_array_equal(gotg, wantg)
    ref = np.concatenate(oligo["ref_groups"])
    mu, sg = api.mean_sd(S, ref)
    mu0, sg0 = orc.mean_sd_over_cells(S, ref)
    assert abs(mu - mu0) < 1e-12 * abs(mu0) + 1e-15 and abs(sg - sg0) < 1e-11 * sg0
    Pi3, d3, mean3, sd3 = orc.i3_hmm_params(S, ref)
    want3 = orc.viterbi_matrix(S, cs, cl, Pi3, d3, mean3, sd3, nthreads=nt)
    got3 = api.viterbi(S, cs, cl, Pi3, d3, mean3, sd3)
    np.testing.assert_array_equal(got3, want3)


def test_viterbi_equals_the_50_digit_restatement_on_c1(api):
    """The i6 and i3 state calls of ten c1 cells against Viterbi.dthmm.adj evaluated with 50 significant digits
    (tests/golden/hmm_mpmath_c1.npz, tools/make_hmm_mpmath_fixture.py; smallest arg-max margin 2e-5): the states every faithful
    double-precision evaluation must return, the reference's R included."""
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "hmm_mpmath_c1.npz"))
    X = np.asfortranarray(d["X"])
    for tag in ("i6", "i3"):
        got = api.viterbi(X, d["chr_start"], d["chr_len"], np.asfortranarray(d[tag + "_Pi"]), d[tag + "_delta"], d[tag + "_mean"],
                          d[tag + "_sd"])
        np.testing.assert_array_equal(got, d[tag + "_states"].astype(got.dtype), err_msg=tag)


def test_multi_slab_host_pipeline_and_fused_call(api, hmm_fixture):
    """More cells than one slab (1024): the pipelined host entry points (H2D / kernels / D2H
    overlapped over cell slabs) and the fused smooth+HMM call against the oracle."""
    rng = np.random.default_rng(77)
    lens = np.array([120, 1, 60, 150, 41])
    cs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    G, C = int(lens.sum()), 2500
    counts = rng.poisson(rng.lognormal(0.5, 1.0, size=(G, 1)) * rng.lognormal(0, 0.2, size=(1, C))).astype(np.float64)
    counts[cs[3]:cs[3] + lens[3], 1200:1400] *= 1.6
    refs = [np.arange(0, 150), np.array([2400, 2401, 2499, 1024, 1023])]
    mean, sd = hmm_fixture["mean"], hmm_fixture["sd"]
    Pi, delta = orc.hmm_params(6)
    nt = orc.max_threads()
    want = orc.smooth_block(counts, cs, lens, refs, window=51, nthreads=nt)
    got = api.smooth_block(counts, cs, lens, refs, window_length=51)
    assert np.max(np.abs(got - want) / np.abs(want)) < 1e-10
    want_st = orc.viterbi_matrix(got, cs, lens, Pi, delta, mean, sd, nthreads=nt)
    np.testing.assert_array_equal(api.viterbi(got, cs, lens, Pi, delta, mean, sd), want_st)
    Y, S = api.smooth_hmm(counts, cs, lens, refs, Pi, delta, mean, sd, window_length=51)
    np.testing.assert_array_equal(Y, got)        # same kernels, same order: bitwise equal
    np.testing.assert_array_equal(S, want_st)
    # one-byte states (icnv_viterbi_u8_f64 / icnv_smooth_hmm_u8_f64): what the R shim binds
    S8 = np.empty((G, C), dtype=np.uint8, order="F")
    np.testing.assert_array_equal(api.viterbi(got, cs, lens, Pi, delta, mean, sd, out=S8), want_st)
    Y8, S8b = api.smooth_hmm(counts, cs, lens, refs, Pi, delta, mean, sd, window_length=51,
                             out_states=np.empty((G, C), dtype=np.uint8, order="F"))
    np.testing.assert_array_equal(Y8, got)
    np.testing.assert_array_equal(S8b, want_st)


# ---- median filter ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("window_size", [3, 7, 9])
def test_median_filter_vs_oracle(api, window_size):
    rng = np.random.default_rng(33)
    lens = [37, 23, 1, 140]
    cs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    G, C = int(np.sum(lens)), 70
    X = np.asfortranarray(rng.normal(size=(G, C)))
    X[:, 5] = np.round(X[:, 5])
    groups = [rng.permutation(np.arange(0, 30)), np.array([40, 41]), np.array([33]), np.arange(45, 70)]
    got = api.median_filter(X, cs, lens, groups, window_size)
    want = orc.median_filter(X, cs, lens, groups, window_size, nthreads=orc.max_threads())
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-15)
    np.testing.assert_array_equal(got[:, 31], X[:, 31])


def test_median_filter_shared_merge_kernel_edges_and_ties(api):
    """window_size 7 runs the shared-merge kernel (sorted 9-key runs per list position, pair / quad merges shared between
    neighbouring outputs, ranks 39..43 of the 81 keys read off per output).  Blocks smaller than the window in either
    direction (every window truncated, even tap counts -> mean of the two middle values), blocks that end inside a tile,
    a de-noised-like matrix (most values one constant), small integers, values closer together than the 24-bit keys
    resolve (the exact rank is then settled on the doubles), and a large spread: all equal to the oracle."""
    rng = np.random.default_rng(77)
    lens = [1, 3, 8, 9, 33, 70, 2, 41]
    cs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    G = int(np.sum(lens))
    sizes = [1, 2, 5, 9, 40, 33, 64, 3]
    C = int(np.sum(sizes)) + 4                      # four cells in no list: copied through
    order = rng.permutation(C)
    groups, pos = [], 0
    for n in sizes:
        groups.append(order[pos:pos + n])
        pos += n
    base = 1.0 + 0.1 * rng.normal(size=(G, C))
    cases = {
        "smooth": base,
        "denoised": np.where(np.abs(base - 1.0) < 0.12, 1.000123, base),
        "states": rng.integers(1, 7, size=(G, C)).astype(float),
        "sub-key": 1.0 + 1e-12 * rng.integers(0, 50, size=(G, C)) + np.where(rng.random((G, C)) < 0.05, 3.0, 0.0),
        "spread": np.exp(rng.normal(scale=6.0, size=(G, C))),
        "constant": np.full((G, C), 2.5),
    }
    for name, X in cases.items():
        X = np.asfortranarray(X)
        got = api.median_filter(X, cs, lens, groups, 7)
        want = orc.median_filter(X, cs, lens, groups, 7, nthreads=orc.max_threads())
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-15, err_msg=name)
        np.testing.assert_array_equal(got[:, order[pos:]], X[:, order[pos:]], err_msg=name)


def test_median_filter_example_object_subclusters(api, example_object):
    ex = example_object
    cs, cl = orc.chr_ranges(ex["chr_codes"])
    X = ex["expr"]
    groups = ex["subclusters"]   # hclust order, as apply_median_filtering walks them
    got = api.median_filter(X, cs, cl, groups, 7)
    want = orc.median_filter(X, cs, cl, groups, 7, nthreads=orc.max_threads())
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-15)


# ---- pairwise distances between cells (the input of every hclust() in the reference, SURVEY 8(f) row 4) -----------------
@pytest.mark.parametrize("G,C,n", [(1000, 300, 257), (17, 9, 5), (333, 130, 129), (48, 2, 2), (1, 40, 40)])
def test_pairwise_dist_vs_oracle(api, G, C, n):
    """icnv_pairwise_dist_f64 = parallelDist(t(X[, cells])) (euclidean) as R's "dist" vector: tile edges (n = 129, 257), a gene
    count that is no multiple of the 16-gene stage, a shuffled subset of the columns, duplicated cells (distance exactly 0)."""
    rng = np.random.default_rng(7 + G)
    X = np.asfortranarray(1.0 + 0.1 * rng.normal(size=(G, C)))
    cells = rng.permutation(C)[:n].astype(np.int32)
    if n >= 5:
        cells[3] = cells[1]          # the same cell twice: distance exactly 0
        X[:, cells[4]] = X[:, cells[0]] + 1e-9   # near-identical cells keep their relative accuracy (difference form)
    got = api.pairwise_dist(X, cells)
    want = orc.pairwise_dist(X, cells, nthreads=orc.max_threads())
    assert got.shape == (n * (n - 1) // 2,)
    np.testing.assert_allclose(got, want, rtol=1e-13, atol=0)
    if n >= 5:
        assert got[n * 1 - 1 * 2 // 2 + (3 - 1 - 1)] == 0.0   # the pair (1, 3)
    # the matrix as parallelDist() receives it (observations x variables = t(X[, cells])): same sums in the same order
    np.testing.assert_array_equal(api.pairwise_dist_rows(np.asfortranarray(X[:, cells].T)), got)
    all_cells = api.pairwise_dist(X)
    np.testing.assert_allclose(all_cells, orc.pairwise_dist(X, nthreads=orc.max_threads()), rtol=1e-13, atol=0)


def test_pairwise_dist_degenerate_shapes_and_errors(api):
    X = np.asfortranarray(np.arange(12, dtype=np.float64).reshape(4, 3))
    assert api.pairwise_dist(X, [2]).size == 0 and api.pairwise_dist(X, []).size == 0
    np.testing.assert_allclose(api.pairwise_dist(X, [0, 2]), [np.sqrt(4 * 2.0 ** 2)])
    with pytest.raises(Exception):
        api.pairwise_dist(X, [0, 3])          # column out of range
    Xn = X.copy(order="F")
    Xn[1, 1] = np.nan                          # NaN propagates to the pairs of that cell only (the R wrapper falls back on NA)
    d = api.pairwise_dist(Xn)
    assert np.isnan(d[0]) and np.isfinite(d[1]) and np.isnan(d[2])


def test_pairwise_dist_example_object(api, example_object):
    """The bundled example's final matrix (4613 genes x 20 cells), observation cells only - the call
    hclust(parallelDist(t(tumor_expr_data))) of define_signif_tumor_subclusters makes (R/inferCNV_tumor_subclusters.R:191)."""
    X = example_object["expr"]
    obs = np.concatenate(example_object["obs_groups"]).astype(np.int32)
    got = api.pairwise_dist(X, obs)
    np.testing.assert_allclose(got, orc.pairwise_dist(X, obs), rtol=1e-13, atol=0)
    assert got.size == len(obs) * (len(obs) - 1) // 2 and np.all(got > 0)
