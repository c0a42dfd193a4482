"""K14 on the GPU: icnv_mask_non_de_f64 against tests/de_reference.py - p_raw within 1e-12 relative, p_adj bit-equal to BH
of the GPU's own p_raw, and Y bit-equal to R's mask from the GPU's p_adj; decisions that differ from the reference's own
p_adj are allowed only within 1e-9 of the threshold (the smallest relative distance is reported).  Under the host
emulation (tests/test_de_emulated_and_r.py) only the small cases run, on a few genes."""
import os

import numpy as np
import pytest

from infercnv_b200 import _lib, api
from infercnv_b200._lib import InfercnvB200Error
from tests import de_reference as dr

pytestmark = pytest.mark.gpu
EMULATED = "_emu" in os.path.basename(_lib.LIB_PATH)
gpu_only = pytest.mark.skipif(EMULATED, reason="GPU only: too large for the host emulation")


@pytest.fixture(scope="module", autouse=True)
def _init():
    api.init(0)


def check(X, refs, subs, test="wilcoxon", thr=0.05, rule="any", jm=1e-4, js=1e-4, seed=0, center_val=None):
    Y, P, A = api.mask_non_de_genes(X, refs, subs, test=test, p_val_thresh=thr, rule=rule, center_val=center_val,
                                    jitter_mean=jm, jitter_sd=js, seed=seed)
    _, RP, RA = dr.mask_non_de(X, refs, subs, test, thr, rule, center_val, jm, js, seed)
    nan = np.isnan(RP)
    assert np.array_equal(np.isnan(P), nan), "NaN pattern of p_raw differs"
    err = np.abs(P[~nan] - RP[~nan]) / np.maximum(np.abs(RP[~nan]), 1e-300)
    assert err.size == 0 or err.max() < 1e-12, f"p_raw: max rel err {err.max():.3e}"
    own = np.column_stack([dr.bh(P[:, c]) for c in range(P.shape[1])]) if P.shape[1] else P
    assert np.array_equal(A.view(np.int64), own.view(np.int64)), "p_adj is not BH of p_raw bit for bit"
    cv = float(np.mean(X)) if center_val is None else center_val
    want_y = dr.mask_from_padj(np.asarray(X, dtype=np.float64), refs, subs, A, thr, rule, cv)
    assert np.array_equal(Y.view(np.int64), want_y.view(np.int64)), "Y differs from R's mask of the GPU's p_adj"
    dec, rdec = A < thr, RA < thr
    close = np.abs(RA - thr) / thr
    if (dec != rdec).any():
        assert close[dec != rdec].max() < 1e-9
    if A.size:
        print(f"\n[non-DE mask] smallest |p_adj - thr| / thr = {np.nanmin(close):.3e}; max rel err p_raw "
              f"{(err.max() if err.size else 0):.3e}")
    return Y, P, A


def dead_band(G, C, seed, frac=0.5):
    """After 2^x the use-bounds dead band leaves many values at exactly 1.0."""
    rng = np.random.default_rng(seed)
    X = 1.0 + rng.normal(scale=0.2, size=(G, C))
    X[rng.uniform(size=(G, C)) < frac] = 1.0
    X[: G // 4, C // 2:] += 0.3
    return np.asfortranarray(X)


def groups(C, sizes, seed):
    perm = np.random.default_rng(seed).permutation(C)
    out, pos = [], 0
    for s in sizes:
        out.append(np.sort(perm[pos:pos + s]))
        pos += s
    return out


G_SMALL = 12 if EMULATED else 300


@pytest.mark.parametrize("js", [0.0, 1e-4])
def test_dead_band_wilcoxon(js):
    X = dead_band(G_SMALL, 240, 1)
    refs, s1, s2, s3, s4 = groups(240, [60, 45, 30, 55, 3], 2)
    check(X, [refs], [s1, s2, s3, s4], js=js, seed=7)


def test_exact_path_and_sizes_around_50():
    X = dead_band(G_SMALL, 400, 3, frac=0.0)
    refs = groups(400, [49, 50, 51], 4)
    subs = groups(400, [1, 49, 50, 51], 5)
    check(X, refs, subs, js=1e-4, seed=11)


def test_t_with_constant_genes():
    X = dead_band(G_SMALL, 200, 5)
    X[0, :] = 2.0                           # constant: NA for every pair
    X[1, :100] = 3.0                        # constant within the groups below
    X[1, 100:] = 4.0
    refs = [np.arange(0, 60), np.arange(60, 100)]
    subs = [np.arange(100, 130), np.arange(130, 131), np.arange(131, 200)]
    _, P, _ = check(X, refs, subs, test="t")
    assert np.isnan(P[0]).all() and np.isnan(P[1]).all() and np.isnan(P[:, 2:4]).all()


@pytest.mark.parametrize("rule", ["any", "most", "all"])
def test_three_reference_groups(rule):
    X = dead_band(G_SMALL, 300, 9, frac=0.2)
    r1, r2, r3, s1, s2, s3 = groups(300, [40, 50, 60, 20, 70, 4], 10)
    extra = np.concatenate([s1[:5], s1[:3]])    # a cell listed twice, and cells in two subclusters
    check(X, [r1, r2, r3], [s1, s2, s3, extra], rule=rule, thr=0.2, seed=3)
    check(X, [r1, r2, r3], [s1, s2, s3], test="t", rule=rule, thr=0.2)


def test_no_tested_subclusters_masks_every_non_reference_cell():
    X = dead_band(G_SMALL, 50, 2)
    refs = [np.arange(10)]
    Y, P, A = check(X, refs, [])
    assert P.shape == (G_SMALL, 0) and (Y[:, 10:] == np.mean(X)).all()


def test_repeatable_and_seeded():
    X = dead_band(G_SMALL, 150, 4, frac=0.1)
    refs, s1, s2 = groups(150, [60, 40, 50], 1)
    a = api.mask_non_de_genes(X, [refs], [s1, s2], seed=5)
    b = api.mask_non_de_genes(X, [refs], [s1, s2], seed=5)
    c = api.mask_non_de_genes(X, [refs], [s1, s2], seed=6)
    for u, v in zip(a, b):
        assert u.tobytes() == v.tobytes()
    assert not np.array_equal(a[1], c[1])


def test_error_codes():
    X = dead_band(8, 20, 0)
    for kw, code in [(dict(refs=[[]]), -3), (dict(subs=[[]]), -3), (dict(refs=[[25]]), -3), (dict(test=2), -3),
                     (dict(rule=3), -3), (dict(js=-1.0), -3)]:
        with pytest.raises(InfercnvB200Error) as e:
            api.mask_non_de_genes(X, kw.get("refs", [[0, 1, 2]]), kw.get("subs", [[5, 6, 7]]), test=kw.get("test", 0),
                                  rule=kw.get("rule", 0), jitter_sd=kw.get("js", 1e-4))
        assert e.value.code == code, kw
    Z = X.copy()
    Z[3, 6] = np.nan
    with pytest.raises(InfercnvB200Error) as e:
        api.mask_non_de_genes(Z, [[0, 1, 2]], [[5, 6, 7]])
    assert e.value.code == -5
    Z = X.copy()
    Z[3, 15] = np.inf                        # outside every list: no error, and masked
    Y, _, _ = api.mask_non_de_genes(Z, [[0, 1, 2]], [[5, 6, 7]], center_val=0.0)
    assert Y[3, 15] == 0.0


def test_oligodendroglioma_step_16(oligo):
    """c1 through the mirror to step 16 (2^x of the smooth block, then the outlier clamp), its two reference groups, each
    tumour group one subcluster."""
    from mirror import ops
    ex = oligo
    G = 40 if EMULATED else ex["counts"].shape[0]
    refs = {f"r{i}": g for i, g in enumerate(ex["ref_groups"])}
    obs = {f"o{i}": g for i, g in enumerate(ex["obs_groups"])}
    o = ops.Infercnv(expr_data=ex["counts"], gene_order_chr=ex["chr_codes"], reference_grouped_cell_indices=refs,
                     observation_grouped_cell_indices=obs)
    o = ops.normalize_counts_by_seq_depth(o)
    o = ops.smooth_block(o, window_length=101, max_centered_threshold=3.0)
    o = ops.remove_outliers_norm(o)
    X = np.asfortranarray(o.expr_data[:G])
    check(X, list(refs.values()), list(obs.values()), seed=20240611)
    o.expr_data = X
    o.tumor_subclusters = {"subclusters": {k: {k: v} for k, v in obs.items()}}
    m = ops.mask_non_DE_genes_basic(o, seed=20240611)
    want, _, _ = api.mask_non_de_genes(X, list(refs.values()), list(obs.values()), seed=20240611)
    assert np.array_equal(m.expr_data, want)
    de = ops.get_DE_genes_basic(o, seed=20240611)
    assert list(de) == [f"{s},{r}" for s in obs for r in refs]


@gpu_only
def test_subcluster_beyond_the_shared_memory_sort():
    X = dead_band(6, 12000, 8, frac=0.3)
    refs, big, small = groups(12000, [2000, 9000, 500], 9)
    check(X, [refs], [big, small], seed=1)
    check(X, [big], [refs, small], seed=2, js=0.0)       # a reference row beyond the bound, ties kept


@gpu_only
def test_engine_equals_api():
    import torch
    from infercnv_b200.device import Engine
    X = dead_band(500, 800, 12)
    refs, s1, s2, s3 = groups(800, [200, 100, 150, 4], 13)
    cv = float(np.mean(X))      # explicit: torch's and NumPy's means may differ in the last bits
    want = api.mask_non_de_genes(X, [refs], [s1, s2, s3], seed=4, center_val=cv)
    eng = Engine(0)
    T = torch.as_tensor(np.ascontiguousarray(X.T), device=eng.tdev)
    Y, P, A = eng.mask_non_de(T, [refs], [s1, s2, s3], seed=4, center_val=cv)
    assert np.array_equal(Y.cpu().numpy().T, want[0])
    assert np.array_equal(P.cpu().numpy().T, want[1]) and np.array_equal(A.cpu().numpy().T, want[2])
    eng.mask_non_de(T, [refs], [s1, s2, s3], seed=4, center_val=cv, out=T)   # in place
    assert np.array_equal(T.cpu().numpy().T, want[0])


@gpu_only
def test_large_run_100k_cells():
    G, C = 2000, 100000
    rng = np.random.default_rng(0)
    X = np.asfortranarray(1.0 + rng.normal(scale=0.1, size=(G, C)))
    X[:200, 50000:] += 0.05
    refs = [np.arange(0, 6000), np.arange(6000, 10000)]
    sizes = rng.integers(50, 500, size=400)
    subs, pos = [], 10000
    for s in sizes:
        if pos + s > C:
            break
        subs.append(np.arange(pos, pos + s))
        pos += s
    Y, P, A = api.mask_non_de_genes(X, refs, subs, seed=3)
    st = api.mask_non_de_stats()
    print(f"\n[non-DE mask 100k x 2000, {len(subs)} subclusters] stages {st}")
    assert P.shape == (G, len(subs) * 2) and np.isfinite(P).all()
    for g in (0, 1, 1999):            # spot check against the reference
        for col in (0, 1, 2 * len(subs) - 1):
            s, j = divmod(col, 2)
            x = dr.jittered(X[g, refs[j]], 3, j, g, 1e-4, 1e-4)
            y = dr.jittered(X[g, subs[s]], 3, dr.SUB_KEY + col, g, 1e-4, 1e-4)
            assert abs(P[g, col] - dr.wilcox_p(x, y)) <= 1e-12 * dr.wilcox_p(x, y)
    assert (A[:200, 160:] < 0.05).mean() > (A[200:, 160:] < 0.05).mean()
