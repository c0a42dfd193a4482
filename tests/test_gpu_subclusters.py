"""K17 on the GPU: the z-score gene filter (icnv_zscore_outlier_genes_f64) against its restatement in exact rationals, and the
group trees (icnv_cluster_groups_f64) bit for bit equal to per-group icnv_pairwise_dist_f64 -> icnv_hclust_f64, whatever the
group sizes, order, gene list or number of waves; then Engine and mirror.ops.define_signif_tumor_subclusters.  Under the
host emulation (tests/test_subclusters_emulated_and_r.py; 4 SMs, so several waves from 5 groups on) the groups are small."""
import os

import numpy as np
import pytest

from infercnv_b200 import _lib, api
from infercnv_b200._lib import InfercnvB200Error
from tests import subclusters_reference as sr

pytestmark = pytest.mark.gpu
EMULATED = "_emu" in os.path.basename(_lib.LIB_PATH)
METHODS = ["single", "complete", "average", "mcquitty", "ward.D", "ward.D2"]
gpu_only = pytest.mark.skipif(EMULATED, reason="GPU only: too large for the host emulation")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module", autouse=True)
def _init():
    api.init(0)


def same_tree(got, want):
    m, h, o = got
    wm, wh, wo = want
    assert np.array_equal(m, wm), "merge differs"
    assert h.tobytes() == np.asarray(wh, dtype=np.float64).tobytes(), "height differs"
    assert np.array_equal(o, wo), "order differs"


def per_group(X, groups, method, keep=None):
    Xk = X if keep is None else np.asfortranarray(X[np.asarray(keep, dtype=np.int64)])
    out = []
    for g in groups:
        n = len(g)
        if n < 2:
            out.append((np.zeros((0, 2), np.int32), np.zeros(0), np.arange(1, n + 1, dtype=np.int32)))
        else:
            out.append(api.hclust(api.pairwise_dist(Xk, g), method))
    return out


def check_all(X, groups, method, keep=None):
    got = api.cluster_groups(X, groups, method=method, keep=keep)
    assert len(got) == len(groups)
    for t, w in zip(got, per_group(X, groups, method, keep)):
        same_tree(t, w)
    return got


def random_groups(rng, C, sizes):
    perm = rng.permutation(C)
    out, at = [], 0
    for n in sizes:
        out.append(perm[at:at + n].astype(np.int32))
        at += n
    return out


# ---- the filter -------------------------------------------------------------------------------------------------------

def scaled(G, C, seed):
    rng = np.random.default_rng(seed)
    return np.asfortranarray(rng.normal(size=(G, C)) * rng.uniform(0.1, 2.0, size=(G, 1)) + rng.normal(size=(G, 1)) * 0.3)


@pytest.mark.parametrize("shape", [(300, 40), (1031, 9)] + ([] if EMULATED else [(10000, 300)]))
def test_filter_equals_the_restatement(shape):
    G, C = shape
    X = scaled(G, C, G + C)
    ref = np.random.default_rng(1).permutation(C)[: max(C // 2, 2)].astype(np.int32)
    mu, sigma = api.mean_sd(X, ref)
    mask = api.zscore_outlier_genes(X, ref)
    want = sr.outlier_mask(X, ref, mu, sigma)
    assert mask.dtype == bool and np.array_equal(mask, want)
    assert 0 < mask.sum() < G
    # mu / sigma are api.mean_sd's bits; against R's mean() / sd() of the whole reference matrix they agree to a few ulp
    from oracle.denoise import r_mean
    vals = X[:, ref]
    assert abs(mu - r_mean(vals)) <= 1e-13 * np.abs(vals).max()
    assert abs(sigma - sr.r_sd(vals.ravel(order="F"))) <= 1e-12 * sigma


def _tune(x, mu, sigma, target):
    """The double near x whose |(x - mu) / sigma| is closest to target."""
    best, bd = x, None
    for s in range(-16, 17):
        v = x
        for _ in range(abs(s)):
            v = np.nextafter(v, np.inf if s > 0 else -np.inf)
        d = abs(float(sr.zscores(np.array([[v]]), [0], mu, sigma)[0, 0]) - target)
        if bd is None or d < bd:
            best, bd = v, d
    return best


def test_filter_at_the_threshold():
    """Genes whose mean |z| sits within a few ulp of 0.8, on both sides and on the midpoints: the last value of each is
    tuned against the mu / sigma the call will use (re-read until they stop moving)."""
    from fractions import Fraction
    rng = np.random.default_rng(5)
    G, n = 400, 12
    X = np.asfortranarray(rng.normal(size=(G, n)) * 1.3)
    ref = np.arange(n, dtype=np.int32)
    mu, sigma = api.mean_sd(X, ref)          # the tuned genes sit near |z| = 0.8, where they barely move mu and sigma
    X[G - 17:] = mu + sigma * (0.8 + 0.05 * rng.normal(size=(17, n))) * rng.choice([-1.0, 1.0], size=(17, n))
    ulp = np.spacing(0.8)
    targets = {g: Fraction(0.8) + Fraction(k - 8) * Fraction(ulp) / 2 for k, g in enumerate(range(G - 17, G))}
    for _ in range(12):
        mu, sigma = api.mean_sd(X, ref)
        for g, t in targets.items():
            z = sr.zscores(X[g:g + 1, : n - 1], np.arange(n - 1), mu, sigma)[0]
            need = t * n - sum((Fraction(float(v)) for v in z), Fraction(0))
            X[g, n - 1] = _tune(mu + float(need) * sigma, mu, sigma, float(need))
        if api.mean_sd(X, ref) == (mu, sigma):
            break
    mu, sigma = api.mean_sd(X, ref)
    Z = sr.zscores(X, ref, mu, sigma)
    exact = sr.row_mean_exact(Z)
    near = np.abs(exact[list(targets)] - 0.8) <= 4 * ulp
    assert near.sum() >= 8
    got = api.zscore_outlier_genes(X, ref)
    assert np.array_equal(got, exact >= 0.8)
    side = got[list(targets)][near]
    assert side.any() and not side.all()
    if sr.HAS_EXTENDED:
        assert np.array_equal(sr.row_mean_r(Z), exact)


def test_constant_reference_flags_no_gene():
    X = np.full((50, 8), 3.0)
    X[:, 5:] = np.random.default_rng(0).normal(size=(50, 3))   # only columns 0 .. 4 are the reference
    ref = np.arange(5, dtype=np.int32)
    assert api.mean_sd(X, ref) == (3.0, 0.0)
    assert not api.zscore_outlier_genes(X, ref).any()
    assert not sr.outlier_mask(X, ref, 3.0, 0.0).any()


def test_filter_errors():
    X = scaled(20, 6, 3)
    for ref, code in [([0, 6], -3), ([-1], -3), ([], -3)]:
        with pytest.raises(InfercnvB200Error) as e:
            api.zscore_outlier_genes(X, np.array(ref, dtype=np.int32))
        assert e.value.code == code
    X[4, 2] = np.nan
    with pytest.raises(InfercnvB200Error) as e:
        api.zscore_outlier_genes(X, [1, 2, 3])
    assert e.value.code == -5
    api.zscore_outlier_genes(X, [0, 1, 3])   # the NaN is in a column that is not listed


# ---- the trees --------------------------------------------------------------------------------------------------------

SIZES = [2, 3, 33, 0, 1, 17, 5] if EMULATED else [2, 3, 33, 1025, 4097, 0, 1]


@pytest.mark.parametrize("method", METHODS)
def test_mixed_sizes_equal_per_group_calls(method):
    rng = np.random.default_rng(11)
    G = 40 if EMULATED else 200
    C = sum(SIZES) + 7
    X = np.asfortranarray(rng.normal(size=(G, C)))
    X[: G // 3, : C // 2] += 1.0
    groups = random_groups(rng, C, SIZES)
    groups.append(np.concatenate([groups[1], groups[0]]))   # a column listed by two groups
    got = check_all(X, groups, method)
    st = api.cluster_groups_stats()
    assert st["waves"] >= 1 and st["widest"] >= 1


@pytest.mark.parametrize("method", METHODS)
def test_tie_laden_data(method):
    rng = np.random.default_rng(2)
    X = np.asfortranarray(np.round(rng.normal(size=(6, 90)) * 1.5) / 2)
    X[:, 40:50] = X[:, 30:40]                                 # duplicated cells: zero distances
    groups = [np.arange(0, 60, dtype=np.int32), np.arange(25, 90, dtype=np.int32)[::-1].copy(), np.arange(60, 67, dtype=np.int32)]
    check_all(X, groups, method)


def test_keep_list_and_no_genes():
    rng = np.random.default_rng(3)
    X = np.asfortranarray(rng.normal(size=(120, 70)))
    groups = random_groups(rng, 70, [30, 9, 2, 20])
    keep = rng.permutation(120)[:47].astype(np.int32)
    check_all(X, groups, "ward.D2", keep=keep)
    check_all(X, groups, "average", keep=np.sort(keep))
    none = api.cluster_groups(X, groups, method="ward.D2", keep=[])
    for t, g in zip(none, groups):
        assert np.all(t[1] == 0.0)                            # every distance is 0
        same_tree(t, api.hclust(np.zeros(len(g) * (len(g) - 1) // 2), "ward.D2"))


def test_many_groups_run_in_several_waves():
    rng = np.random.default_rng(4)
    n_grp = 9 if EMULATED else 200
    sizes = rng.integers(3, 13 if EMULATED else 61, size=n_grp).tolist()
    C = sum(sizes)
    X = np.asfortranarray(rng.normal(size=(30, C)))
    groups = random_groups(rng, C, sizes)
    got = check_all(X, groups, "ward.D2")
    st = api.cluster_groups_stats()
    assert st["waves"] >= 2, st
    # the same trees whatever the order the groups come in
    perm = rng.permutation(n_grp)
    again = api.cluster_groups(X, [groups[i] for i in perm], method="ward.D2")
    for j, i in enumerate(perm):
        same_tree(again[j], got[i])


def test_no_group_with_a_tree():
    X = np.ones((4, 3))
    got = api.cluster_groups(X, [[0], [], [2]])
    assert [t[2].tolist() for t in got] == [[1], [], [1]]
    assert all(t[0].shape == (0, 2) and t[1].size == 0 for t in got)


def test_group_error_codes():
    X = np.asfortranarray(np.random.default_rng(6).normal(size=(10, 8)))
    cases = [(dict(method=5), -4), (dict(method=6), -4), (dict(method=8), -3), (dict(method=-1), -3),
             (dict(groups=[[0, 8]]), -3), (dict(groups=[[0, -1, 2]]), -3), (dict(keep=[0, 10]), -3)]
    for kw, code in cases:
        kw = dict(kw)
        groups = kw.pop("groups", [[0, 1, 2], [3, 4]])
        with pytest.raises(InfercnvB200Error) as e:
            api.cluster_groups(X, groups, **kw)
        assert e.value.code == code, kw
    with pytest.raises(InfercnvB200Error) as e:   # refused before anything is allocated or uploaded
        api.cluster_groups(np.zeros((2, 3)), [[0, 1], np.zeros(65537, dtype=np.int32)])
    assert e.value.code == -4
    Y = X.copy()
    Y[3, 4] = np.nan
    with pytest.raises(InfercnvB200Error) as e:
        api.cluster_groups(Y, [[0, 1, 2], [3, 4]])
    assert e.value.code == -5
    check_all(Y, [[0, 1, 2], [5, 6, 7], [4]], "complete")   # column 4 is only in a one-cell group: no distance uses it


# ---- Engine and the ops mirror -----------------------------------------------------------------------------------------

@gpu_only
def test_engine_equals_the_host_calls():
    import torch
    from infercnv_b200.device import Engine
    rng = np.random.default_rng(8)
    X = scaled(500, 300, 8)
    eng = Engine(0)
    T = torch.as_tensor(np.ascontiguousarray(X.T), device=eng.tdev)
    ref = rng.permutation(300)[:60].astype(np.int32)
    assert np.array_equal(eng.zscore_outlier_genes(T, ref).cpu().numpy(), api.zscore_outlier_genes(X, ref))
    groups = random_groups(rng, 300, [100, 2, 1, 57, 140])
    keep = rng.permutation(500)[:321]
    for kp in (None, keep, []):
        for a, b in zip(eng.cluster_groups(T, groups, "ward.D2", keep=kp), api.cluster_groups(X, groups, "ward.D2", keep=kp)):
            same_tree(a, b)
    with pytest.raises(InfercnvB200Error) as e:
        eng.cluster_groups(T, [[0, 1, 300]])
    assert e.value.code == -3


def restated(obj, partition_method, z_score_filter, p_val=0.1, method="ward.D2"):
    """define_signif_tumor_subclusters by separate calls: filter restatement, per-group distances and hclust, R's cut."""
    refs, obs = obj.reference_grouped_cell_indices, obj.observation_grouped_cell_indices
    keep = None
    if z_score_filter > 0 and refs:
        ref = np.concatenate([np.asarray(v) for v in refs.values()])
        mu, sigma = api.mean_sd(obj.expr_data, ref)
        out = sr.outlier_mask(obj.expr_data, ref, mu, sigma)
        keep = np.flatnonzero(~out) if out.any() else np.zeros(0, np.int64)
    X = obj.expr_data if keep is None else np.asfortranarray(obj.expr_data[keep])
    res = {}
    for g, idx in {**obs, **refs}.items():
        idx = np.asarray(idx)
        if len(idx) <= 2:
            res[g] = (None, {f"{g}_s1": idx})
            continue
        merge, height, order = api.hclust(api.pairwise_dist(X, idx), method)
        cut = sr.cut_height(height, partition_method, p_val)
        grps = sr.cutree(merge, height, k=1) if cut is None else sr.cutree(merge, height, h=cut)
        res[g] = ((merge, height, order), sr.assemble(g, idx, order, grps))
    return res


def check_mirror(obj, partition_method, z_score_filter):
    from mirror import ops
    got, per_chr = ops.define_signif_tumor_subclusters(obj, partition_method=partition_method, z_score_filter=z_score_filter)
    assert per_chr is None
    want = restated(obj, partition_method, z_score_filter)
    ts = got.tumor_subclusters
    assert list(ts["subclusters"]) == list(want)
    for g, (tree, subs) in want.items():
        if tree is None:
            assert ts["hc"][g] is None
        else:
            hc = ts["hc"][g]
            same_tree((hc["merge"], hc["height"], hc["order"]), tree)
            assert hc["method"] == "ward.D2" and hc["dist.method"] == "euclidean"
        assert list(ts["subclusters"][g]) == list(subs)
        for name in subs:
            assert np.array_equal(ts["subclusters"][g][name], subs[name])
    return ts


def example_object():
    from mirror import ops
    z = np.load(os.path.join(GOLD, "example_object.npz"))
    groups = lambda names, idx, off: {str(n): idx[off[k]:off[k + 1]] - 1 for k, n in enumerate(names)}   # noqa: E731
    return ops.Infercnv(expr_data=z["expr"], gene_order_chr=z["chr_codes"],
                        reference_grouped_cell_indices=groups(z["ref_names"], z["ref_idx"], z["ref_off"]),
                        observation_grouped_cell_indices=groups(z["obs_names"], z["obs_idx"], z["obs_off"]))


@pytest.mark.parametrize("partition_method", ["none", "qnorm", "pheight"])
@pytest.mark.parametrize("z_score_filter", [0, 0.8])
def test_mirror_on_the_example(partition_method, z_score_filter):
    check_mirror(example_object(), partition_method, z_score_filter)


@gpu_only
@pytest.mark.parametrize("partition_method", ["none", "qnorm"])
def test_mirror_on_a_seeded_object(partition_method):
    from mirror import ops
    rng = np.random.default_rng(2024)
    G, C = 2000, 5000
    X = rng.normal(size=(G, C)) * 0.2
    X[300:700, :1200] += 0.5
    X[1500:1800, 1200:2000] -= 0.4
    X[:40] *= 6.0                                            # genes the z-score filter removes
    perm = rng.permutation(C)
    obs = {"a": perm[:2000], "b": perm[2000:3500], "c": perm[3500:4500]}
    refs = {"r1": perm[4500:4800], "r2": perm[4800:]}
    obj = ops.Infercnv(expr_data=X, gene_order_chr=np.zeros(G, np.int32), reference_grouped_cell_indices=refs,
                       observation_grouped_cell_indices=obs)
    ts = check_mirror(obj, partition_method, 0.8)
    assert sum(len(v) for v in ts["subclusters"]["a"].values()) == 2000


def test_mirror_refuses_what_is_not_on_the_gpu():
    from mirror import ops
    obj = example_object()
    for kw in (dict(partition_method="leiden"), dict(partition_method="qgamma"),
               dict(partition_method="none", restrict_to_DE_genes=True)):
        with pytest.raises(NotImplementedError):
            ops.define_signif_tumor_subclusters(obj, **kw)
