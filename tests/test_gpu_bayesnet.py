"""K15 on the GPU: icnv_bayesnet_f64 (inferCNVBayesNet's Gibbs sampling) against tests/bayesnet_reference.py - the
log-likelihoods within 1e-12 relative of the NumPy restatement, and the sampled posterior against the exact posterior by
enumeration, every statistical bound at least 5 standard errors wide with fixed seeds.  Under the host emulation
(tests/test_bayesnet_emulated_and_r.py) the small cases run with fewer chains and sweeps."""
import os

import numpy as np
import pytest

from infercnv_b200 import _lib, api
from infercnv_b200._lib import InfercnvB200Error
from tests import bayesnet_reference as br

pytestmark = pytest.mark.gpu
EMULATED = "_emu" in os.path.basename(_lib.LIB_PATH)
gpu_only = pytest.mark.skipif(EMULATED, reason="GPU only: too large for the host emulation")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

MU6 = np.array([0.4, 0.7, 1.0, 1.3, 1.6, 1.9])
TAU6 = np.array([30.0, 40.0, 60.0, 40.0, 30.0, 20.0])


@pytest.fixture(scope="module", autouse=True)
def _init():
    api.init(0)


def overlapping_region(C, G, m, seed):
    """G genes x C cells drawn from random states of mu / tau with heavy overlap: non-degenerate posteriors."""
    rng = np.random.default_rng(seed)
    mu, tau = MU6[:m] if m == 6 else np.array([0.8, 1.0, 1.2]), TAU6[:m] if m == 6 else np.array([30.0, 40.0, 30.0])
    states = rng.integers(0, m, size=C)
    X = np.asfortranarray(rng.normal(mu[states][None, :], 1.0 / np.sqrt(tau[states])[None, :], size=(G, C)))
    return X, mu, tau


def test_loglik_matches_numpy():
    rng = np.random.default_rng(1)
    X = np.asfortranarray(rng.normal(1.0, 0.3, size=(60, 40)))
    genes = [np.arange(5, 30), rng.permutation(60)[:17], np.array([7]), np.array([3, 3, 9])]
    cells = [np.arange(40), rng.permutation(40)[:11], np.array([0, 5, 9, 33]), np.array([2])]
    pooled = [False, False, True, False]
    res = api.bayesnet(X, genes, cells, MU6, TAU6, 2, n_burn=1, n_keep=2, pooled=pooled, want_loglik=True)
    for r in range(4):
        want = br.loglik(X, genes[r], cells[r], MU6, TAU6, pooled=pooled[r])
        got = res["loglik"][r]
        assert got.shape == want.shape
        assert np.all(np.abs(got - want) <= 1e-12 * np.abs(want)), r


def test_decisive_cells_are_certain():
    """Cells whose L margin is >= 200 nats sit in their arg-max state in every kept draw."""
    C, m = 12, 6
    rng = np.random.default_rng(2)
    states = rng.integers(0, m, size=C)
    X = np.asfortranarray(np.repeat(MU6[states][None, :], 400, axis=0) + rng.normal(0, 0.01, size=(400, C)))
    res = api.bayesnet(X, [np.arange(400)], [np.arange(C)], MU6, TAU6, 6, n_burn=20, n_keep=50 if EMULATED else 300,
                       want_loglik=True)
    L = res["loglik"][0]
    srt = np.sort(L, axis=0)
    margin = srt[-1] - srt[-2]
    dec = margin >= 200
    assert dec.sum() >= 6
    P = res["cell_probabilities"][0]
    assert np.all(P[np.argmax(L, axis=0)[dec], np.flatnonzero(dec)] == 1.0)


@pytest.mark.parametrize("m", [3, 6])
def test_many_short_chains_match_the_enumerated_posterior(m):
    C = 4 if m == 6 else 5
    X, mu, tau = overlapping_region(C, 3, m, 10 + m)
    chains = 256 if EMULATED else 4096
    res = api.bayesnet(X, [np.arange(3)], [np.arange(C)], mu, tau, chains, n_burn=50, n_keep=1, seed=7, want_loglik=True)
    P, E = br.enumerate_posterior(res["loglik"][0])
    F = res["cell_probabilities"][0]
    se = np.sqrt(P * (1 - P) / chains)
    assert np.all(np.abs(F - P) <= 5 * se + 2e-3), np.abs(F - P).max()
    th = res["theta"][0]
    se_t = th.std(axis=0) / np.sqrt(chains)
    assert np.all(np.abs(th.mean(axis=0) - E) <= 5 * se_t + 1e-3)
    assert 0.02 < P.max() - P.min()        # not degenerate


@gpu_only
def test_r_defaults_match_the_posterior_by_batch_means():
    X, mu, tau = overlapping_region(5, 4, 6, 21)
    res = api.bayesnet(X, [np.arange(4)], [np.arange(5)], mu, tau, 6, seed=11, want_loglik=True)
    P, E = br.enumerate_posterior(res["loglik"][0])
    th = res["theta"][0]
    assert th.shape == (6000, 6)
    batches = th.reshape(6, 20, 50, 6).mean(axis=2).reshape(120, 6)
    se = batches.std(axis=0, ddof=1) / np.sqrt(120)
    assert np.all(np.abs(th.mean(axis=0) - E) <= 5 * se + 1e-4), (th.mean(axis=0), E, se)
    assert np.all(res["state_counts"][0].sum(axis=0) == 6000)


def test_fixture_regions_and_rao_blackwell():
    """The 9 regions of the reference's JAGS run (data/mcmc_obj.rda) with its mu and sig, on the pre-denoise block of the
    same example reproduced by the oracle (the smooth block of its depth-normalised counts): mean theta against
    (1 + sum_j P(eps_j = k)) / (m + C) within 0.01.  Per-cell modal agreement with the JAGS output is reported, not
    asserted: the fixture does not store the matrix JAGS saw (a NumPy arg-max of L on this block agrees for 71 of 90)."""
    from oracle import oracle as orc
    d = np.load(os.path.join(GOLDEN, "bayesnet_fixture.npz"))
    ex = np.load(os.path.join(GOLDEN, "example_object.npz"))
    cs, cl = orc.chr_ranges(ex["chr_codes"])
    refs = [ex["ref_idx"][ex["ref_off"][i]:ex["ref_off"][i + 1]] - 1 for i in range(len(ex["ref_off"]) - 1)]
    X = np.asfortranarray(orc.smooth_block(orc.normalize_by_seq_depth(ex["counts"].astype(np.float64)), cs, cl, refs))
    go, gi, co, ci = d["gene_off"], d["gene_idx"], d["cell_off"], d["cell_idx"]
    n = 3 if EMULATED else 9
    genes = [gi[go[r]:go[r + 1]] for r in range(n)]
    cells = [ci[co[r]:co[r + 1]] for r in range(n)]
    res = api.bayesnet(X, genes, cells, d["mu"], d["sig"], 6, n_burn=100 if EMULATED else 700,
                       n_keep=200 if EMULATED else 1000, seed=3)
    agree = argmax_agree = 0
    for r in range(n):
        P, th = res["cell_probabilities"][r], res["theta"][r]
        rb = (1.0 + P.sum(axis=1)) / (6 + P.shape[1])
        assert np.abs(rb - th.mean(axis=0)).max() < 0.01, r
        agree += int((P.argmax(axis=0) == d["cell_prob"][r].argmax(axis=0)).sum())
        L = br.loglik(X, genes[r], cells[r], d["mu"], d["sig"])
        argmax_agree += int((L.argmax(axis=0) == d["cell_prob"][r].argmax(axis=0)).sum())
    print(f"\n[bayesnet fixture] per-cell modal state equal to JAGS's for {agree} of {10 * n} cells "
          f"(NumPy arg-max of L: {argmax_agree})")


def test_pooled_one_gene_quirk_and_m3():
    X, mu, tau = overlapping_region(8, 1, 3, 4)
    res = api.bayesnet(X, [np.array([0]), np.array([0])], [np.arange(8), np.arange(8)], mu, tau, 3, n_burn=10, n_keep=40,
                       pooled=[True, False], want_loglik=True)
    assert res["loglik"][0].shape == (3, 1) and res["loglik"][1].shape == (3, 8)
    assert np.allclose(res["loglik"][0][:, 0], res["loglik"][1].sum(axis=1), rtol=1e-12)
    assert res["cell_probabilities"][0].shape == (3, 1)
    assert res["state_counts"][0].sum() == 120 and np.all(res["state_counts"][1].sum(axis=0) == 120)
    assert res["theta"][0].shape == (120, 3)
    assert np.all(np.abs(res["theta"][1].sum(axis=1) - 1.0) <= 1e-12)


def test_error_codes():
    X = np.asfortranarray(np.ones((5, 4)))
    good = dict(genes=[[0, 1]], cells=[[0, 1]], mu=MU6, tau=TAU6, n_chains=2, n_burn=1, n_keep=1)
    cases = [dict(genes=[[]]), dict(cells=[[]]), dict(genes=[[5]]), dict(cells=[[-1]]), dict(mu=MU6[:1], tau=TAU6[:1]),
             dict(mu=np.zeros(9), tau=np.ones(9)), dict(tau=np.r_[TAU6[:5], 0.0]), dict(mu=np.r_[MU6[:5], np.nan]),
             dict(tau=np.r_[TAU6[:5], np.inf]), dict(n_chains=0), dict(n_keep=0), dict(n_burn=-1)]
    for kw in cases:
        a = dict(good, **kw)
        with pytest.raises(InfercnvB200Error) as e:
            api.bayesnet(X, a["genes"], a["cells"], a["mu"], a["tau"], a["n_chains"], n_burn=a["n_burn"], n_keep=a["n_keep"])
        assert e.value.code == -3, kw
    Z = X.copy()
    Z[1, 1] = np.nan
    with pytest.raises(InfercnvB200Error) as e:
        api.bayesnet(Z, [[0, 1]], [[0, 1]], MU6, TAU6, 2, n_burn=1, n_keep=1)
    assert e.value.code == -5
    Z[1, 1], Z[4, 3] = 1.0, np.inf          # outside the region: no error
    api.bayesnet(Z, [[0, 1]], [[0, 1]], MU6, TAU6, 2, n_burn=1, n_keep=1)


def test_repeatable_and_seeded():
    X, mu, tau = overlapping_region(30, 20, 6, 9)
    args = ([np.arange(20), np.arange(5, 12)], [np.arange(30), np.arange(0, 30, 2)], mu, tau, 6)
    a = api.bayesnet(X, *args, n_burn=20, n_keep=30, seed=5)
    b = api.bayesnet(X, *args, n_burn=20, n_keep=30, seed=5)
    c = api.bayesnet(X, *args, n_burn=20, n_keep=30, seed=6)
    for r in range(2):
        assert np.array_equal(a["theta"][r], b["theta"][r]) and np.array_equal(a["state_counts"][r], b["state_counts"][r])
    assert not np.array_equal(a["theta"][0], c["theta"][0])
    # the first chains' draws do not depend on how many chains run beside them
    d = api.bayesnet(X, *args[:4], 2, n_burn=20, n_keep=30, seed=5)
    assert np.array_equal(d["theta"][0], np.concatenate([a["theta"][0][:30], a["theta"][0][30:60]]))


@gpu_only
def test_engine_equals_api():
    import torch
    from infercnv_b200.device import Engine
    X, mu, tau = overlapping_region(300, 120, 6, 12)
    genes = [np.arange(0, 40), np.arange(40, 120), np.array([7])]
    cells = [np.arange(300), np.arange(0, 300, 3), np.arange(50)]
    want = api.bayesnet(X, genes, cells, mu, tau, 6, n_burn=50, n_keep=100, seed=4, pooled=[False, False, True],
                        want_loglik=True)
    eng = Engine(0)
    T = torch.as_tensor(np.ascontiguousarray(X.T), device=eng.tdev)
    got = eng.bayesnet(T, genes, cells, mu, tau, 6, n_burn=50, n_keep=100, seed=4, pooled=[False, False, True],
                       want_loglik=True)
    for k in ("theta", "state_counts", "loglik"):
        for r in range(3):
            assert np.array_equal(got[k][r], want[k][r]), (k, r)


@gpu_only
def test_full_size_3300_regions_100k_cells():
    import torch
    from infercnv_b200.device import Engine
    G, C, K = 10000, 100000, 22
    cl = np.full(K, G // K, dtype=np.int32)
    cl[: G - cl.sum()] += 1
    cs = np.concatenate([[0], np.cumsum(cl)[:-1]]).astype(np.int32)
    eng = Engine(0)
    T = eng.synth(G, cs, cl, np.arange(C), C, 1)
    T = torch.log2(T + 1.0) * 0.25 + 0.6           # around the states' means
    genes, cells = [], []
    for s in range(50):
        sub = np.arange(s * 2000, (s + 1) * 2000, dtype=np.int32)
        for k in range(K):
            b = np.linspace(cs[k], cs[k] + cl[k], 4).astype(int)
            for q in range(3):
                genes.append(np.arange(b[q], b[q + 1], dtype=np.int32))
                cells.append(sub)
    res = eng.bayesnet(T, genes, cells, MU6, TAU6, 6, seed=2)
    st = api.bayesnet_stats()
    print(f"\n[bayesnet {len(genes)} regions x 2000 cells, 10 000 genes] {st}")
    assert st["regions"] == len(genes) == 3300
    for r in range(len(genes)):
        assert np.all(res["state_counts"][r].sum(axis=0) == 6000)
        assert np.all(np.abs(res["theta"][r].sum(axis=1) - 1.0) <= 1e-12)


def test_mirror_regions_from_the_hmm_report_feed_the_sampler():
    """data/HMM_states.rda through the library's region report (by subcluster) and the mirror's @cell_gene gives exactly the
    regions, genes and cells of the reference's own run (data/mcmc_obj.rda@cell_gene), and the mirror's sampling step
    returns R's shapes for them."""
    from mirror import ops
    z = np.load(os.path.join(GOLDEN, "cnv_regions_fixture.npz"))
    d = np.load(os.path.join(GOLDEN, "bayesnet_fixture.npz"))
    levels = [str(s) for s in z["chr_levels"]]
    cell_names = [str(s) for s in z["cell_names"]]
    obj = ops.Infercnv(expr_data=z["hmm_states"].astype(np.float64), gene_order_chr=z["chr_codes"],
                       reference_grouped_cell_indices={"normal": z["ref_idx"] - 1},
                       observation_grouped_cell_indices={"tumor": z["obs_idx"] - 1},
                       tumor_subclusters={"subclusters": {"tumor": {"tumor_s1": z["subcluster_cells"] - 1}}},
                       gene_names=[str(s) for s in z["gene_names"]], gene_order_start=z["gene_start"],
                       gene_order_stop=z["gene_stop"], cell_names=cell_names,
                       chr_names={i + 1: n for i, n in enumerate(levels)})
    cg = ops.cell_gene_from_regions(ops.get_predicted_CNV_regions(obj, by="subcluster"), cell_names, "i6")
    go, gi, co, ci = d["gene_off"], d["gene_idx"], d["cell_off"], d["cell_idx"]
    assert [g["cnv_regions"] for g in cg] == z["region_names"].tolist()
    for r, g in enumerate(cg):
        assert g["Genes"].tolist() == gi[go[r]:go[r + 1]].tolist()
        assert g["Cells"].tolist() == ci[co[r]:co[r + 1]].tolist()
    ex = np.load(os.path.join(GOLDEN, "example_object.npz"))
    mc = ops.inferCNVBayesNet_sampling(ex["expr"], cg, d["mu"], d["sig"], "i6", n_burn=20, n_keep=30, seed=1)
    assert len(mc["cnv_probabilities"]) == len(cg) == 9
    for th, cp, g in zip(mc["cnv_probabilities"], mc["cell_probabilities"], cg):
        assert th.shape == (180, 6) and cp.shape == (6, len(g["Cells"]))
        assert np.allclose(cp.sum(axis=0), 1.0)
