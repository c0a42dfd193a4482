"""CPU checks of tests/bayesnet_reference.py, the expected values of the Bayesian network filter: the enumerated posterior
against quadrature over theta, the Rao-Blackwell identity on the reference's own JAGS output, and the mirror's removeCNV /
reassignCNV on hand cases."""
import os

import numpy as np
import pytest

from tests import bayesnet_reference as br

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("C", [1, 2, 3])
def test_enumeration_matches_quadrature(C):
    rng = np.random.default_rng(C)
    L = rng.normal(scale=1.5, size=(3, C))
    P, E = br.enumerate_posterior(L)
    Pq, Eq = br.simplex_integral(L)
    assert np.allclose(P.sum(axis=0), 1.0) and np.isclose(E.sum(), 1.0)
    assert np.abs(P - Pq).max() < 2e-3
    assert np.abs(E - Eq).max() < 2e-3


def test_rao_blackwell_identity_on_the_jags_fixture():
    d = np.load(os.path.join(GOLDEN, "bayesnet_fixture.npz"))
    cp, tm = d["cell_prob"], d["theta_mean"]
    m, C = cp.shape[1], cp.shape[2]
    assert m == 6 and tm.shape == (9, 6)
    rb = (1.0 + cp.sum(axis=2)) / (m + C)
    assert np.abs(rb - tm).max() < 0.004


def test_loglik_restatement_and_pooled_quirk():
    rng = np.random.default_rng(0)
    X = rng.normal(size=(7, 5))
    mu, tau = np.array([0.5, 1.0, 1.5]), np.array([4.0, 9.0, 2.0])
    L = br.loglik(X, [1, 3, 4], [0, 2], mu, tau)
    direct = np.array([[np.sum(0.5 * np.log(tau[k]) - 0.5 * tau[k] * (X[[1, 3, 4], c] - mu[k]) ** 2) for c in (0, 2)]
                       for k in range(3)])
    assert np.allclose(L, direct, rtol=1e-13)
    Lp = br.loglik(X, [2], [0, 1, 4], mu, tau, pooled=True)
    assert Lp.shape == (3, 1)
    assert np.allclose(Lp[:, 0], br.loglik(X, [2], [0, 1, 4], mu, tau).sum(axis=1), rtol=1e-13)


def test_numpy_gibbs_matches_enumeration():
    rng = np.random.default_rng(5)
    L = rng.normal(scale=1.0, size=(3, 4))
    P, E = br.enumerate_posterior(L)
    theta, counts = br.gibbs(L, 200, 30, 20, rng)
    assert np.abs(counts / 4000.0 - P).max() < 0.04
    assert np.abs(theta.mean(axis=0) - E).max() < 0.02


def _mcmc(theta_means, genes, cells, hmm_type="i6"):
    ths = [np.tile(np.asarray(t, dtype=float), (4, 1)) for t in theta_means]
    cg = [{"cnv_regions": f"r{i}", "Genes": np.asarray(g), "Cells": np.asarray(c), "State": 1} for i, (g, c) in
          enumerate(zip(genes, cells))]
    return {"cell_gene": cg, "cnv_probabilities": ths, "cell_probabilities": [None] * len(ths), "HMM_type": hmm_type}


def test_mirror_remove_and_reassign_by_hand():
    from mirror import ops
    S = np.ones((6, 4), dtype=np.int32)
    tm = [[0.1, 0.1, 0.6, 0.1, 0.05, 0.05],     # P(normal) 0.6 > 0.5: removed, set to 3
          [0.3, 0.3, 0.2, 0.1, 0.05, 0.05],     # kept; tie between states 1 and 2 -> first, state 1
          [0.0, 0.1, 0.5, 0.4, 0.0, 0.0]]       # exactly 0.5: kept; arg-max state 3
    mc = _mcmc(tm, [[0, 1], [2, 3], [4, 5]], [[0, 1], [2, 3], [1, 2]])
    assert br.remove_cnv(np.array(tm), 3, 0.5) == [0]
    assert br.reassign_cnv(np.array(tm)) == [3, 1, 3]
    mc2, S2 = ops.removeCNV(mc, S, 0.5)
    assert len(mc2["cell_gene"]) == 2 and mc2["cell_gene"][0]["cnv_regions"] == "r1"
    assert (S2[np.ix_([0, 1], [0, 1])] == 3).all() and S2.sum() == S.sum() + 2 * 4
    mc3, S3 = ops.reassignCNV(mc2, S2)
    assert [c["State"] for c in mc3["cell_gene"]] == [1, 3]
    assert (S3[np.ix_([4, 5], [1, 2])] == 3).all() and (S3[np.ix_([2, 3], [2, 3])] == 1).all()
    # i3: the normal state is 2
    mc_i3 = _mcmc([[0.2, 0.7, 0.1]], [[0]], [[0, 1]], "i3")
    _, S4 = ops.removeCNV(mc_i3, np.ones((2, 2), dtype=np.int32), 0.5)
    assert (S4[0] == 2).all() and (S4[1] == 1).all()


def _read_table(path):
    with open(path) as f:
        head = f.readline().rstrip("\n").split("\t")
        return [dict(zip(head, line.rstrip("\n").split("\t"))) for line in f]


def get_genes_cells(gene_names, cell_names, pred_cnv_genes, cell_groupings):
    """initializeObject + getGenesCells (R/inferCNV_BayesNet.R:245-339) restated on the two written step-17 files."""
    regions = list(dict.fromkeys(r["gene_region_name"] for r in pred_cnv_genes))      # unique(), file order
    out = []
    for name in regions:
        cur = [r for r in pred_cnv_genes if r["gene_region_name"] == name]
        genes = {r["gene"] for r in cur}
        groups = {r["cell_group_name"] for r in cur}
        cells = {r["cell"] for r in cell_groupings if r["cell_group_name"] in groups}
        out.append({"cnv_regions": name, "Genes": [i for i, g in enumerate(gene_names) if g in genes],
                    "Cells": [j for j, c in enumerate(cell_names) if c in cells],
                    "State": sorted({int(r["state"]) for r in cur})})
    return out


@pytest.mark.parametrize("hmm_type", ["i6", "i3"])
def test_cell_gene_from_regions_matches_r_reading_the_written_reports(tmp_path, monkeypatch, hmm_type):
    """The mirror's @cell_gene equals R's getGenesCells on the files generate_cnv_region_reports writes with
    ignore_neutral_state (neutral regions dropped, genes and cells in ascending matrix order)."""
    from mirror import ops
    neutral = 3 if hmm_type == "i6" else 2
    G, C = 30, 12
    gene_names = [f"g{i}" for i in range(G)]
    cell_names = [f"cell_{(7 * j) % C}" for j in range(C)]          # names not in column order
    # two subclusters, their cells listed out of column order; regions numbered across groups as the report does
    report = [
        {"cell_group_name": "tumor.s1", "cells": [cell_names[j] for j in (9, 2, 5, 0)],
         "cnv_ranges": {"cnv_name": ["1-region_1", "1-region_2", "2-region_3"], "state": np.array([1, neutral, 4]),
                        "chr": ["1", "1", "2"], "start": np.array([1, 50, 200]), "end": np.array([40, 90, 260])},
         "gene_regions": {"first_gene": np.array([0, 5, 15]), "last_gene": np.array([4, 9, 22])}},
        {"cell_group_name": "tumor.s2", "cells": [cell_names[j] for j in (11, 3, 7)],
         "cnv_ranges": {"cnv_name": ["1-region_4", "2-region_5"], "state": np.array([neutral, 1]),
                        "chr": ["1", "2"], "start": np.array([1, 200]), "end": np.array([90, 300])},
         "gene_regions": {"first_gene": np.array([0, 15]), "last_gene": np.array([9, 29])}},
    ]
    monkeypatch.setattr(ops, "get_predicted_CNV_regions", lambda obj, by="consensus": report)
    codes = np.repeat([1, 2], [15, 15]).astype(np.int32)
    obj = ops.Infercnv(expr_data=np.ones((G, C)), gene_order_chr=codes, gene_names=gene_names, cell_names=cell_names,
                       gene_order_start=np.arange(G) * 10.0 + 1, gene_order_stop=np.arange(G) * 10.0 + 9)
    ops.generate_cnv_region_reports(obj, "17_HMM_pred.subcluster", str(tmp_path), ignore_neutral_state=neutral,
                                    by="subcluster")
    want = get_genes_cells(gene_names, cell_names,
                           _read_table(os.path.join(str(tmp_path), "17_HMM_pred.subcluster.pred_cnv_genes.dat")),
                           _read_table(os.path.join(str(tmp_path), "17_HMM_pred.subcluster.cell_groupings")))
    got = ops.cell_gene_from_regions(report, cell_names, hmm_type)
    assert [g["cnv_regions"] for g in got] == [w["cnv_regions"] for w in want]
    assert len(got) == 3 and all(g["State"] != neutral for g in got)
    for g, w in zip(got, want):
        assert g["Genes"].tolist() == w["Genes"] and g["Cells"].tolist() == w["Cells"] and [g["State"]] == w["State"]
    assert got[0]["Cells"].tolist() == sorted(got[0]["Cells"].tolist())
