#!/usr/bin/env python
"""Generate tests/golden/bayesnet_fixture.npz from the reference's bundled JAGS run, `data/mcmc_obj.rda`.

Run in the build container only (needs the read-only reference checkout):

    python tests/golden/make_bayesnet_golden.py [/root/reference]

The object is inferCNVBayesNet's MCMC_inferCNV after its sampling: 9 CNV regions of 10 cells each, sampled by JAGS with the
i6 model (6 chains, 1000 kept draws each).  Stored:

* mu, sig             - the six states' means and precisions (@mu, @sig) the model ran with;
* gene_off / gene_idx - @cell_gene[[r]]$Genes, 0-based rows of the 4613-gene matrix, as CSR;
* cell_off / cell_idx - @cell_gene[[r]]$Cells, 0-based columns of its 20 cells, as CSR;
* theta_mean          - 9 x 6, the posterior means of theta per region (@cnv_probabilities[[1]], stored transposed there);
* cell_prob           - 9 x 6 x 10, the per-cell state frequencies (@cell_probabilities[[r]]).

It is the reference's data reduced to arrays, not reference code.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from rda_reader import read_rda  # noqa: E402


def main(ref: str) -> None:
    m = read_rda(os.path.join(ref, "data/mcmc_obj.rda"))["mcmc_obj"]
    mu = np.asarray(m.attr["mu"].value, dtype=np.float64)
    sig = np.asarray(m.attr["sig"].value, dtype=np.float64)
    genes, cells = [], []
    for cg in m.attr["cell_gene"].value:
        fields = dict(zip(cg.attr["names"].value, cg.value))
        genes.append(np.asarray(fields["Genes"].value, dtype=np.int32) - 1)
        cells.append(np.asarray(fields["Cells"].value, dtype=np.int32) - 1)
    cp = m.attr["cnv_probabilities"].value[0]
    d = cp.attr["dim"].value                                   # 6 x 9, column-major
    theta_mean = np.asarray(cp.value, dtype=np.float64).reshape((d[1], d[0]))
    cell_prob = np.stack([np.asarray(c.value, dtype=np.float64).reshape(tuple(c.attr["dim"].value[::-1])).T
                          for c in m.attr["cell_probabilities"].value])
    np.savez_compressed(
        os.path.join(HERE, "bayesnet_fixture.npz"), mu=mu, sig=sig,
        gene_off=np.cumsum([0] + [len(g) for g in genes]).astype(np.int32), gene_idx=np.concatenate(genes),
        cell_off=np.cumsum([0] + [len(c) for c in cells]).astype(np.int32), cell_idx=np.concatenate(cells),
        theta_mean=theta_mean, cell_prob=cell_prob)
    print("bayesnet_fixture.npz:", len(genes), "regions, genes per region", [len(g) for g in genes],
          "cells per region", [len(c) for c in cells])


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
