#!/usr/bin/env python
"""Time K15, the Bayesian network filter (icnv_bayes.cu; inferCNVBayesNet's Gibbs sampling, run() step 18), on the GPU
(DESIGN section 3, K15).

    python tools/bench_bayesnet.py [--genes 10000] [--cells 100000] [--cases A,B] [--reps 2] [--no-host] [--json out.json]

Workload: Engine.synth's G genes x C cells, mapped to log2(x + 1) / 4 + 0.6 so the values sit around the i6 states' means,
bench.chr_layout's chromosomes, i6 defaults (6 chains, 700 discarded + 1000 kept sweeps, m = 6):
  (A) 50 subclusters of C / 50 cells, each chromosome split into 3 regions: 3 300 regions at the default shape;
  (B) analysis_mode = "samples": one group of all C cells, each chromosome split into 3 regions - 66 regions of C cells,
      396 chains, each one CTA walking C cells per sweep (the one-CTA-per-chain design at its worst).
Per case:
  * the call on device memory (icnv_dev_bayesnet_f64 through Engine.bayesnet), host clock around it, warm, best of --reps,
    with the CUDA-event times of (a) the log-likelihood pass and (b) the sampler from icnv_debug_bayesnet, and two host-side
    parts of it timed apart: building the region lists and copying a tensor the size of the theta draws to the host;
  * the call through the host ABI (icnv_bayesnet_f64) from pageable NumPy memory, as an R matrix arrives;
  * a CPU stand-in: tests/bayesnet_reference.gibbs (NumPy, one core), one chain of the case's first region, scaled to
    6 chains of every region - "NumPy Gibbs, scaled; not JAGS".  JAGS was not measured.
The card's name, power limit and maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MU = np.array([0.4, 0.7, 1.0, 1.3, 1.6, 1.9])
TAU = np.array([30.0, 40.0, 60.0, 40.0, 30.0, 20.0])


def regions(cs, cl, groups):
    genes, cells = [], []
    for g in groups:
        for s, n in zip(cs, cl):
            b = np.linspace(s, s + n, 4).astype(int)
            for q in range(3):
                genes.append(np.arange(b[q], b[q + 1], dtype=np.int32))
                cells.append(g)
    return genes, cells


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genes", type=int, default=10000)
    ap.add_argument("--cells", type=int, default=100000)
    ap.add_argument("--cases", default="A,B")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--no-host", action="store_true")
    ap.add_argument("--json")
    args = ap.parse_args()

    import torch
    import bench
    from infercnv_b200 import api
    from infercnv_b200.device import Engine
    from tests import bayesnet_reference as br
    from tools.bench_random_trees import card

    G, C = args.genes, args.cells
    eng = Engine(0)
    cs, cl = bench.chr_layout(G)
    X = eng.synth(G, cs, cl, np.arange(C), C, 1234)
    X = torch.log2(X + 1.0) * 0.25 + 0.6
    torch.cuda.synchronize()
    out = {"card": card(), "genes": G, "cells": C, "results": {}}
    print(json.dumps({k: out[k] for k in ("card", "genes", "cells")}), flush=True)
    Xh = np.asfortranarray(X.cpu().numpy().T) if not args.no_host else None
    for case in args.cases.split(","):
        if case == "A":
            per = C // 50
            groups = [np.arange(s * per, (s + 1) * per, dtype=np.int32) for s in range(50)]
        else:
            groups = [np.arange(C, dtype=np.int32)]
        genes, cells = regions(cs, cl, groups)
        r = {"regions": len(genes), "cells_per_region": len(cells[0])}
        best = None
        for _ in range(args.reps + 1):           # the first call warms up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.bayesnet(X, genes, cells, MU, TAU, 6, seed=1)
            t = time.perf_counter() - t0
            st = api.bayesnet_stats()
            if best is None or t < best[0]:
                best = (t, st)
        r["device_call_s"] = best[0]
        r["loglik_ms"] = best[1]["loglik_ms"]
        r["sampler_ms"] = best[1]["sampler_ms"]
        r["ctas"] = best[1]["ctas"]
        # the host side of the device call, timed apart: the region lists as CSR, and the copy of the theta draws to the host
        t0 = time.perf_counter()
        api._bayesnet_args(genes, cells, MU, TAU, None)
        r["region_lists_s"] = time.perf_counter() - t0
        th = torch.empty(len(genes) * 6 * 1000 * 6, dtype=torch.float64, device=X.device)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        th.cpu()
        r["theta_to_host_s"] = time.perf_counter() - t0
        del th
        if Xh is not None:
            t0 = time.perf_counter()
            api.bayesnet(Xh, genes, cells, MU, TAU, 6, seed=1)
            r["host_abi_pageable_s"] = time.perf_counter() - t0
        rng = np.random.default_rng(0)
        L = br.loglik(Xh if Xh is not None else X.cpu().numpy().T, genes[0], cells[0], MU, TAU)
        t0 = time.perf_counter()
        br.gibbs(L, 1, 700, 1000, rng)
        r["numpy_gibbs_scaled_s"] = (time.perf_counter() - t0) * 6 * len(genes)
        r["numpy_note"] = "NumPy Gibbs, one chain of one region on one core, scaled to 6 chains of every region; not JAGS"
        out["results"][case] = r
        print(json.dumps({case: r}), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
