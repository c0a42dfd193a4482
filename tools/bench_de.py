#!/usr/bin/env python
"""Time K14, the masking of non-DE genes (icnv_de.cu; mask_non_DE_genes_basic, run() step 21), on the GPU (DESIGN
section 3, K14).

    python tools/bench_de.py [--genes 10000] [--cells 100000] [--tests wilcoxon,t] [--reps 2] [--no-host] [--json out.json]

Workload: c4's shape - Engine.synth's depth-normalised expression (G genes x C cells), bench.ref_groups_global's two
reference groups (6 % / 4 % of the cells) and bench.subclusters_global's 50-500-cell subclusters of the four observation
groups, every subcluster tested against both reference groups, p < 0.05, "any".  Per test:
  * the call on device memory (icnv_dev_mask_non_de_f64), host clock around it, warm, best of --reps, with the CUDA-event
    stage times (a) gather, (b) reference sorts / group statistics, (c) pair tests, (d) BH, (e) mask from
    icnv_debug_mask_non_de;
  * the call through the host ABI (icnv_mask_non_de_f64) from pageable NumPy memory, as an R matrix arrives;
  * a CPU stand-in: scipy's mannwhitneyu / ttest_ind on one pair over all genes on one core, scaled to every pair.
    "scipy on one pair, scaled; not R" - R was not measured.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genes", type=int, default=10000)
    ap.add_argument("--cells", type=int, default=100000)
    ap.add_argument("--tests", default="wilcoxon,t")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--no-host", action="store_true")
    ap.add_argument("--json")
    args = ap.parse_args()

    import torch
    import bench
    from infercnv_b200 import api
    from infercnv_b200.device import Engine
    from tools.bench_random_trees import card

    G, C = args.genes, args.cells
    eng = Engine(0)
    cs, cl = bench.chr_layout(G)
    X = eng.synth(G, cs, cl, np.arange(C), C, 1234)
    refs = bench.ref_groups_global(C)
    subs = bench.subclusters_global(C, 1234)
    n_pairs = len(subs) * len(refs)
    out = {"card": card(), "genes": G, "cells": C, "subclusters": len(subs), "pairs": n_pairs, "results": {}}
    print(json.dumps({k: out[k] for k in ("card", "genes", "cells", "subclusters", "pairs")}), flush=True)
    Xh = np.asfortranarray(X.cpu().numpy().T) if not args.no_host else None
    for test in args.tests.split(","):
        r = {}
        Y = torch.empty_like(X)
        eng.mask_non_de(X, refs, subs, test=test, center_val=0.0, seed=1, out=Y)     # warm
        torch.cuda.synchronize()
        best = None
        for _ in range(args.reps):
            t0 = time.perf_counter()
            eng.mask_non_de(X, refs, subs, test=test, center_val=0.0, seed=1, out=Y)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if best is None or dt < best:
                best, stages = dt, api.mask_non_de_stats()
        r["device_s"] = best
        r["stages"] = stages
        if Xh is not None:
            t0 = time.perf_counter()
            api.mask_non_de_genes(Xh, refs, subs, test=test, center_val=0.0, seed=1)
            r["host_abi_pageable_s"] = time.perf_counter() - t0
        from scipy import stats
        xs = X[refs[0]].cpu().numpy()
        ys = X[subs[0]].cpu().numpy()
        t0 = time.perf_counter()
        for g in range(G):
            if test == "wilcoxon":
                stats.mannwhitneyu(xs[:, g], ys[:, g], alternative="two-sided")
            else:
                stats.ttest_ind(xs[:, g], ys[:, g], equal_var=False)
        one = time.perf_counter() - t0
        r["cpu_standin_s"] = one * n_pairs
        r["cpu_standin_label"] = "scipy on one pair, scaled; not R"
        out["results"][test] = r
        print(json.dumps({test: r}), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
