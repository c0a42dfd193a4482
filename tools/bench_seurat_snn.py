#!/usr/bin/env python
"""Benchmark of K18, the SNN graph of the Leiden PCA route (api.seurat_snn / Engine.seurat_snn), on planted-clone data:

  1. one group of 100 000 cells x 10 000 genes through the host ABI from pageable memory;
  2. 8 groups x 5 000 cells x 10 000 genes (K17's shape), one host call per group;
  3. the per-chromosome PCA route: 22 gene ranges of a resident 100 000 x 10 000 (cells, genes) tensor, Engine.seurat_snn
     on each view.

Per shape: wall time, the device ms of every stage (icnv_debug_seurat_snn) and the Gram matrix's FP64 rate (the DMMA work
the tile schedule executes, over the Gram stage's device time) against the data sheet's 67 TFLOP/s FP64 tensor-core figure
of the H100 SXM.  --cpu adds a labelled CPU stand-in at 5 000 cells (NumPy eigh of the Gram matrix + scipy cKDTree); it is
not Seurat.  The GPU's name and power limit are read in the same run and printed with the numbers.

    python tools/bench_seurat_snn.py [--shapes 1,2,3] [--cpu] [--out /tmp/bench_seurat_snn.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from infercnv_b200 import api  # noqa: E402

FP64_TC_PEAK = 67e12
GT = 64   # the Gram tile of icnv_snn.cu


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        return f"unknown ({e})"


def planted_cells_by_genes(n, G, clones=6, seed=0):
    """(n, G) float64 torch tensor on the GPU: planted CNV clones, positive values."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.rand(G, generator=g, device="cuda", dtype=torch.float64) * 3 + 0.5
    lab = torch.randint(0, clones, (n,), generator=g, device="cuda")
    cnv = torch.ones(clones, G, device="cuda", dtype=torch.float64)
    rng = np.random.default_rng(seed)
    for c in range(clones):
        for _ in range(4):
            a = int(rng.integers(0, G - G // 10))
            cnv[c, a:a + G // 10] = float(rng.choice([0.5, 1.5, 2.0]))
    noise = torch.randn(n, G, generator=g, device="cuda", dtype=torch.float64).mul_(0.3).exp_()
    return noise.mul_(base).mul_(cnv[lab])


def gram_flop(F, n):
    T = (F + GT - 1) // GT
    return T * (T + 1) // 2 * GT * GT * 2 * n


def record(tag, wall, st, n):
    ms = st["ms"]
    fl = gram_flop(st["F"], n)
    rate = fl / (ms["gram"] * 1e-3) if ms["gram"] > 0 else float("nan")
    return {"shape": tag, "wall_s": wall, "F": st["F"], "iterations": st["iterations"], "residual": st["residual"],
            "hub_rows": st["hub_rows"], "stage_ms": ms, "gram_flop": fl, "gram_tflops": rate / 1e12,
            "gram_share_of_67tf": rate / FP64_TC_PEAK}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1,2,3")
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from infercnv_b200.device import Engine
    api.init(0)
    res = {"gpu": gpu_info(), "runs": []}
    shapes = {int(s) for s in a.shapes.split(",")}
    G = 10000
    if 1 in shapes:
        X = planted_cells_by_genes(100000, G, seed=1).cpu().numpy().T       # genes x cells, Fortran order, pageable
        api.seurat_snn(X[:, :5000], k=20)                                    # warm-up
        for rep in range(2):
            t = time.perf_counter()
            r = api.seurat_snn(X, k=20)
            res["runs"].append(record(f"1: 100000 x 10000 host ABI (rep {rep})", time.perf_counter() - t, r.stats, 100000))
        del X, r
    if 2 in shapes:
        X = planted_cells_by_genes(40000, G, seed=2).cpu().numpy().T
        groups = np.arange(40000).reshape(8, 5000)
        api.seurat_snn(X, k=20, cells=groups[0])
        t = time.perf_counter()
        per = []
        for g in groups:
            r = api.seurat_snn(X, k=20, cells=g)
            per.append(record("2: one group of 5000", 0.0, r.stats, 5000))
        wall = time.perf_counter() - t
        res["runs"].append({"shape": "2: 8 groups x 5000 x 10000 host ABI", "wall_s": wall,
                            "stage_ms_sum": {s: sum(p["stage_ms"][s] for p in per) for s in api.SNN_STAGES},
                            "iterations": [p["iterations"] for p in per], "F": [p["F"] for p in per]})
        del X
    if 3 in shapes:
        eng = Engine(0)
        T = planted_cells_by_genes(100000, G, seed=3)                       # resident (cells, genes)
        bounds = np.linspace(0, G, 23).astype(int)
        eng.seurat_snn(T[:, bounds[0]:bounds[1]], 20)
        torch.cuda.synchronize()
        t = time.perf_counter()
        per = []
        for c in range(22):
            r = eng.seurat_snn(T[:, bounds[c]:bounds[c + 1]], 20)
            per.append(record(f"3: chr {c}", 0.0, r.stats, 100000))
        torch.cuda.synchronize()
        wall = time.perf_counter() - t
        res["runs"].append({"shape": "3: 22 gene ranges of a resident 100000 x 10000", "wall_s": wall,
                            "stage_ms_sum": {s: sum(p["stage_ms"][s] for p in per) for s in api.SNN_STAGES},
                            "iterations": [p["iterations"] for p in per], "F": [p["F"] for p in per]})
        del T
    if a.cpu:
        from scipy.spatial import cKDTree
        X = planted_cells_by_genes(5000, G, seed=2).cpu().numpy().T
        r = api.seurat_snn(X, k=20)
        feats = np.sort(r.features)
        mu, sd = X[feats].mean(axis=1), X[feats].std(axis=1, ddof=1)
        t = time.perf_counter()
        Z = np.minimum((X[feats] - mu[:, None]) / sd[:, None], 10.0)
        lam, U = np.linalg.eigh(Z @ Z.T)
        E = Z.T @ U[:, ::-1][:, :10]
        cKDTree(E).query(E, k=20)
        res["runs"].append({"shape": "CPU stand-in (NumPy eigh + cKDTree, not Seurat): 5000 x 2000 features",
                            "wall_s": time.perf_counter() - t, "cpu_threads": os.cpu_count()})
    for run in res["runs"]:
        print(json.dumps(run))
    print(json.dumps({"gpu": res["gpu"]}))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
