#!/usr/bin/env python
"""Time K19, the packed-triangle hclust() linkage, against K11 on the GPU (DESIGN section 3, K19).

    python tools/bench_hclust_tri.py [--sizes 10000,30000,65536] [--big 100000] [--genes 10000] [--reps 1] [--json out.json]

Cells are seeded synthetic blobs (16 blobs in 64 genes, as tools/bench_hclust.py draws them) -> Engine.pairwise_dist ->
the device "dist" vector.  For each n of --sizes, ward.D2:
  * K11 alone (icnv_dev_hclust_f64: fill + mirror + NN-chain kernel) and K19 alone (icnv_dev_hclust_tri_f64: prepare +
    NN-chain kernel), CUDA events on the library's stream, best of --reps, the two trees compared bit for bit;
  * per-row cost = linkage time / n, and the K19 / K11 ratio.
At --big (past K11's 65 536 limit) K19 through Engine.cluster_cells on resident 64-gene cells (the device vector and K19's
own triangle would not both fit; the distances add a few per cent), then icnv_cluster_cells_f64 end to end from a pageable
--genes x --big host matrix (upload, distances into the triangle, linkage, order), host clock.  Both kernels are warmed
once at 2 000 cells first (module load).  The card's name, power limit and maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def cells(n: int, G: int = 64, seed: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    centres = rng.normal(scale=3.0, size=(16, G))
    return centres[rng.integers(0, 16, size=n)] + rng.normal(size=(n, G))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000,30000,65536")
    ap.add_argument("--big", type=int, default=100000)
    ap.add_argument("--genes", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch

    from infercnv_b200 import _lib, api
    from infercnv_b200.device import Engine, _stream_ptr
    api.init(0)
    eng = Engine(0)
    lib = _lib.load()
    print(f"card: {card()}", flush=True)

    def timed(fn, D, n, reps):
        merge = torch.empty(2 * (n - 1), dtype=torch.int32, device="cuda:0")
        height = torch.empty(n - 1, dtype=torch.float64, device="cuda:0")
        st = _stream_ptr()   # torch's stream, so the events bracket the library's launches
        best = None
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(fn(D.data_ptr(), n, 7, merge.data_ptr(), height.data_ptr(), st))
            e1.record()
            torch.cuda.synchronize()
            t = e0.elapsed_time(e1) / 1e3
            best = t if best is None else min(best, t)
        return best, merge.cpu().numpy(), height.cpu().numpy()

    D = eng.pairwise_dist(torch.as_tensor(cells(2000), device="cuda:0"))
    timed(lib.icnv_dev_hclust_f64, D, 2000, 1)
    timed(lib.icnv_dev_hclust_tri_f64, D, 2000, 1)
    del D
    rows = []
    for n in (int(s) for s in a.sizes.split(",") if s):
        D = eng.pairwise_dist(torch.as_tensor(cells(n), device="cuda:0"))
        torch.cuda.synchronize()
        t_sq, m_sq, h_sq = timed(lib.icnv_dev_hclust_f64, D, n, a.reps)
        t_tri, m_tri, h_tri = timed(lib.icnv_dev_hclust_tri_f64, D, n, a.reps)
        del D
        torch.cuda.empty_cache()
        same = bool(np.array_equal(m_sq, m_tri) and h_sq.tobytes() == h_tri.tobytes())
        row = {"n": n, "k11_s": t_sq, "k19_s": t_tri, "k19_over_k11": t_tri / t_sq, "k11_us_per_row": 1e6 * t_sq / n,
               "k19_us_per_row": 1e6 * t_tri / n, "k11_matrix_GB": n * (n + (n & 1)) * 8 / 1e9,
               "k19_triangle_GB": n * (n - 1) * 4 / 1e9, "bit_identical": same}
        print(json.dumps(row), flush=True)
        rows.append(row)
    if a.big:
        n = a.big
        # the device vector and K19's own triangle would not both fit: the cells stay resident and Engine.cluster_cells
        # writes the 64-gene distances straight into the triangle (host clock; the call ends in a synchronise)
        Xd = torch.as_tensor(cells(n), device="cuda:0")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.cluster_cells(Xd, None, "ward.D2")
        t_tri = time.perf_counter() - t0
        del Xd
        torch.cuda.empty_cache()
        row = {"n": n, "genes": 64, "k19_with_distances_s": t_tri, "k19_us_per_row": 1e6 * t_tri / n,
               "k19_triangle_GB": n * (n - 1) * 4 / 1e9}
        print(json.dumps(row), flush=True)
        rows.append(row)
        X = np.asfortranarray(cells(n, a.genes, seed=1).T)   # genes x cells, pageable
        t0 = time.perf_counter()
        merge, height, order = api.cluster_cells(X, method="ward.D2")
        t_e2e = time.perf_counter() - t0
        row = {"n": n, "genes": a.genes, "cluster_cells_host_s": t_e2e, "upload_GB": X.nbytes / 1e9,
               "dist_TFLOP": 2.0 * a.genes * n * (n - 1) / 2 / 1e12, "valid_order": bool(np.array_equal(np.sort(order), np.arange(1, n + 1)))}
        print(json.dumps(row), flush=True)
        rows.append(row)
    out = {"card": card(), "rows": rows}
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        json.dump(out, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
