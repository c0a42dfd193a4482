#!/usr/bin/env python
"""Time K12, the exact k-nearest-neighbour kernel (icnv_dist.cu; nn2() of the per-chromosome Leiden subclustering), on the
GPU, next to K10 on the same cells (DESIGN section 3, K12).

    python tools/bench_knn.py [--sizes 10000,30000,100000] [--genes 455] [--k 20] [--reps 3] [--ckdtree-max 10000]
                              [--chr-pass 100000x22] [--wide 10000x10000] [--json out.json]

Workloads: seeded normal cells (torch's CUDA generator) at each of --sizes x --genes (455 genes = one average chromosome of
c3's 10 000); the whole per-chromosome pass at c3 scale (--chr-pass: cells x chromosomes of --genes each, one device call
per gene-range view of the resident matrix, as Engine.knn makes it); and --wide (cells x genes, one call).  Per workload:
  * K12 on device memory (icnv_dev_knn_f64: partial + merge kernels, and the one synchronise that reports non-finite
    input), CUDA events, warm (one untimed call first), best of --reps;
  * K10 (icnv_dev_pairwise_dist_f64) on the same cells, the same way;
  * the host ABI (icnv_knn_rows_f64) from pageable memory, host clock (it ends in a synchronise);
  * scipy's cKDTree(x).query(x, k, workers=1) for n <= --ckdtree-max: a CPU stand-in for RANN's kd-tree, not RANN.
Rates: K12 computes all n^2 ordered pairs, K10 the n (n + 1) / 2 of the upper triangle's tiles (counted as n^2 / 2);
pair-genes / s over those; FP64-pipe fraction as in DESIGN K10: 2 FP64 instructions per pair-gene against 64 lanes per
clock per SM at the card's maximum SM clock (an upper bound on the pipe's rate, so the fraction is a lower bound).
The card's name, power limit and clocks are read in the same run.
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


def card() -> dict:
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, mx, cur = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit_W": float(pl), "max_sm_MHz": float(mx), "sm_MHz_now": float(cur)}
    except (OSError, subprocess.SubprocessError, ValueError, IndexError) as e:
        return {"name": f"unknown ({e})"}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000,30000,100000")
    ap.add_argument("--genes", type=int, default=455)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ckdtree-max", type=int, default=10000)
    ap.add_argument("--chr-pass", default="100000x22")
    ap.add_argument("--wide", default="10000x10000")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch

    from infercnv_b200 import _lib, api
    from infercnv_b200.device import _stream_ptr
    api.init(0)
    lib = _lib.load()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    info = card()
    print(f"card: {info}, {sms} SMs", flush=True)
    st = _stream_ptr()
    k = a.k

    def best(fn):
        fn()
        torch.cuda.synchronize()
        times = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3)
        return min(times)

    def pipe_frac(pair_genes_per_s):
        mhz = info.get("max_sm_MHz")
        return None if not mhz else 2.0 * pair_genes_per_s / (64.0 * sms * mhz * 1e6)

    def cells(n, G, seed):
        g = torch.Generator(device="cuda:0")
        g.manual_seed(seed)
        return torch.randn((n, G), generator=g, dtype=torch.float64, device="cuda:0")   # cells x genes, row-major

    rows = []
    workloads = [(int(s), a.genes, 1) for s in a.sizes.split(",") if s]
    if a.wide:
        n, G = (int(v) for v in a.wide.split("x"))
        workloads.append((n, G, 1))
    if a.chr_pass:
        n, K = (int(v) for v in a.chr_pass.split("x"))
        workloads.append((n, a.genes, K))
    for n, G, K in workloads:
        X = cells(n, G * K, n + G + K)
        idx = torch.empty((k, n), dtype=torch.int32, device="cuda:0")
        dist = torch.empty((k, n), dtype=torch.float64, device="cuda:0")
        ld = X.stride(0)

        def knn_all():
            for c in range(K):
                _lib.check(lib.icnv_dev_knn_f64(X.data_ptr() + 8 * c * G, G, ld, None, n, k, idx.data_ptr(),
                                                dist.data_ptr(), st))

        t12 = best(knn_all)
        pg12 = float(n) * n * G * K
        row = {"n": n, "G": G, "chromosomes": K, "k": k, "knn_s": t12, "knn_pair_genes_per_s": pg12 / t12,
               "knn_fp64_pipe_frac": pipe_frac(pg12 / t12)}
        if n <= 65535 * 128 and n * (n - 1) // 2 * 8 <= 45e9:
            D = torch.empty(n * (n - 1) // 2, dtype=torch.float64, device="cuda:0")

            def k10_all():
                for c in range(K):
                    _lib.check(lib.icnv_dev_pairwise_dist_f64(X.data_ptr() + 8 * c * G, G, ld, None, n, D.data_ptr(), st))

            t10 = best(k10_all)
            pg10 = float(n) * n * G * K / 2
            row.update({"k10_s": t10, "k10_pair_genes_per_s": pg10 / t10, "k10_fp64_pipe_frac": pipe_frac(pg10 / t10),
                        "knn_over_k10": t12 / t10})
            del D
            torch.cuda.empty_cache()
        if K == 1:
            x = np.ascontiguousarray(X.cpu().numpy())
            xf = np.asfortranarray(x)                          # observations x variables, as nn2() receives it
            t0 = time.perf_counter()
            hi, hd = api.knn_rows(xf, k)
            row["host_abi_s"] = time.perf_counter() - t0
            torch.cuda.synchronize()
            assert np.array_equal(hi, idx.T.cpu().numpy()), "host ABI and device entry differ"
            if n <= a.ckdtree_max and G <= 1000:
                from scipy.spatial import cKDTree
                t0 = time.perf_counter()
                td, ti = cKDTree(x).query(x, k=k, eps=0, workers=1)
                row["ckdtree_1core_s"] = time.perf_counter() - t0
                row["ckdtree_dist_max_rel"] = float(np.max(np.abs(td - hd) / np.maximum(td, 1e-300)))
            del x, xf
        del X
        torch.cuda.empty_cache()
        print(json.dumps(row), flush=True)
        rows.append(row)
    info_after = card()
    print(f"card after: {info_after}", flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        json.dump({"card": info, "card_after": info_after, "sms": sms, "rows": rows}, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
