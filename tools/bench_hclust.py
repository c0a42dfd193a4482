#!/usr/bin/env python
"""Time K11, the hclust() linkage kernel, on the GPU (DESIGN section 3, K11).

    python tools/bench_hclust.py [--sizes 2000,10000,30000,65536] [--reps 2] [--scipy-max 30000] [--json out.json]

For each n: seeded synthetic cells (16 blobs in 64 genes) -> Engine.pairwise_dist -> the device "dist" vector; then
  * linkage alone (icnv_dev_hclust_f64, ward.D2: fill + mirror + NN-chain kernel), CUDA events, warm (one untimed call
    first), best of --reps;
  * the host-ABI call (icnv_hclust_f64) from a pageable host copy of the vector, host clock (it ends in a synchronise);
  * scipy.cluster.hierarchy.linkage(method="ward") on the same vector for n <= --scipy-max: scipy's NN-chain on one CPU
    core.  This is NOT fastcluster (not installed here), only a CPU comparator.
Row scans are counted by replaying the same chain in NumPy (tests/hclust_reference.py) for n <= 10 000; bytes scanned =
scans x ld x 8 (the kernel reads whole rows), effective scan bandwidth = bytes scanned / linkage time (it includes the
updates and the fill, so it is a lower bound on the scan rate).  The card's name and power limit are read in the same run.
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
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def cells(n: int, seed: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    centres = rng.normal(scale=3.0, size=(16, 64))
    return centres[rng.integers(0, 16, size=n)] + rng.normal(size=(n, 64))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="2000,10000,30000,65536")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--scipy-max", type=int, default=30000)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch

    from infercnv_b200 import _lib, api
    from infercnv_b200.device import Engine, _stream_ptr
    api.init(0)
    eng = Engine(0)
    lib = _lib.load()
    print(f"card: {card()}", flush=True)
    rows = []
    for n in (int(s) for s in a.sizes.split(",")):
        D = eng.pairwise_dist(torch.as_tensor(cells(n), device="cuda:0"))
        nm = n - 1
        merge = torch.empty(2 * nm, dtype=torch.int32, device="cuda:0")
        height = torch.empty(nm, dtype=torch.float64, device="cuda:0")
        st = _stream_ptr()   # torch's stream, so the events bracket the library's launches

        def run():
            _lib.check(lib.icnv_dev_hclust_f64(D.data_ptr(), n, 7, merge.data_ptr(), height.data_ptr(), st))

        run()
        torch.cuda.synchronize()
        times = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3)
        t_dev = min(times)
        h_dev = height.cpu().numpy()
        d_host = D.cpu().numpy()
        del D
        torch.cuda.empty_cache()
        t0 = time.perf_counter()
        m_h, h_h, _ = api.hclust(d_host, "ward.D2")
        t_host = time.perf_counter() - t0
        assert np.array_equal(h_h.view(np.int64), h_dev.view(np.int64)), "host ABI and device entry differ"
        row = {"n": n, "linkage_s": t_dev, "host_abi_s": t_host, "matrix_GB": n * (n + (n & 1)) * 8 / 1e9}
        if n <= 10000:
            from tests import hclust_reference as hr
            scans = count_scans(hr, d_host, n)
            row["scans"] = scans
            row["GB_scanned"] = scans * (n + (n & 1)) * 8 / 1e9
            row["scan_GBps"] = row["GB_scanned"] / t_dev
        if n <= a.scipy_max:
            from scipy.cluster.hierarchy import linkage
            t0 = time.perf_counter()
            Z = linkage(d_host, "ward")
            row["scipy_1core_s"] = time.perf_counter() - t0
            row["scipy_height_max_rel"] = float(np.max(np.abs(Z[:, 2] - h_h) / np.maximum(np.abs(Z[:, 2]), 1e-300)))
        del d_host
        print(json.dumps(row), flush=True)
        rows.append(row)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        json.dump({"card": card(), "rows": rows}, open(a.json, "w"), indent=1)


def count_scans(hr, d, n) -> int:
    """Row scans of the kernel's chain = chain extensions + merges; replayed with the reference's rules (ward.D2)."""
    M = hr.square(d, n)
    M = M * M
    np.fill_diagonal(M, np.inf)
    active = np.ones(n, dtype=bool)
    size = np.ones(n)
    chain, merges, scans = [], 0, 0
    while merges < n - 1:
        if not chain:
            chain = [int(np.flatnonzero(active)[0])]
        a = chain[-1]
        p = chain[-2] if len(chain) >= 2 else -1
        row = np.where(active, M[a], np.inf)
        row[a] = np.inf
        b = int(np.argmin(row))
        scans += 1
        if p >= 0 and M[a, p] == row[b]:
            b = p
        if b != p:
            chain.append(b)
            continue
        i, j = min(a, b), max(a, b)
        k = np.flatnonzero(active)
        k = k[(k != i) & (k != j)]
        w = hr.lance_williams(7, M[i, k], M[j, k], M[a, b], size[i], size[j], size[k])
        M[j, k] = w
        M[k, j] = w
        size[j] += size[i]
        active[i] = False
        chain = chain[:-2]
        merges += 1
    return scans


if __name__ == "__main__":
    main()
