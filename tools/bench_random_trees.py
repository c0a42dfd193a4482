#!/usr/bin/env python
"""Time K13b, the random-trees permutation null (icnv_random_trees.cu; .parameterize_random_cluster_heights_smoothed_trees
of random-trees subclustering), on the GPU (DESIGN section 3, K13).

    python tools/bench_random_trees.py [--sizes 500,2000,5000] [--genes 10000] [--n-perm 100] [--reps 2]
                                       [--cpu-perms 2] [--cpu-max 2000] [--json out.json]

Workload: a seeded genes x cells clade (torch's CUDA generator, normal values, the first half of the cells with a +1
offset on a third of the genes: two planted clades), ward.D2, window 101, n_perm permutations - one clade call each.
Per size:
  * the call on device memory (icnv_dev_random_tree_heights_f64), host clock around it (it ends in a synchronise), warm
    (one untimed call first), best of --reps; B and the waves, and the device time of its stages (shuffle + runmean +
    centring, distances, linkages) from icnv_debug_random_trees;
  * one stand-alone linkage of the same n (icnv_dev_hclust_f64 on the observed distances): a linkage stage close to it
    means the B chains of a wave ran side by side;
  * K10 stand-alone (icnv_dev_pairwise_dist_f64) on the clade, pair-genes / s, against the rate inside the call
    ((n_perm + 1) n^2 / 2 G pair-genes over the distance stage);
  * a CPU stand-in for one permutation - NumPy runmean (cumulative sums) + median centring + scipy pdist + linkage on one
    core, --cpu-perms of them, scaled linearly to n_perm + 1 trees.  Not R: R was not measured.
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


def cpu_tree_max(Xc, window, rng):
    """One permuted tree on the CPU: shuffle each gene, runmean (cumulative sums), median centring, pdist, ward.D2."""
    from scipy.cluster.hierarchy import linkage
    from scipy.spatial.distance import pdist
    G, n = Xc.shape
    P = np.take_along_axis(Xc, np.argsort(rng.random((G, n)), axis=1), axis=1)
    k = min(window, G)
    k2 = k // 2
    k1 = k - 1 - k2
    cs = np.vstack([np.zeros((1, n)), np.cumsum(P, axis=0)])
    p = np.arange(G)
    a, b = np.maximum(0, p - k1), np.minimum(G - 1, p + k2)
    sm = (cs[b + 1] - cs[a]) / (b - a + 1)[:, None]
    sm -= np.median(sm, axis=0)
    return linkage(pdist(sm.T), "ward")[:, 2].max()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="500,2000,5000")
    ap.add_argument("--genes", type=int, default=10000)
    ap.add_argument("--n-perm", type=int, default=100)
    ap.add_argument("--window", type=int, default=101)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--cpu-perms", type=int, default=2)
    ap.add_argument("--cpu-max", type=int, default=2000)
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
    G, NP = a.genes, a.n_perm

    def events(fn, reps):
        fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / 1e3)
        return min(ts)

    rows = []
    for n in (int(s) for s in a.sizes.split(",") if s):
        g = torch.Generator(device="cuda:0")
        g.manual_seed(n)
        X = torch.randn((n, G), generator=g, dtype=torch.float64, device="cuda:0")   # cells x genes: column-major G x n
        X[: n // 2, : G // 3] += 1.0
        nm = n - 1
        merge = torch.empty(2 * nm, dtype=torch.int32, device="cuda:0")
        height = torch.empty(nm, dtype=torch.float64, device="cuda:0")
        pm = torch.empty(max(NP, 1), dtype=torch.float64, device="cuda:0")

        def call():
            _lib.check(lib.icnv_dev_random_tree_heights_f64(X.data_ptr(), G, G, None, n, a.window, 7, NP, 12345,
                                                            merge.data_ptr(), height.data_ptr(), pm.data_ptr(), st))

        call()
        torch.cuda.synchronize()
        walls = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            call()
            torch.cuda.synchronize()
            walls.append(time.perf_counter() - t0)
        stats = api.random_trees_stats()
        # stand-alone pieces on the same clade
        D = torch.empty(n * (n - 1) // 2, dtype=torch.float64, device="cuda:0")
        t_dist = events(lambda: _lib.check(lib.icnv_dev_pairwise_dist_f64(X.data_ptr(), G, G, None, n, D.data_ptr(), st)),
                        a.reps)
        m1 = torch.empty(2 * nm, dtype=torch.int32, device="cuda:0")
        h1 = torch.empty(nm, dtype=torch.float64, device="cuda:0")
        t_link1 = events(lambda: _lib.check(lib.icnv_dev_hclust_f64(D.data_ptr(), n, 7, m1.data_ptr(), h1.data_ptr(), st)),
                         a.reps)
        pg = n * n / 2.0 * G
        row = {"n": n, "G": G, "n_perm": NP, "wall_s": min(walls), "B": stats["B"], "waves": stats["waves"],
               "prep_s": stats["prep_ms"] / 1e3, "dist_s": stats["dist_ms"] / 1e3, "link_s": stats["link_ms"] / 1e3,
               "one_linkage_s": t_link1, "k10_alone_pair_genes_per_s": pg / t_dist,
               "k10_in_call_pair_genes_per_s": (NP + 1) * pg / (stats["dist_ms"] / 1e3)}
        if n <= a.cpu_max and a.cpu_perms > 0:
            Xc = X.T.cpu().numpy()
            rng = np.random.default_rng(0)
            t0 = time.perf_counter()
            for _ in range(a.cpu_perms):
                cpu_tree_max(Xc, a.window, rng)
            row["cpu_standin_s_scaled"] = (time.perf_counter() - t0) / a.cpu_perms * (NP + 1)
        rows.append(row)
        print(json.dumps(row), flush=True)
        del X, D, merge, height, pm, m1, h1
        torch.cuda.empty_cache()

    print(f"\n{info.get('name')}, power limit {info.get('power_limit_W')} W, max SM clock {info.get('max_sm_MHz')} MHz, "
          f"ward.D2, window {a.window}, {NP} permutations")
    print("| n | G | call | shuffle+runmean+centre | distances | linkages | one linkage | B x waves | K10 in call / alone "
          "(pair-genes/s) | CPU stand-in, scaled |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        cpu = f"{r['cpu_standin_s_scaled']:.1f} s" if "cpu_standin_s_scaled" in r else "not run"
        print(f"| {r['n']} | {r['G']} | {r['wall_s']:.3f} s | {r['prep_s']:.3f} s | {r['dist_s']:.3f} s | {r['link_s']:.3f} s "
              f"| {r['one_linkage_s'] * 1e3:.1f} ms | {r['B']} x {r['waves']} | {r['k10_in_call_pair_genes_per_s']:.3g} / "
              f"{r['k10_alone_pair_genes_per_s']:.3g} | {cpu} |")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": info, "sms": sms, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
