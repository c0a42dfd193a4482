#!/usr/bin/env python
"""Time K17, the subclustering trees of run() step 15 (icnv_subclusters.cu; define_signif_tumor_subclusters), on the GPU
(DESIGN section 3, K17).

    python tools/bench_subclusters.py [--genes 10000] [--shapes groups,single,leiden] [--json out.json]

Seeded genes x cells data (NumPy, normal values with a per-gene scale; the first 5 % of the genes are wider, so the z-score
filter has outliers to drop), ward.D2, three shapes of groups:
  * groups:  8 groups x 5 000 cells (cluster_by_groups with many cells per group);
  * single:  one group of 30 000 cells;
  * leiden:  40 groups of 50 .. 2 000 cells (the trees of a Leiden partition).
A reference list of 2 000 other cells feeds the filter.  Per shape:
  * the filter call (api.zscore_outlier_genes, host clock around a call that ends in a synchronise);
  * the trees call (api.cluster_groups with the filter's gene list), host clock, and its stages from CUDA events
    (api.cluster_groups_stats: the gene gather, the distances, the linkages, summed over the waves);
  * the same trees as separate host calls per group, api.pairwise_dist on the group's columns then api.hclust - the GPU
    work this step does today without R in between (the distance vector crosses PCIe twice per tree);
  * a bitwise comparison of every tree of the two sides.
Every timed call is run once untimed first.  The card's name, power limit and SM clock are read in the same run.
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


def shape_sizes(name: str, rng) -> list:
    if name == "groups":
        return [5000] * 8
    if name == "single":
        return [30000]
    if name == "leiden":
        return sorted(rng.integers(50, 2001, size=40).tolist(), reverse=True)
    raise ValueError(name)


def timed(fn):
    fn()
    t0 = time.perf_counter()
    out = fn()
    return out, time.perf_counter() - t0


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--genes", type=int, default=10000)
    ap.add_argument("--shapes", default="groups,single,leiden")
    ap.add_argument("--n-ref", type=int, default=2000)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    from infercnv_b200 import api
    api.init(0)
    info = card()
    print(f"card: {info}", flush=True)
    G = a.genes
    rows = []
    for shape in a.shapes.split(","):
        rng = np.random.default_rng(17)
        sizes = shape_sizes(shape, rng)
        C = sum(sizes) + a.n_ref
        X = rng.standard_normal((G, C)) * rng.uniform(0.5, 1.5, size=(G, 1))
        X[: G // 20] *= 4.0
        X = np.asfortranarray(X)
        perm = rng.permutation(C).astype(np.int32)
        ref = perm[:a.n_ref]
        groups, at = [], a.n_ref
        for n in sizes:
            groups.append(perm[at:at + n])
            at += n
        out, t_filter = timed(lambda: api.zscore_outlier_genes(X, ref))
        keep = np.flatnonzero(~out).astype(np.int32)
        trees, t_call = timed(lambda: api.cluster_groups(X, groups, "ward.D2", keep=keep))
        st = api.cluster_groups_stats()
        Xk = np.asfortranarray(X[keep])
        t_sep, same = 0.0, True
        for g, t in zip(groups, trees):
            Xg = np.asfortranarray(Xk[:, g])
            if g is groups[0]:
                api.hclust(api.pairwise_dist(Xg), "ward.D2")          # warm
            t0 = time.perf_counter()
            w = api.hclust(api.pairwise_dist(Xg), "ward.D2")
            t_sep += time.perf_counter() - t0
            same &= np.array_equal(t[0], w[0]) and t[1].tobytes() == w[1].tobytes() and np.array_equal(t[2], w[2])
        row = {"shape": shape, "groups": len(sizes), "cells": sum(sizes), "G": G, "G_kept": int(keep.size),
               "filter_s": t_filter, "trees_call_s": t_call, "gather_s": st["gather_ms"] / 1e3, "dist_s": st["dist_ms"] / 1e3,
               "link_s": st["link_ms"] / 1e3, "waves": st["waves"], "widest_wave": st["widest"], "per_group_calls_s": t_sep,
               "bitwise_equal": bool(same)}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del X, Xk
    print(f"\n{info.get('name')}, power limit {info.get('power_limit_W')} W, SM clock {info.get('sm_MHz_now')} MHz now "
          f"(max {info.get('max_sm_MHz')}), ward.D2, {G} genes")
    print("| shape | groups x cells | filter | trees call | gather / distances / linkages | waves | per-group calls | "
          "bitwise |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['shape']} | {r['groups']} / {r['cells']} | {r['filter_s']:.3f} s | {r['trees_call_s']:.3f} s | "
              f"{r['gather_s']:.3f} / {r['dist_s']:.3f} / {r['link_s']:.3f} s | {r['waves']} (widest {r['widest_wave']}) | "
              f"{r['per_group_calls_s']:.3f} s | {'equal' if r['bitwise_equal'] else 'DIFFERENT'} |")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)
    if not all(r["bitwise_equal"] for r in rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
