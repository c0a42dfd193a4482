#!/usr/bin/env python
"""Time the non-DE mask split over ranks (Engine.mask_non_de_sharded) and over the device slots of the host entry point.

    torchrun --nproc-per-node N tools/bench_de_sharded.py [--genes 10000] [--cells 100000] [--tests wilcoxon,t] [--reps 2]
                                                           [--host] [--json out.json]

Workload: as tools/bench_de.py (c4's shape by default): Engine.synth's expression, bench.ref_groups_global's two reference
groups and bench.subclusters_global's subclusters, each tested against both references, p < 0.05, "any".  The cells are cut
into N contiguous blocks, one per rank, so the reference groups are cut across ranks.  --cells is the TOTAL; a c5-shaped
slice per rank is --genes 20000 --cells 62500 on one rank (c5's 500 000 cells over 8 ranks).
  * the sharded device call, host clock around it with a barrier before and after, warm, best of --reps (the slowest rank's
    time is the call's time);
  * --host (rank 0, after the ranks are done): icnv_mask_non_de_f64 from pageable NumPy memory with one device slot and, when
    the box has more than one GPU, with every GPU (icnv_init_devices).
    ICNV_DIST_BACKEND=gloo ICNV_ONE_GPU=1: every rank on cuda:0, the exchange through host memory - this shows correctness
    and overhead, not scaling.  The card's name, power limit and maximum SM clock are read in the same run.
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
    ap.add_argument("--host", action="store_true")
    ap.add_argument("--json")
    args = ap.parse_args()

    import torch
    import torch.distributed as dist
    import bench
    from infercnv_b200 import api
    from infercnv_b200.device import Engine
    from tools.bench_random_trees import card

    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", "0"), ("WORLD_SIZE", "1"), ("LOCAL_RANK", "0")))
    backend = os.environ.get("ICNV_DIST_BACKEND", "nccl")
    if os.environ.get("ICNV_ONE_GPU", "0") == "1":
        local = 0
    torch.cuda.set_device(local)
    if world > 1:
        if backend == "nccl":
            dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend)
    eng = Engine(local)
    G, C = args.genes, args.cells
    cs, cl = bench.chr_layout(G)
    c0, c1 = C * rank // world, C * (rank + 1) // world
    X = eng.synth(G, cs, cl, np.arange(c0, c1), C, 1234)
    refs = bench.ref_groups_global(C)
    subs = bench.subclusters_global(C, 1234)

    def local_lists(groups):
        out = []
        for g in groups:
            g = np.sort(np.asarray(g, dtype=np.int64))
            out.append((g[(g >= c0) & (g < c1)] - c0).astype(np.int32))
        return out

    ref_l, sub_l = local_lists(refs), local_lists(subs)
    out = {"card": card() if rank == 0 else None, "ranks": world, "backend": backend if world > 1 else None, "genes": G,
           "cells": C, "subclusters": len(subs), "pairs": len(subs) * len(refs), "results": {}}

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()

    for test in args.tests.split(","):
        Y = torch.empty_like(X)
        eng.mask_non_de_sharded(X, ref_l, sub_l, test=test, center_val=0.0, seed=1, out=Y)     # warm
        best = None
        for _ in range(args.reps):
            barrier()
            t0 = time.perf_counter()
            eng.mask_non_de_sharded(X, ref_l, sub_l, test=test, center_val=0.0, seed=1, out=Y)
            barrier()
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
        out["results"][test] = {"device_s": best}
        if rank == 0:
            print(json.dumps({test: out["results"][test], "ranks": world}), flush=True)
    del X, Y
    torch.cuda.empty_cache()
    if args.host and rank == 0:
        Xh = np.asfortranarray(eng.synth(G, cs, cl, np.arange(C), C, 1234).cpu().numpy().T)
        torch.cuda.empty_cache()
        slots = [1] + ([torch.cuda.device_count()] if torch.cuda.device_count() > 1 else [])
        for n in slots:
            if n == 1:
                api.init(local)
            else:
                api.init_devices(None)
            for test in args.tests.split(","):
                t0 = time.perf_counter()
                api.mask_non_de_genes(Xh, refs, subs, test=test, center_val=0.0, seed=1)
                dt = time.perf_counter() - t0
                out["results"].setdefault(test, {})[f"host_abi_{n}_slots_s"] = dt
                print(json.dumps({test: {f"host_abi_{n}_slots_s": dt, "stages": api.mask_non_de_stats()}}), flush=True)
        api.init(local)
    if rank == 0:
        print(json.dumps(out), flush=True)
        if args.json:
            with open(args.json, "w") as f:
                json.dump(out, f, indent=1)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
