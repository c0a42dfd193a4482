#!/usr/bin/env python
"""Time K16, coordinate-weighted smoothing (icnv_smooth_coords.cu; smooth_by_chromosome_coordinates, run() step 10 with
smooth_method = "coordinates"), on the GPU (DESIGN section 3, K16).

    python tools/bench_smooth_coordinates.py [--genes 10000] [--cells 100000] [--windows 1e7,1e6] [--reps 3]
                                             [--host-cells N] [--json out.json]

Workload: tests/coordinates_reference.synthetic_coordinates (seeded: the example's chromosomes in its proportions, gene
lengths drawn from its genes), Engine.synth's G x C values through log2(x + 1) and per-gene centring, as at step 10.
Per window:
  * the call on device memory (Engine.smooth_coordinates: host stencil build, its upload, the kernel), host clock around
    it with a synchronise, warm, best of --reps; the kernel alone from torch.profiler (CUDA activity "smooth_coords_kernel")
    in a separate call;
  * terms (sum over rows of the band length, times C), terms per second, and the share of the FP64 pipe: 8 FP64
    instructions per term (one product, a six-operation two-sum, one compensation add) over SMs x 64 per clock x the
    maximum SM clock; HBM bytes (X in, Y out) and their time at the data sheet's 3.35 TB/s;
  * the call through the host ABI (icnv_smooth_coordinates_f64) from pageable NumPy memory, as an R matrix arrives, on
    --host-cells cells;
  * the outputs of 16 seeded cells checked against the R-arithmetic restatement (the bound, and the bit-identical share);
  * a CPU stand-in: the restatement (NumPy, one core) on 4 cells, scaled to C cells.  R was not measured.
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
GOLDEN = os.path.join(ROOT, "tests", "golden")
FP64_PER_TERM = 8
HBM_BPS = 3.35e12


def kernel_ms(fn) -> float:
    """Device time of the smoothing kernel in one call of fn, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "smooth_coords_kernel" in e.key)
    if us <= 0:
        raise RuntimeError("the profiler saw no smooth_coords_kernel")
    return us / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genes", type=int, default=10000)
    ap.add_argument("--cells", type=int, default=100000)
    ap.add_argument("--windows", default="1e7,1e6")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-cells", type=int, default=None)
    ap.add_argument("--json")
    args = ap.parse_args()

    import torch
    from infercnv_b200 import api
    from infercnv_b200.device import Engine
    from tests import coordinates_reference as cr
    from tools.bench_random_trees import card

    G, C = args.genes, args.cells
    hc = min(args.host_cells or C, C)
    eng = Engine(0)
    st, sp, cs, cl = cr.synthetic_coordinates(G, 7, GOLDEN)
    X = torch.log2(eng.synth(G, cs, cl, np.arange(C), C, 1234) + 1.0)
    X = X - X.mean(dim=0, keepdim=True)
    Y = torch.empty_like(X)
    torch.cuda.synchronize()
    props = torch.cuda.get_device_properties(0)
    info = card()
    out = {"card": info, "sms": props.multi_processor_count, "genes": G, "cells": C, "results": {}}
    print(json.dumps({k: out[k] for k in ("card", "sms", "genes", "cells")}), flush=True)
    sample = np.sort(np.random.default_rng(0).choice(C, min(16, C), replace=False))
    Xs = np.asfortranarray(X[torch.as_tensor(sample, device=X.device)].cpu().numpy().T)
    Xh = np.asfortranarray(X[:hc].cpu().numpy().T)
    for W in [float(w) for w in args.windows.split(",")]:
        rows = cr.stencil(G, cs, cl, st, sp, W)
        band = np.array([r[1] for r in rows], dtype=np.int64)
        terms = int(band.sum()) * C
        r = {"window": W, "band_mean": float(band.mean()), "band_max": int(band.max()), "stencil_MB": band.sum() * 8 / 1e6}
        call = lambda: eng.smooth_coordinates(X, cs, cl, st, sp, W, out=Y)   # noqa: E731
        best = None
        for _ in range(args.reps + 1):          # the first call warms up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            call()
            torch.cuda.synchronize()
            t = time.perf_counter() - t0
            best = t if best is None else min(best, t)
        r["device_call_s"] = best
        r["kernel_ms"] = kernel_ms(call)
        ks = r["kernel_ms"] / 1e3
        r["terms"] = terms
        r["terms_per_s"] = terms / ks
        peak = props.multi_processor_count * 64 * info.get("max_sm_MHz", float("nan")) * 1e6
        r["fp64_pipe_share"] = terms * FP64_PER_TERM / peak / ks
        r["hbm_bytes"] = 2 * 8 * G * C
        r["hbm_floor_ms"] = r["hbm_bytes"] / HBM_BPS * 1e3
        t0 = time.perf_counter()
        api.smooth_coordinates(Xh, cs, cl, st, sp, W)
        r["host_abi_pageable_s"] = time.perf_counter() - t0
        r["host_abi_cells"] = hc
        Ys = Y[torch.as_tensor(sample, device=Y.device)].cpu().numpy().T
        ref = cr.smooth_ld(Xs, cs, cl, st, sp, W, rows)
        r["bit_identical_share"] = cr.check_coordinates(Ys, Xs, cs, cl, st, sp, W, ref)
        t0 = time.perf_counter()
        cr.smooth_ld(Xs[:, :4], cs, cl, st, sp, W, rows)
        r["numpy_restatement_scaled_s"] = (time.perf_counter() - t0) / 4 * C
        r["numpy_note"] = "the long-double NumPy restatement on 4 cells, one core, scaled to C cells; not R"
        out["results"][f"{W:g}"] = r
        print(json.dumps({f"{W:g}": r}), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
