#!/usr/bin/env python
"""Time the fused group-mode call (icnv_smooth_hmm_groups_u8_f64, i6) against the two host calls it replaces.

    python tools/bench_group_fused.py [--cells 100000] [--genes 10000] [--reps 2] [--cases samples,subclusters,singletons]
                                      [--pinned] [--fused-only] [--json out.json]

Workload: bench.py's generators - Engine.synth's matrix in the 22-chromosome layout, the first 10 % of the cells as two
reference groups - with three sets of HMM lists, the shapes analysis_mode "samples" and "subclusters" give run() step 17:
  samples      8 observation groups of consecutive cells, then the 2 reference groups (cluster_by_groups = TRUE);
  subclusters  40 subclusters scattered through the observation and reference cells (a random label per cell);
  singletons   every observation cell a group of its own, then the reference groups (cluster_by_groups = FALSE).
The composition is icnv_smooth_block_f64 then icnv_viterbi_u8_f64 with the lists: two uploads of the matrix, the second
one whole, on one device.  Both read from and write to pageable NumPy memory (an R matrix is pageable; --pinned: torch
page-locked buffers instead, for the fused call only) and share the output buffers.  Per case they run alternately,
--reps times each after one warm call each, host clock around every call; then one fused call and one composition are
compared bitwise on 2048 seeded columns.  --fused-only times the fused call alone (shapes whose composition does not fit
on one device, such as bench.py's c5: 500 000 x 20 000).  Prints one JSON line per case with the card's name and power
limit, read in the same run.
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


def device_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    name, limit, clk = [v.strip() for v in r.stdout.strip().splitlines()[0].rsplit(",", 2)]
    return {"name": name, "power_limit_w": float(limit), "max_sm_clock_mhz": float(clk)}


def hmm_lists(case, C, refs, rng):
    first = int(refs[-1][-1]) + 1
    obs = np.arange(first, C, dtype=np.int32)
    if case == "samples":
        return [g.astype(np.int32) for g in np.array_split(obs, 8)] + refs
    if case == "subclusters":
        cells = np.arange(C, dtype=np.int32)
        lab = rng.integers(0, 40, size=C)
        return [cells[lab == k] for k in range(40)]
    if case == "singletons":
        return [obs[i:i + 1] for i in range(len(obs))] + refs
    raise SystemExit(f"unknown case {case}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=100_000)
    ap.add_argument("--genes", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--cases", default="samples,subclusters,singletons")
    ap.add_argument("--pinned", action="store_true")
    ap.add_argument("--fused-only", action="store_true")
    ap.add_argument("--json")
    args = ap.parse_args()

    import torch

    import bench
    from infercnv_b200 import _lib, api
    from infercnv_b200.device import Engine
    from oracle import oracle as orc

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    G, C = args.genes, args.cells
    seed = bench.SEED0 + bench.CONFIGS["c4"]["index"]
    cs, cl = bench.chr_layout(G)
    refs = [g.astype(np.int32) for g in bench.ref_groups_global(C)]
    if args.pinned:
        hX = torch.empty((C, G), dtype=torch.float64).pin_memory()
        hY = torch.empty((C, G), dtype=torch.float64).pin_memory()
        hS = torch.empty((C, G), dtype=torch.uint8).pin_memory()
        X, Y, S = hX.numpy().T, hY.numpy().T, hS.numpy().T     # Fortran-ordered views of the page-locked buffers
    else:
        X = np.empty((G, C), dtype=np.float64, order="F")
        Y = np.empty_like(X, order="F")
        S = np.empty((G, C), dtype=np.uint8, order="F")
    eng = Engine(0)
    step = max(1, min(C, (2 << 30) // (8 * G)))
    for c0 in range(0, C, step):   # synthesised a block of cells at a time: c5's matrix does not fit on the device
        Xd = eng.synth(G, cs, cl, np.arange(c0, min(C, c0 + step)), C, seed)
        X.T[c0:c0 + step] = Xd.cpu().numpy()
        del Xd
    torch.cuda.empty_cache()
    api.init(0)
    lib = _lib.load()
    off, idx = api.groups_to_csr(refs)
    Pi, delta = orc.hmm_params(6, 1e-6)
    mean = np.array([0.01, 0.5, 1.0, 1.5, 2.0, 3.0])
    base = np.array([0.05, 0.12, 0.1, 0.14, 0.2, 0.3])
    dev = device_info()
    rng = np.random.default_rng(seed)
    for case in args.cases.split(","):
        groups = hmm_lists(case, C, refs, rng)
        sd = np.concatenate([base * (1.0 + 3.0 / np.sqrt(len(g))) for g in groups])
        hoff, hidx = api.groups_to_csr(groups)

        def fused():
            _lib.check(lib.icnv_smooth_hmm_groups_u8_f64(X.ctypes.data, Y.ctypes.data, S.ctypes.data, G, C, cs.ctypes.data,
                                                         cl.ctypes.data, len(cs), off.ctypes.data, idx.ctypes.data,
                                                         len(refs), 1, 3.0, 101, 1, hoff.ctypes.data, hidx.ctypes.data,
                                                         len(groups), 6, Pi.ctypes.data, delta.ctypes.data,
                                                         mean.ctypes.data, sd.ctypes.data))

        def composed():
            api.smooth_block(X, cs, cl, refs, apply_log=True, threshold=3.0, window_length=101, out=Y)
            api.viterbi(Y, cs, cl, Pi, delta, mean, sd, groups=groups, out=S)

        def timed(fn):
            t0 = time.perf_counter()
            fn()
            return time.perf_counter() - t0

        out = {"case": case, "lists": len(groups), "cells": C, "genes": G,
               "memory": "page-locked" if args.pinned else "pageable", "device": dev}
        fused()
        t_fused, t_comp = [], []
        if args.fused_only or args.pinned:
            t_fused = [timed(fused) for _ in range(args.reps)]
        else:
            composed()
            for _ in range(args.reps):
                t_fused.append(timed(fused))
                t_comp.append(timed(composed))
            cols = np.sort(np.random.default_rng(seed).choice(C, size=min(C, 2048), replace=False))
            fused()
            Yf, Sf = Y[:, cols], S[:, cols]
            composed()
            out["outputs_bit_identical"] = bool(np.array_equal(Yf, Y[:, cols]) and np.array_equal(Sf, S[:, cols]))
            out["composed_s"] = t_comp
            out["composed_best_s"] = min(t_comp)
            out["speedup_best"] = min(t_comp) / min(t_fused)
        out["fused_s"] = t_fused
        out["fused_best_s"] = min(t_fused)
        line = json.dumps(out)
        print(line, flush=True)
        if args.json:
            with open(args.json, "a") as fh:
                fh.write(line + "\n")


if __name__ == "__main__":
    main()
