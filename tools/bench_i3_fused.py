#!/usr/bin/env python
"""Time the fused i3 pass (icnv_smooth_i3_hmm_u8_f64) against the four host calls it replaces, on c4's workload.

    python tools/bench_i3_fused.py [--cells 100000] [--genes 10000] [--reps 3] [--json out.json]

Workload: bench.py's c4 generators - Engine.synth's matrix in the 22-chromosome layout, the first 10 % of the cells as two
reference groups, the observation cells as 50-500-cell subclusters; the median filter runs over the subclusters and the
reference groups with window 7, the smoothing window is 101, i3_p_val 0.05, t 1e-6.  Both paths read from and write to
pageable NumPy memory (an R matrix is pageable) and share the output buffers; they are run alternately, --reps times
each after one warm call each, host clock around every call.  The four-call composition is what bench.py's c4 e2e leg
times: icnv_smooth_block_f64, icnv_mean_sd_f64, icnv_viterbi_u8_f64, icnv_median_filter_f64.  After the timed calls
the outputs of one fused call are compared with those of one composition (bitwise, on 2048 seeded columns).  Prints one JSON line with the
card's name and power limit, read in the same run.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=100_000)
    ap.add_argument("--genes", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json")
    args = ap.parse_args()

    import torch

    import bench
    from infercnv_b200 import _lib, api, hmm
    from infercnv_b200.device import Engine

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    G, C = args.genes, args.cells
    seed = bench.SEED0 + bench.CONFIGS["c4"]["index"]
    cs, cl = bench.chr_layout(G)
    refs = [g.astype(np.int32) for g in bench.ref_groups_global(C)]
    subs = [s.astype(np.int32) for s in bench.subclusters_global(C, seed)]
    lists = subs + refs
    eng = Engine(0)
    X = np.empty((G, C), dtype=np.float64, order="F")      # pageable
    Xd = eng.synth(G, cs, cl, np.arange(C), C, seed)
    X.T[...] = Xd.cpu().numpy()
    del Xd
    torch.cuda.empty_cache()
    api.init(0)
    lib = _lib.load()
    Y = np.empty_like(X, order="F")
    F = np.empty_like(X, order="F")
    S = np.empty((G, C), dtype=np.uint8, order="F")
    off, idx = api.groups_to_csr(refs)
    moff, midx = api.groups_to_csr(lists)
    model = np.zeros(3)
    ref_all = np.concatenate(refs)

    def fused():
        _lib.check(lib.icnv_smooth_i3_hmm_u8_f64(X.ctypes.data, Y.ctypes.data, S.ctypes.data, F.ctypes.data, G, C, cs.ctypes.data,
                                                 cl.ctypes.data, len(cs), off.ctypes.data, idx.ctypes.data, len(refs), 1, 3.0,
                                                 101, 1, 0.05, 1e-6, moff.ctypes.data, midx.ctypes.data, len(lists), 7,
                                                 model.ctypes.data))

    def four_calls():
        api.smooth_block(X, cs, cl, refs, apply_log=True, threshold=3.0, window_length=101, out=Y)
        mu, sg = api.mean_sd(Y, ref_all)
        Pi, delta, mean, sd = hmm.i3HMM_get_HMM({"mu": mu, "sigma": sg, "mean_delta": hmm.i3_mean_delta(sg, 0.05),
                                                "KS_delta": None}, 1e-6)
        api.viterbi(Y, cs, cl, Pi, delta, mean, sd, out=S)
        api.median_filter(Y, cs, cl, lists, 7, out=F)
        return mu, sg

    def timed(fn):
        t0 = time.perf_counter()
        fn()
        return time.perf_counter() - t0

    fused()
    four_calls()
    t_fused, t_four = [], []
    for _ in range(args.reps):
        t_fused.append(timed(fused))
        t_four.append(timed(four_calls))
    # outputs: one fused call against one composition, on 2048 seeded columns (a full copy would double the host memory)
    cols = np.sort(np.random.default_rng(seed).choice(C, size=min(C, 2048), replace=False))
    fused()
    Yf, Sf, Ff, mf = Y[:, cols], S[:, cols], F[:, cols], model.copy()
    mu, sg = four_calls()
    same = bool(np.array_equal(Yf, Y[:, cols]) and np.array_equal(Sf, S[:, cols]) and np.array_equal(Ff, F[:, cols])
                and mf[0] == mu and mf[1] == sg)
    out = {
        "workload": f"c4 through the host ABI: {C} cells x {G} genes, pageable NumPy memory, i3 per cell, "
                    f"apply_median_filtering(window 7) over {len(subs)} subclusters and {len(refs)} reference groups",
        "fused_s": t_fused, "four_calls_s": t_four,
        "fused_best_s": min(t_fused), "four_calls_best_s": min(t_four), "speedup_best": min(t_four) / min(t_fused),
        "bytes_fused": {"h2d": 8 * G * C, "d2h": 17 * G * C},
        "outputs_bit_identical": same, "mu": float(mf[0]), "sigma": float(mf[1]), "mean_delta": float(mf[2]),
        "device": device_info(),
    }
    line = json.dumps(out)
    print(line)
    if args.json:
        with open(args.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
