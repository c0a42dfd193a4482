#!/usr/bin/env python
"""Timings of the secondary kernels at configs[1] size (10 000 x 10 000): 2-D median filter
(apply_median_filtering, window 7, subclusters of 50-500 cells) and the i3 HMM.  CUDA events, 5 runs."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from infercnv_b200 import dist as shard  # noqa: E402
from infercnv_b200.device import Engine  # noqa: E402
from infercnv_b200.hmm import i3HMM_get_HMM  # noqa: E402

eng = Engine(0)
G, C = 10000, 10000
cs, cl = bench.chr_layout(G)
refs = bench.ref_groups_global(C)
plan = shard.plan_shards(C, refs, 1)[0]
X = eng.synth(G, cs, cl, plan.local_cells, C, bench.SEED)
Y, _ = eng.smooth_block(X, cs, cl, plan.local_ref_groups(), plan.ref_sizes, plan.max_chunks)
rng = np.random.default_rng(4)
groups, pos = [], 0
while pos < C:
    n = int(rng.integers(50, 501))
    groups.append(np.arange(pos, min(C, pos + n)))
    pos += n


def timed(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


out = {}
F = torch.empty_like(Y)
ms = timed(lambda: eng.median_filter(Y, cs, cl, groups, 7, out=F))
out["median_filter_w7"] = {"ms": ms, "cell_genes_per_s": G * C / ms * 1e3, "algorithmic_GBps": 16 * G * C / ms / 1e6,
                           "blocks": len(groups) * len(cs)}
ref_cells = np.concatenate(plan.local_ref_groups())
mu = float(Y[ref_cells].mean().item())
sg = float(Y[ref_cells].std().item())
from statistics import NormalDist  # noqa: E402
Pi3, d3, mean3, sd3 = i3HMM_get_HMM({"mu": mu, "sigma": sg, "mean_delta": abs(NormalDist(0, sg).inv_cdf(0.05)), "KS_delta": None}, 1e-6)
ms = timed(lambda: eng.viterbi(Y, cs, cl, Pi3, d3, mean3, sd3))
out["viterbi_i3"] = {"ms": ms, "cell_genes_per_s": G * C / ms * 1e3, "algorithmic_GBps": 9 * G * C / ms / 1e6}
# ---- pairwise distances among the cells of one group (hclust input): FP64-pipe bound, 2 FP64 instructions per (pair, gene)
n_d = 9000
D = torch.empty(n_d * (n_d - 1) // 2, dtype=torch.float64, device=Y.device)
cells_d = np.arange(1000, 1000 + n_d, dtype=np.int32)   # the observation cells of the c2 matrix
ms = timed(lambda: eng.pairwise_dist(Y, cells_d, out=D))
pair_genes = n_d * (n_d - 1) / 2 * G
sm_mhz = float(torch.cuda.clock_rate()) if hasattr(torch.cuda, "clock_rate") else 1980.0
out["pairwise_dist_9000_cells"] = {"ms": ms, "pair_genes_per_s": pair_genes / ms * 1e3, "fp64_instr_per_s": 2 * pair_genes / ms * 1e3,
                                   "fp64_pipe_frac_at_64_per_clk_per_sm": 2 * pair_genes / (ms * 1e-3) / (64 * torch.cuda.get_device_properties(0).multi_processor_count * sm_mhz * 1e6),
                                   "tiles_computed": ((n_d + 127) // 128) * ((n_d + 127) // 128 + 1) // 2,
                                   "sm_mhz": sm_mhz}
# ---- region calling on the device-resident i6 states (K7), ingest (K8) and the element-wise steps (K9) ----
from infercnv_b200.hmm import CNV_LEVELS, get_HMM  # noqa: E402
Pi6, d6, _, _ = get_HMM({k: {"mean": m, "sd": s} for k, m, s in zip(CNV_LEVELS, bench.I6_MEAN, bench.I6_SD)}, 1e-6)
S, _ = eng.viterbi(Y, cs, cl, Pi6, d6, bench.I6_MEAN, bench.I6_SD)
gs = np.arange(G, dtype=np.float64) * 1000.0
ge = gs + 5000.0
ms = timed(lambda: eng.state_consensus(S, groups))
out["state_consensus_subclusters"] = {"ms": ms, "cell_genes_per_s": G * C / ms * 1e3, "algorithmic_GBps": 1 * G * C / ms / 1e6,
                                      "groups": len(groups)}
cons = eng.state_consensus(S, groups)
ms = timed(lambda: eng.cnv_regions(cons, cs, cl, gs, ge))
out["cnv_regions_subclusters"] = {"ms": ms, "sequences": len(groups), "regions": int(len(eng.cnv_regions(cons, cs, cl, gs, ge)["seq"]))}
cells_all = np.arange(C)
ms = timed(lambda: eng.cnv_regions(S, cs, cl, gs, ge, cols=cells_all), reps=3)
reg = eng.cnv_regions(S, cs, cl, gs, ge, cols=cells_all)
out["cnv_regions_by_cell"] = {"ms": ms, "cell_genes_per_s": G * C / ms * 1e3, "algorithmic_GBps": 2 * G * C / ms / 1e6,
                              "regions": int(len(reg["seq"])), "note": "includes the D2H fetch of the records"}
import ctypes as ct  # noqa: E402
from infercnv_b200 import _lib  # noqa: E402
from infercnv_b200.device import _stream_ptr  # noqa: E402
lib = _lib.load()
sums = torch.empty(G, dtype=torch.float64, device="cuda")
npos = torch.empty(G, dtype=torch.int32, device="cuda")
ms = timed(lambda: _lib.check(lib.icnv_dev_gene_stats_f64(X.data_ptr(), G, G, C, sums.data_ptr(), npos.data_ptr(), _stream_ptr())))
out["gene_stats_dense"] = {"ms": ms, "cell_genes_per_s": G * C / ms * 1e3, "algorithmic_GBps": 8 * G * C / ms / 1e6}
keep = torch.arange(0, G, 1, dtype=torch.int32, device="cuda")[torch.rand(G, device="cuda") > 0.15].contiguous()
Z = torch.empty((C, int(keep.numel())), dtype=torch.float64, device="cuda")
ms = timed(lambda: _lib.check(lib.icnv_dev_gather_rows_f64(X.data_ptr(), G, keep.data_ptr(), int(keep.numel()), Z.data_ptr(), C,
                                                          _stream_ptr())))
out["remove_genes"] = {"ms": ms, "algorithmic_GBps": 8 * (G + int(keep.numel())) * C / ms / 1e6, "kept": int(keep.numel())}
mins = torch.empty(C, dtype=torch.float64, device="cuda")
maxs = torch.empty(C, dtype=torch.float64, device="cuda")
ms = timed(lambda: _lib.check(lib.icnv_dev_column_minmax_f64(Y.data_ptr(), G, C, mins.data_ptr(), maxs.data_ptr(), _stream_ptr())))
out["column_minmax"] = {"ms": ms, "algorithmic_GBps": 8 * G * C / ms / 1e6}
ms = timed(lambda: _lib.check(lib.icnv_dev_clamp_bounds_f64(Y.data_ptr(), F.data_ptr(), G * C, 0.9, 1.1, _stream_ptr())))
out["clamp_bounds"] = {"ms": ms, "algorithmic_GBps": 16 * G * C / ms / 1e6}
print(json.dumps(out))
