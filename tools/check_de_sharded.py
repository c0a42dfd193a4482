#!/usr/bin/env python
"""torchrun --nproc-per-node N tools/check_de_sharded.py : Engine.mask_non_de_sharded on a cell shard must give, on every rank,
the bytes of api.mask_non_de_genes on the whole matrix (p_raw, p_adj, and this rank's columns of Y) for the cases of
tests/de_shards.py - reference groups cut over the ranks, subclusters whole, the last rank without listed cells (N > 2),
forced gene sub-slabs - and a NaN in one rank's listed cell must raise ICNV_E_NONFINITE on every rank.  Prints BITWISE EQUAL.

    ICNV_DIST_BACKEND=gloo ICNV_ONE_GPU=1   every rank on cuda:0, the exchange through host memory (tests/test_gpu_de_mask_sharded.py);
                                            default: NCCL, one GPU per rank
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from infercnv_b200 import api  # noqa: E402
from infercnv_b200._lib import InfercnvB200Error  # noqa: E402
from infercnv_b200.device import Engine  # noqa: E402
from tests import de_shards  # noqa: E402

rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", "0"), ("WORLD_SIZE", "1"), ("LOCAL_RANK", "0")))
backend = os.environ.get("ICNV_DIST_BACKEND", "nccl")
if os.environ.get("ICNV_ONE_GPU", "0") == "1":
    local = 0
torch.cuda.set_device(local)
if backend == "nccl":
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
else:
    dist.init_process_group(backend)
eng = Engine(local)
ok = True
for name, G, ref_sizes, sub_sizes, kw, mk in de_shards.CASES:
    for slab in (None, 5):
        X, shards, refs, subs = de_shards.make_case(world, G * 7, ref_sizes, sub_sizes, seed=17 + len(name),
                                                     empty_rank=world - 1 if world > 2 else None, **mk)
        cv = float(np.mean(X))
        want = api.mask_non_de_genes(X, refs, subs, center_val=cv, **kw)
        c0, c1, ref_local, sub_local = shards[rank]
        Xl = torch.as_tensor(np.ascontiguousarray(X[:, c0:c1].T), device=eng.tdev)
        Y, P, A = eng.mask_non_de_sharded(Xl, ref_local, sub_local, center_val=cv, slab_genes=slab, **kw)
        good = (Y.cpu().numpy().T.tobytes() == np.ascontiguousarray(want[0][:, c0:c1]).tobytes()
                and P.cpu().numpy().T.tobytes() == want[1].tobytes() and A.cpu().numpy().T.tobytes() == want[2].tobytes())
        if not good:
            print(f"[rank {rank}] {name}, slab {slab}: MISMATCH", flush=True)
        ok &= good
# the default centre: the mean over all ranks, the same for any number of ranks
X, shards, refs, subs = de_shards.make_case(world, 50, [40, 30], [20, 60], seed=5)
c0, c1, ref_local, sub_local = shards[rank]
Xl = torch.as_tensor(np.ascontiguousarray(X[:, c0:c1].T), device=eng.tdev)
eng.collective = False   # the same mean computed by this rank alone over the whole matrix
cv1 = eng.mean_sd(torch.as_tensor(np.ascontiguousarray(X.T), device=eng.tdev), [np.arange(X.shape[1])])[0]
eng.collective = True
Y, _, _ = eng.mask_non_de_sharded(Xl, ref_local, sub_local)
want = api.mask_non_de_genes(X, refs, subs, center_val=cv1)
ok &= Y.cpu().numpy().T.tobytes() == np.ascontiguousarray(want[0][:, c0:c1]).tobytes()
# a NaN in one rank's listed cell: every rank raises
Z = X.copy()
Z[7, refs[1][-1]] = np.nan
Zl = torch.as_tensor(np.ascontiguousarray(Z[:, c0:c1].T), device=eng.tdev)
try:
    eng.mask_non_de_sharded(Zl, ref_local, sub_local, center_val=0.0)
    ok = False
    print(f"[rank {rank}] NaN not reported", flush=True)
except InfercnvB200Error as e:
    ok &= e.code == -5
t = torch.tensor([int(ok)], dtype=torch.int32, device=eng.tdev if backend == "nccl" else "cpu")
dist.all_reduce(t, op=dist.ReduceOp.MIN)
all_ok = bool(t.item())
if rank == 0:
    print(f"[check_de_sharded] {world} ranks ({backend}): {'BITWISE EQUAL' if all_ok else 'MISMATCH'}", flush=True)
dist.destroy_process_group()
sys.exit(0 if all_ok else 1)
