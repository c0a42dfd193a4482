"""Cell-sharded inputs of the non-DE mask for the rank-split checks (tools/check_de_sharded.py, tests/test_gpu_de_stages.py):
a genes x cells matrix cut into one contiguous block of columns per rank, every reference group cut over the ranks (uneven
slices, some empty), every subcluster whole on one rank, the local lists in a shuffled column order, and a few unlisted cells
per rank.  `empty_rank` holds no listed cell.  Global list order = group by group, rank by rank, as Engine.mask_non_de_sharded
reads the local lists."""
from __future__ import annotations

import numpy as np


def dead_band(G, C, rng, frac):
    """After 2^x the use-bounds dead band leaves many values at exactly 1.0 (ties)."""
    X = 1.0 + rng.normal(scale=0.2, size=(G, C))
    X[rng.uniform(size=(G, C)) < frac] = 1.0
    X[: G // 3, C // 2:] += 0.3
    return np.asfortranarray(X)


def make_case(world, G, ref_sizes, sub_sizes, seed, frac=0.3, empty_rank=None, extra=3):
    """Returns (X, shards, refs, subs): X the whole G x C matrix, shards[r] = (c0, c1, ref_local, sub_local) with the LOCAL
    column lists of rank r, refs / subs the global lists in list order."""
    rng = np.random.default_rng(seed)
    holders = [r for r in range(world) if r != empty_rank] or [0]
    # per rank: how many cells of each reference group, which subclusters
    ref_cnt = np.zeros((world, len(ref_sizes)), dtype=np.int64)
    for j, n in enumerate(ref_sizes):
        cuts = np.sort(rng.integers(0, n + 1, size=len(holders) - 1))
        ref_cnt[holders, j] = np.diff(np.concatenate([[0], cuts, [n]]))
    owner = [holders[s % len(holders)] for s in range(len(sub_sizes))]
    n_local = [int(ref_cnt[r].sum()) + sum(n for s, n in enumerate(sub_sizes) if owner[s] == r) + extra + r for r in range(world)]
    cb = np.concatenate([[0], np.cumsum(n_local)]).astype(np.int64)
    X = dead_band(G, int(cb[-1]), rng, frac)
    shards = []
    refs = [[] for _ in ref_sizes]
    subs = [None] * len(sub_sizes)
    for r in range(world):
        perm = rng.permutation(n_local[r]).astype(np.int32)
        pos = 0
        ref_local = []
        for j in range(len(ref_sizes)):
            ref_local.append(perm[pos:pos + ref_cnt[r, j]])
            pos += int(ref_cnt[r, j])
        sub_local = []
        for s, n in enumerate(sub_sizes):
            if owner[s] == r:
                sub_local.append(perm[pos:pos + n])
                pos += n
            else:
                sub_local.append(np.zeros(0, np.int32))
        shards.append((int(cb[r]), int(cb[r + 1]), ref_local, sub_local))
        for j in range(len(ref_sizes)):
            refs[j].append(cb[r] + ref_local[j])
        for s in range(len(sub_sizes)):
            if owner[s] == r:
                subs[s] = cb[r] + sub_local[s]
    refs = [np.concatenate(g).astype(np.int32) for g in refs]
    subs = [np.asarray(g, dtype=np.int32) for g in subs]
    return X, shards, refs, subs


# (name, G, reference group sizes, subcluster sizes, kwargs of mask_non_de_genes, kwargs of make_case)
CASES = [
    ("wilcoxon exact and asymptotic", 45, [60, 45], [30, 55, 3, 49, 50, 51], dict(seed=7), dict(frac=0.3)),
    ("wilcoxon all ties kept", 37, [50, 20], [12, 70, 5], dict(seed=3, jitter_sd=0.0, rule="most"), dict(frac=0.6)),
    ("t test", 33, [40, 25], [20, 60, 1, 4], dict(test="t", rule="most", p_val_thresh=0.2), dict(frac=0.2)),
    ("three references, rule all", 41, [40, 50, 35], [20, 70, 4], dict(rule="all", p_val_thresh=0.2, seed=11), dict(frac=0.2)),
    ("no tested subcluster", 29, [30], [], dict(), dict()),
]
