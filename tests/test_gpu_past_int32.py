"""The whole-matrix calls on one GPU past 2^31 elements: a (C, G) float64 matrix of 10 007 genes x 230 000 cells
(2.30e9 entries, and as many in the uint8 state matrix), checked on sampled columns on both sides of the entry 2^31.

A kernel that forms one 32-bit product (an `int` column times an `int` leading dimension, a `(int)` cast of an offset, an
`unsigned` byte count) runs correctly at every size the rest of the suite uses and writes into the wrong column past
element 2 147 483 648.  Every check here compares two things:

- the same call on a small matrix made of only the columns it needs (sampled cells, reference groups, index lists), which
  must give the same bits: only where the columns sit differs, so any difference is an addressing bug;
- the existing independent reference (tests/cellpipe_reference.py, oracle/, tests/de_reference.py) on those columns.

G = 10 007 is prime, so no column boundary lands on 2^31 and no tile width divides G; the chromosome layout is bench.py's
scaled to G, with a chromosome of one gene and one of two inserted.  The reference groups (6 % and 4 % of the cells, as
in bench.py) sit at the end of the matrix instead of the start, cells [205 000, 228 000): the first group straddles column
214 598, the one that holds entries 2^31 - 1 and 2^31, the second lies wholly past it, so every reference-mean pass
(partial sums, bounds, mean_sd, group means) reads past the boundary.  The last 2 000 cells belong to no reference group:
the subclusters, median-filter lists and distance lists are drawn from them.

X, Y and the states take 18.4 + 18.4 + 2.3 GB; with the small calls the measured peak was 44.9 GB of torch allocations
(47.5 GB in use on the device) and the whole module took 220 s, on an H100 80GB HBM3 at a 700 W power limit.  The test
skips when the device has less free memory than it needs.  The host-pointer check runs only when the host has the RAM
for two 18.4 GB matrices.
"""
import math
import os
import time
from itertools import chain

import numpy as np
import pytest

from infercnv_b200 import _lib

pytestmark = pytest.mark.gpu
EMULATED = "_emu" in os.path.basename(_lib.LIB_PATH)
if EMULATED:
    pytestmark = [pytest.mark.gpu, pytest.mark.skip(reason="GPU only: 2.3e9-entry matrices are far too large for the host emulation")]

G = 10007
C = 230000
TAIL = 2000                          # cells behind the reference groups
SEED = 20261017
U = 2.0 ** -53
BOUNDARY = 2 ** 31
B_COL = (BOUNDARY - 1) // G          # column holding entries 2^31 - 1 and 2^31
FLOAT_BYTES = G * C * 8
STATE_BYTES = G * C


def past(cols, ld=G):
    """the columns whose last entry lies at or past element 2^31 of a matrix with leading dimension ld"""
    return [int(c) for c in np.asarray(cols).ravel() if (int(c) + 1) * ld > BOUNDARY]


def layout():
    import bench
    cs, cl = bench.chr_layout(G - 3)
    lens = list(cl)
    lens.insert(5, 1)
    lens.insert(13, 2)
    lens = np.asarray(lens, dtype=np.int32)
    assert int(lens.sum()) == G and 1 in lens and 2 in lens
    return np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32), lens


def gather(t, cols):
    import torch
    return t[torch.as_tensor(np.asarray(cols, dtype=np.int64), device=t.device)].contiguous()


def local(cols_small, cells):
    """positions of `cells` in the sorted column list of a small matrix"""
    pos = np.searchsorted(cols_small, cells)
    assert np.array_equal(cols_small[pos], cells)
    return pos.astype(np.int32)


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def ulps(a, b):
    return abs(a - b) / math.ulp(max(abs(a), abs(b)))


def log(msg):
    print(f"[past 2^31] {msg}", flush=True)


@pytest.fixture(scope="module")
def world():
    import torch

    import bench
    from infercnv_b200 import api
    from infercnv_b200.device import Engine

    free, total = torch.cuda.mem_get_info()
    need = 2 * FLOAT_BYTES + STATE_BYTES + (12 << 30)
    if free < need:
        pytest.skip(f"needs {need / 1e9:.1f} GB of free device memory, the device has {free / 1e9:.1f} GB free")
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    props = torch.cuda.get_device_properties(0)
    try:
        import subprocess
        power = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    log(f"device {props.name}, power limit {power}; free memory at start {free / 1e9:.2f} GB of {total / 1e9:.2f} GB")
    log(f"G = {G}, C = {C}, G * C = {G * C}; entry 2^31 lies in column {B_COL} (rows {B_COL * G} .. {B_COL * G + G - 1})")
    assert B_COL * G <= BOUNDARY - 1 and BOUNDARY < (B_COL + 1) * G and G * C > BOUNDARY
    # the uint8 state matrix has the same leading dimension: its byte 2^31 is in the same column
    assert (BOUNDARY // G) == B_COL

    eng = Engine(0)
    cs, cl = layout()
    rng = np.random.default_rng(SEED)
    n_a, n_b = int(round(0.06 * C)), int(round(0.04 * C))
    r0 = C - TAIL - n_a - n_b
    refs = [np.arange(r0, r0 + n_a, dtype=np.int32), np.arange(r0 + n_a, r0 + n_a + n_b, dtype=np.int32)]
    ref_all = np.concatenate(refs)
    assert refs[0][0] < B_COL < refs[0][-1] and refs[1][0] > B_COL
    sampled = np.unique(np.concatenate([
        [0, C - 1, B_COL - 1, B_COL, B_COL + 1],
        rng.choice(np.arange(1, B_COL - 1), 17, replace=False),
        rng.choice(np.arange(B_COL + 2, C - TAIL), 12, replace=False),
        rng.choice(np.arange(C - TAIL, C - 1), 5, replace=False)])).astype(np.int32)
    nan_cell = C - TAIL + 777
    assert nan_cell not in sampled and past([nan_cell])
    log(f"{len(sampled)} sampled columns, {len(past(sampled))} of them past the boundary; reference groups "
        f"[{refs[0][0]}, {refs[0][-1] + 1}) and [{refs[1][0]}, {refs[1][-1] + 1})")

    X = eng.synth(G, cs, cl, np.arange(C), C, SEED)
    Xs = X[torch.as_tensor(sampled, device=X.device).long()].cpu().numpy()
    Xref = X[torch.as_tensor(ref_all, device=X.device).long()].cpu().numpy()
    Y = torch.empty_like(X)
    w = dict(torch=torch, api=api, bench=bench, eng=eng, cs=cs, cl=cl, refs=refs, ref_all=ref_all, sampled=sampled,
             rng=rng, X=X, Y=Y, Xs=Xs, Xref=Xref, t0=t0, used=[total - free])

    def mark():
        f, _ = torch.cuda.mem_get_info()
        w["used"].append(total - f)

    # 1. one NaN in a column past the boundary sets the flag
    g_nan = 5003
    keep = float(X[nan_cell, g_nan].item())
    X[nan_cell, g_nan] = float("nan")
    _, flag = eng.smooth_block(X, cs, cl, refs, out=Y)
    w["nan_flag"] = int(flag.item())
    X[nan_cell, g_nan] = keep

    # 2. reference cells leading: pass 2 takes the reuse_reference_pass branch (T[:n_ref], then X[n_ref:])
    lead = [np.arange(0, n_a, dtype=np.int32), np.arange(n_a, n_a + n_b, dtype=np.int32)]
    assert eng.reuse_reference_pass
    _, flag = eng.smooth_block(X, cs, cl, lead, out=Y)
    w["lead_flag"] = int(flag.item())
    w["lead_big"] = Y[torch.as_tensor(sampled, device=Y.device).long()].cpu().numpy()
    cols_l = np.unique(np.concatenate(lead + [sampled])).astype(np.int32)
    Xsm = gather(X, cols_l)
    Ysm, flag = eng.smooth_block(Xsm, cs, cl, [local(cols_l, g) for g in lead])
    w["lead_small"] = Ysm[torch.as_tensor(local(cols_l, sampled), device=Ysm.device).long()].cpu().numpy()
    w["lead_small_flag"] = int(flag.item())
    mark()
    del Xsm, Ysm

    # 3. the main run: reference groups at the end
    _, flag = eng.smooth_block(X, cs, cl, refs, out=Y)
    torch.cuda.synchronize()
    w["flag"] = int(flag.item())
    w["sel"] = api.last_cell_kernel()
    w["b1"] = eng._bounds[0].cpu().numpy().copy()
    w["b2"] = eng._bounds[1].cpu().numpy().copy()
    w["Ys"] = Y[torch.as_tensor(sampled, device=Y.device).long()].cpu().numpy()
    cols_s = np.unique(np.concatenate([ref_all, sampled])).astype(np.int32)
    Xsm = gather(X, cols_s)
    Ysm, flag = eng.smooth_block(Xsm, cs, cl, [local(cols_s, g) for g in refs])
    w["small_flag"] = int(flag.item())
    w["Ys_small"] = Ysm[torch.as_tensor(local(cols_s, sampled), device=Ysm.device).long()].cpu().numpy()
    mark()
    del Xsm, Ysm
    eng._T = None
    eng._plan_cache.clear()

    # per-cell i6 states (and margins) of the whole matrix
    Pi, delta, mean, sd = bench.i6_model()
    S, vflag, mg = eng.viterbi(Y, cs, cl, Pi, delta, mean, sd, want_margins=True)
    torch.cuda.synchronize()
    w.update(Pi=Pi, delta=delta, mean=mean, sd=sd, S=S, vflag=int(vflag.item()), mg=mg, mark=mark)
    mark()
    del X, Y, S, mg                  # w holds them: test_host_pointer_path frees them before it runs
    yield w
    peak = torch.cuda.max_memory_allocated()
    log(f"peak torch allocation {peak / 1e9:.2f} GB; largest device-wide use seen {max(w['used']) / 1e9:.2f} GB; "
        f"wall time {time.perf_counter() - t0:.1f} s")


def test_smooth_block(world):
    from tests import cellpipe_reference as cref
    w = world
    sampled = w["sampled"]
    assert w["nan_flag"] != 0, "a NaN past the boundary did not set the non-finite flag"
    assert w["flag"] == 0 and w["small_flag"] == 0 and w["lead_flag"] == 0 and w["lead_small_flag"] == 0
    assert past(sampled)
    assert same_bits(w["Ys"], w["Ys_small"]), "smooth_block: sampled columns differ from the small call"
    assert same_bits(w["lead_big"], w["lead_small"]), "smooth_block (reference cells leading): differs from the small call"
    log(f"smooth_block: {len(sampled)} columns bit-identical to the small call in both layouts; NaN flag {w['nan_flag']}")

    # reference means on the host from the copied reference columns (before the transform) against the device bounds;
    # the extended-precision reference below then takes the device bounds, so its error bound covers the cell alone
    LD = cref.LD
    Xref, refs, cs, cl = w["Xref"], w["refs"], w["cs"], w["cl"]
    lo1, hi1 = w["b1"][0], w["b1"][1]
    lo2, hi2 = w["b2"][0], w["b2"][1]
    m1, m2, pos = [], [], 0
    for g in refs:
        n = len(g)
        s1 = np.zeros(G, dtype=LD)
        s2 = np.zeros(G, dtype=np.float64)
        for a in range(pos, pos + n, 1000):
            blk = Xref[a:min(a + 1000, pos + n)]
            s1 += np.sum(np.log2(blk.astype(LD) + LD(1)), axis=0)
            s2 += np.sum(cref.prefix_sum_model(blk, cs, cl, apply_log=True, lo1=lo1, hi1=hi1, threshold=3.0, window=101,
                                               center=1), axis=0)
        m1.append((s1 / n).astype(np.float64))
        m2.append(s2 / n)
        pos += n
    d1 = max(np.abs(np.min(m1, axis=0) - lo1).max(), np.abs(np.max(m1, axis=0) - hi1).max())
    d2 = max(np.abs(np.min(m2, axis=0) - lo2).max(), np.abs(np.max(m2, axis=0) - hi2).max())
    log(f"reference bounds: host vs device max |diff| {d1:.2e} (log means), {d2:.2e} (smoothed means)")
    assert d1 < 1e-11 and d2 < 1e-10

    if not cref.HAS_EXTENDED:
        pytest.skip("np.longdouble is not an extended type here: no extended-precision reference")
    sel = w["sel"]
    want, bound = cref.cell_pipeline(w["Xs"], cs, cl, apply_log=True, lo1=lo1, hi1=hi1, threshold=3.0, window=101, center=1,
                                     lo2=lo2, hi2=hi2, apply_exp2=True, L=sel[5], NW=sel[1] // 32)
    r = cref.error_ratio(w["Ys"], want, bound)
    rp = cref.error_ratio(w["Ys"][np.isin(sampled, past(sampled))], want[np.isin(sampled, past(sampled))],
                          bound[np.isin(sampled, past(sampled))])
    log(f"smooth_block vs the extended-precision reference: worst error_ratio {r:.3g} ({rp:.3g} past the boundary), "
        f"kernel {sel}")
    assert r <= 1.0


def test_mean_sd(world):
    w = world
    torch, eng, refs = w["torch"], w["eng"], w["refs"]
    mu, sg = eng.mean_sd(w["Y"], refs)
    ref_all = w["ref_all"]
    Yr = gather(w["Y"], ref_all)
    mu2, sg2 = eng.mean_sd(Yr, [np.arange(len(refs[0]), dtype=np.int32),
                                np.arange(len(refs[0]), len(ref_all), dtype=np.int32)])
    assert past(ref_all)
    assert (mu, sg) == (mu2, sg2), "mean_sd differs from the small call"
    vals = Yr.cpu().numpy()
    del Yr
    n = vals.size
    blocks = range(0, len(vals), 500)
    ref_mu = math.fsum(chain.from_iterable(vals[a:a + 500].ravel().tolist() for a in blocks)) / n
    ss = math.fsum(chain.from_iterable(((vals[a:a + 500] - ref_mu) ** 2).ravel().tolist() for a in blocks))
    ref_sg = math.sqrt(ss / (n - 1))
    del vals
    # the library sums each cell's G values and then the cells in double: (G + n_cells) roundings at most
    k = G + len(ref_all)
    log(f"mean_sd over {len(ref_all)} reference cells ({len(past(ref_all))} past the boundary): mu {ulps(mu, ref_mu):.0f} ulp, "
        f"sigma {ulps(sg, ref_sg):.0f} ulp from the fsum two-pass values (bound {k} / {2 * k} ulp)")
    assert abs(mu - ref_mu) <= k * U * abs(ref_mu) * 2 and abs(sg - ref_sg) <= 2 * k * U * abs(ref_sg) * 2


def test_viterbi(world):
    from oracle import oracle as orc
    w = world
    torch, eng, sampled = w["torch"], w["eng"], w["sampled"]
    assert w["vflag"] == 0
    S, mg = w["S"], w["mg"]
    idx = torch.as_tensor(sampled, device=S.device).long()
    got = S[idx].cpu().numpy()
    Ysm = gather(w["Y"], sampled)
    S2, f2, mg2 = eng.viterbi(Ysm, w["cs"], w["cl"], w["Pi"], w["delta"], w["mean"], w["sd"], want_margins=True)
    assert int(f2.item()) == 0
    assert same_bits(got, S2.cpu().numpy()), "viterbi: states differ from the small call"
    assert same_bits(mg[idx].cpu().numpy(), mg2.cpu().numpy()), "viterbi: margins differ from the small call"
    want = orc.viterbi_matrix(np.asfortranarray(w["Ys"].T), w["cs"], w["cl"], w["Pi"], w["delta"], w["mean"], w["sd"])
    assert np.array_equal(got.T.astype(np.int32), want), "viterbi: states differ from the oracle"
    log(f"viterbi: {len(sampled)} columns ({len(past(sampled))} past the boundary) equal to the small call (states and "
        f"margins) and to the oracle")


def test_state_counts_consensus_regions(world):
    from oracle import regions as orr
    w = world
    torch, eng, S = w["torch"], w["eng"], w["S"]
    tail = np.arange(C - TAIL, C, dtype=np.int32)
    groups = [np.arange(B_COL - 100, B_COL + 120, dtype=np.int32), tail[-300:], w["rng"].permutation(tail[:700]).astype(np.int32),
              w["sampled"]]
    for g in groups[:3]:
        assert past(g)
    cols = np.unique(np.concatenate(groups)).astype(np.int32)
    Ssm = gather(S, cols)
    lg = [local(cols, g) for g in groups]
    counts = eng.state_counts(S, groups).cpu().numpy()
    assert same_bits(counts, eng.state_counts(Ssm, lg).cpu().numpy()), "state_counts differ from the small call"
    Sh = Ssm.cpu().numpy()                                  # (n, G) = the gathered columns
    for k, g in enumerate(lg):
        sub = Sh[g]
        want = np.stack([(sub == 255).sum(axis=0)] + [(sub == v).sum(axis=0) for v in range(7)], axis=1)
        assert np.array_equal(counts[k], want), f"state_counts of group {k} differ from numpy"
    cons = eng.state_consensus(S, groups)
    assert same_bits(cons.cpu().numpy(), eng.state_consensus(Ssm, lg).cpu().numpy())
    want_cons = np.stack([orr.state_consensus(np.asfortranarray(Sh.T), g) for g in lg], axis=0)
    assert np.array_equal(cons.cpu().numpy(), want_cons), "state_consensus differs from the oracle"
    gs = np.arange(G, dtype=np.float64) * 1000.0
    ge = gs + 1500.0
    cs, cl = w["cs"], w["cl"]
    reg = eng.cnv_regions(cons, cs, cl, gs, ge)
    want = orr.cnv_regions(want_cons.T, cs, cl, gs, ge)
    for k in want:
        assert np.array_equal(reg[k], want[k]), k
    # by cell: rows of the state matrix itself, listed past the boundary in shuffled order
    cells = w["rng"].permutation(np.concatenate([[B_COL, C - 1], tail[:40]])).astype(np.int32)
    reg = eng.cnv_regions(S, cs, cl, gs, ge, cols=cells)
    small = eng.cnv_regions(Ssm, cs, cl, gs, ge, cols=local(cols, cells))
    want = orr.cnv_regions(np.asfortranarray(Sh[local(cols, cells)].T), cs, cl, gs, ge)
    for k in want:
        assert np.array_equal(reg[k], small[k]) and np.array_equal(reg[k], want[k]), k
    log(f"state_counts / state_consensus / cnv_regions: {len(groups)} groups and {len(cells)} cells "
        f"({len(past(cols))} columns past byte 2^31) equal to the small call, numpy and oracle/regions.py")


def test_viterbi_groups(world):
    from oracle import oracle as orc
    w = world
    torch, eng = w["torch"], w["eng"]
    groups = [w["rng"].permutation(np.arange(B_COL - 150, B_COL + 150)).astype(np.int32),
              np.arange(C - 400, C, dtype=np.int32)]
    assert min(groups[0]) < B_COL < max(groups[0]) and min(groups[1]) > B_COL
    out = torch.empty((C, G), dtype=torch.uint8, device=w["X"].device)
    St, flag = eng.viterbi_groups(w["Y"], w["cs"], w["cl"], w["Pi"], w["delta"], w["mean"], w["sd"], groups, out=out)
    cols = np.unique(np.concatenate(groups + [w["sampled"]])).astype(np.int32)
    Ysm = gather(w["Y"], cols)
    lg = [local(cols, g) for g in groups]
    S2, f2 = eng.viterbi_groups(Ysm, w["cs"], w["cl"], w["Pi"], w["delta"], w["mean"], w["sd"], lg)
    assert int(flag.item()) == 0 and int(f2.item()) == 0
    got = gather(St, cols).cpu().numpy()
    del St, out
    assert same_bits(got, S2.cpu().numpy()), "viterbi_groups differs from the small call"
    want = orc.viterbi_matrix(np.asfortranarray(Ysm.cpu().numpy().T), w["cs"], w["cl"], w["Pi"], w["delta"], w["mean"],
                              w["sd"], groups=lg)
    g8 = np.where(got.T == 255, -1, got.T.astype(np.int32))
    assert np.array_equal(g8, want), "viterbi_groups differs from the oracle's group mode"
    outside = ~np.isin(cols, np.concatenate(groups))
    assert (got[outside] == 255).all()
    log(f"viterbi_groups: {len(cols)} columns (a group straddling column {B_COL}, one past it) equal to the small call and "
        f"the oracle; {int(outside.sum())} cells in no group stay 255")


def test_pairwise_dist_knn_cluster_cells(world):
    w = world
    torch, eng, Y = w["torch"], w["eng"], w["Y"]
    cells = w["rng"].permutation(np.arange(C - 300, C)).astype(np.int32)
    assert len(past(cells)) == len(cells)
    Ysm = gather(Y, cells)
    own = np.arange(len(cells), dtype=np.int32)
    assert same_bits(eng.pairwise_dist(Y, cells).cpu().numpy(), eng.pairwise_dist(Ysm, own).cpu().numpy())
    a, b = eng.knn(Y, 20, cells), eng.knn(Ysm, 20, own)
    assert same_bits(a[0].cpu().numpy(), b[0].cpu().numpy()) and same_bits(a[1].cpu().numpy(), b[1].cpu().numpy())
    a, b = eng.cluster_cells(Y, cells), eng.cluster_cells(Ysm, own)
    assert all(same_bits(u, v) for u, v in zip(a, b))
    log(f"pairwise_dist / knn / cluster_cells: {len(cells)} cells past the boundary equal to the small call")


@pytest.mark.parametrize("window", [5, 7, 11])
def test_median_filter(world, window):
    from oracle import oracle as orc
    w = world
    torch, eng, Y, X = w["torch"], w["eng"], w["Y"], w["X"]
    rng = np.random.default_rng(SEED + window)
    tail = np.arange(C - TAIL, C)
    lists = [rng.permutation(np.arange(B_COL - 150, B_COL + 151)),
             rng.permutation(tail[-400:]),
             rng.permutation(np.concatenate([rng.choice(np.arange(1, B_COL - 200), 40, replace=False),
                                             rng.choice(np.arange(B_COL + 200, C - TAIL), 40, replace=False)]))]
    lists = [v.astype(np.int32) for v in lists]
    assert B_COL in lists[0] and C - 1 in lists[1]
    through = np.setdiff1d(w["sampled"], np.concatenate(lists)).astype(np.int32)
    assert past(through)
    eng.median_filter(Y, w["cs"], w["cl"], lists, window, out=X)        # X is no longer needed: the output goes there
    cols = np.unique(np.concatenate(lists + [through])).astype(np.int32)
    Ysm = gather(Y, cols)
    F = eng.median_filter(Ysm, w["cs"], w["cl"], [local(cols, v) for v in lists], window)
    got = gather(X, cols).cpu().numpy()
    assert same_bits(got, F.cpu().numpy()), f"median_filter (window {window}) differs from the small call"
    Yh = Ysm.cpu().numpy()
    pos = local(cols, through)
    assert same_bits(got[pos], Yh[pos]), "cells in no list are not copied through"
    for v in lists:
        p = local(cols, v)
        want = orc.median_filter(np.asfortranarray(Yh[p].T), w["cs"], w["cl"], [np.arange(len(v))], window)
        assert np.array_equal(got[p], want.T), f"median_filter (window {window}) differs from the oracle"
    log(f"median_filter window {window}: {len(cols)} columns ({len(past(cols))} past the boundary, lists in shuffled order) "
        f"equal to the small call and the oracle; {len(through)} cells copied through")


@pytest.mark.parametrize("test", ["wilcoxon", "t"])
def test_mask_non_de(world, test):
    from tests import de_reference as dr
    w = world
    torch, eng, Y, X, refs = w["torch"], w["eng"], w["Y"], w["X"], w["refs"]
    tail = np.arange(C - TAIL, C, dtype=np.int32)
    subs = [tail[:400], tail[400:650], tail[-60:]]
    assert all(len(past(g)) == len(g) for g in subs + refs[1:]) and past(refs[0])
    cv = 1.0
    _, P, A = eng.mask_non_de(Y, refs, subs, test=test, center_val=cv, seed=11, out=X)
    cols = np.unique(np.concatenate(refs + subs + [w["sampled"]])).astype(np.int32)
    Ysm = gather(Y, cols)
    Ym, P2, A2 = eng.mask_non_de(Ysm, [local(cols, g) for g in refs], [local(cols, g) for g in subs], test=test, center_val=cv,
                                 seed=11)
    P, A = P.cpu().numpy(), A.cpu().numpy()
    assert same_bits(P, P2.cpu().numpy()) and same_bits(A, A2.cpu().numpy()), f"mask_non_de ({test}): p differ from the small call"
    assert same_bits(gather(X, cols).cpu().numpy(), Ym.cpu().numpy()), f"mask_non_de ({test}): Y differs from the small call"
    del Ym, P2, A2
    genes = np.unique(np.concatenate([[0, 1, G - 1], w["rng"].choice(G, 5, replace=False)]))
    Yg = Ysm[:, torch.as_tensor(genes, device=Ysm.device).long()].cpu().numpy()
    worst = 0.0
    n_ref = len(refs)
    for gi, g in enumerate(genes):
        for s, sub in enumerate(subs):
            for j, ref in enumerate(refs):
                col = s * n_ref + j
                x, y = Yg[local(cols, ref), gi], Yg[local(cols, sub), gi]
                if test == "wilcoxon":
                    want = dr.wilcox_p(dr.jittered(x, 11, j, int(g), 1e-4, 1e-4),
                                       dr.jittered(y, 11, dr.SUB_KEY + col, int(g), 1e-4, 1e-4))
                else:
                    want = dr.welch_p(x, y)
                got = P[col, g]
                if np.isnan(want):
                    assert np.isnan(got)
                    continue
                err = abs(got - want) / max(abs(want), 1e-300)
                worst = max(worst, err)
                assert err <= 1e-12, (test, g, col, got, want)
    log(f"mask_non_de ({test}): p_raw / p_adj / Y of {len(cols)} columns equal to the small call; {len(genes)} genes x "
        f"{P.shape[0]} pairs against tests/de_reference.py, worst relative error {worst:.2e}")


def test_host_pointer_path(world):
    """api.smooth_block and api.viterbi on a pageable (G, C) Fortran array: the pinned staging ring and the slab loop."""
    w = world
    torch, api = w["torch"], w["api"]
    avail = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    need = 2 * FLOAT_BYTES + STATE_BYTES + (16 << 30)
    if avail < need:
        pytest.skip(f"the host path needs {need / 1e9:.1f} GB of free RAM, the host has {avail / 1e9:.1f} GB")
    for k in ("X", "Y", "S", "mg"):
        w.pop(k, None)
    torch.cuda.empty_cache()
    eng, cs, cl, refs, sampled = w["eng"], w["cs"], w["cl"], w["refs"], w["sampled"]
    X = eng.synth(G, cs, cl, np.arange(C), C, SEED)
    hX = X.cpu().numpy().T                                    # (G, C), Fortran order, pageable
    del X
    torch.cuda.empty_cache()
    hY = api.smooth_block(hX, cs, cl, refs)
    hS = np.empty((G, C), dtype=np.uint8, order="F")
    api.viterbi(hY, cs, cl, w["Pi"], w["delta"], w["mean"], w["sd"], out=hS)
    cols = np.unique(np.concatenate([w["ref_all"], sampled])).astype(np.int32)
    sX = np.asfortranarray(hX[:, cols])
    del hX
    sY = api.smooth_block(sX, cs, cl, [local(cols, g) for g in refs])
    sS = np.empty(sY.shape, dtype=np.uint8, order="F")
    api.viterbi(sY, cs, cl, w["Pi"], w["delta"], w["mean"], w["sd"], out=sS)
    p = local(cols, sampled)
    assert same_bits(hY[:, sampled], sY[:, p]), "api.smooth_block: sampled columns differ from the small call"
    assert same_bits(hS[:, sampled], sS[:, p]), "api.viterbi: sampled columns differ from the small call"
    log(f"host-pointer path: api.smooth_block + api.viterbi on a pageable {G} x {C} array, {len(sampled)} columns "
        f"({len(past(sampled))} past the boundary) equal to the small call")
