"""Size-independent properties of the CUDA path at BASELINE.json's full single-GPU size
(configs[1]: 10 000 cells x 10 000 genes), where the CPU oracle is too slow to be the checker."""
import ctypes as ct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def world():
    import torch

    import bench
    from infercnv_b200 import dist as shard
    from infercnv_b200.device import Engine
    from infercnv_b200.hmm import CNV_LEVELS, get_HMM
    eng = Engine(0)
    G, C = 10000, 10000
    cs, cl = bench.chr_layout(G)
    refs = bench.ref_groups_global(C)
    plan = shard.plan_shards(C, refs, 1)[0]
    X = eng.synth(G, cs, cl, plan.local_cells, C, bench.SEED)
    Pi, delta, _, _ = get_HMM({k: {"mean": m, "sd": s} for k, m, s in zip(CNV_LEVELS, bench.I6_MEAN, bench.I6_SD)}, 1e-6)
    Y, flag = eng.smooth_block(X, cs, cl, plan.local_ref_groups(), plan.ref_sizes, plan.max_chunks)
    torch.cuda.synchronize()
    assert int(flag.item()) == 0
    return dict(torch=torch, eng=eng, G=G, C=C, cs=cs, cl=cl, plan=plan, X=X, Y=Y, Pi=Pi, delta=delta, bench=bench)


def test_full_size_hmm_fast_path_equals_reference_order_arithmetic(world):
    """1e8 state calls: the certified fast path and the reference-order kernel must agree everywhere."""
    w = world
    from infercnv_b200 import api
    torch, eng = w["torch"], w["eng"]
    S_fast, f1 = eng.viterbi(w["Y"], w["cs"], w["cl"], w["Pi"], w["delta"], w["bench"].I6_MEAN, w["bench"].I6_SD)
    torch.cuda.synchronize()
    reruns = api.hmm_rerun_count()
    api.set_hmm_mode("exact")
    try:
        S_exact, f2 = eng.viterbi(w["Y"], w["cs"], w["cl"], w["Pi"], w["delta"], w["bench"].I6_MEAN, w["bench"].I6_SD)
        torch.cuda.synchronize()
    finally:
        api.set_hmm_mode("fast")
    assert int(f1.item()) == 0 and int(f2.item()) == 0
    diff = int((S_fast != S_exact).sum().item())
    print(f"\n[full size] fast vs reference-order: {diff} differing states of {S_fast.numel()}; {reruns} of "
          f"{w['C'] * len(w['cs'])} sequences re-run")
    assert diff == 0
    assert int(S_fast.min().item()) >= 1 and int(S_fast.max().item()) <= 6
    # non-trivial workload: CNV calls exist and neutral dominates
    frac_neutral = float((S_fast == 3).float().mean().item())
    assert 0.5 < frac_neutral < 0.999


def test_cell_permutation_invariance_is_bitwise(world):
    """Cells are independent given the reference means, and the means depend only on the ORDER of the
    reference lists: permuting the columns (and the lists with them) permutes the output bit for bit."""
    w = world
    torch, eng = w["torch"], w["eng"]
    C = w["C"]
    perm = torch.randperm(C, device=w["X"].device, generator=torch.Generator(device=w["X"].device).manual_seed(3))
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(C, device=perm.device)
    Xp = w["X"][perm].contiguous()                      # new column j holds old cell perm[j]
    inv_h = inv.cpu().numpy()
    refs_p = [inv_h[g].astype(np.int32) for g in w["plan"].local_ref_groups()]   # same cells, same list order
    Yp, flag = eng.smooth_block(Xp, w["cs"], w["cl"], refs_p, w["plan"].ref_sizes, w["plan"].max_chunks)
    torch.cuda.synchronize()
    assert int(flag.item()) == 0
    assert bool(torch.equal(Yp, w["Y"][perm]))
    S, _ = eng.viterbi(w["Y"], w["cs"], w["cl"], w["Pi"], w["delta"], w["bench"].I6_MEAN, w["bench"].I6_SD)
    Sp, _ = eng.viterbi(Yp, w["cs"], w["cl"], w["Pi"], w["delta"], w["bench"].I6_MEAN, w["bench"].I6_SD)
    torch.cuda.synchronize()
    assert bool(torch.equal(Sp, S[perm]))


def test_smooth_of_constant_shift_and_median_idempotence(world):
    """Renormalised weights: smooth(x + c) = smooth(x) + c; smooth(const) = const; centring twice = once."""
    w = world
    torch, eng = w["torch"], w["eng"]
    G = w["G"]
    X = torch.log2(w["X"][:512] + 1.0)
    out = torch.empty_like(X)
    out2 = torch.empty_like(X)
    eng.cell_pipeline(X, None, out, w["cs"], w["cl"], False, None, 0.0, 101, 0, None, False)
    eng.cell_pipeline(X + 2.5, None, out2, w["cs"], w["cl"], False, None, 0.0, 101, 0, None, False)
    torch.cuda.synchronize()
    assert float((out2 - out - 2.5).abs().max().item()) < 1e-9
    const = torch.full_like(X, 0.75)
    eng.cell_pipeline(const, None, out2, w["cs"], w["cl"], False, None, 0.0, 101, 0, None, False)
    torch.cuda.synchronize()
    assert float((out2 - 0.75).abs().max().item()) < 1e-12
    # median centring: afterwards every cell's median is (numerically) zero, and a second pass changes nothing
    c1 = torch.empty_like(X)
    c2 = torch.empty_like(X)
    eng.cell_pipeline(out, None, c1, w["cs"], w["cl"], False, None, 0.0, 0, 1, None, False)
    eng.cell_pipeline(c1, None, c2, w["cs"], w["cl"], False, None, 0.0, 0, 1, None, False)
    torch.cuda.synchronize()
    med = torch.median(c1, dim=1).values          # lower median for even G: |.| <= gap to the upper one
    srt = torch.sort(c1, dim=1).values
    mid = 0.5 * (srt[:, G // 2 - 1] + srt[:, G // 2])
    assert float(mid.abs().max().item()) < 1e-15
    assert float((c2 - c1).abs().max().item()) < 1e-15
    del med


def test_smooth_block_output_range_and_reference_centering(world):
    w = world
    torch = w["torch"]
    Y = w["Y"]
    assert bool(torch.isfinite(Y).all())
    assert float(Y.min().item()) > 2.0 ** -3.5 and float(Y.max().item()) < 2.0 ** 3.5   # clamp +-3 then smoothing
    # inside the dead band of the second reference subtraction values are exactly 2^0 (ops.R:1768)
    ref_cols = np.concatenate(w["plan"].local_ref_groups())
    frac_one = float((Y[ref_cols] == 1.0).float().mean().item())
    assert frac_one > 0.0


def test_engine_mean_sd_matches_host_entry_point(world):
    w = world
    from infercnv_b200 import api
    groups = w["plan"].local_ref_groups()
    mu, sg = w["eng"].mean_sd(w["Y"], groups)
    Yh = w["Y"][:1200].cpu().numpy().T                         # (G, 1200) Fortran view; refs are the first 1000 cells
    mu2, sg2 = api.mean_sd(Yh, np.concatenate(groups))
    assert mu == mu2 and sg == sg2
    vals = Yh[:, np.concatenate(groups)]
    assert abs(mu - vals.mean()) < 1e-13 and abs(sg - vals.std(ddof=1)) < 1e-12


def test_median_filter_properties(world):
    """Median of a constant block is the constant; positive scaling commutes with the median."""
    w = world
    torch, eng = w["torch"], w["eng"]
    X = w["Y"][:600].contiguous()
    groups = [np.arange(0, 250), np.arange(250, 600)]
    F1 = eng.median_filter(X, w["cs"], w["cl"], groups, 7)
    F2 = eng.median_filter(X * 4.0, w["cs"], w["cl"], groups, 7)
    const = torch.full_like(X, 1.25)
    F3 = eng.median_filter(const, w["cs"], w["cl"], groups, 7)
    torch.cuda.synchronize()
    assert bool(torch.equal(F2, F1 * 4.0))
    assert bool(torch.equal(F3, const))
    assert float(F1.min().item()) >= float(X.min().item()) and float(F1.max().item()) <= float(X.max().item())


def test_full_size_pairwise_distances_against_an_independent_implementation(world):
    """3000 smoothed cells x 10 000 genes (4.5e6 pairs): the distance kernel against torch's own FP64 `cdist` on the
    same device data (an independent implementation: |a|^2 + |b|^2 - 2 a.b form), in R's "dist" order."""
    w = world
    torch, eng = w["torch"], w["eng"]
    cells = np.arange(2000, 5000, dtype=np.int32)
    d = eng.pairwise_dist(w["Y"], cells)
    torch.cuda.synchronize()
    sub = w["Y"][torch.as_tensor(cells, device=w["Y"].device).long()]
    ref = torch.cdist(sub, sub, compute_mode="donot_use_mm_for_euclid_dist")          # exact difference form
    iu = torch.triu_indices(len(cells), len(cells), offset=1, device=ref.device)
    want = ref[iu[0], iu[1]]                    # pairs (a, b), a < b, by a then b = the strict lower triangle by columns
    err = float(((d - want).abs() / want.clamp_min(1e-300)).max().item())
    print(f"\n[full size] {d.numel()} pairwise distances: max relative deviation from torch.cdist {err:.2e}")
    assert d.numel() == len(cells) * (len(cells) - 1) // 2 and err < 1e-12
    assert float(d.min().item()) > 0.0
