#!/usr/bin/env python
"""TEST INFRASTRUCTURE: the torch-tensor layer (infercnv_b200/device.py: Engine) and the multi-rank path driven on the
CPU - CPU tensors stand in for device tensors (the emulated library's "device memory" is host memory), gloo stands in
for NCCL, and the kernels run from their own source under tests/host/emu/cuda_runtime.h.

    python tests/host/engine_emulated.py            single process: Engine vs the oracle
    python tests/host/engine_emulated.py --world 2  two gloo ranks: sharded smooth block + HMM + i3 mu/sigma + region
                                                    consensus must be BITWISE equal to the single-rank run

The same checks as tests/test_gpu_widen_regions.py::test_device_resident_* and tools/check_multigpu.py make on GPUs."""
import ctypes as ct
import os
import socket
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def make_engine():
    """An Engine whose tensors live on the CPU and whose library is the emulated build."""
    import build_emu
    from infercnv_b200 import _lib
    _lib.LIB_PATH = build_emu.build()
    torch.cuda.set_device = lambda d: None
    torch.cuda.synchronize = lambda *a, **k: None
    torch.cuda.current_stream = lambda *a, **k: types.SimpleNamespace(cuda_stream=1)
    from infercnv_b200 import device
    device._stream_ptr = lambda: ct.c_void_p(1)          # any non-NULL handle: the emulation has no streams
    eng = device.Engine(0)
    eng.tdev = torch.device("cpu")
    return eng


I6_MEAN = np.array([0.41234766, 0.84075773, 1.01693983, 1.12238786, 1.23842619, 1.44298781])
I6_SD = np.array([0.028893, 0.164549, 0.105553, 0.190574, 0.244093, 0.290072])
LENS = np.array([180, 75, 1, 40, 2, 110], dtype=np.int32)
CS = np.concatenate([[0], np.cumsum(LENS)[:-1]]).astype(np.int32)
G = int(LENS.sum())
SEED = 20260923


def single():
    from oracle import oracle as orc
    from oracle import regions as orr
    eng = make_engine()
    C = 70
    refs = [np.arange(0, 9), np.arange(9, 14)]
    X = eng.synth(G, CS, LENS, np.arange(C), C, SEED)
    Y, flag = eng.smooth_block(X, CS, LENS, refs)
    Xh = np.asfortranarray(X.numpy().T)
    want = orc.smooth_block(Xh, CS, LENS, refs)
    rel = float(np.max(np.abs(Y.numpy().T - want) / np.abs(want)))
    assert rel < 1e-11 and int(flag.item()) == 0, rel
    # re-using pass 1's reference columns in pass 2 (the default when they are the leading columns) changes no bit
    assert eng.reuse_reference_pass
    eng.reuse_reference_pass = False
    Y_full, _ = eng.smooth_block(X, CS, LENS, refs)
    eng.reuse_reference_pass = True
    assert torch.equal(Y, Y_full)
    # a strided view (column stride G + 1, G even): aligned columns take the bulk copy, the others the element-wise load,
    # alternating inside each CTA's persistent loop and its prefetch of the next cell - same bits as the contiguous matrix
    wide = torch.zeros((C, G + 1), dtype=torch.float64)
    wide[:, :G] = X
    assert G % 2 == 0 and wide[:, :G].stride(0) == G + 1
    Y_wide, flag_w = eng.smooth_block(wide[:, :G], CS, LENS, refs)
    assert torch.equal(Y_wide, Y) and int(flag_w.item()) == 0
    b = tuple(torch.from_numpy(np.ascontiguousarray(v)) for v in (np.full(G, 0.2), np.full(G, 0.6), np.full(G, 0.4)))
    cols = torch.from_numpy(np.array([69, 68, 3, 3, 0, 41, 0, 2], dtype=np.int32))     # pass 1's form: any order, repeats
    outs = []
    for Xin in (wide[:, :G], X):
        Yc = torch.empty((len(cols), G), dtype=torch.float64)
        eng.cell_pipeline(Xin, cols, Yc, CS, LENS, True, b, 3.0, 101, 1, b, True)
        outs.append(Yc)
    assert torch.equal(outs[0], outs[1])
    Y_scattered, _ = eng.smooth_block(X, CS, LENS, [np.array([3, 50, 7]), np.array([11, 60])])      # not leading: full pipeline
    want2 = orc.smooth_block(Xh, CS, LENS, [np.array([3, 50, 7]), np.array([11, 60])])
    assert float(np.max(np.abs(Y_scattered.numpy().T - want2) / np.abs(want2))) < 1e-11
    Pi, delta = orc.hmm_params(6)
    S, f2 = eng.viterbi(Y, CS, LENS, Pi, delta, I6_MEAN, I6_SD)
    want_s = orc.viterbi_matrix(np.asfortranarray(Y.numpy().T), CS, LENS, Pi, delta, I6_MEAN, I6_SD)
    assert np.array_equal(S.numpy().T, want_s) and int(f2.item()) == 0
    # the slab-pipelined host path (sequential on the CPU) is the same computation
    hY, hS = torch.empty_like(X), torch.empty((C, G), dtype=torch.uint8)
    fl = eng.smooth_hmm_host(X.clone(), hY, hS, torch.empty_like(X), torch.empty_like(X), torch.empty((C, G), dtype=torch.uint8), CS,
                             LENS, refs, None, None, Pi, delta, I6_MEAN, I6_SD, slab_cells=16)
    assert torch.equal(hY, Y) and torch.equal(hS, S) and all(int(f.item()) == 0 for f in fl)
    mu, sg = eng.mean_sd(Y, refs)
    mu_o, sg_o = orc.mean_sd_over_cells(np.asfortranarray(Y.numpy().T), np.concatenate(refs))
    assert abs(mu - mu_o) < 1e-14 and abs(sg - sg_o) < 1e-13
    # device-resident states -> consensus -> regions, contiguous and strided (column stride > G)
    Sh = np.asfortranarray(S.numpy().T)
    gs, ge = np.arange(G) * 10.0, np.arange(G) * 10.0 + 95
    wide = torch.zeros((C, G + 4), dtype=torch.uint8)
    wide[:, :G] = S
    groups = [np.arange(0, 40), np.arange(40, 69), np.array([7])]
    for dS in (S, wide[:, :G]):
        cons = eng.state_consensus(dS, groups)
        want_c = np.stack([orr.state_consensus(Sh, g) for g in groups], axis=0)
        assert np.array_equal(cons.numpy(), want_c)
        got, ref = eng.cnv_regions(cons, CS, LENS, gs, ge), orr.cnv_regions(want_c.T, CS, LENS, gs, ge)
        assert all(np.array_equal(got[k], ref[k]) for k in ref)
        cells = [5, 0, 69, 33]
        got, ref = eng.cnv_regions(dS, CS, LENS, gs, ge, cols=cells), orr.cnv_regions(Sh[:, cells], CS, LENS, gs, ge)
        assert all(np.array_equal(got[k], ref[k]) for k in ref)
    sds_g = np.concatenate([I6_SD * len(g) ** -0.5 for g in groups])
    Sg, fg = eng.viterbi_groups(Y, CS, LENS, Pi, delta, I6_MEAN, sds_g, groups)
    want_g = orc.viterbi_matrix(np.asfortranarray(Y.numpy().T), CS, LENS, Pi, delta, I6_MEAN, sds_g, groups=groups)
    got_g = Sg.numpy().T.astype(np.int32)
    got_g[got_g == 255] = -1
    assert np.array_equal(got_g, want_g) and int(fg.item()) == 0, "group-mode HMM differs from the oracle"
    F = eng.median_filter(Y, CS, LENS, groups[:2], 7)
    want_f = orc.median_filter(np.asfortranarray(Y.numpy().T), CS, LENS, groups[:2], 7)
    assert np.allclose(F.numpy().T, want_f, rtol=0, atol=1e-15)
    # pairwise distances of a shuffled subset of the local cells on "device" tensors (Engine.pairwise_dist)
    sub = np.random.default_rng(3).permutation(Y.shape[0])[:37].astype(np.int32)
    D = eng.pairwise_dist(Y, sub)
    assert np.allclose(D.numpy(), orc.pairwise_dist(np.asfortranarray(Y.numpy().T), sub), rtol=1e-13, atol=0)
    print(f"engine (emulated, 1 rank): smooth block rel err {rel:.1e}, {S.numel()} states identical, consensus / regions / "
          f"median filter / pairwise distances equal to the oracle")


def rank_main(rank, world, port):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from infercnv_b200 import dist as shard
    from oracle import oracle as orc
    eng = make_engine()
    C_total = 61 * world + 5
    refs = [np.arange(0, 70), np.arange(80, 80 + 37)]                 # 3 and 2 chunks of 32: cut differently per world
    refs = [r[r < C_total] for r in refs]
    plan = shard.plan_shards(C_total, refs, world)[rank]
    X = eng.synth(G, CS, LENS, plan.local_cells, C_total, SEED)
    Y, f = eng.smooth_block(X, CS, LENS, plan.local_ref_groups(), plan.ref_sizes, plan.max_chunks)
    Pi, delta = orc.hmm_params(6)
    S, f2 = eng.viterbi(Y, CS, LENS, Pi, delta, I6_MEAN, I6_SD)
    Cl = X.shape[0]
    hY, hS = torch.empty_like(X), torch.empty((Cl, G), dtype=torch.uint8)
    eng.smooth_hmm_host(X.clone(), hY, hS, torch.empty_like(X), torch.empty_like(X), torch.empty((Cl, G), dtype=torch.uint8), CS, LENS,
                        plan.local_ref_groups(), plan.ref_sizes, plan.max_chunks, Pi, delta, I6_MEAN, I6_SD, slab_cells=24)
    assert torch.equal(hY, Y) and torch.equal(hS, S), "slab-pipelined host path differs from smooth_block + viterbi"
    mu_d, sg_d = eng.mean_sd(Y, plan.local_ref_groups())
    obs_global = [np.arange(int(0.3 * C_total), int(0.6 * C_total)), np.arange(int(0.6 * C_total), C_total)]
    pos_of = {int(c): i for i, c in enumerate(plan.local_cells)}
    obs_local = [np.array([pos_of[int(c)] for c in g if int(c) in pos_of], dtype=np.int32) for g in obs_global]
    cons_d = eng.state_consensus(S, obs_local)
    assert int(f.item()) == 0 and int(f2.item()) == 0
    # median filter on the shard: the reference groups are cut over the ranks (halos of 4 list entries from the neighbours),
    # the other cells form one list per rank
    Yext = torch.zeros((Cl + 8 * len(refs), G), dtype=torch.float64)
    Yext[:Cl] = Y
    n_ref_local = sum(len(g) for g in plan.local_ref_groups())
    own = [np.arange(n_ref_local, Cl, dtype=np.int32)] if Cl > n_ref_local else []
    Fd = eng.median_filter_sharded(Yext, Cl, own, plan.local_ref_groups(), CS, LENS, 7)[:Cl]
    # group-mode HMM ("samples"): every cell in one of three groups, each cut over the ranks at chunk boundaries
    all_groups = refs + [np.setdiff1d(np.arange(C_total), np.concatenate(refs))]
    gplan = shard.plan_shards(C_total, all_groups, world)[rank]
    Xg = eng.synth(G, CS, LENS, gplan.local_cells, C_total, SEED)
    sds_g = np.concatenate([I6_SD * len(g) ** -0.5 for g in all_groups])
    Sgd, _ = eng.viterbi_groups(Xg, CS, LENS, Pi, delta, I6_MEAN + 1.0, sds_g, gplan.local_ref_groups(), gplan.ref_sizes, gplan.max_chunks)
    n_local = torch.tensor([X.shape[0]])
    sizes = [torch.zeros_like(n_local) for _ in range(world)]
    dist.all_gather(sizes, n_local)
    nmax = int(max(s.item() for s in sizes))
    Yp = torch.zeros((nmax, G), dtype=torch.float64); Yp[: X.shape[0]] = Y
    Sp = torch.zeros((nmax, G), dtype=torch.uint8); Sp[: X.shape[0]] = S
    Fp = torch.zeros((nmax, G), dtype=torch.float64); Fp[: X.shape[0]] = Fd
    Ys = [torch.zeros_like(Yp) for _ in range(world)]
    Ss = [torch.zeros_like(Sp) for _ in range(world)]
    Fs = [torch.zeros_like(Fp) for _ in range(world)]
    ng = torch.tensor([Xg.shape[0]])
    gsz = [torch.zeros_like(ng) for _ in range(world)]
    dist.all_gather(gsz, ng)
    gmax = int(max(v.item() for v in gsz))
    Gp = torch.zeros((gmax, G), dtype=torch.uint8); Gp[: Xg.shape[0]] = Sgd
    Gs = [torch.zeros_like(Gp) for _ in range(world)]
    dist.all_gather(Gs, Gp)
    dist.all_gather(Ys, Yp)
    dist.all_gather(Ss, Sp)
    dist.all_gather(Fs, Fp)
    ok = True
    if rank == 0:
        plans = shard.plan_shards(C_total, refs, world)
        p1 = shard.plan_shards(C_total, refs, 1)[0]
        X1 = eng.synth(G, CS, LENS, p1.local_cells, C_total, SEED)
        eng.collective = False
        Y1, _ = eng.smooth_block(X1, CS, LENS, p1.local_ref_groups(), p1.ref_sizes, [(len(g) + 31) // 32 for g in refs])
        S1, _ = eng.viterbi(Y1, CS, LENS, Pi, delta, I6_MEAN, I6_SD)
        mu_1, sg_1 = eng.mean_sd(Y1, p1.local_ref_groups())
        pos1 = {int(c): i for i, c in enumerate(p1.local_cells)}
        lists1 = [np.array([pos1[int(c)] for c in p.other_cells], dtype=np.int32) for p in plans if len(p.other_cells)] + \
            [np.array([pos1[int(c)] for c in g], dtype=np.int32) for g in refs]
        F1 = eng.median_filter(Y1, CS, LENS, lists1, 7)
        bad_y = bad_s = bad_f = 0
        for r, p in enumerate(plans):
            idx = torch.tensor([pos1[int(c)] for c in p.local_cells])
            bad_y += int((Ys[r][: len(idx)] != Y1[idx]).sum().item())
            bad_s += int((Ss[r][: len(idx)] != S1[idx]).sum().item())
            bad_f += int((Fs[r][: len(idx)] != F1[idx]).sum().item())
        cons_1 = eng.state_consensus(S1, [np.array([pos1[int(c)] for c in g], dtype=np.int32) for g in obs_global])
        bad_c = int((cons_1 != cons_d).sum().item())
        g1 = shard.plan_shards(C_total, all_groups, 1)[0]
        Xg1 = eng.synth(G, CS, LENS, g1.local_cells, C_total, SEED)
        Sg1, _ = eng.viterbi_groups(Xg1, CS, LENS, Pi, delta, I6_MEAN + 1.0, sds_g, g1.local_ref_groups())
        posg = {int(c): i for i, c in enumerate(g1.local_cells)}
        bad_g = 0
        for r, p in enumerate(shard.plan_shards(C_total, all_groups, world)):
            idx = torch.tensor([posg[int(c)] for c in p.local_cells])
            bad_g += int((Gs[r][: len(idx)] != Sg1[idx]).sum().item())
        ok = bad_y == 0 and bad_s == 0 and bad_f == 0 and bad_c == 0 and bad_g == 0 and mu_d == mu_1 and sg_d == sg_1
        print(f"engine (emulated, {world} gloo ranks, {C_total} cells): values differing from the 1-rank run {bad_y}, states "
              f"{bad_s}, group-mode HMM states {bad_g}, median filter (halo exchange) {bad_f}, consensus {bad_c}, mu/sigma {'equal' if (mu_d, sg_d) == (mu_1, sg_1) else 'DIFFER'} -> "
              f"{'BITWISE EQUAL' if ok else 'MISMATCH'}")
    flag = torch.tensor([1 if ok else 0])
    dist.broadcast(flag, 0)
    dist.barrier()
    dist.destroy_process_group()
    if not int(flag.item()):
        sys.exit(1)


if __name__ == "__main__":
    if "--world" in sys.argv:
        import torch.multiprocessing as mp
        world = int(sys.argv[sys.argv.index("--world") + 1])
        import build_emu
        build_emu.build()                      # once, before the ranks race for it
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
        s.close()
        mp.spawn(rank_main, args=(world, port), nprocs=world)
    else:
        single()
