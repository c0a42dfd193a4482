"""The stages of the non-DE mask on their own (icnv_dev_de_pack_f64, icnv_dev_de_place_f64, icnv_dev_de_slab_tests_f64,
icnv_dev_de_bh_mask_f64), driven in one process the way Engine.mask_non_de_sharded drives them across ranks: every "rank"
packs its listed cells for every rank's gene range, the blocks are exchanged as all_to_all_single would exchange them, each
rank places what it received and tests its genes in sub-slabs, and every rank runs BH on the whole p and masks its own cells.
p_raw, p_adj and Y must equal icnv_mask_non_de_f64 on the whole matrix byte for byte.  Gene counts and sub-slabs are not
multiples of 32, so the pack's transpose tiles, the exchange and the slabs all end mid-tile.  Under the host emulation
(tests/test_de_stages_emulated.py) a few genes of the small cases run."""
import os

import numpy as np
import pytest

from infercnv_b200 import _lib, api
from infercnv_b200.api import DE_RULES, DE_TESTS, groups_to_csr
from tests import de_shards

pytestmark = pytest.mark.gpu
EMULATED = "_emu" in os.path.basename(_lib.LIB_PATH)


@pytest.fixture(scope="module", autouse=True)
def _init():
    api.init(0)


class Mem:
    """device buffers: torch CUDA tensors on the GPU, host arrays under the emulation (its device memory is host memory)"""

    def __init__(self):
        if EMULATED:
            self.stream = None
        else:
            from infercnv_b200.device import _stream_ptr
            self.stream = _stream_ptr()

    def up(self, a):
        a = np.ascontiguousarray(a)
        if EMULATED:
            return a, a.ctypes.data
        import torch
        t = torch.as_tensor(a).cuda()
        return t, t.data_ptr()

    def empty(self, n, dtype=np.float64):
        return self.up(np.full(max(int(n), 1), np.nan if dtype == np.float64 else 0, dtype=dtype))

    def down(self, t):
        if EMULATED:
            return t
        import torch
        torch.cuda.synchronize()
        return t.cpu().numpy()


def by_stages(X, shards, refs, subs, slab, center_val, test="wilcoxon", p_val_thresh=0.05, rule="any", jitter_mean=1e-4,
              jitter_sd=1e-4, seed=0):
    lib, mem = _lib.load(), Mem()
    G = X.shape[0]
    world, n_ref, n_sub = len(shards), len(refs), len(subs)
    npair, ng = n_ref * n_sub, n_ref + n_sub
    all_lens = np.asarray([[len(g) for g in sh[2] + sh[3]] for sh in shards], dtype=np.int64).reshape(world, ng)
    goff = np.concatenate([[0], np.cumsum(all_lens.sum(axis=0))]).astype(np.int64)
    T = int(goff[-1])
    m = np.ascontiguousarray(all_lens.sum(axis=1), dtype=np.int64)
    gb = [G * d // world for d in range(world + 1)]
    n_max = max(gb[d + 1] - gb[d] for d in range(world))
    locals_ = [mem.up(np.asfortranarray(X[:, sh[0]:sh[1]]).ravel(order="F")) for sh in shards]
    cols = [mem.up(np.concatenate(sh[2] + sh[3]).astype(np.int32) if m[r] else np.zeros(1, np.int32))
            for r, sh in enumerate(shards)]
    tags = np.concatenate([goff[k] + all_lens[:q, k].sum() + np.arange(all_lens[q, k]) for q in range(world)
                           for k in range(ng)]).astype(np.int32)
    d_tags = mem.up(tags)
    flag = mem.up(np.zeros(1, np.int32))
    P, p_ptr = mem.empty(npair * G)
    roff, soff = goff[:n_ref + 1].astype(np.int32), (goff[n_ref:] - goff[n_ref]).astype(np.int32)
    test_c, rule_c = DE_TESTS[test], DE_RULES[rule]
    if npair:
        for s0 in range(0, n_max, slab):
            lo = np.asarray([min(gb[d] + s0, gb[d + 1]) for d in range(world)], dtype=np.int64)
            hi = np.asarray([min(gb[d] + s0 + slab, gb[d + 1]) for d in range(world)], dtype=np.int64)
            sends = []
            for r, sh in enumerate(shards):
                buf, ptr = mem.empty(int((hi - lo).sum()) * m[r])
                _lib.check(lib.icnv_dev_de_pack_f64(locals_[r][1], G, cols[r][1], int(m[r]), world, lo.ctypes.data,
                                                    hi.ctypes.data, ptr, flag[1], mem.stream))
                sends.append(mem.down(buf))
            for d in range(world):
                n = int(hi[d] - lo[d])
                if n == 0:
                    continue
                # what all_to_all_single hands rank d: source q's block for d, sources in rank order
                recv = np.concatenate([sends[q][int(((hi - lo)[:d]).sum() * m[q]):][:n * int(m[q])] for q in range(world)])
                R, r_ptr = mem.up(recv)
                Z, z_ptr = mem.empty(n * T)
                _lib.check(lib.icnv_dev_de_place_f64(r_ptr, n, world, m.ctypes.data, d_tags[1], T, z_ptr, mem.stream))
                _lib.check(lib.icnv_dev_de_slab_tests_f64(z_ptr, T, int(lo[d]), n, roff.ctypes.data, n_ref, soff.ctypes.data,
                                                          n_sub, test_c, jitter_mean, jitter_sd, seed, p_ptr + 8 * int(lo[d]), G,
                                                          mem.stream))
    bad = int(mem.down(flag[0])[0])
    sub_size = np.ascontiguousarray(goff[n_ref + 1:] - goff[n_ref:-1], dtype=np.int32) if n_sub else np.zeros(1, np.int32)
    Ys, A = [], None
    for r, sh in enumerate(shards):
        C = sh[1] - sh[0]
        Yb, y_ptr = mem.empty(C * G)
        Ab, a_ptr = mem.empty(npair * G)
        ridx = np.concatenate(sh[2]).astype(np.int32) if sum(len(g) for g in sh[2]) else np.zeros(1, np.int32)
        so, si = groups_to_csr(sh[3])
        _lib.check(lib.icnv_dev_de_bh_mask_f64(p_ptr if npair else None, G, n_ref, n_sub, sub_size.ctypes.data, p_val_thresh,
                                               a_ptr if npair else None, locals_[r][1], G, y_ptr, G, C, ridx.ctypes.data,
                                               sum(len(g) for g in sh[2]), so.ctypes.data, si.ctypes.data, rule_c, center_val,
                                               mem.stream))
        Ys.append(mem.down(Yb)[:C * G].reshape(G, C, order="F"))
        a = mem.down(Ab)[:npair * G]
        assert A is None or a.tobytes() == A.tobytes(), "BH differs between ranks"
        A = a
    Y = np.concatenate(Ys, axis=1)
    return Y, mem.down(P)[:npair * G].reshape(npair, G).T, A.reshape(npair, G).T, bad


CASES = de_shards.CASES[:2] + de_shards.CASES[-1:] if EMULATED else de_shards.CASES


@pytest.mark.parametrize("world,slab", [(1, 7), (2, 64), (3, 5)] if EMULATED else [(1, 1000), (2, 7), (3, 5), (4, 32), (5, 13)])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_stages_equal_one_call(case, world, slab):
    name, G, ref_sizes, sub_sizes, kw, mk = case
    if EMULATED:
        G = 13
    X, shards, refs, subs = de_shards.make_case(world, G, ref_sizes, sub_sizes, seed=world * 100 + len(name),
                                                 empty_rank=world - 1 if world > 2 else None, **mk)
    cv = float(np.mean(X))
    want = api.mask_non_de_genes(X, refs, subs, center_val=cv, **kw)
    Y, P, A, bad = by_stages(X, shards, refs, subs, slab, cv, **kw)
    assert bad == 0
    assert P.tobytes() == want[1].tobytes(), "p_raw differs"
    assert A.tobytes() == want[2].tobytes(), "p_adj differs"
    assert Y.tobytes() == np.asfortranarray(want[0]).tobytes(), "Y differs"


def test_pack_reports_a_non_finite_listed_value():
    X, shards, refs, subs = de_shards.make_case(2, 13, [20], [10], seed=1)
    Z = X.copy()
    Z[5, refs[0][0]] = np.inf
    _, _, _, bad = by_stages(Z, shards, refs, subs, 4, 0.0)
    assert bad == 1
    c0, c1, ref_local, sub_local = shards[1]
    unlisted = sorted(set(range(c1 - c0)) - set(np.concatenate(ref_local + sub_local).tolist()))
    Z = X.copy()
    Z[5, c0 + unlisted[0]] = np.nan           # a cell of rank 1 listed nowhere
    _, _, _, bad = by_stages(Z, shards, refs, subs, 4, 0.0)
    assert bad == 0
