"""torch-tensor wrappers of the device-pointer C ABI (icnv_dev_*), used by the benchmark and the
multi-GPU driver.  torch is plumbing only (device memory, streams, torch.distributed); every
kernel is in libinfercnv_b200.so.

A device matrix is a torch.float64 tensor of shape (C, G), C-contiguous: that is exactly R's
column-major G x C (a cell's genes contiguous).
"""
from __future__ import annotations

import ctypes as ct
import os

import numpy as np
import torch

from . import _lib, dist as shard
from .api import _fetch_snn, _i32, groups_to_csr

_E_NONFINITE = -5   # ICNV_E_NONFINITE


def _stream_ptr():
    """torch's current stream as the `void *stream` of the device ABI.  torch's default stream is
    the legacy NULL stream (handle 0), which the ABI reserves for "the library's own stream": pass
    cudaStreamLegacy (handle 0x1) for it instead, so our launches stay ordered with torch's ops."""
    h = torch.cuda.current_stream().cuda_stream
    return ct.c_void_p(h if h else 1)


class Engine:
    """One per process / GPU."""

    def __init__(self, device: int = 0):
        self.lib = _lib.load()
        self.device = int(device)
        torch.cuda.set_device(self.device)
        _lib.check(self.lib.icnv_init(self.device))
        self.tdev = torch.device("cuda", self.device)
        self.timing = None   # when set to a list, smooth_block appends (name, start_event, end_event)
        self.collective = True   # False: never enter a collective even if a process group exists
        # pass 2 re-uses pass 1's reference columns instead of recomputing them (ICNV_REF_REUSE=0 turns it off)
        self.reuse_reference_pass = os.environ.get("ICNV_REF_REUSE", "1") != "0"
        self._plan_cache = {}
        self._T = None

    # ---- process-group plumbing -------------------------------------------------------------------------------------
    def _world(self) -> int:
        import torch.distributed as tdist
        return tdist.get_world_size() if (self.collective and tdist.is_available() and tdist.is_initialized()) else 1

    def _all_gather(self, out: torch.Tensor, part: torch.Tensor) -> None:
        """out[(world,) + part.shape] <- every rank's `part`.  NCCL: one ncclAllGather on torch's current stream over
        NVLink.  Any other backend (gloo: several ranks sharing one GPU in the tests, or CPU-only plumbing tests) goes
        through host memory - same values, same order."""
        import torch.distributed as tdist
        if tdist.get_backend() == "nccl":
            tdist.all_gather_into_tensor(out, part)
            return
        host = part.detach().cpu().contiguous()
        parts = [torch.empty_like(host) for _ in range(tdist.get_world_size())]
        tdist.all_gather(parts, host)
        out.copy_(torch.stack(parts).to(out.device))

    def _all_gather_list(self, t: torch.Tensor):
        """every rank's `t` (same shape on all ranks) as a list in rank order"""
        import torch.distributed as tdist
        world = tdist.get_world_size()
        if tdist.get_backend() == "nccl":
            parts = [torch.empty_like(t) for _ in range(world)]
            tdist.all_gather(parts, t)
            return parts
        host = t.detach().cpu().contiguous()
        parts = [torch.empty_like(host) for _ in range(world)]
        tdist.all_gather(parts, host)
        return [x.to(t.device) for x in parts]

    def _all_reduce_sum(self, t: torch.Tensor) -> None:
        import torch.distributed as tdist
        if tdist.get_backend() == "nccl":
            tdist.all_reduce(t, op=tdist.ReduceOp.SUM)
            return
        host = t.detach().cpu().contiguous()
        tdist.all_reduce(host, op=tdist.ReduceOp.SUM)
        t.copy_(host.to(t.device))

    # ---- data ---------------------------------------------------------------------------------------
    def synth(self, G, chr_start, chr_len, cells_global, C_total, seed) -> torch.Tensor:
        """Synthetic depth-normalised expression for the given GLOBAL cell indices (runs of
        consecutive indices are generated with one launch each)."""
        cells_global = np.asarray(cells_global, dtype=np.int64)
        cs, cl = _i32(chr_start), _i32(chr_len)
        X = torch.empty((len(cells_global), G), dtype=torch.float64, device=self.tdev)
        if len(cells_global) == 0:
            return X
        breaks = np.flatnonzero(np.diff(cells_global) != 1) + 1
        starts = np.concatenate([[0], breaks])
        ends = np.concatenate([breaks, [len(cells_global)]])
        for s, e in zip(starts, ends):
            ptr = X.data_ptr() + int(s) * G * 8
            _lib.check(self.lib.icnv_dev_synth_f64(ptr, G, int(cells_global[s]), int(e - s), int(C_total), cs.ctypes.data,
                                                   cl.ctypes.data, len(cs), ct.c_uint64(seed), _stream_ptr()))
        return X

    # ---- building blocks ----------------------------------------------------------------------------
    def group_partial_sums(self, X: torch.Tensor, cells: torch.Tensor, apply_log: bool) -> torch.Tensor:
        """(n_chunks, G) partial sums over chunks of CHUNK list entries (fixed order)."""
        n = int(cells.numel())
        G = X.shape[1]
        n_chunks = (n + shard.CHUNK - 1) // shard.CHUNK
        out = torch.empty((n_chunks, G), dtype=torch.float64, device=self.tdev)
        if n:
            _lib.check(self.lib.icnv_dev_group_partial_sums_f64(X.data_ptr(), G, X.stride(0), cells.data_ptr(), n,
                                                                shard.CHUNK, int(bool(apply_log)), out.data_ptr(),
                                                                _stream_ptr()))
        return out

    def combine_partials(self, partial: torch.Tensor, count: int) -> torch.Tensor:
        G = partial.shape[1]
        out = torch.empty(G, dtype=torch.float64, device=self.tdev)
        _lib.check(self.lib.icnv_dev_combine_partials_f64(partial.data_ptr(), G, partial.shape[0], int(count),
                                                          out.data_ptr(), _stream_ptr()))
        return out

    def bounds(self, means: torch.Tensor):
        """means: (n_grp, G) -> lo, hi, mid (each G)."""
        n_grp, G = means.shape
        lo, hi, mid = (torch.empty(G, dtype=torch.float64, device=self.tdev) for _ in range(3))
        _lib.check(self.lib.icnv_dev_bounds_from_means_f64(means.data_ptr(), G, n_grp, lo.data_ptr(), hi.data_ptr(),
                                                           mid.data_ptr(), _stream_ptr()))
        return lo, hi, mid

    def cell_pipeline(self, X, cols, Y, chr_start, chr_len, apply_log, b1, threshold, window, center, b2, apply_exp2,
                      use_bounds=True, err_flag=None):
        G = X.shape[1]
        cs, cl = _i32(chr_start), _i32(chr_len)
        n_cols = int(cols.numel()) if cols is not None else X.shape[0]

        def sel(b):
            if b is None:
                return None, None, None
            lo, hi, mid = b
            return (lo.data_ptr(), hi.data_ptr(), None) if use_bounds else (None, None, mid.data_ptr())

        lo1, hi1, mid1 = sel(b1)
        lo2, hi2, mid2 = sel(b2)
        _lib.check(self.lib.icnv_dev_cell_pipeline_f64(
            X.data_ptr(), G, X.stride(0), cols.data_ptr() if cols is not None else None, n_cols, Y.data_ptr(),
            Y.stride(0), cs.ctypes.data, cl.ctypes.data, len(cs), int(bool(apply_log)), lo1, hi1, mid1, float(threshold),
            int(window), int(center), lo2, hi2, mid2, int(bool(apply_exp2)),
            err_flag.data_ptr() if err_flag is not None else None, _stream_ptr()))

    # ---- the hot path ---------------------------------------------------------------------------------------
    def _reference_bounds(self, X, chr_start, chr_len, ref_groups_local, ref_sizes, max_chunks, apply_log, threshold, window,
                          use_bounds, flag):
        """The two reference-mean steps of the smooth block (ops.R:1678, run() steps 8 and 12): bounds b1 of the log
        values, pass 1 of the cell pipeline over this rank's reference cells (-> T, centred and smoothed), bounds b2 of T.
        Only the reference columns of X are read.  Returns (b1, b2, T, n_ref, ref_leading)."""
        C, G = X.shape
        ref_groups_local = [np.asarray(g, dtype=np.int32) for g in ref_groups_local]
        n_grp = len(ref_groups_local)
        if ref_sizes is None:
            ref_sizes = [len(g) for g in ref_groups_local]
        if max_chunks is None:
            max_chunks = [(len(g) + shard.CHUNK - 1) // shard.CHUNK for g in ref_groups_local]
        key = (tuple(g.tobytes() for g in ref_groups_local), C)
        cached = self._plan_cache.get(key)
        if cached is None:       # device copies of the index lists are built once per partition, not per call
            d_groups = [torch.from_numpy(g).to(self.tdev) for g in ref_groups_local]
            t_lists, pos = [], 0
            for g in ref_groups_local:
                t_lists.append(torch.arange(pos, pos + len(g), dtype=torch.int32, device=self.tdev))
                pos += len(g)
            all_ref = torch.cat(d_groups) if pos else None
            self._plan_cache.clear()
            cached = self._plan_cache[key] = (d_groups, t_lists, all_ref)
        d_groups, t_lists, all_ref = cached

        world = self._world()
        tot = int(sum(max_chunks)) if world > 1 else int(sum((len(g) + shard.CHUNK - 1) // shard.CHUNK for g in ref_groups_local))
        rows = [0]
        for k in range(n_grp):
            rows.append(rows[-1] + (int(max_chunks[k]) if world > 1 else (len(ref_groups_local[k]) + shard.CHUNK - 1) // shard.CHUNK))
        row_off = np.asarray(rows, dtype=np.int32)
        counts = np.asarray([int(v) for v in ref_sizes], dtype=np.int64)
        # persistent exchange buffers: every group's chunk sums are written straight into this rank's block of `packed`
        # (rows past a group's local chunk count are never written and stay zero), ONE all-gather per reference-mean step
        # carries them, and one kernel turns the gathered rows into the bounds - no per-step torch ops in between
        bkey = (G, tot, world, tuple(int(v) for v in row_off), tuple(len(g) for g in ref_groups_local))   # stale rows would poison the padding
        if getattr(self, "_xbuf_key", None) != bkey:
            self._xbuf_key = bkey
            self._packed = torch.zeros((max(tot, 1), G), dtype=torch.float64, device=self.tdev)
            self._gathered = torch.empty((world, max(tot, 1), G), dtype=torch.float64, device=self.tdev) if world > 1 else None
            self._bounds = [torch.empty((3, G), dtype=torch.float64, device=self.tdev) for _ in range(2)]

        def group_bounds(src, lists, log, slot):
            for k in range(n_grp):
                n = int(lists[k].numel())
                if n:
                    _lib.check(self.lib.icnv_dev_group_partial_sums_f64(
                        src.data_ptr(), G, src.stride(0), lists[k].data_ptr(), n, shard.CHUNK, int(bool(log)),
                        self._packed.data_ptr() + 8 * G * int(row_off[k]), _stream_ptr()))
            part = self._packed
            if world > 1:
                self._all_gather(self._gathered, self._packed)
                part = self._gathered
            b = self._bounds[slot]
            _lib.check(self.lib.icnv_dev_bounds_from_partials_f64(part.data_ptr(), G, world, max(tot, 1), n_grp,
                                                                  row_off.ctypes.data, counts.ctypes.data, b[0].data_ptr(),
                                                                  b[1].data_ptr(), b[2].data_ptr(), _stream_ptr()))
            return b[0], b[1], b[2]

        b1 = group_bounds(X, d_groups, apply_log, 0)
        # pass 1: reference cells only, up to the median centring
        n_ref = int(sum(len(g) for g in ref_groups_local))
        ref_leading = n_ref > 0 and np.array_equal(np.concatenate(ref_groups_local), np.arange(n_ref))
        if self._T is None or self._T.shape != (max(n_ref, 1), G):
            self._T = torch.empty((max(n_ref, 1), G), dtype=torch.float64, device=self.tdev)
        T = self._T
        if n_ref:
            self.cell_pipeline(X, all_ref, T, chr_start, chr_len, apply_log, b1, threshold, window, 1, None, False,
                               use_bounds, flag)
        b2 = group_bounds(T, t_lists, False, 1)
        return b1, b2, T, n_ref, ref_leading

    def smooth_block(self, X, chr_start, chr_len, ref_groups_local, ref_sizes=None, max_chunks=None, apply_log=True,
                     threshold=3.0, window=101, use_bounds=True, out=None):
        """run() steps 4, 8-12, 14 on this rank's cells.  ref_groups_local: per reference group the
        LOCAL column indices this rank owns (possibly empty); ref_sizes: GLOBAL group sizes
        (defaults to the local ones = single GPU).  With a process group initialised the
        partial sums of the two reference-mean steps are all-gathered (NCCL)."""
        C, G = X.shape
        Y = torch.empty_like(X) if out is None else out
        flag = torch.zeros(1, dtype=torch.int32, device=self.tdev)
        b1, b2, T, n_ref, ref_leading = self._reference_bounds(X, chr_start, chr_len, ref_groups_local, ref_sizes, max_chunks,
                                                               apply_log, threshold, window, use_bounds, flag)
        # pass 2: every local cell, one read and one write of the matrix
        if self.timing is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        if self.reuse_reference_pass and 0 < n_ref < C and ref_leading:
            # the reference cells are the leading columns (the shard planner's layout): pass 1 already left their centred,
            # smoothed values in T, so they only need the second subtraction and 2^x (stage D, bit-identical to running
            # the whole pipeline again: x - 0.0 == x); the other cells take the full pipeline
            self.cell_pipeline(T[:n_ref], None, Y[:n_ref], chr_start, chr_len, False, None, 0.0, 0, 0, b2, True, use_bounds, flag)
            self.cell_pipeline(X[n_ref:], None, Y[n_ref:], chr_start, chr_len, apply_log, b1, threshold, window, 1, b2, True,
                               use_bounds, flag)
        else:
            self.cell_pipeline(X, None, Y, chr_start, chr_len, apply_log, b1, threshold, window, 1, b2, True, use_bounds, flag)
        if self.timing is not None:
            e1.record()
            self.timing.append(("cell_pipeline_pass2", e0, e1))
        return Y, flag

    def smooth_hmm_host(self, hX, hY, hS, dX, Y, states, chr_start, chr_len, ref_groups_local, ref_sizes, max_chunks, Pi, delta,
                        mean, sd, slab_cells=1024, apply_log=True, threshold=3.0, window=101, use_bounds=True):
        """Smooth block + per-cell HMM from / to pinned HOST tensors hX -> hY (float64) and hS (uint8), all (C, G), with the
        copies pipelined against the kernels over slabs of cells: the multi-rank counterpart of the C host pipeline
        (icnv_smooth_hmm_u8_f64, which knows no collectives).  The reference columns must be the leading local columns (the
        shard planner's layout); they go up first, the reference bounds are formed (two all-gathers across ranks), then
        H2D of slab i+1, pass 2 + Viterbi of slab i and D2H of slab i-1 overlap on three streams.  dX / Y / states are
        (C, G) device work buffers.  Bit-identical to smooth_block + viterbi on the uploaded matrix."""
        C, G = hX.shape
        refs = [np.asarray(g, dtype=np.int32) for g in ref_groups_local]
        n_ref = int(sum(len(g) for g in refs))
        if n_ref and not np.array_equal(np.concatenate(refs), np.arange(n_ref)):
            raise ValueError("smooth_hmm_host: the reference cells must be the leading local columns")
        on_gpu = dX.is_cuda
        flag = torch.zeros(1, dtype=torch.int32, device=self.tdev)
        if n_ref:
            dX[:n_ref].copy_(hX[:n_ref], non_blocking=True)
        b1, b2, _, _, _ = self._reference_bounds(dX, chr_start, chr_len, refs, ref_sizes, max_chunks, apply_log, threshold, window,
                                                 use_bounds, flag)
        if on_gpu:
            if getattr(self, "_copy_streams", None) is None:
                self._copy_streams = (torch.cuda.Stream(), torch.cuda.Stream())
            s_in, s_out = self._copy_streams
            main = torch.cuda.current_stream()
            s_in.wait_stream(main)     # the work buffers may still be in use by what was queued before this call
            s_out.wait_stream(main)
        flags = [flag]
        for c0 in range(0, C, slab_cells):
            c1 = min(C, c0 + slab_cells)
            u0 = max(c0, n_ref)        # the reference columns are already on the device
            if on_gpu:
                ev_in = torch.cuda.Event()
                with torch.cuda.stream(s_in):
                    if u0 < c1:
                        dX[u0:c1].copy_(hX[u0:c1], non_blocking=True)
                    ev_in.record(s_in)
                main.wait_event(ev_in)
            elif u0 < c1:
                dX[u0:c1].copy_(hX[u0:c1])
            self.cell_pipeline(dX[c0:c1], None, Y[c0:c1], chr_start, chr_len, apply_log, b1, threshold, window, 1, b2, True,
                               use_bounds, flag)
            _, f2 = self.viterbi(Y[c0:c1], chr_start, chr_len, Pi, delta, mean, sd, out=states[c0:c1])
            flags.append(f2)
            if on_gpu:
                ev_c = torch.cuda.Event()
                ev_c.record(main)
                with torch.cuda.stream(s_out):
                    s_out.wait_event(ev_c)
                    hY[c0:c1].copy_(Y[c0:c1], non_blocking=True)
                    hS[c0:c1].copy_(states[c0:c1], non_blocking=True)
            else:
                hY[c0:c1].copy_(Y[c0:c1])
                hS[c0:c1].copy_(states[c0:c1])
        if on_gpu:
            main.wait_stream(s_out)
            torch.cuda.synchronize()
        return flags

    def viterbi(self, X, chr_start, chr_len, Pi, delta, mean, sd, out=None, want_margins=False):
        """Per-cell i6 / i3 Viterbi on device data -> uint8 states (C, G)."""
        C, G = X.shape
        cs, cl = _i32(chr_start), _i32(chr_len)
        Pi = np.asfortranarray(Pi, dtype=np.float64)
        m = Pi.shape[0]
        delta, mean, sd = (np.ascontiguousarray(v, dtype=np.float64) for v in (delta, mean, sd))
        st = torch.empty((C, G), dtype=torch.uint8, device=self.tdev) if out is None else out
        mg = torch.empty((C, len(cs)), dtype=torch.float64, device=self.tdev) if want_margins else None
        flag = torch.zeros(1, dtype=torch.int32, device=self.tdev)
        _lib.check(self.lib.icnv_dev_viterbi_f64(X.data_ptr(), G, C, cs.ctypes.data, cl.ctypes.data, len(cs), m,
                                                 Pi.ctypes.data, delta.ctypes.data, mean.ctypes.data, sd.ctypes.data, 0,
                                                 st.data_ptr(), mg.data_ptr() if mg is not None else None,
                                                 flag.data_ptr(), _stream_ptr()))
        return (st, flag, mg) if want_margins else (st, flag)

    def viterbi_groups(self, X, chr_start, chr_len, Pi, delta, mean, sds, groups_local, group_sizes=None, max_chunks=None, out=None):
        """Group modes of the HMM (predict_CNV_via_HMM_on_tumor_subclusters / _on_whole_tumor_samples and the i3 twins,
        R/inferCNV_HMM.R:345-408, 509-567): per group x = rowMeans(X[, group]) (:383), ONE trace per (group, chromosome),
        written to every cell of the group; cells in no group stay 255.  groups_local: per group this rank's LOCAL columns,
        a contiguous slice of the group's list cut at multiples of CHUNK (what plan_shards does for the groups it is given) or
        the whole group; group_sizes / max_chunks: the global sizes and the largest per-rank chunk count (defaults: this
        rank holds every group whole).  sds: m values per group (.get_state_emission_params), or m values for all.
        Across ranks the groups' chunk sums are all-gathered (32 groups per exchange) and combined in list order, every rank
        runs the few group sequences itself and scatters the states to its own cells: identical bits for any rank count."""
        C, G = X.shape
        cs, cl = _i32(chr_start), _i32(chr_len)
        Pi = np.asfortranarray(Pi, dtype=np.float64)
        m = Pi.shape[0]
        delta, mean = (np.ascontiguousarray(v, dtype=np.float64) for v in (delta, mean))
        groups_local = [np.asarray(g, dtype=np.int32) for g in groups_local]
        n_grp = len(groups_local)
        sizes = [len(g) for g in groups_local] if group_sizes is None else [int(v) for v in group_sizes]
        world = self._world()
        if max_chunks is None:
            if world > 1 and group_sizes is not None:
                raise ValueError("viterbi_groups: max_chunks is needed when groups are spread over ranks")
            max_chunks = [(len(g) + shard.CHUNK - 1) // shard.CHUNK for g in groups_local]
        sds = np.asarray(sds, dtype=np.float64).reshape(-1)
        if sds.size == m:
            sds = np.tile(sds, n_grp)
        sd_med = np.median(sds.reshape(n_grp, m), axis=1)          # object$pm$sd = median(object$pm$sd), HMM.R:1122
        means = torch.empty((n_grp, G), dtype=torch.float64, device=self.tdev)
        for k0 in range(0, n_grp, 32):
            k1 = min(n_grp, k0 + 32)
            rows = np.concatenate([[0], np.cumsum([int(max_chunks[k]) for k in range(k0, k1)])]).astype(np.int32)
            tot = max(int(rows[-1]), 1)
            packed = torch.zeros((tot, G), dtype=torch.float64, device=self.tdev)
            for k in range(k0, k1):
                n = len(groups_local[k])
                if n:
                    idx = torch.as_tensor(groups_local[k], device=self.tdev)
                    _lib.check(self.lib.icnv_dev_group_partial_sums_f64(X.data_ptr(), G, X.stride(0), idx.data_ptr(), n, shard.CHUNK, 0,
                                                                        packed.data_ptr() + 8 * G * int(rows[k - k0]), _stream_ptr()))
            part = packed
            if world > 1:
                part = torch.empty((world, tot, G), dtype=torch.float64, device=self.tdev)
                self._all_gather(part, packed)
            counts = np.asarray(sizes[k0:k1], dtype=np.int64)
            _lib.check(self.lib.icnv_dev_means_from_partials_f64(part.data_ptr(), G, world, tot, k1 - k0, rows.ctypes.data,
                                                                 counts.ctypes.data, means[k0].data_ptr(), _stream_ptr()))
        d_sd = torch.as_tensor(sd_med, device=self.tdev)
        gst = torch.empty((n_grp, G), dtype=torch.uint8, device=self.tdev)
        flag = torch.zeros(1, dtype=torch.int32, device=self.tdev)
        _lib.check(self.lib.icnv_dev_viterbi_f64(means.data_ptr(), G, n_grp, cs.ctypes.data, cl.ctypes.data, len(cs), m, Pi.ctypes.data,
                                                 delta.ctypes.data, mean.ctypes.data, d_sd.data_ptr(), 1, gst.data_ptr(), None,
                                                 flag.data_ptr(), _stream_ptr()))
        grp_of = np.full(C, -1, dtype=np.int32)
        for k, g in enumerate(groups_local):
            grp_of[g] = k
        d_grp_of = torch.as_tensor(grp_of, device=self.tdev)
        st = torch.empty((C, G), dtype=torch.uint8, device=self.tdev) if out is None else out
        _lib.check(self.lib.icnv_dev_scatter_group_states_u8(gst.data_ptr(), G, C, d_grp_of.data_ptr(), st.data_ptr(), _stream_ptr()))
        return st, flag

    def pairwise_dist(self, X, cells=None, out=None):
        """Euclidean distances between the listed local cells (rows of X; default all) as R's "dist" vector, on the device
        (`hclust(parallelDist(t(expr[, cells])))`, R/inferCNV_tumor_subclusters.R:191): n (n - 1) / 2 doubles."""
        G = X.shape[1]
        idx = None if cells is None else torch.as_tensor(np.asarray(cells, dtype=np.int32), device=self.tdev)
        n = X.shape[0] if idx is None else int(idx.numel())
        if out is None:
            out = torch.empty(n * (n - 1) // 2, dtype=torch.float64, device=self.tdev)
        _lib.check(self.lib.icnv_dev_pairwise_dist_f64(X.data_ptr(), G, X.stride(0), idx.data_ptr() if idx is not None else None,
                                                       n, out.data_ptr(), _stream_ptr()))
        return out

    def knn(self, X, k, cells=None):
        """The k nearest of the listed local cells (rows of X; default all) for each of them, on the device - the nn2() of
        .leiden_simple_snn (R/inferCNV_tumor_subclusters.R:725-741).  X is a (C, G) float64 tensor with contiguous genes,
        or a gene-range view of one (X[:, a:b], one chromosome): the view's stride is the column stride.  Returns device
        tensors (idx int32, dist float64), each (n, k) with 0-based list positions, as api.knn."""
        if X.dtype != torch.float64 or X.dim() != 2 or (X.shape[1] > 1 and X.stride(1) != 1):
            raise ValueError("X must be a (cells, genes) float64 tensor with contiguous genes")
        G = X.shape[1]
        idx = None if cells is None else torch.as_tensor(np.asarray(cells, dtype=np.int32), device=self.tdev)
        n = X.shape[0] if idx is None else int(idx.numel())
        kk = max(int(k), 0) if n > 0 else 0
        nn_idx = torch.empty((kk, n), dtype=torch.int32, device=self.tdev)    # column-major n x k
        nn_dist = torch.empty((kk, n), dtype=torch.float64, device=self.tdev)
        _lib.check(self.lib.icnv_dev_knn_f64(X.data_ptr(), G, max(X.stride(0), G), idx.data_ptr() if idx is not None else None,
                                             n, int(k), nn_idx.data_ptr(), nn_dist.data_ptr(), _stream_ptr()))
        return nn_idx.T, nn_dist.T

    def seurat_snn(self, X, k=20, cells=None, n_features=2000, npcs=10):
        """api.seurat_snn on the listed local cells (rows of X; default all) on the device: X is a (C, G) float64 tensor
        with contiguous genes or a gene-range view of one (X[:, a:b], one chromosome - the per-chromosome PCA route).
        Returns an api.SeuratSNN with host arrays (the graph goes to igraph on the host)."""
        if X.dtype != torch.float64 or X.dim() != 2 or (X.shape[1] > 1 and X.stride(1) != 1):
            raise ValueError("X must be a (cells, genes) float64 tensor with contiguous genes")
        G = X.shape[1]
        idx = None if cells is None else torch.as_tensor(np.asarray(cells, dtype=np.int32), device=self.tdev)
        n = X.shape[0] if idx is None else int(idx.numel())
        nnz = ct.c_int64(0)
        _lib.check(self.lib.icnv_dev_seurat_snn_f64(X.data_ptr(), G, max(X.stride(0), G),
                                                    idx.data_ptr() if idx is not None else None, n, int(n_features),
                                                    int(npcs), int(k), ct.byref(nnz), _stream_ptr()))
        return _fetch_snn(nnz.value, n, min(int(n_features), G), int(npcs), int(k))

    def hclust(self, D, n, method="ward.D2"):
        """hclust() on the device "dist" vector D of n observations (what pairwise_dist returns), fastcluster's methods
        (api.HCLUST_METHODS): (merge, height, order) as numpy arrays in R's convention.  Only merge comes back to the
        host before `order` is computed from it; height follows with it."""
        from .api import hclust_method_code, hclust_order
        if D.dtype != torch.float64 or not D.is_contiguous() or D.numel() != n * (n - 1) // 2:
            raise ValueError("D must be a contiguous float64 device vector of n (n - 1) / 2 entries")
        merge = torch.empty((2, max(n - 1, 0)), dtype=torch.int32, device=self.tdev)   # column-major (n - 1) x 2
        height = torch.empty(max(n - 1, 0), dtype=torch.float64, device=self.tdev)
        _lib.check(self.lib.icnv_dev_hclust_f64(D.data_ptr(), n, hclust_method_code(method), merge.data_ptr(),
                                                height.data_ptr(), _stream_ptr()))
        m = merge.cpu().numpy().T
        return m, height.cpu().numpy(), hclust_order(m)

    def hclust_tri(self, D, n, method="ward.D2"):
        """Engine.hclust on the packed triangle (icnv_dev_hclust_tri_f64): any n that fits the device, bit-identical to
        Engine.hclust where both run.  D is left unchanged."""
        from .api import hclust_method_code, hclust_order
        if D.dtype != torch.float64 or not D.is_contiguous() or D.numel() != n * (n - 1) // 2:
            raise ValueError("D must be a contiguous float64 device vector of n (n - 1) / 2 entries")
        merge = torch.empty((2, max(n - 1, 0)), dtype=torch.int32, device=self.tdev)   # column-major (n - 1) x 2
        height = torch.empty(max(n - 1, 0), dtype=torch.float64, device=self.tdev)
        _lib.check(self.lib.icnv_dev_hclust_tri_f64(D.data_ptr(), n, hclust_method_code(method), merge.data_ptr(),
                                                    height.data_ptr(), _stream_ptr()))
        m = merge.cpu().numpy().T
        return m, height.cpu().numpy(), hclust_order(m)

    def cluster_cells(self, X, cells=None, method="ward.D2", keep=None):
        """api.cluster_cells on the listed local cells (rows of X; default all) on the device: X is a (C, G) float64 tensor
        with contiguous genes, or a gene-range view of one (X[:, a:b], one chromosome), as Engine.knn takes it.  keep: gene
        indices within X's columns (host list or device tensor).  Returns (merge, height, order) as numpy arrays; no
        distance vector leaves the device."""
        from .api import hclust_method_code, hclust_order
        if X.dtype != torch.float64 or X.dim() != 2 or (X.shape[1] > 1 and X.stride(1) != 1):
            raise ValueError("X must be a (cells, genes) float64 tensor with contiguous genes")
        C, G = X.shape
        idx = None if cells is None else torch.as_tensor(np.asarray(cells, dtype=np.int32), device=self.tdev)
        n = C if idx is None else int(idx.numel())
        d_keep = None
        if keep is not None:
            d_keep = torch.as_tensor(np.asarray(keep.cpu() if torch.is_tensor(keep) else keep, dtype=np.int32), device=self.tdev)
        n_keep = 0 if d_keep is None else int(d_keep.numel())
        if d_keep is not None and n_keep == 0:
            d_keep = torch.zeros(1, dtype=torch.int32, device=self.tdev)   # non-NULL: "no genes", never read
        merge = torch.empty((2, max(n - 1, 0)), dtype=torch.int32, device=self.tdev)   # column-major (n - 1) x 2
        height = torch.empty(max(n - 1, 0), dtype=torch.float64, device=self.tdev)
        _lib.check(self.lib.icnv_dev_cluster_cells_f64(
            X.data_ptr(), G, max(X.stride(0), G), C, None if d_keep is None else d_keep.data_ptr(), n_keep,
            idx.data_ptr() if idx is not None else None, n, hclust_method_code(method), merge.data_ptr(), height.data_ptr(),
            _stream_ptr()))
        m = merge.cpu().numpy().T
        return m, height.cpu().numpy(), hclust_order(m)

    def random_tree_heights(self, X, cells=None, window=101, method="ward.D2", n_perm=100, seed=0):
        """The random-trees permutation null of the clade `cells` (rows of the resident (C, G) float64 tensor X with
        contiguous genes; default all) on the device: (merge, height, order, perm_max) as numpy arrays, as
        api.random_tree_heights returns them.  Nothing but the cell list goes up and the results come back."""
        from .api import hclust_method_code, hclust_order
        if X.dtype != torch.float64 or X.dim() != 2 or (X.shape[1] > 1 and X.stride(1) != 1):
            raise ValueError("X must be a (cells, genes) float64 tensor with contiguous genes")
        G = X.shape[1]
        idx = None if cells is None else torch.as_tensor(np.asarray(cells, dtype=np.int32), device=self.tdev)
        n = X.shape[0] if idx is None else int(idx.numel())
        nm = max(n - 1, 0)
        merge = torch.empty((2, nm), dtype=torch.int32, device=self.tdev)   # column-major (n - 1) x 2
        height = torch.empty(nm, dtype=torch.float64, device=self.tdev)
        perm_max = torch.empty(max(int(n_perm), 0), dtype=torch.float64, device=self.tdev)
        _lib.check(self.lib.icnv_dev_random_tree_heights_f64(
            X.data_ptr(), G, max(X.stride(0), G), idx.data_ptr() if idx is not None else None, n, int(window),
            hclust_method_code(method), int(n_perm), int(seed) & 0xFFFFFFFFFFFFFFFF, merge.data_ptr(), height.data_ptr(),
            perm_max.data_ptr() if perm_max.numel() else None, _stream_ptr()))
        m = merge.cpu().numpy().T
        return m, height.cpu().numpy(), hclust_order(m), perm_max.cpu().numpy()

    def zscore_outlier_genes(self, X, ref_cells):
        """api.zscore_outlier_genes on the resident (C, G) float64 tensor X (rows = cells, contiguous): a boolean device
        tensor of G genes, bit-identical to the host call."""
        if X.dtype != torch.float64 or X.dim() != 2 or not X.is_contiguous():
            raise ValueError("X must be a contiguous (cells, genes) float64 tensor")
        G = X.shape[1]
        idx = torch.as_tensor(np.asarray(ref_cells, dtype=np.int32), device=self.tdev)
        out = torch.empty(G, dtype=torch.uint8, device=self.tdev)
        _lib.check(self.lib.icnv_dev_zscore_outlier_genes_f64(X.data_ptr(), G, idx.data_ptr(), int(idx.numel()), out.data_ptr(),
                                                              _stream_ptr()))
        return out.bool()

    def cluster_groups(self, X, groups, method="ward.D2", keep=None):
        """api.cluster_groups on the resident (C, G) float64 tensor X with contiguous genes: one (merge, height, order) per
        group as numpy arrays, bit-identical to the host call.  keep: gene indices (host list or device tensor)."""
        from .api import _tree_split, hclust_method_code, hclust_order
        if X.dtype != torch.float64 or X.dim() != 2 or (X.shape[1] > 1 and X.stride(1) != 1):
            raise ValueError("X must be a (cells, genes) float64 tensor with contiguous genes")
        C, G = X.shape
        off, idx = groups_to_csr(groups)
        sizes = np.diff(off).tolist()
        d_idx = torch.as_tensor(idx, device=self.tdev)
        d_keep = None
        if keep is not None:
            d_keep = torch.as_tensor(np.asarray(keep.cpu() if torch.is_tensor(keep) else keep, dtype=np.int32), device=self.tdev)
        n_keep = 0 if d_keep is None else int(d_keep.numel())
        if d_keep is not None and n_keep == 0:
            d_keep = torch.zeros(1, dtype=torch.int32, device=self.tdev)   # non-NULL: "no genes", never read
        rows = sum(max(n - 1, 0) for n in sizes)
        merge = torch.empty(max(2 * rows, 1), dtype=torch.int32, device=self.tdev)
        height = torch.empty(max(rows, 1), dtype=torch.float64, device=self.tdev)
        _lib.check(self.lib.icnv_dev_cluster_groups_f64(
            X.data_ptr(), G, max(X.stride(0), G), C, None if d_keep is None else d_keep.data_ptr(), n_keep, off.ctypes.data,
            d_idx.data_ptr(), len(sizes), hclust_method_code(method), merge.data_ptr(), height.data_ptr(), _stream_ptr()))
        m, h = merge.cpu().numpy(), height.cpu().numpy()
        order = np.empty(max(int(off[-1]), 1), dtype=np.int32)
        r = 0
        for k, n in enumerate(sizes):
            if n >= 2:
                order[off[k]:off[k] + n] = hclust_order(m[2 * r:2 * r + 2 * (n - 1)].reshape((n - 1, 2), order="F"))
                r += n - 1
            elif n == 1:
                order[off[k]] = 1
        return _tree_split(m, h, order, sizes)

    def smooth_coordinates(self, X, chr_start, chr_len, gene_start, gene_stop, window_length, out=None):
        """smooth_by_chromosome_coordinates on the resident (C, G) float64 tensor X with contiguous genes, as
        api.smooth_coordinates and bit-identical to it: returns Y (C, G), `out` or a new tensor (never X itself)."""
        from .api import _coordinate_args
        if X.dtype != torch.float64 or X.dim() != 2 or (X.shape[1] > 1 and X.stride(1) != 1):
            raise ValueError("X must be a (cells, genes) float64 tensor with contiguous genes")
        C, G = X.shape
        cs, cl, st, sp = _coordinate_args(G, chr_start, chr_len, gene_start, gene_stop)
        Y = torch.empty_like(X) if out is None else out
        if Y.data_ptr() == X.data_ptr():
            raise ValueError("out must not be X: every output reads its neighbours' inputs")
        _lib.check(self.lib.icnv_dev_smooth_coordinates_f64(
            X.data_ptr(), max(X.stride(0), G), Y.data_ptr(), max(Y.stride(0), G), G, C, cs.ctypes.data, cl.ctypes.data,
            len(cs), st.ctypes.data, sp.ctypes.data, float(window_length), _stream_ptr()))
        return Y

    def mask_non_de(self, X, ref_groups, subclusters, test="wilcoxon", p_val_thresh=0.05, rule="any", center_val=None,
                    jitter_mean=1e-4, jitter_sd=1e-4, seed=0, out=None):
        """mask_non_DE_genes_basic on the resident (C, G) float64 tensor X (single GPU), as api.mask_non_de_genes: returns
        device tensors (Y, p_raw, p_adj), Y (C, G) like X (`out`, which may be X itself, or a new tensor), p_raw / p_adj
        (n_pairs, G), row s * n_ref + j.  center_val defaults to the mean of X."""
        from .api import DE_RULES, DE_TESTS, _code
        if X.dtype != torch.float64 or X.dim() != 2 or (X.shape[1] > 1 and X.stride(1) != 1):
            raise ValueError("X must be a (cells, genes) float64 tensor with contiguous genes")
        C, G = X.shape
        if center_val is None:
            center_val = float(X.mean())
        roff, ridx = groups_to_csr(ref_groups)
        soff, sidx = groups_to_csr(subclusters)
        npair = len(subclusters) * len(ref_groups)
        Y = torch.empty_like(X) if out is None else out
        p_raw = torch.empty((npair, G), dtype=torch.float64, device=self.tdev)
        p_adj = torch.empty((npair, G), dtype=torch.float64, device=self.tdev)
        _lib.check(self.lib.icnv_dev_mask_non_de_f64(
            X.data_ptr(), max(X.stride(0), G), Y.data_ptr(), max(Y.stride(0), G), G, C, roff.ctypes.data, ridx.ctypes.data,
            len(ref_groups), soff.ctypes.data, sidx.ctypes.data, len(subclusters), _code(DE_TESTS, test, "test"),
            float(p_val_thresh), _code(DE_RULES, rule, "rule"), float(center_val), float(jitter_mean), float(jitter_sd),
            int(seed) & 0xFFFFFFFFFFFFFFFF, p_raw.data_ptr() if npair else None, p_adj.data_ptr() if npair else None,
            _stream_ptr()))
        return Y, p_raw, p_adj

    def _all_to_all(self, out: torch.Tensor, inp: torch.Tensor, out_splits, in_splits) -> None:
        """all_to_all_single of flat tensors.  NCCL: on torch's current stream; any other backend through host memory, as
        _all_gather - same bytes, same order."""
        import torch.distributed as tdist
        if tdist.get_backend() == "nccl":
            tdist.all_to_all_single(out, inp, out_splits, in_splits)
            return
        host = torch.empty(out.shape, dtype=out.dtype)
        tdist.all_to_all_single(host, inp.detach().cpu(), out_splits, in_splits)
        out.copy_(host.to(out.device))

    def mask_non_de_sharded(self, X_local, ref_groups_local, subclusters_local, test="wilcoxon", p_val_thresh=0.05, rule="any",
                            center_val=None, jitter_mean=1e-4, jitter_sd=1e-4, seed=0, out=None, slab_genes=None):
        """mask_non_DE_genes_basic on a cell shard: X_local is this rank's resident (C_local, G) float64 tensor with contiguous
        genes; ref_groups_local / subclusters_local are, per group, this rank's LOCAL columns (the planner's slices, possibly
        empty), so rank order restores each group's global list order (as mean_sd).  Each rank owns a contiguous range of
        genes: the listed cells are packed for every rank's range and exchanged (all-to-all) in gene sub-slabs sized from free
        memory (`slab_genes` forces the size), each rank tests its genes, the p rows are all-gathered, and every rank runs BH
        on all of them and masks its own cells.  Returns (Y_local, p_raw, p_adj): p_raw / p_adj the whole (n_pairs, G) on
        every rank, row s * n_ref + j.  The bytes equal api.mask_non_de_genes on the gathered matrix with the same seed and
        center_val, for any number of ranks.  center_val defaults to the mean over all ranks, combined in a fixed order
        (icnv_combine_cell_stats), so it does not depend on the number of ranks either.  NaN / Inf in a listed cell of any
        rank raises ICNV_E_NONFINITE on every rank."""
        import torch.distributed as tdist
        from .api import DE_RULES, DE_TESTS, _code
        if X_local.dtype != torch.float64 or X_local.dim() != 2 or (X_local.shape[1] > 1 and X_local.stride(1) != 1):
            raise ValueError("X_local must be a (cells, genes) float64 tensor with contiguous genes")
        C, G = X_local.shape
        world = self._world()
        rank = tdist.get_rank() if world > 1 else 0
        refs = [np.asarray(g, dtype=np.int32) for g in ref_groups_local]
        subs = [np.asarray(g, dtype=np.int32) for g in subclusters_local]
        n_ref, n_sub = len(refs), len(subs)
        npair, ng = n_ref * n_sub, n_ref + n_sub
        test_c, rule_c = _code(DE_TESTS, test, "test"), _code(DE_RULES, rule, "rule")
        mine = np.concatenate(refs + subs) if ng and sum(len(g) for g in refs + subs) else np.zeros(0, np.int32)
        if mine.size and (mine.min() < 0 or mine.max() >= C):
            raise ValueError("a listed column is outside this rank's cells")
        if center_val is None:
            center_val = self.mean_sd(X_local.contiguous(), [np.arange(C, dtype=np.int32)])[0]
        # every rank's entry count per group -> global group offsets and each rank's list positions
        lens = np.asarray([len(g) for g in refs + subs], dtype=np.int64)
        if world > 1:
            all_lens = np.stack([t.cpu().numpy() for t in self._all_gather_list(torch.as_tensor(lens, device=self.tdev))])
        else:
            all_lens = lens[None, :]
        sizes = all_lens.sum(axis=0)
        if n_ref < 1 or (sizes == 0).any():
            raise ValueError("every reference group and subcluster needs at least one cell on some rank")
        goff = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        T = int(goff[-1])
        m = all_lens.sum(axis=1)                                         # listed entries per rank
        gb = [G * d // world for d in range(world + 1)]                  # rank d tests genes [gb[d], gb[d + 1])
        n_max = max(gb[d + 1] - gb[d] for d in range(world))
        Y = torch.empty_like(X_local) if out is None else out
        p_raw = torch.empty((npair, G), dtype=torch.float64, device=self.tdev)
        p_adj = torch.empty((npair, G), dtype=torch.float64, device=self.tdev)
        if npair:
            roff = goff[:n_ref + 1].astype(np.int32)
            soff = (goff[n_ref:] - goff[n_ref]).astype(np.int32)
            # received entries in source order, each tagged with its global list position
            tags = np.concatenate([goff[k] + all_lens[:q, k].sum() + np.arange(all_lens[q, k]) for q in range(world)
                                   for k in range(ng)]).astype(np.int32)
            d_tags = torch.as_tensor(tags, device=self.tdev)
            d_cols = torch.as_tensor(mine if mine.size else np.zeros(1, np.int32), device=self.tdev)
            src_m = np.ascontiguousarray(m, dtype=np.int64)
            flag = torch.zeros(1, dtype=torch.int32, device=self.tdev)
            if slab_genes is None:
                # per gene of a sub-slab: send (at most world blocks of this rank's entries), receive, slab rows, the tests'
                # scratch (a sorted reference row, group statistics) and the p slab
                per_gene = 8 * (world * int(m[rank]) + 2 * T + int(goff[n_ref]) + 3 * ng + npair)
                free, _ = torch.cuda.mem_get_info(self.tdev)
                slab = max(1, min(n_max, (free - (1 << 30)) // per_gene))
                if world > 1:
                    slab = int(min(int(t.item()) for t in self._all_gather_list(torch.tensor([slab], device=self.tdev))))
            else:
                slab = max(1, int(slab_genes))
            p_loc = torch.empty((npair, max(n_max, 1)), dtype=torch.float64, device=self.tdev)
            for s0 in range(0, n_max, slab):
                lo = np.asarray([min(gb[d] + s0, gb[d + 1]) for d in range(world)], dtype=np.int64)
                hi = np.asarray([min(gb[d] + s0 + slab, gb[d + 1]) for d in range(world)], dtype=np.int64)
                n_s = int(hi[rank] - lo[rank])
                send = torch.empty(int((hi - lo).sum()) * int(m[rank]), dtype=torch.float64, device=self.tdev)
                _lib.check(self.lib.icnv_dev_de_pack_f64(X_local.data_ptr(), max(X_local.stride(0), G), d_cols.data_ptr(),
                                                         int(m[rank]), world, lo.ctypes.data, hi.ctypes.data,
                                                         send.data_ptr(), flag.data_ptr(), _stream_ptr()))
                if world > 1:
                    recv = torch.empty(n_s * T, dtype=torch.float64, device=self.tdev)
                    self._all_to_all(recv, send, [n_s * int(m[q]) for q in range(world)],
                                     [int(hi[d] - lo[d]) * int(m[rank]) for d in range(world)])
                else:
                    recv = send
                Z = torch.empty(n_s * T, dtype=torch.float64, device=self.tdev)
                _lib.check(self.lib.icnv_dev_de_place_f64(recv.data_ptr(), n_s, world, src_m.ctypes.data, d_tags.data_ptr(), T,
                                                          Z.data_ptr(), _stream_ptr()))
                _lib.check(self.lib.icnv_dev_de_slab_tests_f64(
                    Z.data_ptr(), T, int(lo[rank]), n_s, roff.ctypes.data, n_ref, soff.ctypes.data, n_sub, test_c,
                    float(jitter_mean), float(jitter_sd), int(seed) & 0xFFFFFFFFFFFFFFFF, p_loc.data_ptr() + 8 * s0,
                    p_loc.stride(0), _stream_ptr()))
                del send, recv, Z
            if world > 1:
                self._all_reduce_sum(flag)
            if int(flag.item()):
                raise _lib.InfercnvB200Error(_E_NONFINITE, "mask_non_de_sharded: NaN or Inf in a listed cell")
            if world > 1:
                gathered = torch.empty((world,) + tuple(p_loc.shape), dtype=torch.float64, device=self.tdev)
                self._all_gather(gathered, p_loc)
                for d in range(world):
                    p_raw[:, gb[d]:gb[d + 1]] = gathered[d, :, :gb[d + 1] - gb[d]]
                del gathered
            else:
                p_raw.copy_(p_loc[:, :G])
            del p_loc
        # BH of every pair on every rank (deterministic), then the mask of this rank's cells
        sub_size = np.ascontiguousarray(goff[n_ref + 1:] - goff[n_ref:-1], dtype=np.int32) if n_sub else np.zeros(1, np.int32)
        ridx = np.concatenate(refs) if sum(len(g) for g in refs) else np.zeros(1, np.int32)
        soff_l, sidx_l = groups_to_csr(subs)
        _lib.check(self.lib.icnv_dev_de_bh_mask_f64(
            p_raw.data_ptr() if npair else None, G, n_ref, n_sub, sub_size.ctypes.data, float(p_val_thresh),
            p_adj.data_ptr() if npair else None, X_local.data_ptr() if C else None, max(X_local.stride(0), G),
            Y.data_ptr() if C else None, max(Y.stride(0), G), C, _i32(ridx).ctypes.data, sum(len(g) for g in refs),
            soff_l.ctypes.data, sidx_l.ctypes.data, rule_c, float(center_val), _stream_ptr()))
        return Y, p_raw, p_adj

    def bayesnet(self, X, regions_genes, regions_cells, mu, tau, n_chains, n_burn=700, n_keep=1000, seed=0, pooled=None,
                 want_loglik=False) -> dict:
        """inferCNVBayesNet's Gibbs sampling on the resident (C, G) float64 tensor X (single GPU), as api.bayesnet and
        bit-identical to it; the outputs come back to the host as the same per-region lists."""
        from .api import _bayesnet_args, _bayesnet_split
        if X.dtype != torch.float64 or X.dim() != 2 or (X.shape[1] > 1 and X.stride(1) != 1):
            raise ValueError("X must be a (cells, genes) float64 tensor with contiguous genes")
        C, G = X.shape
        goff, gidx, coff, cidx, pool, mu, tau, ncol = _bayesnet_args(regions_genes, regions_cells, mu, tau, pooled)
        n_reg, m = len(regions_genes), len(mu)
        rows = int(n_chains) * int(n_keep)
        mm = m if 2 <= m <= 8 else 2
        theta = torch.empty(max(n_reg * max(rows, 1) * mm, 1), dtype=torch.float64, device=self.tdev)
        counts = torch.empty(max(int(ncol.sum()) * mm, 1), dtype=torch.int32, device=self.tdev)
        loglik = torch.empty(max(int(ncol.sum()) * mm, 1), dtype=torch.float64, device=self.tdev) if want_loglik else None
        _lib.check(self.lib.icnv_dev_bayesnet_f64(
            X.data_ptr(), max(X.stride(0), G), G, C, goff.ctypes.data, gidx.ctypes.data, coff.ctypes.data, cidx.ctypes.data,
            pool.ctypes.data, n_reg, m, mu.ctypes.data, tau.ctypes.data, int(n_chains), int(n_burn), int(n_keep),
            int(seed) & 0xFFFFFFFFFFFFFFFF, theta.data_ptr(), counts.data_ptr(),
            loglik.data_ptr() if loglik is not None else None, _stream_ptr()))
        return _bayesnet_split(theta.cpu().numpy(), counts.cpu().numpy(), None if loglik is None else loglik.cpu().numpy(),
                               ncol, m, rows)

    def mean_sd(self, X, groups_local):
        """mu / sigma over all values of the listed cells across ALL ranks (.i3HMM_get_sd_trend_by_num_cells_fit,
        R/inferCNV_i3HMM.R:17-30).  groups_local: per group, this rank's LOCAL columns (the planner's slices).
        Per-cell (sum, sd) are computed on each GPU, all-gathered group by group in rank order - which restores
        the global list order - and combined by the routine the single-GPU entry point uses: identical bits for
        any rank count."""
        import torch.distributed as tdist
        G = X.shape[1]
        multi = self.collective and tdist.is_available() and tdist.is_initialized() and tdist.get_world_size() > 1
        world = tdist.get_world_size() if multi else 1
        lens = [len(g) for g in groups_local]
        cat = np.concatenate([np.asarray(g, dtype=np.int32) for g in groups_local]) if sum(lens) else np.zeros(0, np.int32)
        n = len(cat)
        stats = torch.zeros((2, max(n, 1)), dtype=torch.float64, device=self.tdev)
        if n:
            idx = torch.as_tensor(cat, device=self.tdev)
            _lib.check(self.lib.icnv_dev_column_stats_f64(X.data_ptr(), G, idx.data_ptr(), n, stats[0].data_ptr(),
                                                          stats[1].data_ptr(), _stream_ptr()))
        if not multi:
            allstats = stats[:, :n].cpu().numpy()
        else:
            mine = torch.tensor(lens, dtype=torch.int64, device=self.tdev)
            all_lens = [t.cpu().numpy() for t in self._all_gather_list(mine)]
            nmax = int(max(int(l.sum()) for l in all_lens))
            padded = torch.zeros((2, max(nmax, 1)), dtype=torch.float64, device=self.tdev)
            padded[:, :n] = stats[:, :n]
            gathered = [g.cpu().numpy() for g in self._all_gather_list(padded)]
            cols = []
            for k in range(len(lens)):          # group-major, rank-minor = the global list order
                for r in range(world):
                    off = int(all_lens[r][:k].sum())
                    cols.append(gathered[r][:, off:off + int(all_lens[r][k])])
            allstats = np.concatenate(cols, axis=1)
        sums, sds = np.ascontiguousarray(allstats[0]), np.ascontiguousarray(allstats[1])
        mu, sg = ct.c_double(), ct.c_double()
        self.lib.icnv_combine_cell_stats(sums.ctypes.data, sds.ctypes.data, len(sums), G, ct.addressof(mu), ct.addressof(sg))
        return mu.value, sg.value

    def median_filter(self, X, chr_start, chr_len, groups_local, window_size=7, out=None):
        C, G = X.shape
        cs, cl = _i32(chr_start), _i32(chr_len)
        off, idx = groups_to_csr(groups_local)
        Y = torch.empty_like(X) if out is None else out
        _lib.check(self.lib.icnv_dev_median_filter_f64(X.data_ptr(), Y.data_ptr(), G, C, cs.ctypes.data, cl.ctypes.data,
                                                       len(cs), off.ctypes.data, idx.ctypes.data, len(groups_local),
                                                       int(window_size), _stream_ptr()))
        return Y

    def median_filter_sharded(self, Xext, n_local, whole_lists, split_slices, chr_start, chr_len, window_size=7, out=None):
        """apply_median_filtering (R/noise_reduction.R:43-113) on a cell shard.  Xext: (n_local + n_scratch, G) - the
        shard's columns followed by scratch rows for the halo columns (n_scratch >= 2 r per split list, r = (window_size
        + 1) / 2).  whole_lists: index lists (LOCAL columns) that live entirely on this rank (tumour subclusters - the
        planner keeps them whole).  split_slices: for lists cut over ranks in list order (the reference groups, cut at
        chunk boundaries by plan_shards), this rank's contiguous slice as LOCAL columns (possibly empty).  The r entries
        either side of a slice are fetched from the neighbouring ranks (one all-gather of every rank's first / last r
        columns per split list) into the scratch rows; their own outputs land in scratch rows of `out` and are
        meaningless.  The first n_local rows of the result equal the single-GPU result bit for bit."""
        import torch.distributed as tdist
        r = (int(window_size) + 1) // 2
        G = Xext.shape[1]
        world = self._world()
        Y = torch.empty_like(Xext) if out is None else out
        lists = [np.asarray(v, dtype=np.int32) for v in whole_lists]
        n_split = len(split_slices)
        if world == 1 or n_split == 0:
            lists += [np.asarray(v, dtype=np.int32) for v in split_slices if len(v)]
            return self.median_filter(Xext, chr_start, chr_len, lists, window_size, out=Y)
        if Xext.shape[0] < n_local + 2 * r * n_split:
            raise ValueError("median_filter_sharded: not enough scratch rows behind the shard")
        rank = tdist.get_rank()
        # every rank's first / last r columns of every split list, and the slice lengths
        edge = torch.zeros((n_split, 2, r, G), dtype=torch.float64, device=self.tdev)
        lens = torch.zeros(n_split, dtype=torch.float64, device=self.tdev)
        for k, sl in enumerate(split_slices):
            n = len(sl)
            lens[k] = n
            if n:
                idx = torch.as_tensor(np.asarray(sl, dtype=np.int64), device=self.tdev)
                h = min(r, n)
                edge[k, 0, :h] = Xext[idx[:h]]
                edge[k, 1, r - h:] = Xext[idx[n - h:]]
        all_edge = torch.empty((world,) + tuple(edge.shape), dtype=torch.float64, device=self.tdev)
        all_lens = torch.empty((world, n_split), dtype=torch.float64, device=self.tdev)
        self._all_gather(all_edge, edge)
        self._all_gather(all_lens, lens)
        lens_h = all_lens.cpu().numpy().astype(np.int64)
        pos = n_local
        for k, sl in enumerate(split_slices):
            if not len(sl):
                continue
            prev, nxt = shard.halo_sources(lens_h[:, k], rank, r)
            ext = []
            for q, cnt in prev:          # the last cnt columns of rank q's slice sit at the end of its tail block
                Xext[pos:pos + cnt] = all_edge[q, k, 1, r - cnt:]
                ext += list(range(pos, pos + cnt))
                pos += cnt
            ext += [int(v) for v in sl]
            for q, cnt in nxt:
                Xext[pos:pos + cnt] = all_edge[q, k, 0, :cnt]
                ext += list(range(pos, pos + cnt))
                pos += cnt
            lists.append(np.asarray(ext, dtype=np.int32))
        return self.median_filter(Xext, chr_start, chr_len, lists, window_size, out=Y)

    # ---- CNV region calling on device-resident states (R/inferCNV_HMM.R:706-1087) --------------------------------------
    def state_counts(self, S: torch.Tensor, groups_local) -> torch.Tensor:
        """(n_grp, G, 8) int32 counts of the listed LOCAL cells' states per gene (slot 0: unassigned, v + 1: state v)."""
        C, G = S.shape
        off, idx = groups_to_csr(groups_local)
        n_grp = len(groups_local)
        counts = torch.empty((n_grp, G, 8), dtype=torch.int32, device=self.tdev)
        d_idx = torch.as_tensor(idx if len(idx) else np.zeros(1, np.int32), device=self.tdev)   # a rank may own no listed cell
        flag = torch.zeros(1, dtype=torch.int32, device=self.tdev)
        _lib.check(self.lib.icnv_dev_state_counts_u8(S.data_ptr(), G, S.stride(0), d_idx.data_ptr(), off.ctypes.data, n_grp,
                                                     counts.data_ptr(), flag.data_ptr(), _stream_ptr()))
        if int(flag.item()) & 4:
            raise ValueError("state outside 0..6 / 255 in the state matrix")
        return counts

    def state_consensus(self, S: torch.Tensor, groups_local) -> torch.Tensor:
        """.get_state_consensus for every group -> (n_grp, G) uint8.  groups_local: per group, this rank's LOCAL
        columns (possibly empty).  With a process group the integer counts are summed over ranks (all-reduce), so
        the consensus is the same for any partition of a group's cells."""
        import torch.distributed as tdist
        counts = self.state_counts(S, groups_local)
        if self.collective and tdist.is_available() and tdist.is_initialized() and tdist.get_world_size() > 1:
            self._all_reduce_sum(counts)
        n_grp, G, _ = counts.shape
        cons = torch.empty((n_grp, G), dtype=torch.uint8, device=self.tdev)
        _lib.check(self.lib.icnv_dev_consensus_from_counts(counts.data_ptr(), G, n_grp, cons.data_ptr(), _stream_ptr()))
        return cons

    def cnv_regions(self, seqs: torch.Tensor, chr_start, chr_len, gene_start, gene_stop, cols=None) -> dict:
        """Run-length regions + bounds of the rows of `seqs` ((n_seq, G) uint8: consensus sequences, or the state
        matrix itself with `cols` = the cells to report, by = "cell").  Returns host arrays (api.REGION_FIELDS)."""
        from .api import REGION_FIELDS
        n_rows, G = seqs.shape
        cs, cl = _i32(chr_start), _i32(chr_len)
        gs, ge = (np.ascontiguousarray(v, dtype=np.float64) for v in (gene_start, gene_stop))
        d_cols = torch.as_tensor(np.asarray(cols, dtype=np.int32), device=self.tdev) if cols is not None else None
        n_seq = int(d_cols.numel()) if d_cols is not None else n_rows
        n = ct.c_int64(0)
        _lib.check(self.lib.icnv_dev_cnv_regions_u8(seqs.data_ptr(), G, seqs.stride(0), n_seq,
                                                    d_cols.data_ptr() if d_cols is not None else None, cs.ctypes.data,
                                                    cl.ctypes.data, len(cs), gs.ctypes.data, ge.ctypes.data,
                                                    ct.addressof(n), _stream_ptr()))
        out = {k: np.empty(int(n.value), dtype=dt) for k, dt in REGION_FIELDS}
        _lib.check(self.lib.icnv_cnv_regions_fetch(int(n.value), *[out[k].ctypes.data for k, _ in REGION_FIELDS]))
        return out

    def launch_count(self) -> int:
        return int(self.lib.icnv_launch_count())
