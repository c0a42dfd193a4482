"""NumPy-facing wrappers of the host-pointer C ABI (the same entry points the R shim binds).

Matrices are (G genes, C cells) float64, Fortran order (R column-major: a cell's genes are
contiguous).  Indices are 0-based.  Every call goes H2D -> sm_90a kernels -> D2H inside the
library; nothing here computes on the CPU.
"""
from __future__ import annotations

import ctypes as ct
from collections import namedtuple

import numpy as np

from . import _lib


def _f64(a) -> np.ndarray:
    a = np.asarray(a, dtype=np.float64)
    if a.ndim != 2:
        raise ValueError("expected a genes x cells matrix")
    return np.asfortranarray(a)


def _i32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.int32)


def _p(a: np.ndarray | None):
    return None if a is None else a.ctypes.data


def chr_ranges(chr_codes):
    """Contiguous row range of every chromosome in order of appearance (rows are pre-sorted by
    chr in the reference, R/inferCNV.R:407-413).  A chromosome that re-appears is an error."""
    codes = np.asarray(chr_codes)
    change = np.flatnonzero(codes[1:] != codes[:-1]) + 1
    starts = np.concatenate([[0], change]).astype(np.int32)
    lens = np.diff(np.concatenate([starts, [len(codes)]])).astype(np.int32)
    if len(set(codes[starts].tolist())) != len(starts):
        raise ValueError("gene_order$chr is not sorted: a chromosome appears in two separate runs")
    return starts, lens


def groups_to_csr(groups):
    off = np.cumsum([0] + [len(g) for g in groups]).astype(np.int32)
    idx = np.concatenate([np.asarray(g, dtype=np.int32) for g in groups]) if len(groups) else np.zeros(1, np.int32)
    return off, _i32(idx)


def init(device: int = 0) -> None:
    _lib.check(_lib.load().icnv_init(int(device)))


def init_devices(device_ids=None) -> int:
    """Single-process multi-GPU (what the R shim does): the host-pointer calls that stream cells shard them over these
    devices.  None = every device present.  Returns the number of devices in use."""
    lib = _lib.load()
    if device_ids is None:
        _lib.check(lib.icnv_init_devices(0, None))
    else:
        ids = np.ascontiguousarray(device_ids, dtype=np.int32)
        _lib.check(lib.icnv_init_devices(len(ids), ids.ctypes.data))
    return int(lib.icnv_devices_in_use())


def shutdown() -> None:
    _lib.load().icnv_shutdown()


def reinit(device: int = 0) -> None:
    """Free everything and initialise again - the ICNV_* tuning switches are read from the environment at icnv_init only."""
    shutdown()
    init(device)


def set_host_threads(n: int) -> None:
    _lib.check(_lib.load().icnv_set_host_threads(int(n)))


def device_count() -> int:
    return int(_lib.load().icnv_device_count())


def launch_count() -> int:
    return int(_lib.load().icnv_launch_count())


def set_hmm_mode(mode) -> None:
    """0 / "exact": reference-order arithmetic; 1 / "fast" / "fast64": certified FP64 pass (default).  What the certified
    pass cannot certify is recomputed in reference-order arithmetic."""
    m = {"exact": 0, "fast": 1, "fast64": 1}.get(mode, mode)
    _lib.check(_lib.load().icnv_set_hmm_mode(int(m)))


def last_cell_kernel() -> tuple:
    """(family, NT, MINB, PADQ, LFIX, L) of the fused cell-pipeline instantiation the last smooth-block / cell-pipeline call
    launched (icnv_debug_cell_kernel); all zero when it launched nothing."""
    out = (ct.c_int * 6)()
    _lib.check(_lib.load().icnv_debug_cell_kernel(ct.addressof(out)))
    return tuple(int(v) for v in out)


def hmm_rerun_count() -> int:
    return int(_lib.load().icnv_hmm_rerun_count())


def hmm_second_pass_count() -> int:
    """always 0: no HMM mode hands sequences to a second pass"""
    return int(_lib.load().icnv_hmm_second_pass_count())


def ref_means(X, groups, inv_log=False) -> np.ndarray:
    X = _f64(X)
    G, C = X.shape
    off, idx = groups_to_csr(groups)
    M = np.empty((G, len(groups)), dtype=np.float64, order="F")
    _lib.check(_lib.load().icnv_ref_means_f64(_p(X), G, C, _p(off), _p(idx), len(groups), int(bool(inv_log)), _p(M)))
    return M


def subtract_ref(X, means, use_bounds=True) -> np.ndarray:
    X = _f64(X)
    M = _f64(means)
    G, C = X.shape
    if M.shape[0] != G:
        raise ValueError("means must have one row per gene")
    Y = np.empty_like(X, order="F")
    _lib.check(_lib.load().icnv_subtract_ref_f64(_p(X), _p(Y), G, C, _p(M), M.shape[1], int(bool(use_bounds))))
    return Y


def smooth(X, chr_start, chr_len, window_length) -> np.ndarray:
    X = _f64(X)
    G, C = X.shape
    cs, cl = _i32(chr_start), _i32(chr_len)
    Y = np.empty_like(X, order="F")
    _lib.check(_lib.load().icnv_smooth_f64(_p(X), _p(Y), G, C, _p(cs), _p(cl), len(cs), int(window_length)))
    return Y


def center(X, method="median") -> np.ndarray:
    X = _f64(X)
    G, C = X.shape
    Y = np.empty_like(X, order="F")
    _lib.check(_lib.load().icnv_center_f64(_p(X), _p(Y), G, C, int(method == "median")))
    return Y


def normalize_counts_by_seq_depth(X, normalize_factor=None) -> np.ndarray:
    X = _f64(X)
    G, C = X.shape
    Y = np.empty_like(X, order="F")
    nf = -1.0 if normalize_factor is None else float(normalize_factor)
    _lib.check(_lib.load().icnv_normalize_counts_by_seq_depth_f64(_p(X), _p(Y), G, C, nf))
    return Y


def clear_noise_via_ref_mean_sd(X, cells, sd_amplifier=1.5) -> np.ndarray:
    X = _f64(X)
    G, C = X.shape
    idx = _i32(cells)
    Y = np.empty_like(X, order="F")
    _lib.check(_lib.load().icnv_clear_noise_via_ref_mean_sd_f64(_p(X), _p(Y), G, C, _p(idx), len(idx), float(sd_amplifier)))
    return Y


def log2xplus1(X) -> np.ndarray:
    X = _f64(X)
    Y = np.empty_like(X, order="F")
    _lib.check(_lib.load().icnv_log2xplus1_f64(_p(X), _p(Y), X.size))
    return Y


def invert_log2(X) -> np.ndarray:
    X = _f64(X)
    Y = np.empty_like(X, order="F")
    _lib.check(_lib.load().icnv_invert_log2_f64(_p(X), _p(Y), X.size))
    return Y


def apply_max_threshold_bounds(X, threshold) -> np.ndarray:
    X = _f64(X)
    Y = np.empty_like(X, order="F")
    _lib.check(_lib.load().icnv_apply_max_threshold_bounds_f64(_p(X), _p(Y), X.size, float(threshold)))
    return Y


def smooth_block(X, chr_start, chr_len, ref_groups, apply_log=True, threshold=3.0, window_length=101,
                 use_bounds=True, out=None) -> np.ndarray:
    X = _f64(X)
    G, C = X.shape
    cs, cl = _i32(chr_start), _i32(chr_len)
    off, idx = groups_to_csr(ref_groups)
    Y = np.empty_like(X, order="F") if out is None else out
    _lib.check(_lib.load().icnv_smooth_block_f64(_p(X), _p(Y), G, C, _p(cs), _p(cl), len(cs), _p(off), _p(idx),
                                                 len(ref_groups), int(bool(apply_log)), float(threshold),
                                                 int(window_length), int(bool(use_bounds))))
    return Y


def smooth_hmm(X, chr_start, chr_len, ref_groups, Pi, delta, mean, sd, apply_log=True, threshold=3.0, window_length=101,
               use_bounds=True, out=None, out_states=None, groups=None):
    """Fused smooth block + per-cell HMM (one upload of the matrix).  Returns (Y, states).  States come back as int32
    by default; pass a uint8 `out_states` for the one-byte wire format (icnv_smooth_hmm_u8_f64).

    groups: the HMM lists of analysis_mode "samples" / "subclusters" (icnv_smooth_hmm_groups_u8_f64): states are the group
    Viterbi's, uint8 with 255 for cells in no group, and sd holds m entries per group (or m, shared)."""
    X = _f64(X)
    G, C = X.shape
    cs, cl = _i32(chr_start), _i32(chr_len)
    off, idx = groups_to_csr(ref_groups)
    Pi = np.asfortranarray(Pi, dtype=np.float64)
    delta, mean, sd = (np.ascontiguousarray(v, dtype=np.float64) for v in (delta, mean, sd))
    Y = np.empty_like(X, order="F") if out is None else out
    if groups is not None:
        m, ng = Pi.shape[0], len(groups)
        if sd.size == m:
            sd = np.tile(sd, ng)
        if sd.size != m * ng:
            raise ValueError("sd must have m entries per group")
        S = np.empty((G, C), dtype=np.uint8, order="F") if out_states is None else out_states
        if S.dtype != np.uint8 or S.shape != (G, C) or not S.flags.f_contiguous:
            raise ValueError("with groups, out_states must be a Fortran-ordered (G, C) uint8 array")
        hoff, hidx = groups_to_csr(groups)
        _lib.check(_lib.load().icnv_smooth_hmm_groups_u8_f64(
            _p(X), _p(Y), _p(S), G, C, _p(cs), _p(cl), len(cs), _p(off), _p(idx), len(ref_groups), int(bool(apply_log)),
            float(threshold), int(window_length), int(bool(use_bounds)), _p(hoff), _p(hidx), ng, m, _p(Pi), _p(delta),
            _p(mean), _p(sd)))
        return Y, S
    S = np.empty((G, C), dtype=np.int32, order="F") if out_states is None else out_states
    if S.dtype not in (np.int32, np.uint8) or S.shape != (G, C) or not S.flags.f_contiguous:
        raise ValueError("out_states must be a Fortran-ordered (G, C) int32 or uint8 array")
    lib = _lib.load()
    fn = lib.icnv_smooth_hmm_u8_f64 if S.dtype == np.uint8 else lib.icnv_smooth_hmm_f64
    _lib.check(fn(_p(X), _p(Y), _p(S), G, C, _p(cs), _p(cl), len(cs), _p(off), _p(idx), len(ref_groups), int(bool(apply_log)),
                  float(threshold), int(window_length), int(bool(use_bounds)), Pi.shape[0], _p(Pi), _p(delta), _p(mean),
                  _p(sd)))
    return Y, S


def smooth_i3_hmm(X, chr_start, chr_len, ref_groups, i3_p_val=0.05, t=1e-6, median_lists=None, median_window=7,
                  apply_log=True, threshold=3.0, window_length=101, use_bounds=True, groups=None):
    """Fused i3 pass (icnv_smooth_i3_hmm_u8_f64): smooth block, the i3 model of the reference cells' smoothed values,
    per-cell i3 HMM and, with `median_lists`, apply_median_filtering(window = median_window) over those index lists, in one
    pass over the matrix.  Returns (Y, states uint8, F or None, {"mu", "sigma", "mean_delta"}).

    groups: the HMM lists of analysis_mode "samples" / "subclusters" (icnv_smooth_i3_hmm_groups_u8_f64): the group i3 HMM,
    255 for cells in no group.  It has no median filter (F is None): run median_filter on Y."""
    X = _f64(X)
    G, C = X.shape
    cs, cl = _i32(chr_start), _i32(chr_len)
    off, idx = groups_to_csr(ref_groups)
    Y = np.empty_like(X, order="F")
    S = np.empty((G, C), dtype=np.uint8, order="F")
    if groups is not None:
        if median_lists is not None:
            raise ValueError("the group-mode i3 pass has no median filter: run median_filter on Y")
        hoff, hidx = groups_to_csr(groups)
        model = np.zeros(3, dtype=np.float64)
        _lib.check(_lib.load().icnv_smooth_i3_hmm_groups_u8_f64(
            _p(X), _p(Y), _p(S), G, C, _p(cs), _p(cl), len(cs), _p(off), _p(idx), len(ref_groups), int(bool(apply_log)),
            float(threshold), int(window_length), int(bool(use_bounds)), _p(hoff), _p(hidx), len(groups), float(i3_p_val),
            float(t), _p(model)))
        return Y, S, None, {"mu": float(model[0]), "sigma": float(model[1]), "mean_delta": float(model[2])}
    lists = [] if median_lists is None else list(median_lists)
    moff, midx = groups_to_csr(lists)
    F = np.empty_like(X, order="F") if median_lists is not None else None
    model = np.zeros(3, dtype=np.float64)
    _lib.check(_lib.load().icnv_smooth_i3_hmm_u8_f64(_p(X), _p(Y), _p(S), _p(F), G, C, _p(cs), _p(cl), len(cs), _p(off), _p(idx),
                                                     len(ref_groups), int(bool(apply_log)), float(threshold), int(window_length),
                                                     int(bool(use_bounds)), float(i3_p_val), float(t), _p(moff), _p(midx),
                                                     len(lists), int(median_window), _p(model)))
    return Y, S, F, {"mu": float(model[0]), "sigma": float(model[1]), "mean_delta": float(model[2])}


def viterbi(X, chr_start, chr_len, Pi, delta, mean, sd, groups=None, want_margins=False, out=None):
    """States (G, C): int32 with -1 = unassigned by default; a uint8 `out` selects the one-byte wire format
    (icnv_viterbi_u8_f64, 255 = unassigned)."""
    X = _f64(X)
    G, C = X.shape
    cs, cl = _i32(chr_start), _i32(chr_len)
    K = len(cs)
    Pi = np.asfortranarray(Pi, dtype=np.float64)
    m = Pi.shape[0]
    delta = np.ascontiguousarray(delta, dtype=np.float64)
    mean = np.ascontiguousarray(mean, dtype=np.float64)
    sd = np.ascontiguousarray(sd, dtype=np.float64)
    if groups is None:
        off = idx = None
        ng, nseq = 0, C
        if sd.size != m:
            raise ValueError("sd must have m entries in per-cell mode")
    else:
        off, idx = groups_to_csr(groups)
        ng = nseq = len(groups)
        if sd.size == m:
            sd = np.tile(sd, ng)
        if sd.size != m * ng:
            raise ValueError("sd must have m entries per group")
    states = np.empty((G, C), dtype=np.int32, order="F") if out is None else out
    if states.dtype not in (np.int32, np.uint8) or states.shape != (G, C) or not states.flags.f_contiguous:
        raise ValueError("out must be a Fortran-ordered (G, C) int32 or uint8 array")
    margins = np.empty((K, nseq), dtype=np.float64, order="F") if want_margins else None
    lib = _lib.load()
    fn = lib.icnv_viterbi_u8_f64 if states.dtype == np.uint8 else lib.icnv_viterbi_f64
    _lib.check(fn(_p(X), G, C, _p(cs), _p(cl), K, _p(off), _p(idx), ng, m, _p(Pi), _p(delta), _p(mean), _p(sd), _p(states),
                  _p(margins)))
    return (states, margins) if want_margins else states


def median_filter(X, chr_start, chr_len, groups, window_size=7, out=None) -> np.ndarray:
    X = _f64(X)
    G, C = X.shape
    cs, cl = _i32(chr_start), _i32(chr_len)
    off, idx = groups_to_csr(groups)
    Y = np.empty_like(X, order="F") if out is None else out
    _lib.check(_lib.load().icnv_median_filter_f64(_p(X), _p(Y), G, C, _p(cs), _p(cl), len(cs), _p(off), _p(idx),
                                                  len(groups), int(window_size)))
    return Y


def mean_sd(X, cells):
    X = _f64(X)
    G, C = X.shape
    idx = _i32(cells)
    mu, sg = ct.c_double(), ct.c_double()
    _lib.check(_lib.load().icnv_mean_sd_f64(_p(X), G, C, _p(idx), len(idx), ct.addressof(mu), ct.addressof(sg)))
    return mu.value, sg.value


def pairwise_dist(X, cells=None, out=None):
    """parallelDist(t(X[, cells])) (euclidean): R's "dist" vector - n (n - 1) / 2 doubles, the strict lower triangle by
    columns - for the listed cells (default: all), R/inferCNV_tumor_subclusters.R:191 and the other hclust() call sites."""
    X = _f64(X)
    G, C = X.shape
    idx = None if cells is None else _i32(cells)
    n = C if idx is None else len(idx)
    n_out = n * (n - 1) // 2
    if out is None:
        out = np.empty(n_out, dtype=np.float64)
    if out.dtype != np.float64 or out.size != n_out or not out.flags.c_contiguous:
        raise ValueError("out must be a contiguous float64 vector of n (n - 1) / 2 entries")
    _lib.check(_lib.load().icnv_pairwise_dist_f64(_p(X), G, C, _p(idx) if idx is not None else None, n, _p(out)))
    return out


def pairwise_dist_rows(x, out=None):
    """parallelDist(x) for x = observations x variables (the t(expr.data[, cells]) the reference passes), without
    transposing it back: icnv_pairwise_dist_rows_f64."""
    x = np.asfortranarray(np.asarray(x, dtype=np.float64))
    if x.ndim != 2:
        raise ValueError("x must be a matrix (observations x variables)")
    n, G = x.shape
    n_out = n * (n - 1) // 2
    if out is None:
        out = np.empty(n_out, dtype=np.float64)
    if out.dtype != np.float64 or out.size != n_out or not out.flags.c_contiguous:
        raise ValueError("out must be a contiguous float64 vector of n (n - 1) / 2 entries")
    _lib.check(_lib.load().icnv_pairwise_dist_rows_f64(_p(x), n, G, _p(out)))
    return out


KNN_MAX_K = 64   # ICNV_KNN_MAX_K


def _knn_out(n: int, k: int):
    shape = (n, max(int(k), 0)) if n > 0 else (0, 0)
    return np.empty(shape, dtype=np.int32, order="F"), np.empty(shape, dtype=np.float64, order="F")


def knn(X, k, cells=None):
    """The k nearest of the listed cells (default: all columns of the genes x cells matrix X) for each of them, itself
    included - RANN::nn2(t(X[, cells]), k = k) exactly: (idx, dist), each (n, k), idx 0-based list positions.  Rows are
    ordered by squared distance, then position (icnv_knn_f64); distances have the bits of pairwise_dist's."""
    X = _f64(X)
    G, C = X.shape
    idx = None if cells is None else _i32(cells)
    n = C if idx is None else len(idx)
    nn_idx, nn_dist = _knn_out(n, k)
    _lib.check(_lib.load().icnv_knn_f64(_p(X), G, C, _p(idx) if idx is not None else None, n, int(k), _p(nn_idx),
                                        _p(nn_dist)))
    return nn_idx, nn_dist


def knn_rows(x, k):
    """knn() on x = observations x variables, the matrix nn2() receives (t(expr.data[, cells])): icnv_knn_rows_f64."""
    x = np.asfortranarray(np.asarray(x, dtype=np.float64))
    if x.ndim != 2:
        raise ValueError("x must be a matrix (observations x variables)")
    n, G = x.shape
    nn_idx, nn_dist = _knn_out(n, k)
    _lib.check(_lib.load().icnv_knn_rows_f64(_p(x), n, G, int(k), _p(nn_idx), _p(nn_dist)))
    return nn_idx, nn_dist


# hclust() methods with an exact nearest-neighbour chain, coded as fastcluster orders them (centroid 5 and median 6 are not
# reducible and have no GPU path)
HCLUST_METHODS = {"single": 0, "complete": 1, "average": 2, "mcquitty": 3, "ward.D": 4, "ward.D2": 7}


def hclust_method_code(method) -> int:
    if isinstance(method, str):
        if method not in HCLUST_METHODS:
            raise ValueError(f"hclust method {method!r}: one of {sorted(HCLUST_METHODS)}")
        return HCLUST_METHODS[method]
    return int(method)


def _dist_size(n_d: int) -> int:
    n = int(round((1 + np.sqrt(1 + 8 * n_d)) / 2))
    if n * (n - 1) // 2 != n_d:
        raise ValueError(f"{n_d} entries are not a \"dist\" vector (n (n - 1) / 2 for some n)")
    return n


def hclust(d, method="ward.D2"):
    """fastcluster::hclust(d, method) on R's "dist" vector d (strict lower triangle by columns, e.g. pairwise_dist's
    output): returns (merge, height, order) in R's convention - merge (n - 1) x 2 int32 (singleton -(i + 1), cluster of
    step s +s), height (n - 1), order (n, 1-based).  Methods: HCLUST_METHODS (or their codes)."""
    d = np.ascontiguousarray(d, dtype=np.float64).ravel()
    n = _dist_size(d.size)
    merge = np.empty((max(n - 1, 0), 2), dtype=np.int32, order="F")
    height = np.empty(max(n - 1, 0), dtype=np.float64)
    order = np.empty(n, dtype=np.int32)
    _lib.check(_lib.load().icnv_hclust_f64(_p(d), n, hclust_method_code(method), _p(merge), _p(height), _p(order)))
    return merge, height, order


# the largest n the square-matrix linkage (icnv_hclust_f64, cluster_groups) accepts; hclust_tri / cluster_cells go past it
HCLUST_NMAX = 65536


def hclust_tri(d, method="ward.D2"):
    """hclust() as api.hclust returns it, on the packed triangle (icnv_hclust_tri_f64): bit-identical to api.hclust where
    both run, and for any n whose 4 n (n - 1) bytes (plus the scratch) fit the free device memory - past HCLUST_NMAX."""
    d = np.ascontiguousarray(d, dtype=np.float64).ravel()
    n = _dist_size(d.size)
    merge = np.empty((max(n - 1, 0), 2), dtype=np.int32, order="F")
    height = np.empty(max(n - 1, 0), dtype=np.float64)
    order = np.empty(n, dtype=np.int32)
    _lib.check(_lib.load().icnv_hclust_tri_f64(_p(d), n, hclust_method_code(method), _p(merge), _p(height), _p(order)))
    return merge, height, order


def cluster_cells(X, cells=None, method="ward.D2", keep=None):
    """hclust(parallelDist(t(X[keep, cells])), method) for one cell list (default: all columns of the genes x cells matrix X)
    of any size that fits the device, in one call (icnv_cluster_cells_f64): (merge, height, order), bit-identical to
    hclust_tri(pairwise_dist(X[keep], cells), method).  keep: genes to use (default all; an empty list uses none)."""
    X = _f64(X)
    G, C = X.shape
    idx = None if cells is None else _i32(cells)
    n = C if idx is None else len(idx)
    k = None if keep is None else _i32(keep)
    kp = np.zeros(1, np.int32) if k is not None and k.size == 0 else k   # non-NULL: "no genes", never read
    merge = np.empty((max(n - 1, 0), 2), dtype=np.int32, order="F")
    height = np.empty(max(n - 1, 0), dtype=np.float64)
    order = np.empty(max(n, 1), dtype=np.int32)
    _lib.check(_lib.load().icnv_cluster_cells_f64(
        _p(X), G, C, _p(kp), 0 if k is None else len(k), _p(idx) if idx is not None else None, n, hclust_method_code(method),
        _p(merge), _p(height), _p(order)))
    return merge, height, order[:n]


def hclust_order(merge) -> np.ndarray:
    """R's `order` from a merge matrix ((n - 1) x 2): hcass2's traversal, on the host (icnv_hclust_order)."""
    m = np.asfortranarray(merge, dtype=np.int32)
    n = m.shape[0] + 1
    order = np.empty(n, dtype=np.int32)
    _lib.check(_lib.load().icnv_hclust_order(_p(m), n, _p(order)))
    return order


def runmean(X, k, chr_start=None, chr_len=None) -> np.ndarray:
    """caTools::runmean(x, k) (endrule "mean", align "center") down every column of the genes x cells matrix X, per row
    range (default: the whole column): smooth_by_chromosome_runmeans with the chromosomes as ranges.  Genes outside every
    range, ranges of fewer than 2 genes and k <= 1 are copied (icnv_runmean_f64)."""
    X = _f64(X)
    G, C = X.shape
    Y = np.empty_like(X, order="F")
    if chr_start is None:
        _lib.check(_lib.load().icnv_runmean_f64(_p(X), _p(Y), G, C, None, None, 0, int(k)))
    else:
        cs, cl = _i32(chr_start), _i32(chr_len)
        if len(cs) != len(cl):
            raise ValueError("chr_start and chr_len differ in length")
        _lib.check(_lib.load().icnv_runmean_f64(_p(X), _p(Y), G, C, _p(cs), _p(cl), len(cs), int(k)))
    return Y


def _coordinate_args(G, chr_start, chr_len, gene_start, gene_stop):
    cs, cl = _i32(chr_start), _i32(chr_len)
    st = np.ascontiguousarray(gene_start, dtype=np.float64)
    sp = np.ascontiguousarray(gene_stop, dtype=np.float64)
    if len(cs) != len(cl):
        raise ValueError("chr_start and chr_len differ in length")
    if st.shape != (G,) or sp.shape != (G,):
        raise ValueError("gene_start and gene_stop need one entry per gene")
    return cs, cl, st, sp


def smooth_coordinates(X, chr_start, chr_len, gene_start, gene_stop, window_length) -> np.ndarray:
    """smooth_by_chromosome_coordinates on the genes x cells matrix X with the row ranges (chr_start, chr_len) as its
    chromosomes: every gene's value becomes the weighted mean over the genes within window_length of its midpoint, with
    R's padding and recycling (icnv_smooth_coordinates_f64).  gene_start / gene_stop are per row of X.  Genes outside every
    range, ranges of one gene and window_length < 2 are copied."""
    X = _f64(X)
    G, C = X.shape
    cs, cl, st, sp = _coordinate_args(G, chr_start, chr_len, gene_start, gene_stop)
    Y = np.empty_like(X, order="F")
    _lib.check(_lib.load().icnv_smooth_coordinates_f64(_p(X), _p(Y), G, C, _p(cs), _p(cl), len(cs), _p(st), _p(sp),
                                                       float(window_length)))
    return Y


def random_tree_heights(X, window=101, method="ward.D2", n_perm=100, seed=0, cells=None):
    """The permutation null of random-trees subclustering for the clade X[:, cells] (default: all columns) of the genes x
    cells matrix X: (merge, height, order, perm_max).  merge / height / order are the observed tree, runmean(window) ->
    median centring -> Euclidean distances -> hclust(method), as hclust() returns it; perm_max (n_perm) holds the largest
    height of each permuted tree (every gene shuffled across the cells by the generator of icnv_random_tree_heights_f64)."""
    X = _f64(X)
    G, C = X.shape
    idx = None if cells is None else _i32(cells)
    n = C if idx is None else len(idx)
    nm = max(n - 1, 0)
    merge = np.empty((nm, 2), dtype=np.int32, order="F")
    height = np.empty(nm, dtype=np.float64)
    order = np.empty(max(n, 1), dtype=np.int32)
    perm_max = np.empty(max(int(n_perm), 0), dtype=np.float64)
    _lib.check(_lib.load().icnv_random_tree_heights_f64(
        _p(X), G, C, _p(idx) if idx is not None else None, n, int(window), hclust_method_code(method), int(n_perm),
        int(seed) & 0xFFFFFFFFFFFFFFFF, _p(merge), _p(height), _p(order), _p(perm_max) if perm_max.size else None))
    return merge, height, order[:n], perm_max


def random_trees_stats() -> dict:
    """What the last random_tree_heights call did: the wave size B, the number of waves and the device time (ms) of its
    stages (icnv_debug_random_trees)."""
    out = np.zeros(5, dtype=np.float64)
    _lib.check(_lib.load().icnv_debug_random_trees(_p(out)))
    return {"B": int(out[0]), "waves": int(out[1]), "prep_ms": out[2], "dist_ms": out[3], "link_ms": out[4]}


def zscore_outlier_genes(X, ref_cells) -> np.ndarray:
    """The z-score gene filter of define_signif_tumor_subclusters (R/inferCNV_tumor_subclusters.R:45-68) on the genes x cells
    matrix X: a boolean mask of the genes with mean(|z|) >= 0.8 over the reference columns `ref_cells` (in that order), z
    standardised by api.mean_sd's mu and sigma of those columns (icnv_zscore_outlier_genes_f64)."""
    X = _f64(X)
    G, C = X.shape
    idx = _i32(ref_cells)
    out = np.empty(G, dtype=np.uint8)
    _lib.check(_lib.load().icnv_zscore_outlier_genes_f64(_p(X), G, C, _p(idx), len(idx), _p(out)))
    return out.astype(bool)


def _tree_split(merge, height, order, sizes):
    """The packed outputs of icnv_cluster_groups_f64 -> one (merge, height, order) per group."""
    trees, r, o = [], 0, 0
    for n in sizes:
        nm = max(n - 1, 0)
        m = np.asfortranarray(merge[2 * r:2 * r + 2 * nm].reshape((nm, 2), order="F"))
        trees.append((m, height[r:r + nm].copy(), order[o:o + n].copy()))
        r += nm
        o += n
    return trees


def cluster_groups(X, groups, method="ward.D2", keep=None):
    """hclust(parallelDist(t(X[keep, g])), method) for every cell list g of `groups` (columns of the genes x cells matrix X)
    in one call (icnv_cluster_groups_f64): a list of (merge, height, order), each bit-identical to
    hclust(pairwise_dist(X[keep], g), method).  keep: genes to use (default all; an empty list uses none, so every distance
    is 0).  A group of fewer than 2 cells gets an empty merge / height and order 1 .. n."""
    X = _f64(X)
    G, C = X.shape
    off, idx = groups_to_csr(groups)
    sizes = np.diff(off).tolist()
    k = None if keep is None else _i32(keep)
    kp = np.zeros(1, np.int32) if k is not None and k.size == 0 else k   # non-NULL: "no genes", never read
    rows = sum(max(n - 1, 0) for n in sizes)
    merge = np.empty(max(2 * rows, 1), dtype=np.int32)
    height = np.empty(max(rows, 1), dtype=np.float64)
    order = np.empty(max(int(off[-1]), 1), dtype=np.int32)
    _lib.check(_lib.load().icnv_cluster_groups_f64(
        _p(X), G, C, _p(kp), 0 if k is None else len(k), _p(off), _p(idx), len(sizes), hclust_method_code(method), _p(merge), _p(height),
        _p(order)))
    return _tree_split(merge, height, order, sizes)


def cluster_groups_stats() -> dict:
    """What the last cluster_groups call did: waves, groups in the largest wave, device ms of the gene gather, the distances
    and the linkages (icnv_debug_cluster_groups)."""
    out = np.zeros(5, dtype=np.float64)
    _lib.check(_lib.load().icnv_debug_cluster_groups(_p(out)))
    return {"waves": int(out[0]), "widest": int(out[1]), "gather_ms": out[2], "dist_ms": out[3], "link_ms": out[4]}


SeuratSNN = namedtuple("SeuratSNN", "indptr indices data features embeddings idx stats")
SeuratSNN.__doc__ = """What seurat_snn returns: the graph as CSR (indptr int64 n + 1, indices int32, data float64; symmetric,
columns ascending per row), the variable features (0-based gene indices in rank order), the embeddings (n x npcs), the kNN
lists (n x k, 0-based positions) and the call's statistics (seurat_snn_stats)."""


def _fetch_snn(nnz: int, n: int, nf: int, npcs: int, k: int) -> SeuratSNN:
    indptr = np.empty(n + 1, dtype=np.int64)
    indices = np.empty(max(nnz, 1), dtype=np.int32)
    data = np.empty(max(nnz, 1), dtype=np.float64)
    feats = np.empty(max(nf, 1), dtype=np.int32)
    emb = np.empty((n, npcs), dtype=np.float64)       # row-major n x npcs = the library's npcs x n column-major
    idx = np.empty((k, n), dtype=np.int32)             # column-major n x k
    _lib.check(_lib.load().icnv_seurat_snn_fetch(_p(indptr), _p(indices), _p(data), _p(feats), _p(emb), _p(idx)))
    return SeuratSNN(indptr, indices[:nnz], data[:nnz], feats[:nf], emb, np.ascontiguousarray(idx.T), seurat_snn_stats())


def seurat_snn(X, k=20, cells=None, n_features=2000, npcs=10) -> SeuratSNN:
    """The SNN graph .leiden_seurat_preprocess_routine builds with Seurat (vst variable features, ScaleData, RunPCA(npcs),
    FindNeighbors(k.param = k)) on the columns `cells` (default all) of the genes x cells matrix X, computed exactly on the
    device (icnv_seurat_snn_f64; see include/infercnv_b200.h for the contract)."""
    X = _f64(X)
    G, C = X.shape
    idx = None if cells is None else _i32(cells)
    n = C if idx is None else len(idx)
    nnz = ct.c_int64(0)
    _lib.check(_lib.load().icnv_seurat_snn_f64(_p(X), G, C, _p(idx), n, int(n_features), int(npcs), int(k),
                                               ct.byref(nnz)))
    return _fetch_snn(nnz.value, n, min(int(n_features), G), int(npcs), int(k))


SNN_STAGES = ("stats", "trend", "stdvar", "gram", "eigen", "embed", "knn", "snn")


def seurat_snn_stats() -> dict:
    """What the last seurat_snn call did (icnv_debug_seurat_snn): F, npcs used, eigen-iterations, the largest relative
    residual, the eigen-gap ratio, the standardised-variance gap at the n_features cut, singular trend fits, device ms per
    stage and the hub rows that took the global-memory path."""
    out = np.zeros(16, dtype=np.float64)
    _lib.check(_lib.load().icnv_debug_seurat_snn(_p(out)))
    return {"F": int(out[0]), "npcs": int(out[1]), "iterations": int(out[2]), "residual": out[3], "eig_ratio": out[4],
            "sv_gap": out[5], "singular_fits": int(out[6]), "ms": dict(zip(SNN_STAGES, out[7:15].tolist())),
            "hub_rows": int(out[15])}


DE_TESTS = {"wilcoxon": 0, "t": 1}
DE_RULES = {"any": 0, "most": 1, "all": 2}


def _code(table, v, what) -> int:
    if isinstance(v, str):
        if v not in table:
            raise ValueError(f"unknown {what} {v!r}")
        return table[v]
    return int(v)


def mask_non_de_genes(X, ref_groups, subclusters, test="wilcoxon", p_val_thresh=0.05, rule="any", center_val=None,
                      jitter_mean=1e-4, jitter_sd=1e-4, seed=0, want_y=True):
    """mask_non_DE_genes_basic on the genes x cells matrix X (icnv_mask_non_de_f64): ref_groups and subclusters are lists
    of 0-based column lists, the subclusters the TESTED ones in R's loop order.  Returns (Y, p_raw, p_adj): Y the masked
    matrix (None when want_y is False), p_raw / p_adj G x (len(subclusters) * len(ref_groups)), column s * n_ref + j.
    center_val defaults to the mean of X, as in R."""
    X = _f64(X)
    G, C = X.shape
    if center_val is None:
        center_val = float(np.mean(X))
    roff, ridx = groups_to_csr(ref_groups)
    soff, sidx = groups_to_csr(subclusters)
    npair = len(subclusters) * len(ref_groups)
    Y = np.empty_like(X, order="F") if want_y else None
    p_raw = np.empty((G, npair), dtype=np.float64, order="F")
    p_adj = np.empty((G, npair), dtype=np.float64, order="F")
    _lib.check(_lib.load().icnv_mask_non_de_f64(
        _p(X), _p(Y), G, C, _p(roff), _p(ridx), len(ref_groups), _p(soff), _p(sidx), len(subclusters),
        _code(DE_TESTS, test, "test"), float(p_val_thresh), _code(DE_RULES, rule, "rule"), float(center_val),
        float(jitter_mean), float(jitter_sd), int(seed) & 0xFFFFFFFFFFFFFFFF, _p(p_raw) if npair else None,
        _p(p_adj) if npair else None))
    return Y, p_raw, p_adj


def mask_non_de_stats() -> dict:
    """What the last mask call did: gene tiles, genes per tile and the device time (ms) of its stages
    (icnv_debug_mask_non_de)."""
    out = np.zeros(7, dtype=np.float64)
    _lib.check(_lib.load().icnv_debug_mask_non_de(_p(out)))
    return {"tiles": int(out[0]), "genes_per_tile": int(out[1]), "gather_ms": out[2], "group_ms": out[3],
            "pairs_ms": out[4], "bh_ms": out[5], "mask_ms": out[6]}


def _bayesnet_args(regions_genes, regions_cells, mu, tau, pooled):
    goff, gidx = groups_to_csr(regions_genes)
    coff, cidx = groups_to_csr(regions_cells)
    n_reg = len(regions_genes)
    if len(regions_cells) != n_reg:
        raise ValueError("regions_genes and regions_cells differ in length")
    pool = np.zeros(max(n_reg, 1), dtype=np.uint8)
    if pooled is not None:
        pool[:n_reg] = np.asarray(pooled, dtype=bool)
    mu = np.ascontiguousarray(mu, dtype=np.float64)
    tau = np.ascontiguousarray(tau, dtype=np.float64)
    if mu.shape != tau.shape or mu.ndim != 1:
        raise ValueError("mu and tau must be vectors of the same length")
    ncol = np.where(pool[:n_reg] > 0, 1, np.diff(coff)).astype(np.int64)
    return goff, gidx, coff, cidx, pool, mu, tau, ncol


def _bayesnet_split(theta, counts, loglik, ncol, m, rows):
    """Flat library outputs -> per-region lists."""
    off = np.concatenate([[0], np.cumsum(ncol)]) * m
    th = [theta[r * rows * m:(r + 1) * rows * m].reshape((rows, m), order="F") for r in range(len(ncol))]
    cnt = [counts[off[r]:off[r + 1]].reshape((m, int(ncol[r])), order="F") for r in range(len(ncol))]
    ll = None if loglik is None else [loglik[off[r]:off[r + 1]].reshape((m, int(ncol[r])), order="F") for r in range(len(ncol))]
    return {"theta": th, "cell_probabilities": [c / float(rows) for c in cnt], "state_counts": cnt, "loglik": ll}


def bayesnet(X, regions_genes, regions_cells, mu, tau, n_chains, n_burn=700, n_keep=1000, seed=0, pooled=None,
             want_loglik=False) -> dict:
    """inferCNVBayesNet's Gibbs sampling (icnv_bayesnet_f64) for every region of the genes x cells matrix X: region r is
    the block X[regions_genes[r], regions_cells[r]] (0-based lists), mu / tau the m states' means and precisions; pooled[r]
    marks R's one-gene quirk (the region is one pseudo-cell).  Returns {"theta": per region the (n_chains n_keep) x m draws,
    chains stacked; "cell_probabilities": per region m x C'_r state frequencies; "state_counts": the same as integer counts;
    "loglik": per region the m x C'_r log-likelihoods L, or None}.  Same posterior as JAGS, not its draws."""
    X = _f64(X)
    G, C = X.shape
    goff, gidx, coff, cidx, pool, mu, tau, ncol = _bayesnet_args(regions_genes, regions_cells, mu, tau, pooled)
    n_reg, m = len(regions_genes), len(mu)
    rows = int(n_chains) * int(n_keep)
    mm = m if 2 <= m <= 8 else 2
    theta = np.empty(max(n_reg * max(rows, 1) * mm, 1), dtype=np.float64)
    counts = np.empty(max(int(ncol.sum()) * mm, 1), dtype=np.int32)
    loglik = np.empty(max(int(ncol.sum()) * mm, 1), dtype=np.float64) if want_loglik else None
    _lib.check(_lib.load().icnv_bayesnet_f64(
        _p(X), G, C, _p(goff), _p(gidx), _p(coff), _p(cidx), _p(pool), n_reg, m, _p(mu), _p(tau), int(n_chains), int(n_burn),
        int(n_keep), int(seed) & 0xFFFFFFFFFFFFFFFF, _p(theta), _p(counts), _p(loglik)))
    return _bayesnet_split(theta, counts, loglik, ncol, m, rows)


def bayesnet_stats() -> dict:
    """What the last Bayesian network call did: regions, sampler CTAs and the device time (ms) of the log-likelihood pass
    and of the sampler (icnv_debug_bayesnet)."""
    out = np.zeros(4, dtype=np.float64)
    _lib.check(_lib.load().icnv_debug_bayesnet(_p(out)))
    return {"regions": int(out[0]), "ctas": int(out[1]), "loglik_ms": out[2], "sampler_ms": out[3]}


# ---- CNV region calling on the state matrix (R/inferCNV_HMM.R:706-1087) ---------------------------------------

def _u8(a) -> np.ndarray:
    """State matrix in the one-byte wire format (0..6, 255 = unassigned).  int / float matrices as R holds them
    (-1 = unassigned) are narrowed here; that is marshalling, like the R shim's double -> byte loop."""
    a = np.asarray(a)
    if a.ndim == 1:
        a = a[:, None]
    if a.dtype != np.uint8:
        if np.any(a != np.floor(a)) or a.min() < -1 or a.max() > 254:
            raise ValueError("states must be integers in -1..254")
        a = np.where(a < 0, 255, a).astype(np.uint8)
    return np.asfortranarray(a)


REGION_FIELDS = (("seq", np.int32), ("chr", np.int32), ("first_gene", np.int32), ("last_gene", np.int32),
                 ("state", np.int32), ("start", np.float64), ("end", np.float64))


def _fetch_regions(n: int) -> dict:
    out = {k: np.empty(n, dtype=dt) for k, dt in REGION_FIELDS}
    _lib.check(_lib.load().icnv_cnv_regions_fetch(n, *[_p(out[k]) for k, _ in REGION_FIELDS]))
    return out


def state_consensus(states, groups) -> np.ndarray:
    """Modal state per gene per group, (G, n_grp) uint8 (icnv_state_consensus_u8)."""
    S = _u8(states)
    G, C = S.shape
    off, idx = groups_to_csr(groups)
    cons = np.empty((G, len(groups)), dtype=np.uint8, order="F")
    _lib.check(_lib.load().icnv_state_consensus_u8(_p(S), G, C, _p(off), _p(idx), len(groups), _p(cons)))
    return cons


def cnv_regions(seqs, chr_start, chr_len, gene_start, gene_stop) -> dict:
    """Run-length regions of every column of `seqs` (icnv_cnv_regions_u8 + icnv_cnv_regions_fetch): dict of arrays
    seq, chr, first_gene, last_gene, state, start, end in (sequence, chromosome, position) order."""
    S = _u8(seqs)
    G, n_seq = S.shape
    cs, cl = _i32(chr_start), _i32(chr_len)
    gs, ge = (np.ascontiguousarray(v, dtype=np.float64) for v in (gene_start, gene_stop))
    n = ct.c_int64(0)
    _lib.check(_lib.load().icnv_cnv_regions_u8(_p(S), G, n_seq, _p(cs), _p(cl), len(cs), _p(gs), _p(ge), ct.addressof(n)))
    return _fetch_regions(int(n.value))


def predicted_cnv_regions(states, chr_start, chr_len, gene_start, gene_stop, groups, want_consensus=False):
    """Consensus of every cell group + region calling in one upload (icnv_predicted_cnv_regions_u8).
    Returns the region dict, or (regions, consensus) with want_consensus."""
    S = _u8(states)
    G, C = S.shape
    cs, cl = _i32(chr_start), _i32(chr_len)
    gs, ge = (np.ascontiguousarray(v, dtype=np.float64) for v in (gene_start, gene_stop))
    off, idx = groups_to_csr(groups)
    cons = np.empty((G, len(groups)), dtype=np.uint8, order="F") if want_consensus else None
    n = ct.c_int64(0)
    _lib.check(_lib.load().icnv_predicted_cnv_regions_u8(_p(S), G, C, _p(cs), _p(cl), len(cs), _p(gs), _p(ge), _p(off), _p(idx),
                                                         len(groups), _p(cons), ct.addressof(n)))
    reg = _fetch_regions(int(n.value))
    return (reg, cons) if want_consensus else reg


# ---- gene filters and counts ingest (run() steps 2-3) -----------------------------------------------------------

def gene_stats(X):
    """Per-gene (sums, n_pos, means) of a dense matrix (icnv_gene_stats_f64): what .below_min_mean_expr_cutoff and
    require_above_min_cells_ref compare with their thresholds."""
    X = _f64(X)
    G, C = X.shape
    sums, means = np.empty(G), np.empty(G)
    n_pos = np.empty(G, dtype=np.int32)
    _lib.check(_lib.load().icnv_gene_stats_f64(_p(X), G, C, _p(sums), _p(n_pos), _p(means)))
    return sums, n_pos, means


def remove_genes(X, keep) -> np.ndarray:
    """X[keep, ] for increasing row indices `keep` (icnv_remove_genes_f64)."""
    X = _f64(X)
    G, C = X.shape
    keep = _i32(keep)
    Y = np.empty((len(keep), C), dtype=np.float64, order="F")
    _lib.check(_lib.load().icnv_remove_genes_f64(_p(X), G, C, _p(keep), len(keep), _p(Y)))
    return Y


def _csc(p, i, x):
    p, i = _i32(p), _i32(i)
    x = np.ascontiguousarray(x, dtype=np.float64)
    if len(i) != len(x) or len(p) < 2 or p[-1] != len(x):
        raise ValueError("inconsistent compressed-column arrays")
    return p, i, x


def csc_gene_stats(p, i, x, n_genes):
    """gene_stats for a compressed-sparse-column counts matrix (dgCMatrix @p / @i / @x)."""
    p, i, x = _csc(p, i, x)
    G, C = int(n_genes), len(p) - 1
    sums, means = np.empty(G), np.empty(G)
    n_pos = np.empty(G, dtype=np.int32)
    _lib.check(_lib.load().icnv_csc_gene_stats_f64(_p(p), _p(i), _p(x), G, C, _p(sums), _p(n_pos), _p(means)))
    return sums, n_pos, means


def csc_normalize(p, i, x, n_genes, keep=None, normalize_factor=None, want_col_sums=False):
    """Dense depth-normalised matrix (kept genes x cells) straight from compressed columns (icnv_csc_normalize_f64)."""
    p, i, x = _csc(p, i, x)
    G, C = int(n_genes), len(p) - 1
    keep = None if keep is None else _i32(keep)
    G_out = G if keep is None else len(keep)
    Y = np.empty((G_out, C), dtype=np.float64, order="F")
    cs = np.empty(C) if want_col_sums else None
    nf = -1.0 if normalize_factor is None else float(normalize_factor)
    _lib.check(_lib.load().icnv_csc_normalize_f64(_p(p), _p(i), _p(x), G, C, _p(keep), 0 if keep is None else len(keep), nf,
                                                  _p(Y), _p(cs)))
    return (Y, cs) if want_col_sums else Y


# ---- outlier clamp and noise clearing (run() steps 16, 22) --------------------------------------------------------

def remove_outliers_norm(X, lower_bound=None, upper_bound=None, want_bounds=False):
    """.remove_outliers_norm (icnv_remove_outliers_norm_f64); a missing bound selects out_method "average_bound"."""
    X = _f64(X)
    G, C = X.shape
    Y = np.empty_like(X, order="F")
    b = np.empty(2)
    lo = float("nan") if lower_bound is None else float(lower_bound)
    hi = float("nan") if upper_bound is None else float(upper_bound)
    _lib.check(_lib.load().icnv_remove_outliers_norm_f64(_p(X), _p(Y), G, C, lo, hi, _p(b)))
    return (Y, (float(b[0]), float(b[1]))) if want_bounds else Y


def clear_noise(X, cells, threshold, noise_logistic=False) -> np.ndarray:
    """clear_noise (icnv_clear_noise_f64); cells = reference cells, or None / empty for "all data"."""
    X = _f64(X)
    G, C = X.shape
    idx = None if cells is None or len(cells) == 0 else _i32(cells)
    Y = np.empty_like(X, order="F")
    _lib.check(_lib.load().icnv_clear_noise_f64(_p(X), _p(Y), G, C, _p(idx), 0 if idx is None else len(idx), float(threshold),
                                                int(bool(noise_logistic))))
    return Y


def clear_noise_via_ref_mean_sd_logistic(X, cells, sd_amplifier=1.5) -> np.ndarray:
    X = _f64(X)
    G, C = X.shape
    idx = _i32(cells)
    Y = np.empty_like(X, order="F")
    _lib.check(_lib.load().icnv_clear_noise_via_ref_mean_sd_logistic_f64(_p(X), _p(Y), G, C, _p(idx), len(idx),
                                                                        float(sd_amplifier)))
    return Y


def assign_hmm_states_to_proxy_expr_vals(states, m=6) -> np.ndarray:
    """State matrix -> proxy expression values (icnv_assign_hmm_states_to_proxy_expr_vals_f64)."""
    X = _f64(states)
    Y = np.empty_like(X, order="F")
    _lib.check(_lib.load().icnv_assign_hmm_states_to_proxy_expr_vals_f64(_p(X), _p(Y), X.size, int(m)))
    return Y


# ---- per-chromosome subcluster HMM (R/inferCNV_HMM.R:412-487) -----------------------------------------------------

def viterbi_per_chr(X, chr_start, chr_len, groups_per_chr, Pi, delta, mean, sds) -> np.ndarray:
    """One Viterbi sequence per (chromosome, subcluster of that chromosome) on the subcluster's rowMeans
    (icnv_viterbi_per_chr_u8_f64).  groups_per_chr: per chromosome a list of cell-index arrays; sds: m values per group,
    chromosome-major in the same order.  Returns uint8 states (G, C), 255 where a cell has no subcluster."""
    X = _f64(X)
    G, C = X.shape
    cs, cl = _i32(chr_start), _i32(chr_len)
    if len(groups_per_chr) != len(cs):
        raise ValueError("one list of subclusters per chromosome is needed")
    flat = [np.asarray(g) for per in groups_per_chr for g in per]
    chr_off = np.cumsum([0] + [len(per) for per in groups_per_chr]).astype(np.int32)
    off, idx = groups_to_csr(flat)
    Pi = np.asfortranarray(Pi, dtype=np.float64)
    m = Pi.shape[0]
    delta, mean = (np.ascontiguousarray(v, dtype=np.float64) for v in (delta, mean))
    sds = np.ascontiguousarray(sds, dtype=np.float64)
    if sds.size == m:
        sds = np.tile(sds, len(flat))
    if sds.size != m * len(flat):
        raise ValueError("sds must have m entries per (chromosome, subcluster)")
    S = np.empty((G, C), dtype=np.uint8, order="F")
    _lib.check(_lib.load().icnv_viterbi_per_chr_u8_f64(_p(X), G, C, _p(cs), _p(cl), len(cs), _p(chr_off), _p(off), _p(idx), m,
                                                       _p(Pi), _p(delta), _p(mean), _p(sds), _p(S)))
    return S


def apply_state_consensus(states, chr_start, chr_len, groups) -> np.ndarray:
    """Every cell of a group takes the group's consensus state on the genes region calling covers
    (icnv_apply_state_consensus_u8)."""
    S = _u8(states)
    G, C = S.shape
    cs, cl = _i32(chr_start), _i32(chr_len)
    off, idx = groups_to_csr(groups)
    out = np.empty((G, C), dtype=np.uint8, order="F")
    _lib.check(_lib.load().icnv_apply_state_consensus_u8(_p(S), G, C, _p(cs), _p(cl), len(cs), _p(off), _p(idx), len(groups),
                                                         _p(out)))
    return out


def scale_infercnv_expr(X) -> np.ndarray:
    """Per-gene z-scores across the cells (icnv_scale_infercnv_expr_f64)."""
    X = _f64(X)
    G, C = X.shape
    Y = np.empty_like(X, order="F")
    _lib.check(_lib.load().icnv_scale_infercnv_expr_f64(_p(X), _p(Y), G, C))
    return Y


def gather_genes(X, idx) -> np.ndarray:
    """X[idx, ] for any row order (icnv_gather_genes_f64)."""
    X = _f64(X)
    G, C = X.shape
    idx = _i32(idx)
    Y = np.empty((len(idx), C), dtype=np.float64, order="F")
    _lib.check(_lib.load().icnv_gather_genes_f64(_p(X), G, C, _p(idx), len(idx), _p(Y)))
    return Y
