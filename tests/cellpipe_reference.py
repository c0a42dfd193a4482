"""Extended-precision restatement of the fused cell pipeline (icnv_dev_cell_pipeline_f64) and a per-element error bound for
its FP64 prefix-sum formulation.  Test infrastructure: used by tests/test_gpu_cell_pipeline_variants.py and checked itself by
tests/test_cellpipe_reference.py.

The stages, with the options of the device entry point (include/infercnv_b200.h):
  A  [log2(x + 1)], [dead-band subtraction lo1 / hi1 (strict inequalities) | x - mid1], [clamp to +-threshold]
  B  pyramid smoothing per chromosome as the DIRECT weighted window sum  sum_{|d| <= h} (h + 1 - |d|) x'[j + d] / D(j)  over the
     genes inside the chromosome, D(j) = ((w - 1) / 2)^2 + w - rl (rl + 1) / 2 - rr (rr + 1) / 2 with rl, rr the parts of the
     window cut off at either end (the reference's edge denominators, R/inferCNV_ops.R:2483-2532); chromosomes of one gene
     and windows < 2 leave x' unchanged
  C  centring: none, median (mean of the order statistics (n - 1) // 2 and n // 2) or mean
  D  [dead-band subtraction lo2 / hi2 | x - mid2], [2^x]
all in np.longdouble.  Nothing here uses prefix sums, so a kernel and this reference share no arithmetic.

The bound (bound=True) follows the kernel's arithmetic, not a blanket rtol.  The smoothed value is
N(j) / D(j) with N(j) = (Q(j+h) - Q(j-1)) - (Q(j-1) - Q(j-h-2)), P and Q the prefix sums of x' and of P inside the chromosome
(Q continued linearly past the last gene).  Every rounding in a sum is at most u = 2^-53 times the absolute value of a partial
sum, and a partial sum of P(i), i <= j, is bounded by PA(j) = sum_{i <= j} |x'_i|; each term passes through at most
    d = (L - 1) + 5 + 31 + 1 + L  additions  (its thread's slice total, five shuffle levels of the warp scan, at most 31 warp
                                               carries, the join of the two, the in-slice running sum; L = slice length)
on its way into P(j), and as many more into Q(j).  So |dQ(j)| <= 2 (d + 1) u QA(j), QA = the prefix sum of PA, and the three
subtractions of N add at most u (QA(j+h) + 2 QA(j-1) + QA(j-h-2)).  With K_S = 2 (d + 1) + 3 = 4 L + 77:
    |dN(j)| <= K_S u (QA(j+h) + 2 QA(j-1) + QA(j-h-2)),   |d out(j)| <= |dN(j)| / D(j) + 2 u |out(j)| + sum_d w_d |dx'| / D(j)
(2 u: the reciprocal / quotient and the product).  Stage A contributes |dx'| <= 5 u max(1, |log2(x + 1)|) + u |x'| (the
table-plus-polynomial log2 is within 3e-16 relative / absolute below 1, plus the rounding of x + 1 and of the subtraction).
The centre inherits max |d out| (median: order statistics are 1-Lipschitz in the sup norm) or the mean of |d out| plus the
reduction's own d_mean u mean |out|; stage D adds u |y| per subtraction, and 2^y multiplies the error by 2^y (e^(ln2 |dy|) - 1)
and adds 4 u 2^y for the exp2 polynomial.  These are first-order worst-case bounds: an FP64 kernel that sums in the stated
tree stays far below them (ratios of 1e-3 .. 1e-2 are typical), while a wrong index, pad or denominator is off by orders of
magnitude more.
"""
from __future__ import annotations

import numpy as np

LD = np.longdouble
U = 2.0 ** -53
HAS_EXTENDED = float(np.finfo(np.longdouble).eps) <= 1e-18


def deadband(x, lo, hi):
    return np.where(x > hi, x - hi, np.where(x < lo, x - lo, LD(0)))


def summation_depth(L: int) -> int:
    return (L - 1) + 5 + 31 + 1 + L


def cell_pipeline(X, chr_start, chr_len, *, apply_log=False, lo1=None, hi1=None, mid1=None, threshold=0.0, window=0, center=0,
                  lo2=None, hi2=None, mid2=None, apply_exp2=False, L=1, NW=32, window_shrink=0, edge_denominator_shift=False,
                  median_shift=0):
    """X: (n_cells, G) float64, a cell per row.  Returns (value, bound): the pipeline's result in np.longdouble and the
    per-element error bound (float64) of an FP64 prefix-sum kernel whose segment table has slices of L genes in CTAs of
    NW warps.  window_shrink / edge_denominator_shift / median_shift perturb the reference (tests of the checker only): a
    window narrower by 2 * window_shrink, the first gene of every chromosome divided by its neighbour's denominator, the
    median taken median_shift order statistics higher."""
    X = np.asarray(X, dtype=np.float64)
    n_cells, G = X.shape
    cs = np.asarray(chr_start, dtype=np.int64)
    cl = np.asarray(chr_len, dtype=np.int64)
    K = len(cs)
    x = X.astype(LD)

    # ---- A -------------------------------------------------------------------------------------------------------
    with np.errstate(divide="ignore", invalid="ignore"):
        if apply_log:
            lx = np.log2(x + LD(1))
            la = np.abs(lx.astype(np.float64))
            ea = np.where(np.isfinite(la), 5 * U * np.maximum(1.0, la), 0.0)
        else:
            lx = x.copy()
            ea = np.zeros(X.shape)
        if lo1 is not None:
            v = deadband(lx, np.asarray(lo1, dtype=LD)[None, :], np.asarray(hi1, dtype=LD)[None, :])
            ea = ea + U * np.abs(v.astype(np.float64))
        elif mid1 is not None:
            v = lx - np.asarray(mid1, dtype=LD)[None, :]
            ea = ea + U * np.abs(v.astype(np.float64))
        else:
            v = lx
        if threshold > 0.0:
            over = np.abs(v.astype(np.float64)) - threshold
            v = np.clip(v, LD(-threshold), LD(threshold))
            ea = np.where(over > ea, 0.0, ea)   # clamped with room to spare: the kernel writes +-threshold exactly
        ea = np.where(np.isfinite(ea), ea, 0.0)

    # ---- B -------------------------------------------------------------------------------------------------------
    s = v.copy()
    eb = ea.copy()
    if window >= 2:
        h = (window - 1) // 2 - window_shrink
        hb = (window - 1) // 2                        # the bound always follows the kernel's window
        KS = 2 * (summation_depth(L) + 1) + 3
        for c0, n in zip(cs, cl):
            if n < 2:
                continue
            xs = v[:, c0:c0 + n]
            acc = np.zeros((n_cells, n), dtype=LD)
            eprop = np.zeros((n_cells, n))
            for d in range(-h, h + 1):
                wgt = h + 1 - abs(d)
                a, b = max(0, -d), min(n, n - d)     # outputs j in [a, b) have j + d inside the chromosome
                if a < b:
                    acc[:, a:b] += LD(wgt) * xs[:, a + d:b + d]
            for d in range(-hb, hb + 1):
                a, b = max(0, -d), min(n, n - d)
                if a < b:
                    eprop[:, a:b] += (hb + 1 - abs(d)) * ea[:, c0 + a + d:c0 + b + d]
            j = np.arange(n)
            rl = np.maximum(h - j, 0)
            rr = np.maximum(h - (n - 1 - j), 0)
            if edge_denominator_shift:
                rl = np.where(j == 0, np.maximum(h - 1, 0), rl)
                rr = np.where(j == 0, np.maximum(h - (n - 2), 0), rr)
            D = LD((h + 1) * (h + 1)) - LD(0.5) * (rl * (rl + 1)).astype(LD) - LD(0.5) * (rr * (rr + 1)).astype(LD)
            s[:, c0:c0 + n] = acc / D[None, :]
            # bound: |x'| through the kernel's prefix sums, Q continued linearly past the last gene
            rlb = np.maximum(hb - j, 0)
            rrb = np.maximum(hb - (n - 1 - j), 0)
            Db = (hb + 1) * (hb + 1) - 0.5 * rlb * (rlb + 1) - 0.5 * rrb * (rrb + 1)
            A = np.abs(v[:, c0:c0 + n].astype(np.float64))
            PA = np.cumsum(A, axis=1)
            QA = np.cumsum(PA, axis=1)

            def qa(i):
                i = np.asarray(i)
                inside = np.clip(i, 0, n - 1)
                past = np.maximum(i - (n - 1), 0)
                val = QA[:, inside] + past[None, :] * PA[:, n - 1:n]
                return np.where((i >= 0)[None, :], val, 0.0)

            en = KS * U * (qa(j + hb) + 2 * qa(j - 1) + qa(j - hb - 2))
            sv = np.abs(s[:, c0:c0 + n].astype(np.float64))
            eb[:, c0:c0 + n] = (en + eprop) / Db[None, :] * (1 + 4 * U) + 2 * U * sv

    # ---- C -------------------------------------------------------------------------------------------------------
    if center == 1:
        srt = np.sort(s, axis=1)
        kA, kB = (G - 1) // 2 + median_shift, G // 2 + median_shift
        c = (srt[:, kA] + srt[:, kB]) / LD(2)
        ec = np.max(eb, axis=1) + U * np.abs(c.astype(np.float64))
    elif center == 2:
        c = np.sum(s, axis=1) / LD(G)
        nch = int(np.sum((cl + 31) // 32))
        d_mean = -(-nch // NW) + L + 12        # a lane's outputs (v3: its slice; v4: its chunks), two warp-level folds
        ec = np.mean(eb, axis=1) + d_mean * U * np.mean(np.abs(s.astype(np.float64)), axis=1) + U * np.abs(c.astype(np.float64))
    else:
        c = np.zeros(n_cells, dtype=LD)
        ec = np.zeros(n_cells)

    # ---- D -------------------------------------------------------------------------------------------------------
    z = s - c[:, None]
    e = eb + ec[:, None] + U * np.abs(z.astype(np.float64))
    if lo2 is not None:
        y = deadband(z, np.asarray(lo2, dtype=LD)[None, :], np.asarray(hi2, dtype=LD)[None, :])
        e = e + U * np.abs(y.astype(np.float64))
    elif mid2 is not None:
        y = z - np.asarray(mid2, dtype=LD)[None, :]
        e = e + U * np.abs(y.astype(np.float64))
    else:
        y = z
    if apply_exp2:
        out = np.exp2(y)
        o = out.astype(np.float64)
        e = o * (np.expm1(np.log(2.0) * e) + 4 * U)
    else:
        out = y
    return out, e


def error_ratio(got, want, bound):
    """max over the elements of |got - want| / bound (an element with a zero bound must be exact); non-finite output or a
    mismatch where the bound is zero gives inf."""
    got = np.asarray(got, dtype=np.float64)
    if not np.all(np.isfinite(got)):
        return float("inf")
    err = np.abs(got.astype(LD) - want).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    return float(np.max(r)) if r.size else 0.0


def prefix_sum_model(X, chr_start, chr_len, *, apply_log=False, lo1=None, hi1=None, mid1=None, threshold=0.0, window=0,
                     center=0, lo2=None, hi2=None, mid2=None, apply_exp2=False):
    """An FP64 implementation of the kernel's formulation in NumPy: sequential prefix sums P, Q per chromosome (the kernel
    with one slice per chromosome, L = the longest chromosome), N(j) = (Q(j+h) - Q(j-1)) - (Q(j-1) - Q(j-h-2)) times the
    reciprocal denominator.  A stand-in for a kernel in the checker's own tests."""
    X = np.asarray(X, dtype=np.float64)
    n_cells, G = X.shape
    with np.errstate(divide="ignore"):
        v = np.log2(X + 1.0) if apply_log else X.copy()
    if lo1 is not None:
        v = np.where(v > hi1, v - hi1, np.where(v < lo1, v - lo1, 0.0))
    elif mid1 is not None:
        v = v - mid1
    if threshold > 0.0:
        v = np.clip(v, -threshold, threshold)
    s = v.copy()
    if window >= 2:
        h = (window - 1) // 2
        full = float((h + 1) * (h + 1))
        for c0, n in zip(chr_start, chr_len):
            if n < 2:
                continue
            P = np.cumsum(v[:, c0:c0 + n], axis=1)
            Q = np.cumsum(P, axis=1)
            k = np.arange(1, h + 1, dtype=np.float64)
            Qx = np.concatenate([np.zeros((n_cells, h + 2)), Q, Q[:, -1:] + k[None, :] * P[:, -1:]], axis=1)   # Q(-h-2 ..)
            j = np.arange(n)
            qa, qb, qc = Qx[:, j + h + h + 2], Qx[:, j - 1 + h + 2], Qx[:, j - h - 2 + h + 2]
            N = (qa - qb) - (qb - qc)
            rl, rr = np.maximum(h - j, 0), np.maximum(h - (n - 1 - j), 0)
            D = full - 0.5 * rl * (rl + 1) - 0.5 * rr * (rr + 1)
            s[:, c0:c0 + n] = N * (1.0 / D)
    if center == 1:
        c = np.median(s, axis=1)
    elif center == 2:
        c = np.sum(s, axis=1) / G
    else:
        c = np.zeros(n_cells)
    y = s - c[:, None]
    if lo2 is not None:
        y = np.where(y > hi2, y - hi2, np.where(y < lo2, y - lo2, 0.0))
    elif mid2 is not None:
        y = y - mid2
    return np.exp2(y) if apply_exp2 else y
