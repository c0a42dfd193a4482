// icnv_median_select.cuh - exact median of one (2R+1) x (2R+1) window of apply_median_filtering
// (.median_filter, R/noise_reduction.R:93-113), written once for device and host: the CUDA kernel in
// icnv_median_filter.cu runs it per thread, tests/test_median_select_host.py compiles the same text with g++ and
// checks it against std::nth_element on random, tie-heavy and truncated windows.
//
// The window lives in a shared "halo" array (taps outside the block hold +inf there and 0 in a second copy used
// for the moments).  Selection of the k-th smallest, k = (n-1)/2, never moves values - only counts and a
// per-thread list of 16-bit tap offsets:
//   1. mean / sd of the window place a first bracket (mean - sd/2, mean + sd/2];
//   2. one pass over the taps counts the values at or below the bracket and lists the taps inside it; if the
//      target rank fell outside (skewed or bimodal window) the pass is repeated on the side that holds it;
//   3. the bracket is narrowed by counting over the LIST only: four value pivots placed by interpolation while
//      that shrinks it (one round is then enough for all but ~1 % of the windows - a warp runs as many rounds as its
//      slowest lane), otherwise one three-way round (less / equal / greater) around an element of the list,
//      which always makes progress and finishes tie-dominated windows (de-noised matrices, state matrices) in
//      one round;
//   4. at most 16 candidates are left: a sorting network orders them and the rank is read off.
// Even n (truncated windows only) averages the two middle values as median.default does.
#pragma once
#include <cfloat>
#include <cmath>
#include <cstring>

#ifdef __CUDACC__
#define ICNV_HD __host__ __device__ __forceinline__
#else
#define ICNV_HD inline
#endif

namespace icnv {

ICNV_HD void mf_cswap(double &a, double &b) {
    const bool s = b < a;
    const double lo = s ? b : a, hi = s ? a : b;
    a = lo;
    b = hi;
}

// largest double below a finite x (the bracket's upper end after a three-way round excludes the pivot itself)
ICNV_HD double mf_pred(double x) {
    if (x == 0.0) return -4.9406564584124654e-324;
    long long b;
#ifdef __CUDA_ARCH__
    b = __double_as_longlong(x);
#else
    memcpy(&b, &x, sizeof(b));
#endif
    b += (x > 0.0) ? -1 : 1;
#ifdef __CUDA_ARCH__
    return __longlong_as_double(b);
#else
    double r;
    memcpy(&r, &b, sizeof(r));
    return r;
#endif
}

// Batcher's odd-even merge sort for 16 keys (63 comparators)
ICNV_HD void mf_sort16(double (&c)[16]) {
    mf_cswap(c[0], c[1]); mf_cswap(c[2], c[3]); mf_cswap(c[0], c[2]); mf_cswap(c[1], c[3]);
    mf_cswap(c[1], c[2]); mf_cswap(c[4], c[5]); mf_cswap(c[6], c[7]); mf_cswap(c[4], c[6]);
    mf_cswap(c[5], c[7]); mf_cswap(c[5], c[6]); mf_cswap(c[0], c[4]); mf_cswap(c[2], c[6]);
    mf_cswap(c[2], c[4]); mf_cswap(c[1], c[5]); mf_cswap(c[3], c[7]); mf_cswap(c[3], c[5]);
    mf_cswap(c[1], c[2]); mf_cswap(c[3], c[4]); mf_cswap(c[5], c[6]); mf_cswap(c[8], c[9]);
    mf_cswap(c[10], c[11]); mf_cswap(c[8], c[10]); mf_cswap(c[9], c[11]); mf_cswap(c[9], c[10]);
    mf_cswap(c[12], c[13]); mf_cswap(c[14], c[15]); mf_cswap(c[12], c[14]); mf_cswap(c[13], c[15]);
    mf_cswap(c[13], c[14]); mf_cswap(c[8], c[12]); mf_cswap(c[10], c[14]); mf_cswap(c[10], c[12]);
    mf_cswap(c[9], c[13]); mf_cswap(c[11], c[15]); mf_cswap(c[11], c[13]); mf_cswap(c[9], c[10]);
    mf_cswap(c[11], c[12]); mf_cswap(c[13], c[14]); mf_cswap(c[0], c[8]); mf_cswap(c[4], c[12]);
    mf_cswap(c[4], c[8]); mf_cswap(c[2], c[10]); mf_cswap(c[6], c[14]); mf_cswap(c[6], c[10]);
    mf_cswap(c[2], c[4]); mf_cswap(c[6], c[8]); mf_cswap(c[10], c[12]); mf_cswap(c[1], c[9]);
    mf_cswap(c[5], c[13]); mf_cswap(c[5], c[9]); mf_cswap(c[3], c[11]); mf_cswap(c[7], c[15]);
    mf_cswap(c[7], c[11]); mf_cswap(c[3], c[5]); mf_cswap(c[7], c[9]); mf_cswap(c[11], c[13]);
    mf_cswap(c[1], c[2]); mf_cswap(c[3], c[4]); mf_cswap(c[5], c[6]); mf_cswap(c[7], c[8]);
    mf_cswap(c[9], c[10]); mf_cswap(c[11], c[12]); mf_cswap(c[13], c[14]);
}

// halo / halo0: the tile's values (+inf resp. 0 outside the block), row stride HR (genes are the fast index);
// idx0: index of the window's first tap; list: this thread's tap-offset list, entries ls apart, (2R+1)^2 entries;
// n: number of taps inside the block (>= 1).  stats (optional): [0] += list rounds, [1] += second build passes.
constexpr int MF_CAND = 16;   // candidates ordered directly at the end

template <int R>
ICNV_HD double window_median(const double *halo, const double *halo0, int HR, int idx0, unsigned short *list, int ls, int n,
                             unsigned *stats = nullptr) {
    constexpr int D = 2 * R + 1;
    const int k = (n - 1) >> 1;
    const bool even = (n & 1) == 0;
    const double *w = halo + idx0;
    const double *w0 = halo0 + idx0;

    // ---- 1. moments -> first bracket -----------------------------------------------------------------------------
    double s1 = 0.0, s2 = 0.0;
#pragma unroll
    for (int dj = 0; dj < D; ++dj)
#pragma unroll
        for (int di = 0; di < D; ++di) {
            const double v = w0[dj * HR + di];
            s1 += v;
            s2 = fma(v, v, s2);
        }
    const double mean = s1 / (double)n;
    const double var = s2 / (double)n - mean * mean;
    double blo = -INFINITY, bhi = DBL_MAX;   // bracket (blo, bhi]; +inf padding is never inside
    if (var > 0.0) {
        const double half = 0.5 * sqrt(var);
        const double p1 = mean - half, p2 = mean + half;
        if (p1 < p2 && p2 < DBL_MAX) {
            blo = p1;
            bhi = p2;
        }
    }

    // ---- 2. list the taps inside the bracket, count the values at or below it ------------------------------------
    int c_lo = 0, cnt = 0;
    for (int attempt = 0; attempt < 3; ++attempt) {
        c_lo = 0;
        cnt = 0;
#pragma unroll
        for (int dj = 0; dj < D; ++dj)
#pragma unroll
            for (int di = 0; di < D; ++di) {
                const double v = w[dj * HR + di];
                const bool below = v <= blo;
                const bool inside = !below && (v <= bhi);
                c_lo += below ? 1 : 0;
                if (inside) {
                    list[cnt * ls] = (unsigned short)(dj * HR + di);
                    ++cnt;
                }
            }
        if (k < c_lo) {   // the target is below the bracket: everything at or below its lower end
            bhi = blo;
            blo = -INFINITY;
        } else if (k >= c_lo + cnt) {   // above it
            blo = bhi;
            bhi = DBL_MAX;
        } else {
            break;
        }
        if (stats) stats[1] += 1;
    }
    const int L0 = c_lo;                       // window values at or below the list's lower end
    double lo = blo, hi = bhi;                 // invariant: #(v <= lo) = Flo <= k < Fhi = #(v <= hi)
    int Flo = c_lo, Fhi = c_lo + cnt;
    double result = 0.0, next = 0.0;
    bool have_result = false, have_next = false;

    // ---- 3. narrow the bracket by counting over the list ----------------------------------------------------------
    bool stagnant = false;
    bool first = true;
    for (int iter = 0; iter < 4 * D * D && !have_result; ++iter) {
        const int m = Fhi - Flo;
        if (m <= MF_CAND) break;
        if (stats) stats[0] += 1;
        bool elem_mode = stagnant;
        if (first) {   // three probes equal: a tie-dominated window, go straight for an element pivot
            const double a = w[list[0]], b = w[list[(cnt >> 1) * ls]], c = w[list[(cnt - 1) * ls]];
            elem_mode = (a == b) && (b == c);
            first = false;
        }
        const double span = hi - lo;
        if (!(span < DBL_MAX)) elem_mode = true;   // open-ended bracket: nothing to interpolate in
        if (elem_mode) {
            double x = 0.0;
            for (int t = 0; t < cnt; ++t) {   // first listed value still inside the bracket (one exists: m > MF_CAND)
                const double v = w[list[t * ls]];
                if (v > lo && v <= hi) {
                    x = v;
                    break;
                }
            }
            int less = 0, eq = 0;
            for (int t = 0; t < cnt; ++t) {
                const double v = w[list[t * ls]];
                less += (v < x) ? 1 : 0;
                eq += (v == x) ? 1 : 0;
            }
            const int L = L0 + less;
            if (k < L) {
                hi = mf_pred(x);
                Fhi = L;
            } else if (k < L + eq) {
                result = x;
                have_result = true;
                if (k + 1 < L + eq) {
                    next = x;
                    have_next = true;
                } else {   // the upper middle value is the smallest one above x
                    hi = x;
                    Fhi = L + eq;
                }
            } else {
                lo = x;
                Flo = L + eq;
            }
            stagnant = false;
        } else {
            // k sits at fraction f of the bracket's m values.  Four value pivots placed by interpolation at about -12, -4,
            // +4 and +12 ranks around it cut the bracket into pieces of ~8 ranks, so that for the usual m of 25..40 whichever
            // piece holds the target fits the final network: one round per window, and - what matters on the GPU, where a warp
            // runs as many rounds as its slowest lane - practically never a second one (two pivots at +-6 left 8..28 % of the
            // windows with more than MF_CAND candidates).  The counts are exact whatever the placement.
            const double f = ((double)(k - Flo) + 0.5) / (double)m;
            const double w1 = fmax(4.0 / (double)m, 0.05), w2 = fmax(12.0 / (double)m, 0.15);
            const double pv0 = lo + span * (f - w2), pv1 = lo + span * (f - w1), pv2 = lo + span * (f + w1),
                         pv3 = lo + span * (f + w2);
            int c0 = 0, c1 = 0, c2 = 0, c3 = 0;
            for (int t = 0; t < cnt; ++t) {
                const double v = w[list[t * ls]];
                c0 += (v <= pv0) ? 1 : 0;
                c1 += (v <= pv1) ? 1 : 0;
                c2 += (v <= pv2) ? 1 : 0;
                c3 += (v <= pv3) ? 1 : 0;
            }
            // ascending pivots: the last one with #(v <= p) <= k becomes the lower end, the first one above it the upper end
            // (pivots outside the open bracket are ignored; the invariant #(v <= lo) = Flo <= k < Fhi = #(v <= hi) is kept)
            const double lo_in = lo, hi_in = hi;
            bool have_hi = false;
#define ICNV_MF_PIVOT(PV, CV)                                  \
            if ((PV) > lo_in && (PV) < hi_in && !have_hi) {    \
                const int Cq = L0 + (CV);                      \
                if (k >= Cq) {                                 \
                    lo = (PV);                                 \
                    Flo = Cq;                                  \
                } else {                                       \
                    hi = (PV);                                 \
                    Fhi = Cq;                                  \
                    have_hi = true;                            \
                }                                              \
            }
            ICNV_MF_PIVOT(pv0, c0)
            ICNV_MF_PIVOT(pv1, c1)
            ICNV_MF_PIVOT(pv2, c2)
            ICNV_MF_PIVOT(pv3, c3)
#undef ICNV_MF_PIVOT
            stagnant = (Fhi - Flo == m);
        }
    }

    // ---- 4. <= MF_CAND candidates in (lo, hi]: order them, read off rank k (and k + 1 for even n) ------------------
    if (!have_result) {
        int c = 0;
        for (int t = 0; t < cnt; ++t) {   // in place: the write position never passes the read position
            const unsigned short e = list[t * ls];
            const double v = w[e];
            if (v > lo && v <= hi) {
                list[c * ls] = e;
                ++c;
            }
        }
        double cand[MF_CAND];
#pragma unroll
        for (int q = 0; q < MF_CAND; ++q) cand[q] = (q < c) ? w[list[q * ls]] : INFINITY;
        mf_sort16(cand);
        const int r = k - Flo;
#pragma unroll
        for (int q = 0; q < MF_CAND; ++q) {
            if (q == r) result = cand[q];
            if (q == r + 1 && q < c) {
                next = cand[q];
                have_next = true;
            }
        }
    }
    if (!even) return result;
    if (!have_next) {   // the upper middle value lies above the bracket: smallest value greater than hi
        double mn = INFINITY;
#pragma unroll
        for (int dj = 0; dj < D; ++dj)
#pragma unroll
            for (int di = 0; di < D; ++di) {
                const double v = w[dj * HR + di];
                if (v > hi && v < mn) mn = v;
            }
        next = mn;
    }
    return (result + next) * 0.5;
}

}  // namespace icnv
