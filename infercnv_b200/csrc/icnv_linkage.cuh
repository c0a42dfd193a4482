// icnv_linkage.cuh - the arithmetic and the tie rules shared by the two nearest-neighbour-chain linkage kernels: K11 on the
// square matrix (icnv_hclust.cu) and K19 on the packed triangle (icnv_hclust_tri.cu).  Both must return the same bits on
// the same input, so the Lance-Williams update, the key order of the row scans and the end of the launch (stable sort of
// the raw merges, conversion to R's merge matrix) live here once.
#pragma once

#include "icnv_common.cuh"

namespace icnv {

#ifdef __CUDACC__

// total order on doubles with -0 == +0 (what a numeric comparison does): key of v + 0.0
__device__ __forceinline__ unsigned long long dkey(double v) { return key_of(__dadd_rn(v, 0.0)); }

__device__ __forceinline__ bool key_less(unsigned long long ka, int ia, unsigned long long kb, int ib) {
    return ka < kb || (ka == kb && ia < ib);
}

// d(k, i u j) from d(k, i), d(k, j), d(i, j) and the sizes, in the operation order of icnv_hclust.cu's header comment
__device__ __forceinline__ double lance_williams(int method, double dki, double dkj, double dij, double ni, double nj,
                                                 double nk) {
    switch (method) {
    case 0: return dki < dkj ? dki : dkj;
    case 1: return dki > dkj ? dki : dkj;
    case 2: return __ddiv_rn(__dadd_rn(__dmul_rn(ni, dki), __dmul_rn(nj, dkj)), __dadd_rn(ni, nj));
    case 3: return __ddiv_rn(__dadd_rn(dki, dkj), 2.0);
    default:  // 4 ward.D, 7 ward.D2 (squared input)
        return __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(__dadd_rn(ni, nk), dki), __dmul_rn(__dadd_rn(nj, nk), dkj)),
                                   -__dmul_rn(nk, dij)),
                         __dadd_rn(__dadd_rn(ni, nj), nk));
    }
}

// The end of a linkage, run by all NT threads of its CTA: the n - 1 raw merges (slots raw_i < raw_j merged at height raw_h,
// in chain order) stably sorted by height - bitonic on (key, raw step) over P (a power of two >= n - 1) entries of skey /
// sidx - then converted to R's merge matrix by a union-find over the slots in sorted order (uf, node: n entries each).
// Heights are rooted for ward.D2 (method 7).  merge: (n - 1) x 2 column-major.
template <int NT>
__device__ __forceinline__ void linkage_finish(int64_t n, int method, int P, const double *raw_h, const int32_t *raw_i,
                                               const int32_t *raw_j, unsigned long long *skey, int32_t *sidx, int32_t *uf,
                                               int32_t *node, int32_t *merge, double *height) {
    const int tid = threadIdx.x;
    const int nm = (int)(n - 1);
    for (int t = tid; t < P; t += NT) {
        skey[t] = t < nm ? dkey(raw_h[t]) : ~0ull;
        sidx[t] = t < nm ? t : 0x7fffffff;
    }
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1)
        for (int jj = k >> 1; jj > 0; jj >>= 1) {
            for (int t = tid; t < P; t += NT) {
                const int l = t ^ jj;
                if (l <= t) continue;
                const unsigned long long ka = skey[t], kb = skey[l];
                const int ia = sidx[t], ib = sidx[l];
                const bool up = (t & k) == 0;
                if (up ? key_less(kb, ib, ka, ia) : key_less(ka, ia, kb, ib)) {
                    skey[t] = kb; skey[l] = ka;
                    sidx[t] = ib; sidx[l] = ia;
                }
            }
            __syncthreads();
        }
    for (int64_t k = tid; k < n; k += NT) {
        uf[k] = (int32_t)k;
        node[k] = (int32_t)k;
    }
    __syncthreads();
    if (tid == 0) {
        auto find = [&](int x) {
            while (uf[x] != x) {
                const int gp = uf[uf[x]];
                uf[x] = gp;
                x = gp;
            }
            return x;
        };
        for (int s = 0; s < nm; ++s) {
            const int t = sidx[s];
            const int x = find(raw_i[t]), y = find(raw_j[t]);
            const int nx = node[x], ny = node[y];
            const int lo = nx < ny ? nx : ny, hi = nx < ny ? ny : nx;
            merge[s] = lo < n ? -(lo + 1) : lo - (int)n + 1;
            merge[nm + s] = hi < n ? -(hi + 1) : hi - (int)n + 1;
            const double h = raw_h[t];
            height[s] = method == 7 ? sqrt(h) : h;
            uf[x] = y;
            node[y] = (int)n + s;
        }
    }
}

#endif  // __CUDACC__

}  // namespace icnv
