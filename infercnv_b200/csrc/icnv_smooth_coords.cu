// Coordinate-weighted smoothing - K16 in DESIGN section 3.
//
// smooth_by_chromosome_coordinates (R/inferCNV_ops.R:2534-2622): per chromosome range of n >= 2 genes and window W >= 2,
// every cell's value of gene i becomes a weighted mean over a band of genes whose weights depend only on the genes'
// coordinates and W.  The host builds that stencil once (stencil_build, R's which() scan literally, O(n^2) per range):
//     pos = (s[i] + e[i]) / 2,  around = {j : s[j] > pos - W and e[j] < pos + W}  (ascending; {i} if empty),
//     w_j = 1 - |(e[j] + s[j]) / 2 - pos| / W,  to_add = floor(|around| / 2),
//     lo = max(0, min(around) - to_add),  hi = min(n - 1, max(around) + to_add),
//     wv = (0.1 x (min(around) - lo), w_around, 0.1 x (hi - max(around)))           (Lw entries)
// The band x[lo .. hi] has L = hi - lo + 1 >= Lw entries; where `around` has holes, R's `*` recycles wv, so term k uses
// wv[k mod Lw].  The table stores those L recycled weights per row, and den = the sequential long-double sum of the Lw
// unrecycled weights rounded to double (on x86-64 the host's long double is R's LDOUBLE: den is R's sum(w) bit for bit).
// Rows outside every smoothed range are the stencil lo = i, L = 1, weight 1, den 1: a copy.
//
// The kernel: Y[i, c] = fl( fl(sum_k fl(X[lo + k, c] w_k)) / den ).  Products are __dmul_rn (never contracted into an FMA:
// R's products are rounded on their own); the numerator is Ogita-Rump-Oishi Sum2 (cascaded two-sum) in increasing k,
// rounded once, then divided.  One CTA takes SC_RB consecutive rows and SC_TC cells; the rows' band slab (with the rows
// themselves, so every gene is checked for NaN / Inf) goes through shared memory in chunks of SC_CH genes, loaded along
// each cell's contiguous genes; lanes are cells, so each weight load is a warp-wide broadcast.  A row's terms are added in
// increasing k across the chunks, so the result does not depend on the chunk size or the launch geometry.
#include "icnv_common.cuh"

#include <algorithm>
#include <cmath>
#include <new>
#include <vector>

namespace icnv {
namespace sc {

constexpr int SC_TC = 32;              // cells per CTA: the lanes of a warp
constexpr int SC_NW = 8;               // warps per CTA
constexpr int SC_NT = SC_TC * SC_NW;
constexpr int SC_RB = 32;              // rows per CTA
constexpr int SC_RPW = SC_RB / SC_NW;  // rows per warp
constexpr int SC_CH = 128;             // slab genes per chunk
constexpr int SC_LD = SC_TC + 1;       // padded slab row

// blockIdx.x: tile of SC_TC cells, blockIdx.y: block of SC_RB rows.  Row r: band [lo[r], lo[r] + len[r]) with the weights
// w[off[r] ..], denominator den[r]; row block b: slab [blo[b], bhi[b]].  flag |= 1 on NaN / Inf in the slab.
__global__ void __launch_bounds__(SC_NT, 4) smooth_coords_kernel(const double *__restrict__ X, int64_t ldx,
                                                                 double *__restrict__ Y, int64_t ldy, int64_t G, int64_t C,
                                                                 const int32_t *__restrict__ lo, const int32_t *__restrict__ len,
                                                                 const int64_t *__restrict__ off, const double *__restrict__ w,
                                                                 const double *__restrict__ den, const int32_t *__restrict__ blo,
                                                                 const int32_t *__restrict__ bhi, int *flag) {
    __shared__ double slab[SC_CH * SC_LD];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t c0 = (int64_t)blockIdx.x * SC_TC, r0 = (int64_t)blockIdx.y * SC_RB;
    const int ncell = (int)(C - c0 < SC_TC ? C - c0 : SC_TC);
    const int64_t g_lo = blo[blockIdx.y], g_hi = bhi[blockIdx.y];
    int64_t rlo[SC_RPW], rlen[SC_RPW], roff[SC_RPW];
    double s[SC_RPW], e[SC_RPW];
#pragma unroll
    for (int j = 0; j < SC_RPW; ++j) {
        const int64_t r = r0 + warp + SC_NW * j;
        rlo[j] = r < G ? lo[r] : 0;
        rlen[j] = r < G ? len[r] : 0;
        roff[j] = r < G ? off[r] : 0;
        s[j] = 0.0;
        e[j] = 0.0;
    }
    bool bad = false;
    for (int64_t cb = g_lo; cb <= g_hi; cb += SC_CH) {
        __syncthreads();   // the previous chunk has been read
        for (int t = threadIdx.x; t < SC_TC * SC_CH; t += SC_NT) {
            const int cell = t / SC_CH, g = t % SC_CH;
            double v = 0.0;
            if (cell < ncell && cb + g <= g_hi) {
                v = X[cb + g + ldx * (c0 + cell)];
                bad |= !is_finite_d(v);
            }
            slab[g * SC_LD + cell] = v;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < SC_RPW; ++j) {
            int64_t kb = cb - rlo[j], ke = cb + SC_CH - rlo[j];
            kb = kb > 0 ? kb : 0;
            ke = ke < rlen[j] ? ke : rlen[j];
            if (kb >= ke) continue;
            const double *xs = slab + (rlo[j] + kb - cb) * SC_LD + lane;   // gene lo + k sits at xs[(k - kb) * SC_LD]
            const double *wr = w + roff[j];
            int64_t k = kb;
            if (k == 0) {   // the first term starts the sum (a one-term row is then an exact copy, -0.0 included)
                s[j] = __dmul_rn(xs[0], wr[0]);
                k = 1;
            }
            for (; k < ke; ++k) {
                const double t = __dmul_rn(xs[(k - kb) * SC_LD], wr[k]);
                double hi, err;
                two_sum(s[j], t, hi, err);
                s[j] = hi;
                e[j] = __dadd_rn(e[j], err);
            }
        }
    }
    __syncthreads();   // stage the outputs in the slab: rows down, cells across, then store each cell's rows contiguously
#pragma unroll
    for (int j = 0; j < SC_RPW; ++j) {
        const int64_t r = r0 + warp + SC_NW * j;
        if (r < G) slab[(warp + SC_NW * j) * SC_LD + lane] = __dadd_rn(s[j], e[j]) / den[r];
    }
    __syncthreads();
    for (int t = threadIdx.x; t < SC_TC * SC_RB; t += SC_NT) {
        const int cell = t / SC_RB, rr = t % SC_RB;
        if (cell < ncell && r0 + rr < G) Y[r0 + rr + ldy * (c0 + cell)] = slab[rr * SC_LD + cell];
    }
    if (bad) atomicOr(flag, 1);
}

// The stencil of every row of [0, G) (see the file comment), and each row block's slab.
struct Stencil {
    std::vector<int32_t> lo, len, blo, bhi;
    std::vector<int64_t> off;
    std::vector<double> w, den;
};

void stencil_build(Stencil &t, int64_t G, const int32_t *chr_start, const int32_t *chr_len, int K, const double *st,
                   const double *sp, double W) {
    t.lo.resize((size_t)G);
    t.len.resize((size_t)G);
    t.off.resize((size_t)G);
    t.den.resize((size_t)G);
    t.w.clear();
    auto identity = [&](int64_t i) {
        t.lo[i] = (int32_t)i;
        t.len[i] = 1;
        t.off[i] = (int64_t)t.w.size();
        t.w.push_back(1.0);
        t.den[i] = 1.0;
    };
    std::vector<int64_t> around;
    std::vector<double> wv;
    int64_t pos_g = 0;
    for (int r = 0; r <= K; ++r) {
        const int64_t s0 = r < K ? chr_start[r] : G, n = r < K ? chr_len[r] : 0;
        for (; pos_g < s0; ++pos_g) identity(pos_g);
        if (n <= 0) continue;
        if (n < 2 || W < 2.0) {
            for (int64_t i = s0; i < s0 + n; ++i) identity(i);
        } else {
            const double *s = st + s0, *e = sp + s0;
            for (int64_t i = 0; i < n; ++i) {
                const double pos = (s[i] + e[i]) / 2, a = pos - W, b = pos + W;
                around.clear();
                for (int64_t j = 0; j < n; ++j)
                    if (s[j] > a && e[j] < b) around.push_back(j);
                if (around.empty()) around.push_back(i);
                const int64_t mn = around.front(), mx = around.back(), to_add = (int64_t)around.size() / 2;
                const int64_t l = std::max<int64_t>(0, mn - to_add), h = std::min<int64_t>(n - 1, mx + to_add);
                wv.assign((size_t)(mn - l), 0.1);
                for (int64_t j : around) wv.push_back(1 - std::fabs((e[j] + s[j]) / 2 - pos) / W);
                wv.insert(wv.end(), (size_t)(h - mx), 0.1);
                long double d = 0.0L;
                for (double v : wv) d += v;
                const int64_t L = h - l + 1, Lw = (int64_t)wv.size();
                t.lo[s0 + i] = (int32_t)(s0 + l);
                t.len[s0 + i] = (int32_t)L;
                t.off[s0 + i] = (int64_t)t.w.size();
                for (int64_t k = 0; k < L; ++k) t.w.push_back(wv[(size_t)(k % Lw)]);
                t.den[s0 + i] = (double)d;
            }
        }
        pos_g = s0 + n;
    }
    const int64_t nb = (G + SC_RB - 1) / SC_RB;
    t.blo.resize((size_t)nb);
    t.bhi.resize((size_t)nb);
    for (int64_t b = 0; b < nb; ++b) {
        const int64_t r0 = b * SC_RB, r1 = std::min<int64_t>(G, r0 + SC_RB);
        int64_t a = r0, z = r1 - 1;
        for (int64_t i = r0; i < r1; ++i) {
            a = std::min<int64_t>(a, t.lo[i]);
            z = std::max<int64_t>(z, (int64_t)t.lo[i] + t.len[i] - 1);
        }
        t.blo[b] = (int32_t)a;
        t.bhi[b] = (int32_t)z;
    }
}

}  // namespace sc

using namespace sc;

// X, Y device (ld >= G, Y must not overlap X); ranges and coordinates host; arguments checked by the caller.
int smooth_coords_dev(const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t G, int64_t C, const int32_t *chr_start,
                      const int32_t *chr_len, int K, const double *gene_start, const double *gene_stop, double W,
                      cudaStream_t st, const char *who) {
    Stencil t;
    try {
        stencil_build(t, G, chr_start, chr_len, K, gene_start, gene_stop, W);
    } catch (const std::bad_alloc &) {
        return set_error(ICNV_E_NOMEM, "%s: no host memory for the stencil of %lld genes", who, (long long)G);
    }
    const int64_t nb = (int64_t)t.blo.size(), nw = (int64_t)t.w.size();
    const size_t bytes = sizeof(double) * (size_t)(nw + G) + sizeof(int64_t) * (size_t)G +
                         sizeof(int32_t) * (size_t)(2 * G + 2 * nb) + 64;
    char *buf = nullptr;
    if (cudaMallocAsync((void **)&buf, bytes, st) != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NOMEM, "%s: no device memory for a stencil of %lld weights", who, (long long)nw);
    }
    double *d_w = (double *)buf, *d_den = d_w + nw;
    int64_t *d_off = (int64_t *)(d_den + G);
    int32_t *d_lo = (int32_t *)(d_off + G), *d_len = d_lo + G, *d_blo = d_len + G, *d_bhi = d_blo + nb;
    int *d_flag = (int *)(d_bhi + nb);
    auto body = [&]() -> int {
        ICNV_CUDA(cudaMemcpyAsync(d_w, t.w.data(), sizeof(double) * (size_t)nw, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_den, t.den.data(), sizeof(double) * (size_t)G, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_off, t.off.data(), sizeof(int64_t) * (size_t)G, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_lo, t.lo.data(), sizeof(int32_t) * (size_t)G, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_len, t.len.data(), sizeof(int32_t) * (size_t)G, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_blo, t.blo.data(), sizeof(int32_t) * (size_t)nb, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_bhi, t.bhi.data(), sizeof(int32_t) * (size_t)nb, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
        smooth_coords_kernel<<<dim3((unsigned)((C + SC_TC - 1) / SC_TC), (unsigned)nb), SC_NT, 0, st>>>(
            X, ldx, Y, ldy, G, C, d_lo, d_len, d_off, d_w, d_den, d_blo, d_bhi, d_flag);
        ICNV_CHECK_LAUNCH("smooth_coords_kernel");
        int h = 0;
        ICNV_CUDA(cudaMemcpyAsync(&h, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaStreamSynchronize(st));   // the host stencil is freed on return
        if (h) return set_error(ICNV_E_NONFINITE, "%s: NaN or Inf in X", who);
        return ICNV_OK;
    };
    const int rc = body();
    cudaFreeAsync(buf, st);
    return rc;
}

}  // namespace icnv
