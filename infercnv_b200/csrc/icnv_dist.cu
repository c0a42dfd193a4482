// Pairwise Euclidean distances between cells - what every `hclust(parallelDist(t(expr[, cells])))` of the reference
// asks for (R/inferCNV_tumor_subclusters.R:191,411,472,582,609; R/inferCNV_ops.R:1930,3242; R/inferCNV_heatmap.R:719,755,
// 1062,1079; parallelDist's default method "euclidean": sqrt(sum((a - b)^2)) over the genes) - SURVEY section 8(f) row 4.
//
// out[] is R's "dist" layout: the strict lower triangle by columns, i.e. for list positions a < b
//     out[n a - a (a + 1) / 2 + (b - a - 1)] = sqrt(sum_g (X[g, cells[a]] - X[g, cells[b]])^2).
//
// The sum is taken in the DIFFERENCE form, gene by gene in gene order, one fused multiply-add per term: no |a|^2 + |b|^2 -
// 2 a.b cancellation, so near-identical cells (which hclust merges first) keep full relative accuracy.  That form is two
// FP64 instructions per (pair, gene) and nothing else matters: the kernel is bound by the FP64 pipe (64 lanes per clock per
// SM on H100; its FP64 tensor path is twice that, but only for the cancelling a.b form), not by HBM - a 128 x 128 tile of pairs re-uses every value it loads
// 128 times from shared memory.
//
// One CTA = one 128 x 128 tile of the upper triangle (tiles below the diagonal exit at once), 256 threads, 8 x 8 pairs per
// thread in registers (rows ty + 16 p, columns tx + 16 q, so the 16 lanes of a half-warp read consecutive cells of the
// column tile - stride 17 doubles, bank-conflict free - and write 128 contiguous bytes of out[]).  The genes arrive 16 at a
// time per cell (128 contiguous bytes of its column) by cp.async into a double-buffered [cell][16 + 1] layout.
#include "icnv_common.cuh"

namespace icnv {

constexpr int PD_T = 128;        // cells per tile side
constexpr int PD_K = 16;         // genes per stage
constexpr int PD_LD = PD_K + 1;  // padded row (doubles)
constexpr int PD_NT = 256;

struct DistParams {
    const double *X;
    int64_t G, ldx;
    const int32_t *cells;  // n list entries, or nullptr: cells 0 .. n-1
    int64_t n;
    double *out;
    int rows;              // 1: X is observations x variables, column-major (cell a, gene g at X[a + ldx g]) - what R hands to
                           // parallelDist(); 0: genes x cells (gene g of cell c at X[g + ldx c]) - expr.data itself
};

__device__ __forceinline__ void cp_async8(void *smem_dst, const void *gsrc, bool valid) {
    unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    int sz = valid ? 8 : 0;  // src-size 0: zero-fill, nothing is read
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}

__global__ void __launch_bounds__(PD_NT, 1) pairwise_dist_kernel(const DistParams p) {
    const int bi = blockIdx.y, bj = blockIdx.x;
    if (bi > bj) return;   // the lower triangle is the upper one's mirror image
    extern __shared__ __align__(16) double pd_smem[];
    double *As = pd_smem;                          // [2][PD_T][PD_LD]
    double *Bs = pd_smem + 2 * PD_T * PD_LD;       // [2][PD_T][PD_LD]
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int64_t i0 = (int64_t)bi * PD_T, j0 = (int64_t)bj * PD_T;
    // staging: thread t copies genes (t & 15) of 8 cells of either tile per stage: 16 lanes cover one cell's 128 bytes
    const int sk = tid & 15;
    const double *srcA[8], *srcB[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
        const int row = (tid >> 4) + 16 * u;
        int64_t a = i0 + row, b = j0 + row;
        a = a < p.n ? a : p.n - 1;   // rows behind the list: any valid cell, never written
        b = b < p.n ? b : p.n - 1;
        srcA[u] = p.rows ? p.X : p.X + p.ldx * (p.cells ? (int64_t)p.cells[a] : a);
        srcB[u] = p.rows ? p.X : p.X + p.ldx * (p.cells ? (int64_t)p.cells[b] : b);
    }
    // observations x variables: a warp copies one gene of 32 consecutive cells (256 contiguous bytes); thread t takes cell
    // t & 127 of either tile and the genes (t >> 7) + 2 u of the stage
    const int rc = tid & 127, rk = tid >> 7;
    const int64_t ra = (i0 + rc < p.n) ? i0 + rc : p.n - 1, rb = (j0 + rc < p.n) ? j0 + rc : p.n - 1;
    auto issue = [&](int64_t g0, int buf) {
        double *da = As + buf * (PD_T * PD_LD), *db = Bs + buf * (PD_T * PD_LD);
        if (p.rows) {
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int k = rk + 2 * u;
                const int64_t g = g0 + k;
                const bool ok = g < p.G;
                cp_async8(da + rc * PD_LD + k, p.X + ra + p.ldx * (ok ? g : 0), ok);
                cp_async8(db + rc * PD_LD + k, p.X + rb + p.ldx * (ok ? g : 0), ok);
            }
            return;
        }
        const int64_t g = g0 + sk;
        const bool ok = g < p.G;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int row = (tid >> 4) + 16 * u;
            cp_async8(da + row * PD_LD + sk, srcA[u] + (ok ? g : 0), ok);
            cp_async8(db + row * PD_LD + sk, srcB[u] + (ok ? g : 0), ok);
        }
    };
    double acc[8][8];
#pragma unroll
    for (int pp = 0; pp < 8; ++pp)
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[pp][q] = 0.0;
    const int64_t n_st = (p.G + PD_K - 1) / PD_K;
    if (n_st > 0) {
        issue(0, 0);
        cp_async_commit();
    }
    for (int64_t s = 0; s < n_st; ++s) {
        const int buf = (int)(s & 1);
        if (s + 1 < n_st) {
            issue((s + 1) * PD_K, buf ^ 1);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const double *A = As + buf * (PD_T * PD_LD) + ty * PD_LD, *B = Bs + buf * (PD_T * PD_LD) + tx * PD_LD;
#pragma unroll
        for (int k = 0; k < PD_K; ++k) {
            double a[8], b[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                a[u] = A[u * 16 * PD_LD + k];
                b[u] = B[u * 16 * PD_LD + k];
            }
#pragma unroll
            for (int pp = 0; pp < 8; ++pp)
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const double d = a[pp] - b[q];
                    acc[pp][q] = fma(d, d, acc[pp][q]);
                }
        }
        __syncthreads();   // the buffer is refilled by the next iteration's copies
    }
#pragma unroll
    for (int pp = 0; pp < 8; ++pp) {
        const int64_t a = i0 + ty + 16 * pp;
        if (a >= p.n) continue;
        const int64_t base = p.n * a - a * (a + 1) / 2 - a - 1;   // + b
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const int64_t b = j0 + tx + 16 * q;
            if (b > a && b < p.n) p.out[base + b] = sqrt(acc[pp][q]);
        }
    }
}

}  // namespace icnv

using namespace icnv;

extern "C" {

static int launch_pairwise_dist(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n, double *out, int rows,
                                void *stream, const char *who) {
    ICNV_REQUIRE_READY();
    if (!X || G < 0 || ldx < (rows ? n : G) || n < 0 || (n >= 2 && !out) || (rows && d_cells)) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    if (n < 2) return ICNV_OK;   // an empty "dist" object
    const int64_t T = (n + PD_T - 1) / PD_T;
    if (T > 65535) return set_error(ICNV_E_UNSUPPORTED, "%s: %lld cells (limit %d)", who, (long long)n, 65535 * PD_T);
    DistParams p{X, G, ldx, d_cells, n, out, rows};
    const size_t smem = sizeof(double) * 4 * PD_T * PD_LD;
    ICNV_CUDA(cudaFuncSetAttribute(pairwise_dist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    pairwise_dist_kernel<<<dim3((unsigned)T, (unsigned)T), PD_NT, smem, pick_stream(stream)>>>(p);
    ICNV_CHECK_LAUNCH("pairwise_dist_kernel");
    return ICNV_OK;
}

int icnv_dev_pairwise_dist_f64(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n, double *out,
                               void *stream) {
    return launch_pairwise_dist(X, G, ldx, d_cells, n, out, 0, stream, "icnv_dev_pairwise_dist_f64");
}

int icnv_dev_pairwise_dist_rows_f64(const double *x, int64_t n, int64_t ldx, int64_t G, double *out, void *stream) {
    return launch_pairwise_dist(x, G, ldx, nullptr, n, out, 1, stream, "icnv_dev_pairwise_dist_rows_f64");
}

}  // extern "C"
