// Hierarchical clustering of cells - the hclust() half of every `hclust(parallelDist(t(expr[, cells])), method)` of the
// reference (R/inferCNV_tumor_subclusters.R:191,411,474,498,582,609; R/inferCNV_ops.R:1930,3242; R/inferCNV_heatmap.R:719,
// 755,1062,1079; infercnv imports fastcluster::hclust, default method "ward.D2") - K11 in DESIGN section 3.
//
// Algorithm: nearest-neighbour chain with Lance-Williams updates on a device-resident, symmetric, square FP64 matrix
// (row stride ld = n rounded up to even, so every row starts on 16 bytes).  Exact for the reducible methods, coded as
// fastcluster orders them: 0 single, 1 complete, 2 average, 3 mcquitty, 4 ward.D, 7 ward.D2 (5 centroid and 6 median are
// not reducible: ICNV_E_UNSUPPORTED).  For clusters i, j merged and any other active k (n_* = sizes):
//   single   min(d_ki, d_kj)                 complete  max(d_ki, d_kj)
//   average  (n_i d_ki + n_j d_kj) / (n_i + n_j)                 mcquitty  (d_ki + d_kj) / 2
//   ward.D   ((n_i + n_k) d_ki + (n_j + n_k) d_kj - n_k d_ij) / (n_i + n_j + n_k)
//   ward.D2  ward.D on the squared input, sqrt of every height at the end
// each evaluated in exactly this operation order with __dmul_rn / __dadd_rn / __ddiv_rn (no FMA contraction), so a plain
// C / NumPy restatement of the same rules reproduces the output bit for bit.
//
// Rules that fix the tree under ties:
//   * a chain starts at the smallest active index;
//   * the nearest neighbour of the chain tip is the strict minimum of its row over the other active clusters; the element
//     before the tip in the chain wins a tie, otherwise the smallest index does;
//   * two reciprocal nearest neighbours i < j merge into slot j, and i is deactivated;
//   * the raw merges are stably sorted by height;
//   * then converted to R's convention by a union-find in sorted order: a singleton is -(position + 1), the cluster made at
//     sorted step s is +s, and in each row the smaller node comes first with singletons numbered 0 .. n-1 and clusters
//     n .. 2n-2 (a singleton before a cluster, the older cluster first).
//
// Shape: one persistent 1024-thread CTA runs the whole chain loop.  A row scan streams the tip's row through shared memory
// in 16 KB chunks with cp.async.bulk and mbarrier completion (four stages); the arg-min is a block reduction on
// (value, index).  A merge rewrites row j (contiguous) and column j (one strided store per row) in place.  The active set
// is not compacted: every scan reads the full row, and the flags of the inactive slots (shared memory, one byte each) mask
// them out.  The stable sort (bitonic on (height, raw step) in global scratch) and the conversion to R's merge matrix run
// in the same launch.  The matrix is filled from R's condensed "dist" layout by two grid-wide kernels before it.
#include "icnv_common.cuh"
#include "icnv_linkage.cuh"

#include <algorithm>

namespace icnv {
namespace hc {

constexpr int HC_NT = 1024;
constexpr int HC_S = 4;             // pipeline stages of the row scan
constexpr int HC_CH = 2048;         // doubles per chunk (16 KB)
constexpr int64_t HC_NMAX = 65536;

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(void *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(void *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, void *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(void *bar, unsigned parity) {
    unsigned ok = 0;
    const unsigned a = smem_u32(bar);
    while (!ok) {
        asm volatile(
            "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
            : "=r"(ok)
            : "r"(a), "r"(parity)
            : "memory");
    }
}
// generic-proxy stores to global memory (the row / column update) made visible to the bulk copies of later scans
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.global;\n" ::: "memory"); }

struct HcParams {
    double *M;               // n x ld, symmetric, diagonal +inf
    int64_t n, ld;
    int method;
    int32_t *chain;          // n
    int32_t *size;           // n
    int32_t *raw_i, *raw_j;  // n - 1: slots merged at raw step t (i < j)
    double *raw_h;           // n - 1
    unsigned long long *skey;  // P >= n - 1 (power of two): sort keys
    int32_t *sidx;           // P: raw step of each key
    int32_t *uf;             // n: union-find parent of each slot
    int32_t *node;           // n: node number of each union-find root
    int32_t *merge;          // (n - 1) x 2, column-major
    double *height;          // n - 1
    int P;
    // a batched launch runs one linkage per CTA: member z = blockIdx.x works on M + z sM, raw_h / skey + z s8,
    // chain .. sidx + z s4, merge + z 2 (n - 1) and height + z (n - 1)
    int64_t sM, s8, s4;
    // or, members of different n (K17): member z = blockIdx.x takes n, ld, P and its offsets from mem[z] (raw_h and chain
    // are then the bases of the 8-byte and the int32 scratch)
    const HcMember *mem;
};

// Condensed "dist" rows [a0, a1) -> upper triangle of M (squared for ward.D2), diagonal +inf.  src holds the entries of
// those rows back to back (row a starts at off(a) - off(a0), off(a) = n a - a (a + 1) / 2).  flag |= 1 on NaN / Inf.
__global__ void __launch_bounds__(256) hclust_fill_kernel(const double *__restrict__ src, int64_t a0, int64_t a1, int64_t n,
                                                          int64_t ld, int square, double *__restrict__ M, int *flag) {
    const int64_t base = n * a0 - a0 * (a0 + 1) / 2;
    bool bad = false;
    for (int64_t a = a0 + blockIdx.x; a < a1; a += gridDim.x) {
        const double *row = src + (n * a - a * (a + 1) / 2 - base) - (a + 1);   // row[b], b > a
        double *dst = M + a * ld;
        for (int64_t b = a + 1 + threadIdx.x; b < n; b += blockDim.x) {
            double v = row[b];
            bad |= !is_finite_d(v);
            dst[b] = square ? __dmul_rn(v, v) : v;
        }
        if (threadIdx.x == 0) dst[a] = __longlong_as_double(0x7ff0000000000000ll);
    }
    if (bad) atomicOr(flag, 1);
}

// lower triangle from the upper one, 32 x 32 tiles through shared memory
__global__ void __launch_bounds__(256) hclust_mirror_kernel(double *M, int64_t n, int64_t ld) {
    __shared__ double t[32][33];
    const int64_t bi = blockIdx.y, bj = blockIdx.x;   // tile (bi, bj) of the upper triangle -> tile (bj, bi)
    if (bi > bj) return;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int r = ty; r < 32; r += 8) {
        const int64_t a = bi * 32 + r, b = bj * 32 + tx;
        t[r][tx] = (a < n && b < n && b > a) ? M[a * ld + b] : 0.0;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int64_t b = bj * 32 + r, a = bi * 32 + tx;   // M[b, a] = M[a, b] for a < b
        if (a < n && b < n && b > a) M[b * ld + a] = t[tx][r];
    }
}

__global__ void __launch_bounds__(HC_NT, 1) hclust_nn_chain_kernel(const HcParams p0) {
    HcParams p = p0;
    {   // both layouts keep a member's scratch as [raw_h | skey] (n + P doubles) and [chain | size | raw_i | raw_j | uf | node |
        // sidx] (6 n + P int32) from its two bases
        int64_t oM, o8, o4, oo;
        if (p0.mem) {
            const HcMember m = p0.mem[blockIdx.x];
            p.n = m.n;
            p.ld = m.ld;
            p.P = m.P;
            oM = m.m_off;
            o8 = m.s8_off;
            o4 = m.s4_off;
            oo = m.out_off;
        } else {
            const int64_t z = blockIdx.x;
            oM = z * p0.sM;
            o8 = z * p0.s8;
            o4 = z * p0.s4;
            oo = z * (p0.n - 1);
        }
        const int64_t n = p.n;
        p.M += oM;
        p.raw_h += o8;
        p.skey = reinterpret_cast<unsigned long long *>(p.raw_h + n);
        p.chain += o4;
        p.size = p.chain + n;
        p.raw_i = p.chain + 2 * n;
        p.raw_j = p.chain + 3 * n;
        p.uf = p.chain + 4 * n;
        p.node = p.chain + 5 * n;
        p.sidx = p.chain + 6 * n;
        p.merge += 2 * oo;
        p.height += oo;
    }
    extern __shared__ __align__(16) unsigned char hc_smem[];
    double *buf = reinterpret_cast<double *>(hc_smem);                    // [HC_S][HC_CH]
    unsigned char *active = hc_smem + sizeof(double) * HC_S * HC_CH;      // [n]
    __shared__ __align__(8) unsigned long long s_bar[2 * HC_S];
    __shared__ unsigned long long s_wkey[HC_NT / 32];
    __shared__ int s_widx[HC_NT / 32];
    __shared__ int s_a, s_p, s_len, s_lo, s_merged, s_done, s_i, s_j;
    __shared__ int s_steps;
    __shared__ double s_dprev, s_dij, s_ni, s_nj;

    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int64_t n = p.n, ld = p.ld;
    const int nch = (int)((ld + HC_CH - 1) / HC_CH);
    for (int64_t k = tid; k < n; k += HC_NT) {
        active[k] = 1;
        p.size[k] = 1;
    }
    if (tid == 0) {
        for (int s = 0; s < HC_S; ++s) mbar_init(&s_bar[2 * s], 1);
        s_len = 0;
        s_lo = 0;
        s_steps = 0;
    }
    __syncthreads();
    unsigned long long g = 0;   // chunks consumed so far (every thread counts the same): stage g % HC_S, parity (g / HC_S) & 1
    for (;;) {
        if (tid == 0) {
            s_done = s_steps == n - 1;
            if (!s_done) {
                if (s_len == 0) {
                    while (!active[s_lo]) ++s_lo;
                    p.chain[0] = s_lo;
                    s_len = 1;
                }
                s_a = p.chain[s_len - 1];
                s_p = s_len >= 2 ? p.chain[s_len - 2] : -1;
                s_dprev = 0.0;
            }
        }
        __syncthreads();
        if (s_done) break;
        const int a = s_a, pv = s_p;
        const double *row = p.M + (int64_t)a * ld;
        auto issue = [&](int c, unsigned long long gc) {
            const int s = (int)(gc % HC_S);
            const int64_t c0 = (int64_t)c * HC_CH;
            const unsigned bytes = (unsigned)(sizeof(double) * (size_t)min((int64_t)HC_CH, ld - c0));
            mbar_expect_tx(&s_bar[2 * s], bytes);
            bulk_g2s(buf + s * HC_CH, row + c0, bytes, &s_bar[2 * s]);
        };
        if (tid == 0)
            for (int c = 0; c < nch && c < HC_S; ++c) issue(c, g + c);
        unsigned long long bk = ~0ull;
        int bi = 0x7fffffff;
        for (int c = 0; c < nch; ++c, ++g) {
            const int s = (int)(g % HC_S);
            mbar_wait(&s_bar[2 * s], (unsigned)((g / HC_S) & 1));
            const double *v = buf + s * HC_CH;
            const int64_t c0 = (int64_t)c * HC_CH;
            const int m = (int)min((int64_t)HC_CH, n - c0);
            for (int e = tid; e < m; e += HC_NT) {
                const int k = (int)(c0 + e);
                if (k == pv) s_dprev = v[e];
                if (!active[k] || k == a) continue;
                const unsigned long long kk = dkey(v[e]);
                if (kk < bk) { bk = kk; bi = k; }   // ascending k: the first of equal values stays
            }
            __syncthreads();   // every thread is done with stage s
            if (tid == 0 && c + HC_S < nch) issue(c + HC_S, g + HC_S);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long ok = __shfl_xor_sync(0xffffffffu, bk, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (key_less(ok, oi, bk, bi)) { bk = ok; bi = oi; }
        }
        if (lane == 0) { s_wkey[wid] = bk; s_widx[wid] = bi; }
        __syncthreads();
        if (wid == 0) {
            bk = s_wkey[lane];
            bi = s_widx[lane];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const unsigned long long ok = __shfl_xor_sync(0xffffffffu, bk, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (key_less(ok, oi, bk, bi)) { bk = ok; bi = oi; }
            }
            if (tid == 0) {
                int b = bi;
                if (pv >= 0 && dkey(s_dprev) == bk) b = pv;   // the element before the tip wins a tie
                s_merged = b == pv;
                if (b == pv) {
                    const int i = a < b ? a : b, j = a < b ? b : a;
                    p.raw_i[s_steps] = i;
                    p.raw_j[s_steps] = j;
                    p.raw_h[s_steps] = s_dprev;
                    s_dij = s_dprev;
                    s_i = i;
                    s_j = j;
                    s_ni = (double)p.size[i];
                    s_nj = (double)p.size[j];
                    p.size[j] = p.size[i] + p.size[j];
                    active[i] = 0;
                    s_len -= 2;
                    s_steps += 1;
                } else {
                    if (s_len == (int)n) s_len = 0;   // cannot happen in exact arithmetic; keeps the chain in bounds
                    p.chain[s_len++] = b;
                }
            }
        }
        __syncthreads();
        if (s_merged) {
            const int i = s_i, j = s_j;
            const double dij = s_dij, ni = s_ni, nj = s_nj;
            const double *ri = p.M + (int64_t)i * ld;
            double *rj = p.M + (int64_t)j * ld;
            for (int64_t k = tid; k < n; k += HC_NT) {
                if (!active[k] || k == j) continue;
                const double w = lance_williams(p.method, ri[k], rj[k], dij, ni, nj, (double)p.size[k]);
                rj[k] = w;
                p.M[k * ld + j] = w;
            }
            fence_proxy_async();
        }
    }

    // ---- stable sort of the raw merges by height, then R's merge matrix ----
    linkage_finish<HC_NT>(n, p.method, p.P, p.raw_h, p.raw_i, p.raw_j, p.skey, p.sidx, p.uf, p.node, p.merge, p.height);
}

}  // namespace hc
}  // namespace icnv

namespace icnv {

using namespace hc;

// Checks shared by the entry points; ICNV_OK when the linkage can run.
int hclust_check_args(int64_t n, int method, const char *who) {
    if (n < 2) return set_error(ICNV_E_BAD_ARG, "%s: n = %lld (at least 2 observations)", who, (long long)n);
    if (method == 5 || method == 6)
        return set_error(ICNV_E_UNSUPPORTED, "%s: method %d (centroid / median) is not reducible", who, method);
    if (method < 0 || method > 7) return set_error(ICNV_E_BAD_ARG, "%s: unknown method code %d", who, method);
    if (n > HC_NMAX) return set_error(ICNV_E_UNSUPPORTED, "%s: n = %lld (limit %lld)", who, (long long)n, (long long)HC_NMAX);
    return ICNV_OK;
}

// The square matrix of n observations: n x ld doubles, ld = n rounded up to even.
int64_t hclust_ld(int64_t n) { return (n + 1) & ~(int64_t)1; }

// Fill rows [a0, a1) of M from the condensed entries of those rows in src (device), flag |= 1 on a non-finite entry.
static int hclust_fill_rows(const double *src, int64_t a0, int64_t a1, int64_t n, int method, double *M, int *flag,
                            cudaStream_t st) {
    if (a1 <= a0) return ICNV_OK;
    const int64_t ld = hclust_ld(n);
    const unsigned grid = (unsigned)std::min<int64_t>(a1 - a0, 4096);
    hclust_fill_kernel<<<grid, 256, 0, st>>>(src, a0, a1, n, ld, method == 7, M, flag);
    ICNV_CHECK_LAUNCH("hclust_fill_kernel");
    return ICNV_OK;
}

// B linkages of n observations in one launch, one CTA (one SM) each: member z's filled matrix (symmetric, diagonal +inf,
// squared for ward.D2) at M + z n ld, its merge / height at merge + z 2 (n - 1) / height + z (n - 1).  Every member is
// the same function of its own matrix as a single-tree launch (B = 1).  The scratch is freed on `st` after the launch.
int hclust_batch(double *M, int64_t n, int method, int B, int32_t *merge, double *height, cudaStream_t st) {
    const int64_t ld = hclust_ld(n);
    int P = 1;
    while (P < n - 1) P <<= 1;
    // scratch of a linkage: chain, size, raw_i, raw_j, uf, node, sidx (int32) and raw_h, skey (8 bytes)
    const int64_t s8 = n + P, s4 = 6 * n + P;
    const size_t b8 = sizeof(double) * (size_t)s8 * (size_t)B, b4 = sizeof(int32_t) * (size_t)s4 * (size_t)B;
    char *w = nullptr;
    ICNV_CUDA(cudaMallocAsync((void **)&w, b8 + b4 + 64, st));
    HcParams q{};
    q.M = M;
    q.n = n;
    q.ld = ld;
    q.method = method;
    q.raw_h = (double *)w;            // the kernel derives skey and size .. sidx from these two bases
    q.chain = (int32_t *)(w + b8);
    q.merge = merge;
    q.height = height;
    q.P = P;
    q.sM = n * ld;
    q.s8 = s8;
    q.s4 = s4;
    q.mem = nullptr;
    const size_t smem = sizeof(double) * HC_S * HC_CH + (size_t)((n + 15) & ~15);
    ICNV_CUDA(cudaFuncSetAttribute(hclust_nn_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    hclust_nn_chain_kernel<<<B, HC_NT, smem, st>>>(q);
    ICNV_CHECK_LAUNCH("hclust_nn_chain_kernel");
    ICNV_CUDA(cudaFreeAsync(w, st));
    return ICNV_OK;
}

// K17: B linkages of members of different n in one launch, one CTA each (member z = d_mem[z], device).  The filled
// matrices are at M + m_off, the scratch at w8 + s8_off / w4 + s4_off, the results at merge / height + the member's
// out_off.  Dynamic shared memory is sized by n_max, the largest member's n.  Every member is the same function of its
// own matrix as a single-tree launch.
int hclust_member_batch(const HcMember *d_mem, int B, int64_t n_max, int method, double *M, double *w8, int32_t *w4,
                        int32_t *merge, double *height, cudaStream_t st) {
    if (B <= 0) return ICNV_OK;
    HcParams q{};
    q.M = M;
    q.n = n_max;
    q.ld = hclust_ld(n_max);
    q.method = method;
    q.raw_h = w8;
    q.chain = w4;
    q.merge = merge;
    q.height = height;
    q.mem = d_mem;
    const size_t smem = sizeof(double) * HC_S * HC_CH + (size_t)((n_max + 15) & ~15);
    ICNV_CUDA(cudaFuncSetAttribute(hclust_nn_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    hclust_nn_chain_kernel<<<B, HC_NT, smem, st>>>(q);
    ICNV_CHECK_LAUNCH("hclust_nn_chain_kernel");
    return ICNV_OK;
}

// Bytes of device scratch hclust_batch allocates per member.
size_t hclust_batch_scratch(int64_t n) {
    int64_t P = 1;
    while (P < n - 1) P <<= 1;
    return sizeof(double) * (size_t)(n + P) + sizeof(int32_t) * (size_t)(6 * n + P);
}

// Mirror the upper triangle, check the flag (one synchronisation), then enqueue the linkage.  M is freed on `st` after it.
static int hclust_run(double *M, int64_t n, int method, int *d_flag, int32_t *merge, double *height, cudaStream_t st) {
    const int64_t ld = hclust_ld(n);
    const unsigned T = (unsigned)((n + 31) / 32);
    hclust_mirror_kernel<<<dim3(T, T), 256, 0, st>>>(M, n, ld);
    ICNV_CHECK_LAUNCH("hclust_mirror_kernel");
    int h_flag = 0;
    ICNV_CUDA(cudaMemcpyAsync(&h_flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    if (h_flag) return set_error(ICNV_E_NONFINITE, "hclust: NaN or Inf in the dissimilarities");
    return hclust_batch(M, n, method, 1, merge, height, st);
}

}  // namespace icnv

namespace icnv {

// The bodies of icnv_dev_hclust_f64 / icnv_hclust_f64 (icnv_api.cu holds the exported entry points).

int hclust_dev(const double *d_dist, int64_t n, int method, int32_t *merge, double *height, void *stream) {
    ICNV_REQUIRE_READY();
    int rc = hclust_check_args(n, method, "icnv_dev_hclust_f64");
    if (rc) return rc;
    if (!d_dist || !merge || !height) return set_error(ICNV_E_BAD_ARG, "icnv_dev_hclust_f64: bad argument");
    cudaStream_t st = pick_stream(stream);
    const int64_t ld = hclust_ld(n);
    double *M = nullptr;
    int *d_flag = nullptr;
    if (cudaMallocAsync((void **)&M, sizeof(double) * (size_t)n * (size_t)ld + 16, st) != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NOMEM, "icnv_dev_hclust_f64: no room for the %lld x %lld matrix", (long long)n, (long long)n);
    }
    d_flag = (int *)(M + (size_t)n * (size_t)ld);
    if (cudaMemsetAsync(d_flag, 0, sizeof(int), st) != cudaSuccess) rc = set_error(ICNV_E_CUDA, "icnv_dev_hclust_f64: memset failed");
    if (!rc) rc = hclust_fill_rows(d_dist, 0, n, n, method, M, d_flag, st);
    if (!rc) rc = hclust_run(M, n, method, d_flag, merge, height, st);
    cudaFreeAsync(M, st);
    return rc;
}

/* hclust on a host "dist" vector: the square matrix is filled slab by slab - whole rows of the condensed vector, copied
 * from the caller's (pageable) memory through two page-locked slabs and two device slabs - so the device holds n^2
 * doubles plus the slab pair, never the whole condensed vector as well. */
int hclust_host(const double *d, int64_t n, int method, int32_t *merge, double *height, int32_t *order) {
    ICNV_REQUIRE_READY();
    Ctx &c = ctx();
    std::lock_guard<std::mutex> lk(c.mu);
    ICNV_CUDA(cudaSetDevice(c.device));
    cudaStream_t st = c.stream;
    int rc = hclust_check_args(n, method, "icnv_hclust_f64");
    if (rc) return rc;
    if (!d || !merge || !height || !order) return set_error(ICNV_E_BAD_ARG, "icnv_hclust_f64: bad argument");
    const int64_t ld = hclust_ld(n), nm = n - 1, total = n * (n - 1) / 2;
    const int64_t slab = std::min<int64_t>((int64_t)8 << 20, total);   // doubles per slab (64 MB at most); a row is shorter
    double *M = nullptr, *pin[2] = {nullptr, nullptr};
    if (cudaMallocAsync((void **)&M, sizeof(double) * ((size_t)n * (size_t)ld + 2), st) != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NOMEM, "icnv_hclust_f64: no room for the %lld x %lld matrix", (long long)n, (long long)n);
    }
    int *d_flag = (int *)(M + (size_t)n * (size_t)ld);
    int32_t *d_merge = nullptr;
    double *d_height = nullptr;
    auto body = [&]() -> int {
        ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
        d_height = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)nm + sizeof(int32_t) * 2 * (size_t)nm);
        if (!d_height) return ICNV_E_NOMEM;
        d_merge = (int32_t *)(d_height + nm);
        for (int b = 0; b < 2; ++b) {
            if (cudaHostAlloc((void **)&pin[b], sizeof(double) * (size_t)slab, cudaHostAllocPortable) != cudaSuccess) {
                pin[b] = nullptr;
                cudaGetLastError();
                return set_error(ICNV_E_NOMEM, "icnv_hclust_f64: cudaHostAlloc of the staging slab failed");
            }
        }
        int64_t a0 = 0;
        int b = 0;
        while (a0 < n) {   // rows [a0, a1) of the condensed vector per slab (the last row holds only its diagonal)
            const int64_t off0 = n * a0 - a0 * (a0 + 1) / 2;
            int64_t a1 = a0;
            while (a1 < n && (n * (a1 + 1) - (a1 + 1) * (a1 + 2) / 2) - off0 <= slab) ++a1;
            const size_t cnt = (size_t)((n * a1 - a1 * (a1 + 1) / 2) - off0);
            double *dev = (double *)scratch(SLOT_SLAB_IN0 + b, sizeof(double) * (size_t)slab);
            if (!dev) return ICNV_E_NOMEM;
            ICNV_CUDA(cudaEventSynchronize(c.ev_h2d[b]));   // the copy of two slabs ago has read this staging slab
            memcpy(pin[b], d + off0, sizeof(double) * cnt);
            ICNV_CUDA(cudaMemcpyAsync(dev, pin[b], sizeof(double) * cnt, cudaMemcpyHostToDevice, st));
            ICNV_CUDA(cudaEventRecord(c.ev_h2d[b], st));
            int r = hclust_fill_rows(dev, a0, a1, n, method, M, d_flag, st);
            if (r) return r;
            a0 = a1;
            b ^= 1;
        }
        return hclust_run(M, n, method, d_flag, d_merge, d_height, st);
    };
    rc = body();
    cudaFreeAsync(M, st);
    if (!rc) {
        if (cudaMemcpyAsync(height, d_height, sizeof(double) * (size_t)nm, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaMemcpyAsync(merge, d_merge, sizeof(int32_t) * 2 * (size_t)nm, cudaMemcpyDeviceToHost, st) != cudaSuccess)
            rc = set_error(ICNV_E_CUDA, "icnv_hclust_f64: copy of the result failed");
    }
    const cudaError_t e = cudaStreamSynchronize(st);
    for (double *p : pin)
        if (p) cudaFreeHost(p);
    if (rc) return rc;
    if (e != cudaSuccess) return set_error(ICNV_E_CUDA, "icnv_hclust_f64: %s", cudaGetErrorString(e));
    return icnv_hclust_order(merge, n, order);
}

}  // namespace icnv
