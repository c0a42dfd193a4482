// Hierarchical clustering past the square matrix's reach - K19 in DESIGN section 3.  The same nearest-neighbour chain as K11
// (icnv_hclust.cu: methods, Lance-Williams arithmetic, tie rules, sort and merge convention, all shared through
// icnv_linkage.cuh), run on the packed strict lower triangle in R's "dist" layout instead of an n x n matrix: half the
// memory, so about 130 000 observations fit an 80 GB device where K11 stops at 65 536.
//
// Layout: entry (i, j), i > j, at T[j n - j (j + 1) / 2 + (i - j - 1)] = T[tri_col(j) + i] (64-bit offsets) - column j holds
// the rows below the diagonal back to back, exactly the caller's "dist" vector (the host entry copies it in unchanged).
//
// Row scan of the chain tip a: the entries d(a, k), k > a, are one contiguous run (column a); the entries k < a are a
// gather, one from each column k (stride n - k - 1 doubles between consecutive k).  One persistent 1024-thread CTA runs the
// chain, as K11 does; every thread keeps HT_U independent loads in flight (k = k0 + u 1024 + tid, u < HT_U, all issued
// before the first is compared), so the SM has up to 8192 outstanding 8-byte loads to cover the gather's latency.  Slots
// already merged away are not read at all (their bit in the shared active mask is clear), so the gathered half shrinks as
// the tree grows.  A merge of i < j into j rewrites the active entries d(j, k) from d(i, k) and d(j, k) - the same two
// halves per slot - with HT_UM slots (three loads each: d(i, k), d(j, k), size k) in flight per thread; HT_U of them
// would not fit the 64 registers a 1024-thread CTA leaves a thread.  Per thread the k are visited in ascending order and the block
// reduction orders (key, index), so the arg-min and every tie resolve as in K11's scan.
//
// Per-linkage state: the active mask is one bit per slot in dynamic shared memory ((n + 31) / 32 words: 4 KB at 130 000),
// the chain / sizes / raw merges and the sort keys are global (n + P doubles, 6 n + P int32, P = power of two >= n - 1).
#include "icnv_common.cuh"
#include "icnv_linkage.cuh"

#include <algorithm>

namespace icnv {

namespace sc {   // icnv_subclusters.cu
int check_indices(const int32_t *d_idx, int64_t n, int64_t lim, int *flag, cudaStream_t st);
}

namespace ht {

constexpr int HT_NT = 1024;
constexpr int HT_U = 8;                        // loads in flight per thread in a row scan
constexpr int HT_UM = 4;                       // slots per thread and batch in a merge (three loads each)
constexpr int64_t HT_NMAX = (int64_t)1 << 30;  // int32 slots and sort indices; far beyond any device's memory
constexpr size_t HT_HEADROOM = (size_t)256 << 20;   // free memory left to the runtime

struct HtParams {
    double *T;               // the prepared triangle (squared for ward.D2)
    int64_t n;
    int method;
    int32_t *chain, *size, *raw_i, *raw_j, *uf, *node, *sidx;   // n each, sidx P
    double *raw_h;           // n - 1
    unsigned long long *skey;  // P
    int P;
    int32_t *merge;          // (n - 1) x 2, column-major
    double *height;          // n - 1
};

// entry (i, j), i > j, is T[tri_col(n, j) + i]
__device__ __forceinline__ int64_t tri_col(int64_t n, int64_t j) { return j * n - j * (j + 1) / 2 - j - 1; }

// dst[e] = src[e] (squared for ward.D2) over the whole triangle; flag |= 1 on NaN / Inf.  src may be dst.
__global__ void __launch_bounds__(256) hclust_tri_prepare_kernel(const double *src, double *dst, int64_t len, int square,
                                                                 int *flag) {
    bool bad = false;
    for (int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x; e < len; e += (int64_t)gridDim.x * 256) {
        const double v = src[e];
        bad |= !is_finite_d(v);
        dst[e] = square ? __dmul_rn(v, v) : v;
    }
    if (bad) atomicOr(flag, 1);
}

__global__ void __launch_bounds__(HT_NT, 1) hclust_tri_kernel(const HtParams p) {
    extern __shared__ __align__(16) unsigned char ht_smem[];
    unsigned *act = reinterpret_cast<unsigned *>(ht_smem);   // [(n + 31) / 32]: bit k & 31 of word k >> 5 = slot k active
    __shared__ unsigned long long s_wkey[HT_NT / 32];
    __shared__ int s_widx[HT_NT / 32];
    __shared__ int s_a, s_p, s_len, s_lo, s_merged, s_done, s_i, s_j;
    __shared__ int s_steps;
    __shared__ double s_dprev, s_dij, s_ni, s_nj;

    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int64_t n = p.n, nw = (n + 31) / 32;
    double *T = p.T;
    for (int64_t w = tid; w < nw; w += HT_NT) act[w] = (w < nw - 1 || (n & 31) == 0) ? ~0u : (1u << (n & 31)) - 1u;
    for (int64_t k = tid; k < n; k += HT_NT) p.size[k] = 1;
    if (tid == 0) {
        s_len = 0;
        s_lo = 0;
        s_steps = 0;
    }
    __syncthreads();
    auto active = [&](int64_t k) { return (act[k >> 5] >> (k & 31)) & 1u; };
    for (;;) {
        if (tid == 0) {
            s_done = s_steps == n - 1;
            if (!s_done) {
                if (s_len == 0) {
                    while (!active(s_lo)) ++s_lo;
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
        const int64_t a = s_a;
        const int pv = s_p;
        const int64_t ca = tri_col(n, a);
        unsigned long long bk = ~0ull;
        int bi = 0x7fffffff;
        for (int64_t k0 = 0; k0 < n; k0 += (int64_t)HT_NT * HT_U) {
            double v[HT_U];
            bool ok[HT_U];
#pragma unroll
            for (int u = 0; u < HT_U; ++u) {   // every load of the batch is issued before any is used
                const int64_t k = k0 + (int64_t)u * HT_NT + tid;
                ok[u] = k < n && k != a && active(k);
                v[u] = ok[u] ? T[k < a ? tri_col(n, k) + a : ca + k] : 0.0;
            }
#pragma unroll
            for (int u = 0; u < HT_U; ++u) {   // ascending k: the first of equal values stays
                if (!ok[u]) continue;
                const int k = (int)(k0 + (int64_t)u * HT_NT + tid);
                if (k == pv) s_dprev = v[u];
                const unsigned long long kk = dkey(v[u]);
                if (kk < bk) { bk = kk; bi = k; }
            }
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
                    const int i = (int)a < b ? (int)a : b, j = (int)a < b ? b : (int)a;
                    p.raw_i[s_steps] = i;
                    p.raw_j[s_steps] = j;
                    p.raw_h[s_steps] = s_dprev;
                    s_dij = s_dprev;
                    s_i = i;
                    s_j = j;
                    s_ni = (double)p.size[i];
                    s_nj = (double)p.size[j];
                    p.size[j] = p.size[i] + p.size[j];
                    act[i >> 5] &= ~(1u << (i & 31));
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
            const int64_t i = s_i, j = s_j;
            const double dij = s_dij, ni = s_ni, nj = s_nj;
            const int64_t ci = tri_col(n, i), cj = tri_col(n, j);
            for (int64_t k0 = 0; k0 < n; k0 += (int64_t)HT_NT * HT_UM) {
                double di[HT_UM], dj[HT_UM], nk[HT_UM];
                int64_t oj[HT_UM];
                bool ok[HT_UM];
#pragma unroll
                for (int u = 0; u < HT_UM; ++u) {   // i is inactive already: k != i
                    const int64_t k = k0 + (int64_t)u * HT_NT + tid;
                    ok[u] = k < n && k != j && active(k);
                    oj[u] = k < j ? tri_col(n, k) + j : cj + k;
                    di[u] = ok[u] ? T[k < i ? tri_col(n, k) + i : ci + k] : 0.0;
                    dj[u] = ok[u] ? T[oj[u]] : 0.0;
                    nk[u] = ok[u] ? (double)p.size[k] : 0.0;
                }
#pragma unroll
                for (int u = 0; u < HT_UM; ++u)
                    if (ok[u]) T[oj[u]] = lance_williams(p.method, di[u], dj[u], dij, ni, nj, nk[u]);
            }
        }
    }
    linkage_finish<HT_NT>(n, p.method, p.P, p.raw_h, p.raw_i, p.raw_j, p.skey, p.sidx, p.uf, p.node, p.merge, p.height);
}

int64_t sort_size(int64_t n) {
    int64_t P = 1;
    while (P < n - 1) P <<= 1;
    return P;
}

// device bytes of the triangle, and of the linkage's scratch (with the non-finite flag)
size_t tri_bytes(int64_t n) { return sizeof(double) * (size_t)(n * (n - 1) / 2); }
size_t work_bytes(int64_t n) {
    const int64_t P = sort_size(n);
    return sizeof(double) * (size_t)(n + P) + sizeof(int32_t) * (size_t)(6 * n + P) + 256;
}
size_t mask_bytes(int64_t n) { return (sizeof(unsigned) * (size_t)((n + 31) / 32) + 15) & ~(size_t)15; }

}  // namespace ht

using namespace ht;

// Checks on n and the method, before anything else.
int hclust_tri_check(int64_t n, int method, const char *who) {
    if (n < 2) return set_error(ICNV_E_BAD_ARG, "%s: n = %lld (at least 2 observations)", who, (long long)n);
    if (method == 5 || method == 6)
        return set_error(ICNV_E_UNSUPPORTED, "%s: method %d (centroid / median) is not reducible", who, method);
    if (method < 0 || method > 7) return set_error(ICNV_E_BAD_ARG, "%s: unknown method code %d", who, method);
    if (n > HT_NMAX) return set_error(ICNV_E_NOMEM, "%s: n = %lld observations cannot fit a device", who, (long long)n);
    return ICNV_OK;
}

// ICNV_OK when the triangle of n observations, the linkage's scratch and `extra` more bytes fit the free device memory
// (less 256 MB for the runtime) and the active mask fits shared memory; otherwise ICNV_E_NOMEM.  Allocates nothing.
int hclust_tri_room(int64_t n, size_t extra, const char *who) {
    size_t free_b = 0, total_b = 0;
    ICNV_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const size_t need = tri_bytes(n) + work_bytes(n) + extra + HT_HEADROOM;
    if (need > free_b)
        return set_error(ICNV_E_NOMEM, "%s: %lld observations need %.2f GB of device memory, %.2f GB are free", who,
                         (long long)n, need / 1e9, free_b / 1e9);
    if (mask_bytes(n) > (size_t)ctx().smem_optin)
        return set_error(ICNV_E_NOMEM, "%s: the active mask of %lld observations exceeds shared memory", who, (long long)n);
    return ICNV_OK;
}

// Prepare the triangle T (device, n (n - 1) / 2 entries + an int flag behind them) from src (device; may be T), check it
// (one synchronisation of `st`), then enqueue the linkage; its scratch is freed on `st` after it.
static int tri_prepare_and_link(const double *src, double *T, int64_t n, int method, int32_t *merge, double *height,
                                cudaStream_t st, const char *who) {
    const int64_t len = n * (n - 1) / 2;
    int *d_flag = (int *)(T + len);
    ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
    const unsigned grid = (unsigned)std::min<int64_t>((len + 255) / 256, (int64_t)ctx().sm_count * 8);
    hclust_tri_prepare_kernel<<<grid, 256, 0, st>>>(src, T, len, method == 7, d_flag);
    ICNV_CHECK_LAUNCH("hclust_tri_prepare_kernel");
    int h_flag = 0;
    ICNV_CUDA(cudaMemcpyAsync(&h_flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    if (h_flag) return set_error(ICNV_E_NONFINITE, "%s: NaN or Inf in the dissimilarities", who);
    const int64_t P = sort_size(n);
    char *w = nullptr;
    if (cudaMallocAsync((void **)&w, work_bytes(n), st) != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NOMEM, "%s: no room for the linkage's scratch", who);
    }
    HtParams q{};
    q.T = T;
    q.n = n;
    q.method = method;
    q.raw_h = (double *)w;
    q.skey = (unsigned long long *)(q.raw_h + n);
    q.chain = (int32_t *)(w + sizeof(double) * (size_t)(n + P));
    q.size = q.chain + n;
    q.raw_i = q.chain + 2 * n;
    q.raw_j = q.chain + 3 * n;
    q.uf = q.chain + 4 * n;
    q.node = q.chain + 5 * n;
    q.sidx = q.chain + 6 * n;
    q.P = (int)P;
    q.merge = merge;
    q.height = height;
    const size_t smem = mask_bytes(n);
    int rc = ICNV_OK;
    if (cudaFuncSetAttribute(hclust_tri_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
        cudaGetLastError();
        rc = set_error(ICNV_E_CUDA, "%s: cudaFuncSetAttribute failed", who);
    } else {
        hclust_tri_kernel<<<1, HT_NT, smem, st>>>(q);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) rc = set_error(ICNV_E_CUDA, "launch of hclust_tri_kernel failed: %s", cudaGetErrorString(e));
        else count_launch();
    }
    cudaFreeAsync(w, st);
    return rc;
}

// The bodies of icnv_dev_hclust_tri_f64 / icnv_hclust_tri_f64 / icnv_dev_cluster_cells_f64 (icnv_api.cu holds the exported
// entry points and the host half of icnv_cluster_cells_f64).

int hclust_tri_dev(const double *d_dist, int64_t n, int method, int32_t *merge, double *height, void *stream,
                   const char *who) {
    ICNV_REQUIRE_READY();
    int rc = hclust_tri_check(n, method, who);
    if (rc) return rc;
    if (!d_dist || !merge || !height) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    if ((rc = hclust_tri_room(n, 0, who))) return rc;
    cudaStream_t st = pick_stream(stream);
    double *T = nullptr;
    if (cudaMallocAsync((void **)&T, tri_bytes(n) + 16, st) != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NOMEM, "%s: no room for the triangle of %lld observations", who, (long long)n);
    }
    rc = tri_prepare_and_link(d_dist, T, n, method, merge, height, st, who);
    cudaFreeAsync(T, st);
    return rc;
}

/* hclust on a host "dist" vector: the vector is the triangle's layout, so it goes up unchanged in 64 MB pieces through two
 * page-locked slabs straight into the device triangle - no second full copy on either side. */
int hclust_tri_host(const double *d, int64_t n, int method, int32_t *merge, double *height, int32_t *order, const char *who) {
    ICNV_REQUIRE_READY();
    Ctx &c = ctx();
    std::lock_guard<std::mutex> lk(c.mu);
    ICNV_CUDA(cudaSetDevice(c.device));
    cudaStream_t st = c.stream;
    int rc = hclust_tri_check(n, method, who);
    if (rc) return rc;
    if (!d || !merge || !height || !order) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    const int64_t nm = n - 1, total = n * (n - 1) / 2;
    const size_t out_bytes = (sizeof(double) + 2 * sizeof(int32_t)) * (size_t)nm;
    if ((rc = hclust_tri_room(n, out_bytes > c.slot_bytes[SLOT_OUT] ? out_bytes : 0, who))) return rc;
    const int64_t slab = std::min<int64_t>((int64_t)8 << 20, total);   // doubles per piece (64 MB at most)
    double *T = nullptr, *pin[2] = {nullptr, nullptr};
    if (cudaMallocAsync((void **)&T, tri_bytes(n) + 16, st) != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NOMEM, "%s: no room for the triangle of %lld observations", who, (long long)n);
    }
    int32_t *d_merge = nullptr;
    double *d_height = nullptr;
    auto body = [&]() -> int {
        d_height = (double *)scratch(SLOT_OUT, out_bytes);
        if (!d_height) return ICNV_E_NOMEM;
        d_merge = (int32_t *)(d_height + nm);
        for (int b = 0; b < 2; ++b) {
            if (cudaHostAlloc((void **)&pin[b], sizeof(double) * (size_t)slab, cudaHostAllocPortable) != cudaSuccess) {
                pin[b] = nullptr;
                cudaGetLastError();
                return set_error(ICNV_E_NOMEM, "%s: cudaHostAlloc of the staging slab failed", who);
            }
        }
        int b = 0;
        for (int64_t off = 0; off < total; off += slab, b ^= 1) {
            const size_t cnt = (size_t)std::min<int64_t>(slab, total - off);
            ICNV_CUDA(cudaEventSynchronize(c.ev_h2d[b]));   // the copy of two pieces ago has read this staging slab
            memcpy(pin[b], d + off, sizeof(double) * cnt);
            ICNV_CUDA(cudaMemcpyAsync(T + off, pin[b], sizeof(double) * cnt, cudaMemcpyHostToDevice, st));
            ICNV_CUDA(cudaEventRecord(c.ev_h2d[b], st));
        }
        return tri_prepare_and_link(T, T, n, method, d_merge, d_height, st, who);
    };
    rc = body();
    cudaFreeAsync(T, st);
    if (!rc) {
        if (cudaMemcpyAsync(height, d_height, sizeof(double) * (size_t)nm, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaMemcpyAsync(merge, d_merge, sizeof(int32_t) * 2 * (size_t)nm, cudaMemcpyDeviceToHost, st) != cudaSuccess)
            rc = set_error(ICNV_E_CUDA, "%s: copy of the result failed", who);
    }
    const cudaError_t e = cudaStreamSynchronize(st);
    for (double *p : pin)
        if (p) cudaFreeHost(p);
    if (rc) return rc;
    if (e != cudaSuccess) return set_error(ICNV_E_CUDA, "%s: %s", who, cudaGetErrorString(e));
    return icnv_hclust_order(merge, n, order);
}

/* hclust(parallelDist(t(X[keep, cells])), method) on device data: K10's tiles write the distances straight into the
 * triangle, which is then prepared and linked as a "dist" vector would be.  X: genes x C columns (stride ldx >= G);
 * d_keep (device; NULL: all G genes, non-NULL with n_keep = 0: none); d_cells (device, n columns; NULL: columns 0 .. n-1). */
int cluster_cells_dev(const double *X, int64_t G, int64_t ldx, int64_t C, const int32_t *d_keep, int64_t n_keep,
                      const int32_t *d_cells, int64_t n, int method, int32_t *merge, double *height, void *stream,
                      const char *who) {
    ICNV_REQUIRE_READY();
    int rc = hclust_tri_check(n, method, who);
    if (rc) return rc;
    if (!X || G < 0 || n_keep < 0 || ldx < G || C < 1 || (!d_cells && n > C) || !merge || !height ||
        (d_keep && n_keep > 0 && G < 1))
        return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    cudaStream_t st = pick_stream(stream);
    const int64_t Gk = d_keep ? n_keep : G;   // genes the distances run over
    const size_t y_bytes = d_keep && Gk > 0 ? sizeof(double) * (size_t)Gk * (size_t)C : 0;
    if ((rc = hclust_tri_room(n, y_bytes + 256, who))) return rc;
    char *fb = nullptr;   // [flag | gathered genes]
    if (cudaMallocAsync((void **)&fb, 256 + y_bytes, st) != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NOMEM, "%s: no room for the gathered genes", who);
    }
    int *d_flag = (int *)fb;
    double *Y = (double *)(fb + 256), *T = nullptr;
    auto body = [&]() -> int {
        ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
        int r = d_cells ? sc::check_indices(d_cells, n, C, d_flag, st) : ICNV_OK;
        if (!r && d_keep) r = sc::check_indices(d_keep, n_keep, G, d_flag, st);
        if (r) return r;
        int hf = 0;
        ICNV_CUDA(cudaMemcpyAsync(&hf, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        if (hf & 2) return set_error(ICNV_E_BAD_ARG, "%s: cell or gene index out of range", who);
        const double *Xd = X;
        int64_t ldd = ldx;
        if (d_keep && Gk > 0) {
            if ((r = icnv_dev_gather_rows_f64(X, ldx, d_keep, Gk, Y, C, st))) return r;
            Xd = Y;
            ldd = Gk;
        }
        if (cudaMallocAsync((void **)&T, tri_bytes(n) + 16, st) != cudaSuccess) {
            cudaGetLastError();
            T = nullptr;
            return set_error(ICNV_E_NOMEM, "%s: no room for the triangle of %lld cells", who, (long long)n);
        }
        if ((r = icnv_dev_pairwise_dist_f64(Xd, Gk, ldd, d_cells, n, T, st))) return r;
        return tri_prepare_and_link(T, T, n, method, merge, height, st, who);
    };
    rc = body();
    if (T) cudaFreeAsync(T, st);
    cudaFreeAsync(fb, st);
    if (rc) cudaStreamSynchronize(st);   // nothing enqueued by a failed call outlives it
    return rc;
}

}  // namespace icnv
