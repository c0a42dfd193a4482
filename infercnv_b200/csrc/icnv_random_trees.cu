// Running means and the permutation null of random-trees subclustering - K13 in DESIGN section 3.
//
// K13a, caTools::runmean(x, k) with its defaults (alg "C", endrule "mean", align "center") down each column, per row range:
// for a range of L genes, k' = min(k, L), k2 = k' / 2, k1 = k' - 1 - k2, and
//     out[p] = mean(x[max(0, p - k1) .. min(L - 1, p + k2)])
// - a centred box mean whose window is cut at the ends of the range.  k <= 1 and ranges of fewer than 2 genes are copies, as
// are the genes outside every range.  Arithmetic: one thread walks a column range in gene order with a double-double
// running sum (two-sum of each added / removed value, the error term renormalised by a second two-sum), and the mean is the
// double-double sum over the count with one remainder correction.  Each output is a function of its column's range alone,
// whatever the launch geometry, and
//     |out[p] - m[p]| <= 2 u |m[p]| + 8 L u^2 T / cnt[p]         (u = 2^-53, T = sum of |x| over the range)
// where m[p] is the exact mean (tests/runmean_reference.py states and enforces it).
//
// K13b, .parameterize_random_cluster_heights_smoothed_trees (R/inferCNV_tumor_subclusters.random_smoothed_trees.R:217-304):
// the observed tree and n_perm permuted trees of one clade, each runmean(window) over [0, G) -> median centring (the cell
// pipeline with centring only, icnv_center_f64's kernel) -> Euclidean distances (K10's tiles, written into a square matrix)
// -> NN-chain linkage (K11).  Permutation p shuffles every gene independently across the n cells: with
// key(p, g, i) = mix64(hash3(seed, p, g, i)) and pi_{p,g} the stable ascending argsort of the keys over the list positions i,
// X_p[g, i] = X[g, cells[pi_{p,g}(i)]].  (hash3's last argument enters through an XOR only: its raw values would order the
// positions of one (p, g) in a few ways only - 8 of the 24 orders of four; the final mix64 spreads them.)  The members (the observed tree first, then the permutations in order) go through
// the device in waves of B: a gather / sort kernel (one CTA per member and gene) writes the permuted matrices, then one
// launch each smooths, centres and measures all B of them, and one linkage launch runs the B chains, one per SM.
#include "icnv_common.cuh"

#include <algorithm>
#include <vector>

extern "C" int icnv_dev_cell_pipeline_f64(const double *X, int64_t G, int64_t ldx, const int32_t *cols, int64_t n_cols,
                                          double *Y, int64_t ldy, const int32_t *chr_start, const int32_t *chr_len, int K,
                                          int apply_log, const double *lo1, const double *hi1, const double *mid1,
                                          double threshold, int window, int center, const double *lo2, const double *hi2,
                                          const double *mid2, int apply_exp2, int *err_flag, void *stream);

namespace icnv {

// icnv_hclust.cu / icnv_dist.cu
int hclust_check_args(int64_t n, int method, const char *who);
int64_t hclust_ld(int64_t n);
int hclust_batch(double *M, int64_t n, int method, int B, int32_t *merge, double *height, cudaStream_t st);
size_t hclust_batch_scratch(int64_t n);
int dist_square_launch(const double *X, int64_t G, int64_t ldx, int64_t sx, int64_t n, int B, double *M, int64_t ld,
                       int64_t sm, int square, int *flag, cudaStream_t st);

namespace rt {

constexpr int RM_NT = 128;
constexpr int PG_NT = 256;

// One column range [s, s + L) of x -> y.
__device__ void runmean_range(const double *x, double *y, int64_t L, int k) {
    const int64_t kk = k < L ? k : L;
    const int64_t k2 = kk / 2, k1 = kk - 1 - k2;
    double hi = 0.0, lo = 0.0;
    for (int64_t g = 0; g <= k2; ++g) dd_add(hi, lo, x[g]);   // window of p = 0: [0, k2]
    for (int64_t p = 0; p < L; ++p) {
        const int64_t a = p - k1 > 0 ? p - k1 : 0, b = p + k2 < L - 1 ? p + k2 : L - 1;
        y[p] = dd_div(hi, lo, (double)(b - a + 1));
        if (p + 1 + k2 < L) dd_add(hi, lo, x[p + 1 + k2]);    // the window of p + 1 gains its right end
        if (p - k1 >= 0) dd_add(hi, lo, -x[p - k1]);          // and loses its left end
    }
}

// One thread per column: the K ranges (rs / rl; rs == nullptr: the single range [0, G)) in order, genes outside them copied.
// flag |= 1 on a non-finite value anywhere in the column.
__global__ void __launch_bounds__(RM_NT) runmean_kernel(const double *__restrict__ X, int64_t ldx, double *__restrict__ Y,
                                                        int64_t ldy, int64_t G, int64_t ncols, const int32_t *rs,
                                                        const int32_t *rl, int K, int k, int *flag) {
    const int64_t c = (int64_t)blockIdx.x * RM_NT + threadIdx.x;
    if (c >= ncols) return;
    const double *x = X + ldx * c;
    double *y = Y + ldy * c;
    bool bad = false;
    int64_t pos = 0;
    const int nr = rs ? K : 1;
    for (int r = 0; r <= nr; ++r) {
        const int64_t s = r < nr ? (rs ? rs[r] : 0) : G, L = r < nr ? (rs ? rl[r] : G) : 0;
        for (; pos < s; ++pos) {
            const double v = x[pos];
            bad |= !is_finite_d(v);
            y[pos] = v;
        }
        if (L <= 0) continue;
        if (k > 1 && L >= 2) {
            for (int64_t g = s; g < s + L; ++g) bad |= !is_finite_d(x[g]);
            runmean_range(x + s, y + s, L, k);
        } else {
            for (int64_t g = s; g < s + L; ++g) {
                const double v = x[g];
                bad |= !is_finite_d(v);
                y[g] = v;
            }
        }
        pos = s + L;
    }
    if (bad) atomicOr(flag, 1);
}

// (key, position) ascending; positions are distinct, so this is a total order and the sort is the stable argsort
__device__ __forceinline__ bool pg_less(unsigned long long ka, int ia, unsigned long long kb, int ib) {
    return ka < kb || (ka == kb && ia < ib);
}

// Members q0 + blockIdx.y (q = 0: the observed matrix, q >= 1: permutation p = q - 1), genes 0 .. G - 1 grid-stride over
// blockIdx.x: one (member, gene) segment at a time.  Permutations sort their n keys (bitonic over P = power of two >= n, padded with
// (~0, INT_MAX)) in `keys` / `idx`: shared memory, or global scratch of P entries per CTA when `gkeys` is given.
// W (G x nb n): member z's columns at W + G n z.
__global__ void __launch_bounds__(PG_NT) perm_gather_kernel(const double *__restrict__ X, int64_t ldx,
                                                            const int32_t *__restrict__ cells, int64_t n, int64_t G, int P,
                                                            unsigned long long seed, int64_t q0, double *W,
                                                            unsigned long long *gkeys, int32_t *gidx) {
    extern __shared__ __align__(16) unsigned char pg_smem[];
    const size_t cta = (size_t)blockIdx.y * gridDim.x + blockIdx.x;
    unsigned long long *keys = gkeys ? gkeys + cta * P : reinterpret_cast<unsigned long long *>(pg_smem);
    int32_t *idx = gkeys ? gidx + cta * P : reinterpret_cast<int32_t *>(pg_smem + sizeof(unsigned long long) * P);
    const int tid = threadIdx.x;
    const int64_t z = blockIdx.y, q = q0 + z;
    for (int64_t g = blockIdx.x; g < G; g += gridDim.x) {
        double *w = W + G * n * z + g;
        if (q == 0) {
            for (int i = tid; i < n; i += PG_NT) w[G * i] = X[g + ldx * (cells ? cells[i] : i)];
            continue;
        }
        const unsigned long long p = (unsigned long long)(q - 1);
        for (int i = tid; i < P; i += PG_NT) {
            keys[i] = i < n ? mix64(hash3(seed, p, (unsigned long long)g, (unsigned long long)i)) : ~0ull;
            idx[i] = i < n ? i : 0x7fffffff;
        }
        __syncthreads();
        for (int kb = 2; kb <= P; kb <<= 1)
            for (int jj = kb >> 1; jj > 0; jj >>= 1) {
                for (int e = tid; e < P / 2; e += PG_NT) {   // pair e: t has bit jj clear, l = t + jj
                    const int t = ((e & ~(jj - 1)) << 1) | (e & (jj - 1)), l = t + jj;
                    const unsigned long long ka = keys[t], kl = keys[l];
                    const int ia = idx[t], il = idx[l];
                    const bool up = (t & kb) == 0;
                    if (up ? pg_less(kl, il, ka, ia) : pg_less(ka, ia, kl, il)) {
                        keys[t] = kl; keys[l] = ka;
                        idx[t] = il; idx[l] = ia;
                    }
                }
                __syncthreads();
            }
        for (int i = tid; i < n; i += PG_NT) {
            const int j = idx[i];
            w[G * i] = X[g + ldx * (cells ? cells[j] : j)];
        }
        __syncthreads();   // keys / idx are rewritten by the next segment
    }
}

// perm_max[q - 1] = the largest height of member z = q - q0 (its sorted heights end with it), for q >= 1
__global__ void perm_max_kernel(const double *height, int64_t nm, int64_t q0, int nb, double *perm_max) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    if (z >= nb || q0 + z == 0) return;
    perm_max[q0 + z - 1] = height[(int64_t)z * nm + nm - 1];
}

}  // namespace rt

using namespace rt;

int runmean_launch(const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t G, int64_t ncols, const int32_t *d_rs,
                   const int32_t *d_rl, int K, int k, int *flag, cudaStream_t st) {
    if (ncols <= 0) return ICNV_OK;
    runmean_kernel<<<(unsigned)((ncols + RM_NT - 1) / RM_NT), RM_NT, 0, st>>>(X, ldx, Y, ldy, G, ncols, d_rs, d_rl, K, k, flag);
    ICNV_CHECK_LAUNCH("runmean_kernel");
    return ICNV_OK;
}

// What the last random-trees call of the process did: B, waves, and the device time of its stages (ms).
static double g_rt_stats[5];

int random_trees_dev(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n, int window, int method,
                     int n_perm, unsigned long long seed, int32_t *merge, double *height, double *perm_max, void *stream,
                     const char *who) {
    ICNV_REQUIRE_READY();
    if (n_perm < 0) return set_error(ICNV_E_BAD_ARG, "%s: n_perm = %d", who, n_perm);
    int rc = hclust_check_args(n, method, who);
    if (rc) return rc;
    if (!X || G < 1 || ldx < G || !merge || !height || (n_perm > 0 && !perm_max))
        return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    Ctx &c = ctx();
    cudaStream_t st = pick_stream(stream);
    const int64_t Q = (int64_t)n_perm + 1, ld = hclust_ld(n), nm = n - 1;
    int P = 1;
    while (P < n) P <<= 1;
    const size_t sort_smem = (sizeof(unsigned long long) + sizeof(int32_t)) * (size_t)P;
    const bool sort_global = sort_smem > (size_t)c.smem_optin;
    const int64_t sort_grid = (int64_t)c.sm_count * 8;   // CTAs of a global-memory sort launch (at most; gx nb <= it)
    // per member: two G x n working copies, the n x ld matrix, the linkage scratch, merge and height
    const size_t per = sizeof(double) * (2 * (size_t)G * (size_t)n + (size_t)n * (size_t)ld + (size_t)nm) +
                       sizeof(int32_t) * 2 * (size_t)nm + hclust_batch_scratch(n) + 1024;
    const size_t fixed = (sort_global ? sort_smem * (size_t)sort_grid : 0) + 4096;
    size_t free_b = 0, total_b = 0;
    ICNV_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const size_t usable = free_b > (size_t)(256 << 20) ? free_b - (size_t)(256 << 20) : 0;   // headroom for the runtime
    const int64_t fit = usable > fixed ? (int64_t)((usable - fixed) / per) : 0;
    const int B = (int)std::min<int64_t>(std::min<int64_t>(Q, c.sm_count), fit);
    if (B < 1) return set_error(ICNV_E_NOMEM, "%s: one member of %lld cells x %lld genes does not fit", who, (long long)n, (long long)G);
    const size_t wn = (size_t)G * (size_t)n * (size_t)B, mn = (size_t)n * (size_t)ld * (size_t)B;
    char *buf = nullptr;
    const size_t bytes = sizeof(double) * (2 * wn + mn + (size_t)nm * B) + sizeof(int32_t) * 2 * (size_t)nm * B + fixed + 256;
    if (cudaMallocAsync((void **)&buf, bytes, st) != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NOMEM, "%s: no room for %d members", who, B);
    }
    double *W1 = (double *)buf, *W2 = W1 + wn, *M = W2 + wn, *hgt = M + mn;
    int32_t *mrg = (int32_t *)(hgt + (size_t)nm * B);
    int *d_flag = (int *)(mrg + 2 * (size_t)nm * B);
    char *tail = (char *)d_flag + 256;
    unsigned long long *gkeys = sort_global ? (unsigned long long *)tail : nullptr;
    int32_t *gidx = sort_global ? (int32_t *)(tail + sizeof(unsigned long long) * (size_t)P * (size_t)sort_grid) : nullptr;
    const int32_t one_start = 0, one_len = (int32_t)G;
    const int64_t waves = (Q + B - 1) / B;
    std::vector<cudaEvent_t> ev((size_t)(4 * waves), nullptr);
    for (auto &e : ev) ICNV_CUDA(cudaEventCreate(&e));
    auto body = [&]() -> int {
        ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
        if (!sort_global) ICNV_CUDA(cudaFuncSetAttribute(perm_gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sort_smem));
        for (int64_t w = 0; w < waves; ++w) {
            const int64_t q0 = w * B;
            const int nb = (int)std::min<int64_t>(B, Q - q0);
            ICNV_CUDA(cudaEventRecord(ev[4 * w], st));
            const unsigned gx = (unsigned)std::min<int64_t>(G, sort_global ? std::max<int64_t>(sort_grid / nb, 1) : 65535);
            perm_gather_kernel<<<dim3(gx, (unsigned)nb), PG_NT, sort_global ? 0 : sort_smem, st>>>(X, ldx, d_cells, n, G, P,
                                                                                                seed, q0, W1, gkeys, gidx);
            ICNV_CHECK_LAUNCH("perm_gather_kernel");
            int r = runmean_launch(W1, G, W2, G, G, (int64_t)nb * n, nullptr, nullptr, 1, window, d_flag, st);
            if (r) return r;
            r = icnv_dev_cell_pipeline_f64(W2, G, G, nullptr, (int64_t)nb * n, W1, G, &one_start, &one_len, 1, 0, nullptr,
                                           nullptr, nullptr, 0.0, 0, 1, nullptr, nullptr, nullptr, 0, d_flag, st);
            if (r) return r;
            ICNV_CUDA(cudaEventRecord(ev[4 * w + 1], st));
            r = dist_square_launch(W1, G, G, G * n, n, nb, M, ld, n * ld, method == 7, d_flag, st);
            if (r) return r;
            ICNV_CUDA(cudaEventRecord(ev[4 * w + 2], st));
            if (w == 0) {   // the values of every member are those of the observed one, reordered: one check covers all
                int h = 0;
                ICNV_CUDA(cudaMemcpyAsync(&h, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
                ICNV_CUDA(cudaStreamSynchronize(st));
                if (h) return set_error(ICNV_E_NONFINITE, "%s: NaN or Inf in the input (or in its distances)", who);
            }
            if ((r = hclust_batch(M, n, method, nb, mrg, hgt, st))) return r;
            if (w == 0) {
                ICNV_CUDA(cudaMemcpyAsync(merge, mrg, sizeof(int32_t) * 2 * (size_t)nm, cudaMemcpyDeviceToDevice, st));
                ICNV_CUDA(cudaMemcpyAsync(height, hgt, sizeof(double) * (size_t)nm, cudaMemcpyDeviceToDevice, st));
            }
            if (n_perm > 0) {
                perm_max_kernel<<<(nb + 127) / 128, 128, 0, st>>>(hgt, nm, q0, nb, perm_max);
                ICNV_CHECK_LAUNCH("perm_max_kernel");
            }
            ICNV_CUDA(cudaEventRecord(ev[4 * w + 3], st));
        }
        ICNV_CUDA(cudaStreamSynchronize(st));
        double t[3] = {0.0, 0.0, 0.0};
        for (int64_t w = 0; w < waves; ++w)
            for (int s = 0; s < 3; ++s) {
                float ms = 0.0f;
                ICNV_CUDA(cudaEventElapsedTime(&ms, ev[4 * w + s], ev[4 * w + s + 1]));
                t[s] += ms;
            }
        g_rt_stats[0] = B;
        g_rt_stats[1] = (double)waves;
        for (int s = 0; s < 3; ++s) g_rt_stats[2 + s] = t[s];
        return ICNV_OK;
    };
    rc = body();
    cudaFreeAsync(buf, st);
    for (auto &e : ev)
        if (e) cudaEventDestroy(e);
    return rc;
}

void random_trees_stats(double *out5) {
    for (int i = 0; i < 5; ++i) out5[i] = g_rt_stats[i];
}

}  // namespace icnv
