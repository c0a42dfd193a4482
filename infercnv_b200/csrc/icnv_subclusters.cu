// Subclustering trees of run() step 15, define_signif_tumor_subclusters (R/inferCNV_tumor_subclusters.R:2-177) - K17 in
// DESIGN section 3.
//
// K17a, the z-score gene filter (:45-68): with ref the columns of unlist(reference_grouped_cell_indices) in that order,
//     z = (ref - mean(ref)) / sd(ref),   outliers = which(apply(abs(z), 1, mean) >= 0.8).
// mu and sigma are icnv_mean_sd_f64's bits (per-cell statistics on the device, combined on the host by
// icnv_combine_cell_stats).  One thread per (gene, eighth of the cell list) forms |__ddiv_rn(x - mu, sigma)| - one rounding
// per operation, as R evaluates the matrix expression element by element - and adds it to a double-double sum (two_sum);
// the eight partial sums of a gene are added in a fixed order, and dd_div divides by n.  R's mean() is s = sum / n in long
// double followed by s += sum(x - s) / n; dd_div is that refinement with both sums exact to ~2^-100, so the mean is the
// correctly rounded mean of the z values (R's long double can differ only where the exact mean lies within ~n 2^-64 of a
// rounding midpoint).  Non-finite z values follow R: a NaN (0 / 0, a constant reference) makes the mean NaN, which fails
// >= 0.8; +Inf (x != mu with sigma = 0) makes it +Inf.  The threshold is the literal 0.8 of the reference.
//
// K17b, the trees (:191, :582, :609): hclust(parallelDist(t(expr.data[keep, cells_g])), method) for every group g with
// n_g >= 2, in one call.  The kept genes are gathered once (icnv_dev_gather_rows_f64); the members (groups) are ordered
// largest first and cut into waves of at most one member per SM that fit the free device memory.  Per wave, one
// dist_square_kernel launch walks a tile-work table (member, tile row, tile column) over all its members - K10's tiles, so
// every distance has the bits of icnv_pairwise_dist_f64 - and one hclust_nn_chain_kernel launch runs its linkages, one
// CTA each, every member reading its n, ld and offsets from the member table.  A member's tree is a function of its own
// cells only: whatever the wave split, member order or SM count, it equals icnv_pairwise_dist_f64 -> icnv_hclust_f64 on
// that group, bit for bit.
#include "icnv_common.cuh"

#include <algorithm>
#include <numeric>
#include <vector>

namespace icnv {

// icnv_hclust.cu / icnv_dist.cu
int64_t hclust_ld(int64_t n);
size_t hclust_batch_scratch(int64_t n);
int hclust_member_batch(const HcMember *d_mem, int B, int64_t n_max, int method, double *M, double *w8, int32_t *w4,
                        int32_t *merge, double *height, cudaStream_t st);
int dist_square_members_launch(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, const int4 *d_tiles,
                               int64_t n_tiles, const HcMember *d_mem, double *M, int square, int *flag, cudaStream_t st);

namespace sc {

constexpr int ZS_GENES = 32;   // genes per CTA: a warp reads 256 contiguous bytes of one cell's column
constexpr int ZS_WARPS = 8;    // warp w takes the list positions w, w + 8, ...
constexpr int64_t SC_NMAX = 65536;
constexpr int SC_PD_T = 128;   // dist_square_kernel's tile side (PD_T of icnv_dist.cu)

// outlier[g] = (mean over the list of |(X[g, cells[i]] - mu) / sigma|) >= 0.8.  flag |= 1 on a non-finite input value.
__global__ void __launch_bounds__(ZS_GENES *ZS_WARPS) zscore_outlier_kernel(const double *__restrict__ X, int64_t G,
                                                                            const int32_t *__restrict__ cells, int64_t n,
                                                                            double mu, double sigma, uint8_t *outlier,
                                                                            int *flag) {
    __shared__ double s_hi[ZS_WARPS][ZS_GENES], s_lo[ZS_WARPS][ZS_GENES];
    __shared__ int s_sp[ZS_WARPS][ZS_GENES];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t g = (int64_t)blockIdx.x * ZS_GENES + lane;
    double hi = 0.0, lo = 0.0;
    int sp = 0;   // 1: a +Inf z, 2: a NaN z
    bool bad = false;
    if (g < G)
        for (int64_t i = w; i < n; i += ZS_WARPS) {
            const double x = X[g + G * (int64_t)cells[i]];
            bad |= !is_finite_d(x);
            const double z = fabs(__ddiv_rn(__dadd_rn(x, -mu), sigma));
            if (is_finite_d(z))
                dd_add(hi, lo, z);
            else
                sp |= z == z ? 1 : 2;
        }
    s_hi[w][lane] = hi;
    s_lo[w][lane] = lo;
    s_sp[w][lane] = sp;
    __syncthreads();
    if (w == 0 && g < G) {
        hi = s_hi[0][lane];
        lo = s_lo[0][lane];
        for (int k = 1; k < ZS_WARPS; ++k) {
            dd_add(hi, lo, s_hi[k][lane]);
            dd_add(hi, lo, s_lo[k][lane]);
            sp |= s_sp[k][lane];
        }
        const double m = dd_div(hi, lo, (double)n);
        outlier[g] = (sp & 2) ? 0 : ((sp & 1) ? 1 : (m >= 0.8 ? 1 : 0));
    }
    if (bad) atomicOr(flag, 1);
}

// flag |= 2 when an entry of idx is outside [0, lim)
__global__ void __launch_bounds__(256) index_check_kernel(const int32_t *__restrict__ idx, int64_t n, int64_t lim, int *flag) {
    bool bad = false;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
        const int32_t v = idx[i];
        bad |= v < 0 || v >= lim;
    }
    if (bad) atomicOr(flag, 2);
}

int check_indices(const int32_t *d_idx, int64_t n, int64_t lim, int *flag, cudaStream_t st) {
    if (n <= 0) return ICNV_OK;
    const unsigned grid = (unsigned)std::min<int64_t>((n + 255) / 256, 1024);
    index_check_kernel<<<grid, 256, 0, st>>>(d_idx, n, lim, flag);
    ICNV_CHECK_LAUNCH("index_check_kernel");
    return ICNV_OK;
}

}  // namespace sc

using namespace sc;

// ---- K17a ------------------------------------------------------------------------------------------------------------

// X: G x (listed columns), ld G, on the device; d_cells: n device indices.  Synchronises `stream` twice (the statistics
// come to the host to be combined; the non-finite check).
int zscore_outlier_dev(const double *X, int64_t G, const int32_t *d_cells, int64_t n, uint8_t *outlier, void *stream,
                       const char *who) {
    ICNV_REQUIRE_READY();
    if (!X || !d_cells || !outlier || G <= 1 || n <= 0) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    cudaStream_t st = pick_stream(stream);
    char *w = nullptr;
    if (cudaMallocAsync((void **)&w, sizeof(double) * 2 * (size_t)n + 16, st) != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NOMEM, "%s: no room for the per-cell statistics", who);
    }
    double *d_stats = (double *)w;
    int *d_flag = (int *)(d_stats + 2 * n);
    auto body = [&]() -> int {
        ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
        int rc = icnv_dev_column_stats_f64(X, G, d_cells, n, d_stats, d_stats + n, st);
        if (rc) return rc;
        std::vector<double> h(2 * (size_t)n);
        ICNV_CUDA(cudaMemcpyAsync(h.data(), d_stats, sizeof(double) * 2 * (size_t)n, cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        double mu = 0.0, sigma = 0.0;
        icnv_combine_cell_stats(h.data(), h.data() + n, n, G, &mu, &sigma);
        zscore_outlier_kernel<<<(unsigned)((G + ZS_GENES - 1) / ZS_GENES), ZS_GENES * ZS_WARPS, 0, st>>>(X, G, d_cells, n, mu,
                                                                                                        sigma, outlier, d_flag);
        ICNV_CHECK_LAUNCH("zscore_outlier_kernel");
        int hf = 0;
        ICNV_CUDA(cudaMemcpyAsync(&hf, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        if (hf) return set_error(ICNV_E_NONFINITE, "%s: NaN or Inf in the reference columns", who);
        return ICNV_OK;
    };
    const int rc = body();
    cudaFreeAsync(w, st);
    return rc;
}

// ---- K17b ------------------------------------------------------------------------------------------------------------

// What the last group-trees call did: waves, members of the largest wave, device ms of the gene gather, the distances and
// the linkages (summed over the waves).
static double g_cg_stats[5];

// Checks on the host-visible arguments, before anything is allocated.
int cluster_groups_check(int64_t G, const int32_t *keep, int64_t n_keep, const int32_t *grp_off, int n_grp, int method,
                         const char *who) {
    if (G < 0 || n_keep < 0 || n_grp < 0 || (n_grp > 0 && !grp_off) || (keep && n_keep > 0 && G < 1))
        return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    if (method == 5 || method == 6)
        return set_error(ICNV_E_UNSUPPORTED, "%s: method %d (centroid / median) is not reducible", who, method);
    if (method < 0 || method > 7) return set_error(ICNV_E_BAD_ARG, "%s: unknown method code %d", who, method);
    for (int k = 0; k < n_grp; ++k) {
        const int64_t n = (int64_t)grp_off[k + 1] - grp_off[k];
        if (grp_off[k] < 0 || n < 0) return set_error(ICNV_E_BAD_ARG, "%s: group offsets are not ascending", who);
        if (n > SC_NMAX)
            return set_error(ICNV_E_UNSUPPORTED, "%s: group %d has %lld cells (limit %lld)", who, k, (long long)n,
                             (long long)SC_NMAX);
    }
    return ICNV_OK;
}

// merge / height rows of the trees before group k: sum over the earlier groups of max(n - 1, 0)
int64_t cluster_groups_rows(const int32_t *grp_off, int n_grp) {
    int64_t r = 0;
    for (int k = 0; k < n_grp; ++k) r += std::max<int64_t>((int64_t)grp_off[k + 1] - grp_off[k] - 1, 0);
    return r;
}

// X (genes x cells, column stride ldx >= G, C columns), d_keep / n_keep (device; NULL: all genes), grp_off (host, n_grp + 1),
// d_idx (device, grp_off[n_grp] columns), merge / height (device, packed per group).
int cluster_groups_dev(const double *X, int64_t G, int64_t ldx, int64_t C, const int32_t *d_keep, int64_t n_keep,
                       const int32_t *grp_off, const int32_t *d_idx, int n_grp, int method, int32_t *merge, double *height,
                       void *stream, const char *who) {
    ICNV_REQUIRE_READY();
    int rc = cluster_groups_check(G, d_keep, n_keep, grp_off, n_grp, method, who);
    if (rc) return rc;
    const int64_t rows = cluster_groups_rows(grp_off, n_grp);
    for (double &v : g_cg_stats) v = 0.0;
    if (rows == 0) return ICNV_OK;   // no group of two or more cells: nothing to write
    if (!X || ldx < G || C < 1 || !d_idx || !merge || !height) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    Ctx &c = ctx();
    cudaStream_t st = pick_stream(stream);
    const int64_t Gk = d_keep ? n_keep : G;   // genes the distances run over
    const int64_t n_list = grp_off[n_grp];

    // members, largest first (ties: group order); their output offsets follow the group order
    std::vector<int> mem_grp;
    std::vector<int64_t> out_off((size_t)n_grp, 0);
    int64_t row = 0;
    for (int k = 0; k < n_grp; ++k) {
        const int64_t n = (int64_t)grp_off[k + 1] - grp_off[k];
        out_off[(size_t)k] = row;
        if (n >= 2) {
            mem_grp.push_back(k);
            row += n - 1;
        }
    }
    auto size_of = [&](int k) { return (int64_t)grp_off[k + 1] - grp_off[k]; };
    std::stable_sort(mem_grp.begin(), mem_grp.end(), [&](int a, int b) { return size_of(a) > size_of(b); });

    // one allocation for the flag, the gathered genes and the tables; the wave buffer after it
    int64_t n_tiles = 0;
    for (int k : mem_grp) {
        const int64_t T = (size_of(k) + SC_PD_T - 1) / SC_PD_T;
        n_tiles += T * (T + 1) / 2;
    }
    const size_t nm = mem_grp.size();
    const size_t y_bytes = d_keep && Gk > 0 ? sizeof(double) * (size_t)Gk * (size_t)C : 0;
    const size_t fixed = 256 + ((y_bytes + 255) & ~(size_t)255) + sizeof(HcMember) * nm + sizeof(int4) * (size_t)n_tiles;
    char *fb = nullptr;
    if (cudaMallocAsync((void **)&fb, fixed, st) != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NOMEM, "%s: no room for the gathered genes and the tables", who);
    }
    int *d_flag = (int *)fb;
    double *Y = (double *)(fb + 256);
    HcMember *d_mem = (HcMember *)(fb + 256 + ((y_bytes + 255) & ~(size_t)255));
    int4 *d_tiles = (int4 *)(d_mem + nm);
    char *wb = nullptr;
    std::vector<cudaEvent_t> ev;

    auto body = [&]() -> int {
        ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
        int r = check_indices(d_idx, n_list, C, d_flag, st);
        if (!r && d_keep) r = check_indices(d_keep, n_keep, G, d_flag, st);
        if (r) return r;
        int hf = 0;
        ICNV_CUDA(cudaMemcpyAsync(&hf, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        if (hf & 2) return set_error(ICNV_E_BAD_ARG, "%s: cell or gene index out of range", who);

        // waves: the next members in size order while one more fits the free memory and an SM is left for it
        size_t free_b = 0, total_b = 0;
        ICNV_CUDA(cudaMemGetInfo(&free_b, &total_b));
        const size_t usable = free_b > (size_t)(256 << 20) ? free_b - (size_t)(256 << 20) : 0;   // headroom for the runtime
        auto per = [&](int64_t n) { return sizeof(double) * (size_t)n * (size_t)hclust_ld(n) + hclust_batch_scratch(n) + 64; };
        std::vector<size_t> wave_at;   // first member of each wave (positions in mem_grp), then nm
        for (size_t i = 0; i < nm;) {
            wave_at.push_back(i);
            size_t used = 0, j = i;
            while (j < nm && (int64_t)(j - i) < c.sm_count && used + per(size_of(mem_grp[j])) <= usable) used += per(size_of(mem_grp[j++]));
            if (j == i)
                return set_error(ICNV_E_NOMEM, "%s: one linkage of %lld cells does not fit the free device memory", who,
                                 (long long)size_of(mem_grp[i]));
            i = j;
        }
        wave_at.push_back(nm);
        const size_t waves = wave_at.size() - 1;

        // member and tile tables, offsets within the wave buffer: [matrices | 8-byte scratch | int32 scratch]
        std::vector<HcMember> hm(nm);
        std::vector<int4> ht;
        ht.reserve((size_t)n_tiles);
        std::vector<int64_t> tile_at;
        int64_t mM = 0, m8 = 0, m4 = 0;
        for (size_t w = 0; w < waves; ++w) {
            int64_t oM = 0, o8 = 0, o4 = 0;
            tile_at.push_back((int64_t)ht.size());
            for (size_t i = wave_at[w]; i < wave_at[w + 1]; ++i) {
                const int k = mem_grp[i];
                const int64_t n = size_of(k), ld = hclust_ld(n);
                int64_t P = 1;
                while (P < n - 1) P <<= 1;
                hm[i] = HcMember{grp_off[k], n, ld, oM, o8, o4, out_off[(size_t)k], (int32_t)P, 0};
                oM += n * ld;
                o8 += n + P;
                o4 += 6 * n + P;
                const int T = (int)((n + SC_PD_T - 1) / SC_PD_T);
                for (int bi = 0; bi < T; ++bi)
                    for (int bj = bi; bj < T; ++bj) ht.push_back(make_int4((int)(i - wave_at[w]), bi, bj, 0));
            }
            mM = std::max(mM, oM);
            m8 = std::max(m8, o8);
            m4 = std::max(m4, o4);
        }
        tile_at.push_back((int64_t)ht.size());
        ICNV_CUDA(cudaMemcpyAsync(d_mem, hm.data(), sizeof(HcMember) * nm, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_tiles, ht.data(), sizeof(int4) * ht.size(), cudaMemcpyHostToDevice, st));
        const size_t bM = sizeof(double) * (size_t)mM, b8 = sizeof(double) * (size_t)m8;
        if (cudaMallocAsync((void **)&wb, bM + b8 + sizeof(int32_t) * (size_t)m4 + 64, st) != cudaSuccess) {
            cudaGetLastError();
            wb = nullptr;
            return set_error(ICNV_E_NOMEM, "%s: no room for the linkage matrices", who);
        }
        double *M = (double *)wb, *w8 = (double *)(wb + bM);
        int32_t *w4 = (int32_t *)(wb + bM + b8);

        ev.assign(3 * waves + 2, nullptr);
        for (auto &e : ev) ICNV_CUDA(cudaEventCreate(&e));
        ICNV_CUDA(cudaEventRecord(ev[0], st));
        const double *Xd = X;
        int64_t ldd = ldx;
        if (d_keep && Gk > 0) {
            if ((r = icnv_dev_gather_rows_f64(X, ldx, d_keep, Gk, Y, C, st))) return r;
            Xd = Y;
            ldd = Gk;
        }
        ICNV_CUDA(cudaEventRecord(ev[1], st));
        for (size_t w = 0; w < waves; ++w) {
            const HcMember *wm = d_mem + wave_at[w];
            const int nb = (int)(wave_at[w + 1] - wave_at[w]);
            const int64_t n_max = hm[wave_at[w]].n;   // the wave's first member is its largest
            r = dist_square_members_launch(Xd, Gk, ldd, d_idx, d_tiles + tile_at[w], tile_at[w + 1] - tile_at[w], wm, M,
                                           method == 7, d_flag, st);
            if (r) return r;
            ICNV_CUDA(cudaEventRecord(ev[2 + 3 * w], st));
            ICNV_CUDA(cudaMemcpyAsync(&hf, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
            ICNV_CUDA(cudaStreamSynchronize(st));
            if (hf) return set_error(ICNV_E_NONFINITE, "%s: NaN or Inf in the input (or in its distances)", who);
            ICNV_CUDA(cudaEventRecord(ev[3 + 3 * w], st));
            if ((r = hclust_member_batch(wm, nb, n_max, method, M, w8, w4, merge, height, st))) return r;
            ICNV_CUDA(cudaEventRecord(ev[4 + 3 * w], st));
        }
        ICNV_CUDA(cudaStreamSynchronize(st));
        float ms = 0.0f;
        double t[3] = {0.0, 0.0, 0.0};
        ICNV_CUDA(cudaEventElapsedTime(&ms, ev[0], ev[1]));
        t[0] = ms;
        for (size_t w = 0; w < waves; ++w) {
            ICNV_CUDA(cudaEventElapsedTime(&ms, w ? ev[1 + 3 * w] : ev[1], ev[2 + 3 * w]));
            t[1] += ms;
            ICNV_CUDA(cudaEventElapsedTime(&ms, ev[3 + 3 * w], ev[4 + 3 * w]));
            t[2] += ms;
        }
        size_t widest = 0;
        for (size_t w = 0; w < waves; ++w) widest = std::max(widest, wave_at[w + 1] - wave_at[w]);
        g_cg_stats[0] = (double)waves;
        g_cg_stats[1] = (double)widest;
        for (int s = 0; s < 3; ++s) g_cg_stats[2 + s] = t[s];
        return ICNV_OK;
    };
    rc = body();
    if (wb) cudaFreeAsync(wb, st);
    cudaFreeAsync(fb, st);
    if (rc) cudaStreamSynchronize(st);   // nothing enqueued by a failed call outlives it
    for (auto &e : ev)
        if (e) cudaEventDestroy(e);
    return rc;
}

void cluster_groups_stats(double *out5) {
    for (int i = 0; i < 5; ++i) out5[i] = g_cg_stats[i];
}

}  // namespace icnv
