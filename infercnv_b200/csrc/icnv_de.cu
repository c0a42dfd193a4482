// Masking of non-DE genes - K14 in DESIGN section 3: mask_non_DE_genes_basic (R/inferCNV_mask_non_DE.R:28-52) in one call.
//
// Pairs (get_DE_genes_basic, :209-255): tested subcluster s (the caller's lists, in R's loop order) x reference group j,
// column s * n_ref + j; x = the reference cells, y = the subcluster.  Per (pair, gene):
//   wilcoxon (:191-203)  both sides jittered, then wilcox.test(x, y) with R's defaults: W = sum of the average ranks of x in
//                        x u y - n_x (n_x + 1) / 2; exact when n_x < 50, n_y < 50 and no ties in x u y (p = min(1, 2 P(W' <=
//                        min(W, n_x n_y - W))) from a host table of the rank-sum null), else the normal approximation with the
//                        continuity and tie corrections, p = 2 pnorm(-|z|).
//   t (:166-176)         Welch's t.test(x, y), no jitter; NaN where R's try() would catch an error (n < 2, or "essentially
//                        constant": stderr < 10 eps max(|m_x|, |m_y|)); p = 2 pt(-|t|, df) = I_{df / (df + t^2)}(df / 2, 1 / 2).
// BH per pair over the genes in R's operation order (:237; p.adjust's pmin(1, cummin(n / i * p[o]))[ro], n = the non-NA
// count); DE = p_adj < p_thresh (NaN: not DE).  Mask (.mask_DE_genes, :77-134): per cell and gene a count - reference cells
// and cells of tested subclusters of < 5 list entries start at n_ref, every cell of a tested subcluster of >= 5 entries adds
// 1 per reference group where the gene is DE for that subcluster (once per subcluster however often the cell is listed),
// other cells start at 0; "any" masks count == 0, "most" count < n_ref / 2, "all" count != n_ref.
//
// Generator: jitter = mean + sd z (__dadd_rn / __dmul_rn, no contraction), added to the value; z is Box-Muller on two (0, 1]
// uniforms u_k = ((mix64(hash3(seed, a, g, 2 i + k)) >> 11) + 1) 2^-53 (k = 0, 1), z = sqrt(-2 log u_0) cospi(2 u_1), with
// a = j for reference group j's draws (shared by every subcluster) and a = 2^32 + pair for the subcluster's draws, g the
// absolute gene and i the list position within the group.  Keys are absolute, so nothing depends on the gene tiling or the
// launch shape.
//
// Shape, per tile of genes sized from free memory: (a) a transpose-gather of the listed cells into gene-major rows, (b) per
// (reference group, gene) the jittered row sorted once, with its own tie count (Wilcoxon), or per (group, gene) mean and
// variance (t), (c) per (pair, gene) the jittered subcluster row sorted and each run of equal values located in the sorted
// reference row by binary search - W and sum(t^3 - t) in exact integers - then p; after all tiles (d) BH per pair and (e)
// one streaming pass per cell column.  Sorts are bitonic in shared memory up to SORT_SMEM bytes and in global scratch
// beyond, as in icnv_random_trees.cu.
#include "icnv_common.cuh"

#include <algorithm>
#include <cmath>
#include <vector>

namespace icnv {
namespace de {

constexpr int NT = 256;
constexpr int EXACT_N = 50;                   // wilcox.test's exact rule: n_x < 50 and n_y < 50
constexpr size_t SORT_SMEM = 64 * 1024;       // larger sorts run in global scratch

__device__ __forceinline__ double pos_inf() { return __longlong_as_double(0x7ff0000000000000ll); }

// jitter of list position i of the group keyed a, gene g
__device__ __forceinline__ double jitter(unsigned long long seed, unsigned long long a, unsigned long long g,
                                         unsigned long long i, double jm, double js) {
    const unsigned long long h0 = mix64(hash3(seed, a, g, 2 * i)), h1 = mix64(hash3(seed, a, g, 2 * i + 1));
    const double u0 = (double)((h0 >> 11) + 1) * 0x1p-53, u1 = (double)((h1 >> 11) + 1) * 0x1p-53;
    const double z = __dmul_rn(sqrt(-2.0 * log(u0)), cospi(2.0 * u1));
    return __dadd_rn(jm, __dmul_rn(js, z));
}

// ascending bitonic sort of key[0, P) (P a power of two) with an optional int32 payload (then ordered by (key, idx));
// starts and ends with a barrier
__device__ void block_sort(double *key, int32_t *idx, int P) {
    __syncthreads();
    for (int kb = 2; kb <= P; kb <<= 1)
        for (int jj = kb >> 1; jj > 0; jj >>= 1) {
            for (int e = threadIdx.x; e < P / 2; e += NT) {   // pair e: t has bit jj clear, l = t + jj
                const int t = ((e & ~(jj - 1)) << 1) | (e & (jj - 1)), l = t + jj;
                const double a = key[t], b = key[l];
                const bool up = (t & kb) == 0;
                bool sw;
                if (idx) {
                    const int ia = idx[t], ib = idx[l];
                    const bool b_lt_a = b < a || (b == a && ib < ia), a_lt_b = a < b || (a == b && ia < ib);
                    sw = up ? b_lt_a : a_lt_b;
                    if (sw) { idx[t] = ib; idx[l] = ia; }
                } else {
                    sw = up ? b < a : a < b;
                }
                if (sw) { key[t] = b; key[l] = a; }
            }
            __syncthreads();
        }
}

__device__ __forceinline__ long long warp_sum_ll(long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// block sum of an exact integer; every thread gets it
__device__ long long block_sum_ll(long long v, long long *sh) {
    v = warp_sum_ll(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    long long s = 0;
    for (int w = 0; w < NT / 32; ++w) s += sh[w];
    return s;
}

__device__ __forceinline__ long long tie_term(long long t) { return t * t * t - t; }
__device__ __forceinline__ int pow2_at_least(int n) {
    int p = 1;
    while (p < n) p <<= 1;
    return p;
}
// first position in x[0, n) with x >= v (lower) or x > v (upper)
__device__ __forceinline__ int bound(const double *x, int n, double v, bool upper) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int m = (lo + hi) >> 1;
        if (upper ? x[m] <= v : x[m] < v) lo = m + 1; else hi = m;
    }
    return lo;
}

// (a) Z[gl T + t] = X[g0 + gl + ldx cols[t]]: 32 x 32 tiles through shared memory, coalesced both ways.  flag |= 1 on a
// non-finite listed value.
__global__ void __launch_bounds__(NT) gather_kernel(const double *__restrict__ X, int64_t ldx, const int32_t *__restrict__ cols,
                                                    int64_t T, int64_t g0, int64_t gt, double *__restrict__ Z, int *flag) {
    __shared__ double tile[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int64_t t0 = (int64_t)blockIdx.x * 32, gb = (int64_t)blockIdx.y * 32;
    bool bad = false;
    for (int r = ty; r < 32; r += NT / 32) {       // r: list position within the tile, tx: gene
        const int64_t t = t0 + r, gl = gb + tx;
        if (t < T && gl < gt) {
            const double v = X[g0 + gl + ldx * (int64_t)cols[t]];
            bad |= !is_finite_d(v);
            tile[r][tx] = v;
        }
    }
    __syncthreads();
    for (int r = ty; r < 32; r += NT / 32) {       // r: gene within the tile, tx: list position
        const int64_t t = t0 + tx, gl = gb + r;
        if (t < T && gl < gt) Z[gl * T + t] = tile[tx][r];
    }
    if (bad) atomicOr(flag, 1);
}

// (b) Wilcoxon: per item (gene gl, reference group j) the jittered row sorted into RS (same layout as Z's reference part)
// and its own tie count sum(t^3 - t) into TS[gl n_ref + j].  `gbuf` (P doubles per CTA) when the sort is in global memory.
__global__ void __launch_bounds__(NT) ref_sort_kernel(const double *__restrict__ Z, int64_t T, int64_t gt, int64_t g0,
                                                      const int32_t *__restrict__ ref_off, int n_ref, int64_t R_tot,
                                                      unsigned long long seed, double jm, double js, double *RS,
                                                      long long *TS, double *gbuf, int P) {
    extern __shared__ __align__(16) unsigned char de_smem[];
    __shared__ long long red[NT / 32];
    double *buf = gbuf ? gbuf + (size_t)blockIdx.x * P : reinterpret_cast<double *>(de_smem);
    const int64_t items = gt * n_ref;
    for (int64_t it = blockIdx.x; it < items; it += gridDim.x) {
        const int64_t gl = it / n_ref;
        const int j = (int)(it % n_ref);
        const int a = ref_off[j], n = ref_off[j + 1] - a, Pn = pow2_at_least(n);
        const double *z = Z + gl * T + a;
        for (int i = threadIdx.x; i < Pn; i += NT)
            buf[i] = i < n ? __dadd_rn(z[i], jitter(seed, (unsigned long long)j, (unsigned long long)(g0 + gl), i, jm, js)) : pos_inf();
        block_sort(buf, nullptr, Pn);
        double *out = RS + gl * R_tot + a;
        long long ties = 0;
        for (int i = threadIdx.x; i < n; i += NT) {
            const double v = buf[i];
            out[i] = v;
            if (i == 0 || buf[i - 1] != v) {
                int e = i + 1;
                while (e < n && buf[e] == v) ++e;
                ties += tie_term(e - i);
            }
        }
        ties = block_sum_ll(ties, red);
        if (threadIdx.x == 0) TS[gl * n_ref + j] = ties;
        __syncthreads();   // buf is rewritten by the next item
    }
}

// wilcox.test(x, y) p from U_x (twice it, an exact integer) and sum(t^3 - t) over x u y
__device__ double wilcox_p(long long u2, long long ties, int nx, int ny, const int32_t *cdf_idx, const double *cdf) {
    if (nx < EXACT_N && ny < EXACT_N && ties == 0) {
        const long long w = u2 / 2, mn = (long long)nx * ny;
        const double p = 2.0 * cdf[cdf_idx[nx * EXACT_N + ny] + (w < mn - w ? w : mn - w)];
        return p < 1.0 ? p : 1.0;
    }
    const double nxd = (double)nx, nyd = (double)ny, N = __dadd_rn(nxd, nyd);
    double z = __dadd_rn((double)u2 * 0.5, -(__dmul_rn(nxd, nyd) / 2.0));
    const double sigma = sqrt(__dmul_rn(__dmul_rn(nxd, nyd) / 12.0,
                                        __dadd_rn(__dadd_rn(N, 1.0), -((double)ties / __dmul_rn(N, __dadd_rn(N, -1.0))))));
    const double corr = z > 0.0 ? 0.5 : (z < 0.0 ? -0.5 : 0.0);
    z = __dadd_rn(z, -corr) / sigma;
    return erfc(fabs(z) * 0.70710678118654752440);   // 2 pnorm(-|z|); NaN when every value is tied (sigma = 0)
}

// (c) Wilcoxon: per item (gene gl, pair) the subcluster's jittered row sorted; each run of equal values v (b of them) adds
// b (2 lo + a) to 2 U_y and (a + b)^3 - (a + b) - (a^3 - a) to the ties, a = #(x == v), lo = #(x < v) in the sorted
// reference row.  p into PR[pair G + g0 + gl].
__global__ void __launch_bounds__(NT) pair_wilcox_kernel(const double *__restrict__ Z, int64_t T, int64_t gt, int64_t g0,
                                                         int64_t G, const int32_t *__restrict__ ref_off,
                                                         const int32_t *__restrict__ sub_off, int n_ref, int n_sub,
                                                         int64_t R_tot, unsigned long long seed, double jm, double js,
                                                         const double *__restrict__ RS, const long long *__restrict__ TS,
                                                         const int32_t *__restrict__ cdf_idx, const double *__restrict__ cdf,
                                                         double *PR, double *gbuf, int P) {
    extern __shared__ __align__(16) unsigned char de_smem[];
    __shared__ long long red[NT / 32];
    double *buf = gbuf ? gbuf + (size_t)blockIdx.x * P : reinterpret_cast<double *>(de_smem);
    const int64_t npair = (int64_t)n_sub * n_ref, items = gt * npair;
    for (int64_t it = blockIdx.x; it < items; it += gridDim.x) {
        const int64_t gl = it / npair, pair = it % npair;
        const int s = (int)(pair / n_ref), j = (int)(pair % n_ref);
        const int ys = sub_off[s], ny = sub_off[s + 1] - ys, xs = ref_off[j], nx = ref_off[j + 1] - xs, Pn = pow2_at_least(ny);
        const double *z = Z + gl * T + ys;   // sub_off: list positions within the row (the subclusters follow R_tot)
        const unsigned long long key = (1ull << 32) + (unsigned long long)pair;
        for (int i = threadIdx.x; i < Pn; i += NT)
            buf[i] = i < ny ? __dadd_rn(z[i], jitter(seed, key, (unsigned long long)(g0 + gl), i, jm, js)) : pos_inf();
        block_sort(buf, nullptr, Pn);
        const double *x = RS + gl * R_tot + xs;
        long long u2y = 0, ties = 0;
        for (int i = threadIdx.x; i < ny; i += NT) {
            const double v = buf[i];
            if (i > 0 && buf[i - 1] == v) continue;
            int e = i + 1;
            while (e < ny && buf[e] == v) ++e;
            const long long b = e - i, lo = bound(x, nx, v, false), a = bound(x, nx, v, true) - lo;
            u2y += b * (2 * lo + a);
            ties += tie_term(a + b) - tie_term(a);
        }
        u2y = block_sum_ll(u2y, red);
        ties = block_sum_ll(ties, red);
        if (threadIdx.x == 0) {
            const long long u2x = 2 * (long long)nx * ny - u2y;
            PR[pair * G + g0 + gl] = wilcox_p(u2x, ties + TS[gl * n_ref + j], nx, ny, cdf_idx, cdf);
        }
        __syncthreads();
    }
}

// block double-double sum in a fixed tree order; every thread gets hi + lo as (hi, lo)
__device__ void block_dd_sum(double &hi, double &lo, double *sh) {
    __syncthreads();
    sh[threadIdx.x] = hi;
    sh[NT + threadIdx.x] = lo;
    __syncthreads();
    for (int w = NT / 2; w > 0; w >>= 1) {
        if ((int)threadIdx.x < w) {
            double h = sh[threadIdx.x], l = sh[NT + threadIdx.x];
            dd_add(h, l, sh[threadIdx.x + w]);
            dd_add(h, l, sh[NT + threadIdx.x + w]);
            sh[threadIdx.x] = h;
            sh[NT + threadIdx.x] = l;
        }
        __syncthreads();
    }
    hi = sh[0];
    lo = sh[NT];
}

// (b) t: per item (gene gl, group k of the n_ref + n_sub groups over the T list positions) the mean (double-double sum,
// one division) and the variance (two-pass, double-double sum of the squared deviations) into ST[(gl ng + k) 2 + {0, 1}]
__global__ void __launch_bounds__(NT) group_stats_kernel(const double *__restrict__ Z, int64_t T, int64_t gt,
                                                         const int32_t *__restrict__ all_off, int ng, double *ST) {
    __shared__ double sh[2 * NT];
    const int64_t items = gt * ng;
    for (int64_t it = blockIdx.x; it < items; it += gridDim.x) {
        const int64_t gl = it / ng;
        const int k = (int)(it % ng);
        const int a = all_off[k], n = all_off[k + 1] - a;
        const double *z = Z + gl * T + a;
        double hi = 0.0, lo = 0.0;
        for (int i = threadIdx.x; i < n; i += NT) dd_add(hi, lo, z[i]);
        block_dd_sum(hi, lo, sh);
        const double m = dd_div(hi, lo, (double)n);
        hi = lo = 0.0;
        for (int i = threadIdx.x; i < n; i += NT) {
            const double d = z[i] - m;
            dd_add(hi, lo, __dmul_rn(d, d));
        }
        block_dd_sum(hi, lo, sh);
        if (threadIdx.x == 0) {
            ST[(gl * ng + k) * 2] = m;
            ST[(gl * ng + k) * 2 + 1] = n > 1 ? dd_div(hi, lo, (double)(n - 1)) : 0.0;
        }
    }
}

// lbeta(a, 1/2): lgamma(1/2) + lgamma(a) - lgamma(a + 1/2); for a >= 8 the difference of Stirling's series, written so that
// nothing cancels (|error| ~ 1e-16 absolute)
__device__ double lbeta_half(double a) {
    const double lg_half = 0.57236494292470008707;   // log(sqrt(pi))
    if (a < 8.0) return lg_half + lgamma(a) - lgamma(a + 0.5);
    auto cor = [](double x) {
        const double r = 1.0 / x, r2 = r * r;
        return r * (1.0 / 12 - r2 * (1.0 / 360 - r2 * (1.0 / 1260 - r2 * (1.0 / 1680 - r2 * (1.0 / 1188 - r2 * (691.0 / 360360))))));
    };
    return lg_half - 0.5 * log(a) + (0.5 - a * log1p(0.5 / a)) + (cor(a) - cor(a + 0.5));
}

// continued fraction of I_x(a, b) (modified Lentz)
__device__ double betacf(double a, double b, double x) {
    const double tiny = 1e-300, eps = 3e-16;
    const double qab = a + b, qap = a + 1.0, qam = a - 1.0;
    double c = 1.0, d = 1.0 - qab * x / qap;
    if (fabs(d) < tiny) d = tiny;
    d = 1.0 / d;
    double h = d;
    for (int m = 1; m <= 20000; ++m) {
        const double m2 = 2.0 * m;
        double aa = m * (b - m) * x / ((qam + m2) * (a + m2));
        d = 1.0 + aa * d;
        if (fabs(d) < tiny) d = tiny;
        c = 1.0 + aa / c;
        if (fabs(c) < tiny) c = tiny;
        d = 1.0 / d;
        h *= d * c;
        aa = -(a + m) * (qab + m) * x / ((a + m2) * (qap + m2));
        d = 1.0 + aa * d;
        if (fabs(d) < tiny) d = tiny;
        c = 1.0 + aa / c;
        if (fabs(c) < tiny) c = tiny;
        d = 1.0 / d;
        const double del = d * c;
        h *= del;
        if (fabs(del - 1.0) < eps) break;
    }
    return h;
}

// 2 pt(-|t|, df) = I_x(df / 2, 1 / 2), x = df / (df + t^2) = 1 / (1 + r), 1 - x = r / (1 + r), r = (t / df) t
__device__ double t_two_sided(double t, double df) {
    const double a = 0.5 * df, b = 0.5, r = (fabs(t) / df) * fabs(t);
    if (r == 0.0) return 1.0;
    if (isinf(r)) return 0.0;
    const double lx = -log1p(r), ly = log(r) - log1p(r), x = 1.0 / (1.0 + r), y = r / (1.0 + r);
    const double bt = exp(a * lx + b * ly - lbeta_half(a));
    if (x < (a + 1.0) / (a + b + 2.0)) return bt * betacf(a, b, x) / a;
    return 1.0 - bt * betacf(b, a, y) / b;
}

// (c) t: per (pair, gene gl), one thread each.  t.test.default's arithmetic in its order.
__global__ void __launch_bounds__(NT) pair_t_kernel(const double *__restrict__ ST, int64_t gt, int64_t g0, int64_t G,
                                                    const int32_t *__restrict__ all_off, int n_ref, int n_sub, double *PR) {
    const int ng = n_ref + n_sub;
    const int64_t npair = (int64_t)n_sub * n_ref, items = gt * npair;
    for (int64_t it = (int64_t)blockIdx.x * NT + threadIdx.x; it < items; it += (int64_t)gridDim.x * NT) {
        const int64_t pair = it / gt, gl = it % gt;
        const int s = (int)(pair / n_ref), j = (int)(pair % n_ref);
        const int kx = j, ky = n_ref + s;
        const int nx = all_off[kx + 1] - all_off[kx], ny = all_off[ky + 1] - all_off[ky];
        const double mx = ST[(gl * ng + kx) * 2], vx = ST[(gl * ng + kx) * 2 + 1];
        const double my = ST[(gl * ng + ky) * 2], vy = ST[(gl * ng + ky) * 2 + 1];
        double p = __longlong_as_double(0x7ff8000000000000ll);   // R's try() error: NA
        if (nx >= 2 && ny >= 2) {
            const double sx = sqrt(vx / nx), sy = sqrt(vy / ny);
            const double se = sqrt(__dadd_rn(__dmul_rn(sx, sx), __dmul_rn(sy, sy)));
            const double df = pow(se, 4.0) / __dadd_rn(pow(sx, 4.0) / (nx - 1), pow(sy, 4.0) / (ny - 1));
            const double lim = 10.0 * 2.220446049250313e-16 * fmax(fabs(mx), fabs(my));
            if (!(se < lim)) p = t_two_sided((mx - my) / se, df);   // se = 0 = lim: t and df NaN, so p NaN as in R
            if (se == 0.0 && !(se < lim)) p = __longlong_as_double(0x7ff8000000000000ll);
        }
        PR[pair * G + g0 + gl] = p;
    }
}

// (d) BH per pair over the G genes: p_adj[k] = min(1, min over the run ends i >= k's of (n / (i + 1)) p_(i)) on the
// ascending sort of the n non-NaN values - p.adjust's cummin, where a run of equal values all take the value of its last
// rank.  NaN stays NaN.  DE[pair G + g] = p_adj < thr.
__global__ void __launch_bounds__(NT) bh_kernel(const double *__restrict__ PR, int64_t G, int64_t npair, double thr,
                                                double *PA, unsigned char *DE, double *gkey, int32_t *gidx, int P) {
    extern __shared__ __align__(16) unsigned char de_smem[];
    __shared__ long long red[NT / 32];
    __shared__ double cmin[NT];
    double *key = gkey ? gkey + (size_t)blockIdx.x * P : reinterpret_cast<double *>(de_smem);
    int32_t *idx = gkey ? gidx + (size_t)blockIdx.x * P : reinterpret_cast<int32_t *>(de_smem + sizeof(double) * P);
    for (int64_t pair = blockIdx.x; pair < npair; pair += gridDim.x) {
        const double *p = PR + pair * G;
        long long valid = 0;
        for (int i = threadIdx.x; i < P; i += NT) {
            const double v = i < G ? p[i] : pos_inf();
            const bool ok = i < G && !isnan(v);
            valid += ok;
            key[i] = ok ? v : pos_inf();
            idx[i] = i;
        }
        const int n = (int)block_sum_ll(valid, red);
        block_sort(key, idx, P);
        // per thread a contiguous chunk of the n sorted values: q at the run ends, suffix minimum within the chunk
        const int chunk = (n + NT - 1) / NT, c0 = threadIdx.x * chunk, c1 = min(n, c0 + chunk);
        double m = pos_inf();
        for (int i = c1 - 1; i >= c0; --i)
            if (i == n - 1 || key[i + 1] != key[i]) m = fmin(m, ((double)n / (double)(i + 1)) * key[i]);
        cmin[threadIdx.x] = m;
        __syncthreads();
        double run = pos_inf();   // minimum over the later chunks
        for (int t = threadIdx.x + 1; t < NT; ++t) run = fmin(run, cmin[t]);
        for (int i = c1 - 1; i >= c0; --i) {
            if (i == n - 1 || key[i + 1] != key[i]) run = fmin(run, ((double)n / (double)(i + 1)) * key[i]);
            const double adj = fmin(1.0, run);
            PA[pair * G + idx[i]] = adj;
            DE[pair * G + idx[i]] = adj < thr;
        }
        for (int i = n + threadIdx.x; i < G; i += NT) {
            PA[pair * G + idx[i]] = __longlong_as_double(0x7ff8000000000000ll);
            DE[pair * G + idx[i]] = 0;
        }
        __syncthreads();
    }
}

// (e) one CTA per cell column (grid-stride): count = base[c] n_ref + sum over the >= 5-entry subclusters s holding c of
// sum_j DE[(s n_ref + j) G + g]; Y = masked ? mask_val : X
__global__ void __launch_bounds__(NT) mask_kernel(const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t G, int64_t C,
                                                  const unsigned char *__restrict__ base, const int32_t *__restrict__ cell_off,
                                                  const int32_t *__restrict__ cell_sub, int n_ref,
                                                  const unsigned char *__restrict__ DE, int rule, double mask_val) {
    for (int64_t c = blockIdx.x; c < C; c += gridDim.x) {
        const int b = base[c] ? n_ref : 0, s0 = cell_off[c], s1 = cell_off[c + 1];
        for (int64_t g = threadIdx.x; g < G; g += NT) {
            int cnt = b;
            for (int q = s0; q < s1; ++q) {
                const unsigned char *de = DE + (int64_t)cell_sub[q] * n_ref * G + g;
                for (int j = 0; j < n_ref; ++j) cnt += de[(int64_t)j * G];
            }
            const bool masked = rule == 0 ? cnt == 0 : (rule == 1 ? (double)cnt < (double)n_ref / 2.0 : cnt != n_ref);
            const double v = X[g + ldx * c];
            Y[g + ldy * c] = masked ? mask_val : v;
        }
    }
}

}  // namespace de

using namespace de;

// P(W <= w), w = 0 .. floor(m n / 2), of the rank-sum null of (m, n): the coefficients of the Gaussian binomial
// [m + n choose m]_q, built as prod_{k=1..m} (1 - q^(n+k)) / (1 - q^k) in exact 128-bit integers, summed and divided once
static void rank_sum_cdf(int m, int n, std::vector<double> &out) {
    const int mn = m * n;
    std::vector<unsigned __int128> c((size_t)mn + 1, 0);
    c[0] = 1;
    int deg = 0;
    for (int k = 1; k <= m; ++k) {
        const int sh = n + k;
        deg += n;
        for (int u = deg; u >= sh; --u) c[u] -= c[u - sh];   // * (1 - q^(n+k)); values stay exact modulo 2^128
        for (int u = k; u <= deg; ++u) c[u] += c[u - k];      // / (1 - q^k)
    }
    unsigned __int128 total = 0;
    for (int u = 0; u <= mn; ++u) total += c[u];
    unsigned __int128 cum = 0;
    for (int u = 0; u <= mn / 2; ++u) {
        cum += c[u];
        out.push_back((double)cum / (double)total);
    }
}

// What the last mask call of the process did: gene tiles, genes per tile, device ms of stages (a) - (e).
static double g_de_stats[7];

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

int de_mask_dev(const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t G, int64_t C, const int32_t *ref_off,
                const int32_t *ref_idx, int n_ref, const int32_t *sub_off, const int32_t *sub_idx, int n_sub, int test,
                double p_thresh, int rule, double mask_val, double jitter_mean, double jitter_sd, unsigned long long seed,
                double *p_raw, double *p_adj, void *stream, const char *who) {
    ICNV_REQUIRE_READY();
    if (!X || G < 1 || C < 1 || ldx < G || (Y && ldy < G) || n_ref < 1 || n_sub < 0 || !ref_off || !ref_idx ||
        (n_sub > 0 && (!sub_off || !sub_idx)))
        return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    if (test != 0 && test != 1) return set_error(ICNV_E_BAD_ARG, "%s: unknown test code %d", who, test);
    if (rule < 0 || rule > 2) return set_error(ICNV_E_BAD_ARG, "%s: unknown rule code %d", who, rule);
    if (!std::isfinite(jitter_mean) || !std::isfinite(jitter_sd) || jitter_sd < 0.0 || std::isnan(p_thresh))
        return set_error(ICNV_E_BAD_ARG, "%s: bad jitter or threshold", who);
    if (ref_off[0] != 0 || (n_sub > 0 && sub_off[0] != 0)) return set_error(ICNV_E_BAD_ARG, "%s: offsets must start at 0", who);
    for (int k = 0; k < n_ref; ++k)
        if (ref_off[k + 1] <= ref_off[k]) return set_error(ICNV_E_BAD_ARG, "%s: reference group %d is empty", who, k);
    for (int k = 0; k < n_sub; ++k)
        if (sub_off[k + 1] <= sub_off[k]) return set_error(ICNV_E_BAD_ARG, "%s: subcluster %d is empty", who, k);
    const int64_t R_tot = ref_off[n_ref], S_tot = n_sub > 0 ? sub_off[n_sub] : 0, T = R_tot + S_tot;
    if (T > (int64_t)INT32_MAX / 2) return set_error(ICNV_E_UNSUPPORTED, "%s: %lld listed cells", who, (long long)T);
    std::vector<int32_t> cols((size_t)T);
    for (int64_t i = 0; i < R_tot; ++i) cols[(size_t)i] = ref_idx[i];
    for (int64_t i = 0; i < S_tot; ++i) cols[(size_t)(R_tot + i)] = sub_idx[i];
    for (int32_t v : cols)
        if (v < 0 || v >= C) return set_error(ICNV_E_BAD_ARG, "%s: cell index %d out of range", who, v);
    // every group's offsets over the T list positions: reference groups, then subclusters
    std::vector<int32_t> all_off((size_t)(n_ref + n_sub + 1));
    for (int k = 0; k <= n_ref; ++k) all_off[(size_t)k] = ref_off[k];
    for (int k = 1; k <= n_sub; ++k) all_off[(size_t)(n_ref + k)] = (int32_t)(R_tot + sub_off[k]);
    // the count's start per cell and, per cell, the >= 5-entry subclusters holding it (each once)
    std::vector<unsigned char> base((size_t)C, 0);
    for (int64_t i = 0; i < R_tot; ++i) base[(size_t)ref_idx[i]] = 1;
    std::vector<int32_t> cnt((size_t)C + 1, 0), last((size_t)C, -1);
    for (int s = 0; s < n_sub; ++s) {
        const bool small = sub_off[s + 1] - sub_off[s] < 5;
        for (int32_t i = sub_off[s]; i < sub_off[s + 1]; ++i) {
            const int32_t c = sub_idx[i];
            if (small) base[(size_t)c] = 1;
            else if (last[(size_t)c] != s) { last[(size_t)c] = s; cnt[(size_t)c + 1]++; }
        }
    }
    for (int64_t c = 0; c < C; ++c) cnt[(size_t)c + 1] += cnt[(size_t)c];
    std::vector<int32_t> cell_sub((size_t)std::max<int32_t>(cnt[(size_t)C], 1)), fill(cnt.begin(), cnt.end() - 1);
    std::fill(last.begin(), last.end(), -1);
    for (int s = 0; s < n_sub; ++s) {
        if (sub_off[s + 1] - sub_off[s] < 5) continue;
        for (int32_t i = sub_off[s]; i < sub_off[s + 1]; ++i) {
            const int32_t c = sub_idx[i];
            if (last[(size_t)c] != s) { last[(size_t)c] = s; cell_sub[(size_t)fill[(size_t)c]++] = s; }
        }
    }
    // exact null tables of the pairs with both sizes < 50 (Wilcoxon)
    std::vector<int32_t> cdf_idx((size_t)EXACT_N * EXACT_N, -1);
    std::vector<double> cdf;
    int max_ny = 1, max_nx = 1;
    for (int j = 0; j < n_ref; ++j) max_nx = std::max(max_nx, ref_off[j + 1] - ref_off[j]);
    for (int s = 0; s < n_sub; ++s) max_ny = std::max(max_ny, sub_off[s + 1] - sub_off[s]);
    if (test == 0)
        for (int s = 0; s < n_sub; ++s)
            for (int j = 0; j < n_ref; ++j) {
                const int nx = ref_off[j + 1] - ref_off[j], ny = sub_off[s + 1] - sub_off[s];
                if (nx >= EXACT_N || ny >= EXACT_N || cdf_idx[(size_t)(nx * EXACT_N + ny)] >= 0) continue;
                cdf_idx[(size_t)(nx * EXACT_N + ny)] = (int32_t)cdf.size();
                rank_sum_cdf(nx, ny, cdf);
            }
    if (cdf.empty()) cdf.push_back(0.0);

    Ctx &c = ctx();
    cudaStream_t st = pick_stream(stream);
    const int64_t npair = (int64_t)n_sub * n_ref;
    const int ng = n_ref + n_sub;
    int Psort = 1;   // the largest row sort
    while (Psort < std::max(max_nx, max_ny)) Psort <<= 1;
    int PG = 1;
    while (PG < G) PG <<= 1;
    const bool sort_global = sizeof(double) * (size_t)Psort > SORT_SMEM;
    const bool bh_global = (sizeof(double) + sizeof(int32_t)) * (size_t)PG > SORT_SMEM;
    const int grid_sort = c.sm_count * (sort_global ? 4 : 16);
    const int grid_bh = (int)std::min<int64_t>(std::max<int64_t>(npair, 1), (int64_t)c.sm_count * 2);
    // fixed part of the one device allocation
    size_t fixed = 0;
    auto take = [&](size_t b) { const size_t o = fixed; fixed += align256(b); return o; };
    const size_t o_cols = take(sizeof(int32_t) * (size_t)T), o_alloff = take(sizeof(int32_t) * all_off.size()),
                 o_base = take((size_t)C), o_celloff = take(sizeof(int32_t) * cnt.size()),
                 o_cellsub = take(sizeof(int32_t) * cell_sub.size()), o_cdfidx = take(sizeof(int32_t) * cdf_idx.size()),
                 o_cdf = take(sizeof(double) * cdf.size()), o_flag = take(sizeof(int)),
                 o_pr = p_raw ? 0 : take(sizeof(double) * (size_t)(G * std::max<int64_t>(npair, 1))),
                 o_pa = p_adj ? 0 : take(sizeof(double) * (size_t)(G * std::max<int64_t>(npair, 1))),
                 o_de = take((size_t)(G * std::max<int64_t>(npair, 1))),
                 o_sort = take(sort_global ? sizeof(double) * (size_t)Psort * grid_sort : 0),
                 o_bhk = take(bh_global ? sizeof(double) * (size_t)PG * grid_bh : 0),
                 o_bhi = take(bh_global ? sizeof(int32_t) * (size_t)PG * grid_bh : 0);
    const size_t per_gene = sizeof(double) * (size_t)(T + (test == 0 ? R_tot : 0)) +
                            (test == 0 ? sizeof(long long) * (size_t)n_ref : sizeof(double) * 2 * (size_t)ng);
    size_t free_b = 0, total_b = 0;
    ICNV_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const size_t usable = free_b > (size_t)(512 << 20) ? free_b - (size_t)(512 << 20) : 0;
    if (usable < fixed + per_gene + 4096) return set_error(ICNV_E_NOMEM, "%s: not even one gene fits in device memory", who);
    const int64_t gt = std::min<int64_t>(G, (int64_t)((usable - fixed - 4096) / per_gene));
    const size_t o_z = take(sizeof(double) * (size_t)(gt * T)), o_rs = take(test == 0 ? sizeof(double) * (size_t)(gt * R_tot) : 0),
                 o_ts = take(test == 0 ? sizeof(long long) * (size_t)(gt * n_ref) : sizeof(double) * 2 * (size_t)(gt * ng));
    char *buf = nullptr;
    if (cudaMallocAsync((void **)&buf, fixed, st) != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NOMEM, "%s: no room for %lld bytes", who, (long long)fixed);
    }
    int32_t *d_cols = (int32_t *)(buf + o_cols), *d_alloff = (int32_t *)(buf + o_alloff), *d_celloff = (int32_t *)(buf + o_celloff),
            *d_cellsub = (int32_t *)(buf + o_cellsub), *d_cdfidx = (int32_t *)(buf + o_cdfidx);
    unsigned char *d_base = (unsigned char *)(buf + o_base), *d_de = (unsigned char *)(buf + o_de);
    double *d_cdf = (double *)(buf + o_cdf), *PR = p_raw ? p_raw : (double *)(buf + o_pr), *PA = p_adj ? p_adj : (double *)(buf + o_pa);
    double *d_sort = sort_global ? (double *)(buf + o_sort) : nullptr, *d_bhk = bh_global ? (double *)(buf + o_bhk) : nullptr;
    int32_t *d_bhi = bh_global ? (int32_t *)(buf + o_bhi) : nullptr;
    int *d_flag = (int *)(buf + o_flag);
    double *Z = (double *)(buf + o_z), *RS = (double *)(buf + o_rs);
    long long *TS = (long long *)(buf + o_ts);
    double *ST = (double *)(buf + o_ts);
    const int32_t *d_refoff = d_alloff, *d_suboff = d_alloff + n_ref;   // list positions of every group within a Z row
    cudaEvent_t ev[6] = {};
    for (auto &e : ev) ICNV_CUDA(cudaEventCreate(&e));
    auto body = [&]() -> int {
        ICNV_CUDA(cudaMemcpyAsync(d_cols, cols.data(), sizeof(int32_t) * (size_t)T, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_alloff, all_off.data(), sizeof(int32_t) * all_off.size(), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_base, base.data(), (size_t)C, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_celloff, cnt.data(), sizeof(int32_t) * cnt.size(), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_cellsub, cell_sub.data(), sizeof(int32_t) * cell_sub.size(), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_cdfidx, cdf_idx.data(), sizeof(int32_t) * cdf_idx.size(), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_cdf, cdf.data(), sizeof(double) * cdf.size(), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
        double t[5] = {0, 0, 0, 0, 0};
        const size_t smem_sort = sort_global ? 0 : sizeof(double) * (size_t)Psort;
        if (smem_sort > 48 * 1024) {
            ICNV_CUDA(cudaFuncSetAttribute(ref_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sort));
            ICNV_CUDA(cudaFuncSetAttribute(pair_wilcox_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sort));
        }
        for (int64_t g0 = 0; g0 < G; g0 += gt) {
            const int64_t n = std::min<int64_t>(gt, G - g0);
            ICNV_CUDA(cudaEventRecord(ev[0], st));
            gather_kernel<<<dim3((unsigned)((T + 31) / 32), (unsigned)((n + 31) / 32)), NT, 0, st>>>(X, ldx, d_cols, T, g0, n, Z, d_flag);
            ICNV_CHECK_LAUNCH("gather_kernel");
            ICNV_CUDA(cudaEventRecord(ev[1], st));
            if (test == 0) {
                const unsigned gb = (unsigned)std::min<int64_t>(n * n_ref, grid_sort);
                ref_sort_kernel<<<gb, NT, smem_sort, st>>>(Z, T, n, g0, d_refoff, n_ref, R_tot, seed, jitter_mean, jitter_sd, RS,
                                                           TS, d_sort, Psort);
                ICNV_CHECK_LAUNCH("ref_sort_kernel");
            } else {
                const unsigned gb = (unsigned)std::min<int64_t>(n * ng, (int64_t)c.sm_count * 16);
                group_stats_kernel<<<gb, NT, 0, st>>>(Z, T, n, d_alloff, ng, ST);
                ICNV_CHECK_LAUNCH("group_stats_kernel");
            }
            ICNV_CUDA(cudaEventRecord(ev[2], st));
            if (npair > 0 && test == 0) {
                const unsigned gb = (unsigned)std::min<int64_t>(n * npair, grid_sort);
                pair_wilcox_kernel<<<gb, NT, smem_sort, st>>>(Z, T, n, g0, G, d_refoff, d_suboff, n_ref, n_sub, R_tot,
                                                              seed, jitter_mean, jitter_sd, RS, TS, d_cdfidx, d_cdf, PR,
                                                              d_sort, Psort);
                ICNV_CHECK_LAUNCH("pair_wilcox_kernel");
            } else if (npair > 0) {
                const unsigned gb = (unsigned)std::min<int64_t>((n * npair + NT - 1) / NT, (int64_t)c.sm_count * 32);
                pair_t_kernel<<<gb, NT, 0, st>>>(ST, n, g0, G, d_alloff, n_ref, n_sub, PR);
                ICNV_CHECK_LAUNCH("pair_t_kernel");
            }
            ICNV_CUDA(cudaEventRecord(ev[3], st));
            int h = 0;   // each tile's gather reports its own non-finite values
            ICNV_CUDA(cudaMemcpyAsync(&h, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
            ICNV_CUDA(cudaStreamSynchronize(st));
            if (h) return set_error(ICNV_E_NONFINITE, "%s: NaN or Inf in a listed cell", who);
            float ms = 0.0f;
            for (int s = 0; s < 3; ++s) {
                ICNV_CUDA(cudaEventElapsedTime(&ms, ev[s], ev[s + 1]));
                t[s] += ms;
            }
        }
        ICNV_CUDA(cudaEventRecord(ev[3], st));
        if (npair > 0) {
            const size_t smem_bh = bh_global ? 0 : (sizeof(double) + sizeof(int32_t)) * (size_t)PG;
            if (smem_bh > 48 * 1024) ICNV_CUDA(cudaFuncSetAttribute(bh_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bh));
            bh_kernel<<<(unsigned)grid_bh, NT, smem_bh, st>>>(PR, G, npair, p_thresh, PA, d_de, d_bhk, d_bhi, PG);
            ICNV_CHECK_LAUNCH("bh_kernel");
        }
        ICNV_CUDA(cudaEventRecord(ev[4], st));
        if (Y) {
            mask_kernel<<<(unsigned)std::min<int64_t>(C, 65535), NT, 0, st>>>(X, ldx, Y, ldy, G, C, d_base, d_celloff, d_cellsub,
                                                                               n_ref, d_de, rule, mask_val);
            ICNV_CHECK_LAUNCH("mask_kernel");
        }
        ICNV_CUDA(cudaEventRecord(ev[5], st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        float ms = 0.0f;
        ICNV_CUDA(cudaEventElapsedTime(&ms, ev[3], ev[4]));
        t[3] = ms;
        ICNV_CUDA(cudaEventElapsedTime(&ms, ev[4], ev[5]));
        t[4] = ms;
        g_de_stats[0] = (double)((G + gt - 1) / gt);
        g_de_stats[1] = (double)gt;
        for (int s = 0; s < 5; ++s) g_de_stats[2 + s] = t[s];
        return ICNV_OK;
    };
    const int rc = body();
    cudaFreeAsync(buf, st);
    for (auto &e : ev)
        if (e) cudaEventDestroy(e);
    return rc;
}

void de_mask_stats(double *out7) {
    for (int i = 0; i < 7; ++i) out7[i] = g_de_stats[i];
}

}  // namespace icnv
