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
//
// The stages are also entry points of their own, for callers that split the genes over devices or ranks: the pack of a
// rank's listed cells per destination gene range (the gather's transpose), the placing of received blocks by list position,
// (b) + (c) on a slab of genes, and (d) + (e) on a block of cells.  A split gives the bytes of one call for any number of
// parts (icnv_de_multi.cu, device.py's Engine.mask_non_de_sharded).
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
// reference row.  p into PR[pair ldp + gl] (g0 + gl the absolute gene).
__global__ void __launch_bounds__(NT) pair_wilcox_kernel(const double *__restrict__ Z, int64_t T, int64_t gt, int64_t g0,
                                                         int64_t ldp, const int32_t *__restrict__ ref_off,
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
            PR[pair * ldp + gl] = wilcox_p(u2x, ties + TS[gl * n_ref + j], nx, ny, cdf_idx, cdf);
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

// (c) t: per (pair, gene gl), one thread each.  t.test.default's arithmetic in its order.  p into PR[pair ldp + gl].
__global__ void __launch_bounds__(NT) pair_t_kernel(const double *__restrict__ ST, int64_t gt, int64_t ldp,
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
        PR[pair * ldp + gl] = p;
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

// Receiving side of the gene exchange of the rank-sharded path: `blk` is one source rank's gene-major block (n genes x m
// listed cells, in that rank's list order) and tags[k] the global list position of its entry k, so each value goes
// straight to its place in the slab rows Z (n x T, every row in global list order).
__global__ void __launch_bounds__(NT) place_kernel(const double *__restrict__ blk, int64_t n, int64_t m,
                                                   const int32_t *__restrict__ tags, int64_t T, double *__restrict__ Z) {
    for (int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x; i < n * m; i += (int64_t)gridDim.x * NT) {
        const int64_t gl = i / m, k = i - gl * m;
        Z[gl * T + tags[k]] = blk[i];
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

namespace {

// one device allocation carved into 256-byte aligned pieces
struct Layout {
    size_t bytes = 0;
    size_t take(size_t b) {
        const size_t o = bytes;
        bytes += align256(b);
        return o;
    }
};

// Host side of the tests (stages (b) and (c)) for one set of groups: every group's offsets over the T list positions
// (reference groups, then subclusters), the exact null tables of the Wilcoxon pairs with both sizes < 50, the sort sizes.
struct TestPlan {
    int n_ref = 0, n_sub = 0, test = 0;
    int64_t R_tot = 0, T = 0;
    std::vector<int32_t> all_off, cdf_idx;
    std::vector<double> cdf;
    int Psort = 1;   // the largest row sort
    bool sort_global = false;
};

int make_test_plan(const int32_t *ref_off, int n_ref, const int32_t *sub_off, int n_sub, int test, TestPlan &p,
                   const char *who) {
    if (n_ref < 1 || n_sub < 0 || !ref_off || (n_sub > 0 && !sub_off)) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    if (test != 0 && test != 1) return set_error(ICNV_E_BAD_ARG, "%s: unknown test code %d", who, test);
    if (ref_off[0] != 0 || (n_sub > 0 && sub_off[0] != 0)) return set_error(ICNV_E_BAD_ARG, "%s: offsets must start at 0", who);
    for (int k = 0; k < n_ref; ++k)
        if (ref_off[k + 1] <= ref_off[k]) return set_error(ICNV_E_BAD_ARG, "%s: reference group %d is empty", who, k);
    for (int k = 0; k < n_sub; ++k)
        if (sub_off[k + 1] <= sub_off[k]) return set_error(ICNV_E_BAD_ARG, "%s: subcluster %d is empty", who, k);
    p.n_ref = n_ref;
    p.n_sub = n_sub;
    p.test = test;
    p.R_tot = ref_off[n_ref];
    p.T = p.R_tot + (n_sub > 0 ? sub_off[n_sub] : 0);
    if (p.T > (int64_t)INT32_MAX / 2) return set_error(ICNV_E_UNSUPPORTED, "%s: %lld listed cells", who, (long long)p.T);
    p.all_off.assign((size_t)(n_ref + n_sub + 1), 0);
    for (int k = 0; k <= n_ref; ++k) p.all_off[(size_t)k] = ref_off[k];
    for (int k = 1; k <= n_sub; ++k) p.all_off[(size_t)(n_ref + k)] = (int32_t)(p.R_tot + sub_off[k]);
    p.cdf_idx.assign((size_t)EXACT_N * EXACT_N, -1);
    p.cdf.clear();
    int max_ny = 1, max_nx = 1;
    for (int j = 0; j < n_ref; ++j) max_nx = std::max(max_nx, ref_off[j + 1] - ref_off[j]);
    for (int s = 0; s < n_sub; ++s) max_ny = std::max(max_ny, sub_off[s + 1] - sub_off[s]);
    if (test == 0)
        for (int s = 0; s < n_sub; ++s)
            for (int j = 0; j < n_ref; ++j) {
                const int nx = ref_off[j + 1] - ref_off[j], ny = sub_off[s + 1] - sub_off[s];
                if (nx >= EXACT_N || ny >= EXACT_N || p.cdf_idx[(size_t)(nx * EXACT_N + ny)] >= 0) continue;
                p.cdf_idx[(size_t)(nx * EXACT_N + ny)] = (int32_t)p.cdf.size();
                rank_sum_cdf(nx, ny, p.cdf);
            }
    if (p.cdf.empty()) p.cdf.push_back(0.0);
    p.Psort = 1;
    while (p.Psort < std::max(max_nx, max_ny)) p.Psort <<= 1;
    p.sort_global = sizeof(double) * (size_t)p.Psort > SORT_SMEM;
    return ICNV_OK;
}

// Device side of a TestPlan: its tables and sort scratch (fixed) and the per-gene scratch of tiles of up to gt genes.
struct TestDev {
    size_t o_alloff = 0, o_cdfidx = 0, o_cdf = 0, o_sort = 0, o_rs = 0, o_ts = 0;
    int32_t *alloff = nullptr, *cdfidx = nullptr;
    double *cdf = nullptr, *sort = nullptr, *RS = nullptr, *ST = nullptr;
    long long *TS = nullptr;
    int grid_sort = 0;

    void fixed(const TestPlan &p, int sm_count, Layout &L) {
        grid_sort = sm_count * (p.sort_global ? 4 : 16);
        o_alloff = L.take(sizeof(int32_t) * p.all_off.size());
        o_cdfidx = L.take(sizeof(int32_t) * p.cdf_idx.size());
        o_cdf = L.take(sizeof(double) * p.cdf.size());
        o_sort = L.take(p.sort_global ? sizeof(double) * (size_t)p.Psort * grid_sort : 0);
    }
    static size_t per_gene(const TestPlan &p) {
        return p.test == 0 ? sizeof(double) * (size_t)p.R_tot + sizeof(long long) * (size_t)p.n_ref
                           : sizeof(double) * 2 * (size_t)(p.n_ref + p.n_sub);
    }
    void tiles(const TestPlan &p, int64_t gt, Layout &L) {
        const int ng = p.n_ref + p.n_sub;
        o_rs = L.take(p.test == 0 ? sizeof(double) * (size_t)(gt * p.R_tot) : 0);
        o_ts = L.take(p.test == 0 ? sizeof(long long) * (size_t)(gt * p.n_ref) : sizeof(double) * 2 * (size_t)(gt * ng));
    }
    void bind(const TestPlan &p, char *buf) {
        alloff = (int32_t *)(buf + o_alloff);
        cdfidx = (int32_t *)(buf + o_cdfidx);
        cdf = (double *)(buf + o_cdf);
        sort = p.sort_global ? (double *)(buf + o_sort) : nullptr;
        RS = (double *)(buf + o_rs);
        TS = (long long *)(buf + o_ts);
        ST = (double *)(buf + o_ts);
    }
    int upload(const TestPlan &p, cudaStream_t st) const {
        ICNV_CUDA(cudaMemcpyAsync(alloff, p.all_off.data(), sizeof(int32_t) * p.all_off.size(), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(cdfidx, p.cdf_idx.data(), sizeof(int32_t) * p.cdf_idx.size(), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(cdf, p.cdf.data(), sizeof(double) * p.cdf.size(), cudaMemcpyHostToDevice, st));
        const size_t smem_sort = p.sort_global ? 0 : sizeof(double) * (size_t)p.Psort;
        if (smem_sort > 48 * 1024) {
            ICNV_CUDA(cudaFuncSetAttribute(ref_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sort));
            ICNV_CUDA(cudaFuncSetAttribute(pair_wilcox_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sort));
        }
        return ICNV_OK;
    }
    // stages (b) and (c) on the n gene-major rows Z (absolute genes g0 ..): p into PR[pair ldp + gl].  `mid`, when given,
    // is recorded between the two stages.
    int launch(const TestPlan &p, const double *Z, int64_t g0, int64_t n, double *PR, int64_t ldp, double jm, double js,
               unsigned long long seed, int sm_count, cudaStream_t st, cudaEvent_t mid) const {
        const int64_t npair = (int64_t)p.n_sub * p.n_ref;
        const int ng = p.n_ref + p.n_sub;
        const size_t smem_sort = p.sort_global ? 0 : sizeof(double) * (size_t)p.Psort;
        const int32_t *refoff = alloff, *suboff = alloff + p.n_ref;   // list positions of every group within a Z row
        if (p.test == 0) {
            const unsigned gb = (unsigned)std::min<int64_t>(n * p.n_ref, grid_sort);
            ref_sort_kernel<<<gb, NT, smem_sort, st>>>(Z, p.T, n, g0, refoff, p.n_ref, p.R_tot, seed, jm, js, RS, TS, sort,
                                                       p.Psort);
            ICNV_CHECK_LAUNCH("ref_sort_kernel");
        } else {
            const unsigned gb = (unsigned)std::min<int64_t>(n * ng, (int64_t)sm_count * 16);
            group_stats_kernel<<<gb, NT, 0, st>>>(Z, p.T, n, alloff, ng, ST);
            ICNV_CHECK_LAUNCH("group_stats_kernel");
        }
        if (mid) ICNV_CUDA(cudaEventRecord(mid, st));
        if (npair > 0 && p.test == 0) {
            const unsigned gb = (unsigned)std::min<int64_t>(n * npair, grid_sort);
            pair_wilcox_kernel<<<gb, NT, smem_sort, st>>>(Z, p.T, n, g0, ldp, refoff, suboff, p.n_ref, p.n_sub, p.R_tot, seed,
                                                          jm, js, RS, TS, cdfidx, cdf, PR, sort, p.Psort);
            ICNV_CHECK_LAUNCH("pair_wilcox_kernel");
        } else if (npair > 0) {
            const unsigned gb = (unsigned)std::min<int64_t>((n * npair + NT - 1) / NT, (int64_t)sm_count * 32);
            pair_t_kernel<<<gb, NT, 0, st>>>(ST, n, ldp, alloff, p.n_ref, p.n_sub, PR);
            ICNV_CHECK_LAUNCH("pair_t_kernel");
        }
        return ICNV_OK;
    }
};

// Host side of the mask (stage (e)) for a block of C columns: per cell the count's start (reference cells and the cells of a
// tested subcluster of < 5 list entries start at n_ref) and the >= 5-entry subclusters holding it, each once.  sub_size[s]
// is subcluster s's whole list length; sub_off / sub_idx list the cells of the block it holds (possibly none).
struct MaskPlan {
    std::vector<unsigned char> base;
    std::vector<int32_t> cell_off, cell_sub;
};

int make_mask_plan(int64_t C, const int32_t *ref_idx, int64_t n_ref_cells, const int32_t *sub_off, const int32_t *sub_idx,
                   int n_sub, const int32_t *sub_size, MaskPlan &m, const char *who) {
    for (int64_t i = 0; i < n_ref_cells; ++i)
        if (ref_idx[i] < 0 || ref_idx[i] >= C) return set_error(ICNV_E_BAD_ARG, "%s: cell index %d out of range", who, ref_idx[i]);
    for (int s = 0; s < n_sub; ++s)
        for (int32_t i = sub_off[s]; i < sub_off[s + 1]; ++i)
            if (sub_idx[i] < 0 || sub_idx[i] >= C) return set_error(ICNV_E_BAD_ARG, "%s: cell index %d out of range", who, sub_idx[i]);
    m.base.assign((size_t)C, 0);
    for (int64_t i = 0; i < n_ref_cells; ++i) m.base[(size_t)ref_idx[i]] = 1;
    std::vector<int32_t> last((size_t)C, -1);
    m.cell_off.assign((size_t)C + 1, 0);
    for (int s = 0; s < n_sub; ++s) {
        const bool small = sub_size[s] < 5;
        for (int32_t i = sub_off[s]; i < sub_off[s + 1]; ++i) {
            const int32_t c = sub_idx[i];
            if (small) m.base[(size_t)c] = 1;
            else if (last[(size_t)c] != s) { last[(size_t)c] = s; m.cell_off[(size_t)c + 1]++; }
        }
    }
    for (int64_t c = 0; c < C; ++c) m.cell_off[(size_t)c + 1] += m.cell_off[(size_t)c];
    m.cell_sub.assign((size_t)std::max<int32_t>(m.cell_off[(size_t)C], 1), 0);
    std::vector<int32_t> fill(m.cell_off.begin(), m.cell_off.end() - 1);
    std::fill(last.begin(), last.end(), -1);
    for (int s = 0; s < n_sub; ++s) {
        if (sub_size[s] < 5) continue;
        for (int32_t i = sub_off[s]; i < sub_off[s + 1]; ++i) {
            const int32_t c = sub_idx[i];
            if (last[(size_t)c] != s) { last[(size_t)c] = s; m.cell_sub[(size_t)fill[(size_t)c]++] = s; }
        }
    }
    return ICNV_OK;
}

// Device side of stages (d) and (e): the DE bytes, BH's sort scratch and a MaskPlan's tables.
struct BhMaskDev {
    size_t o_de = 0, o_bhk = 0, o_bhi = 0, o_base = 0, o_celloff = 0, o_cellsub = 0;
    unsigned char *DE = nullptr, *base = nullptr;
    double *bhk = nullptr;
    int32_t *bhi = nullptr, *celloff = nullptr, *cellsub = nullptr;
    int PG = 1, grid_bh = 1;
    bool bh_global = false;

    void fixed(int64_t G, int64_t npair, const MaskPlan &m, int sm_count, Layout &L) {
        PG = 1;
        while (PG < G) PG <<= 1;
        bh_global = (sizeof(double) + sizeof(int32_t)) * (size_t)PG > SORT_SMEM;
        grid_bh = (int)std::min<int64_t>(std::max<int64_t>(npair, 1), (int64_t)sm_count * 2);
        o_base = L.take(m.base.size());
        o_celloff = L.take(sizeof(int32_t) * m.cell_off.size());
        o_cellsub = L.take(sizeof(int32_t) * m.cell_sub.size());
        o_de = L.take((size_t)(G * std::max<int64_t>(npair, 1)));
        o_bhk = L.take(bh_global ? sizeof(double) * (size_t)PG * grid_bh : 0);
        o_bhi = L.take(bh_global ? sizeof(int32_t) * (size_t)PG * grid_bh : 0);
    }
    void bind(char *buf) {
        DE = (unsigned char *)(buf + o_de);
        base = (unsigned char *)(buf + o_base);
        celloff = (int32_t *)(buf + o_celloff);
        cellsub = (int32_t *)(buf + o_cellsub);
        bhk = bh_global ? (double *)(buf + o_bhk) : nullptr;
        bhi = bh_global ? (int32_t *)(buf + o_bhi) : nullptr;
    }
    int upload(const MaskPlan &m, cudaStream_t st) const {
        ICNV_CUDA(cudaMemcpyAsync(base, m.base.data(), m.base.size(), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(celloff, m.cell_off.data(), sizeof(int32_t) * m.cell_off.size(), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(cellsub, m.cell_sub.data(), sizeof(int32_t) * m.cell_sub.size(), cudaMemcpyHostToDevice, st));
        return ICNV_OK;
    }
    int bh(const double *PR, int64_t G, int64_t npair, double thr, double *PA, cudaStream_t st) const {
        if (npair == 0) return ICNV_OK;
        const size_t smem_bh = bh_global ? 0 : (sizeof(double) + sizeof(int32_t)) * (size_t)PG;
        if (smem_bh > 48 * 1024) ICNV_CUDA(cudaFuncSetAttribute(bh_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bh));
        bh_kernel<<<(unsigned)grid_bh, NT, smem_bh, st>>>(PR, G, npair, thr, PA, DE, bhk, bhi, PG);
        ICNV_CHECK_LAUNCH("bh_kernel");
        return ICNV_OK;
    }
    int mask(const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t G, int64_t C, int n_ref, int rule, double mask_val,
             cudaStream_t st) const {
        if (!Y || C == 0) return ICNV_OK;
        mask_kernel<<<(unsigned)std::min<int64_t>(C, 65535), NT, 0, st>>>(X, ldx, Y, ldy, G, C, base, celloff, cellsub, n_ref,
                                                                           DE, rule, mask_val);
        ICNV_CHECK_LAUNCH("mask_kernel");
        return ICNV_OK;
    }
};

// free device memory less a 512 MB margin
size_t usable_device_bytes() {
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) return 0;
    return free_b > (size_t)(512 << 20) ? free_b - (size_t)(512 << 20) : 0;
}

int alloc_layout(char **buf, const Layout &L, cudaStream_t st, const char *who) {
    if (cudaMallocAsync((void **)buf, L.bytes, st) != cudaSuccess) {
        cudaGetLastError();
        *buf = nullptr;
        return set_error(ICNV_E_NOMEM, "%s: no room for %lld bytes", who, (long long)L.bytes);
    }
    return ICNV_OK;
}

int check_jitter(double jitter_mean, double jitter_sd, double p_thresh, const char *who) {
    if (!std::isfinite(jitter_mean) || !std::isfinite(jitter_sd) || jitter_sd < 0.0 || std::isnan(p_thresh))
        return set_error(ICNV_E_BAD_ARG, "%s: bad jitter or threshold", who);
    return ICNV_OK;
}

}  // namespace

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
    int rc = check_jitter(jitter_mean, jitter_sd, p_thresh, who);
    if (rc) return rc;
    TestPlan tp;
    if ((rc = make_test_plan(ref_off, n_ref, sub_off, n_sub, test, tp, who))) return rc;
    const int64_t R_tot = tp.R_tot, T = tp.T;
    std::vector<int32_t> cols((size_t)T);
    for (int64_t i = 0; i < R_tot; ++i) cols[(size_t)i] = ref_idx[i];
    for (int64_t i = R_tot; i < T; ++i) cols[(size_t)i] = sub_idx[i - R_tot];
    for (int32_t v : cols)
        if (v < 0 || v >= C) return set_error(ICNV_E_BAD_ARG, "%s: cell index %d out of range", who, v);
    std::vector<int32_t> sub_size((size_t)std::max(n_sub, 1));
    for (int s = 0; s < n_sub; ++s) sub_size[(size_t)s] = sub_off[s + 1] - sub_off[s];
    MaskPlan mp;
    if ((rc = make_mask_plan(C, ref_idx, R_tot, sub_off, sub_idx, n_sub, sub_size.data(), mp, who))) return rc;

    Ctx &c = ctx();
    cudaStream_t st = pick_stream(stream);
    const int64_t npair = (int64_t)n_sub * n_ref;
    // fixed part of the one device allocation
    Layout L;
    TestDev td;
    BhMaskDev bm;
    const size_t o_cols = L.take(sizeof(int32_t) * (size_t)T), o_flag = L.take(sizeof(int)),
                 o_pr = p_raw ? 0 : L.take(sizeof(double) * (size_t)(G * std::max<int64_t>(npair, 1))),
                 o_pa = p_adj ? 0 : L.take(sizeof(double) * (size_t)(G * std::max<int64_t>(npair, 1)));
    td.fixed(tp, c.sm_count, L);
    bm.fixed(G, npair, mp, c.sm_count, L);
    const size_t per_gene = sizeof(double) * (size_t)T + TestDev::per_gene(tp);
    const size_t usable = usable_device_bytes();
    if (usable < L.bytes + per_gene + 4096) return set_error(ICNV_E_NOMEM, "%s: not even one gene fits in device memory", who);
    const int64_t gt = std::min<int64_t>(G, (int64_t)((usable - L.bytes - 4096) / per_gene));
    const size_t o_z = L.take(sizeof(double) * (size_t)(gt * T));
    td.tiles(tp, gt, L);
    char *buf = nullptr;
    if ((rc = alloc_layout(&buf, L, st, who))) return rc;
    td.bind(tp, buf);
    bm.bind(buf);
    int32_t *d_cols = (int32_t *)(buf + o_cols);
    int *d_flag = (int *)(buf + o_flag);
    double *PR = p_raw ? p_raw : (double *)(buf + o_pr), *PA = p_adj ? p_adj : (double *)(buf + o_pa);
    double *Z = (double *)(buf + o_z);
    cudaEvent_t ev[6] = {};
    for (auto &e : ev) ICNV_CUDA(cudaEventCreate(&e));
    auto body = [&]() -> int {
        int rc2;
        ICNV_CUDA(cudaMemcpyAsync(d_cols, cols.data(), sizeof(int32_t) * (size_t)T, cudaMemcpyHostToDevice, st));
        if ((rc2 = td.upload(tp, st)) || (rc2 = bm.upload(mp, st))) return rc2;
        ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
        double t[5] = {0, 0, 0, 0, 0};
        for (int64_t g0 = 0; g0 < G; g0 += gt) {
            const int64_t n = std::min<int64_t>(gt, G - g0);
            ICNV_CUDA(cudaEventRecord(ev[0], st));
            gather_kernel<<<dim3((unsigned)((T + 31) / 32), (unsigned)((n + 31) / 32)), NT, 0, st>>>(X, ldx, d_cols, T, g0, n, Z, d_flag);
            ICNV_CHECK_LAUNCH("gather_kernel");
            ICNV_CUDA(cudaEventRecord(ev[1], st));
            if ((rc2 = td.launch(tp, Z, g0, n, PR + g0, G, jitter_mean, jitter_sd, seed, c.sm_count, st, ev[2]))) return rc2;
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
        if ((rc2 = bm.bh(PR, G, npair, p_thresh, PA, st))) return rc2;
        ICNV_CUDA(cudaEventRecord(ev[4], st));
        if ((rc2 = bm.mask(X, ldx, Y, ldy, G, C, n_ref, rule, mask_val, st))) return rc2;
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
    rc = body();
    cudaFreeAsync(buf, st);
    for (auto &e : ev)
        if (e) cudaEventDestroy(e);
    return rc;
}

void de_mask_stats(double *out7) {
    for (int i = 0; i < 7; ++i) out7[i] = g_de_stats[i];
}
void de_mask_set_stats(const double *in7) {
    for (int i = 0; i < 7; ++i) g_de_stats[i] = in7[i];
}

// ---- the stages on their own, for callers that split the genes over devices or ranks ----------------------------------

// Stage (a) for an exchange: per destination d, the gene-major block (gene_hi[d] - gene_lo[d] genes x m listed cells) of
// X's columns d_cols, blocks back to back in destination order - the same 32 x 32 transpose as the gather.
int de_pack_dev(const double *X, int64_t ldx, const int32_t *d_cols, int64_t m, int n_dst, const int64_t *gene_lo,
                const int64_t *gene_hi, double *out, int *flag, void *stream, const char *who) {
    ICNV_REQUIRE_READY();
    if (m < 0 || n_dst < 1 || !gene_lo || !gene_hi) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    int64_t total = 0;
    for (int d = 0; d < n_dst; ++d) {
        if (gene_lo[d] < 0 || gene_hi[d] < gene_lo[d] || gene_hi[d] > ldx)
            return set_error(ICNV_E_BAD_ARG, "%s: gene range %d is [%lld, %lld)", who, d, (long long)gene_lo[d], (long long)gene_hi[d]);
        total += gene_hi[d] - gene_lo[d];
    }
    if (m == 0 || total == 0) return ICNV_OK;
    if (!X || !d_cols || !out || !flag) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    cudaStream_t st = pick_stream(stream);
    double *o = out;
    for (int d = 0; d < n_dst; ++d) {
        const int64_t n = gene_hi[d] - gene_lo[d];
        if (n == 0) continue;
        gather_kernel<<<dim3((unsigned)((m + 31) / 32), (unsigned)((n + 31) / 32)), NT, 0, st>>>(X, ldx, d_cols, m, gene_lo[d], n,
                                                                                                o, flag);
        ICNV_CHECK_LAUNCH("gather_kernel");
        o += n * m;
    }
    return ICNV_OK;
}

// The receiving side: R holds one block (n genes x src_m[q] cells) per source q, back to back in source order; d_tags the
// global list positions of the received entries in the same order.  Fills the n x T slab rows Z.
int de_place_dev(const double *R, int64_t n, int n_src, const int64_t *src_m, const int32_t *d_tags, int64_t T, double *Z,
                 void *stream, const char *who) {
    ICNV_REQUIRE_READY();
    if (n < 0 || n_src < 1 || !src_m || T < 0) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    int64_t tot = 0;
    for (int q = 0; q < n_src; ++q) {
        if (src_m[q] < 0) return set_error(ICNV_E_BAD_ARG, "%s: source %d sends %lld cells", who, q, (long long)src_m[q]);
        tot += src_m[q];
    }
    if (tot != T) return set_error(ICNV_E_BAD_ARG, "%s: the sources send %lld cells, the rows hold %lld", who, (long long)tot, (long long)T);
    if (n == 0 || T == 0) return ICNV_OK;
    if (!R || !d_tags || !Z) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    Ctx &c = ctx();
    cudaStream_t st = pick_stream(stream);
    int64_t e0 = 0;
    for (int q = 0; q < n_src; ++q) {
        const int64_t m = src_m[q];
        if (m > 0) {
            const unsigned gb = (unsigned)std::min<int64_t>((n * m + NT - 1) / NT, (int64_t)c.sm_count * 16);
            place_kernel<<<gb, NT, 0, st>>>(R + n * e0, n, m, d_tags + e0, T, Z);
            ICNV_CHECK_LAUNCH("place_kernel");
        }
        e0 += m;
    }
    return ICNV_OK;
}

// Stages (b) and (c) on the slab rows Z (n genes x T listed cells, gene-major, global list order) of absolute genes g0 ..:
// p into p_raw[pair ldp + gl].  The per-gene scratch is tiled from free memory.  `times`, when given, gets the device ms of
// (b) and (c) added.
int de_slab_tests_dev(const double *Z, int64_t T, int64_t g0, int64_t n, const int32_t *ref_off, int n_ref,
                      const int32_t *sub_off, int n_sub, int test, double jitter_mean, double jitter_sd,
                      unsigned long long seed, double *p_raw, int64_t ldp, void *stream, double *times, const char *who) {
    ICNV_REQUIRE_READY();
    if (n < 0 || g0 < 0 || T < 1) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    int rc = check_jitter(jitter_mean, jitter_sd, 0.0, who);
    if (rc) return rc;
    TestPlan tp;
    if ((rc = make_test_plan(ref_off, n_ref, sub_off, n_sub, test, tp, who))) return rc;
    if (tp.T != T) return set_error(ICNV_E_BAD_ARG, "%s: the groups list %lld cells, the rows hold %lld", who, (long long)tp.T, (long long)T);
    if (n == 0 || n_sub == 0) return ICNV_OK;   // no pair: nothing to write
    if (!Z || !p_raw || ldp < n) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    Ctx &c = ctx();
    cudaStream_t st = pick_stream(stream);
    Layout L;
    TestDev td;
    td.fixed(tp, c.sm_count, L);
    const size_t per_gene = TestDev::per_gene(tp), usable = usable_device_bytes();
    if (usable < L.bytes + per_gene + 4096) return set_error(ICNV_E_NOMEM, "%s: not even one gene fits in device memory", who);
    const int64_t gt = std::min<int64_t>(n, (int64_t)((usable - L.bytes - 4096) / per_gene));
    td.tiles(tp, gt, L);
    char *buf = nullptr;
    if ((rc = alloc_layout(&buf, L, st, who))) return rc;
    td.bind(tp, buf);
    cudaEvent_t ev[3] = {};
    for (auto &e : ev) ICNV_CUDA(cudaEventCreate(&e));
    auto body = [&]() -> int {
        int rc2;
        if ((rc2 = td.upload(tp, st))) return rc2;
        for (int64_t a = 0; a < n; a += gt) {
            const int64_t nn = std::min<int64_t>(gt, n - a);
            ICNV_CUDA(cudaEventRecord(ev[0], st));
            if ((rc2 = td.launch(tp, Z + a * T, g0 + a, nn, p_raw + a, ldp, jitter_mean, jitter_sd, seed, c.sm_count, st, ev[1])))
                return rc2;
            ICNV_CUDA(cudaEventRecord(ev[2], st));
            ICNV_CUDA(cudaStreamSynchronize(st));
            float ms = 0.0f;
            for (int s = 0; s < 2 && times; ++s) {
                ICNV_CUDA(cudaEventElapsedTime(&ms, ev[s], ev[s + 1]));
                times[s] += ms;
            }
        }
        return ICNV_OK;
    };
    rc = body();
    cudaFreeAsync(buf, st);
    for (auto &e : ev)
        if (e) cudaEventDestroy(e);
    return rc;
}

// Stages (d) and (e): BH of the whole p_raw (G x n_pairs, pair rows of G), then the mask of a block of C columns of X
// (nullable Y: BH only).  ref_idx: the block's reference cells; sub_off / sub_idx: per subcluster the block's cells of it
// (possibly none), sub_size its whole list length.  `times`, when given, gets the device ms of (d) and (e).
int de_bh_mask_dev(const double *p_raw, int64_t G, int n_ref, int n_sub, const int32_t *sub_size, double p_thresh,
                   double *p_adj, const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t C, const int32_t *ref_idx,
                   int64_t n_ref_cells, const int32_t *sub_off, const int32_t *sub_idx, int rule, double mask_val,
                   void *stream, double *times, const char *who) {
    ICNV_REQUIRE_READY();
    const int64_t npair = (int64_t)std::max(n_sub, 0) * n_ref;
    if (G < 1 || n_ref < 1 || n_sub < 0 || C < 0 || n_ref_cells < 0 || (npair > 0 && (!p_raw || !sub_size)) ||
        (n_ref_cells > 0 && !ref_idx) || (n_sub > 0 && (!sub_off || !sub_idx)) ||
        (Y && C > 0 && (!X || ldx < G || ldy < G)))
        return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    if (rule < 0 || rule > 2) return set_error(ICNV_E_BAD_ARG, "%s: unknown rule code %d", who, rule);
    if (std::isnan(p_thresh)) return set_error(ICNV_E_BAD_ARG, "%s: bad threshold", who);
    for (int s = 0; s < n_sub; ++s) {
        if (sub_size[s] < 1) return set_error(ICNV_E_BAD_ARG, "%s: subcluster %d is empty", who, s);
        if (sub_off[s + 1] < sub_off[s]) return set_error(ICNV_E_BAD_ARG, "%s: offsets of subcluster %d decrease", who, s);
    }
    if (n_sub > 0 && sub_off[0] != 0) return set_error(ICNV_E_BAD_ARG, "%s: offsets must start at 0", who);
    MaskPlan mp;
    int rc = make_mask_plan(Y ? C : 0, ref_idx, Y ? n_ref_cells : 0, sub_off, sub_idx, Y ? n_sub : 0, sub_size, mp, who);
    if (rc) return rc;
    Ctx &c = ctx();
    cudaStream_t st = pick_stream(stream);
    Layout L;
    BhMaskDev bm;
    const size_t o_pa = p_adj ? 0 : L.take(sizeof(double) * (size_t)(G * std::max<int64_t>(npair, 1)));
    bm.fixed(G, npair, mp, c.sm_count, L);
    char *buf = nullptr;
    if ((rc = alloc_layout(&buf, L, st, who))) return rc;
    bm.bind(buf);
    double *PA = p_adj ? p_adj : (double *)(buf + o_pa);
    cudaEvent_t ev[3] = {};
    for (auto &e : ev) ICNV_CUDA(cudaEventCreate(&e));
    auto body = [&]() -> int {
        int rc2;
        if ((rc2 = bm.upload(mp, st))) return rc2;
        ICNV_CUDA(cudaEventRecord(ev[0], st));
        if ((rc2 = bm.bh(p_raw, G, npair, p_thresh, PA, st))) return rc2;
        ICNV_CUDA(cudaEventRecord(ev[1], st));
        if ((rc2 = bm.mask(X, ldx, Y, ldy, G, C, n_ref, rule, mask_val, st))) return rc2;
        ICNV_CUDA(cudaEventRecord(ev[2], st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        float ms = 0.0f;
        for (int s = 0; s < 2 && times; ++s) {
            ICNV_CUDA(cudaEventElapsedTime(&ms, ev[s], ev[s + 1]));
            times[s] += ms;
        }
        return ICNV_OK;
    };
    rc = body();
    cudaFreeAsync(buf, st);
    for (auto &e : ev)
        if (e) cudaEventDestroy(e);
    return rc;
}

}  // namespace icnv
