// Shared-nearest-neighbour graph of Leiden subclustering, run() step 15 with leiden_method = "PCA" - K18 in DESIGN
// section 3.  .leiden_seurat_preprocess_routine (R/inferCNV_tumor_subclusters.R:699-723) runs Seurat 5's
// FindVariableFeatures (vst) -> ScaleData -> RunPCA(npcs) -> FindNeighbors(k.param) on one group matrix; this file computes
// what those calls define, on the device, in one call:
//
//   1. gene statistics      mu_g, v_g (denominator n - 1) over the n listed cells (gene_stats_kernel, one pass);
//   2. vst trend            direct local quadratic loess of log10 v on log10 mu over the m non-constant genes, span 0.3:
//                           the q = floor(0.3 m) nearest x (a contiguous window of the sorted x), tricube weights on
//                           d / rho with rho the q-th smallest distance (trend_kernel, one warp per gene);
//   3. standardised var.    sum_c min((x - mu) / s, sqrt(n))^2 / (n - 1), s = sqrt(10^yhat) (stdvar_kernel, second pass);
//                           ranked decreasing, ties by gene index (rank_kernel): the first min(n_features, G) genes;
//   4. scaling              z = min((x - mu) / sqrt(v), 10), formed on the fly wherever a tile of Z is staged; constant
//                           genes are dropped (F genes remain);
//   5. PCA                  C = Z Z^T (gram_kernel: FP64 DMMA, upper-triangle 64 x 64 tiles, no atomics), its top npcs
//                           eigenpairs by block subspace iteration with Rayleigh-Ritz (snn_mul_kernel and the eig_*
//                           kernels; stop when every ||C v_j - l_j v_j|| <= 1e-12 l_1), signs so that the largest |entry| of each
//                           vector is positive (ties: the lower variable-feature rank), E = Z^T V (embed_kernel);
//   6. SNN                  K12's exact kNN on E (knn_launch), reverse lists by a counting sort, per row the shared counts
//                           s over the union of its neighbours' reverse lists, w = s / (k + (k - s)), dropped when
//                           w < 1/15; a count pass and a fill pass into CSR (snn_rows_kernel; rows whose candidate list
//                           does not fit shared memory - hubs - go to snn_spill_kernel's global counters).
//
// Every reduction has a fixed order and the only atomics are integer ones whose results do not depend on their order, so two
// calls on the same input return the same bits.  The result stays in the library until the next call
// (icnv_seurat_snn_fetch copies it out).
#include "icnv_common.cuh"

#include <algorithm>
#include <cmath>
#include <numeric>
#include <vector>

namespace icnv {

// K12 (icnv_dist.cu)
int knn_launch(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n, int k, int32_t *idx, double *dist,
               int rows, void *stream, const char *who);

namespace snn {

constexpr double SN_SPAN = 0.3;           // FindVariableFeatures(loess.span)
constexpr double SN_SCALE_MAX = 10.0;     // ScaleData(scale.max)
constexpr double SN_PRUNE = 1.0 / 15.0;   // FindNeighbors(prune.SNN)
constexpr int SN_NPCS_MAX = 16;           // embedding accumulators per lane
constexpr int SN_B = 32;                  // widest subspace block
constexpr int SN_CHECK = 8;               // subspace iterations between Rayleigh-Ritz checks
constexpr int SN_ITER_MAX = 4096;
constexpr int SN_BATCH = 32;              // iterations enqueued between reads of the done flag
constexpr int ST_GENES = 32, ST_WARPS = 8;
constexpr int GT = 64, GKC = 16, GLD = GT + 8;   // Gram tile, cells per staged chunk, staged row stride
constexpr int SN_CAP = 4096;              // candidate slots per warp of snn_rows_kernel
constexpr int SN_ROW_WARPS = 4;
constexpr int SN_SPILL_CTAS = 128;

// state of the subspace iteration (device)
struct EigState {
    int iter, done, status;   // status: 0 converged / running, 1 the block collapsed (Cholesky breakdown)
    int pad;
    double max_res;           // largest ||C v_j - l_j v_j|| / l_1 at the last check
    double theta[SN_B];       // Ritz values, decreasing
    int perm[SN_B];           // column of W holding the j-th Ritz vector
    double W[SN_B][SN_B + 1]; // eigenvectors of H = Q^T C Q (columns)
    double R[SN_B][SN_B + 1]; // Cholesky factor of the column-scaled Y^T Y
    double dsc[SN_B];         // the column scaling
};

// ---- 1 and 3: gene passes --------------------------------------------------------------------------------------------

// mu[g], var[g] over the listed cells (shifted by the first value: a constant gene gets exactly 0); flag |= 1 on a
// non-finite value; n_var counts the genes with var > 0, flag |= 4 when one of them has mu <= 0 (log10 mu undefined).
__global__ void __launch_bounds__(ST_GENES *ST_WARPS) gene_stats_kernel(const double *__restrict__ X, int64_t G, int64_t ldx,
                                                                        const int32_t *__restrict__ cells, int64_t n,
                                                                        double *mu, double *var, int *n_var, int *flag) {
    __shared__ double s1[ST_WARPS][ST_GENES], s2[ST_WARPS][ST_GENES];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t g = (int64_t)blockIdx.x * ST_GENES + lane;
    double a = 0.0, b = 0.0, x0 = 0.0;
    bool bad = false;
    if (g < G) {
        x0 = X[g + ldx * (int64_t)(cells ? cells[0] : 0)];
        for (int64_t i = w; i < n; i += ST_WARPS) {
            const double x = X[g + ldx * (int64_t)(cells ? cells[i] : i)];
            bad |= !is_finite_d(x);
            const double d = x - x0;
            a += d;
            b = fma(d, d, b);
        }
    }
    s1[w][lane] = a;
    s2[w][lane] = b;
    __syncthreads();
    if (w == 0 && g < G) {
        a = s1[0][lane];
        b = s2[0][lane];
        for (int k = 1; k < ST_WARPS; ++k) {
            a += s1[k][lane];
            b += s2[k][lane];
        }
        const double m = x0 + a / (double)n;
        const double v = fmax((b - a * (a / (double)n)) / (double)(n - 1), 0.0);
        mu[g] = m;
        var[g] = v;
        if (v > 0.0) {
            atomicAdd(n_var, 1);
            if (!(m > 0.0)) atomicOr(flag, 4);
        }
    }
    if (bad) atomicOr(flag, 1);
}

// sv[g] = sum over the cells of min((x - mu) / s, vmax = sqrt(n))^2 / (n - 1), 0 where s = 0
__global__ void __launch_bounds__(ST_GENES *ST_WARPS, 1) stdvar_kernel(const double *__restrict__ X, int64_t G, int64_t ldx,
                                                                    const int32_t *__restrict__ cells, int64_t n,
                                                                    const double *__restrict__ mu,
                                                                    const double *__restrict__ sexp, double vmax, double *sv) {
    __shared__ double s1[ST_WARPS][ST_GENES];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t g = (int64_t)blockIdx.x * ST_GENES + lane;
    double a = 0.0;
    if (g < G && sexp[g] > 0.0) {
        const double m = mu[g], s = sexp[g];
        const double *xg = X + g;
        for (int64_t i = w; i < n; i += ST_WARPS) {
            const double z = fmin(__ddiv_rn(xg[ldx * (int64_t)(cells ? cells[i] : i)] - m, s), vmax);
            a = fma(z, z, a);
        }
    }
    s1[w][lane] = a;
    __syncthreads();
    if (w == 0 && g < G) {
        a = s1[0][lane];
        for (int k = 1; k < ST_WARPS; ++k) a += s1[k][lane];
        sv[g] = a / (double)(n - 1);
    }
}

// ---- 2: the vst trend --------------------------------------------------------------------------------------------------

// key[g] = log10 mu (ascending sort of the non-constant genes; constant genes get +inf and sort last)
__global__ void trend_keys_kernel(const double *mu, const double *var, int64_t G, double *key) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g < G) key[g] = var[g] > 0.0 ? log10(mu[g]) : __longlong_as_double(0x7ff0000000000000ll);
}

// pos[i] = the place of key i in the stable order: ascending (desc = 0) or decreasing (desc = 1), ties by index
__global__ void __launch_bounds__(256) rank_kernel(const double *__restrict__ key, int64_t m, int desc, int32_t *pos) {
    __shared__ double tile[256];
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const double ki = i < m ? key[i] : 0.0;
    int64_t r = 0;
    for (int64_t t0 = 0; t0 < m; t0 += 256) {
        __syncthreads();
        if (t0 + threadIdx.x < m) tile[threadIdx.x] = key[t0 + threadIdx.x];
        __syncthreads();
        const int lim = (int)min((int64_t)256, m - t0);
        for (int t = 0; t < lim; ++t) {
            const double kj = tile[t];
            const int64_t j = t0 + t;
            r += desc ? (kj > ki || (kj == ki && j < i)) : (kj < ki || (kj == ki && j < i));
        }
    }
    if (i < m) pos[i] = (int32_t)r;
}

__global__ void scatter_sorted_kernel(const int32_t *pos, const double *mu, const double *var, int64_t G, double *xs,
                                      double *ys, int32_t *gene_at) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const int32_t p = pos[g];
    gene_at[p] = (int32_t)g;
    if (var[g] > 0.0) {
        xs[p] = log10(mu[g]);
        ys[p] = log10(var[g]);
    }
}

// One warp per non-constant gene (sorted position p): the q-point window around x_p with the smallest q-th distance rho,
// tricube weights on u = (x_j - x_p) / rho, the weighted normal equations of y ~ 1 + u + u^2 solved in FP64; yhat = the
// intercept.  A singular system (pivot <= 1e-12 of the first) or rho = 0 - where loess would warn - takes the weighted mean
// of the window and counts in n_sing.  sexp[gene] = sqrt(10^yhat); constant genes keep 0.
__global__ void __launch_bounds__(256) trend_kernel(const double *__restrict__ xs, const double *__restrict__ ys,
                                                    const int32_t *__restrict__ gene_at, int64_t m, int64_t q,
                                                    double *sexp, int *n_sing) {
    const int64_t p = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (p >= m) return;
    const int lane = threadIdx.x & 31;
    const double xp = xs[p];
    int64_t lo = max((int64_t)0, p - q + 1), hi = min(p, m - q);   // window starts [lo, hi]
    // the first start whose right distance reaches its left distance; rho is the smaller of it and its predecessor
    int64_t a = lo, b = hi;
    while (a < b) {
        const int64_t c = (a + b) >> 1;
        if (xs[c + q - 1] - xp >= xp - xs[c]) b = c; else a = c + 1;
    }
    double rho = fmax(xp - xs[a], xs[a + q - 1] - xp);
    if (a > lo) {
        const double r2 = fmax(xp - xs[a - 1], xs[a - 1 + q - 1] - xp);
        if (r2 < rho) {
            rho = r2;
            a = a - 1;
        }
    }
    double S[5] = {0, 0, 0, 0, 0}, T[3] = {0, 0, 0};
    for (int64_t j = a + lane; j < a + q; j += 32) {
        const double d = fabs(xs[j] - xp);
        double w;
        if (rho > 0.0) {
            const double u = d / rho;
            if (u >= 1.0) continue;
            const double t = 1.0 - u * u * u;
            w = t * t * t;
        } else {
            w = 1.0;
        }
        const double u = rho > 0.0 ? (xs[j] - xp) / rho : 0.0, y = ys[j];
        double up = w;
        for (int e = 0; e < 5; ++e) {
            S[e] += up;
            if (e < 3) T[e] += up * y;
            up *= u;
        }
    }
#pragma unroll
    for (int e = 0; e < 5; ++e) S[e] = warp_sum_d(S[e]);
#pragma unroll
    for (int e = 0; e < 3; ++e) T[e] = warp_sum_d(T[e]);
    if (lane) return;
    double yhat;
    bool sing = !(rho > 0.0);
    if (!sing) {   // LDL^T of [[S0 S1 S2] [S1 S2 S3] [S2 S3 S4]]
        const double d0 = S[0];
        const double l10 = S[1] / d0, l20 = S[2] / d0;
        const double d1 = S[2] - l10 * S[1];
        const double l21 = d1 > 0.0 ? (S[3] - l20 * S[1]) / d1 : 0.0;
        const double d2 = S[4] - l20 * S[2] - l21 * l21 * d1;
        sing = !(d1 > 1e-12 * d0) || !(d2 > 1e-12 * d0);
        if (!sing) {
            const double z0 = T[0], z1 = T[1] - l10 * z0, z2 = T[2] - l20 * z0 - l21 * z1;
            const double c2 = z2 / d2, c1 = z1 / d1 - l21 * c2, c0 = z0 / d0 - l10 * c1 - l20 * c2;
            yhat = c0;
        }
    }
    if (sing) {
        yhat = T[0] / S[0];
        atomicAdd(n_sing, 1);
    }
    sexp[gene_at[p]] = sqrt(pow(10.0, yhat));
}

// ---- 5: the Gram matrix (FP64 tensor cores) --------------------------------------------------------------------------

// D(16 x 8) += A(16 x 4, row) B(4 x 8, col), PTX fragment layout with g = lane / 4, t = lane % 4:
// a0 = A[g][t], a1 = A[g + 8][t]; b = B[t][g]; d[i] = D[g + 8 (i / 2)][2 t + i % 2].
__device__ __forceinline__ void dmma_16x8x4(double *d, double a0, double a1, double b) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                 : "d"(a0), "d"(a1), "d"(b));
}

struct GramParams {
    const double *X;
    int64_t ldx;
    const int32_t *cells;   // NULL: column a is cell a
    int64_t n;
    const int32_t *feat;    // F genes, ascending
    const double *mu, *sd;  // per feature
    int F;
    const int2 *tiles;      // (bi, bj), bi <= bj
    double *C;              // F x F, ld F, both triangles written
};

// One CTA per upper-triangle tile pair: the 64 x 64 block C[bi, bj] over all n cells, 16 cells per staged chunk (z formed
// while staging, the next chunk's loads in flight during this chunk's DMMA); warp w owns rows 16 (w % 4) .. +16 and columns
// 32 (w / 4) .. +32 of the tile.  Chunks and k-steps run in ascending cell order.
__global__ void __launch_bounds__(256, 1) gram_kernel(const GramParams p) {
    __shared__ __align__(16) double As[GKC][GLD], Bs[GKC][GLD];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, g = lane >> 2, t = lane & 3;
    const int2 tl = p.tiles[blockIdx.x];
    const bool diag = tl.x == tl.y;
    const int fl = tid & (GT - 1), cl = tid >> 6;   // staging: feature within the tile, first cell of the chunk (+4 i)
    const int fa = tl.x * GT + fl, fb = tl.y * GT + fl;
    const bool va = fa < p.F, vb = fb < p.F;
    const int64_t ga = va ? p.feat[fa] : 0, gb = vb ? p.feat[fb] : 0;
    const double ma = va ? p.mu[fa] : 0.0, sa = va ? p.sd[fa] : 1.0, mb = vb ? p.mu[fb] : 0.0, sb = vb ? p.sd[fb] : 1.0;
    double ra[4], rb[4];
    auto load = [&](int64_t c0) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t c = c0 + cl + 4 * i;
            ra[i] = rb[i] = 0.0;
            if (c < p.n) {
                const int64_t col = p.ldx * (int64_t)(p.cells ? p.cells[c] : c);
                if (va) ra[i] = fmin(__ddiv_rn(p.X[ga + col] - ma, sa), SN_SCALE_MAX);
                if (vb && !diag) rb[i] = fmin(__ddiv_rn(p.X[gb + col] - mb, sb), SN_SCALE_MAX);
            }
        }
    };
    double acc[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[j][i] = 0.0;
    const double(*Bp)[GLD] = diag ? As : Bs;
    const int r0 = (w & 3) * 16, c0w = (w >> 2) * 32;
    load(0);
    for (int64_t c0 = 0; c0 < p.n; c0 += GKC) {
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            As[cl + 4 * i][fl] = ra[i];
            Bs[cl + 4 * i][fl] = rb[i];
        }
        __syncthreads();
        if (c0 + GKC < p.n) load(c0 + GKC);
#pragma unroll
        for (int kk = 0; kk < GKC / 4; ++kk) {
            const double a0 = As[4 * kk + t][r0 + g], a1 = As[4 * kk + t][r0 + g + 8];
#pragma unroll
            for (int j = 0; j < 4; ++j) dmma_16x8x4(acc[j], a0, a1, Bp[4 * kk + t][c0w + 8 * j + g]);
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t r = (int64_t)tl.x * GT + r0 + g + 8 * (i >> 1), c = (int64_t)tl.y * GT + c0w + 8 * j + 2 * t + (i & 1);
            if (r < p.F && c < p.F) {
                p.C[r + p.F * c] = acc[j][i];
                if (!diag) p.C[c + p.F * r] = acc[j][i];
            }
        }
}

// ---- 5: eigenpairs -----------------------------------------------------------------------------------------------------

// Y = C Q (F x SN_B, row-major; the columns >= b of Q are 0).  16 rows per CTA, h in chunks of 64, ascending.
__global__ void __launch_bounds__(256) snn_mul_kernel(const double *__restrict__ C, int F, const double *__restrict__ Q,
                                                      double *Y, const EigState *s) {
    if (s->done) return;
    __shared__ double Cs[16][65], Qs[64][SN_B];
    const int tid = threadIdx.x, r = tid >> 4, jc = tid & 15;
    const int64_t f0 = (int64_t)blockIdx.x * 16;
    double y0 = 0.0, y1 = 0.0;
    for (int h0 = 0; h0 < F; h0 += 64) {
        __syncthreads();
        for (int e = tid; e < 16 * 64; e += 256) {
            const int rr = e >> 6, hh = e & 63;
            Cs[rr][hh] = (f0 + rr < F && h0 + hh < F) ? C[(h0 + hh) + (int64_t)F * (f0 + rr)] : 0.0;
        }
        for (int e = tid; e < 64 * SN_B; e += 256) {
            const int hh = e / SN_B, j = e % SN_B;
            Qs[hh][j] = h0 + hh < F ? Q[(int64_t)(h0 + hh) * SN_B + j] : 0.0;
        }
        __syncthreads();
#pragma unroll 8
        for (int hh = 0; hh < 64; ++hh) {
            y0 = fma(Cs[r][hh], Qs[hh][jc], y0);
            y1 = fma(Cs[r][hh], Qs[hh][jc + 16], y1);
        }
    }
    if (f0 + r < F) {
        Y[(f0 + r) * SN_B + jc] = y0;
        Y[(f0 + r) * SN_B + jc + 16] = y1;
    }
}

// Every iteration: Y = C Q (snn_mul_kernel), the partial Gram matrices of Y over row blocks (eig_gram_kernel; Q^T Y too at a
// check), their fixed-order sums, the Cholesky factor of the column-scaled Y^T Y and, at a check, the eigenpairs of
// H = Q^T Y (eig_small_kernel), then Q = Y D R^-1 row by row (eig_apply_kernel).  At a check (every SN_CHECK-th iteration)
// eig_resid_kernel forms the Ritz vectors V = Q W[:, :npcs] and their residuals ||Y w_j - l_j Q w_j|| per row block, and
// eig_decide_kernel adds them in block order and stops the iteration when every one is <= 1e-12 l_1.
constexpr int EG_ROWS = 64;   // rows per partial block of eig_gram_kernel and eig_resid_kernel

__global__ void __launch_bounds__(1024) eig_gram_kernel(const double *__restrict__ Q, const double *__restrict__ Y, int F,
                                                        int check, double *part, const EigState *s) {
    if (s->done) return;
    __shared__ double Ys[EG_ROWS][SN_B], Qs[EG_ROWS][SN_B];
    const int i = threadIdx.x >> 5, j = threadIdx.x & 31;
    const int64_t f0 = (int64_t)blockIdx.x * EG_ROWS;
    const int rows = (int)min((int64_t)EG_ROWS, F - f0);
    for (int e = threadIdx.x; e < rows * SN_B; e += 1024) {
        Ys[e / SN_B][e % SN_B] = Y[f0 * SN_B + e];
        if (check) Qs[e / SN_B][e % SN_B] = Q[f0 * SN_B + e];
    }
    __syncthreads();
    double g = 0.0, h = 0.0;
    for (int r = 0; r < rows; ++r) {
        g = fma(Ys[r][i], Ys[r][j], g);
        if (check) h = fma(Qs[r][i], Ys[r][j], h);
    }
    double *out = part + (int64_t)blockIdx.x * 2 * SN_B * SN_B;
    out[i * SN_B + j] = g;
    if (check) out[SN_B * SN_B + i * SN_B + j] = h;
}

constexpr int EG_SMALL_NT = 256;

// Jacobi on the b x b symmetric A by the whole CTA, in round-robin order: each step rotates b/2 disjoint (p, q) planes at
// once (the circle method over m = b rounded up to even; pairs with the dummy index b are skipped); V accumulates the
// rotations.  Sweeps stop when the off-diagonal norm is within 1e-15 of the diagonal's.
__device__ void jacobi_block(double (*A)[SN_B + 1], double (*V)[SN_B + 1], int b) {
    __shared__ int P[SN_B / 2], Qx[SN_B / 2];
    __shared__ double Cs[SN_B / 2], Ss[SN_B / 2];
    __shared__ int go;
    const int tid = threadIdx.x, m = (b + 1) & ~1, np = m / 2;
    for (int e = tid; e < SN_B * SN_B; e += EG_SMALL_NT) V[e / SN_B][e % SN_B] = (e / SN_B == e % SN_B) ? 1.0 : 0.0;
    __syncthreads();
    for (int sweep = 0; sweep < 30; ++sweep) {
        if (tid == 0) {
            double off = 0.0, dia = 0.0;
            for (int p = 0; p < b; ++p) {
                dia += A[p][p] * A[p][p];
                for (int q = p + 1; q < b; ++q) off += A[p][q] * A[p][q];
            }
            go = off > 1e-30 * dia;
        }
        __syncthreads();
        if (!go) break;
        for (int r = 0; r < m - 1; ++r) {
            if (tid < np) {
                int p = tid == 0 ? m - 1 : (r + tid) % (m - 1), q = tid == 0 ? r : (r - tid + m - 1) % (m - 1);
                if (p > q) {
                    const int t = p;
                    p = q;
                    q = t;
                }
                double c = 1.0, sn = 0.0;
                if (q < b) {
                    const double apq = A[p][q];
                    if (fabs(apq) > 1e-18 * sqrt(fabs(A[p][p] * A[q][q]))) {
                        const double th = (A[q][q] - A[p][p]) / (2.0 * apq);
                        const double tt = (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
                        c = 1.0 / sqrt(tt * tt + 1.0);
                        sn = tt * c;
                    }
                }
                P[tid] = p;
                Qx[tid] = q < b ? q : p;   // a pair with the dummy rotates nothing
                Cs[tid] = c;
                Ss[tid] = q < b ? sn : 0.0;
            }
            __syncthreads();
            for (int e = tid; e < np * b; e += EG_SMALL_NT) {   // columns: A J
                const int k = e / b, l = e % b, p = P[k], q = Qx[k];
                if (p == q) continue;
                const double akp = A[l][p], akq = A[l][q];
                A[l][p] = Cs[k] * akp - Ss[k] * akq;
                A[l][q] = Ss[k] * akp + Cs[k] * akq;
            }
            __syncthreads();
            for (int e = tid; e < np * b; e += EG_SMALL_NT) {   // rows: J^T (A J); and V J
                const int k = e / b, l = e % b, p = P[k], q = Qx[k];
                if (p == q) continue;
                const double apk = A[p][l], aqk = A[q][l];
                A[p][l] = Cs[k] * apk - Ss[k] * aqk;
                A[q][l] = Ss[k] * apk + Cs[k] * aqk;
                const double vkp = V[l][p], vkq = V[l][q];
                V[l][p] = Cs[k] * vkp - Ss[k] * vkq;
                V[l][q] = Ss[k] * vkp + Cs[k] * vkq;
            }
            __syncthreads();
        }
    }
}

// One CTA: the partial sums added in block order; warp 0 factors the column-scaled Y^T Y (upper R, G = R^T R); then, at a
// check, the whole CTA diagonalises the symmetrised H and thread 0 orders its eigenpairs by decreasing value, ties by index.
__global__ void __launch_bounds__(EG_SMALL_NT) eig_small_kernel(const double *__restrict__ part, int n_part, int b, int check,
                                                                EigState *s) {
    if (s->done) return;
    __shared__ double Gs[SN_B][SN_B + 1], Hs[SN_B][SN_B + 1], Ws[SN_B][SN_B + 1], dsc[SN_B];
    for (int e = threadIdx.x; e < SN_B * SN_B; e += EG_SMALL_NT) {
        double g = 0.0, h = 0.0;
        for (int p = 0; p < n_part; ++p) {
            g += part[(int64_t)p * 2 * SN_B * SN_B + e];
            if (check) h += part[(int64_t)p * 2 * SN_B * SN_B + SN_B * SN_B + e];
        }
        Gs[e / SN_B][e % SN_B] = g;
        Hs[e / SN_B][e % SN_B] = h;
    }
    __syncthreads();
    const int l = threadIdx.x & 31;
    if (threadIdx.x < 32) {   // Cholesky
        dsc[l] = l < b && Gs[l][l] > 0.0 ? 1.0 / sqrt(Gs[l][l]) : 0.0;
        __syncwarp();
        for (int i = 0; i < SN_B; ++i) Gs[i][l] *= dsc[i] * dsc[l];
        __syncwarp();
        bool bad = false;
        for (int kc = 0; kc < b; ++kc) {
            const double d = Gs[kc][kc];
            bad |= !(d > 1e-24);
            const double r = sqrt(fmax(d, 1e-300));
            __syncwarp();
            if (l == kc) Gs[kc][kc] = r;
            if (l > kc && l < b) Gs[kc][l] /= r;
            __syncwarp();
            if (l > kc && l < b)
                for (int i = kc + 1; i <= l; ++i) Gs[i][l] -= Gs[kc][i] * Gs[kc][l];
            __syncwarp();
        }
        for (int i = 0; i < SN_B; ++i) s->R[i][l] = Gs[i][l];
        s->dsc[l] = dsc[l];
        if (bad && l == 0) {
            s->status = 1;
            s->done = 1;
        }
    }
    if (!check) return;
    // Rayleigh-Ritz (Q^T C Q is symmetric up to rounding)
    for (int e = threadIdx.x; e < SN_B * SN_B; e += EG_SMALL_NT) Ws[e / SN_B][e % SN_B] = 0.5 * (Hs[e / SN_B][e % SN_B] + Hs[e % SN_B][e / SN_B]);
    __syncthreads();
    for (int e = threadIdx.x; e < SN_B * SN_B; e += EG_SMALL_NT) Hs[e / SN_B][e % SN_B] = Ws[e / SN_B][e % SN_B];
    __syncthreads();
    jacobi_block(Hs, Ws, b);
    if (threadIdx.x == 0) {
        int perm[SN_B];
        for (int i = 0; i < b; ++i) perm[i] = i;
        for (int i = 1; i < b; ++i) {
            const int v = perm[i];
            int j = i;
            while (j > 0 && Hs[perm[j - 1]][perm[j - 1]] < Hs[v][v]) {
                perm[j] = perm[j - 1];
                --j;
            }
            perm[j] = v;
        }
        for (int i = 0; i < SN_B; ++i) {
            s->perm[i] = i < b ? perm[i] : i;
            s->theta[i] = i < b ? Hs[perm[i]][perm[i]] : 0.0;
        }
    }
    for (int e = threadIdx.x; e < SN_B * SN_B; e += EG_SMALL_NT) s->W[e / SN_B][e % SN_B] = Ws[e / SN_B][e % SN_B];
}

// At a check: V[f][j] = sum_i Q[f][i] W[i][perm j] and this block's sum of (Y w - l_j Q w)^2 per component (rows in order)
__global__ void __launch_bounds__(256) eig_resid_kernel(const double *__restrict__ Q, const double *__restrict__ Y, int F,
                                                        int b, int npcs, double *V, double *rpart, const EigState *s) {
    if (s->done) return;
    __shared__ double Ws[SN_B][SN_NPCS_MAX], th[SN_NPCS_MAX], acc[EG_ROWS][SN_NPCS_MAX];
    for (int e = threadIdx.x; e < SN_B * SN_NPCS_MAX; e += 256) {
        const int i = e / SN_NPCS_MAX, j = e % SN_NPCS_MAX;
        Ws[i][j] = j < npcs ? s->W[i][s->perm[j]] : 0.0;
    }
    if (threadIdx.x < SN_NPCS_MAX) th[threadIdx.x] = s->theta[threadIdx.x];
    __syncthreads();
    const int64_t f0 = (int64_t)blockIdx.x * EG_ROWS;
    for (int e = threadIdx.x; e < EG_ROWS * SN_NPCS_MAX; e += 256) {
        const int r = e / SN_NPCS_MAX, j = e % SN_NPCS_MAX;
        const int64_t f = f0 + r;
        double c = 0.0;
        if (f < F && j < npcs) {
            double u = 0.0, cu = 0.0;
            for (int i = 0; i < b; ++i) {
                u = fma(Q[f * SN_B + i], Ws[i][j], u);
                cu = fma(Y[f * SN_B + i], Ws[i][j], cu);
            }
            V[f * npcs + j] = u;
            const double d = cu - th[j] * u;
            c = d * d;
        }
        acc[r][j] = c;
    }
    __syncthreads();
    if (threadIdx.x < SN_NPCS_MAX) {
        double t = 0.0;
        for (int r = 0; r < EG_ROWS; ++r) t += acc[r][threadIdx.x];
        rpart[(int64_t)blockIdx.x * SN_NPCS_MAX + threadIdx.x] = t;
    }
}

__global__ void eig_decide_kernel(const double *rpart, int n_part, int npcs, int it, EigState *s) {
    if (s->done || threadIdx.x) return;
    double rmax = 0.0;
    for (int j = 0; j < npcs; ++j) {
        double t = 0.0;
        for (int p = 0; p < n_part; ++p) t += rpart[(int64_t)p * SN_NPCS_MAX + j];
        rmax = fmax(rmax, sqrt(t));
    }
    rmax = s->theta[0] > 0.0 ? rmax / s->theta[0] : rmax;
    s->max_res = rmax;
    s->iter = it;
    if (rmax <= 1e-12 || it >= SN_ITER_MAX) s->done = 1;
}

// Q = Y D R^-1, one row per thread (32 rows per CTA, staged in shared memory)
__global__ void __launch_bounds__(32) eig_apply_kernel(const double *__restrict__ Y, double *Q, int F, int b, int it,
                                                       EigState *s) {
    if (s->done) return;
    __shared__ double Rs[SN_B][SN_B + 1], ds[SN_B], Ys[32][SN_B + 1];
    const int l = threadIdx.x;
    for (int i = 0; i < SN_B; ++i) Rs[i][l] = s->R[i][l];
    ds[l] = s->dsc[l];
    const int64_t f0 = (int64_t)blockIdx.x * 32;
    for (int r = 0; r < 32; ++r) Ys[r][l] = f0 + r < F ? Y[(f0 + r) * SN_B + l] : 0.0;
    __syncwarp();
    double *y = Ys[l];
    for (int j = 0; j < b; ++j) {
        double v = y[j] * ds[j];
        for (int i = 0; i < j; ++i) v -= y[i] * Rs[i][j];
        y[j] = v / Rs[j][j];
    }
    __syncwarp();
    for (int r = 0; r < 32; ++r)
        if (f0 + r < F) Q[(f0 + r) * SN_B + l] = Ys[r][l];
    if (blockIdx.x == 0 && l == 0) s->iter = it;
}

// deterministic start: hashed uniforms in [-0.5, 0.5) on the first b columns
__global__ void subspace_start_kernel(double *Q, int F, int b) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)F * SN_B) return;
    const int j = (int)(e % SN_B);
    Q[e] = j < b ? u01(hash3(0x5eed5eedull, (uint64_t)(e / SN_B), (uint64_t)j, 18)) - 0.5 : 0.0;
}

// column j of V: the entry of largest magnitude made positive (ties: the lower variable-feature rank, rank_of[f])
__global__ void __launch_bounds__(256) sign_kernel(double *V, int F, int npcs, const int32_t *rank_of) {
    __shared__ double sm[256];
    __shared__ int sr[256], sf[256];
    const int j = blockIdx.x;
    double best = -1.0;
    int br = 0x7fffffff, bf = 0;
    for (int f = threadIdx.x; f < F; f += 256) {
        const double a = fabs(V[(int64_t)f * npcs + j]);
        if (a > best || (a == best && rank_of[f] < br)) {
            best = a;
            br = rank_of[f];
            bf = f;
        }
    }
    sm[threadIdx.x] = best;
    sr[threadIdx.x] = br;
    sf[threadIdx.x] = bf;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            const double a = sm[threadIdx.x + o];
            const int r = sr[threadIdx.x + o];
            if (a > sm[threadIdx.x] || (a == sm[threadIdx.x] && r < sr[threadIdx.x])) {
                sm[threadIdx.x] = a;
                sr[threadIdx.x] = r;
                sf[threadIdx.x] = sf[threadIdx.x + o];
            }
        }
        __syncthreads();
    }
    const bool flip = V[(int64_t)sf[0] * npcs + j] < 0.0;
    __syncthreads();
    if (flip)
        for (int f = threadIdx.x; f < F; f += 256) V[(int64_t)f * npcs + j] = -V[(int64_t)f * npcs + j];
}

// E[j + npcs c] = sum_f z_fc V[f][j]: one warp per cell, lanes over the features, a fixed shuffle tree per component
__global__ void __launch_bounds__(256) embed_kernel(const GramParams p, const double *__restrict__ V, int npcs, double *E) {
    const int64_t c = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (c >= p.n) return;
    const int lane = threadIdx.x & 31;
    const int64_t col = p.ldx * (int64_t)(p.cells ? p.cells[c] : c);
    double acc[SN_NPCS_MAX];
#pragma unroll
    for (int j = 0; j < SN_NPCS_MAX; ++j) acc[j] = 0.0;
    for (int f = lane; f < p.F; f += 32) {
        const double z = fmin(__ddiv_rn(p.X[p.feat[f] + col] - p.mu[f], p.sd[f]), SN_SCALE_MAX);
#pragma unroll
        for (int j = 0; j < SN_NPCS_MAX; ++j)
            if (j < npcs) acc[j] = fma(z, V[(int64_t)f * npcs + j], acc[j]);
    }
#pragma unroll
    for (int j = 0; j < SN_NPCS_MAX; ++j)
        if (j < npcs) {
            const double v = warp_sum_d(acc[j]);
            if (lane == 0) E[j + (int64_t)npcs * c] = v;
        }
}

// ---- 6: the SNN graph --------------------------------------------------------------------------------------------------

__global__ void indegree_kernel(const int32_t *idx, int64_t nk, int32_t *deg) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nk; e += (int64_t)gridDim.x * blockDim.x)
        atomicAdd(&deg[idx[e]], 1);
}

// out[i] = sum of in[0 .. i) for i <= n (one CTA of 1024 threads)
__global__ void __launch_bounds__(1024) exclusive_scan_kernel(const int32_t *in, int64_t n, int64_t *out) {
    using U = int64_t;
    __shared__ U part[1024];
    const int64_t per = (n + 1023) / 1024, a = min(n, per * threadIdx.x), b = min(n, a + per);
    U s = 0;
    for (int64_t i = a; i < b; ++i) s += (U)in[i];
    part[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        U run = 0;
        for (int i = 0; i < 1024; ++i) {
            const U v = part[i];
            part[i] = run;
            run += v;
        }
        out[n] = run;
    }
    __syncthreads();
    U run = part[threadIdx.x];
    for (int64_t i = a; i < b; ++i) {
        const U v = (U)in[i];
        out[i] = run;
        run += v;
    }
}

__global__ void reverse_fill_kernel(const int32_t *idx, int64_t n, int k, const int64_t *roff, int32_t *cursor, int32_t *rev) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n * k; e += (int64_t)gridDim.x * blockDim.x) {
        const int32_t m = idx[e];
        rev[roff[m] + atomicAdd(&cursor[m], 1)] = (int32_t)(e % n);
    }
}

// cand[i] = sum over m in N(i) of |R(m)|
__global__ void candidates_kernel(const int32_t *idx, int64_t n, int k, const int64_t *roff, int64_t *cand) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int64_t s = 0;
    for (int r = 0; r < k; ++r) {
        const int32_t m = idx[i + n * r];
        s += roff[m + 1] - roff[m];
    }
    cand[i] = s;
}

__device__ __forceinline__ bool snn_keep(int s, int k) { return !((double)s / (double)(k + (k - s)) < SN_PRUNE); }

struct SnnParams {
    const int32_t *idx;
    int64_t n;
    int k;
    const int64_t *roff;
    const int32_t *rev;
    const int64_t *cand;
    int32_t *row_nnz;         // count pass
    const int64_t *row_ptr;   // fill pass (NULL: count pass)
    int32_t *col;
    double *w;
};

// One warp per row whose candidates fit SN_CAP: gather, bitonic sort, runs -> shared counts -> Jaccard, prune; count or fill.
__global__ void __launch_bounds__(32 * SN_ROW_WARPS) snn_rows_kernel(const SnnParams p) {
    extern __shared__ int32_t snn_smem[];
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    const int64_t i = (int64_t)blockIdx.x * SN_ROW_WARPS + wl;
    if (i >= p.n || p.cand[i] > SN_CAP) return;
    int32_t *buf = snn_smem + wl * SN_CAP;
    const int T = (int)p.cand[i];
    int base = 0;
    for (int r = 0; r < p.k; ++r) {
        const int32_t m = p.idx[i + p.n * r];
        const int64_t o = p.roff[m];
        const int d = (int)(p.roff[m + 1] - o);
        for (int t = lane; t < d; t += 32) buf[base + t] = p.rev[o + t];
        base += d;
    }
    int P = 1;
    while (P < T) P <<= 1;
    for (int t = T + lane; t < P; t += 32) buf[t] = 0x7fffffff;
    __syncwarp();
    for (int kk = 2; kk <= P; kk <<= 1)
        for (int j = kk >> 1; j > 0; j >>= 1) {
            for (int t = lane; t < P; t += 32) {
                const int u = t ^ j;
                if (u > t) {
                    const int32_t a = buf[t], b = buf[u];
                    const bool up = (t & kk) == 0;
                    if ((a > b) == up) {
                        buf[t] = b;
                        buf[u] = a;
                    }
                }
            }
            __syncwarp();
        }
    int64_t out = p.row_ptr ? p.row_ptr[i] : 0;
    int cnt = 0;
    for (int t0 = 0; t0 < T; t0 += 32) {
        const int t = t0 + lane;
        bool keep = false;
        int32_t j = 0;
        int s = 0;
        if (t < T && (t == 0 || buf[t] != buf[t - 1])) {
            j = buf[t];
            s = 1;
            while (t + s < T && buf[t + s] == j) ++s;
            keep = snn_keep(s, p.k);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (keep && p.row_ptr) {
            const int64_t at = out + __popc(bal & ((1u << lane) - 1u));
            p.col[at] = j;
            p.w[at] = (double)s / (double)(p.k + (p.k - s));
        }
        out += __popc(bal);
        cnt += __popc(bal);
    }
    if (lane == 0 && !p.row_ptr) p.row_nnz[i] = cnt;
}

// Rows whose candidates exceed SN_CAP (hubs): each CTA owns n int32 counters in global memory (zero between rows), adds the
// candidates with integer atomics, then walks j = 0 .. n-1 in order, compacting the kept pairs and clearing the counters.
__global__ void __launch_bounds__(256) snn_spill_kernel(const SnnParams p, const int32_t *spill, int n_spill, int32_t *cnt_all) {
    __shared__ int wsum[8];
    __shared__ int64_t s_out;
    int32_t *cnt = cnt_all + (int64_t)blockIdx.x * p.n;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int b = blockIdx.x; b < n_spill; b += gridDim.x) {
        const int64_t i = spill[b];
        for (int r = 0; r < p.k; ++r) {
            const int32_t m = p.idx[i + p.n * r];
            for (int64_t t = p.roff[m] + threadIdx.x; t < p.roff[m + 1]; t += 256) atomicAdd(&cnt[p.rev[t]], 1);
        }
        if (threadIdx.x == 0) s_out = p.row_ptr ? p.row_ptr[i] : 0;
        __syncthreads();
        for (int64_t j0 = 0; j0 < p.n; j0 += 256) {
            const int64_t j = j0 + threadIdx.x;
            int s = 0;
            if (j < p.n) {   // volatile: the counts were added by other threads' atomics, past this SM's L1
                s = *(volatile int32_t *)&cnt[j];
                cnt[j] = 0;
            }
            const bool keep = s > 0 && snn_keep(s, p.k);
            const unsigned bal = __ballot_sync(0xffffffffu, keep);
            if (lane == 0) wsum[w] = __popc(bal);
            __syncthreads();
            int before = 0, tot = 0;
            for (int q = 0; q < 8; ++q) {
                before += q < w ? wsum[q] : 0;
                tot += wsum[q];
            }
            if (keep && p.row_ptr) {
                const int64_t at = s_out + before + __popc(bal & ((1u << lane) - 1u));
                p.col[at] = (int32_t)j;
                p.w[at] = (double)s / (double)(p.k + (p.k - s));
            }
            __syncthreads();
            if (threadIdx.x == 0) s_out += tot;
            __syncthreads();
        }
        if (threadIdx.x == 0 && !p.row_ptr) p.row_nnz[i] = (int32_t)s_out;
        __syncthreads();
    }
}

// ---- the last call's result and statistics -----------------------------------------------------------------------------

struct Result {
    char *buf = nullptr;   // one device allocation: row_ptr | emb | w | idx | features | col
    int64_t n = 0, nnz = 0;
    int nfeat = 0, npcs = 0, k = 0;
    int64_t *row_ptr = nullptr;
    double *emb = nullptr, *w = nullptr;
    int32_t *idx = nullptr, *feat = nullptr, *col = nullptr;
    int device = -1;
};
static Result g_res;
static double g_stats[16];

static size_t al(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace snn

void seurat_snn_release();

using namespace snn;

// Host-visible checks, before anything is allocated or read on the device.
int seurat_snn_check(int64_t G, int64_t n, int n_features, int npcs, int k, const char *who) {
    if (G < 1 || n < 1 || n_features < 1 || npcs < 1 || k < 1) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    if (k > ICNV_KNN_MAX_K) return set_error(ICNV_E_UNSUPPORTED, "%s: k = %d (limit %d)", who, k, ICNV_KNN_MAX_K);
    if (npcs > SN_NPCS_MAX) return set_error(ICNV_E_UNSUPPORTED, "%s: npcs = %d (limit %d)", who, npcs, SN_NPCS_MAX);
    if (n <= npcs) return set_error(ICNV_E_UNSUPPORTED, "%s: %lld cells for %d components", who, (long long)n, npcs);
    if (k > n) return set_error(ICNV_E_BAD_ARG, "%s: k = %d for %lld cells (1 <= k <= n)", who, k, (long long)n);
    if (n > 0x7ffffffell) return set_error(ICNV_E_UNSUPPORTED, "%s: %lld cells", who, (long long)n);
    return ICNV_OK;
}

// The host entry uploads the listed columns once and does not stream them: a group that does not fit is refused.
int seurat_snn_room(int64_t G, int64_t n, const char *who) {
    size_t free_b = 0, total_b = 0;
    ICNV_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const double need = 8.0 * (double)G * (double)n;
    if (need + (double)(512 << 20) > (double)free_b)
        return set_error(ICNV_E_UNSUPPORTED, "%s: the group (%.3g GB) does not fit the free device memory (%.3g GB)", who,
                         need / 1e9, (double)free_b / 1e9);
    return ICNV_OK;
}

// X: genes x columns (stride ldx >= G) on the device; d_cells: n device column indices (NULL: columns 0 .. n-1, already
// checked by the caller when given).  Synchronises `stream`.  Leaves the result in g_res.
int seurat_snn_dev(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n, int n_features, int npcs,
                   int k, int64_t *nnz_out, void *stream, const char *who) {
    ICNV_REQUIRE_READY();
    int rc = seurat_snn_check(G, n, n_features, npcs, k, who);
    if (rc) return rc;
    if (!X || ldx < G || !nnz_out) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    cudaStream_t st = pick_stream(stream);
    const int nf = (int)std::min<int64_t>(n_features, G);
    for (double &v : g_stats) v = 0.0;
    seurat_snn_release();   // the previous call's result

    // work area: gene arrays (7 G doubles / ints), eigen arrays (C F^2, Q, Y, V), embeddings, kNN, SNN
    const size_t bG = al(sizeof(double) * (size_t)G), bI = al(sizeof(int32_t) * (size_t)G);
    char *wg = nullptr, *we = nullptr, *ws = nullptr;
    std::vector<cudaEvent_t> ev(10, nullptr);
    auto body = [&]() -> int {
        if (cudaMallocAsync((void **)&wg, 6 * bG + 2 * bI + 256, st) != cudaSuccess) {
            cudaGetLastError();
            wg = nullptr;
            return set_error(ICNV_E_NOMEM, "%s: no room for the gene statistics", who);
        }
        double *mu = (double *)wg, *var = (double *)(wg + bG), *key = (double *)(wg + 2 * bG), *xs = (double *)(wg + 3 * bG),
               *ys = (double *)(wg + 4 * bG), *sexp = (double *)(wg + 5 * bG);
        int32_t *pos = (int32_t *)(wg + 6 * bG), *gene_at = (int32_t *)(wg + 6 * bG + bI);
        int *flags = (int *)(wg + 6 * bG + 2 * bI);   // [0] flag, [1] non-constant genes, [2] singular fits
        for (auto &e : ev) ICNV_CUDA(cudaEventCreate(&e));
        ICNV_CUDA(cudaEventRecord(ev[0], st));
        ICNV_CUDA(cudaMemsetAsync(flags, 0, 4 * sizeof(int), st));
        ICNV_CUDA(cudaMemsetAsync(sexp, 0, sizeof(double) * (size_t)G, st));
        const unsigned gb = (unsigned)((G + ST_GENES - 1) / ST_GENES);
        gene_stats_kernel<<<gb, ST_GENES * ST_WARPS, 0, st>>>(X, G, ldx, d_cells, n, mu, var, flags + 1, flags);
        ICNV_CHECK_LAUNCH("gene_stats_kernel");
        int hf[4] = {0, 0, 0, 0};
        ICNV_CUDA(cudaMemcpyAsync(hf, flags, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaEventRecord(ev[1], st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        if (hf[0] & 1) return set_error(ICNV_E_NONFINITE, "%s: NaN or Inf in a listed column", who);
        if (hf[0] & 4)
            return set_error(ICNV_E_UNSUPPORTED, "%s: a non-constant gene has mean <= 0: log10 of it is undefined (vst warns)", who);
        const int64_t m = hf[1], q = (int64_t)std::floor((double)m * SN_SPAN);
        if (q < 3) return set_error(ICNV_E_UNSUPPORTED, "%s: %lld non-constant genes leave a loess window of %lld", who,
                                    (long long)m, (long long)q);

        // 2. the trend over the sorted log10 means
        const unsigned g256 = (unsigned)((G + 255) / 256);
        trend_keys_kernel<<<g256, 256, 0, st>>>(mu, var, G, key);
        ICNV_CHECK_LAUNCH("trend_keys_kernel");
        rank_kernel<<<g256, 256, 0, st>>>(key, G, 0, pos);
        ICNV_CHECK_LAUNCH("rank_kernel");
        scatter_sorted_kernel<<<g256, 256, 0, st>>>(pos, mu, var, G, xs, ys, gene_at);
        ICNV_CHECK_LAUNCH("scatter_sorted_kernel");
        trend_kernel<<<(unsigned)((m + 7) / 8), 256, 0, st>>>(xs, ys, gene_at, m, q, sexp, flags + 2);
        ICNV_CHECK_LAUNCH("trend_kernel");
        ICNV_CUDA(cudaEventRecord(ev[2], st));

        // 3. standardised variances, their ranking, the variable features
        stdvar_kernel<<<gb, ST_GENES * ST_WARPS, 0, st>>>(X, G, ldx, d_cells, n, mu, sexp, std::sqrt((double)n), key);
        ICNV_CHECK_LAUNCH("stdvar_kernel");
        rank_kernel<<<g256, 256, 0, st>>>(key, G, 1, pos);
        ICNV_CHECK_LAUNCH("rank_kernel");
        std::vector<int32_t> hpos((size_t)G);
        std::vector<double> hsv((size_t)G), hvar((size_t)G), hmu((size_t)G);
        ICNV_CUDA(cudaMemcpyAsync(hpos.data(), pos, sizeof(int32_t) * (size_t)G, cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaMemcpyAsync(hsv.data(), key, sizeof(double) * (size_t)G, cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaMemcpyAsync(hvar.data(), var, sizeof(double) * (size_t)G, cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaMemcpyAsync(hmu.data(), mu, sizeof(double) * (size_t)G, cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaMemcpyAsync(hf, flags, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaEventRecord(ev[3], st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        std::vector<int32_t> ranked((size_t)G);
        for (int64_t g = 0; g < G; ++g) ranked[(size_t)hpos[(size_t)g]] = (int32_t)g;
        // the features PCA uses: the non-constant variable features, ascending gene index, with their rank
        std::vector<int32_t> feat;
        for (int r = 0; r < nf; ++r)
            if (hvar[(size_t)ranked[(size_t)r]] > 0.0) feat.push_back(ranked[(size_t)r]);
        std::sort(feat.begin(), feat.end());
        const int F = (int)feat.size();
        g_stats[0] = F;
        g_stats[1] = npcs;
        g_stats[5] = nf < G ? hsv[(size_t)ranked[(size_t)nf - 1]] - hsv[(size_t)ranked[(size_t)nf]] : INFINITY;
        g_stats[6] = hf[2];
        if (F <= npcs) return set_error(ICNV_E_UNSUPPORTED, "%s: %d non-constant variable features for %d components", who, F, npcs);
        std::vector<int32_t> rank_of((size_t)F);
        std::vector<double> fmu((size_t)F), fsd((size_t)F);
        for (int f = 0; f < F; ++f) {
            rank_of[(size_t)f] = hpos[(size_t)feat[(size_t)f]];
            fmu[(size_t)f] = hmu[(size_t)feat[(size_t)f]];
            fsd[(size_t)f] = std::sqrt(hvar[(size_t)feat[(size_t)f]]);
        }

        // 5. Gram matrix, eigenpairs, embeddings
        const int TB = (F + GT - 1) / GT, n_tiles = TB * (TB + 1) / 2;
        const int b = (int)std::min<int64_t>(std::min(SN_B, F), n - 1);
        const size_t bC = al(sizeof(double) * (size_t)F * F), bQ = al(sizeof(double) * (size_t)F * SN_B),
                     bV = al(sizeof(double) * (size_t)F * npcs), bF = al(sizeof(int32_t) * (size_t)F),
                     bFd = al(sizeof(double) * (size_t)F), bT = al(sizeof(int2) * (size_t)n_tiles);
        const size_t bP = al(sizeof(double) * 2 * SN_B * SN_B * (size_t)((F + EG_ROWS - 1) / EG_ROWS)),
                     bR = al(sizeof(double) * SN_NPCS_MAX * (size_t)((F + EG_ROWS - 1) / EG_ROWS));
        if (cudaMallocAsync((void **)&we, bC + 2 * bQ + bV + 2 * bF + 2 * bFd + bT + bP + bR + al(sizeof(EigState)), st) !=
            cudaSuccess) {
            cudaGetLastError();
            we = nullptr;
            return set_error(ICNV_E_NOMEM, "%s: no room for the %d x %d Gram matrix", who, F, F);
        }
        char *e = we;
        double *Cm = (double *)e; e += bC;
        double *Q = (double *)e; e += bQ;
        double *Y = (double *)e; e += bQ;
        double *V = (double *)e; e += bV;
        int32_t *d_feat = (int32_t *)e; e += bF;
        int32_t *d_rank = (int32_t *)e; e += bF;
        double *d_mu = (double *)e; e += bFd;
        double *d_sd = (double *)e; e += bFd;
        int2 *d_tiles = (int2 *)e; e += bT;
        double *part = (double *)e; e += bP;
        double *rpart = (double *)e; e += bR;
        EigState *d_st = (EigState *)e;
        std::vector<int2> tiles;
        for (int bi = 0; bi < TB; ++bi)
            for (int bj = bi; bj < TB; ++bj) tiles.push_back(make_int2(bi, bj));
        ICNV_CUDA(cudaMemcpyAsync(d_feat, feat.data(), sizeof(int32_t) * (size_t)F, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_rank, rank_of.data(), sizeof(int32_t) * (size_t)F, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_mu, fmu.data(), sizeof(double) * (size_t)F, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_sd, fsd.data(), sizeof(double) * (size_t)F, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_tiles, tiles.data(), sizeof(int2) * tiles.size(), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemsetAsync(d_st, 0, sizeof(EigState), st));
        GramParams gp{X, ldx, d_cells, n, d_feat, d_mu, d_sd, F, d_tiles, Cm};
        ICNV_CUDA(cudaEventRecord(ev[4], st));
        gram_kernel<<<(unsigned)n_tiles, 256, 0, st>>>(gp);
        ICNV_CHECK_LAUNCH("gram_kernel");
        ICNV_CUDA(cudaEventRecord(ev[5], st));
        subspace_start_kernel<<<(unsigned)(((int64_t)F * SN_B + 255) / 256), 256, 0, st>>>(Q, F, b);
        ICNV_CHECK_LAUNCH("subspace_start_kernel");
        const int n_part = (F + EG_ROWS - 1) / EG_ROWS;
        EigState hs{};
        for (int it0 = 0; it0 < SN_ITER_MAX && !hs.done; it0 += SN_BATCH) {
            for (int it = it0 + 1; it <= it0 + SN_BATCH && it <= SN_ITER_MAX; ++it) {
                const int check = it % SN_CHECK == 0 || it == SN_ITER_MAX;
                snn_mul_kernel<<<(unsigned)((F + 15) / 16), 256, 0, st>>>(Cm, F, Q, Y, d_st);
                ICNV_CHECK_LAUNCH("snn_mul_kernel");
                eig_gram_kernel<<<(unsigned)n_part, 1024, 0, st>>>(Q, Y, F, check, part, d_st);
                ICNV_CHECK_LAUNCH("eig_gram_kernel");
                eig_small_kernel<<<1, EG_SMALL_NT, 0, st>>>(part, n_part, b, check, d_st);
                ICNV_CHECK_LAUNCH("eig_small_kernel");
                if (check) {
                    eig_resid_kernel<<<(unsigned)n_part, 256, 0, st>>>(Q, Y, F, b, npcs, V, rpart, d_st);
                    ICNV_CHECK_LAUNCH("eig_resid_kernel");
                    eig_decide_kernel<<<1, 32, 0, st>>>(rpart, n_part, npcs, it, d_st);
                    ICNV_CHECK_LAUNCH("eig_decide_kernel");
                }
                eig_apply_kernel<<<(unsigned)((F + 31) / 32), 32, 0, st>>>(Y, Q, F, b, it, d_st);
                ICNV_CHECK_LAUNCH("eig_apply_kernel");
            }
            ICNV_CUDA(cudaMemcpyAsync(&hs, d_st, sizeof(EigState), cudaMemcpyDeviceToHost, st));
            ICNV_CUDA(cudaStreamSynchronize(st));
        }
        g_stats[2] = hs.iter;
        g_stats[3] = hs.max_res;
        g_stats[4] = b > npcs && hs.theta[npcs] > 0.0 ? hs.theta[npcs - 1] / hs.theta[npcs] : INFINITY;
        if (hs.status == 1) return set_error(ICNV_E_UNSUPPORTED, "%s: the subspace collapsed (rank of Z below %d)", who, b);
        if (!(hs.max_res <= 1e-12))
            return set_error(ICNV_E_UNSUPPORTED, "%s: no convergence in %d subspace iterations (residual %.3g of l_1)", who,
                             hs.iter, hs.max_res);
        sign_kernel<<<(unsigned)npcs, 256, 0, st>>>(V, F, npcs, d_rank);
        ICNV_CHECK_LAUNCH("sign_kernel");
        ICNV_CUDA(cudaEventRecord(ev[6], st));

        // result buffer (everything but the CSR columns and weights, whose size is known after the count pass)
        const size_t nk = (size_t)n * (size_t)k;
        const size_t bRP = al(sizeof(int64_t) * (size_t)(n + 1)), bE = al(sizeof(double) * (size_t)n * npcs),
                     bIdx = al(sizeof(int32_t) * nk), bFe = al(sizeof(int32_t) * (size_t)nf);
        const int64_t n_sp_ctas = SN_SPILL_CTAS;
        const size_t bN = al(sizeof(int32_t) * (size_t)(n + 1)), bN8 = al(sizeof(int64_t) * (size_t)(n + 2));
        // SNN work: dist (n k), deg, cursor, row_nnz (n each), roff, cand (n + 1, int64), rev (n k), spill list, counters
        const size_t bw = al(sizeof(double) * nk) + 3 * bN + 2 * bN8 + al(sizeof(int32_t) * nk) + bN;
        if (cudaMallocAsync((void **)&ws, bw, st) != cudaSuccess) {
            cudaGetLastError();
            ws = nullptr;
            return set_error(ICNV_E_NOMEM, "%s: no room for the neighbour lists", who);
        }
        Result R;
        R.n = n;
        R.nfeat = nf;
        R.npcs = npcs;
        R.k = k;
        R.device = ctx().device;
        // the result's first part; the CSR columns and weights follow once nnz is known (reallocated below)
        char *rb = nullptr;
        if (cudaMalloc((void **)&rb, bRP + bE + bIdx + bFe) != cudaSuccess) {
            cudaGetLastError();
            return set_error(ICNV_E_NOMEM, "%s: no room for the result", who);
        }
        R.buf = rb;
        R.row_ptr = (int64_t *)rb;
        R.emb = (double *)(rb + bRP);
        R.idx = (int32_t *)(rb + bRP + bE);
        R.feat = (int32_t *)(rb + bRP + bE + bIdx);
        g_res = R;
        ICNV_CUDA(cudaMemcpyAsync(R.feat, ranked.data(), sizeof(int32_t) * (size_t)nf, cudaMemcpyHostToDevice, st));
        embed_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(gp, V, npcs, R.emb);
        ICNV_CHECK_LAUNCH("embed_kernel");
        ICNV_CUDA(cudaEventRecord(ev[7], st));

        // 6. kNN (K12) and the SNN graph
        char *s = ws;
        double *dist = (double *)s; s += al(sizeof(double) * nk);
        int32_t *deg = (int32_t *)s; s += bN;
        int32_t *cursor = (int32_t *)s; s += bN;
        int32_t *row_nnz = (int32_t *)s; s += bN;
        int64_t *roff = (int64_t *)s; s += bN8;
        int64_t *cand = (int64_t *)s; s += bN8;
        int32_t *rev = (int32_t *)s; s += al(sizeof(int32_t) * nk);
        int32_t *spill = (int32_t *)s;
        if ((rc = knn_launch(R.emb, npcs, npcs, nullptr, n, k, R.idx, dist, 0, st, who))) return rc;
        ICNV_CUDA(cudaEventRecord(ev[8], st));
        ICNV_CUDA(cudaMemsetAsync(deg, 0, 2 * bN, st));   // deg and cursor
        const unsigned gk = (unsigned)std::min<int64_t>(((int64_t)nk + 255) / 256, 4096), gn = (unsigned)((n + 255) / 256);
        indegree_kernel<<<gk, 256, 0, st>>>(R.idx, (int64_t)nk, deg);
        ICNV_CHECK_LAUNCH("indegree_kernel");
        exclusive_scan_kernel<<<1, 1024, 0, st>>>(deg, n, roff);
        ICNV_CHECK_LAUNCH("exclusive_scan_kernel");
        reverse_fill_kernel<<<gk, 256, 0, st>>>(R.idx, n, k, roff, cursor, rev);
        ICNV_CHECK_LAUNCH("reverse_fill_kernel");
        candidates_kernel<<<gn, 256, 0, st>>>(R.idx, n, k, roff, cand);
        ICNV_CHECK_LAUNCH("candidates_kernel");
        std::vector<int64_t> hc((size_t)n);
        ICNV_CUDA(cudaMemcpyAsync(hc.data(), cand, sizeof(int64_t) * (size_t)n, cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        std::vector<int32_t> hsp;
        for (int64_t i = 0; i < n; ++i)
            if (hc[(size_t)i] > SN_CAP) hsp.push_back((int32_t)i);
        const int n_spill = (int)hsp.size();
        g_stats[15] = n_spill;
        int32_t *cnt_all = nullptr;
        if (n_spill) {
            ICNV_CUDA(cudaMemcpyAsync(spill, hsp.data(), sizeof(int32_t) * (size_t)n_spill, cudaMemcpyHostToDevice, st));
            const size_t bcnt = sizeof(int32_t) * (size_t)n * (size_t)std::min<int64_t>(n_spill, n_sp_ctas);
            if (cudaMallocAsync((void **)&cnt_all, bcnt, st) != cudaSuccess) {
                cudaGetLastError();
                return set_error(ICNV_E_NOMEM, "%s: no room for the hub rows' counters", who);
            }
            ICNV_CUDA(cudaMemsetAsync(cnt_all, 0, bcnt, st));
        }
        SnnParams sp{R.idx, n, k, roff, rev, cand, row_nnz, nullptr, nullptr, nullptr};
        const size_t rsm = sizeof(int32_t) * SN_CAP * SN_ROW_WARPS;
        ICNV_CUDA(cudaFuncSetAttribute(snn_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rsm));
        const unsigned gr = (unsigned)((n + SN_ROW_WARPS - 1) / SN_ROW_WARPS);
        const unsigned gsp = (unsigned)std::min(n_spill, SN_SPILL_CTAS);
        auto pass = [&]() -> int {
            snn_rows_kernel<<<gr, 32 * SN_ROW_WARPS, rsm, st>>>(sp);
            ICNV_CHECK_LAUNCH("snn_rows_kernel");
            if (n_spill) {
                snn_spill_kernel<<<gsp, 256, 0, st>>>(sp, spill, n_spill, cnt_all);
                ICNV_CHECK_LAUNCH("snn_spill_kernel");
            }
            return ICNV_OK;
        };
        rc = pass();
        if (!rc) {
            exclusive_scan_kernel<<<1, 1024, 0, st>>>(row_nnz, n, R.row_ptr);
            ICNV_CHECK_LAUNCH("exclusive_scan_kernel");
            int64_t nnz = 0;
            ICNV_CUDA(cudaMemcpyAsync(&nnz, R.row_ptr + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
            ICNV_CUDA(cudaStreamSynchronize(st));
            char *cb = nullptr;
            if (cudaMalloc((void **)&cb, al(sizeof(double) * (size_t)nnz) + al(sizeof(int32_t) * (size_t)nnz) + 256) != cudaSuccess) {
                cudaGetLastError();
                rc = set_error(ICNV_E_NOMEM, "%s: no room for %lld graph entries", who, (long long)nnz);
            } else {
                // keep both allocations reachable from the result: the CSR part is freed with it (see release below)
                g_res.w = (double *)cb;
                g_res.col = (int32_t *)(cb + al(sizeof(double) * (size_t)nnz));
                g_res.nnz = nnz;
                sp.row_ptr = R.row_ptr;
                sp.col = g_res.col;
                sp.w = g_res.w;
                rc = pass();
                if (!rc) {
                    ICNV_CUDA(cudaStreamSynchronize(st));
                    *nnz_out = nnz;
                }
            }
        }
        if (cnt_all) cudaFreeAsync(cnt_all, st);
        if (rc) return rc;
        ICNV_CUDA(cudaEventRecord(ev[9], st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        // stage times: statistics, trend, standardised variance + ranking, Gram, eigenpairs, embedding, kNN, SNN
        const int from[8] = {0, 1, 2, 4, 5, 6, 7, 8};
        const int to[8] = {1, 2, 3, 5, 6, 7, 8, 9};
        float ms = 0.0f;
        for (int i = 0; i < 8; ++i) {
            ICNV_CUDA(cudaEventElapsedTime(&ms, ev[from[i]], ev[to[i]]));
            g_stats[7 + i] = ms;
        }
        return ICNV_OK;
    };
    rc = body();
    if (ws) cudaFreeAsync(ws, st);
    if (we) cudaFreeAsync(we, st);
    if (wg) cudaFreeAsync(wg, st);
    cudaStreamSynchronize(st);
    for (auto &e : ev)
        if (e) cudaEventDestroy(e);
    if (rc) seurat_snn_release();
    return rc;
}

void seurat_snn_release() {
    if (g_res.w) cudaFree(g_res.w);
    if (g_res.buf) cudaFree(g_res.buf);
    g_res = Result{};
}

int seurat_snn_fetch(int64_t *row_ptr, int32_t *col, double *w, int32_t *features, double *emb, int32_t *idx,
                     cudaStream_t st, const char *who) {
    if (!g_res.buf) return set_error(ICNV_E_BAD_ARG, "%s: no SNN graph has been computed", who);
    const Result &R = g_res;
    if (row_ptr) ICNV_CUDA(cudaMemcpyAsync(row_ptr, R.row_ptr, sizeof(int64_t) * (size_t)(R.n + 1), cudaMemcpyDeviceToHost, st));
    if (col && R.nnz) ICNV_CUDA(cudaMemcpyAsync(col, R.col, sizeof(int32_t) * (size_t)R.nnz, cudaMemcpyDeviceToHost, st));
    if (w && R.nnz) ICNV_CUDA(cudaMemcpyAsync(w, R.w, sizeof(double) * (size_t)R.nnz, cudaMemcpyDeviceToHost, st));
    if (features) ICNV_CUDA(cudaMemcpyAsync(features, R.feat, sizeof(int32_t) * (size_t)R.nfeat, cudaMemcpyDeviceToHost, st));
    if (emb) ICNV_CUDA(cudaMemcpyAsync(emb, R.emb, sizeof(double) * (size_t)R.n * R.npcs, cudaMemcpyDeviceToHost, st));
    if (idx) ICNV_CUDA(cudaMemcpyAsync(idx, R.idx, sizeof(int32_t) * (size_t)R.n * R.k, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

void seurat_snn_stats(double *out16) {
    for (int i = 0; i < 16; ++i) out16[i] = g_stats[i];
}

}  // namespace icnv
