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

#include <algorithm>

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

// The 128 x 128 tile of squared distances between list positions i0 + r and j0 + c (r, c < 128): thread (tx, ty) ends with
// the sums of rows ty + 16 p and columns tx + 16 q in acc[p][q].  Positions past the list stage cell n - 1 (their sums are
// meaningless and never used).  Ends with a block barrier when there is a gene, so the staging buffers As / Bs
// ([2][PD_T][PD_LD] each) may be refilled as soon as it returns.  K10 and K12 both call it: one gene loop, one set of bits.
__device__ __forceinline__ void dist_tile(const DistParams &p, int64_t i0, int64_t j0, double *As, double *Bs, double (&acc)[8][8]) {
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
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
}

__global__ void __launch_bounds__(PD_NT, 1) pairwise_dist_kernel(const DistParams p) {
    const int bi = blockIdx.y, bj = blockIdx.x;
    if (bi > bj) return;   // the lower triangle is the upper one's mirror image
    extern __shared__ __align__(16) double pd_smem[];
    double *As = pd_smem;                          // [2][PD_T][PD_LD]
    double *Bs = pd_smem + 2 * PD_T * PD_LD;       // [2][PD_T][PD_LD]
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int64_t i0 = (int64_t)bi * PD_T, j0 = (int64_t)bj * PD_T;
    double acc[8][8];
    dist_tile(p, i0, j0, As, Bs, acc);
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

// ---- K13b's distances: pairwise_dist_kernel's tiles written straight into the linkage's square matrices -----------------
// Member z = blockIdx.x / T (tile column blockIdx.x % T, T tiles per side): columns X + z * sx (ldx, no cell list), matrix M + z * sm (n x ld).  Entry (a, b), a != b, is the
// value hclust_fill_kernel would store from pairwise_dist_kernel's entry of the pair, v = sqrt(sum) (v * v for ward.D2), in
// both triangles; the diagonal is +inf.  flag |= 1 when a value is not finite, as that kernel reports it.
// K17's members of different n (tiles != nullptr): a 1-D grid over a tile-work table, tiles[blockIdx.x] = (member, bi, bj)
// with bi <= bj; the member's cells are d.cells + cell_off (X and ldx shared), its matrix M + m_off with its own ld.
struct DistSqParams {
    DistParams d;         // X, G, ldx, n, rows = 0, cells = out = nullptr (a member table: cells = the groups' lists)
    int64_t sx, sm, ld;
    unsigned T;
    double *M;
    int square;
    int *flag;
    const int4 *tiles;
    const HcMember *mem;
};

__global__ void __launch_bounds__(PD_NT, 1) dist_square_kernel(const DistSqParams q) {
    int bi, bj;
    int64_t n, ld;
    DistParams p = q.d;
    double *M;
    if (q.tiles) {
        const int4 t = q.tiles[blockIdx.x];
        const HcMember m = q.mem[t.x];
        bi = t.y;
        bj = t.z;
        n = p.n = m.n;
        ld = m.ld;
        p.cells += m.cell_off;
        M = q.M + m.m_off;
    } else {
        const unsigned z = blockIdx.x / q.T;
        bi = blockIdx.y;
        bj = (int)(blockIdx.x - z * q.T);
        if (bi > bj) return;
        n = q.d.n;
        ld = q.ld;
        p.X += (int64_t)z * q.sx;
        M = q.M + (int64_t)z * q.sm;
    }
    extern __shared__ __align__(16) double pd_smem[];
    double *As = pd_smem;
    double *Bs = pd_smem + 2 * PD_T * PD_LD;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int64_t i0 = (int64_t)bi * PD_T, j0 = (int64_t)bj * PD_T;
    double acc[8][8];
    dist_tile(p, i0, j0, As, Bs, acc);
    bool bad = false;
#pragma unroll
    for (int pp = 0; pp < 8; ++pp) {
        const int64_t a = i0 + ty + 16 * pp;
        if (a >= n) continue;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int64_t b = j0 + tx + 16 * c;
            if (b == a) M[a * ld + a] = __longlong_as_double(0x7ff0000000000000ll);
            if (b <= a || b >= n) continue;
            const double v = sqrt(acc[pp][c]);
            bad |= !is_finite_d(v);
            const double w = q.square ? __dmul_rn(v, v) : v;
            M[a * ld + b] = w;
            M[b * ld + a] = w;
        }
    }
    if (bad) atomicOr(q.flag, 1);
}

// B members of n cells each (genes x cells, member z's columns at X + z * sx) -> their n x ld matrices (M + z * sm)
int dist_square_launch(const double *X, int64_t G, int64_t ldx, int64_t sx, int64_t n, int B, double *M, int64_t ld,
                       int64_t sm, int square, int *flag, cudaStream_t st) {
    const int64_t T = (n + PD_T - 1) / PD_T;
    if (T > 65535) return set_error(ICNV_E_UNSUPPORTED, "distances: %lld cells (limit %d)", (long long)n, 65535 * PD_T);
    DistSqParams q{{X, G, ldx, nullptr, n, nullptr, 0}, sx, sm, ld, (unsigned)T, M, square, flag, nullptr, nullptr};
    const size_t smem = sizeof(double) * 4 * PD_T * PD_LD;
    ICNV_CUDA(cudaFuncSetAttribute(dist_square_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dist_square_kernel<<<dim3((unsigned)(T * B), (unsigned)T), PD_NT, smem, st>>>(q);
    ICNV_CHECK_LAUNCH("dist_square_kernel");
    return ICNV_OK;
}

// K17: the n_tiles tiles of d_tiles (device; (member, bi, bj), bi <= bj) over the members d_mem (device), whose cells are
// columns X + ldx d_cells[cell_off + a] (genes x cells) -> each member's matrix in M.
int dist_square_members_launch(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, const int4 *d_tiles,
                               int64_t n_tiles, const HcMember *d_mem, double *M, int square, int *flag, cudaStream_t st) {
    if (n_tiles <= 0) return ICNV_OK;
    if (n_tiles > 0x7fffffff) return set_error(ICNV_E_UNSUPPORTED, "distances: %lld tiles in one launch", (long long)n_tiles);
    DistSqParams q{{X, G, ldx, d_cells, 0, nullptr, 0}, 0, 0, 0, 1u, M, square, flag, d_tiles, d_mem};
    const size_t smem = sizeof(double) * 4 * PD_T * PD_LD;
    ICNV_CUDA(cudaFuncSetAttribute(dist_square_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dist_square_kernel<<<(unsigned)n_tiles, PD_NT, smem, st>>>(q);
    ICNV_CHECK_LAUNCH("dist_square_kernel");
    return ICNV_OK;
}

// ---- K12: exact k nearest neighbours (RANN::nn2(data, k = k) with the query set = the data set) --------------------------
//
// Order: ascending squared distance, then ascending list position - a total order, so the result does not depend on launch
// geometry or thread order, and a cell comes first in its own row (distance exactly 0) unless a duplicate of it has a lower
// position.  The squared distances are dist_tile's sums, the very bits K10 roots: every reported distance equals the
// parallelDist() value of the same pair.
//
// One CTA = one 128-cell query tile x one split of the candidate tiles (blockIdx.y of S; S from n and the SM count, never from
// a switch).  Per candidate tile, the 128 candidates of a query row sit in the registers of the 16 lanes (one half-warp) that
// hold that row, and that half-warp owns the row's running list of its k best in shared memory - no block barrier: each lane
// compares its 8 candidates with the row's current k-th entry, the warp ballots the survivors (usually none after the first
// tiles), and one survivor at a time replaces the list's greatest entry, whose successor the half-warp finds with shuffles.
// The list starts as k copies of (+inf, INT_MAX), which every real candidate precedes.  Each split's k best per row go to a
// partial buffer (split-major, n x k per split); knn_merge_kernel ranks the S k entries of a row and roots the first k.
constexpr int KNN_KMAX = ICNV_KNN_MAX_K;   // cap on k: 128 lists of 64 x 12 bytes fit beside the staging buffers
constexpr int KNN_SMAX = 16;     // cap on the splits
constexpr int KNN_MMAX = 512;    // cap on S k, the entries the merge ranks per row
constexpr int KNN_NONE = 0x7fffffff;

struct KnnParams {
    DistParams d;       // X, G, ldx, cells, n, rows (out unused)
    int64_t T;          // query / candidate tiles
    int k, S;
    double *part_d;     // [S][n][k] squared distances of each split's k best
    int32_t *part_j;    // [S][n][k] their list positions
    int *flag;          // |= 1: a non-finite value in some cell - its distance to itself is NaN
};

// index of the lowest set bit of v != 0
__device__ __forceinline__ int lowest_bit(unsigned v) { return __popc((v & (0u - v)) - 1u); }
__device__ __forceinline__ bool knn_less(double d, int j, double D, int J) { return d < D || (d == D && j < J); }
// (d, j, slot) after (D, J, S): the list's greatest entry; the slot breaks the ties of the identical initial entries
__device__ __forceinline__ bool knn_after(double d, int j, int s, double D, int J, int S) {
    return d > D || (d == D && (j > J || (j == J && s > S)));
}

__global__ void __launch_bounds__(PD_NT, 1) knn_partial_kernel(const KnnParams q) {
    extern __shared__ __align__(16) double pd_smem[];
    double *As = pd_smem;                          // [2][PD_T][PD_LD]
    double *Bs = pd_smem + 2 * PD_T * PD_LD;       // [2][PD_T][PD_LD]
    const int k = q.k;
    double *Ld = pd_smem + 4 * PD_T * PD_LD;       // [PD_T][k] each row's list: squared distances
    double *Rd = Ld + PD_T * k;                    // [PD_T] the list's greatest entry: squared distance,
    int32_t *Lj = (int32_t *)(Rd + PD_T);          // [PD_T][k] list positions
    int32_t *Rj = Lj + PD_T * k;                   // [PD_T] position,
    int32_t *Rs = Rj + PD_T;                       // [PD_T] slot
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4, lane = tid & 31, hbase = lane & 16;
    const double inf = __longlong_as_double(0x7ff0000000000000ll);
    for (int e = tid; e < PD_T * k; e += PD_NT) {
        Ld[e] = inf;
        Lj[e] = KNN_NONE;
    }
    for (int r = tid; r < PD_T; r += PD_NT) {
        Rd[r] = inf;
        Rj[r] = KNN_NONE;
        Rs[r] = 0;
    }
    __syncthreads();
    const int64_t n = q.d.n, i0 = (int64_t)blockIdx.x * PD_T;
    const int s = blockIdx.y;
    const int64_t t1 = q.T * (s + 1) / q.S;
    for (int64_t t = q.T * s / q.S; t < t1; ++t) {
        const int64_t j0 = t * PD_T;
        double acc[8][8];
        dist_tile(q.d, i0, j0, As, Bs, acc);
        if (j0 == i0 && tx == ty) {   // x - x is 0 unless x is NaN or +-Inf
#pragma unroll
            for (int pp = 0; pp < 8; ++pp)
                if (i0 + ty + 16 * pp < n && !(acc[pp][pp] == acc[pp][pp])) atomicOr(q.flag, 1);
        }
#pragma unroll
        for (int pp = 0; pp < 8; ++pp) {
            const int r = ty + 16 * pp;
            const bool row_ok = i0 + r < n;
            double td = Rd[r];
            int tj = Rj[r], ts = Rs[r];
            unsigned m = 0;   // this lane's candidates of the row that precede its greatest entry
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const int64_t j = j0 + tx + 16 * c;
                if (row_ok && j < n && knn_less(acc[pp][c], (int)j, td, tj)) m |= 1u << c;
            }
            bool changed = false;
            for (;;) {   // warp-uniform: both half-warps take part in every collective
                const unsigned any = __ballot_sync(0xffffffffu, m != 0);
                if (!any) break;
                const unsigned mine = (any >> hbase) & 0xffffu;
                const int src = mine ? hbase + lowest_bit(mine) : lane;
                const int c0 = m ? lowest_bit(m) : 0;   // this lane's first candidate; src's is the one broadcast
                double cd = 0.0;
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    if (c == c0) cd = acc[pp][c];
                cd = __shfl_sync(0xffffffffu, cd, src);
                const int cj = __shfl_sync(0xffffffffu, (int)(j0 + tx + 16 * c0), src);
                if (lane == src) m &= m - 1;
                const bool act = mine != 0 && knn_less(cd, cj, td, tj);   // the same in all 16 lanes of the half
                if (act && tx == 0) {
                    Ld[r * k + ts] = cd;
                    Lj[r * k + ts] = cj;
                }
                __syncwarp();
                double bd = -1.0;
                int bj = -1, bs = -1;
                if (act)
                    for (int e = tx; e < k; e += 16) {
                        const double d = Ld[r * k + e];
                        const int j = Lj[r * k + e];
                        if (knn_after(d, j, e, bd, bj, bs)) {
                            bd = d;
                            bj = j;
                            bs = e;
                        }
                    }
#pragma unroll
                for (int o = 8; o > 0; o >>= 1) {
                    const double od = __shfl_xor_sync(0xffffffffu, bd, o);
                    const int oj = __shfl_xor_sync(0xffffffffu, bj, o), os = __shfl_xor_sync(0xffffffffu, bs, o);
                    if (knn_after(od, oj, os, bd, bj, bs)) {
                        bd = od;
                        bj = oj;
                        bs = os;
                    }
                }
                if (act) {
                    td = bd;
                    tj = bj;
                    ts = bs;
                    changed = true;
#pragma unroll
                    for (int c = 0; c < 8; ++c)
                        if (((m >> c) & 1u) && !knn_less(acc[pp][c], (int)(j0 + tx + 16 * c), td, tj)) m &= ~(1u << c);
                }
            }
            if (changed && tx == 0) {
                Rd[r] = td;
                Rj[r] = tj;
                Rs[r] = ts;
            }
            __syncwarp();
        }
    }
    __syncthreads();
    const int64_t base = ((int64_t)s * n + i0) * k;
    for (int e = tid; e < PD_T * k; e += PD_NT)
        if (i0 + e / k < n) {
            q.part_d[base + e] = Ld[e];
            q.part_j[base + e] = Lj[e];
        }
}

// One warp per row: the rank of each of the row's S k partial entries among them (entries are distinct: a position
// appears in one split only, and the (+inf, INT_MAX) fillers rank behind the n >= k real ones), the first k written
// column-major with their distance rooted.
__global__ void __launch_bounds__(256) knn_merge_kernel(const double *part_d, const int32_t *part_j, int64_t n, int S, int k,
                                                        int32_t *idx, double *dist) {
    const int64_t i = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (i >= n) return;
    const int lane = threadIdx.x & 31, M = S * k;
    for (int e = lane; e < M; e += 32) {
        const int64_t pe = ((int64_t)(e / k) * n + i) * k + e % k;
        const double d = part_d[pe];
        const int j = part_j[pe];
        if (j == KNN_NONE) continue;
        int rank = 0;
        for (int f = 0; f < M && rank < k; ++f) {
            const int64_t pf = ((int64_t)(f / k) * n + i) * k + f % k;
            rank += knn_less(part_d[pf], part_j[pf], d, j);
        }
        if (rank < k) {
            idx[i + n * rank] = j;
            dist[i + n * rank] = sqrt(d);
        }
    }
}

// Splits of the candidate range: S (at most KNN_SMAX, S k at most KNN_MMAX, at least one tile each) against the launch's
// time in units of one unsplit CTA, ceil(T S / slots) / S, where slots = resident CTAs of the device: the smallest S within
// 5 % of the best such time (more splits only add partial lists and merge work).
static int knn_splits(int64_t T, int64_t slots, int k) {
    const int64_t s_max = std::min<int64_t>(std::min<int64_t>(KNN_SMAX, T), KNN_MMAX / k);
    int64_t best = 1, best_w = (T + slots - 1) / slots;
    for (int64_t S = 2; S <= s_max; ++S) {
        const int64_t w = (T * S + slots - 1) / slots;
        if (w * best < best_w * S) {
            best = S;
            best_w = w;
        }
    }
    for (int64_t S = 1; S <= s_max; ++S)
        if (100 * ((T * S + slots - 1) / slots) * best <= 105 * best_w * S) return (int)S;
    return (int)best;
}

// K12 on device memory in either of K10's layouts (rows: observations x variables); icnv_api.cu's host entry points call it
// too.  Enqueues both kernels on the stream, then synchronises it once to report non-finite input.
int knn_launch(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n, int k, int32_t *idx, double *dist,
               int rows, void *stream, const char *who) {
    ICNV_REQUIRE_READY();
    if (n < 0 || G < 0 || (n > 0 && (!X || !idx || !dist || ldx < (rows ? n : G))) || (rows && d_cells))
        return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    if (n == 0) return ICNV_OK;
    if (k < 1 || k > n) return set_error(ICNV_E_BAD_ARG, "%s: k = %d for %lld cells (1 <= k <= n)", who, k, (long long)n);
    if (k > KNN_KMAX) return set_error(ICNV_E_UNSUPPORTED, "%s: k = %d (limit %d)", who, k, KNN_KMAX);
    if (n > KNN_NONE - 1) return set_error(ICNV_E_UNSUPPORTED, "%s: %lld cells (limit %d)", who, (long long)n, KNN_NONE - 1);
    Ctx &c = ctx();
    cudaStream_t st = pick_stream(stream);
    const int64_t T = (n + PD_T - 1) / PD_T;
    const size_t smem = sizeof(double) * 4 * PD_T * PD_LD + (sizeof(double) + sizeof(int32_t)) * PD_T * (size_t)k +
                        (sizeof(double) + 2 * sizeof(int32_t)) * PD_T;
    ICNV_CUDA(cudaFuncSetAttribute(knn_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    ICNV_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, knn_partial_kernel, PD_NT, smem));
    const int S = knn_splits(T, (int64_t)c.sm_count * std::max(per_sm, 1), k);
    const size_t n_part = (size_t)S * (size_t)n * (size_t)k;
    char *w = (char *)scratch(SLOT_KNN, (sizeof(double) + sizeof(int32_t)) * n_part + 16);
    if (!w) return ICNV_E_NOMEM;
    int *flag = (int *)w;
    KnnParams q{{X, G, ldx, d_cells, n, nullptr, rows}, T, k, S, (double *)(w + 16), (int32_t *)(w + 16 + sizeof(double) * n_part), flag};
    ICNV_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));
    knn_partial_kernel<<<dim3((unsigned)T, (unsigned)S), PD_NT, smem, st>>>(q);
    ICNV_CHECK_LAUNCH("knn_partial_kernel");
    knn_merge_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(q.part_d, q.part_j, n, S, k, idx, dist);
    ICNV_CHECK_LAUNCH("knn_merge_kernel");
    int h_flag = 0;
    ICNV_CUDA(cudaMemcpyAsync(&h_flag, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    if (h_flag) return set_error(ICNV_E_NONFINITE, "%s: NaN or Inf in the input", who);
    return ICNV_OK;
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

int icnv_dev_knn_f64(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n, int k, int32_t *idx,
                     double *dist, void *stream) {
    return knn_launch(X, G, ldx, d_cells, n, k, idx, dist, 0, stream, "icnv_dev_knn_f64");
}

}  // extern "C"
