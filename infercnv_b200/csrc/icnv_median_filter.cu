// icnv_median_filter.cu - K4: apply_median_filtering / .median_filter (R/noise_reduction.R:43-113).
//
// out[i, j] = median(B[max(0,i-r) .. min(n-1,i+r), max(0,j-r) .. min(m-1,j+r)]) on every block
// B = (genes of one chromosome) x (cells of one index list, in list order), r = (window_size+1)/2
// as in the reference (noise_reduction.R:102-106: half_window + 1).  Even-count windows average
// the two middle values (median.default).  Reads the un-filtered input throughout.
//
// One thread per output element.  Window sizes 3, 5 and 9 (radius 2, 3, 5) run median_filter_select_kernel: the tile's
// halo is staged in shared memory and every thread selects its window's median by counting (icnv_median_select.cuh - no
// data-dependent partitioning, so the lanes of a warp stay together).  Window size 7 (radius 4, the reference's default)
// runs the shared-merge kernel further down.  Larger window sizes use the generic kernel below (in-place Wirth selection
// over a private index array).
#include <cfloat>
#include <cmath>
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "icnv_common.cuh"
#include "icnv_median_select.cuh"

namespace icnv {

struct MfTile {
    int start;  // first gene (or first list position) of the tile
    int len;    // valid entries in the tile
    int lo;     // block start (chromosome start / group offset in the concatenated list)
    int hi;     // block end, exclusive
};

struct MfParams {
    const double *X;
    double *Y;
    int64_t G;
    const int32_t *cells;     // concatenated index lists (device)
    const MfTile *gene_tiles; // gridDim.y entries
    const MfTile *cell_tiles; // gridDim.x entries
    int r;
    int *err_flag;
    // shared-merge kernel: the matrix' range (keys quantise over it) and its dominant value (NaN: none), found before the launch
    double vmin, vmax, mode;
    double scale;             // (2^24 - 3) / (vmax - vmin), 0 if the matrix is constant
    const long long *coloff;  // shared-merge kernel: G * cells[i] per list entry
};

// One CTA = a tile of TI genes x TJ list positions (TI*TJ threads, one output each).  The tile's halo
// ((TI+2r) x (TJ+2r) values, clamped to the chromosome / index-list block) is loaded ONCE into shared
// memory, coalesced along genes; every thread then selects its median over a private array of 16-bit
// indices into that shared halo - nothing but indices ever moves.  12 KB of shared memory per 64-thread
// CTA for the default window (against 83 KB of private value copies before) keeps ~36 warps per SM busy
// on what is a chain of dependent shared-memory reads.
constexpr int MF_TI = 8, MF_TJ = 8, MF_NT = MF_TI * MF_TJ;

__global__ void __launch_bounds__(MF_NT) median_filter_kernel(const MfParams p) {
    extern __shared__ __align__(16) unsigned char mf_smem[];
    const int r = p.r;
    const int HR = MF_TI + 2 * r, HC = MF_TJ + 2 * r;       // halo rows (genes, fast) x cols (cells)
    const int W = (2 * r + 1) * (2 * r + 1);
    double *halo = reinterpret_cast<double *>(mf_smem);
    unsigned short *idx_all = reinterpret_cast<unsigned short *>(halo + HR * HC);
    const MfTile gt = p.gene_tiles[blockIdx.y];
    const MfTile ct = p.cell_tiles[blockIdx.x];
    const int hi0 = gt.start - r, hj0 = ct.start - r;
    bool bad = false;
    // ---- halo: rows inside [gt.lo, gt.hi), list positions inside [ct.lo, ct.hi) -------------------------
    for (int e = threadIdx.x; e < HR * HC; e += MF_NT) {
        const int hr = e % HR, hc = e / HR;
        const int ii = hi0 + hr, jj = hj0 + hc;
        double v = 0.0;
        if (ii >= gt.lo && ii < gt.hi && jj >= ct.lo && jj < ct.hi) {
            v = p.X[ii + p.G * (int64_t)p.cells[jj]];
            bad |= !is_finite_d(v);
        }
        halo[e] = v;
    }
    __syncthreads();
    const int ti = threadIdx.x % MF_TI, tj = threadIdx.x / MF_TI;
    if (ti < gt.len && tj < ct.len) {
        const int i = gt.start + ti, j = ct.start + tj;
        const int xa = max(gt.lo, i - r), xb = min(gt.hi - 1, i + r);
        const int ya = max(ct.lo, j - r), yb = min(ct.hi - 1, j + r);
        unsigned short *a = idx_all + threadIdx.x;   // [tap][thread]
        int n = 0;
        for (int jj = ya; jj <= yb; ++jj)
            for (int ii = xa; ii <= xb; ++ii) {
                a[n * MF_NT] = (unsigned short)((jj - hj0) * HR + (ii - hi0));
                ++n;
            }
        (void)W;
#define MF_VAL(q) halo[a[(q) * MF_NT]]
        // k-th smallest, k = (n-1)/2 (Wirth); afterwards val[0..k-1] <= val[k] <= val[k+1..n-1]
        const int k = (n - 1) >> 1;
        int l = 0, rr = n - 1;
        while (l < rr) {
            const double x = MF_VAL(k);
            int u = l, w = rr;
            do {
                while (MF_VAL(u) < x) ++u;
                while (x < MF_VAL(w)) --w;
                if (u <= w) {
                    const unsigned short t = a[u * MF_NT];
                    a[u * MF_NT] = a[w * MF_NT];
                    a[w * MF_NT] = t;
                    ++u;
                    --w;
                }
            } while (u <= w);
            if (w < k) l = u;
            if (k < u) rr = w;
        }
        double med = MF_VAL(k);
        if ((n & 1) == 0) {  // mean of the two middle values
            double nxt = DBL_MAX;
            for (int q = k + 1; q < n; ++q) nxt = fmin(nxt, MF_VAL(q));
            med = (med + nxt) * 0.5;
        }
#undef MF_VAL
        p.Y[i + p.G * (int64_t)p.cells[j]] = med;
    }
    if (bad && p.err_flag) atomicExch(p.err_flag, 1);
}

// Tile of 32 genes x 8 list positions, 256 threads; a warp covers 32 consecutive genes of one cell, so its halo reads
// are consecutive doubles (no bank conflicts) and the per-thread tap lists interleave at 2-byte granularity.
constexpr int MS_TI = 32, MS_TJ = 8, MS_NT = MS_TI * MS_TJ;

template <int R>
__global__ void __launch_bounds__(MS_NT) median_filter_select_kernel(const MfParams p) {
    extern __shared__ __align__(16) unsigned char mf_smem[];
    constexpr int D = 2 * R + 1, HR = MS_TI + 2 * R, HC = MS_TJ + 2 * R;
    double *halo = reinterpret_cast<double *>(mf_smem);          // +inf outside the block: never counted
    double *halo0 = halo + HR * HC;                              // 0 outside the block: for the window moments
    unsigned short *list = reinterpret_cast<unsigned short *>(halo0 + HR * HC);   // [D*D][MS_NT] tap offsets
    const MfTile gt = p.gene_tiles[blockIdx.y];
    const MfTile ct = p.cell_tiles[blockIdx.x];
    const int hi0 = gt.start - R, hj0 = ct.start - R;
    bool bad = false;
    for (int e = threadIdx.x; e < HR * HC; e += MS_NT) {
        const int hr = e % HR, hc = e / HR;
        const int ii = hi0 + hr, jj = hj0 + hc;
        double v = INFINITY, v0 = 0.0;
        if (ii >= gt.lo && ii < gt.hi && jj >= ct.lo && jj < ct.hi) {
            v = p.X[ii + p.G * (int64_t)p.cells[jj]];
            bad |= !is_finite_d(v);
            v0 = v;
        }
        halo[e] = v;
        halo0[e] = v0;
    }
    __syncthreads();
    const int ti = threadIdx.x % MS_TI, tj = threadIdx.x / MS_TI;
    if (ti < gt.len && tj < ct.len) {
        const int i = gt.start + ti, j = ct.start + tj;
        const int xa = max(gt.lo, i - R), xb = min(gt.hi - 1, i + R);
        const int ya = max(ct.lo, j - R), yb = min(ct.hi - 1, j + R);
        const int n = (xb - xa + 1) * (yb - ya + 1);
        p.Y[i + p.G * (int64_t)p.cells[j]] = window_median<R>(halo, halo0, HR, tj * HR + ti, list + threadIdx.x, MS_NT, n);
    }
    if (bad && p.err_flag) atomicExch(p.err_flag, 1);
}

// Range of the matrix (finite values) for the key quantisation of the shared-merge kernel, and a sample of its values from
// which the host picks the dominant one.  One read of the matrix (~0.13 ms per 10^8 values).
__global__ void __launch_bounds__(256) mf_range_kernel(const double *__restrict__ X, int64_t n, unsigned long long *__restrict__ range,
                                                       double *__restrict__ sample, int n_sample) {
    double mn = INFINITY, mx = -INFINITY;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const double v = X[i];
        if (is_finite_d(v)) {
            mn = v < mn ? v : mn;
            mx = v > mx ? v : mx;
        }
    }
    mn = warp_min_d(mn);
    mx = warp_max_d(mx);
    if ((threadIdx.x & 31) == 0) {
        if (mn <= mx) {   // order-preserving integer keys: min / max by integer atomics
            atomicMin(&range[0], key_of(mn));
            atomicMax(&range[1], key_of(mx));
        }
    }
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n_sample) sample[t] = X[(int64_t)((double)t * (double)n / (double)n_sample)];
}

// =================================================================================================
// window_size 7 (radius 4, 9 x 9 taps - the default of apply_median_filtering): shared-merge networks on 32-bit keys
// =================================================================================================
//
// The counting selection above redoes all of a window's work for every output although neighbouring windows share 72 of
// their 81 taps.  Here a tile of 32 genes x 32 list positions is worked on by the whole CTA in stages that keep what is
// shared (tools/gen_median_merge.py, icnv_median_merge.inc; lane = gene, every list below is per gene):
//   S0  the halo (40 genes x 40 positions) is loaded once; every value gets a 32-bit key = 24 bits of its position
//       between the tile's minimum and maximum (monotone) | an 8-bit tag (gene mod 16, position mod 16) that is unique
//       inside any 9 x 9 window.  Taps outside the chromosome / index-list block get the keys 0 and 0xffffffff in a
//       checkerboard, so that a truncated window is still 81 keys with its median at rank 40, 41 or 42.
//   S1  per halo position: the 9 keys around the gene sorted (a "run", 25 comparators); runs of consecutive positions
//       merged in pairs (P, 18 keys)
//   S2  P + P -> Q (36 keys, four consecutive positions)
//   S3  per pair of outputs: the 8 positions they share = Q + Q, of which only ranks 30..43 can still be a median; each
//       output adds its own ninth run and reads off ranks 39..43 of its 81 keys.
// ~290 min / max operations per output instead of ~1400 for a network per window (or ~4600 instructions of counting).
// The median's key carries its tap in the tag, so its double is one shared-memory load away.  Keys order the values up to
// the 24-bit quantisation: when a neighbour in rank shares the median's quantised value, the rank is settled exactly by
// counting over the doubles of that quantisation cell (mm_exact_rank); identical values - de-noised matrices - stay cheap
// there because a cell whose doubles are all equal needs no further selection.
#define mf_min(a, b) min((unsigned)(a), (unsigned)(b))
#define mf_max(a, b) max((unsigned)(a), (unsigned)(b))
#include "icnv_median_merge.inc"

constexpr int MM_TX = 32;                        // outputs per tile along the genes (lanes)
constexpr int MM_HX = MM_TX + 8;                 // halo genes
constexpr int MM_PW = 20, MM_QW = 36;            // words per gene and list (P padded to a multiple of 4)
constexpr unsigned MM_LOW = 0u, MM_HIGH = 0xffffffffu;

// TY = outputs per tile along the index list.  Halo rows 0 .. TY+9 (row r = list position y0 - 5 + r; rows 1 .. TY+8 are used);
// P lists: rows (2t, 2t+1), t = 1 .. TY/2+3; Q lists: P[q] + P[q+1].
constexpr size_t mm_smem_bytes(int TY) {
    return sizeof(double) * (size_t)(TY + 10) * MM_HX + sizeof(unsigned) * (size_t)(TY + 10) * MM_HX +
           sizeof(unsigned) * (size_t)(TY + 10) * 9 * MM_TX + sizeof(unsigned) * (size_t)(TY / 2 + 3) * MM_TX * MM_PW +
           sizeof(unsigned) * (size_t)(TY / 2 + 2) * MM_TX * MM_QW + 96 * sizeof(double);
}

// The value of real rank `rho` (1-based, among the window's taps inside the block) when the key at that rank has the
// quantised value Q: every tap below the cell ranks below it, so the answer is the (rho - #below)-th smallest double of the
// cell.  (x0, r0): halo coordinates of the window's first tap; Dh: the tile's halo values, [ROWS][HX].
__device__ __noinline__ double mm_exact_rank(const unsigned *__restrict__ Kh, const double *__restrict__ Dh, int x0, int r0, unsigned Q, int rho) {
    int below = 0, g = 0;
    double dmin = INFINITY, dmax = -INFINITY;
    for (int r = 0; r < 9; ++r)
        for (int c = 0; c < 9; ++c) {
            const unsigned key = Kh[(r0 + r) * MM_HX + x0 + c];
            if (key == MM_LOW || key == MM_HIGH) continue;
            const unsigned q = key >> 8;
            below += (q < Q) ? 1 : 0;
            if (q == Q) {
                const double d = Dh[(r0 + r) * MM_HX + x0 + c];
                ++g;
                dmin = d < dmin ? d : dmin;
                dmax = d > dmax ? d : dmax;
            }
        }
    if (dmin == dmax) return dmin;
    const int t = rho - below;   // 1 .. g
    double ans = dmin;
    for (int r = 0; r < 9; ++r)       // distinct doubles in one cell (rare): rank each member among the members
        for (int c = 0; c < 9; ++c) {
            const unsigned key = Kh[(r0 + r) * MM_HX + x0 + c];
            if (key == MM_LOW || key == MM_HIGH || (key >> 8) != Q) continue;
            const double d = Dh[(r0 + r) * MM_HX + x0 + c];
            int lt = 0, eq = 0;
            for (int r2 = 0; r2 < 9; ++r2)
                for (int c2 = 0; c2 < 9; ++c2) {
                    const unsigned k2 = Kh[(r0 + r2) * MM_HX + x0 + c2];
                    if (k2 == MM_LOW || k2 == MM_HIGH || (k2 >> 8) != Q) continue;
                    const double d2 = Dh[(r0 + r2) * MM_HX + x0 + c2];
                    lt += (d2 < d) ? 1 : 0;
                    eq += (d2 == d) ? 1 : 0;
                }
            if (lt < t && t <= lt + eq) ans = d;
        }
    return ans;
}

// the double behind a key of the window whose first tap is (x0, r0): the tag holds the tap's halo coordinates mod 16
__device__ __forceinline__ double mm_value_of(const double *Dh, unsigned key, int x0, int r0) {
    const int tx = (int)((key >> 4) & 15u), ty = (int)(key & 15u);
    const int hx = x0 + ((tx - x0) & 15), r = r0 + ((ty - r0) & 15);
    return Dh[r * MM_HX + hx];
}

template <int MM_TY, int MM_NW, int MINB>
__global__ void __launch_bounds__(MM_NW * 32, MINB) median_filter_merge_kernel(const MfParams p) {
    constexpr int MM_ROWS = MM_TY + 10, MM_NT = MM_NW * 32, MM_NP = MM_TY / 2 + 3, MM_NQ = MM_TY / 2 + 2;
    extern __shared__ __align__(16) unsigned char mf_smem[];
    double *Dh = reinterpret_cast<double *>(mf_smem);                         // [ROWS][HX] values (0 outside the block)
    double *redd = Dh + MM_ROWS * MM_HX;                                      // [96] flags
    unsigned *Kh = reinterpret_cast<unsigned *>(redd + 96);                   // [ROWS][HX] keys
    unsigned *Rs = Kh + MM_ROWS * MM_HX;                                      // [ROWS][9][TX] sorted runs
    unsigned *Ps = Rs + (size_t)MM_ROWS * 9 * MM_TX;                          // [NP][TX][PW]
    unsigned *Qs = Ps + (size_t)MM_NP * MM_TX * MM_PW;                        // [NQ][TX][QW]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const MfTile gt = p.gene_tiles[blockIdx.y];
    const MfTile ct = p.cell_tiles[blockIdx.x];
    const int hi0 = gt.start - 4, hj0 = ct.start - 5;   // halo (hx, r) = gene hi0 + hx, list position hj0 + r
    // ---- S0: halo and keys in one pass.  The keys quantise over the MATRIX' range (found by mf_range_kernel before the launch),
    //      so no tile reduction is needed; lanes cover 32 genes of a row, the 8 genes left of four rows share one more step.
    bool bad = false, dirty = false;
    const double vmin = p.vmin, M = p.mode;
    const double QMAX = 16777213.0;   // quantised values 1 .. 2^24 - 2: strictly between the two padding keys
    const double scale = p.scale;     // QMAX / (vmax - vmin), 0 for a constant matrix (set by the launcher)
    auto quant = [&](double v) -> unsigned {
        double qd = (v - vmin) * scale;
        qd = qd < QMAX ? qd : QMAX;       // (also maps NaN to QMAX)
        qd = qd > 0.0 ? qd : 0.0;
        return 1u + __double2uint_rd(qd);
    };
    // The matrices this filter sees hold ONE value many times over (exactly 1 after the dead-band subtraction and 2^x, the
    // reference mean after de-noising): M, picked by the host from a sample.  A tile whose key cell of M holds nothing but
    // copies of M ("clean") can answer every median that falls into that cell with M, however many ties surround it.
    const unsigned qM = quant(M);
    int *flags = reinterpret_cast<int *>(redd);
    if (tid == 0) flags[0] = 0;
    // a tap's value -> its key and the two halo arrays
    auto put = [&](int r, int hx, bool in, double v) {
        unsigned key = ((hx + r) & 1) ? MM_HIGH : MM_LOW;
        if (in) {
            bad |= !is_finite_d(v);
            const unsigned q = quant(v);
            dirty |= (q == qM) && (v != M);
            key = (q << 8) | (unsigned)((hx & 15) << 4) | (unsigned)(r & 15);
        }
        Dh[r * MM_HX + hx] = in ? v : 0.0;
        Kh[r * MM_HX + hx] = key;
    };
    // every global load of the tile is issued before the first one is used: first the column offsets (G * cell, a table the
    // launcher builds beside the index lists) of this warp's rows and of the four rows whose last 8 genes it takes, then the
    // values - two dependent memory latencies per tile, not two per row
    constexpr int RPW = (MM_ROWS + MM_NW - 1) / MM_NW;          // rows per warp
    constexpr int TPW = (MM_ROWS + 4 * MM_NW - 1) / (4 * MM_NW);  // groups of four row tails per warp
    long long rb[RPW + TPW];
    bool rin[RPW + TPW];
#pragma unroll
    for (int i = 0; i < RPW + TPW; ++i) {
        const int r = i < RPW ? warp + i * MM_NW : 4 * (warp + (i - RPW) * MM_NW) + (lane >> 3);
        const int jj = hj0 + r;
        rin[i] = r < MM_ROWS && jj >= ct.lo && jj < ct.hi && r >= 1 && r <= MM_TY + 8;
        rb[i] = rin[i] ? p.coloff[jj] : 0ll;
    }
    double tv[RPW + TPW];
#pragma unroll
    for (int i = 0; i < RPW + TPW; ++i) {
        const int hx = i < RPW ? lane : 32 + (lane & 7);
        const int ii = hi0 + hx;
        rin[i] = rin[i] && ii >= gt.lo && ii < gt.hi;
        tv[i] = rin[i] ? p.X[ii + rb[i]] : 0.0;
    }
#pragma unroll
    for (int i = 0; i < RPW + TPW; ++i) {
        const int r = i < RPW ? warp + i * MM_NW : 4 * (warp + (i - RPW) * MM_NW) + (lane >> 3);
        const int hx = i < RPW ? lane : 32 + (lane & 7);
        if (r < MM_ROWS) put(r, hx, rin[i], tv[i]);
    }
    __syncthreads();
    if (dirty) flags[0] = 1;
    __syncthreads();
    const bool mode_clean = flags[0] == 0 && (M == M);
    // ---- S1: sorted runs, pairs ----------------------------------------------------------------------------------------------
    for (int t = warp; t <= MM_TY / 2 + 4; t += MM_NW) {      // rows 2t, 2t+1
        unsigned ra[9], rb[9];
        const int r0 = 2 * t, r1 = 2 * t + 1;
        const bool ok0 = r0 >= 1 && r0 <= MM_TY + 8, ok1 = r1 >= 1 && r1 <= MM_TY + 8;
        if (ok0) {
            unsigned k[9];
#pragma unroll
            for (int i = 0; i < 9; ++i) k[i] = Kh[r0 * MM_HX + lane + i];
            MF_SORT9(k, ra);
#pragma unroll
            for (int i = 0; i < 9; ++i) Rs[(r0 * 9 + i) * MM_TX + lane] = ra[i];
        }
        if (ok1) {
            unsigned k[9];
#pragma unroll
            for (int i = 0; i < 9; ++i) k[i] = Kh[r1 * MM_HX + lane + i];
            MF_SORT9(k, rb);
#pragma unroll
            for (int i = 0; i < 9; ++i) Rs[(r1 * 9 + i) * MM_TX + lane] = rb[i];
        }
        if (t >= 1 && t <= MM_NP) {      // P[t-1] = rows (2t, 2t+1), both inside 2 .. TY+7
            unsigned o[MM_PW];
            MF_MERGE9(ra, rb, o);
            o[18] = 0u;
            o[19] = 0u;
            uint4 *dst = reinterpret_cast<uint4 *>(Ps + ((size_t)(t - 1) * MM_TX + lane) * MM_PW);
#pragma unroll
            for (int i = 0; i < MM_PW / 4; ++i) dst[i] = make_uint4(o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
        }
    }
    __syncthreads();
    // ---- S2: Q[q] = P[q] + P[q+1] (rows 2q+2 .. 2q+5) --------------------------------------------------------------------
    for (int q = warp; q < MM_NQ; q += MM_NW) {
        unsigned a[MM_PW], b[MM_PW], o[MM_QW];
        const uint4 *sa = reinterpret_cast<const uint4 *>(Ps + ((size_t)q * MM_TX + lane) * MM_PW);
        const uint4 *sb = reinterpret_cast<const uint4 *>(Ps + ((size_t)(q + 1) * MM_TX + lane) * MM_PW);
#pragma unroll
        for (int i = 0; i < MM_PW / 4; ++i) {
            const uint4 va = sa[i], vb = sb[i];
            a[4 * i] = va.x; a[4 * i + 1] = va.y; a[4 * i + 2] = va.z; a[4 * i + 3] = va.w;
            b[4 * i] = vb.x; b[4 * i + 1] = vb.y; b[4 * i + 2] = vb.z; b[4 * i + 3] = vb.w;
        }
        MF_MERGE18(a, b, o);
        uint4 *dst = reinterpret_cast<uint4 *>(Qs + ((size_t)q * MM_TX + lane) * MM_QW);
#pragma unroll
        for (int i = 0; i < MM_QW / 4; ++i) dst[i] = make_uint4(o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
    }
    __syncthreads();
    // ---- S3: per pair of outputs (2j, 2j+1): core = Q[j] + Q[j+2] (rows 2j+2 .. 2j+9), + row 2j+1 resp. 2j+10 ----------------
    for (int j = warp; j < MM_TY / 2; j += MM_NW) {
        long long ycol[2];   // column offsets of the two outputs, fetched now, needed at the end of the task
#pragma unroll
        for (int half = 0; half < 2; ++half) ycol[half] = (2 * j + half < ct.len) ? p.coloff[ct.start + 2 * j + half] : 0ll;
        unsigned core[14];
        {
            unsigned a[MM_QW], b[MM_QW];
            const uint4 *sa = reinterpret_cast<const uint4 *>(Qs + ((size_t)j * MM_TX + lane) * MM_QW);
            const uint4 *sb = reinterpret_cast<const uint4 *>(Qs + ((size_t)(j + 2) * MM_TX + lane) * MM_QW);
#pragma unroll
            for (int i = 0; i < MM_QW / 4; ++i) {
                const uint4 va = sa[i], vb = sb[i];
                a[4 * i] = va.x; a[4 * i + 1] = va.y; a[4 * i + 2] = va.z; a[4 * i + 3] = va.w;
                b[4 * i] = vb.x; b[4 * i + 1] = vb.y; b[4 * i + 2] = vb.z; b[4 * i + 3] = vb.w;
            }
            MF_CORE(a, b, core);
        }
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int y = 2 * j + half;                       // output row of the tile; its window: rows y+1 .. y+9
            const int rex = half == 0 ? 2 * j + 1 : 2 * j + 10;
            unsigned e[9], s[5];
#pragma unroll
            for (int i = 0; i < 9; ++i) e[i] = Rs[(rex * 9 + i) * MM_TX + lane];
            MF_SELECT(core, e, s);                            // ranks 39 .. 43 of the window's 81 keys
            if (lane < gt.len && y < ct.len) {
                const int i = gt.start + lane, jpos = ct.start + y;
                const int xa = max(gt.lo, i - 4), xb = min(gt.hi - 1, i + 4);
                const int ya = max(ct.lo, jpos - 4), yb = min(ct.hi - 1, jpos + 4);
                const int n = (xb - xa + 1) * (yb - ya + 1);
                // padding keys of the window: a checkerboard, LOW where (hx + r) is even
                const int w_low = ((lane + y + 1) & 1) ? 40 : 41;
                const int in_low = (n + ((((xa - hi0) + (ya - hj0)) & 1) ? 0 : 1)) >> 1;
                const int L = w_low - in_low;
                const int rho = (n + 1) >> 1;                 // lower middle rank among the window's taps
                const int k = rho + L;                        // its rank among the 81 keys: 40, 41 or 42
                const bool even = (n & 1) == 0;
                const int x0 = lane, r0 = y + 1;
                // the value of the key at index ki of s[] (rank 39 + ki), real rank rk: its tap when no rank neighbour shares its
                // key cell; when the whole cell lies inside ranks 40..42 its (at most 3) doubles are read and ordered here;
                // M when the cell is the tile's clean dominant one; the exact-rank scan otherwise
                auto value_at = [&](int ki, int rk) -> double {
                    const unsigned Qc = s[ki] >> 8;
                    const bool tl = (s[ki - 1] >> 8) == Qc, th = (s[ki + 1] >> 8) == Qc;
                    if (!tl && !th) return mm_value_of(Dh, s[ki], x0, r0);
                    if (Qc == qM && mode_clean) return M;
                    int lo = ki, hi = ki;
                    while (lo > 0 && (s[lo - 1] >> 8) == Qc) --lo;
                    while (hi < 4 && (s[hi + 1] >> 8) == Qc) ++hi;
                    if (lo == 0 || hi == 4 || hi - lo > 2) return mm_exact_rank(Kh, Dh, x0, r0, Qc, rk);
                    double d0 = mm_value_of(Dh, s[lo], x0, r0), d1 = mm_value_of(Dh, s[lo + 1], x0, r0);
                    double d2 = (hi - lo == 2) ? mm_value_of(Dh, s[lo + 2], x0, r0) : INFINITY;
                    mf_cswap(d0, d1);
                    mf_cswap(d1, d2);
                    mf_cswap(d0, d1);
                    const int t = ki - lo;
                    return t == 0 ? d0 : (t == 1 ? d1 : d2);
                };
                const double v1 = value_at(k - 39, rho);
                double med = v1;
                if (even) med = (v1 + value_at(k - 38, rho + 1)) * 0.5;
                p.Y[i + ycol[half]] = med;
            }
        }
    }
    if (bad && p.err_flag) atomicExch(p.err_flag, 1);
}

static void make_tiles(const int32_t *start, const int32_t *len, int nblk, int T, std::vector<MfTile> &out) {
    for (int b = 0; b < nblk; ++b) {
        int lo = start[b], hi = start[b] + len[b];
        for (int s = lo; s < hi; s += T) out.push_back(MfTile{s, (hi - s < T ? hi - s : T), lo, hi});
    }
}

}  // namespace icnv

using namespace icnv;

extern "C" int icnv_dev_median_filter_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *chr_start,
                                          const int32_t *chr_len, int K, const int32_t *grp_off, const int32_t *grp_idx,
                                          int n_grp, int window_size, void *stream) {
    ICNV_REQUIRE_READY();
    Ctx &c = ctx();
    if (!X || !Y || X == Y || G <= 0 || C <= 0 || !chr_start || !chr_len || K <= 0 || n_grp < 0)
        return set_error(ICNV_E_BAD_ARG, "icnv_dev_median_filter_f64: bad argument (X and Y must not alias)");
    if (window_size < 3 || (window_size & 1) == 0)
        return set_error(ICNV_E_BAD_ARG, "window_size must be an odd number >= 3 (noise_reduction.R:48-50)");
    const int r = (window_size + 1) / 2;
    const int W = (2 * r + 1) * (2 * r + 1);
    // window_size 7 (radius 4): the shared-merge kernel, tiles of 12 list positions, two 256-thread CTAs per SM; the other
    // windows up to radius 5: the counting selection; larger ones: the generic kernel
    constexpr int mm_ty = 12, mm_nw = 8;
    const bool merge_kernel = r == 4;
    const bool select_kernel = !merge_kernel && r >= 2 && r <= 5;
    const int TI = merge_kernel ? MM_TX : (select_kernel ? MS_TI : MF_TI), TJ = merge_kernel ? mm_ty : (select_kernel ? MS_TJ : MF_TJ);
    const int NT = merge_kernel ? mm_nw * 32 : TI * TJ;
    const size_t smem = merge_kernel ? mm_smem_bytes(mm_ty)
                                     : sizeof(double) * (size_t)(TI + 2 * r) * (size_t)(TJ + 2 * r) * (select_kernel ? 2 : 1) +
                                           sizeof(unsigned short) * (size_t)W * (size_t)NT;
    if (smem > (size_t)c.smem_optin || (TI + 2 * r) * (TJ + 2 * r) > 65535)
        return set_error(ICNV_E_UNSUPPORTED, "window_size %d needs %zu B of shared memory per CTA", window_size, smem);
    cudaStream_t st = pick_stream(stream);
    // cells in no list and genes on no chromosome are copied through - one pass over the matrix that is skipped when the
    // lists and the chromosomes cover everything (the usual call: every cell belongs to one group or subcluster)
    bool covered = n_grp > 0;
    {
        int64_t g_cov = 0;
        for (int k = 0; k < K; ++k) g_cov += chr_len[k] > 0 ? chr_len[k] : 0;
        covered = covered && g_cov >= G && grp_off[n_grp] >= C;
        if (covered) {
            std::vector<unsigned char> seen((size_t)C, 0);
            int64_t n_seen = 0;
            for (int64_t i = 0; i < grp_off[n_grp]; ++i) {
                const int32_t cell = grp_idx[i];
                if (cell >= 0 && cell < C && !seen[(size_t)cell]) {
                    seen[(size_t)cell] = 1;
                    ++n_seen;
                }
            }
            covered = n_seen == C;
            std::vector<unsigned char> gseen((size_t)G, 0);   // chromosomes may overlap or leave gaps in a hand-made layout
            int64_t n_g = 0;
            for (int k = 0; k < K; ++k)
                for (int64_t g = chr_start[k]; g < (int64_t)chr_start[k] + chr_len[k]; ++g)
                    if (g >= 0 && g < G && !gseen[(size_t)g]) {
                        gseen[(size_t)g] = 1;
                        ++n_g;
                    }
            covered = covered && n_g == G;
        }
    }
    if (!covered) ICNV_CUDA(cudaMemcpyAsync(Y, X, sizeof(double) * (size_t)(G * C), cudaMemcpyDeviceToDevice, st));
    if (n_grp == 0) return ICNV_OK;
    std::vector<MfTile> gt, ct;
    make_tiles(chr_start, chr_len, K, TI, gt);
    std::vector<int32_t> g_start(n_grp), g_len(n_grp);
    for (int b = 0; b < n_grp; ++b) {
        g_start[b] = grp_off[b];
        g_len[b] = grp_off[b + 1] - grp_off[b];
    }
    make_tiles(g_start.data(), g_len.data(), n_grp, TJ, ct);
    if (gt.empty() || ct.empty()) return ICNV_OK;
    if (gt.size() > 65535) return set_error(ICNV_E_UNSUPPORTED, "too many gene tiles (%zu)", gt.size());
    const int64_t n_idx = grp_off[n_grp];
    size_t bytes = sizeof(MfTile) * (gt.size() + ct.size()) + sizeof(int32_t) * (size_t)n_idx + 64 +
                   (merge_kernel ? sizeof(long long) * (size_t)n_idx + 16 : 0);
    char *d = (char *)scratch(SLOT_MF, bytes);
    int *d_flag = (int *)scratch(SLOT_MISC, 64);
    if (!d || !d_flag) return ICNV_E_NOMEM;
    MfTile *d_gt = (MfTile *)d;
    MfTile *d_ct = d_gt + gt.size();
    int32_t *d_cells = (int32_t *)(d_ct + ct.size());
    ICNV_CUDA(cudaMemcpyAsync(d_gt, gt.data(), sizeof(MfTile) * gt.size(), cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaMemcpyAsync(d_ct, ct.data(), sizeof(MfTile) * ct.size(), cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaMemcpyAsync(d_cells, grp_idx, sizeof(int32_t) * (size_t)n_idx, cudaMemcpyHostToDevice, st));
    std::vector<long long> coloff;
    long long *d_coloff = nullptr;
    if (merge_kernel) {   // column offsets G * cell beside the lists: one 8-byte load per halo row instead of index + multiply
        coloff.resize((size_t)n_idx);
        for (int64_t i = 0; i < n_idx; ++i) coloff[(size_t)i] = (long long)G * (long long)grp_idx[i];
        d_coloff = reinterpret_cast<long long *>((reinterpret_cast<uintptr_t>(d_cells + n_idx) + 15) & ~(uintptr_t)15);
        ICNV_CUDA(cudaMemcpyAsync(d_coloff, coloff.data(), sizeof(long long) * (size_t)n_idx, cudaMemcpyHostToDevice, st));
    }
    ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
    ICNV_CUDA(cudaStreamSynchronize(st));  // tile tables are stack-lifetime host buffers
    MfParams p{X, Y, G, d_cells, d_gt, d_ct, r, d_flag, 0.0, 0.0, 0.0, 0.0, d_coloff};
    if (merge_kernel) {
        // range of the matrix + a sample of its values (the dominant value is the most frequent one of the sample, if any
        // value takes >= 0.5 % of it)
        constexpr int NS = 4096;
        char *d_pre = (char *)scratch(SLOT_MF_PRE, 16 + sizeof(double) * NS);
        if (!d_pre) return ICNV_E_NOMEM;
        unsigned long long h_range[2] = {~0ull, 0ull};
        ICNV_CUDA(cudaMemcpyAsync(d_pre, h_range, sizeof(h_range), cudaMemcpyHostToDevice, st));
        mf_range_kernel<<<(unsigned)(c.sm_count * 8), 256, 0, st>>>(X, G * C, (unsigned long long *)d_pre, (double *)(d_pre + 16), NS);
        ICNV_CHECK_LAUNCH("mf_range_kernel");
        std::vector<double> smp((size_t)NS);
        ICNV_CUDA(cudaMemcpyAsync(h_range, d_pre, sizeof(h_range), cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaMemcpyAsync(smp.data(), d_pre + 16, sizeof(double) * NS, cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        auto unkey = [](unsigned long long k) {
            unsigned long long u = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
            double d;
            memcpy(&d, &u, 8);
            return d;
        };
        p.vmin = h_range[0] <= h_range[1] ? unkey(h_range[0]) : 0.0;
        p.vmax = h_range[0] <= h_range[1] ? unkey(h_range[1]) : 0.0;
        std::sort(smp.begin(), smp.end(), [](double a, double b) {   // bitwise order: NaNs and -0 / +0 stay apart, runs are exact copies
            long long x, y;
            memcpy(&x, &a, 8);
            memcpy(&y, &b, 8);
            return x < y;
        });
        int best_n = 0;
        double best_v = NAN;
        for (int i = 0; i < NS;) {
            int j = i + 1;
            while (j < NS && memcmp(&smp[(size_t)i], &smp[(size_t)j], 8) == 0) ++j;
            if (j - i > best_n) {
                best_n = j - i;
                best_v = smp[(size_t)i];
            }
            i = j;
        }
        p.mode = (best_n >= NS / 200 && std::isfinite(best_v)) ? best_v : NAN;
        p.scale = (p.vmax > p.vmin) ? 16777213.0 / (p.vmax - p.vmin) : 0.0;
    }
    dim3 grid((unsigned)ct.size(), (unsigned)gt.size());
    auto launch = [&](auto kern) -> int {
        ICNV_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, NT, smem, st>>>(p);
        return ICNV_OK;
    };
    int lrc;
    if (merge_kernel) lrc = launch(median_filter_merge_kernel<mm_ty, mm_nw, 2>);
    else if (!select_kernel) lrc = launch(median_filter_kernel);
    else if (r == 2) lrc = launch(median_filter_select_kernel<2>);
    else if (r == 3) lrc = launch(median_filter_select_kernel<3>);
    else lrc = launch(median_filter_select_kernel<5>);
    if (lrc) return lrc;
    ICNV_CHECK_LAUNCH("median_filter_kernel");
    return ICNV_OK;
}
