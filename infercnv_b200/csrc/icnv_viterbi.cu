// icnv_viterbi.cu - K3: the i6 / i3 HMM of inferCNV as an sm_90a kernel.
//
// Restates Viterbi.dthmm.adj (R/inferCNV_HMM.R:1101-1176) for every (cell-or-group, chromosome)
// sequence at once.  One thread owns one sequence; the 32 lanes of a warp are 32 consecutive
// cells on the SAME chromosome, so the lanes run the same trip count and never diverge on length.
// The m-state trellis row, the running path margins and the emission work all live in registers;
// mean / log Pi / log delta sit in the kernel-parameter constant bank (warp-uniform operands).
// Backpointers (3 bits per state, one 32-bit word per gene) go to a per-warp scratch ring laid out
// [gene][lane], i.e. one coalesced 128-byte line per gene, sized for the longest chromosome and
// re-used for every work item, so its lines are written to and read back from L2.
//
// Arithmetic: "exact" mode follows the reference's operation order in IEEE double without FMA
// contraction (explicit __dmul_rn/__dadd_rn/__ddiv_rn), including nmath's pnorm_both
// (Cody 1969) for pnorm(log.p=TRUE, lower.tail=FALSE) at HMM.R:1129,1156.  What can still differ
// from R on x86-64 by an ulp: log() (CUDA vs glibc) and sum() (R accumulates in long double).
// State calls only change if an arg-max is decided by less than that, which the per-sequence
// margin output makes checkable.
//
// This kernel is FP64-pipe bound (6 pnorm + 12 divisions + 12 logs per cell-gene against 9 bytes
// of HBM traffic); see DESIGN.md for the roofline discussion.
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>
#include <algorithm>

#include "icnv_common.cuh"

namespace icnv {

constexpr int MAXM = 6;

struct VitParams {
    const double *X;
    int64_t G, C;
    const int32_t *item_chr_start;  // per sorted chromosome
    const int32_t *item_chr_len;
    int K;
    int64_t n_tiles;   // ceil(C / 32)
    int64_t n_items;   // K * n_tiles
    int max_len;
    double logPi[MAXM * MAXM];  // [j*M + k] = log P(j -> k)
    double logdelta[MAXM];
    double mean[MAXM];
    double sd;             // median of the state sds (HMM.R:1122)
    const double *sd_col;  // optional per-column median sd (group modes)
    uint8_t *states;
    double *margins;   // K x C (original chromosome order) or nullptr
    const int32_t *item_chr_id;  // original chromosome index of each sorted chromosome
    uint32_t *bp;      // n_warps * max_len * 32 words
    unsigned long long *counter;
    int *err_flag;     // bit 0: non-finite input, bit 1: underflow
    // list mode (exact re-run of the sequences the fast path could not certify): item q is the
    // single sequence (chromosome list[q].x in ORIGINAL order, cell list[q].y), handled by lane 0.
    const int2 *list;
    const unsigned int *list_count;
    const int32_t *chr_start_orig;  // original-order chromosome tables (list mode)
    const int32_t *chr_len_orig;
    // certified fast path
    double a_diag, b_off;      // log Pi diagonal / off-diagonal (all equal)
    double cmove;              // a_diag - b_off: what moving costs against staying
    int near_hi;               // high word of cmove - tau (the fast kernel's near-best check)
    double inv_sd;             // 1 / median sd
    double emis_scale;         // 16 / sd and -mean_k * 16 / sd for the launch-wide sd (the fast kernel's table argument)
    double emis_nms[MAXM];
    double tau;                // decision-margin threshold below which a sequence is re-run exactly
    const double *table;       // device copy of icnv_emis_table
    int means_monotone;        // state means sorted (either direction): the furthest state from any x is an end state
    int2 *list_out;
    unsigned int *list_out_count;
    unsigned int list_cap;
};

// ---- nmath pnorm_both, upper tail, log.p, argument y >= 0 (Cody 1969) -------------------------------
__device__ __forceinline__ double pnorm_upper_log_exact(double y) {
    const double a0 = 2.2352520354606839287, a1 = 161.02823106855587881, a2 = 1067.6894854603709582,
                 a3 = 18154.981253343561249, a4 = 0.065682337918207449113;
    const double b0 = 47.20258190468824187, b1 = 976.09855173777669322, b2 = 10260.932208618978205,
                 b3 = 45507.789335026729956;
    const double c0 = 0.39894151208813466764, c1 = 8.8831497943883759412, c2 = 93.506656132177855979,
                 c3 = 597.27027639480026226, c4 = 2494.5375852903726711, c5 = 6848.1904505362823326,
                 c6 = 11602.651437647350124, c7 = 9842.7148383839780218, c8 = 1.0765576773720192317e-8;
    const double d0 = 22.266688044328115691, d1 = 235.38790178262499861, d2 = 1519.377599407554805,
                 d3 = 6485.558298266760755, d4 = 18615.571640885098091, d5 = 34900.952721145977266,
                 d6 = 38912.003286093271411, d7 = 19685.429676859990727;
    const double p0 = 0.21589853405795699, p1 = 0.1274011611602473639, p2 = 0.022235277870649807,
                 p3 = 0.001421619193227893466, p4 = 2.9112874951168792e-5, p5 = 0.02307344176494017303;
    const double q0 = 1.28426009614491121, q1 = 0.468238212480865118, q2 = 0.0659881378689285515,
                 q3 = 0.00378239633202758244, q4 = 7.29751555083966205e-5;
    const double SQRT32 = 5.656854249492380195206754896838;
    const double INV_SQRT_2PI = 0.398942280401432677939946059934;
#define M_(a, b) __dmul_rn((a), (b))
#define A_(a, b) __dadd_rn((a), (b))
#define D_(a, b) __ddiv_rn((a), (b))
    double arg, A = 0.0;
    bool central = false;
    if (y <= 0.67448975) {
        double xnum = 0.0, xden = 0.0;
        if (y > DBL_EPSILON * 0.5) {
            double xsq = M_(y, y);
            xnum = M_(a4, xsq);
            xden = xsq;
            xnum = M_(A_(xnum, a0), xsq);
            xden = M_(A_(xden, b0), xsq);
            xnum = M_(A_(xnum, a1), xsq);
            xden = M_(A_(xden, b1), xsq);
            xnum = M_(A_(xnum, a2), xsq);
            xden = M_(A_(xden, b2), xsq);
        }
        double temp = D_(M_(y, A_(xnum, a3)), A_(xden, b3));
        arg = A_(0.5, -temp);
        central = true;
    } else if (y <= SQRT32) {
        double xnum = M_(c8, y), xden = y;
        xnum = M_(A_(xnum, c0), y);
        xden = M_(A_(xden, d0), y);
        xnum = M_(A_(xnum, c1), y);
        xden = M_(A_(xden, d1), y);
        xnum = M_(A_(xnum, c2), y);
        xden = M_(A_(xden, d2), y);
        xnum = M_(A_(xnum, c3), y);
        xden = M_(A_(xden, d3), y);
        xnum = M_(A_(xnum, c4), y);
        xden = M_(A_(xden, d4), y);
        xnum = M_(A_(xnum, c5), y);
        xden = M_(A_(xden, d5), y);
        xnum = M_(A_(xnum, c6), y);
        xden = M_(A_(xden, d6), y);
        arg = D_(A_(xnum, c7), A_(xden, d7));
        double xsq = trunc(M_(y, 16.0)) * 0.0625;
        double del = M_(A_(y, -xsq), A_(y, xsq));
        A = A_(M_(M_(-xsq, xsq), 0.5), M_(-del, 0.5));
    } else if (y < 1e170) {
        double xsq = D_(1.0, M_(y, y));
        double xnum = M_(p5, xsq), xden = xsq;
        xnum = M_(A_(xnum, p0), xsq);
        xden = M_(A_(xden, q0), xsq);
        xnum = M_(A_(xnum, p1), xsq);
        xden = M_(A_(xden, q1), xsq);
        xnum = M_(A_(xnum, p2), xsq);
        xden = M_(A_(xden, q2), xsq);
        xnum = M_(A_(xnum, p3), xsq);
        xden = M_(A_(xden, q3), xsq);
        double temp = D_(M_(xsq, A_(xnum, p4)), A_(xden, q4));
        arg = D_(A_(INV_SQRT_2PI, -temp), y);
        double xs = trunc(M_(y, 16.0)) * 0.0625;
        double del = M_(A_(y, -xs), A_(y, xs));
        A = A_(M_(M_(-xs, xs), 0.5), M_(-del, 0.5));
    } else {
        return -INFINITY;
    }
    double r = log(arg);
    return central ? r : A_(A, r);
#undef M_
#undef A_
#undef D_
}

// log emission of every state for one observation, HMM.R:1129-1133 / 1156-1160
template <int M>
__device__ __forceinline__ void emission_exact(double x, const double (&mean)[MAXM], double sd, double (&le)[MAXM]) {
    double e[M];
#pragma unroll
    for (int k = 0; k < M; ++k) {
        double z = __ddiv_rn(fabs(__dadd_rn(x, -mean[k])), sd);
        double lq = pnorm_upper_log_exact(z);
        e[k] = __ddiv_rn(1.0, -lq);  // 1 / (-1 * emission)
    }
    double s = e[0];
#pragma unroll
    for (int k = 1; k < M; ++k) s = __dadd_rn(s, e[k]);
#pragma unroll
    for (int k = 0; k < M; ++k) le[k] = log(__ddiv_rn(e[k], s));
}

template <int M, bool MARGIN>
__global__ void __launch_bounds__(128) viterbi_kernel(const VitParams p) {
    const int lane = threadIdx.x & 31;
    const int64_t warp_global = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    uint32_t *__restrict__ bp = p.bp + warp_global * (int64_t)p.max_len * 32;
    int err = 0;

    const int64_t n_items = p.list ? (int64_t)min(*p.list_count, p.list_cap) : p.n_items;
    for (;;) {
        unsigned long long item = 0;
        if (lane == 0) item = atomicAdd(p.counter, 1ull);
        item = __shfl_sync(0xffffffffu, item, 0);
        if ((int64_t)item >= n_items) break;
        int ks, cs, n;
        int64_t c;
        bool active;
        if (p.list) {
            const int2 e = p.list[item];
            ks = e.x;
            cs = p.chr_start_orig[ks];
            n = p.chr_len_orig[ks];
            c = e.y;
            active = lane == 0;
        } else {
            ks = (int)(item / (unsigned long long)p.n_tiles);   // sorted chromosome (longest first)
            const int64_t tile = (int64_t)(item % (unsigned long long)p.n_tiles);
            cs = p.item_chr_start[ks];
            n = p.item_chr_len[ks];
            c = tile * 32 + lane;
            active = c < p.C;
        }
        const int64_t cc = (c < p.C) ? c : (p.C - 1);  // idle lanes shadow a valid cell, stores masked
        const double *__restrict__ xcol = p.X + p.G * cc + cs;
        uint8_t *__restrict__ scol = p.states + p.G * cc + cs;
        if (n < 2) {  // HMM.R:1104-1107: not enough to run a trace on -> state 3
            if (active && n == 1) scol[0] = 3;
            if (MARGIN && active && p.margins) p.margins[(p.list ? ks : p.item_chr_id[ks]) + (int64_t)p.K * c] = INFINITY;
            continue;
        }
        const double sd = p.sd_col ? p.sd_col[cc] : p.sd;

        double nu[MAXM], mg[MAXM], le[MAXM];
        // ---- forward ---------------------------------------------------------------------------------
        {
            double x = xcol[0];
            if (!is_finite_d(x)) err |= 1;
            emission_exact<M>(x, p.mean, sd, le);
#pragma unroll
            for (int k = 0; k < M; ++k) {
                nu[k] = __dadd_rn(p.logdelta[k], le[k]);
                mg[k] = INFINITY;
            }
        }
        double xnext = xcol[1];
        for (int i = 1; i < n; ++i) {
            double x = xnext;
            if (i + 1 < n) xnext = xcol[i + 1];
            if (!is_finite_d(x)) err |= 1;
            emission_exact<M>(x, p.mean, sd, le);
            double nn[MAXM], mgn[MAXM];
            uint32_t word = 0;
#pragma unroll
            for (int k = 0; k < M; ++k) {
                // max_j(nu[j] + logPi[j,k]) with which.max's first-index tie rule (HMM.R:1162,1173)
                double best = __dadd_rn(nu[0], p.logPi[0 * M + k]);
                double second = -INFINITY;
                int arg = 0;
                double mga = mg[0];
#pragma unroll
                for (int j = 1; j < M; ++j) {
                    double v = __dadd_rn(nu[j], p.logPi[j * M + k]);
                    if (v > best) {
                        second = best;
                        best = v;
                        arg = j;
                        if (MARGIN) mga = mg[j];
                    } else if (MARGIN && v > second) {
                        second = v;
                    }
                }
                nn[k] = __dadd_rn(best, le[k]);
                word |= (uint32_t)arg << (3 * k);
                if (MARGIN) mgn[k] = fmin(mga, best - second);
            }
#pragma unroll
            for (int k = 0; k < M; ++k) {
                nu[k] = nn[k];
                if (MARGIN) mg[k] = mgn[k];
            }
            bp[(int64_t)i * 32 + lane] = word;
        }
        // ---- termination: any(nu[n,] == -Inf) -> "Problems With Underflow" (HMM.R:1165) ---------
        int y = 0;
        {
            double best = nu[0], second = -INFINITY;
            bool under = (nu[0] == -INFINITY);
#pragma unroll
            for (int k = 1; k < M; ++k) {
                under |= (nu[k] == -INFINITY);
                if (nu[k] > best) {
                    second = best;
                    best = nu[k];
                    y = k;
                } else if (nu[k] > second) {
                    second = nu[k];
                }
            }
            if (under && active) err |= 2;
            if (MARGIN && active && p.margins) {
                double m = mg[0];
#pragma unroll
                for (int k = 1; k < M; ++k)
                    if (y == k) m = mg[k];
                p.margins[(p.list ? ks : p.item_chr_id[ks]) + (int64_t)p.K * c] = fmin(m, best - second);
            }
        }
        // ---- traceback: y[i] = which.max(logPi[, y[i+1]] + nu[i, ]) = stored first arg-max ------------
        if (active) scol[n - 1] = (uint8_t)(y + 1);
        for (int i = n - 1; i >= 1; --i) {
            uint32_t word = bp[(int64_t)i * 32 + lane];
            y = (int)((word >> (3 * y)) & 7u);
            if (active) scol[i - 1] = (uint8_t)(y + 1);
        }
        __syncwarp();
    }
    if (err && p.err_flag) atomicOr(p.err_flag, err);
}


// =================================================================================================
// certified fast path
// =================================================================================================
//
// Same recursion, two changes that cannot alter a state call without being noticed:
//  (1) emission.  log(e_k / sum_j e_j) = g(z_k) - log(sum_j e_j) with g(z) = -log(-log Q(z)).  The
//      second term is the same for every state of a gene, so it shifts all path scores equally and
//      no arg-max sees it: it is dropped.  g comes from a piecewise degree-4 table
//      (icnv_emission_table.inc, |error| < 4.5e-13 checked against 50-digit arithmetic, + < 4.8e-13 for keeping
//      the cubic / quartic coefficients to 20 mantissa bits, see the kernel); z beyond the
//      table falls back to the nmath evaluation.
//  (2) max_j(nu[j] + logPi[j,k]) uses the structure of .get_HMM's matrix (one diagonal value a,
//      one off-diagonal value b, R/inferCNV_HMM.R:233-238): the winner is either "stay" (nu[k]+a)
//      or the best state (+b), with which.max's first-index rule.  The scores are kept minus i * a
//      (a shift common to all states), so per gene nu'[k] = max(nu[k], best - cmove) + le[k], cmove = a - b.
// Certificate: every arg-max (all states, all genes, and the final one) records the gap between
// winner and runner-up; a sequence whose smallest gap exceeds tau = 2^-23 = 1.19e-7 has the same trace in both
// arithmetics, the others are appended to a list and recomputed by the exact kernel above (list mode); their count is
// reported.  Error budget, per gene and path, while every score is below 2^15 in magnitude (half an ulp <= 2^-38 = 3.6e-12;
// checked at the end of the sequence): this pass rounds twice (best - cmove, + le) and its emission is off by < 9.3e-13
// (table + shortened coefficients); the reference-order kernel rounds twice (nu + logPi, + le) and its emission is within
// a few ulp of |le| <= 6, < 1e-14; cmove itself is rounded once (< 7.2e-15 for cmove < 64).  Together < 1.6e-11 per gene, so
// the two arithmetics' scores of one path differ by < n * 1.6e-11, two paths' difference by twice that, and the rounded gap
// e adds 3.6e-12: for n <= FAST_MAX_N = 3600 genes that is < 1.16e-7 < tau.  The longest sequence of the benchmark's layouts
// (chromosome 1 at 20 000 genes, ~1 700 genes) stays below 5.5e-8.  Longer sequences go to the exact kernel.
#include "icnv_emission_table.inc"

constexpr int FAST_MAX_N = 3600;   // longest sequence the error budget above certifies
constexpr int TG = 8;        // genes per staged tile
constexpr int TS = TG + 1;   // padded row stride in doubles (bank-conflict-free column reads)
constexpr int FAST_WARPS = 16;   // warps per CTA (one CTA per SM: the replicated table below is shared by all of them)
constexpr int TAB_REP = 8;       // table replicas: lane l reads replica l & 7, so a 16-byte lookup never bank-conflicts

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

// |x - mean| / sd beyond the table (> 24): nmath evaluation, kept out of line (rare)
__device__ __noinline__ double emission_far(double x, double mean, double sd) {
    const double zz = __ddiv_rn(fabs(__dadd_rn(x, -mean)), sd);
    return -log(-pnorm_upper_log_exact(zz));
}

// acc += (v >= lim): a compare and a predicated add (the compiler's own form is compare, select 0 / 1, add)
__device__ __forceinline__ void count_if_ge(int &acc, int v, int lim) {
    asm("{ .reg .pred p; setp.ge.s32 p, %1, %2; @p add.s32 %0, %0, 1; }" : "+r"(acc) : "r"(v), "r"(lim));
}

// c3 rounded to 20 mantissa bits, as the high word of a double whose low word `lo` is already taken (c4's high word): of
// the three high words around c3's own, the one whose pair lies nearest to c3 - within half a unit of the high word,
// |error| <= 2^-21 |c3|
__device__ __forceinline__ int c3_high_word(double c3, int lo) {
    const int h = __double2hiint(c3);
    int best = h;
    double err = fabs(__hiloint2double(h, lo) - c3);
    for (int d = -1; d <= 1; d += 2) {
        const double e = fabs(__hiloint2double(h + d, lo) - c3);
        if (e < err) {
            err = e;
            best = h + d;
        }
    }
    return best;
}

// both 16-byte halves of interval `idx` from the lane's table replica (`tab_lane` -> its copy of interval 0): the address is
// ONE multiply-add (the compiler otherwise forms shift + or per state), the second half sits at a constant offset
__device__ __forceinline__ void table_entry(const double2 *tab_lane, int idx, double2 &c01, double2 &c2f) {
    constexpr int NTAB_BYTES = (ICNV_EMIS_N + 1) * TAB_REP * 16;
    const unsigned base = (unsigned)__cvta_generic_to_shared(tab_lane);   // loop-invariant
    unsigned addr;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(addr) : "r"((unsigned)idx), "n"(TAB_REP * 16), "r"(base));
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(c01.x), "=d"(c01.y) : "r"(addr));
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2+%3];" : "=d"(c2f.x), "=d"(c2f.y) : "r"(addr), "n"(NTAB_BYTES));
}

template <int M, int NWARPS, bool SDCOL>
__global__ void __launch_bounds__(NWARPS * 32, 1) viterbi_fast_kernel(const VitParams p) {
    extern __shared__ __align__(16) double sm[];
    // emission table re-laid as [interval][replica] -> {c0, c1} and {c2, c34}: two 16-byte loads per state (32 B instead
    // of 40 B).  c34 holds c3 and c4 shortened to their high words (20 mantissa bits): read as a double it IS c3 (high word
    // c3's, low word c4's high word, see c3_high_word), and c4 is its low word moved into a high word.  So the whole
    // polynomial runs in FP64 without a conversion.  c3, c4 only weigh u^3, u^4 with |u| <= 1/2: the shortening costs
    // <= 2^-21 * 7.9e-6 / 8 + 2^-20 * 5.0e-8 / 16 < 4.8e-13 (the table's largest |c3|, |c4|).
    // The lanes of a warp look up unrelated intervals, which on a single copy costs ~2.4 x the minimum number of
    // shared-memory wavefronts in bank conflicts - the table reads are this kernel's tightest resource.  With
    // TAB_REP = 8 copies interleaved at 16-byte granularity, lane l always reads bank group l & 7: every quarter
    // warp touches 8 distinct groups, i.e. exactly 4 wavefronts per load.
    constexpr int NTAB = (ICNV_EMIS_N + 1) * TAB_REP;
    double2 *tab01 = reinterpret_cast<double2 *>(sm);
    double2 *tab2f = tab01 + NTAB;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double *tiles = reinterpret_cast<double *>(tab2f + NTAB) + warp * (2 * 32 * TS);   // two staged x tiles per warp
    for (int e = threadIdx.x; e < ICNV_EMIS_N * TAB_REP; e += blockDim.x) {
        const int i = e / TAB_REP;
        tab01[e] = make_double2(p.table[i], p.table[ICNV_EMIS_N + i]);
        const int c4_hi = __double2hiint(p.table[4 * ICNV_EMIS_N + i]);
        tab2f[e] = make_double2(p.table[2 * ICNV_EMIS_N + i], __hiloint2double(c3_high_word(p.table[3 * ICNV_EMIS_N + i], c4_hi), c4_hi));
    }
    __syncthreads();
    // this lane's replica of interval 0; the second halves (tab2f) follow at a constant distance
    const double2 *tab_lane = tab01 + (lane & (TAB_REP - 1));

    const int64_t warp_global = (int64_t)blockIdx.x * NWARPS + warp;
    // backpointers: one 16-bit word per gene and lane - the best previous state (3 bits) and, per state, whether the
    // path into it comes from that best state (1) or stays (0)
    uint16_t *__restrict__ bp = reinterpret_cast<uint16_t *>(p.bp + warp_global * (int64_t)p.max_len * 32);
    const double cmove = p.cmove;   // read from the parameter bank where it is used: no register held for it
    const double MAGIC = 6755399441055744.0;  // 1.5 * 2^52: (v + MAGIC) - MAGIC == rint(v), low word == (int)rint(v)
    // a state is "near the best" when its e = score - (best - cmove) reaches cmove - tau (> 0: the launcher refuses the fast
    // path unless cmove > 8 tau).  Compared by high words: e >= cmove - tau implies hi(e) >= lim_hi, so the count can only
    // come out too large - i.e. the check rejects a little more than the exact one would (a gap below tau + one unit of the
    // high word, 2^-17 for cmove in [8, 16)), and never accepts what the exact one rejects
    const int lim_hi = p.near_hi;   // __double2hiint(cmove - tau), from the launcher (a parameter-bank operand)
    int err = 0;

    for (;;) {
        unsigned long long item = 0;
        if (lane == 0) item = atomicAdd(p.counter, 1ull);
        item = __shfl_sync(0xffffffffu, item, 0);
        if ((int64_t)item >= p.n_items) break;
        const int ks = (int)(item / (unsigned long long)p.n_tiles);
        const int64_t tile = (int64_t)(item % (unsigned long long)p.n_tiles);
        const int cs = p.item_chr_start[ks];
        const int n = p.item_chr_len[ks];
        const int64_t c0 = tile * 32;
        const int64_t c = c0 + lane;
        const bool active = c < p.C;
        const int64_t cc = active ? c : (p.C - 1);
        uint8_t *__restrict__ scol = p.states + p.G * cc;
        if (n < 2) {
            if (active && n == 1) scol[cs] = 3;
            continue;
        }
        const double sd = SDCOL ? p.sd_col[cc] : p.sd;
        // zs_k = 16 * |x - mean_k| / sd = |fma(x, scale, -mean_k * scale)|: one operation per state.  With one sd for the
        // launch, scale and the offsets are the launcher's (same operations, same bits) and stay in the parameter bank: held
        // per lane they cost 12 registers, and under the 128-register cap the compiler would form them again every gene
        const double scale = SDCOL ? (double)ICNV_EMIS_INVW / sd : p.emis_scale;
        double nms[MAXM];
#pragma unroll
        for (int k = 0; k < M; ++k) nms[k] = SDCOL ? -p.mean[k] * scale : p.emis_nms[k];
        const int g_lo = cs, g_hi = cs + n;
        const int b_first = g_lo / TG, b_last = (g_hi - 1) / TG;

        // stage tile `blk` (TG genes x 32 cells) into buffer `buf`: 8 cp.async per lane, each
        // warp instruction covers 4 cells x 8 consecutive genes (4 x 64 contiguous bytes)
        auto issue_tile = [&](int blk, int buf) {
            double *dst = tiles + buf * (32 * TS);
            const int col = lane & 7;
            const int64_t gene = (int64_t)blk * TG + col;
            const bool ok = gene < p.G;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int row = q * 4 + (lane >> 3);
                int64_t cell = c0 + row;
                if (cell >= p.C) cell = p.C - 1;
                const double *src = p.X + p.G * cell + (ok ? gene : 0);
                cp_async8(dst + row * TS + col, src, ok);
            }
        };

        double nu[MAXM];
        // certificate: smallest decision margin seen, tracked through the HIGH WORD of the (non-negative)
        // gap - monotone in the gap, exact for the power-of-two threshold, two integer ops per check
        unsigned mg = 0x7fffffffu;
        int near_best = 0;   // states within tau of the best score, summed over the steps (the best one included)
        issue_tile(b_first, 0);
        cp_async_commit();
        for (int blk = b_first; blk <= b_last; ++blk) {
            const int buf = (blk - b_first) & 1;
            if (blk < b_last) {
                issue_tile(blk + 1, buf ^ 1);
                cp_async_commit();
                cp_async_wait<1>();
            } else {
                cp_async_wait<0>();
            }
            __syncwarp();
            const double *row = tiles + buf * (32 * TS) + lane * TS;
            const int j0 = max(0, g_lo - blk * TG), j1 = min(TG, g_hi - blk * TG);
            // two genes per trip: the next gene's table lookups and polynomials are independent of this gene's recursion, so
            // the compiler can issue them into its dependency gaps (3 % off the kernel at c3).  With per-lane offsets
            // (SDCOL) the registers for that are not there: one gene per trip, spill-free
#pragma unroll(SDCOL ? 1 : 2)
            for (int j = j0; j < j1; ++j) {
                const int i = blk * TG + j - g_lo;
                const double x = row[j];   // a non-finite x makes every zs NaN / Inf: it is caught on the rare path below
                // ---- emissions: g(z_k) from the table ------------------------------------------------
                double le[MAXM], zs[MAXM];
#pragma unroll
                for (int k = 0; k < M; ++k) zs[k] = fabs(fma(x, scale, nms[k]));
                // the state means are monotone (checked by the launcher), so the largest |x - mean_k| is at an end
                // state: one range test per gene instead of one per state, and a branch-free lookup block
                const double LIM = (double)(ICNV_EMIS_N - 1);
                bool in_table = (zs[0] < LIM) && (zs[M - 1] < LIM);
                if (!p.means_monotone) {
#pragma unroll
                    for (int k = 1; k < M - 1; ++k) in_table = in_table && (zs[k] < LIM);
                }
                if (in_table) {
#pragma unroll
                    for (int k = 0; k < M; ++k) {
                        const double m = zs[k] + MAGIC;
                        const double u = zs[k] - (m - MAGIC);
                        double2 c01, c2f;
                        table_entry(tab_lane, __double2loint(m), c01, c2f);
                        double v = fma(u, __hiloint2double(__double2loint(c2f.y), 0), c2f.y);   // c3 + u c4
                        v = fma(u, v, c2f.x);
                        v = fma(u, v, c01.y);
                        le[k] = fma(u, v, c01.x);
                    }
                } else {   // some state further than 24 sd from x (rare): per-state choice, nmath beyond the table
                    if (!is_finite_d(x)) err |= 1;
#pragma unroll
                    for (int k = 0; k < M; ++k) {
                        double v;
                        if (zs[k] < LIM) {
                            const double m = zs[k] + MAGIC;
                            const double u = zs[k] - (m - MAGIC);
                            double2 c01, c2f;
                            table_entry(tab_lane, __double2loint(m), c01, c2f);
                            v = fma(u, __hiloint2double(__double2loint(c2f.y), 0), c2f.y);
                            v = fma(u, v, c2f.x);
                            v = fma(u, v, c01.y);
                            v = fma(u, v, c01.x);
                        } else {
                            v = emission_far(x, p.mean[k], sd);
                        }
                        le[k] = v;
                    }
                }
                if (i == 0) {
#pragma unroll
                    for (int k = 0; k < M; ++k) nu[k] = p.logdelta[k] + le[k];
                    continue;
                }
                // ---- shifted frame: nu holds the scores minus i * a (a common shift: no arg-max sees it), so staying adds
                //      nothing and coming from the best state costs cmove:  nu'[k] = max(nu[k], best - cmove) + le[k].
                //      best = max_k nu[k] and its first index: a tournament of compare / select pairs carries the index along,
                //      the lower-indexed side on the left (strict comparison = which.max's first-index rule).  M - 1
                //      compares as in a chain, but ceil(log2 M) deep: this is the one step of the gene on the recursion's
                //      dependency chain that has width ----
                double bv[MAXM];
                int bi[MAXM];
#pragma unroll
                for (int k = 0; k < M; ++k) {
                    bv[k] = nu[k];
                    bi[k] = k;
                }
#pragma unroll
                for (int s = 1; s < M; s *= 2) {
#pragma unroll
                    for (int k = 0; k + s < M; k += 2 * s) {
                        const bool gt = bv[k + s] > bv[k];   // compare + select: fmax() is ~8 instructions in FP64
                        bv[k] = gt ? bv[k + s] : bv[k];
                        bi[k] = gt ? bi[k + s] : bi[k];
                    }
                }
                const double best = bv[0];
                const int i1 = bi[0];
                const double T = best - cmove;   // "come from the best state"
                // ---- per state: stay (nu[k]) or come from the best state (T).  The best state always stays (e = cmove),
                //      so the runner-up is never a third state unless best - nu[k] is itself small - which the second
                //      check catches. ----------------------------------------------------------------------------------
                uint32_t moved = 0;   // bit k: the path into state k comes from the best state (sign bit of e, shifted in)
#pragma unroll
                for (int k = M - 1; k >= 0; --k) {
                    const double e = nu[k] - T;
                    const int he = __double2hiint(e);
                    const bool stay = he >= 0;
                    mg = min(mg, (unsigned)(he & 0x7fffffff));                      // |stay - from_best|
                    // best vs every other state: best - nu[k] = cmove - e up to two roundings, so the gap is at least tau
                    // iff e <= cmove - tau.  The best state itself has e = cmove: exactly one state per gene may reach the
                    // bound - counted here on the high word (see lim_hi), checked against the number of steps at the end.
                    count_if_ge(near_best, he, lim_hi);
                    nu[k] = (stay ? nu[k] : T) + le[k];
                    moved = __funnelshift_l((uint32_t)he, moved, 1);
                }
                bp[(int64_t)i * 32 + lane] = (uint16_t)(moved | ((uint32_t)i1 << 8));
            }
            __syncwarp();
        }
        // ---- termination ------------------------------------------------------------------------------
        int y = 0;
        {
            double best = nu[0], second = -INFINITY;
            bool under = (nu[0] == -INFINITY);
#pragma unroll
            for (int k = 1; k < M; ++k) {
                under |= (nu[k] == -INFINITY);
                if (nu[k] > best) {
                    second = best;
                    best = nu[k];
                    y = k;
                } else if (nu[k] > second) {
                    second = nu[k];
                }
            }
            if (under && active) err |= 2;
            const double gap = best - second;
            if (!(gap >= p.tau)) mg = 0;   // also catches NaN
            if (near_best != n - 1) mg = 0;   // some step had a second state within tau of the best one (or a NaN score)
            // |score| < 2^15 keeps every rounding of the recursion below 2^-38 (error budget above); the best score rises by
            // at most g(0) < 0.375 per gene, so a final best score above this bound means every earlier one was inside it
            if (!(best - 0.375 * n > -32768.0 + cmove + 8.0) || n > FAST_MAX_N) mg = 0;
        }
        // uncertified sequences go to the exact kernel
        if (active && (int)mg < __double2hiint(p.tau)) {
            unsigned pos = atomicAdd(p.list_out_count, 1u);
            if (pos < p.list_cap) p.list_out[pos] = make_int2(p.item_chr_id[ks], (int)c);
        }
        // ---- traceback in aligned blocks of 8 genes: the 8 backpointer words are loaded together
        //      (independent addresses), states leave as one 8-byte word when the layout allows it -----
        const bool wide = ((p.G & 7) == 0);  // then (G*c + g) is 8-aligned whenever g is
        for (int gb = (g_hi - 1) & ~7; gb + 8 > g_lo; gb -= 8) {
            uint32_t w[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int i = gb + q - g_lo;
                w[q] = (i >= 1 && i < n) ? (uint32_t)bp[(int64_t)i * 32 + lane] : 0u;
            }
            unsigned long long pack = 0;
#pragma unroll
            for (int q = 7; q >= 0; --q) {
                const int g = gb + q;
                if (g >= g_lo && g < g_hi) {
                    pack |= (unsigned long long)(y + 1) << (8 * q);
                    if (g > g_lo) y = ((w[q] >> y) & 1u) ? (int)(w[q] >> 8) : y;
                }
            }
            if (active) {
                if (wide && gb >= g_lo && gb + 8 <= g_hi) {
                    *reinterpret_cast<unsigned long long *>(scol + gb) = pack;
                } else {  // ragged first / last block of the chromosome, or unaligned layout
#pragma unroll
                    for (int q = 0; q < 8; ++q) {
                        const int g = gb + q;
                        if (g >= g_lo && g < g_hi) scol[g] = (uint8_t)(pack >> (8 * q));
                    }
                }
            }
        }
        __syncwarp();
    }
    if (err && p.err_flag) atomicOr(p.err_flag, err);
}

// Exact re-run of the sequences the certificate rejected: one CTA (4 warps) per sequence, reference-order
// arithmetic throughout.  The emissions - ~1100 FP64 instructions per gene, embarrassingly parallel - are
// evaluated a chunk of LIST_CH genes at a time into shared memory by warps 1..3 while warp 0 runs the
// recursion on the previous chunk (double-buffered).  The recursion itself is a dependent chain per gene, so
// it is spread over the states: lane k of warp 0 owns nu[k], fetches the other states' nu by shuffle, forms
// nu[j] + logPi[j,k] and takes the first arg-max with a comparison tree that prefers the lower index on ties
// (which.max, HMM.R:1170).  Backpointers stay in shared memory for sequences of up to LIST_BPS genes.
constexpr int LIST_NT = 128;
constexpr int LIST_CH = 96 * 4;
constexpr int LIST_BPS = 2048;

template <int M>
__global__ void __launch_bounds__(LIST_NT) viterbi_list_kernel(const VitParams p) {
    __shared__ double le_s[2][LIST_CH][M];
    __shared__ uint32_t bp_s[LIST_BPS];
    __shared__ unsigned long long item_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t *__restrict__ bp_g = p.bp + (int64_t)blockIdx.x * 4 * (int64_t)p.max_len * 32;   // this CTA's share of the ring
    const int64_t n_items = (int64_t)min(*p.list_count, p.list_cap);
    const int kk = lane < M ? lane : 0;   // state owned by this lane of warp 0 (lanes >= M shadow state 0)
    double lp[M];                         // logPi[j, kk], j = 0..M-1
#pragma unroll
    for (int j = 0; j < M; ++j) lp[j] = p.logPi[j * M + kk];
    int err = 0;
    for (;;) {
        if (tid == 0) item_s = atomicAdd(p.counter, 1ull);
        __syncthreads();
        const unsigned long long item = item_s;
        __syncthreads();
        if ((int64_t)item >= n_items) break;
        const int2 e = p.list[item];
        const int cs = p.chr_start_orig[e.x], n = p.chr_len_orig[e.x];
        const int64_t c = e.y;
        const double *__restrict__ xcol = p.X + p.G * c + cs;
        uint8_t *__restrict__ scol = p.states + p.G * c + cs;
        const double sd = p.sd_col ? p.sd_col[c] : p.sd;
        uint32_t *bpw = (n <= LIST_BPS) ? bp_s : bp_g;
        auto produce = [&](int chunk, int first_thread, int n_threads) {
            const int base = chunk * LIST_CH;
            for (int q = tid - first_thread; q < LIST_CH && base + q < n; q += n_threads) {
                double le[MAXM];
                emission_exact<M>(xcol[base + q], p.mean, sd, le);
#pragma unroll
                for (int k = 0; k < M; ++k) le_s[chunk & 1][q][k] = le[k];
            }
        };
        const int nch = (n + LIST_CH - 1) / LIST_CH;
        produce(0, 0, LIST_NT);
        __syncthreads();
        double nu = 0.0;
        for (int s = 0; s < nch; ++s) {
            if (warp > 0) {
                if (s + 1 < nch) produce(s + 1, 32, LIST_NT - 32);
            } else {
                const int base = s * LIST_CH;
                const int cnt = min(LIST_CH, n - base);
                for (int q = 0; q < cnt; ++q) {
                    const double le = le_s[s & 1][q][kk];
                    if (base + q == 0) {
                        nu = __dadd_rn(p.logdelta[kk], le);
                        continue;
                    }
                    double v[M];
#pragma unroll
                    for (int j = 0; j < M; ++j) v[j] = __dadd_rn(__shfl_sync(0xffffffffu, nu, j), lp[j]);
                    double best;
                    int arg;
                    if (M == 6) {
                        const bool t01 = v[1] > v[0], t23 = v[3] > v[2], t45 = v[5] > v[4];
                        const double b01 = t01 ? v[1] : v[0], b23 = t23 ? v[3] : v[2], b45 = t45 ? v[5] : v[4];
                        const int a01 = t01 ? 1 : 0, a23 = t23 ? 3 : 2, a45 = t45 ? 5 : 4;
                        const bool u = b23 > b01;
                        const double b03 = u ? b23 : b01;
                        const int a03 = u ? a23 : a01;
                        const bool w = b45 > b03;
                        best = w ? b45 : b03;
                        arg = w ? a45 : a03;
                    } else {
                        best = v[0];
                        arg = 0;
#pragma unroll
                        for (int j = 1; j < M; ++j)
                            if (v[j] > best) {
                                best = v[j];
                                arg = j;
                            }
                    }
                    nu = __dadd_rn(best, le);
                    const uint32_t word = __reduce_or_sync(0xffffffffu, lane < M ? (uint32_t)arg << (3 * lane) : 0u);
                    if (lane == 0) bpw[base + q] = word;
                }
            }
            __syncthreads();
        }
        if (warp == 0) {
            double fin[M];
#pragma unroll
            for (int k = 0; k < M; ++k) fin[k] = __shfl_sync(0xffffffffu, nu, k);
            if (lane == 0) {
                int y = 0;
                double best = fin[0];
                bool under = (fin[0] == -INFINITY);
#pragma unroll
                for (int k = 1; k < M; ++k) {
                    under |= (fin[k] == -INFINITY);
                    if (fin[k] > best) {
                        best = fin[k];
                        y = k;
                    }
                }
                if (under) err |= 2;
                scol[n - 1] = (uint8_t)(y + 1);
                for (int i = n - 1; i >= 1;) {   // backpointer words are fetched 8 at a time: their addresses do not depend on y
                    const int take = min(8, i);
                    uint32_t w[8];
#pragma unroll
                    for (int q = 0; q < 8; ++q) w[q] = (q < take) ? bpw[i - q] : 0u;
#pragma unroll
                    for (int q = 0; q < 8; ++q)
                        if (q < take) {
                            y = (int)((w[q] >> (3 * y)) & 7u);
                            scol[i - q - 1] = (uint8_t)(y + 1);
                        }
                    i -= take;
                }
            }
        }
        __syncthreads();
    }
    if (err && p.err_flag) atomicOr(p.err_flag, err);
}

// uint8 states -> int32 (255 = unassigned -> -1)
__global__ void __launch_bounds__(256) widen_states_kernel(const uint8_t *__restrict__ s, int32_t *__restrict__ out,
                                                           int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        uint8_t v = s[i];
        out[i] = (v == 255) ? -1 : (int32_t)v;
    }
}

// int32 states -> uint8 (-1 = unassigned -> 255): the one-byte wire format of the *_u8 host entry points
__global__ void __launch_bounds__(256) narrow_states_kernel(const int32_t *__restrict__ s, uint8_t *__restrict__ out,
                                                            int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        const int32_t v = s[i];
        out[i] = (v < 0) ? (uint8_t)255 : (uint8_t)v;
    }
}

// group-mode broadcast: states[g, c] = grp_states[g, grp_of[c]] or -1 (HMM.R:368, 399)
__global__ void __launch_bounds__(256) scatter_group_states_kernel(const uint8_t *__restrict__ gs, int64_t G, int64_t C,
                                                                   const int32_t *__restrict__ grp_of,
                                                                   int32_t *__restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < G * C; i += stride) {
        int64_t c = i / G, g = i - c * G;
        int grp = grp_of[c];
        out[i] = grp < 0 ? -1 : (int32_t)gs[g + G * grp];
    }
}

// the same with one byte per state (255 = cell in no group)
__global__ void __launch_bounds__(256) scatter_group_states_u8_kernel(const uint8_t *__restrict__ gs, int64_t G, int64_t C,
                                                                      const int32_t *__restrict__ grp_of, uint8_t *__restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < G * C; i += stride) {
        int64_t c = i / G, g = i - c * G;
        int grp = grp_of[c];
        out[i] = grp < 0 ? (uint8_t)255 : gs[g + G * grp];
    }
}

}  // namespace icnv

using namespace icnv;

extern "C" {

int icnv_dev_scatter_group_states_u8(const uint8_t *gs, int64_t G, int64_t C, const int32_t *grp_of, uint8_t *out, void *stream) {
    ICNV_REQUIRE_READY();
    if (!gs || !grp_of || !out || G <= 0 || C <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_dev_scatter_group_states_u8: bad argument");
    int64_t blocks = (G * C + 255) / 256;
    if (blocks > (int64_t)ctx().sm_count * 32) blocks = (int64_t)ctx().sm_count * 32;
    scatter_group_states_u8_kernel<<<(unsigned)blocks, 256, 0, pick_stream(stream)>>>(gs, G, C, grp_of, out);
    ICNV_CHECK_LAUNCH("scatter_group_states_u8_kernel");
    return ICNV_OK;
}

int icnv_dev_widen_states(const uint8_t *s, int32_t *out, int64_t n, void *stream) {
    ICNV_REQUIRE_READY();
    int64_t blocks = (n + 255) / 256;
    if (blocks > (int64_t)ctx().sm_count * 32) blocks = (int64_t)ctx().sm_count * 32;
    widen_states_kernel<<<(unsigned)blocks, 256, 0, pick_stream(stream)>>>(s, out, n);
    ICNV_CHECK_LAUNCH("widen_states_kernel");
    return ICNV_OK;
}

int icnv_dev_narrow_states(const int32_t *s, uint8_t *out, int64_t n, void *stream) {
    ICNV_REQUIRE_READY();
    int64_t blocks = (n + 255) / 256;
    if (blocks > (int64_t)ctx().sm_count * 32) blocks = (int64_t)ctx().sm_count * 32;
    narrow_states_kernel<<<(unsigned)blocks, 256, 0, pick_stream(stream)>>>(s, out, n);
    ICNV_CHECK_LAUNCH("narrow_states_kernel");
    return ICNV_OK;
}

int icnv_dev_scatter_group_states(const uint8_t *gs, int64_t G, int64_t C, const int32_t *grp_of, int32_t *out,
                                  void *stream) {
    ICNV_REQUIRE_READY();
    int64_t blocks = (G * C + 255) / 256;
    if (blocks > (int64_t)ctx().sm_count * 32) blocks = (int64_t)ctx().sm_count * 32;
    scatter_group_states_kernel<<<(unsigned)blocks, 256, 0, pick_stream(stream)>>>(gs, G, C, grp_of, out);
    ICNV_CHECK_LAUNCH("scatter_group_states_kernel");
    return ICNV_OK;
}

int icnv_dev_viterbi_f64(const double *X, int64_t G, int64_t C, const int32_t *chr_start, const int32_t *chr_len, int K,
                         int m, const double *Pi, const double *delta, const double *mean, const double *sd,
                         int sd_per_col, uint8_t *states_u8, double *margins, int *err_flag, void *stream) {
    ICNV_REQUIRE_READY();
    Ctx &c = ctx();
    if (!X || !states_u8 || G <= 0 || C <= 0 || !chr_start || !chr_len || K <= 0 || !Pi || !delta || !mean || !sd)
        return set_error(ICNV_E_BAD_ARG, "icnv_dev_viterbi_f64: bad argument");
    if (m != 6 && m != 3) return set_error(ICNV_E_BAD_ARG, "m must be 6 (i6) or 3 (i3), got %d", m);
    cudaStream_t st = pick_stream(stream);

    VitParams p;
    p.X = X; p.G = G; p.C = C; p.K = K;
    for (int j = 0; j < m; ++j)
        for (int k = 0; k < m; ++k) p.logPi[j * m + k] = std::log(Pi[j + m * k]);
    for (int k = 0; k < m; ++k) {
        p.logdelta[k] = std::log(delta[k]);
        p.mean[k] = mean[k];
    }
    const double *d_sd_col = nullptr;
    p.sd = 0.0;
    if (sd_per_col) {
        d_sd_col = sd;  // device array, one median sd per column
    } else {
        // object$pm$sd = median(object$pm$sd), HMM.R:1122
        std::vector<double> v(sd, sd + m);
        std::sort(v.begin(), v.end());
        p.sd = (m & 1) ? v[m / 2] : 0.5 * (v[m / 2 - 1] + v[m / 2]);
        if (!(p.sd > 0.0)) return set_error(ICNV_E_BAD_ARG, "state sd must be positive");
    }
    p.sd_col = d_sd_col;

    // chromosomes longest first, so the dynamic scheduler ends with the short ones (LPT)
    std::vector<int> order(K);
    for (int k = 0; k < K; ++k) order[k] = k;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return chr_len[a] > chr_len[b]; });
    std::vector<int32_t> h(5 * (size_t)K);
    int max_len = 1;
    for (int k = 0; k < K; ++k) {
        int o = order[k];
        if (chr_len[o] < 0 || chr_start[o] < 0 || (int64_t)chr_start[o] + chr_len[o] > G)
            return set_error(ICNV_E_BAD_ARG, "chromosome %d out of range", o);
        h[k] = chr_start[o];
        h[K + k] = chr_len[o];
        h[2 * K + k] = o;
        h[3 * K + k] = chr_start[k];
        h[4 * K + k] = chr_len[k];
        max_len = std::max(max_len, (int)chr_len[o]);
    }
    int32_t *d_items = (int32_t *)scratch(SLOT_VIT_ITEMS, sizeof(int32_t) * 5 * (size_t)K + 64);
    if (!d_items) return ICNV_E_NOMEM;
    ICNV_CUDA(upload_if_changed(c.up_items, c.up_items_stream, d_items, h.data(), sizeof(int32_t) * 5 * (size_t)K, st));
    p.item_chr_start = d_items;
    p.item_chr_len = d_items + K;
    p.item_chr_id = d_items + 2 * K;
    p.chr_start_orig = d_items + 3 * K;
    p.chr_len_orig = d_items + 4 * K;
    p.n_tiles = (C + 31) / 32;
    p.n_items = p.n_tiles * K;
    p.max_len = max_len;
    p.list = nullptr;
    p.list_count = nullptr;
    p.states = states_u8;
    p.margins = margins;
    p.err_flag = err_flag;

    // counters: [0] work counter of the main launch, [1] work counter of the list launch, [2] list length
    const size_t counter_bytes = 3 * sizeof(unsigned long long);
    unsigned long long *d_counter = (unsigned long long *)scratch(SLOT_MISC2, counter_bytes + 64);
    if (!d_counter) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemsetAsync(d_counter, 0, counter_bytes, st));
    p.counter = d_counter;
    c.hmm_list_count = reinterpret_cast<unsigned int *>(d_counter + 2);

    const bool want_margin = margins != nullptr;
    // the fast path needs .get_HMM's structure: one diagonal and one off-diagonal value
    bool structured = true;
    for (int j = 0; j < m && structured; ++j)
        for (int k = 0; k < m; ++k)
            if (Pi[j + m * k] != (j == k ? Pi[0] : Pi[1])) structured = false;
    // ... with the diagonal the larger one ("the best state always stays" is what the fast recursion relies on) and every
    // transition possible (log 0 would poison the margins): t <= 1/6 for i6, 1/3 for i3, and t > 0.  The certificate's
    // best-versus-others check reads the gap off e = stay - from_best, which needs log(diag / offdiag) well above tau.
    structured = structured && Pi[0] > Pi[1] && Pi[1] > 0.0 && std::log(Pi[0] / Pi[1]) > 1e-6;
    const bool use_fast = (c.hmm_mode == 1) && structured && !want_margin;

    if (!use_fast) {
        int per_sm = 0;
        auto kern = (m == 6) ? (want_margin ? viterbi_kernel<6, true> : viterbi_kernel<6, false>)
                             : (want_margin ? viterbi_kernel<3, true> : viterbi_kernel<3, false>);
        ICNV_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 128, 0));
        if (per_sm < 1) per_sm = 1;
        int64_t blocks = (int64_t)c.sm_count * per_sm;
        int64_t need_blocks = (p.n_items + 3) / 4;
        if (blocks > need_blocks) blocks = need_blocks;
        uint32_t *d_bp = (uint32_t *)scratch(SLOT_BP, sizeof(uint32_t) * (size_t)(blocks * 4) * (size_t)max_len * 32);
        if (!d_bp) return ICNV_E_NOMEM;
        p.bp = d_bp;
        kern<<<(unsigned)blocks, 128, 0, st>>>(p);
        ICNV_CHECK_LAUNCH("viterbi_kernel");
        return ICNV_OK;
    }

    // ---- certified fast path + exact re-run of the uncertified sequences --------------------------------
    double *d_table = (double *)scratch(SLOT_TABLE, sizeof(icnv_emis_table));
    if (!d_table) return ICNV_E_NOMEM;
    if (!c.table_uploaded) {
        ICNV_CUDA(cudaMemcpyAsync(d_table, icnv_emis_table, sizeof(icnv_emis_table), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        c.table_uploaded = true;
    }
    const size_t list_cap = (size_t)K * (size_t)C;
    int2 *d_list = (int2 *)scratch(SLOT_LIST, sizeof(int2) * list_cap);
    if (!d_list) return ICNV_E_NOMEM;
    p.a_diag = p.logPi[0];
    p.b_off = p.logPi[1];
    p.inv_sd = sd_per_col ? 0.0 : 1.0 / p.sd;
    p.emis_scale = sd_per_col ? 0.0 : (double)ICNV_EMIS_INVW / p.sd;
    for (int k = 0; k < MAXM; ++k) p.emis_nms[k] = (sd_per_col || k >= m) ? 0.0 : -p.mean[k] * p.emis_scale;
    p.tau = 1.1920928955078125e-07;  // 2^-23: power of two, so the high-word comparison in the kernel is exact
    p.cmove = p.a_diag - p.b_off;
    {
        const double lim = p.cmove - p.tau;
        int32_t hi;
        std::memcpy(&hi, reinterpret_cast<const char *>(&lim) + 4, 4);
        p.near_hi = hi;
    }
    p.table = d_table;
    p.list_out = d_list;
    p.list_out_count = c.hmm_list_count;
    p.list_cap = (unsigned int)std::min<size_t>(list_cap, 0xffffffffu);

    auto lkern = (m == 6) ? viterbi_list_kernel<6> : viterbi_list_kernel<3>;
    void (*fkern)(const VitParams) = sd_per_col
        ? ((m == 6) ? viterbi_fast_kernel<6, FAST_WARPS, true> : viterbi_fast_kernel<3, FAST_WARPS, true>)
        : ((m == 6) ? viterbi_fast_kernel<6, FAST_WARPS, false> : viterbi_fast_kernel<3, FAST_WARPS, false>);
    const size_t smem = sizeof(double) * (4 * (ICNV_EMIS_N + 1) * TAB_REP + (size_t)FAST_WARPS * 2 * 32 * TS);
    p.means_monotone = 1;
    for (int k = 1; k + 1 < m; ++k)
        if ((mean[k] - mean[k - 1]) * (mean[k + 1] - mean[k]) < 0.0) p.means_monotone = 0;
    ICNV_CUDA(cudaFuncSetAttribute(fkern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    ICNV_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fkern, FAST_WARPS * 32, smem));
    if (per_sm < 1) per_sm = 1;
    int64_t blocks = (int64_t)c.sm_count * per_sm;
    int64_t need_blocks = (p.n_items + FAST_WARPS - 1) / FAST_WARPS;
    if (blocks > need_blocks) blocks = need_blocks;
    const int64_t list_blocks = c.sm_count;  // 4 warps each; the list is short
    const int64_t n_warps = std::max<int64_t>(blocks * FAST_WARPS, list_blocks * 4);
    uint32_t *d_bp = (uint32_t *)scratch(SLOT_BP, sizeof(uint32_t) * (size_t)n_warps * (size_t)max_len * 32);
    if (!d_bp) return ICNV_E_NOMEM;
    p.bp = d_bp;
    fkern<<<(unsigned)blocks, FAST_WARPS * 32, smem, st>>>(p);
    ICNV_CHECK_LAUNCH("viterbi_fast_kernel");
    // exact re-run of whatever the certificate rejected (list length is read on the device)
    p.list = d_list;
    p.list_count = c.hmm_list_count;
    p.counter = d_counter + 1;
    lkern<<<(unsigned)list_blocks, LIST_NT, 0, st>>>(p);
    ICNV_CHECK_LAUNCH("viterbi_list_kernel");
    return ICNV_OK;
}

int icnv_set_hmm_mode(int mode) {
    if (mode != 0 && mode != 1)
        return set_error(ICNV_E_BAD_ARG, "hmm mode must be 0 (reference-order arithmetic) or 1 (certified FP64 pass, default), got %d", mode);
    ctx().hmm_mode = mode;
    return ICNV_OK;
}

/* always 0: no HMM mode hands sequences to a second pass (kept for callers of the C ABI) */
int64_t icnv_hmm_second_pass_count(void) { return 0; }

int64_t icnv_hmm_rerun_count(void) {
    Ctx &c = ctx();
    if (!c.ready || !c.hmm_list_count) return 0;
    unsigned int h = 0;
    cudaDeviceSynchronize();
    if (cudaMemcpy(&h, c.hmm_list_count, sizeof(h), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    return (int64_t)h;
}

}  // extern "C"
