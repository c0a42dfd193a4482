// Bayesian network filter - K15 in DESIGN section 3: the Gibbs sampling of inferCNVBayesNet (R/inferCNV_BayesNet.R:
// run_gibb_sampling, :1054-1107) for every CNV region of the HMM's report in one call.
//
// Model (inst/BUGS_Mixture_Model, m = 6; ..._i3, m = 3), region r with genes i and cells j:
//   gexp[i, j] ~ dnorm(mu[eps_j], tau[eps_j]),  eps_j ~ dcat(theta),  theta ~ ddirich(1, ..., 1)
// with mu and tau (a precision) data.  Both full conditionals are exact:
//   theta | eps ~ Dirichlet(1 + n_1, ..., 1 + n_m)              (n_k: cells in state k)
//   eps_j | theta ∝ theta_k exp(L[j, k]),  L[j, k] = sum_i (1/2 log tau_k - 1/2 tau_k (x_ij - mu_k)^2)
// L does not change across sweeps, so it is computed once per (region, cell, state):
//   (a) loglik_kernel: one thread per output column (region, cell), every state, FP64, the genes in list order; each term
//       is hl_k - (ht_k d) d with d = x - mu_k, hl_k = 1/2 log tau_k and ht_k = 1/2 tau_k from the host, every operation
//       rounded on its own (no contraction), so a sequential NumPy restatement reproduces it.  A POOLED region (R's
//       one-gene quirk: expr.data[Gene, Cells] drops to a vector that JAGS sees as ONE cell whose genes are the C values)
//       has one column summed over its cells in list order, within a cell its genes in list order.  Non-finite listed
//       values raise a flag.
//   (b) sampler_kernel: one CTA per (region, chain), items taken largest region first from an atomic counter by a
//       persistent grid; threads over the region's columns.  Chain c starts from eps = rep(c mod m, C').  Each sweep:
//       m Marsaglia-Tsang gamma draws (shape 1 + n_k >= 1, so no boost) normalised to theta in FP64; per column the
//       FP64 log-weights log theta_k + L[j, k] with their maximum subtracted, exp and the cumulative sum in FP32 (each
//       normalised weight within 1e-6 absolute: expf's 2 ulp, the FP32
//       rounding of the argument and the FP32 sum of at most 8 terms stay under 8e-7), one uniform against the cumulative sum; an integer block reduction of
//       the m counts.  Sweeps n_burn .. n_burn + n_keep - 1 write their theta row and add 1 to the drawn state of each
//       column in a per-CTA private count buffer (coalesced, no atomics), added to the output once per item.  L sits in
//       shared memory when the region fits (SMEM_L bytes), in global memory otherwise.
//
// Generator: mix64(hash3(seed, a, b, c)) with a = 2 r (gamma draws) or 2 r + 1 (categorical draws), b = chain 2^32 + sweep,
// c = index 2^12 + attempt 2^2 + component (index = state or column; component 0 / 1 the Box-Muller pair, 2 the uniform;
// attempt the Marsaglia-Tsang rejection round, 0 for the categorical draw).  The result is a pure function of (seed,
// inputs): independent of the launch shape, the schedule and thread order; the counts are summed as integers.
#include "icnv_common.cuh"

#include <algorithm>
#include <cmath>
#include <numeric>
#include <vector>

namespace icnv {
namespace bayes {

constexpr int NT = 256;
constexpr int MAXM = 8;
constexpr size_t SMEM_L = 96 * 1024;   // two CTAs per SM with their L in shared memory
constexpr int MT_ATTEMPTS = 1024;      // Marsaglia-Tsang accepts with probability > 0.95 per round

struct Emis {
    double mu[MAXM], hl[MAXM], ht[MAXM];
};

__device__ __forceinline__ uint64_t draw(unsigned long long seed, uint64_t a, uint64_t b, uint64_t c) {
    return mix64(hash3(seed, a, b, c));
}

// upper_bound(off, off + n, v) - off - 1: the region whose column range holds v
__device__ __forceinline__ int region_of(const int32_t *off, int n, int64_t v) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((int64_t)off[mid] <= v) lo = mid + 1; else hi = mid;
    }
    return lo - 1;
}

// (a) L[col m + k] for every output column col of every region
__global__ void __launch_bounds__(NT) loglik_kernel(const double *__restrict__ X, int64_t ldx, const int32_t *__restrict__ gene_off,
                                                    const int32_t *__restrict__ gene_idx, const int32_t *__restrict__ cell_off,
                                                    const int32_t *__restrict__ cell_idx, const int32_t *__restrict__ out_off,
                                                    const unsigned char *__restrict__ pooled, int n_reg, int64_t n_cols, int m,
                                                    Emis e, double *__restrict__ L, int *flag) {
    bool bad = false;
    for (int64_t col = (int64_t)blockIdx.x * NT + threadIdx.x; col < n_cols; col += (int64_t)gridDim.x * NT) {
        const int r = region_of(out_off, n_reg + 1, col);
        const int g0 = gene_off[r], g1 = gene_off[r + 1];
        int c0 = cell_off[r], c1 = cell_off[r + 1];
        if (!pooled[r]) {
            c0 += (int)(col - out_off[r]);
            c1 = c0 + 1;
        }
        double s[MAXM];
#pragma unroll
        for (int k = 0; k < MAXM; ++k) s[k] = 0.0;
        for (int cc = c0; cc < c1; ++cc) {
            const double *x = X + ldx * (int64_t)cell_idx[cc];
            for (int gi = g0; gi < g1; ++gi) {
                const double v = x[gene_idx[gi]];
                bad |= !is_finite_d(v);
#pragma unroll
                for (int k = 0; k < MAXM; ++k)
                    if (k < m) {
                        const double d = __dadd_rn(v, -e.mu[k]);
                        s[k] = __dadd_rn(s[k], __dadd_rn(e.hl[k], -__dmul_rn(__dmul_rn(e.ht[k], d), d)));
                    }
            }
        }
#pragma unroll
        for (int k = 0; k < MAXM; ++k)
            if (k < m) L[col * m + k] = s[k];
    }
    if (bad) atomicOr(flag, 1);
}

// Gamma(a, 1), a >= 1, by Marsaglia and Tsang (2000)
__device__ double gamma_mt(double a, unsigned long long seed, uint64_t ka, uint64_t kb, uint64_t idx) {
    const double d = a - 1.0 / 3.0, c = 1.0 / sqrt(9.0 * d);
    for (uint64_t t = 0; t < (uint64_t)MT_ATTEMPTS; ++t) {
        const uint64_t kc = (idx << 12) | (t << 2);
        const double x = std_normal(draw(seed, ka, kb, kc), draw(seed, ka, kb, kc | 1));
        double v = 1.0 + c * x;
        if (v <= 0.0) continue;
        v = v * v * v;
        const double u = u01(draw(seed, ka, kb, kc | 2));
        if (log(u) < 0.5 * x * x + d - d * v + d * log(v)) return d * v;
    }
    return d;   // not reached in practice: 1024 rejections in a row have probability < 1e-1300
}

// (b) one item = (region order[item / n_chains], chain item % n_chains) at a time per CTA
__global__ void __launch_bounds__(NT, 2) sampler_kernel(const double *__restrict__ L, const int32_t *__restrict__ out_off,
                                                        const int32_t *__restrict__ order, int64_t n_items, int n_chains,
                                                        int m, int n_burn, int n_keep, unsigned long long seed, int smem_cols,
                                                        double *__restrict__ theta, int32_t *__restrict__ counts,
                                                        int32_t *__restrict__ priv, int64_t priv_stride,
                                                        unsigned long long *work) {
    extern __shared__ __align__(16) unsigned char bn_smem[];
    double *sL = reinterpret_cast<double *>(bn_smem);
    __shared__ double s_g[MAXM], s_lt[MAXM];
    __shared__ int s_n[MAXM], s_w[NT / 32][MAXM];
    __shared__ long long s_item;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int32_t *my = priv + (int64_t)blockIdx.x * priv_stride;
    const int64_t rows = (int64_t)n_chains * n_keep;
    for (;;) {
        if (tid == 0) s_item = (long long)atomicAdd(work, 1ull);
        __syncthreads();
        const long long item = s_item;
        if (item >= n_items) break;
        const int r = order[item / n_chains], ch = (int)(item % n_chains);
        const int64_t o = out_off[r];
        const int n = out_off[r + 1] - (int)o;
        const double *Lr = L + o * m;
        const bool in_smem = n <= smem_cols;
        if (in_smem)
            for (int i = tid; i < n * m; i += NT) sL[i] = Lr[i];
        const double *Lp = in_smem ? sL : Lr;
        if (tid < m) s_n[tid] = tid == ch % m ? n : 0;
        double *th_out = theta + (int64_t)r * rows * m + (int64_t)ch * n_keep;
        __syncthreads();
        const uint64_t ka = 2ull * (uint64_t)r;
        for (int s = 0; s < n_burn + n_keep; ++s) {
            const bool kept = s >= n_burn;
            const uint64_t kb = ((uint64_t)ch << 32) | (uint64_t)s;
            if (tid < m) s_g[tid] = gamma_mt(1.0 + (double)s_n[tid], seed, ka, kb, (uint64_t)tid);
            __syncthreads();
            if (tid < m) {
                double tot = 0.0;
                for (int k = 0; k < m; ++k) tot += s_g[k];
                const double th = s_g[tid] / tot;
                s_lt[tid] = log(th);
                if (kept) th_out[(int64_t)tid * rows + (s - n_burn)] = th;
            }
            __syncthreads();
            int cnt[MAXM];
#pragma unroll
            for (int k = 0; k < MAXM; ++k) cnt[k] = 0;
            int q = 0;
            for (int j = tid; j < n; j += NT, ++q) {
                const double *lj = Lp + (int64_t)j * m;
                double lw[MAXM];
                double mx = __longlong_as_double((long long)0xfff0000000000000ull);   // -inf
#pragma unroll
                for (int k = 0; k < MAXM; ++k)
                    if (k < m) {
                        lw[k] = s_lt[k] + lj[k];
                        mx = fmax(mx, lw[k]);
                    }
                float w[MAXM], tot = 0.0f;
#pragma unroll
                for (int k = 0; k < MAXM; ++k)
                    if (k < m) {
                        w[k] = expf((float)(lw[k] - mx));
                        tot += w[k];
                    }
                const float tgt = (float)u01(draw(seed, ka + 1, kb, ((uint64_t)j << 12) | 2)) * tot;
                int pick = m - 1;
                float cum = 0.0f;
                bool found = false;
#pragma unroll
                for (int k = 0; k < MAXM; ++k)
                    if (k < m) {
                        cum += w[k];
                        if (!found && cum >= tgt) {
                            pick = k;
                            found = true;
                        }
                    }
#pragma unroll
                for (int k = 0; k < MAXM; ++k) cnt[k] += k == pick;
                if (kept) my[((int64_t)q * m + pick) * NT + tid] += 1;
            }
#pragma unroll
            for (int k = 0; k < MAXM; ++k)
                if (k < m) {
                    const int v = __reduce_add_sync(0xffffffffu, cnt[k]);
                    if (lane == 0) s_w[warp][k] = v;
                }
            __syncthreads();
            if (tid < m) {
                int t = 0;
                for (int w2 = 0; w2 < NT / 32; ++w2) t += s_w[w2][tid];
                s_n[tid] = t;
            }
            __syncthreads();
        }
        // this chain's state counts into the region's, and the private buffer back to zero
        int q = 0;
        for (int j = tid; j < n; j += NT, ++q)
            for (int k = 0; k < m; ++k) {
                int32_t *p = my + ((int64_t)q * m + k) * NT + tid;
                const int v = *p;
                if (v) {
                    atomicAdd(counts + (o + j) * m + k, v);
                    *p = 0;
                }
            }
        __syncthreads();   // s_item and sL are rewritten by the next item
    }
}

}  // namespace bayes

using namespace bayes;

// What the last call of the process did: regions, sampler CTAs, device ms of (a) the log-likelihoods and (b) the sampler.
static double g_bayes_stats[4];

static size_t align256b(size_t b) { return (b + 255) & ~(size_t)255; }

static int check_lists(const int32_t *off, const int32_t *idx, int n_reg, int64_t bound, const char *what, const char *who) {
    if (!off || !idx) return set_error(ICNV_E_BAD_ARG, "%s: %s lists missing", who, what);
    if (off[0] != 0) return set_error(ICNV_E_BAD_ARG, "%s: %s offsets must start at 0", who, what);
    for (int r = 0; r < n_reg; ++r)
        if (off[r + 1] <= off[r]) return set_error(ICNV_E_BAD_ARG, "%s: region %d has an empty %s list", who, r, what);
    for (int32_t i = 0; i < off[n_reg]; ++i)
        if (idx[i] < 0 || idx[i] >= bound) return set_error(ICNV_E_BAD_ARG, "%s: %s index %d out of range", who, what, idx[i]);
    return ICNV_OK;
}

// Every argument check of the call that needs no device (host entry points run it before they upload the matrix); on
// success *n_cols = sum over the regions of C'_r.
int bayesnet_check(int64_t G, int64_t C, const int32_t *gene_off, const int32_t *gene_idx, const int32_t *cell_off,
                   const int32_t *cell_idx, const uint8_t *pooled, int n_reg, int m, const double *mu, const double *tau,
                   int n_chains, int n_burn, int n_keep, int64_t *n_cols, const char *who) {
    *n_cols = 0;
    if (G < 1 || C < 1 || n_reg < 0 || !mu || !tau) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    if (m < 2 || m > MAXM) return set_error(ICNV_E_BAD_ARG, "%s: m = %d outside 2..%d", who, m, MAXM);
    if (n_chains < 1 || n_keep < 1 || n_burn < 0 || (int64_t)n_burn + n_keep > INT32_MAX)
        return set_error(ICNV_E_BAD_ARG, "%s: bad chain count or sweep counts", who);
    for (int k = 0; k < m; ++k)
        if (!std::isfinite(mu[k]) || !std::isfinite(tau[k]) || !(tau[k] > 0.0))
            return set_error(ICNV_E_BAD_ARG, "%s: mu / tau of state %d invalid (tau must be finite and > 0)", who, k + 1);
    if (n_reg == 0) return ICNV_OK;
    int rc;
    if ((rc = check_lists(gene_off, gene_idx, n_reg, G, "gene", who))) return rc;
    if ((rc = check_lists(cell_off, cell_idx, n_reg, C, "cell", who))) return rc;
    int64_t tot = 0;
    for (int r = 0; r < n_reg; ++r) {
        tot += pooled && pooled[r] ? 1 : cell_off[r + 1] - cell_off[r];
        if (tot * MAXM > INT32_MAX) return set_error(ICNV_E_UNSUPPORTED, "%s: too many output columns", who);
    }
    *n_cols = tot;
    return ICNV_OK;
}

int bayesnet_dev(const double *X, int64_t ldx, int64_t G, int64_t C, const int32_t *gene_off, const int32_t *gene_idx,
                 const int32_t *cell_off, const int32_t *cell_idx, const uint8_t *pooled, int n_reg, int m, const double *mu,
                 const double *tau, int n_chains, int n_burn, int n_keep, unsigned long long seed, double *theta,
                 int32_t *state_counts, double *loglik, void *stream, const char *who) {
    ICNV_REQUIRE_READY();
    if (!X || ldx < G || !theta || !state_counts) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    int64_t n_cols = 0;
    int rc = bayesnet_check(G, C, gene_off, gene_idx, cell_off, cell_idx, pooled, n_reg, m, mu, tau, n_chains, n_burn, n_keep,
                            &n_cols, who);
    if (rc || n_reg == 0) return rc;
    // output columns: 1 for a pooled region, C_r otherwise
    std::vector<int32_t> out_off((size_t)n_reg + 1, 0);
    std::vector<unsigned char> pool_f((size_t)n_reg, 0);
    for (int r = 0; r < n_reg; ++r) {
        pool_f[(size_t)r] = pooled && pooled[r] ? 1 : 0;
        out_off[(size_t)r + 1] = out_off[(size_t)r] + (pool_f[(size_t)r] ? 1 : cell_off[r + 1] - cell_off[r]);
    }
    // largest region first (stable), so the long chains start early
    std::vector<int32_t> order((size_t)n_reg);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) {
        return out_off[(size_t)a + 1] - out_off[(size_t)a] > out_off[(size_t)b + 1] - out_off[(size_t)b];
    });
    int max_cols = 0, smem_cols = 0;
    const int fit = (int)(SMEM_L / (sizeof(double) * (size_t)m));
    for (int r = 0; r < n_reg; ++r) {
        const int w = out_off[(size_t)r + 1] - out_off[(size_t)r];
        max_cols = std::max(max_cols, w);
        if (w <= fit) smem_cols = std::max(smem_cols, w);
    }
    Emis e;
    for (int k = 0; k < MAXM; ++k) {
        e.mu[k] = k < m ? mu[k] : 0.0;
        e.hl[k] = k < m ? 0.5 * std::log(tau[k]) : 0.0;
        e.ht[k] = k < m ? 0.5 * tau[k] : 0.0;
    }

    Ctx &c = ctx();
    cudaStream_t st = pick_stream(stream);
    const int64_t n_items = (int64_t)n_reg * n_chains;
    const size_t smem = sizeof(double) * (size_t)smem_cols * (size_t)m;
    if (smem > 48 * 1024) ICNV_CUDA(cudaFuncSetAttribute(sampler_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 1;
    ICNV_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sampler_kernel, NT, smem));
    const int64_t grid = std::max<int64_t>(1, std::min<int64_t>(n_items, (int64_t)c.sm_count * std::max(per_sm, 1)));
    const int64_t priv_stride = (int64_t)((max_cols + NT - 1) / NT) * m * NT;
    size_t bytes = 0;
    auto take = [&](size_t b) { const size_t o = bytes; bytes += align256b(b); return o; };
    const size_t o_goff = take(sizeof(int32_t) * ((size_t)n_reg + 1)), o_gidx = take(sizeof(int32_t) * (size_t)gene_off[n_reg]),
                 o_coff = take(sizeof(int32_t) * ((size_t)n_reg + 1)), o_cidx = take(sizeof(int32_t) * (size_t)cell_off[n_reg]),
                 o_ooff = take(sizeof(int32_t) * ((size_t)n_reg + 1)), o_pool = take((size_t)n_reg),
                 o_order = take(sizeof(int32_t) * (size_t)n_reg), o_flag = take(sizeof(int)),
                 o_work = take(sizeof(unsigned long long)),
                 o_L = take(loglik ? 0 : sizeof(double) * (size_t)(n_cols * m)),
                 o_priv = take(sizeof(int32_t) * (size_t)(grid * priv_stride));
    char *buf = nullptr;
    if (cudaMallocAsync((void **)&buf, bytes, st) != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NOMEM, "%s: no room for %lld bytes", who, (long long)bytes);
    }
    int32_t *d_goff = (int32_t *)(buf + o_goff), *d_gidx = (int32_t *)(buf + o_gidx), *d_coff = (int32_t *)(buf + o_coff),
            *d_cidx = (int32_t *)(buf + o_cidx), *d_ooff = (int32_t *)(buf + o_ooff), *d_order = (int32_t *)(buf + o_order),
            *d_priv = (int32_t *)(buf + o_priv);
    unsigned char *d_pool = (unsigned char *)(buf + o_pool);
    int *d_flag = (int *)(buf + o_flag);
    unsigned long long *d_work = (unsigned long long *)(buf + o_work);
    double *d_L = loglik ? loglik : (double *)(buf + o_L);
    cudaEvent_t ev[4] = {};
    for (auto &ev_i : ev) ICNV_CUDA(cudaEventCreate(&ev_i));
    auto body = [&]() -> int {
        ICNV_CUDA(cudaMemcpyAsync(d_goff, gene_off, sizeof(int32_t) * ((size_t)n_reg + 1), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_gidx, gene_idx, sizeof(int32_t) * (size_t)gene_off[n_reg], cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_coff, cell_off, sizeof(int32_t) * ((size_t)n_reg + 1), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_cidx, cell_idx, sizeof(int32_t) * (size_t)cell_off[n_reg], cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_ooff, out_off.data(), sizeof(int32_t) * out_off.size(), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_pool, pool_f.data(), (size_t)n_reg, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_order, order.data(), sizeof(int32_t) * (size_t)n_reg, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
        ICNV_CUDA(cudaMemsetAsync(d_work, 0, sizeof(unsigned long long), st));
        ICNV_CUDA(cudaMemsetAsync(d_priv, 0, sizeof(int32_t) * (size_t)(grid * priv_stride), st));
        ICNV_CUDA(cudaMemsetAsync(state_counts, 0, sizeof(int32_t) * (size_t)(n_cols * m), st));
        ICNV_CUDA(cudaEventRecord(ev[0], st));
        const int64_t gl = std::min<int64_t>((n_cols + NT - 1) / NT, (int64_t)c.sm_count * 64);
        loglik_kernel<<<(unsigned)gl, NT, 0, st>>>(X, ldx, d_goff, d_gidx, d_coff, d_cidx, d_ooff, d_pool, n_reg, n_cols, m, e,
                                                   d_L, d_flag);
        ICNV_CHECK_LAUNCH("loglik_kernel");
        ICNV_CUDA(cudaEventRecord(ev[1], st));
        int h = 0;
        ICNV_CUDA(cudaMemcpyAsync(&h, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        if (h) return set_error(ICNV_E_NONFINITE, "%s: NaN or Inf in a listed entry", who);
        ICNV_CUDA(cudaEventRecord(ev[2], st));
        sampler_kernel<<<(unsigned)grid, NT, smem, st>>>(d_L, d_ooff, d_order, n_items, n_chains, m, n_burn, n_keep, seed,
                                                         smem_cols, theta, state_counts, d_priv, priv_stride, d_work);
        ICNV_CHECK_LAUNCH("sampler_kernel");
        ICNV_CUDA(cudaEventRecord(ev[3], st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        float ms_a = 0.0f, ms_b = 0.0f;
        ICNV_CUDA(cudaEventElapsedTime(&ms_a, ev[0], ev[1]));
        ICNV_CUDA(cudaEventElapsedTime(&ms_b, ev[2], ev[3]));
        g_bayes_stats[0] = (double)n_reg;
        g_bayes_stats[1] = (double)grid;
        g_bayes_stats[2] = ms_a;
        g_bayes_stats[3] = ms_b;
        return ICNV_OK;
    };
    rc = body();
    cudaFreeAsync(buf, st);
    cudaStreamSynchronize(st);
    for (auto &ev_i : ev)
        if (ev_i) cudaEventDestroy(ev_i);
    return rc;
}

void bayesnet_stats(double *out4) {
    for (int i = 0; i < 4; ++i) out4[i] = g_bayes_stats[i];
}

}  // namespace icnv
