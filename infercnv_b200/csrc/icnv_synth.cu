// icnv_synth.cu - deterministic synthetic workload written straight into HBM (bench / scale tests).
//
// Counter-based: every value is a pure function of (seed, global cell index, gene index), so any
// partition of the cells over GPUs produces bit-identical data.  Model (SURVEY section 8d):
//   x[g, c] ~ Gamma-Poisson(mean = m_g * f_c * cnv(c, chr(g)), dispersion 0.1)
//   m_g ~ LogNormal(0.5, 1.0), f_c ~ LogNormal(0, 0.2); the first 10 % of the cells are reference
//   cells; 30 % of the remaining cells carry 3 whole-chromosome events with multiplier 0.5 or 1.5.
// Values are stored as float64 "depth-normalised expression" (input of run() step 4).
#include <cmath>
#include <vector>

#include "icnv_common.cuh"

namespace icnv {

__global__ void __launch_bounds__(256) synth_kernel(double *__restrict__ X, int64_t G, int64_t cell0, int64_t n_cells,
                                                    int64_t C_total, const int32_t *__restrict__ chr_of, int K,
                                                    uint64_t seed) {
    for (int64_t ci = blockIdx.x; ci < n_cells; ci += gridDim.x) {
        const uint64_t cell = (uint64_t)(cell0 + ci);
        const double f_c = exp(0.2 * std_normal(hash3(seed, 1, cell, 0), hash3(seed, 1, cell, 1)));
        // events: observation cells only (cells beyond the first 10 %)
        int ev_chr[3] = {-1, -1, -1};
        double ev_mul[3] = {1.0, 1.0, 1.0};
        const bool is_obs = (int64_t)cell >= C_total / 10;
        if (is_obs && u01(hash3(seed, 2, cell, 0)) < 0.3) {
            for (int e = 0; e < 3; ++e) {
                uint64_t h = hash3(seed, 3, cell, (uint64_t)e);
                ev_chr[e] = (int)(h % (uint64_t)K);
                ev_mul[e] = (h >> 40) & 1ull ? 1.5 : 0.5;
            }
        }
        double *col = X + G * ci;
        for (int64_t g = threadIdx.x; g < G; g += blockDim.x) {
            const double m_g = exp(0.5 + std_normal(hash3(seed, 4, (uint64_t)g, 0), hash3(seed, 4, (uint64_t)g, 1)));
            const int chr = chr_of[g];
            double cnv = 1.0;
#pragma unroll
            for (int e = 0; e < 3; ++e)
                if (chr == ev_chr[e]) cnv = ev_mul[e];
            const double mean = m_g * f_c * cnv;
            // Gamma(shape 10, scale mean/10) as minus the log of a product of 10 uniforms
            double prod = 1.0;
#pragma unroll
            for (int i = 0; i < 10; ++i) prod *= u01(hash3(seed, 5 + (uint64_t)i, cell, (uint64_t)g));
            const double lambda = -log(prod) * (mean * 0.1);
            double x;
            if (lambda < 12.0) {  // Poisson by inversion
                double u = u01(hash3(seed, 20, cell, (uint64_t)g));
                double pmf = exp(-lambda), cdf = pmf;
                int k = 0;
                while (u > cdf && k < 64) {
                    ++k;
                    pmf *= lambda / (double)k;
                    cdf += pmf;
                }
                x = (double)k;
            } else {  // normal approximation with continuity rounding
                double z = std_normal(hash3(seed, 21, cell, (uint64_t)g), hash3(seed, 22, cell, (uint64_t)g));
                x = floor(lambda + sqrt(lambda) * z + 0.5);
                if (x < 0.0) x = 0.0;
            }
            col[g] = x;
        }
    }
}

}  // namespace icnv

using namespace icnv;

extern "C" int icnv_dev_synth_f64(double *X, int64_t G, int64_t cell0, int64_t n_cells, int64_t C_total,
                                  const int32_t *chr_start, const int32_t *chr_len, int K, uint64_t seed, void *stream) {
    ICNV_REQUIRE_READY();
    if (!X || G <= 0 || n_cells <= 0 || C_total <= 0 || !chr_start || !chr_len || K <= 0)
        return set_error(ICNV_E_BAD_ARG, "icnv_dev_synth_f64: bad argument");
    cudaStream_t st = pick_stream(stream);
    std::vector<int32_t> chr_of((size_t)G, 0);
    for (int k = 0; k < K; ++k)
        for (int32_t g = chr_start[k]; g < chr_start[k] + chr_len[k] && g < G; ++g) chr_of[g] = k;
    int32_t *d_chr = (int32_t *)scratch(SLOT_SYNTH, sizeof(int32_t) * (size_t)G);
    if (!d_chr) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemcpyAsync(d_chr, chr_of.data(), sizeof(int32_t) * (size_t)G, cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    int64_t blocks = n_cells < (int64_t)ctx().sm_count * 16 ? n_cells : (int64_t)ctx().sm_count * 16;
    synth_kernel<<<(unsigned)blocks, 256, 0, st>>>(X, G, cell0, n_cells, C_total, d_chr, K, seed);
    ICNV_CHECK_LAUNCH("synth_kernel");
    return ICNV_OK;
}
