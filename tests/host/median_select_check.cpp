// Host-side check of infercnv_b200/csrc/icnv_median_select.cuh (the per-thread window median of the CUDA
// median filter, compiled here as plain C++): random / skewed / bimodal / tie-dominated / truncated windows
// against std::nth_element, plus the 0-1 test of the 16-key sorting network.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "icnv_median_select.cuh"

static double ref_median(std::vector<double> v) {
    const size_t n = v.size();
    std::sort(v.begin(), v.end());
    return (n & 1) ? v[n / 2] : (v[n / 2 - 1] + v[n / 2]) * 0.5;   // median.default: mean of the two middle values
}

template <int R>
static int run(std::mt19937_64 &rng, int trials, unsigned *stats) {
    constexpr int D = 2 * R + 1;
    const int HR = D + 3, idx0 = 2;
    std::vector<double> halo((size_t)HR * (D + 1)), halo0(halo.size());
    std::vector<unsigned short> list((size_t)D * D * 4);
    std::normal_distribution<double> nd(0.0, 1.0);
    std::uniform_real_distribution<double> ud(0.0, 1.0);
    int bad = 0;
    for (int t = 0; t < trials; ++t) {
        const int kind = t % 9;
        // valid sub-rectangle (truncated windows at block edges); full window most of the time
        int a0 = 0, a1 = D - 1, b0 = 0, b1 = D - 1;
        if (t % 3 == 0) {
            a0 = (int)(ud(rng) * D); a1 = a0 + (int)(ud(rng) * (D - a0));
            b0 = (int)(ud(rng) * D); b1 = b0 + (int)(ud(rng) * (D - b0));
        }
        std::vector<double> vals;
        const double scale = (kind == 7) ? 1e300 : (kind == 8 ? 1e-300 : 1.0);
        for (int dj = 0; dj < D; ++dj)
            for (int di = 0; di < D; ++di) {
                const bool in = di >= a0 && di <= a1 && dj >= b0 && dj <= b1;
                double v = 0.0;
                switch (kind) {
                    case 0: v = 1.0 + 0.1 * nd(rng); break;                                   // smooth expression values
                    case 1: v = std::exp(nd(rng)); break;                                     // skewed
                    case 2: v = (ud(rng) < 0.6 ? 1.0 : 1.5) + 0.02 * nd(rng); break;          // CNV boundary: bimodal
                    case 3: v = (ud(rng) < 0.7) ? 1.000123 : 1.0 + 0.2 * nd(rng); break;      // de-noised: ties dominate
                    case 4: v = (double)(1 + (int)(ud(rng) * 6.0)); break;                    // state matrix
                    case 5: v = 3.0; break;                                                   // constant
                    case 6: v = (ud(rng) < 0.5) ? (ud(rng) < 0.5 ? 0.0 : -0.0) : 0.01 * nd(rng); break;   // signed zeros
                    default: v = scale * (1.0 + 0.3 * nd(rng)); break;                        // extreme magnitudes
                }
                halo[idx0 + dj * HR + di] = in ? v : INFINITY;
                halo0[idx0 + dj * HR + di] = in ? v : 0.0;
                if (in) vals.push_back(v);
            }
        const double want = ref_median(vals);
        const double got = icnv::window_median<R>(halo.data(), halo0.data(), HR, idx0, list.data(), 3, (int)vals.size(), stats);
        if (!(got == want)) {
            if (bad < 5) std::printf("R=%d trial %d kind %d n=%zu: got %.17g want %.17g\n", R, t, kind, vals.size(), got, want);
            ++bad;
        }
    }
    return bad;
}


int main(int argc, char **argv) {
    const int trials = argc > 1 ? std::atoi(argv[1]) : 20000;
    // sorting network: 0-1 principle
    for (int mask = 0; mask < 65536; ++mask) {
        double c[16];
        for (int q = 0; q < 16; ++q) c[q] = (mask >> q) & 1;
        icnv::mf_sort16(c);
        for (int q = 1; q < 16; ++q)
            if (c[q - 1] > c[q]) {
                std::printf("sort16 fails on mask %d\n", mask);
                return 1;
            }
    }
    std::mt19937_64 rng(12345);
    unsigned stats[2] = {0, 0};
    int bad = 0;
    bad += run<2>(rng, trials, stats);
    bad += run<3>(rng, trials, stats);
    bad += run<4>(rng, trials, stats);
    bad += run<5>(rng, trials, stats);
    std::printf("windows %d, mismatches %d, list rounds per window %.2f, second build passes per window %.3f\n", 4 * trials, bad,
                stats[0] / (4.0 * trials), stats[1] / (4.0 * trials));
    return bad ? 1 : 0;
}
