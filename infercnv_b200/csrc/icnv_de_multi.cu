// Masking of non-DE genes (K14, icnv_de.cu) over several device slots of icnv_init_devices: the host entry point's
// multi-device body.  The genes are cut into one contiguous range per device for the tests; each device uploads only its
// genes of the listed columns (2-D copies, pitch G), packs them into slab rows and tests them, and the p rows meet in host
// memory.  Every device then runs BH on all of them (deterministic: the same DE bits everywhere) and masks its own range of
// cells, streamed through it in chunks.  The stages are icnv_de.cu's, so the bytes are one device's.
#include "icnv_common.cuh"

#include <algorithm>
#include <array>
#include <cmath>
#include <condition_variable>
#include <numeric>
#include <string>
#include <thread>
#include <vector>

namespace icnv {

int de_pack_dev(const double *X, int64_t ldx, const int32_t *d_cols, int64_t m, int n_dst, const int64_t *gene_lo,
                const int64_t *gene_hi, double *out, int *flag, void *stream, const char *who);
int de_slab_tests_dev(const double *Z, int64_t T, int64_t g0, int64_t n, const int32_t *ref_off, int n_ref,
                      const int32_t *sub_off, int n_sub, int test, double jitter_mean, double jitter_sd,
                      unsigned long long seed, double *p_raw, int64_t ldp, void *stream, double *times, const char *who);
int de_bh_mask_dev(const double *p_raw, int64_t G, int n_ref, int n_sub, const int32_t *sub_size, double p_thresh,
                   double *p_adj, const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t C, const int32_t *ref_idx,
                   int64_t n_ref_cells, const int32_t *sub_off, const int32_t *sub_idx, int rule, double mask_val,
                   void *stream, double *times, const char *who);
void de_mask_set_stats(const double *in7);

namespace {

// device memory owned by one scope
struct DevBuf {
    void *p = nullptr;
    ~DevBuf() {
        if (p) cudaFree(p);
    }
    template <class T> T *get(size_t bytes) {
        if (p) cudaFree(p);
        p = nullptr;
        if (cudaMalloc(&p, bytes ? bytes : 16) != cudaSuccess) {
            cudaGetLastError();
            p = nullptr;
            set_error(ICNV_E_NOMEM, "icnv_mask_non_de_f64: no room for %zu bytes", bytes);
        }
        return (T *)p;
    }
};

size_t usable_bytes() {
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    return free_b > (size_t)(1 << 30) ? free_b - (size_t)(1 << 30) : (size_t)0;
}

// One device slot's share of the tests: genes [g_lo, g_hi) of every listed column go up in sub-slabs sized from free memory
// (2-D copies: pitch G, one per run of consecutive columns), are packed into slab rows and tested; the p rows come back to
// h_p (pair rows of G).  stats: tiles, largest tile, ms of (a) - (c).
int mask_tests_slot(cudaStream_t st, const double *X, int64_t G, const std::vector<int32_t> &cols, const int32_t *ref_off,
                           int n_ref, const int32_t *sub_off, int n_sub, int test, double jitter_mean, double jitter_sd,
                           unsigned long long seed, int64_t g_lo, int64_t g_hi, double *h_p, double *stats) {
    static const char *who = "icnv_mask_non_de_f64";
    const int64_t T = (int64_t)cols.size(), R_tot = ref_off[n_ref], npair = (int64_t)n_sub * n_ref;
    if (npair == 0 || g_hi <= g_lo) return ICNV_OK;
    // per gene: the uploaded columns, the slab rows, the p slab and the tests' own scratch
    const size_t per_gene = sizeof(double) * (size_t)(2 * T + npair + R_tot + 3 * (n_ref + n_sub));
    const int64_t nt = std::min<int64_t>(g_hi - g_lo, (int64_t)(usable_bytes() / per_gene));
    if (nt < 1) return set_error(ICNV_E_NOMEM, "%s: not even one gene fits in device memory", who);
    std::vector<int32_t> iota((size_t)T);
    std::iota(iota.begin(), iota.end(), 0);
    DevBuf b_iota, b_u, b_z, b_p, b_flag;
    int32_t *d_iota = b_iota.get<int32_t>(sizeof(int32_t) * (size_t)T);
    double *dU = b_u.get<double>(sizeof(double) * (size_t)(nt * T)), *dZ = b_z.get<double>(sizeof(double) * (size_t)(nt * T));
    double *dP = b_p.get<double>(sizeof(double) * (size_t)(nt * npair));
    int *d_flag = b_flag.get<int>(sizeof(int));
    if (!d_iota || !dU || !dZ || !dP || !d_flag) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemcpyAsync(d_iota, iota.data(), sizeof(int32_t) * (size_t)T, cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
    cudaEvent_t ev[2] = {};
    for (auto &e : ev) ICNV_CUDA(cudaEventCreate(&e));
    auto body = [&]() -> int {
        int rc;
        for (int64_t a = g_lo; a < g_hi; a += nt) {
            const int64_t n = std::min<int64_t>(nt, g_hi - a), lo = 0, hi = n;
            for (int64_t i = 0; i < T;) {   // column-major n x T
                int64_t j = i + 1;
                while (j < T && cols[(size_t)j] == cols[(size_t)j - 1] + 1) ++j;
                ICNV_CUDA(cudaMemcpy2DAsync(dU + i * n, sizeof(double) * (size_t)n, X + (size_t)cols[(size_t)i] * (size_t)G + a,
                                            sizeof(double) * (size_t)G, sizeof(double) * (size_t)n, (size_t)(j - i),
                                            cudaMemcpyHostToDevice, st));
                i = j;
            }
            ICNV_CUDA(cudaEventRecord(ev[0], st));
            if ((rc = de_pack_dev(dU, n, d_iota, T, 1, &lo, &hi, dZ, d_flag, st, who))) return rc;
            ICNV_CUDA(cudaEventRecord(ev[1], st));
            if ((rc = de_slab_tests_dev(dZ, T, a, n, ref_off, n_ref, sub_off, n_sub, test, jitter_mean, jitter_sd, seed, dP, n, st,
                                        stats + 3, who)))
                return rc;
            ICNV_CUDA(cudaMemcpy2DAsync(h_p + a, sizeof(double) * (size_t)G, dP, sizeof(double) * (size_t)n,
                                        sizeof(double) * (size_t)n, (size_t)npair, cudaMemcpyDeviceToHost, st));
            int h = 0;
            ICNV_CUDA(cudaMemcpyAsync(&h, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
            ICNV_CUDA(cudaStreamSynchronize(st));
            if (h) return set_error(ICNV_E_NONFINITE, "%s: NaN or Inf in a listed cell", who);
            float ms = 0.0f;
            ICNV_CUDA(cudaEventElapsedTime(&ms, ev[0], ev[1]));
            stats[0] += 1;
            stats[1] = std::max<double>(stats[1], (double)n);
            stats[2] += ms;
        }
        return ICNV_OK;
    };
    const int rc = body();
    for (auto &e : ev)
        if (e) cudaEventDestroy(e);
    return rc;
}

// One device slot's share of BH + mask: BH of the whole p (h_p, pair rows of G) on this device, then the mask of cells
// [c_lo, c_hi) in chunks that fit beside it, streamed back to Y.  p_adj (nullable) gets BH's output.  stats[5], [6]: ms of
// (d), (e).
int mask_apply_slot(cudaStream_t st, const double *X, double *Y, int64_t G, const int32_t *ref_off, const int32_t *ref_idx,
                           int n_ref, const int32_t *sub_off, const int32_t *sub_idx, int n_sub, const double *h_p,
                           int64_t c_lo, int64_t c_hi, double p_thresh, int rule, double mask_val, double *p_adj,
                           double *stats) {
    static const char *who = "icnv_mask_non_de_f64";
    if (c_hi <= c_lo && !p_adj) return ICNV_OK;
    const int64_t R_tot = ref_off[n_ref], npair = (int64_t)n_sub * n_ref;
    const size_t pbytes = sizeof(double) * (size_t)(G * std::max<int64_t>(npair, 1));
    DevBuf b_p, b_pa, b_x;
    double *d_p = b_p.get<double>(pbytes), *d_pa = p_adj ? b_pa.get<double>(pbytes) : nullptr;
    if (!d_p || (p_adj && !d_pa)) return ICNV_E_NOMEM;
    if (npair > 0) ICNV_CUDA(cudaMemcpyAsync(d_p, h_p, pbytes, cudaMemcpyHostToDevice, st));
    // beside the chunk: BH's DE bytes and sort scratch, and the cell tables
    const size_t reserve = (size_t)(G * std::max<int64_t>(npair, 1)) * 2 + (size_t)(c_hi - c_lo) * 16 + ((size_t)64 << 20);
    const size_t avail = usable_bytes();
    const int64_t cc = std::max<int64_t>(1, std::min<int64_t>(std::max<int64_t>(c_hi - c_lo, 1),
                                                             (int64_t)((avail > reserve ? avail - reserve : 0) / (sizeof(double) * (size_t)G))));
    double *dX = c_hi > c_lo ? b_x.get<double>(sizeof(double) * (size_t)(cc * G)) : nullptr;
    if (c_hi > c_lo && !dX) return ICNV_E_NOMEM;
    std::vector<int32_t> sub_size((size_t)std::max(n_sub, 1));
    for (int s = 0; s < n_sub; ++s) sub_size[(size_t)s] = sub_off[s + 1] - sub_off[s];
    int64_t c0 = c_lo;
    do {
        const int64_t c1 = std::min<int64_t>(c_hi, c0 + cc), n = std::max<int64_t>(c1 - c0, 0);
        // the chunk's reference cells and, per subcluster, its cells, as chunk columns
        std::vector<int32_t> rl, so(1, 0), si;
        for (int64_t i = 0; i < R_tot; ++i)
            if (ref_idx[i] >= c0 && ref_idx[i] < c1) rl.push_back((int32_t)(ref_idx[i] - c0));
        for (int s = 0; s < n_sub; ++s) {
            for (int32_t i = sub_off[s]; i < sub_off[s + 1]; ++i)
                if (sub_idx[i] >= c0 && sub_idx[i] < c1) si.push_back((int32_t)(sub_idx[i] - c0));
            so.push_back((int32_t)si.size());
        }
        si.push_back(0);   // never empty
        if (n > 0) ICNV_CUDA(cudaMemcpyAsync(dX, X + (size_t)c0 * (size_t)G, sizeof(double) * (size_t)(n * G), cudaMemcpyHostToDevice, st));
        const bool first = c0 == c_lo;
        int rc = de_bh_mask_dev(d_p, G, n_ref, n_sub, sub_size.data(), p_thresh, first ? d_pa : nullptr, dX, G, n > 0 ? dX : nullptr,
                                G, n, rl.data(), (int64_t)rl.size(), so.data(), si.data(), rule, mask_val, st, stats + 5, who);
        if (rc) return rc;
        if (n > 0) ICNV_CUDA(cudaMemcpyAsync(Y + (size_t)c0 * (size_t)G, dX, sizeof(double) * (size_t)(n * G), cudaMemcpyDeviceToHost, st));
        if (first && d_pa && npair > 0) ICNV_CUDA(cudaMemcpyAsync(p_adj, d_pa, pbytes, cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        c0 = c1;
    } while (c0 < c_hi);
    return ICNV_OK;
}

}  // namespace

// Several device slots (icnv_init_devices): the genes are cut into one contiguous range per slot for the tests and the p
// rows gathered on the host; then every slot runs BH on all of them (deterministic, so every slot has the same DE bits) and
// masks its own range of cells.  One host thread per slot, as host_pipeline.  The same bytes as one device.
int de_mask_multi(int n_dev, const double *X, double *Y, int64_t G, int64_t C, const int32_t *ref_off,
                             const int32_t *ref_idx, int n_ref, const int32_t *sub_off, const int32_t *sub_idx, int n_sub,
                             int test, double p_thresh, int rule, double mask_val, double jitter_mean, double jitter_sd,
                             uint64_t seed, double *p_raw, double *p_adj) {
    static const char *who = "icnv_mask_non_de_f64";
    if (!ref_off || !ref_idx || (n_sub > 0 && (!sub_off || !sub_idx))) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    if (test != 0 && test != 1) return set_error(ICNV_E_BAD_ARG, "%s: unknown test code %d", who, test);
    if (rule < 0 || rule > 2) return set_error(ICNV_E_BAD_ARG, "%s: unknown rule code %d", who, rule);
    if (!std::isfinite(jitter_mean) || !std::isfinite(jitter_sd) || jitter_sd < 0.0 || std::isnan(p_thresh))
        return set_error(ICNV_E_BAD_ARG, "%s: bad jitter or threshold", who);
    if (ref_off[0] != 0 || (n_sub > 0 && sub_off[0] != 0)) return set_error(ICNV_E_BAD_ARG, "%s: offsets must start at 0", who);
    for (int k = 0; k < n_ref; ++k)
        if (ref_off[k + 1] <= ref_off[k]) return set_error(ICNV_E_BAD_ARG, "%s: reference group %d is empty", who, k);
    for (int k = 0; k < n_sub; ++k)
        if (sub_off[k + 1] <= sub_off[k]) return set_error(ICNV_E_BAD_ARG, "%s: subcluster %d is empty", who, k);
    const int64_t R_tot = ref_off[n_ref], T = R_tot + (n_sub > 0 ? sub_off[n_sub] : 0), npair = (int64_t)n_sub * n_ref;
    if (T > (int64_t)INT32_MAX / 2) return set_error(ICNV_E_UNSUPPORTED, "%s: %lld listed cells", who, (long long)T);
    std::vector<int32_t> cols((size_t)T);
    for (int64_t i = 0; i < R_tot; ++i) cols[(size_t)i] = ref_idx[i];
    for (int64_t i = R_tot; i < T; ++i) cols[(size_t)i] = sub_idx[i - R_tot];
    for (int32_t v : cols)
        if (v < 0 || v >= C) return set_error(ICNV_E_BAD_ARG, "%s: cell index %d out of range", who, v);
    std::vector<double> own;
    double *h_p = p_raw;
    if (!h_p && npair > 0) {
        own.resize((size_t)(G * npair));
        h_p = own.data();
    }
    std::vector<int> rcs((size_t)n_dev, ICNV_OK);
    std::vector<std::string> msgs((size_t)n_dev);
    std::vector<std::array<double, 7>> stats((size_t)n_dev);
    std::mutex mu;
    std::condition_variable cv;
    int arrived = 0, failed = 0;
    // every slot's p rows are in h_p before any slot reads them; false when some slot's tests failed
    auto barrier = [&](int rc) {
        std::unique_lock<std::mutex> lk(mu);
        failed += rc != ICNV_OK;
        if (++arrived == n_dev) cv.notify_all();
        else cv.wait(lk, [&] { return arrived == n_dev; });
        return failed == 0;
    };
    std::vector<std::thread> th;
    const int caller_slot = current_slot();
    for (int d = 0; d < n_dev; ++d) {
        th.emplace_back([&, d] {
            set_current_slot(d);
            Ctx &c = ctx();
            std::unique_lock<std::mutex> lk(c.mu, std::defer_lock);
            if (d != caller_slot) lk.lock();   // the caller already holds its own context's lock
            double *sd = stats[(size_t)d].data();
            stats[(size_t)d].fill(0.0);
            int rc = ICNV_OK;
            if (cudaSetDevice(c.device) != cudaSuccess) rc = set_error(ICNV_E_CUDA, "cudaSetDevice(%d) failed", c.device);
            if (!rc)
                rc = mask_tests_slot(c.stream, X, G, cols, ref_off, n_ref, sub_off, n_sub, test, jitter_mean, jitter_sd, seed,
                                     G * d / n_dev, G * (d + 1) / n_dev, h_p, sd);
            if (barrier(rc) && !rc)
                rc = mask_apply_slot(c.stream, X, Y, G, ref_off, ref_idx, n_ref, sub_off, sub_idx, n_sub, h_p,
                                     Y ? C * d / n_dev : 0, Y ? C * (d + 1) / n_dev : 0, p_thresh, rule, mask_val,
                                     d == 0 ? p_adj : nullptr, sd);
            rcs[(size_t)d] = rc;
            if (rc) msgs[(size_t)d] = icnv_last_error();   // the message is per thread: carry it to the caller
        });
    }
    for (auto &t : th) t.join();
    cudaSetDevice(ctx_of(caller_slot).device);
    for (int d = 0; d < n_dev; ++d)
        if (rcs[(size_t)d]) return set_error(rcs[(size_t)d], "device %d: %s", ctx_of(d).device, msgs[(size_t)d].c_str());
    double out[7] = {0, 0, 0, 0, 0, 0, 0};   // tiles summed; the largest tile and every stage time: the slowest slot's
    for (int d = 0; d < n_dev; ++d) {
        out[0] += stats[(size_t)d][0];
        for (int s = 1; s < 7; ++s) out[s] = std::max(out[s], stats[(size_t)d][s]);
    }
    de_mask_set_stats(out);
    return ICNV_OK;
}
}  // namespace icnv
