// icnv_api.cu - C ABI of libinfercnv_b200.so: lifecycle, the host-pointer entry points the R shim
// binds, and the device-side composition of the smooth block.  See include/infercnv_b200.h.
#if defined(__x86_64__)
#include <emmintrin.h>
#endif
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <functional>
#include <memory>
#include <numeric>
#include <string>
#include <thread>
#include <vector>

#include "icnv_common.cuh"

// device-pointer helpers defined in the other translation units
extern "C" {
int icnv_dev_invlog_finish_f64(double *means, int64_t n, void *stream);
int icnv_dev_widen_states(const uint8_t *s, int32_t *out, int64_t n, void *stream);
int icnv_dev_narrow_states(const int32_t *s, uint8_t *out, int64_t n, void *stream);
int icnv_dev_scatter_group_states(const uint8_t *gs, int64_t G, int64_t C, const int32_t *grp_of, int32_t *out,
                                  void *stream);
int icnv_dev_elementwise_f64(const double *X, double *Y, int64_t n, int op, double param, int *err_flag, void *stream);
int icnv_dev_column_stats_f64(const double *X, int64_t G, const int32_t *cells, int64_t n_cells, double *sums, double *sds,
                              void *stream);
int icnv_dev_scale_columns_f64(const double *X, double *Y, int64_t G, int64_t C, const double *sums, double factor,
                               void *stream);
int icnv_dev_clear_noise_f64(const double *X, double *Y, int64_t n, double lo, double hi, double mu, void *stream);
int icnv_dev_proxy_vals_f64(const double *X, double *Y, int64_t n, int m, void *stream);
int icnv_dev_column_minmax_f64(const double *X, int64_t G, int64_t C, double *mins, double *maxs, void *stream);
int icnv_dev_clamp_bounds_f64(const double *X, double *Y, int64_t n, double lower, double upper, void *stream);
int icnv_dev_logistic_adj_f64(const double *X, double *Y, int64_t n, double expr_mean, double delta_midpt, double slope,
                              void *stream);
int icnv_dev_gene_stats_f64(const double *X, int64_t G, int64_t ldx, int64_t C, double *d_sums, int32_t *d_npos, void *stream);
int icnv_dev_gather_rows_f64(const double *X, int64_t ldx, const int32_t *d_keep, int64_t n_keep, double *Y, int64_t C,
                             void *stream);
int icnv_dev_scale_rows_f64(const double *X, double *Y, int64_t G, int64_t C, double *d_sums, double *d_ss, void *stream);
int icnv_dev_csc_gene_stats_f64(const int32_t *d_i, const double *d_x, int64_t nnz, int64_t G, double *d_sums,
                                int32_t *d_npos, void *stream);
int icnv_dev_csc_col_sums_f64(const int32_t *d_p, const int32_t *d_i, const double *d_x, const int32_t *d_keep_map,
                              int64_t C, double *d_cs, void *stream);
int icnv_dev_csc_expand_f64(const int32_t *d_p, const int32_t *d_i, const double *d_x, const int32_t *d_keep_map,
                            int64_t G_out, int64_t C, const double *d_cs, double factor, double *Y, void *stream);
int icnv_dev_scatter_states_per_chr_u8(const uint8_t *gs, int64_t G, int64_t C, const int32_t *d_chr_id, const int32_t *d_grp_of,
                                       uint8_t *out, void *stream);
int icnv_dev_apply_consensus_u8(const uint8_t *S, const uint8_t *cons, int64_t G, int64_t C, const int32_t *d_chr_of,
                                const int32_t *d_grp_of, uint8_t *out, void *stream);
int icnv_dev_state_consensus_u8(const uint8_t *S, int64_t G, int64_t lds, const int32_t *d_cells, const int32_t *h_grp_off,
                                int n_grp, uint8_t *d_cons, int *d_flag, void *stream);
int icnv_dev_cnv_regions_u8(const uint8_t *d_seqs, int64_t G, int64_t lds, int64_t n_seq, const int32_t *d_cols,
                            const int32_t *chr_start, const int32_t *chr_len, int K, const double *gene_start,
                            const double *gene_stop, int64_t *n_regions, void *stream);
int icnv_dev_cnv_regions_records(int64_t *n, const int32_t **seq, const int32_t **chr, const int32_t **first_gene,
                                 const int32_t **last_gene, const int32_t **state, const double **start,
                                 const double **end);
}
extern "C" ICNV_API void icnv_combine_cell_stats(const double *sums, const double *sds, int64_t n, int64_t G, double *mu,
                                                double *sigma);

namespace icnv {
// K12 in either layout (icnv_dist.cu)
int knn_launch(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n, int k, int32_t *idx, double *dist,
               int rows, void *stream, const char *who);
// K1 over a list-ordered slab (icnv_smooth.cu)
int slab_group_sums(const double *Y, int64_t G, int64_t ldy, const int32_t *d_chunks, int64_t n_chunks, const int32_t *d_segs,
                    int64_t n_segs, double *partial, const double *acc_in, double *acc_out, double *means, void *stream);
}  // namespace icnv

namespace icnv {

static thread_local char g_err[512] = "";

// One context per device the library was initialised on.  A host thread works on one of them at a time (slot 0 unless
// the multi-device host pipeline put the thread on another one): every helper below - scratch(), pick_stream(), the
// launch counter - goes through ctx().
static Ctx g_ctx[ICNV_MAX_DEVICES];
static thread_local int tl_slot = 0;
static int g_slots = 0;

Ctx &ctx() { return g_ctx[tl_slot]; }
Ctx &ctx_of(int slot) { return g_ctx[slot]; }
int current_slot() { return tl_slot; }
void set_current_slot(int s) { tl_slot = s; }
int device_slots() { return g_slots; }

// ---- host copy pool: pageable caller memory <-> the pinned staging ring --------------------------------------------
// cudaMemcpyAsync from pageable memory is staged by the driver on the calling thread at ~10 GB/s and blocks it, which
// serialises the three-stream slab pipeline.  The library therefore owns pinned slabs and a few copy threads that move
// the caller's slab into / out of them at memory bandwidth, so PCIe sees pinned transfers only.
// One thread's share of a staging copy, with NON-TEMPORAL stores: the destination (a pinned ring slot the DMA engine reads
// next, or the caller's result matrix) is not read again by this thread, so writing around the cache saves the write-allocate
// read of every line - glibc's memcpy only does that above ~3/4 of the last-level cache per call.
static void stream_copy(char *d, const char *s, size_t n) {
#if defined(__x86_64__) && defined(__SSE2__)
    if (n < (size_t)1 << 16) {
        memcpy(d, s, n);
        return;
    }
    const size_t head = (16 - (reinterpret_cast<uintptr_t>(d) & 15)) & 15;
    memcpy(d, s, head);
    d += head;
    s += head;
    n -= head;
    const size_t blocks = n / 64;
    for (size_t i = 0; i < blocks; ++i) {
        const __m128i a = _mm_loadu_si128(reinterpret_cast<const __m128i *>(s));
        const __m128i b = _mm_loadu_si128(reinterpret_cast<const __m128i *>(s + 16));
        const __m128i c = _mm_loadu_si128(reinterpret_cast<const __m128i *>(s + 32));
        const __m128i e = _mm_loadu_si128(reinterpret_cast<const __m128i *>(s + 48));
        _mm_stream_si128(reinterpret_cast<__m128i *>(d), a);
        _mm_stream_si128(reinterpret_cast<__m128i *>(d + 16), b);
        _mm_stream_si128(reinterpret_cast<__m128i *>(d + 32), c);
        _mm_stream_si128(reinterpret_cast<__m128i *>(d + 48), e);
        s += 64;
        d += 64;
    }
    _mm_sfence();
    memcpy(d, s, n - blocks * 64);
#else
    memcpy(d, s, n);
#endif
}

class CopyPool {
public:
    explicit CopyPool(int n) : n_(n) {
        for (int t = 0; t < n_; ++t) th_.emplace_back([this, t] { loop(t); });
    }
    ~CopyPool() {
        {
            std::lock_guard<std::mutex> lk(mu_);
            stop_ = true;
            ++gen_;
        }
        cv_.notify_all();
        for (auto &t : th_) t.join();
    }
    int size() const { return n_; }
    struct Job {
        char *d;
        const char *s;
        size_t n;
    };
    // copies the (dst, src, bytes) jobs, their bytes laid end to end and cut into equal ranges over the threads; returns
    // when every job is done
    void copyv(const std::vector<Job> &jobs) {
        size_t total = 0;
        for (const Job &j : jobs) total += j.n;
        if (total == 0) return;
        std::unique_lock<std::mutex> lk(mu_);
        job_ = &jobs;
        pending_ = n_;
        ++gen_;
        cv_.notify_all();
        done_.wait(lk, [this] { return pending_ == 0; });
    }
    void copy2(void *d0, const void *s0, size_t n0, void *d1, const void *s1, size_t n1) {
        copyv({{static_cast<char *>(d0), static_cast<const char *>(s0), n0},
               {static_cast<char *>(d1), static_cast<const char *>(s1), n1}});
    }

private:
    void loop(int t) {
        unsigned long long seen = 0;
        for (;;) {
            const std::vector<Job> *jobs;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return gen_ != seen; });
                seen = gen_;
                if (stop_) return;
                jobs = job_;
            }
            size_t total = 0;
            for (const Job &j : *jobs) total += j.n;
            const size_t per = ((total + (size_t)n_ - 1) / (size_t)n_ + 4095) & ~(size_t)4095;
            const size_t lo = per * (size_t)t, hi = std::min(total, lo + per);
            size_t base = 0;
            for (const Job &j : *jobs) {   // the byte range [lo, hi) of the jobs laid end to end
                if (base >= hi) break;
                const size_t a = std::max(lo, base), b = std::min(hi, base + j.n);
                if (a < b) stream_copy(j.d + (a - base), j.s + (a - base), b - a);
                base += j.n;
            }
            std::lock_guard<std::mutex> lk(mu_);
            if (--pending_ == 0) done_.notify_all();
        }
    }
    int n_;
    std::vector<std::thread> th_;
    std::mutex mu_;
    std::condition_variable cv_, done_;
    const std::vector<Job> *job_ = nullptr;
    int pending_ = 0;
    unsigned long long gen_ = 0;
    bool stop_ = false;
};

static int g_host_threads = 0;   // 0 = default (icnv_set_host_threads)
static int pool_threads_per_device() {
    int n = g_host_threads;
    if (n <= 0) {
        const unsigned hw = std::thread::hardware_concurrency();
        n = (int)std::min<unsigned>(16u, std::max<unsigned>(2u, hw / 2));
    }
    const int slots = std::max(1, g_slots);
    return std::max(2, n / slots);
}

// pinned staging buffer `i` of the current device context (grow-only, freed in icnv_shutdown)
static void *pinned(int i, size_t bytes) {
    Ctx &c = ctx();
    if (c.pin_bytes[i] >= bytes) return c.pin_ptr[i];
    if (c.pin_ptr[i]) {
        cudaFreeHost(c.pin_ptr[i]);
        c.pin_ptr[i] = nullptr;
        c.pin_bytes[i] = 0;
    }
    void *p = nullptr;
    cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocPortable);
    if (e != cudaSuccess) {
        set_error(ICNV_E_NOMEM, "cudaHostAlloc(%zu) for the staging ring failed: %s", bytes, cudaGetErrorString(e));
        cudaGetLastError();
        return nullptr;
    }
    c.pin_ptr[i] = p;
    c.pin_bytes[i] = bytes;
    return p;
}

// true when the driver can DMA straight from / to p (cudaHostAlloc / cudaHostRegister memory)
static bool is_pinned(const void *p) {
    if (!p) return true;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

int set_error(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

void *scratch(int slot, size_t bytes) {
    Ctx &c = ctx();
    if (bytes == 0) bytes = 16;
    if (c.slot_bytes[slot] >= bytes) return c.slot_ptr[slot];
    if (slot == SLOT_SEGS) c.up_segs.clear();          // a new allocation does not hold what was uploaded before
    if (slot == SLOT_VIT_ITEMS) c.up_items.clear();
    if (c.slot_ptr[slot]) {
        cudaStreamSynchronize(c.stream);
        cudaFree(c.slot_ptr[slot]);
        c.slot_ptr[slot] = nullptr;
        c.slot_bytes[slot] = 0;
    }
    size_t want = bytes + 256;  // slack so 16-byte over-reads at a column tail stay inside
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
        set_error(ICNV_E_NOMEM, "cudaMalloc(%zu) for scratch slot %d failed: %s", want, slot, cudaGetErrorString(e));
        cudaGetLastError();
        return nullptr;
    }
    c.slot_ptr[slot] = p;
    c.slot_bytes[slot] = bytes;
    return p;
}

static int validate_chr(int64_t G, const int32_t *chr_start, const int32_t *chr_len, int K) {
    if (!chr_start || !chr_len || K <= 0) return set_error(ICNV_E_BAD_ARG, "chromosome ranges missing");
    int64_t pos = 0;
    for (int k = 0; k < K; ++k) {
        if (chr_start[k] != pos || chr_len[k] < 0)
            return set_error(ICNV_E_BAD_ARG, "chromosome ranges must tile [0, G) contiguously (chr %d)", k);
        pos += chr_len[k];
    }
    if (pos != G) return set_error(ICNV_E_BAD_ARG, "chromosome ranges cover %lld genes, G = %lld", (long long)pos, (long long)G);
    return ICNV_OK;
}

static int validate_groups(int64_t C, const int32_t *grp_off, const int32_t *grp_idx, int n_grp, bool allow_empty) {
    if (n_grp < 0) return set_error(ICNV_E_BAD_ARG, "n_grp < 0");
    if (n_grp == 0) return allow_empty ? ICNV_OK : set_error(ICNV_E_BAD_ARG, "at least one cell group is required");
    if (!grp_off || !grp_idx) return set_error(ICNV_E_BAD_ARG, "group index lists missing");
    if (grp_off[0] != 0) return set_error(ICNV_E_BAD_ARG, "grp_off[0] must be 0");
    for (int k = 0; k < n_grp; ++k) {
        if (grp_off[k + 1] <= grp_off[k]) return set_error(ICNV_E_BAD_ARG, "group %d is empty", k);
    }
    for (int32_t i = 0; i < grp_off[n_grp]; ++i)
        if (grp_idx[i] < 0 || grp_idx[i] >= C) return set_error(ICNV_E_BAD_ARG, "cell index %d out of range", grp_idx[i]);
    return ICNV_OK;
}

static int check_flag(int *d_flag, cudaStream_t st) {
    int h = 0;
    ICNV_CUDA(cudaMemcpyAsync(&h, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    if (h & 1) return set_error(ICNV_E_NONFINITE, "non-finite value (NA/NaN/Inf) in the expression matrix");
    if (h & 2) return set_error(ICNV_E_UNDERFLOW, "Problems With Underflow");
    return ICNV_OK;
}

// group means of the columns listed in d_cells[off[k]..off[k+1]) -> d_means (G x n_grp)
static int dev_group_means(const double *dX, int64_t G, int64_t ldx, const int32_t *d_cells, const int32_t *h_off,
                           int n_grp, int apply_log, double *d_means, cudaStream_t st) {
    const int chunk = 32;  // fixed: the summation tree must not depend on the device count
    int64_t max_chunks = 0;
    for (int k = 0; k < n_grp; ++k) max_chunks = std::max<int64_t>(max_chunks, (h_off[k + 1] - h_off[k] + chunk - 1) / chunk);
    double *d_part = (double *)scratch(SLOT_PARTIAL, sizeof(double) * (size_t)G * (size_t)max_chunks);
    if (!d_part) return ICNV_E_NOMEM;
    for (int k = 0; k < n_grp; ++k) {
        int64_t n = h_off[k + 1] - h_off[k];
        int64_t n_chunks = (n + chunk - 1) / chunk;
        int rc = icnv_dev_group_partial_sums_f64(dX, G, ldx, d_cells + h_off[k], n, chunk, apply_log, d_part, st);
        if (rc) return rc;
        rc = icnv_dev_combine_partials_f64(d_part, G, n_chunks, n, d_means + G * k, st);
        if (rc) return rc;
    }
    return ICNV_OK;
}

static void destroy_streams(Ctx &c) {
    if (c.stream) cudaStreamDestroy(c.stream);
    if (c.s_h2d) cudaStreamDestroy(c.s_h2d);
    if (c.s_d2h) cudaStreamDestroy(c.s_d2h);
    c.stream = c.s_h2d = c.s_d2h = nullptr;
    for (int i = 0; i < 2; ++i) {
        if (c.ev_h2d[i]) cudaEventDestroy(c.ev_h2d[i]);
        if (c.ev_comp[i]) cudaEventDestroy(c.ev_comp[i]);
        if (c.ev_d2h[i]) cudaEventDestroy(c.ev_d2h[i]);
        c.ev_h2d[i] = c.ev_comp[i] = c.ev_d2h[i] = nullptr;
    }
}

}  // namespace icnv

using namespace icnv;

extern "C" {

// ---- lifecycle ------------------------------------------------------------------------------------

int icnv_device_count(void) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NO_DEVICE, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
    }
    return n;
}

static void free_slot(Ctx &c) {
    cudaSetDevice(c.device);
    if (c.stream) cudaStreamSynchronize(c.stream);
    for (int s = 0; s < SLOT_COUNT; ++s) {
        if (c.slot_ptr[s]) cudaFree(c.slot_ptr[s]);
        c.slot_ptr[s] = nullptr;
        c.slot_bytes[s] = 0;
    }
    for (int i = 0; i < 8; ++i) {
        if (c.pin_ptr[i]) cudaFreeHost(c.pin_ptr[i]);
        c.pin_ptr[i] = nullptr;
        c.pin_bytes[i] = 0;
    }
    destroy_streams(c);
    c.ready = false;
}

static int env_int(const char *name, int dflt, bool *set = nullptr) {
    const char *e = getenv(name);
    if (set) *set = e != nullptr;
    return e ? atoi(e) : dflt;
}

// Tuning switches come from the environment ONCE, here - never at launch time - and every one that departs from the
// default is reported, so a stray variable in a user's shell cannot silently change which kernel runs.
static void read_options(Ctx &c, bool verbose) {
    bool set;
    if (const char *e = getenv("ICNV_HMM_MODE")) c.hmm_mode = (e[0] == '0' || e[0] == 'e') ? 0 : 1;
    c.opt_cell_kernel = env_int("ICNV_CELL_KERNEL", 0);
    c.opt_cell_nt = env_int("ICNV_CELL_NT", 0);
    c.opt_cell_variant = env_int("ICNV_CELL_VARIANT", -1);
    c.opt_cell_padq = env_int("ICNV_CELL_PADQ", 1);
    c.opt_cell_lfix = env_int("ICNV_CELL_LFIX", 1);
    c.opt_slab_cells = env_int("ICNV_SLAB_CELLS", 0, &set);
    if (c.opt_slab_cells < 32 || c.opt_slab_cells > 65536) c.opt_slab_cells = 0;
    if (!verbose) return;
    static const char *names[] = {"ICNV_HMM_MODE", "ICNV_CELL_KERNEL", "ICNV_CELL_NT", "ICNV_CELL_VARIANT", "ICNV_CELL_PADQ",
                                  "ICNV_CELL_LFIX", "ICNV_SLAB_CELLS"};
    for (const char *n : names)
        if (const char *e = getenv(n)) fprintf(stderr, "[infercnv_b200] non-default tuning switch %s=%s (read once at icnv_init)\n", n, e);
}

static int init_slot(int slot, int device) {
    Ctx &c = g_ctx[slot];
    std::lock_guard<std::mutex> lk(c.mu);
    if (c.ready && c.device == device) return ICNV_OK;
    if (c.ready) free_slot(c);
    cudaError_t e = cudaSetDevice(device);
    if (e != cudaSuccess) return set_error(ICNV_E_NO_DEVICE, "cudaSetDevice(%d): %s", device, cudaGetErrorString(e));
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) return set_error(ICNV_E_NO_DEVICE, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0)
        return set_error(ICNV_E_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", device,
                         prop.major, prop.minor);
    c.sm_count = prop.multiProcessorCount;
    c.smem_optin = (int)prop.sharedMemPerBlockOptin;
    e = cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c.s_h2d, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c.s_d2h, cudaStreamNonBlocking);
    for (int i = 0; i < 2 && e == cudaSuccess; ++i) {
        e = cudaEventCreateWithFlags(&c.ev_h2d[i], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c.ev_comp[i], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c.ev_d2h[i], cudaEventDisableTiming);
    }
    if (e != cudaSuccess) return set_error(ICNV_E_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e));
    c.device = device;
    c.launches = 0;
    c.table_uploaded = false;
    c.math_tables_uploaded = false;
    c.up_segs.clear();
    c.up_items.clear();
    c.hmm_list_count = nullptr;
    c.rg_n = 0;
    read_options(c, slot == 0);
    c.ready = true;
    return ICNV_OK;
}

static std::mutex g_init_mu;

int icnv_init(int device) {
    std::lock_guard<std::mutex> lk(g_init_mu);
    Ctx &c0 = g_ctx[0];
    if (device < 0) {
        if (c0.ready) return ICNV_OK;   // keep whatever icnv_init / icnv_init_devices set up
        device = 0;
    }
    if (c0.ready && c0.device == device && g_slots == 1) return ICNV_OK;
    int n = icnv_device_count();
    if (n <= 0) return set_error(ICNV_E_NO_DEVICE, "no CUDA device available (the library has no CPU fallback)");
    if (device >= n) return set_error(ICNV_E_BAD_ARG, "device %d out of range (%d devices)", device, n);
    for (int s = 1; s < g_slots; ++s)
        if (g_ctx[s].ready) free_slot(g_ctx[s]);
    int rc = init_slot(0, device);
    if (rc) return rc;
    g_slots = 1;
    cudaSetDevice(device);
    return ICNV_OK;
}

int icnv_init_devices(int n_devices, const int *device_ids) {
    std::lock_guard<std::mutex> lk(g_init_mu);
    int n = icnv_device_count();
    if (n <= 0) return set_error(ICNV_E_NO_DEVICE, "no CUDA device available (the library has no CPU fallback)");
    if (n_devices <= 0) n_devices = n;   // "all of them"
    if (n_devices > ICNV_MAX_DEVICES || n_devices > n)
        return set_error(ICNV_E_BAD_ARG, "icnv_init_devices: %d devices requested, %d present (at most %d)", n_devices, n,
                         ICNV_MAX_DEVICES);
    for (int i = 0; i < n_devices; ++i) {
        const int d = device_ids ? device_ids[i] : i;
        if (d < 0 || d >= n) return set_error(ICNV_E_BAD_ARG, "icnv_init_devices: device %d out of range", d);
        for (int j = 0; j < i; ++j)
            if ((device_ids ? device_ids[j] : j) == d) return set_error(ICNV_E_BAD_ARG, "icnv_init_devices: device %d listed twice", d);
    }
    for (int s = n_devices; s < g_slots; ++s)
        if (g_ctx[s].ready) free_slot(g_ctx[s]);
    for (int i = 0; i < n_devices; ++i) {
        int rc = init_slot(i, device_ids ? device_ids[i] : i);
        if (rc) return rc;
    }
    g_slots = n_devices;
    cudaSetDevice(g_ctx[0].device);
    return ICNV_OK;
}

int icnv_devices_in_use(void) { return g_slots; }

int icnv_set_host_threads(int n) {
    if (n < 0 || n > 256) return set_error(ICNV_E_BAD_ARG, "icnv_set_host_threads: 0 (default) .. 256");
    g_host_threads = n;
    return ICNV_OK;
}

void icnv_shutdown(void) {
    std::lock_guard<std::mutex> lk(g_init_mu);
    for (int s = 0; s < ICNV_MAX_DEVICES; ++s) {
        Ctx &c = g_ctx[s];
        std::lock_guard<std::mutex> lk2(c.mu);
        if (c.ready) free_slot(c);
    }
    g_slots = 0;
}

const char *icnv_last_error(void) { return g_err; }
const char *icnv_version(void) { return "infercnv_b200 0.1.0 (sm_90a)"; }
int64_t icnv_launch_count(void) {
    int64_t n = 0;
    for (int s = 0; s < std::max(1, g_slots); ++s) n += g_ctx[s].launches.load();
    return n;
}

// ---- device-side composition of the smooth block ---------------------------------------------------------

int icnv_dev_smooth_block_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *chr_start,
                              const int32_t *chr_len, int K, const int32_t *grp_off, const int32_t *grp_idx, int n_grp,
                              int apply_log, double threshold, int window, int use_bounds, void *stream) {
    ICNV_REQUIRE_READY();
    if (!X || !Y || G <= 0 || C <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_dev_smooth_block_f64: bad argument");
    int rc = validate_chr(G, chr_start, chr_len, K);
    if (rc) return rc;
    rc = validate_groups(C, grp_off, grp_idx, n_grp, false);
    if (rc) return rc;
    cudaStream_t st = pick_stream(stream);
    const int64_t n_ref = grp_off[n_grp];

    // index lists: [ref cells as given | 0..n_ref-1 (columns of the compact pass-1 buffer)]
    int32_t *d_idx = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * 2 * (size_t)n_ref);
    if (!d_idx) return ICNV_E_NOMEM;
    std::vector<int32_t> iota((size_t)n_ref);
    std::iota(iota.begin(), iota.end(), 0);
    ICNV_CUDA(cudaMemcpyAsync(d_idx, grp_idx, sizeof(int32_t) * (size_t)n_ref, cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaMemcpyAsync(d_idx + n_ref, iota.data(), sizeof(int32_t) * (size_t)n_ref, cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaStreamSynchronize(st));  // iota is a stack-lifetime host buffer

    double *d_means = (double *)scratch(SLOT_MEANS, sizeof(double) * (size_t)G * (size_t)n_grp);
    double *d_b = (double *)scratch(SLOT_BOUNDS, sizeof(double) * (size_t)G * 6);
    double *d_T = (double *)scratch(SLOT_TMP, sizeof(double) * (size_t)G * (size_t)n_ref);
    int *d_flag = (int *)scratch(SLOT_MISC, 64);
    if (!d_means || !d_b || !d_T || !d_flag) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
    double *lo1 = d_b, *hi1 = d_b + G, *mid1 = d_b + 2 * G, *lo2 = d_b + 3 * G, *hi2 = d_b + 4 * G, *mid2 = d_b + 5 * G;

    // pass 0: step-8 reference means on (log-transformed) input   (ops.R:771 -> :1708)
    rc = dev_group_means(X, G, G, d_idx, grp_off, n_grp, apply_log ? 1 : 0, d_means, st);
    if (rc) return rc;
    rc = icnv_dev_bounds_from_means_f64(d_means, G, n_grp, lo1, hi1, mid1, st);
    if (rc) return rc;
    // pass 1: steps 4..11 on the reference cells only -> compact buffer T (one column per list entry)
    rc = icnv_dev_cell_pipeline_f64(X, G, G, d_idx, n_ref, d_T, G, chr_start, chr_len, K, apply_log,
                                    use_bounds ? lo1 : nullptr, use_bounds ? hi1 : nullptr, use_bounds ? nullptr : mid1,
                                    threshold, window, 1, nullptr, nullptr, nullptr, 0, d_flag, st);
    if (rc) return rc;
    // step-12 reference means on the centred, smoothed reference cells   (ops.R:952)
    rc = dev_group_means(d_T, G, G, d_idx + n_ref, grp_off, n_grp, 0, d_means, st);
    if (rc) return rc;
    rc = icnv_dev_bounds_from_means_f64(d_means, G, n_grp, lo2, hi2, mid2, st);
    if (rc) return rc;
    // pass 2: every cell, read once, written once
    rc = icnv_dev_cell_pipeline_f64(X, G, G, nullptr, C, Y, G, chr_start, chr_len, K, apply_log,
                                    use_bounds ? lo1 : nullptr, use_bounds ? hi1 : nullptr, use_bounds ? nullptr : mid1,
                                    threshold, window, 1, use_bounds ? lo2 : nullptr, use_bounds ? hi2 : nullptr,
                                    use_bounds ? nullptr : mid2, 1, d_flag, st);
    if (rc) return rc;
    return ICNV_OK;
}

// ---- host-pointer entry points --------------------------------------------------------------------------------

#define ICNV_HOST_PROLOGUE()                       \
    ICNV_REQUIRE_READY();                          \
    Ctx &c = ctx();                                \
    std::lock_guard<std::mutex> lk(c.mu);          \
    ICNV_CUDA(cudaSetDevice(c.device));            \
    cudaStream_t st = c.stream;                    \
    (void)st

static int upload_matrix(const double *X, int64_t n, double **dX, int slot, cudaStream_t st) {
    *dX = (double *)scratch(slot, sizeof(double) * (size_t)n);
    if (!*dX) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemcpyAsync(*dX, X, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice, st));
    return ICNV_OK;
}

// The columns idx[0 .. n) of the host matrix X (G rows) into a compact device buffer (SLOT_IN), each run of consecutive
// indices as one copy, and the identity list 0 .. n-1 into SLOT_IDX.  The caller has checked the indices.
static int upload_listed_columns(const double *X, int64_t G, const int32_t *idx, int64_t n, double **dX, int32_t **d_ident,
                                 cudaStream_t st) {
    *dX = (double *)scratch(SLOT_IN, sizeof(double) * (size_t)std::max<int64_t>(G * n, 1));
    *d_ident = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)n);
    if (!*dX || !*d_ident) return ICNV_E_NOMEM;
    std::vector<int32_t> ident((size_t)n);
    std::iota(ident.begin(), ident.end(), 0);
    for (int64_t i = 0; G > 0 && i < n;) {
        int64_t j = i + 1;
        while (j < n && idx[j] == idx[j - 1] + 1) ++j;
        ICNV_CUDA(cudaMemcpyAsync(*dX + G * i, X + G * (int64_t)idx[i], sizeof(double) * (size_t)G * (size_t)(j - i),
                                  cudaMemcpyHostToDevice, st));
        i = j;
    }
    ICNV_CUDA(cudaMemcpyAsync(*d_ident, ident.data(), sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaStreamSynchronize(st));   // `ident` is pageable host memory that goes out of scope
    return ICNV_OK;
}

int icnv_ref_means_f64(const double *X, int64_t G, int64_t C, const int32_t *grp_off, const int32_t *grp_idx, int n_grp,
                       int inv_log, double *means) {
    ICNV_HOST_PROLOGUE();
    if (!X || !means || G <= 0 || C <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_ref_means_f64: bad argument");
    int rc = validate_groups(C, grp_off, grp_idx, n_grp, false);
    if (rc) return rc;
    double *dX;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    int64_t n_ref = grp_off[n_grp];
    int32_t *d_idx = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)n_ref);
    double *d_means = (double *)scratch(SLOT_MEANS, sizeof(double) * (size_t)G * (size_t)n_grp);
    if (!d_idx || !d_means) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemcpyAsync(d_idx, grp_idx, sizeof(int32_t) * (size_t)n_ref, cudaMemcpyHostToDevice, st));
    rc = dev_group_means(dX, G, G, d_idx, grp_off, n_grp, inv_log ? 2 : 0, d_means, st);
    if (rc) return rc;
    if (inv_log && (rc = icnv_dev_invlog_finish_f64(d_means, G * n_grp, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(means, d_means, sizeof(double) * (size_t)G * (size_t)n_grp, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

// one pass of the per-cell kernel over a host matrix: upload, run, download
static int host_cell_pipeline(const double *X, double *Y, int64_t G, int64_t C, const int32_t *chr_start,
                              const int32_t *chr_len, int K, const double *h_means, int n_grp, int use_bounds,
                              int window, int center, cudaStream_t st) {
    double *dX, *dY;
    int rc;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(G * C));
    int *d_flag = (int *)scratch(SLOT_MISC, 64);
    if (!dY || !d_flag) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
    double *lo = nullptr, *hi = nullptr, *mid = nullptr;
    if (h_means) {
        double *d_means = (double *)scratch(SLOT_MEANS, sizeof(double) * (size_t)G * (size_t)n_grp);
        double *d_b = (double *)scratch(SLOT_BOUNDS, sizeof(double) * (size_t)G * 6);
        if (!d_means || !d_b) return ICNV_E_NOMEM;
        ICNV_CUDA(cudaMemcpyAsync(d_means, h_means, sizeof(double) * (size_t)G * (size_t)n_grp, cudaMemcpyHostToDevice, st));
        if ((rc = icnv_dev_bounds_from_means_f64(d_means, G, n_grp, d_b, d_b + G, d_b + 2 * G, st))) return rc;
        if (use_bounds) {
            lo = d_b;
            hi = d_b + G;
        } else {
            mid = d_b + 2 * G;
        }
    }
    std::vector<int32_t> one_start{0}, one_len{(int32_t)G};
    const int32_t *cs = chr_start ? chr_start : one_start.data();
    const int32_t *cl = chr_len ? chr_len : one_len.data();
    int kk = chr_start ? K : 1;
    rc = icnv_dev_cell_pipeline_f64(dX, G, G, nullptr, C, dY, G, cs, cl, kk, 0, lo, hi, mid, 0.0, window, center, nullptr,
                                    nullptr, nullptr, 0, d_flag, st);
    if (rc) return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    return check_flag(d_flag, st);
}

int icnv_subtract_ref_f64(const double *X, double *Y, int64_t G, int64_t C, const double *means, int n_grp,
                          int use_bounds) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || !means || G <= 0 || C <= 0 || n_grp <= 0)
        return set_error(ICNV_E_BAD_ARG, "icnv_subtract_ref_f64: bad argument");
    return host_cell_pipeline(X, Y, G, C, nullptr, nullptr, 0, means, n_grp, use_bounds, 0, 0, st);
}

int icnv_smooth_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *chr_start, const int32_t *chr_len,
                    int K, int window) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || G <= 0 || C <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_smooth_f64: bad argument");
    int rc = validate_chr(G, chr_start, chr_len, K);
    if (rc) return rc;
    if (window >= 2 && (window & 1) == 0)
        return set_error(ICNV_E_BAD_ARG, "window_length %d is even: refusing (the reference's result is accidental)", window);
    return host_cell_pipeline(X, Y, G, C, chr_start, chr_len, K, nullptr, 0, 0, window, 0, st);
}

int icnv_center_f64(const double *X, double *Y, int64_t G, int64_t C, int use_median) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || G <= 0 || C <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_center_f64: bad argument");
    return host_cell_pipeline(X, Y, G, C, nullptr, nullptr, 0, nullptr, 0, 0, 0, use_median ? 1 : 2, st);
}

// ---- slab pipeline: cells are independent once the reference means are known, so the matrix moves
// through the GPU in slabs of SLAB_CELLS columns - H2D of slab i+1, kernels on slab i and D2H of slab
// i-1 run concurrently on three streams (double-buffered device slabs).  PCIe, not the kernels, bounds
// the host-pointer entry points; this hides everything but the slower copy direction. ---------------
static const int64_t SLAB_CELLS = 1024;
static const int64_t SLAB_CELLS_SMOOTH = 256;

struct HmmModel {
    int m;
    const double *Pi, *delta, *mean, *sd;
};

/* qnorm(p, mu, sigma) for 0 < p < 1: Wichura's AS241 (PPND16), the algorithm of R's qnorm, with the published
 * coefficients in the order of operations of Python's NormalDist.inv_cdf (hmm.i3_mean_delta gives the same bits). */
static double qnorm_as241(double p, double mu, double sigma) {
    const double q = p - 0.5;
    double r, val;
    if (std::fabs(q) <= .425) {
        r = .180625 - q * q;
        val = q * (((((((r * 2509.0809287301226727 + 33430.575583588128105) * r + 67265.770927008700853) * r +
                        45921.953931549871457) * r + 13731.693765509461125) * r + 1971.5909503065514427) * r +
                     133.14166789178437745) * r + 3.387132872796366608) /
              (((((((r * 5226.4952788528545610 + 28729.085735721942674) * r + 39307.89580009271061) * r +
                   21213.794301586595867) * r + 5394.1960214247511077) * r + 687.1870074920579083) * r +
                42.313330701600911252) * r + 1.);
        return mu + sigma * val;
    }
    r = std::sqrt(-std::log(q < 0 ? p : 1. - p));
    if (r <= 5.) {
        r += -1.6;
        val = (((((((r * 7.7454501427834140764e-4 + .0227238449892691845833) * r + .24178072517745061177) * r +
                   1.27045825245236838258) * r + 3.64784832476320460504) * r + 5.7694972214606914055) * r +
                4.6303378461565452959) * r + 1.42343711074968357734) /
              (((((((r * 1.05075007164441684324e-9 + 5.475938084995344946e-4) * r + .0151986665636164571966) * r +
                   .14810397642748007459) * r + .68976733498510000455) * r + 1.6763848301838038494) * r +
                2.05319162663775882187) * r + 1.);
    } else {
        r += -5.;
        val = (((((((r * 2.01033439929228813265e-7 + 2.71155556874348757815e-5) * r + .0012426609473880784386) * r +
                   .026532189526576123093) * r + .29656057182850489123) * r + 1.7848265399172913358) * r +
                5.4637849111641143699) * r + 6.6579046435011037772) /
              (((((((r * 2.04426310338993978564e-15 + 1.4215117583164458887e-7) * r + 1.8463183175100546818e-5) * r +
                   7.868691311456132591e-4) * r + .0148753612908506148525) * r + .13692988092273580531) * r +
                .59983220655588793769) * r + 1.);
    }
    if (q < 0.0) val = -val;
    return mu + sigma * val;
}

/* What the fused i3 call adds to the slab pipeline: the i3 model, fixed from the reference cells' final values between
 * the reference pre-pass and the first slab, and the median filter over index lists.  With the filter, the cells are cut
 * into units - runs of columns no list's span crosses, at least a slab long - and a unit's Y stays on the device until its
 * last slab is done; the filter then runs on the whole unit and F leaves behind it. */
struct I3Fused {
    double p_val, t;
    double *model;                       // out: mu, sigma, mean_delta (NULL: this device does not report them)
    double *F;                           // median-filtered Y; NULL: no filter
    const int32_t *mf_off, *mf_idx;
    int n_mf, mf_window;
    std::vector<std::pair<int64_t, int64_t>> spans;   // merged [lo, hi) column spans of the lists, ascending
    // the smallest column >= x that no span crosses
    int64_t cut_at_or_after(int64_t x) const {
        auto it = std::upper_bound(spans.begin(), spans.end(), std::make_pair(x, INT64_MAX));
        if (it != spans.begin() && std::prev(it)->first < x && x < std::prev(it)->second) return std::prev(it)->second;
        return x;
    }
    // the column nearest x that no span crosses (ties: the lower one)
    int64_t cut_near(int64_t x) const {
        auto it = std::upper_bound(spans.begin(), spans.end(), std::make_pair(x, INT64_MAX));
        if (it != spans.begin() && std::prev(it)->first < x && x < std::prev(it)->second) {
            const int64_t a = std::prev(it)->first, b = std::prev(it)->second;
            return (x - a <= b - x) ? a : b;
        }
        return x;
    }
};

/* What the fused group-mode calls change in the slab pipeline.  The cells go through it in HMM-list order - every list
 * entry, then the cells in no list in column order - so that a group's 32-entry chunks (dev_group_means' summation tree)
 * lie in one slab each: pipeline position p is column order[p].  Slabs gather their columns from X and scatter Y back,
 * each column written from the one position that owns it (its last listing; an unlisted cell's own position).  The group
 * means build up slab by slab; after the last slab the group Viterbi runs on them and every owned column of `states`
 * takes its group's trace (255: in no list).  A device's positions start and end at group boundaries. */
struct GroupHmm {
    const int32_t *off;              // hmm_off[n_hmm + 1]
    int n_hmm;
    int64_t n_listed;                // off[n_hmm]
    std::vector<int32_t> order;      // position -> column
    std::vector<int32_t> grp_at;     // position -> its group (the listed positions)
    std::vector<char> owns;          // position -> whether it writes its column's Y and states
    std::vector<double> sd_med;      // i6: per-group median sd (viterbi_impl's); empty: i3 (sigma for every group)
    uint8_t *states;
    // the column of position p
    int64_t col(int64_t p) const { return order[(size_t)p]; }
    // the smallest position >= x at which a slab may end: a group boundary, a chunk boundary inside a group, or any
    // position among the unlisted cells
    bool may_cut(int64_t x) const {
        if (x >= n_listed) return true;
        return (x - off[grp_at[(size_t)x]]) % 32 == 0;
    }
    // the position nearest x that is a group boundary (ties: the lower one) - where the devices' shares are cut
    int64_t group_cut_near(int64_t x) const {
        if (x >= n_listed) return x;
        const int k = grp_at[(size_t)x];
        return (x - off[k] <= off[k + 1] - x) ? off[k] : off[k + 1];
    }
    // the first group whose entries start at or after position x
    int group_at_or_after(int64_t x) const {
        return (int)(std::lower_bound(off, off + n_hmm + 1, (int32_t)std::min<int64_t>(x, n_listed)) - off);
    }
};

// Several devices: every device's range allocates its buffers first and waits here for the others, so that a range whose
// buffers do not fit stops every device before any of them has written output.
struct StartGate {
    std::mutex mu;
    std::condition_variable cv;
    int left;
    bool ok = true;
    int first_fail = -1;               // the device whose own failure closed the gate
    std::vector<char> in;
    StartGate(int n_dev, int n_threads) : left(n_threads), in((size_t)n_dev, 0) {}
    // device d has allocated (good) or failed; returns whether every device may start.  A second arrival returns at once.
    bool arrive(int d, bool good) {
        std::unique_lock<std::mutex> lk(mu);
        if (in[(size_t)d]) return ok;
        in[(size_t)d] = 1;
        if (!good && first_fail < 0) first_fail = d;
        ok = ok && good;
        if (--left == 0) cv.notify_all();
        else cv.wait(lk, [&] { return left == 0; });
        return ok;
    }
};

// Y (optional) = smooth block of X; states (optional) = per-cell Viterbi of the block's output (or of X
// itself when do_smooth == 0).
// states (int32, -1 = unassigned) or states8 (uint8, 255 = unassigned): at most one of them is non-NULL.
// Works on the cells [c_lo, c_hi) of the G x C host matrices on the calling thread's device context; the reference
// groups index the whole matrix (every device reduces all reference cells itself, in list order).
// i3 (with do_smooth, hmm == NULL): the per-cell HMM uses the i3 model of the block's reference cells, and F (optional)
// is the median filter of Y; [c_lo, c_hi) must not cut a list's span.
// grp (with do_smooth, states == states8 == NULL, no F): the group-mode HMM of GroupHmm; [c_lo, c_hi) are pipeline positions
// and start and end at group boundaries.
static int host_pipeline_range(Ctx &c, const double *X, double *Y, int32_t *states, uint8_t *states8, int64_t G, int64_t c_lo,
                               int64_t c_hi, const int32_t *chr_start, const int32_t *chr_len, int K, int do_smooth,
                               const int32_t *grp_off, const int32_t *grp_idx, int n_grp, int apply_log, double threshold,
                               int window, int use_bounds, const HmmModel *hmm, CopyPool *pool, const I3Fused *i3 = nullptr,
                               StartGate *gate = nullptr, const GroupHmm *grp = nullptr) {
    cudaStream_t sc = c.stream, sh = c.s_h2d, sd = c.s_d2h;
    int rc;
    const int64_t C = c_hi - c_lo;
    const bool mf = i3 && i3->F;
    const bool has_hmm = (hmm || i3) && !grp;   // the per-cell HMM, slab by slab
    int *d_flag = (int *)scratch(SLOT_MISC, 64);
    if (!d_flag) return ICNV_E_NOMEM;
    if (mf) d_flag += 4;   // icnv_dev_median_filter_f64 clears and sets the slot's first word for itself
    ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), sc));
    double *lo1 = nullptr, *hi1 = nullptr, *mid1 = nullptr, *lo2 = nullptr, *hi2 = nullptr, *mid2 = nullptr;
    // page-locked caller memory goes over PCIe directly; anything else through the pinned ring (pool != NULL)
    const bool stage_in = pool && !is_pinned(X);
    const bool stage_out = pool && ((Y && !is_pinned(Y)) || (states && !is_pinned(states)) || (states8 && !is_pinned(states8)) ||
                                    (mf && !is_pinned(i3->F)));

    // ---- slabs ------------------------------------------------------------------------------------------
    // Fill and drain of the copy pipeline cost one slab each way.  Without the HMM a slab's kernel time (~0.05 ms per 256
    // cells) is far below its PCIe time (0.37 ms), so small slabs only shorten fill / drain; the per-cell Viterbi is bounded
    // below by its longest chromosome's serial recursion whatever the slab size, so HMM calls keep the measured 1024.
    int64_t slab_cells = has_hmm ? SLAB_CELLS : SLAB_CELLS_SMOOTH;
    if (stage_in || stage_out) {
        // pageable caller memory: fewer, larger hand-overs to the copy threads - about 320 MB of input per slab (4000 cells at
        // 10 000 genes), but at least ten slabs so that filling and draining the pipeline stays a small share
        int64_t by_bytes = ((int64_t)(320e6 / (8.0 * (double)G)) + 31) / 32 * 32;
        by_bytes = std::max<int64_t>(256, std::min<int64_t>(8192, by_bytes));
        const int64_t by_count = std::max<int64_t>(SLAB_CELLS, ((C + 9) / 10 + 31) / 32 * 32);
        slab_cells = std::min(by_bytes, by_count);
    }
    if (c.opt_slab_cells) slab_cells = c.opt_slab_cells;
    const int64_t slab = std::max<int64_t>(1, std::min<int64_t>(slab_cells, C));
    // slab i is the cells [c_lo + s_at[i], c_lo + s_at[i + 1]).  With the median filter the slabs are cut inside units (see
    // I3Fused); unit_lo[i] is the first cell of slab i's unit, unit_end[i] marks its last slab.
    std::vector<int64_t> s_at{0}, unit_lo;
    std::vector<char> unit_end;
    int64_t max_unit = 0;
    for (int64_t u0 = 0; grp && u0 < C;) {   // group mode: a slab ends where no 32-entry chunk is cut
        int64_t q = std::min(C, u0 + slab);
        while (!grp->may_cut(c_lo + q)) --q;
        if (q == u0) {   // a slab shorter than a chunk: round up instead
            q = u0 + 1;
            while (!grp->may_cut(c_lo + q)) ++q;
        }
        s_at.push_back(q);
        u0 = q;
    }
    for (int64_t u0 = 0; !grp && u0 < C;) {
        const int64_t u1 = mf ? std::min(C, i3->cut_at_or_after(c_lo + u0 + slab) - c_lo) : C;
        for (int64_t s = u0; s < u1; s += slab) {
            s_at.push_back(std::min(u1, s + slab));
            unit_lo.push_back(u0);
            unit_end.push_back(s + slab >= u1);
        }
        max_unit = std::max(max_unit, u1 - u0);
        u0 = u1;
    }
    int64_t slab_cap = slab;
    for (size_t i = 0; i + 1 < s_at.size(); ++i) slab_cap = std::max(slab_cap, s_at[i + 1] - s_at[i]);
    const size_t slab_elems = (size_t)G * (size_t)slab_cap;
    double *dIn[2], *dOut[2] = {nullptr, nullptr};
    uint8_t *dSt[2] = {nullptr, nullptr};
    int32_t *dW[2] = {nullptr, nullptr};
    double *pIn[2] = {nullptr, nullptr}, *pOut[2] = {nullptr, nullptr}, *pF[2] = {nullptr, nullptr};
    void *pSt[2] = {nullptr, nullptr};
    const size_t st_elem = states ? sizeof(int32_t) : 1;
    // the median filter's unit buffers (Y and F of the unit) take the place of the two output slabs
    double *dYu = nullptr, *dFu = nullptr;
    if (mf) {
        const size_t unit_bytes = sizeof(double) * (size_t)G * (size_t)max_unit;
        dYu = (double *)scratch(SLOT_SLAB_OUT0, unit_bytes);
        dFu = dYu ? (double *)scratch(SLOT_SLAB_OUT1, unit_bytes) : nullptr;
        if (!dYu || !dFu)
            return set_error(ICNV_E_NOMEM, "median filter: a run of %lld cells that no index list's span crosses needs 2 x %zu "
                             "bytes on device %d: %s", (long long)max_unit, unit_bytes, c.device, icnv_last_error());
    }
    for (int b = 0; b < 2; ++b) {
        dIn[b] = (double *)scratch(SLOT_SLAB_IN0 + b, sizeof(double) * slab_elems);
        if (!dIn[b]) return ICNV_E_NOMEM;
        if (do_smooth && !mf) {
            dOut[b] = (double *)scratch(SLOT_SLAB_OUT0 + b, sizeof(double) * slab_elems);
            if (!dOut[b]) return ICNV_E_NOMEM;
        }
        if (has_hmm) {
            dSt[b] = (uint8_t *)scratch(SLOT_SLAB_ST0 + b, slab_elems);
            if (!dSt[b]) return ICNV_E_NOMEM;
            if (states) {
                dW[b] = (int32_t *)scratch(SLOT_SLAB_W0 + b, sizeof(int32_t) * slab_elems);
                if (!dW[b]) return ICNV_E_NOMEM;
            }
        }
        if (stage_in && !(pIn[b] = (double *)pinned(b, sizeof(double) * slab_elems))) return ICNV_E_NOMEM;
        if (stage_out && do_smooth && Y && !(pOut[b] = (double *)pinned(2 + b, sizeof(double) * slab_elems))) return ICNV_E_NOMEM;
        if (stage_out && has_hmm && !(pSt[b] = pinned(4 + b, st_elem * slab_elems))) return ICNV_E_NOMEM;
        if (stage_out && mf && !(pF[b] = (double *)pinned(6 + b, sizeof(double) * slab_elems))) return ICNV_E_NOMEM;
    }
    const int64_t n_slabs = (int64_t)s_at.size() - 1;
    auto slab_cells_of = [&](int64_t i) { return s_at[(size_t)i + 1] - s_at[(size_t)i]; };
    // group mode: runs of consecutive columns among slab i's positions, f(first slab column, first matrix column, length);
    // owners_only: the positions that write their column
    auto col_runs = [&](int64_t i, bool owners_only, const std::function<int(int64_t, int64_t, int64_t)> &f) -> int {
        const int64_t p0 = c_lo + s_at[(size_t)i], p1 = c_lo + s_at[(size_t)i + 1];
        for (int64_t p = p0; p < p1;) {
            if (owners_only && !grp->owns[(size_t)p]) {
                ++p;
                continue;
            }
            int64_t q = p + 1;
            while (q < p1 && (!owners_only || grp->owns[(size_t)q]) && grp->col(q) == grp->col(q - 1) + 1) ++q;
            if (int rc2 = f(p - p0, grp->col(p), q - p)) return rc2;
            p = q;
        }
        return ICNV_OK;
    };
    // group mode: this range's groups [k_lo, k_hi); per slab i its chunks [ch_at[i], ch_at[i + 1]) (pairs: first slab
    // column, entries) and group segments [sg_at[i], sg_at[i + 1]) (see slab_combine_kernel), uploaded once
    const int k_lo = grp ? grp->group_at_or_after(c_lo) : 0, k_hi = grp ? grp->group_at_or_after(c_hi) : 0;
    const int64_t n_loc = k_hi - k_lo;
    std::vector<int64_t> ch_at{0}, sg_at{0};
    double *d_gm = nullptr, *d_gsd = nullptr, *d_part = nullptr;
    int32_t *d_chunks = nullptr, *d_segs = nullptr;
    uint8_t *d_gst = nullptr;
    if (grp) {
        std::vector<int32_t> chunks, segs;
        int64_t max_ch = 1;
        for (int64_t i = 0; i < n_slabs; ++i) {
            const int64_t p0 = c_lo + s_at[(size_t)i], p1 = c_lo + s_at[(size_t)i + 1];
            const int64_t first = (int64_t)chunks.size() / 2;
            for (int k = p0 < grp->n_listed ? grp->grp_at[(size_t)p0] : grp->n_hmm; k < grp->n_hmm && grp->off[k] < p1; ++k) {
                const int64_t a = grp->off[k], e = grp->off[k + 1];
                const int64_t ch0 = (int64_t)chunks.size() / 2 - first;
                for (int64_t q = std::max(a, p0); q < std::min(e, p1); q += 32) {   // max(a, p0) starts a chunk
                    chunks.push_back((int32_t)(q - p0));
                    chunks.push_back((int32_t)std::min<int64_t>(32, e - q));
                }
                segs.insert(segs.end(), {(int32_t)ch0, (int32_t)((int64_t)chunks.size() / 2 - first - ch0), a >= p0, e <= p1,
                                         (int32_t)(e - a), (int32_t)(k - k_lo)});
            }
            ch_at.push_back((int64_t)chunks.size() / 2);
            sg_at.push_back((int64_t)segs.size() / 6);
            max_ch = std::max(max_ch, ch_at.back() - ch_at[ch_at.size() - 2]);
        }
        d_gm = (double *)scratch(SLOT_GRP_MEANS, sizeof(double) * ((size_t)G + 1) * (size_t)n_loc);
        d_part = (double *)scratch(SLOT_GRP_PART, sizeof(double) * (size_t)G * (size_t)(max_ch + 2));
        d_chunks = (int32_t *)scratch(SLOT_GRP_TAB, sizeof(int32_t) * (chunks.size() + segs.size()));
        d_gst = (uint8_t *)scratch(SLOT_GRP_ST, (size_t)G * (size_t)n_loc);
        if (!d_gm || !d_part || !d_chunks || !d_gst)
            return set_error(ICNV_E_NOMEM, "group-mode HMM: the means, traces and slab tables of %lld groups do not fit on device "
                             "%d: %s", (long long)n_loc, c.device, icnv_last_error());
        d_gsd = d_gm + (size_t)G * (size_t)n_loc;
        d_segs = d_chunks + chunks.size();
        ICNV_CUDA(cudaMemcpyAsync(d_chunks, chunks.data(), sizeof(int32_t) * chunks.size(), cudaMemcpyHostToDevice, sc));
        ICNV_CUDA(cudaMemcpyAsync(d_segs, segs.data(), sizeof(int32_t) * segs.size(), cudaMemcpyHostToDevice, sc));
        ICNV_CUDA(cudaStreamSynchronize(sc));   // the tables are pageable host vectors
    }
    // results of slab j leave the pinned ring for the caller's buffers (after its D2H has completed); together with the
    // input of slab `in` entering the ring when in >= 0 - one hand-over to the copy threads for both directions
    auto host_copies = [&](int64_t in, int64_t out) -> int {
        if (grp) {   // the slab's columns gathered into the ring; Y scattered from it to the columns its positions own
            std::vector<CopyPool::Job> jobs;
            if (in >= 0 && in < n_slabs && stage_in) {
                const int b = (int)(in & 1);
                if (in >= 2) ICNV_CUDA(cudaEventSynchronize(c.ev_h2d[b]));
                col_runs(in, false, [&](int64_t r, int64_t col, int64_t n) {
                    jobs.push_back({(char *)(pIn[b] + G * r), (const char *)(X + G * col), sizeof(double) * (size_t)(G * n)});
                    return ICNV_OK;
                });
            }
            if (out >= 0 && out < n_slabs && stage_out) {
                const int b = (int)(out & 1);
                ICNV_CUDA(cudaEventSynchronize(c.ev_d2h[b]));
                col_runs(out, true, [&](int64_t r, int64_t col, int64_t n) {
                    jobs.push_back({(char *)(Y + G * col), (const char *)(pOut[b] + G * r), sizeof(double) * (size_t)(G * n)});
                    return ICNV_OK;
                });
            }
            pool->copyv(jobs);
            return ICNV_OK;
        }
        void *d0 = nullptr, *d1 = nullptr;
        const void *s0 = nullptr, *s1 = nullptr;
        size_t n0 = 0, n1 = 0;
        if (in >= 0 && in < n_slabs && stage_in) {
            const int b = (int)(in & 1);
            if (in >= 2) ICNV_CUDA(cudaEventSynchronize(c.ev_h2d[b]));   // the ring slot has been read by slab in-2's H2D
            d0 = pIn[b];
            s0 = X + G * (c_lo + s_at[(size_t)in]);
            n0 = sizeof(double) * (size_t)G * (size_t)slab_cells_of(in);
        }
        if (out >= 0 && out < n_slabs && stage_out) {
            const int b = (int)(out & 1);
            ICNV_CUDA(cudaEventSynchronize(c.ev_d2h[b]));
            const int64_t c0 = c_lo + s_at[(size_t)out], nc = slab_cells_of(out);
            if (do_smooth && Y) {
                d1 = Y + G * c0;
                s1 = pOut[b];
                n1 = sizeof(double) * (size_t)G * (size_t)nc;
            }
            if (hmm) {   // the states ride along: a third job is not worth a second hand-over
                char *dst = states ? (char *)(states + G * c0) : (char *)(states8 + G * c0);
                if (n1 == 0) {
                    d1 = dst;
                    s1 = pSt[b];
                    n1 = st_elem * (size_t)G * (size_t)nc;
                } else {
                    pool->copy2(d0, s0, n0, d1, s1, n1);
                    d0 = dst;
                    s0 = pSt[b];
                    n0 = st_elem * (size_t)G * (size_t)nc;
                    d1 = nullptr;
                    n1 = 0;
                }
            }
        }
        pool->copy2(d0, s0, n0, d1, s1, n1);
        return ICNV_OK;
    };
    // H2D of slab i (buffer i & 1) may start once the kernels of slab i-2 have consumed the buffer
    auto issue_h2d = [&](int64_t i) -> int {
        const int b = (int)(i & 1);
        const int64_t c0 = c_lo + s_at[(size_t)i], nc = slab_cells_of(i);
        if (i >= 2) ICNV_CUDA(cudaStreamWaitEvent(sh, c.ev_comp[b], 0));
        if (grp && !stage_in) {   // page-locked X: one copy per run of consecutive columns
            int rc2 = col_runs(i, false, [&](int64_t r, int64_t col, int64_t n) -> int {
                ICNV_CUDA(cudaMemcpyAsync(dIn[b] + G * r, X + G * col, sizeof(double) * (size_t)(G * n), cudaMemcpyHostToDevice, sh));
                return ICNV_OK;
            });
            if (rc2) return rc2;
        } else {
            ICNV_CUDA(cudaMemcpyAsync(dIn[b], stage_in ? pIn[b] : X + G * c0, sizeof(double) * (size_t)G * (size_t)nc,
                                      cudaMemcpyHostToDevice, sh));
        }
        ICNV_CUDA(cudaEventRecord(c.ev_h2d[b], sh));
        return ICNV_OK;
    };
    int64_t h2d_issued = 0;
    double i3_Pi[9], i3_delta[3], i3_mean[3], i3_sd[3];
    const HmmModel i3_hmm{3, i3_Pi, i3_delta, i3_mean, i3_sd};
    // the median filter's local lists and events: F of unit u leaves (ev_f) before unit u+1's filter overwrites dFu
    std::vector<int32_t> mf_off_u, mf_idx_u;
    cudaEvent_t ev_mf = nullptr, ev_f[2] = {nullptr, nullptr};
    struct EventsGuard {
        cudaEvent_t *e[3];
        ~EventsGuard() {
            for (cudaEvent_t *p : e)
                if (*p) cudaEventDestroy(*p);
        }
    } ev_guard{{&ev_mf, &ev_f[0], &ev_f[1]}};
    if (mf) {
        ICNV_CUDA(cudaEventCreateWithFlags(&ev_mf, cudaEventDisableTiming));
        ICNV_CUDA(cudaEventCreateWithFlags(&ev_f[0], cudaEventDisableTiming));
        ICNV_CUDA(cudaEventCreateWithFlags(&ev_f[1], cudaEventDisableTiming));
    }

    if (do_smooth) {
        // ---- reference pre-passes on a compact copy of the reference columns (<= ~10 % of the cells) ----
        const int64_t n_ref = grp_off[n_grp];
        double *d_ref = (double *)scratch(SLOT_REFX, sizeof(double) * (size_t)G * (size_t)n_ref);
        double *d_T = (double *)scratch(SLOT_TMP, sizeof(double) * (size_t)G * (size_t)n_ref);
        double *d_means = (double *)scratch(SLOT_MEANS, sizeof(double) * (size_t)G * (size_t)n_grp);
        double *d_b = (double *)scratch(SLOT_BOUNDS, sizeof(double) * (size_t)G * 6);
        int32_t *d_iota = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)n_ref);
        if (!d_ref || !d_T || !d_means || !d_b || !d_iota) return ICNV_E_NOMEM;
        if (gate && !gate->arrive(current_slot(), true))
            return set_error(ICNV_E_NOMEM, "stopped before any output: another device could not allocate its buffers");
        for (int64_t i = 0; i < n_ref;) {  // runs of consecutive cells go up in one copy (staged: a ring slot at a time)
            int64_t j = i + 1;
            while (j < n_ref && grp_idx[j] == grp_idx[j - 1] + 1) ++j;
            if (!stage_in) {
                ICNV_CUDA(cudaMemcpyAsync(d_ref + G * i, X + G * (int64_t)grp_idx[i], sizeof(double) * (size_t)(G * (j - i)),
                                          cudaMemcpyHostToDevice, sc));
            } else {
                for (int64_t q = i; q < j; q += slab) {
                    const int64_t nq = std::min<int64_t>(slab, j - q);
                    const int b = (int)((q / slab) & 1);
                    ICNV_CUDA(cudaEventSynchronize(c.ev_h2d[b]));   // (a recorded-never event is complete)
                    pool->copy2(pIn[b], X + G * ((int64_t)grp_idx[i] + (q - i)), sizeof(double) * (size_t)(G * nq), nullptr, nullptr, 0);
                    ICNV_CUDA(cudaMemcpyAsync(d_ref + G * q, pIn[b], sizeof(double) * (size_t)(G * nq), cudaMemcpyHostToDevice, sc));
                    ICNV_CUDA(cudaEventRecord(c.ev_h2d[b], sc));
                }
            }
            i = j;
        }
        std::vector<int32_t> iota((size_t)n_ref);
        std::iota(iota.begin(), iota.end(), 0);
        ICNV_CUDA(cudaMemcpyAsync(d_iota, iota.data(), sizeof(int32_t) * (size_t)n_ref, cudaMemcpyHostToDevice, sc));
        if (!stage_in) {
            // the first two slabs queue up behind the reference columns and cross PCIe while the pre-passes run
            for (; h2d_issued < std::min<int64_t>(2, n_slabs); ++h2d_issued)
                if ((rc = issue_h2d(h2d_issued))) return rc;
        }
        ICNV_CUDA(cudaStreamSynchronize(sc));
        lo1 = d_b; hi1 = d_b + G; mid1 = d_b + 2 * G; lo2 = d_b + 3 * G; hi2 = d_b + 4 * G; mid2 = d_b + 5 * G;
        if ((rc = dev_group_means(d_ref, G, G, d_iota, grp_off, n_grp, apply_log ? 1 : 0, d_means, sc))) return rc;
        if ((rc = icnv_dev_bounds_from_means_f64(d_means, G, n_grp, lo1, hi1, mid1, sc))) return rc;
        rc = icnv_dev_cell_pipeline_f64(d_ref, G, G, nullptr, n_ref, d_T, G, chr_start, chr_len, K, apply_log,
                                        use_bounds ? lo1 : nullptr, use_bounds ? hi1 : nullptr, use_bounds ? nullptr : mid1,
                                        threshold, window, 1, nullptr, nullptr, nullptr, 0, d_flag, sc);
        if (rc) return rc;
        if ((rc = dev_group_means(d_T, G, G, d_iota, grp_off, n_grp, 0, d_means, sc))) return rc;
        if ((rc = icnv_dev_bounds_from_means_f64(d_means, G, n_grp, lo2, hi2, mid2, sc))) return rc;
        if (!use_bounds) lo1 = hi1 = lo2 = hi2 = nullptr;
        else mid1 = mid2 = nullptr;
        if (i3) {
            // .i3HMM_get_sd_trend_by_num_cells_fit (i3HMM.R:17-80): mu and sigma over every value of the reference cells after
            // step 14.  Their final columns are a stage-D-only launch away from T (bit-identical to pass 2's: x - 0.0 == x); the
            // per-cell (sum, sd) pairs are combined in list order, exactly as icnv_mean_sd_f64 forms them.  T then holds the pairs.
            rc = icnv_dev_cell_pipeline_f64(d_T, G, G, nullptr, n_ref, d_ref, G, chr_start, chr_len, K, 0, nullptr, nullptr,
                                            nullptr, 0.0, 0, 0, lo2, hi2, mid2, 1, d_flag, sc);
            if (rc) return rc;
            if ((rc = icnv_dev_column_stats_f64(d_ref, G, d_iota, n_ref, d_T, d_T + n_ref, sc))) return rc;
            std::vector<double> h(2 * (size_t)n_ref);
            ICNV_CUDA(cudaMemcpyAsync(h.data(), d_T, sizeof(double) * 2 * (size_t)n_ref, cudaMemcpyDeviceToHost, sc));
            ICNV_CUDA(cudaStreamSynchronize(sc));
            double mu, sigma;
            icnv_combine_cell_stats(h.data(), h.data() + n_ref, n_ref, G, &mu, &sigma);
            // .i3HMM_get_HMM (i3HMM.R:99-156) with use_KS = FALSE: states at mu -+ |qnorm(p, 0, sigma)|, sd sigma, transition
            // diagonal 1 - 5t as the reference writes it
            const double d = std::fabs(qnorm_as241(i3->p_val, 0.0, sigma));
            for (int k = 0; k < 9; ++k) i3_Pi[k] = (k % 4 == 0) ? 1 - 5 * i3->t : i3->t;
            i3_delta[0] = i3_delta[2] = i3->t;
            i3_delta[1] = 1 - 5 * i3->t;
            i3_mean[0] = mu - d; i3_mean[1] = mu; i3_mean[2] = mu + d;
            i3_sd[0] = i3_sd[1] = i3_sd[2] = sigma;
            if (i3->model) {
                i3->model[0] = mu;
                i3->model[1] = sigma;
                i3->model[2] = d;
            }
            hmm = &i3_hmm;
        }
    }

    // apply_median_filtering on the unit that slab i closes: the lists inside it with unit-local indices, K4 on the unit's Y,
    // then F down - straight into the caller's matrix, or through two pinned chunks while the copy threads empty the other
    auto unit_median_filter = [&](int64_t i) -> int {
        const int64_t u0 = unit_lo[(size_t)i], nu = s_at[(size_t)i + 1] - u0;
        mf_off_u.assign(1, 0);
        mf_idx_u.clear();
        for (int k = 0; k < i3->n_mf; ++k) {
            const int32_t a = i3->mf_off[k], e = i3->mf_off[k + 1];
            if (i3->mf_idx[a] < c_lo + u0 || i3->mf_idx[a] >= c_lo + u0 + nu) continue;   // a list lies inside one unit
            for (int32_t q = a; q < e; ++q) mf_idx_u.push_back((int32_t)(i3->mf_idx[q] - (c_lo + u0)));
            mf_off_u.push_back((int32_t)mf_idx_u.size());
        }
        ICNV_CUDA(cudaStreamWaitEvent(sc, ev_f[0], 0));   // (a recorded-never event is complete)
        int rc2 = icnv_dev_median_filter_f64(dYu, dFu, G, nu, chr_start, chr_len, K, mf_off_u.data(), mf_idx_u.data(),
                                             (int)mf_off_u.size() - 1, i3->mf_window, sc);
        if (rc2) return rc2;
        ICNV_CUDA(cudaEventRecord(ev_mf, sc));
        ICNV_CUDA(cudaStreamWaitEvent(sd, ev_mf, 0));
        double *F0 = i3->F + G * (c_lo + u0);
        if (!stage_out) {
            ICNV_CUDA(cudaMemcpyAsync(F0, dFu, sizeof(double) * (size_t)G * (size_t)nu, cudaMemcpyDeviceToHost, sd));
            ICNV_CUDA(cudaEventRecord(ev_f[0], sd));
            return ICNV_OK;
        }
        const int64_t n_chunks = (nu + slab - 1) / slab;
        auto chunk_bytes = [&](int64_t k) { return sizeof(double) * (size_t)G * (size_t)std::min<int64_t>(slab, nu - k * slab); };
        for (int64_t k = 0; k <= n_chunks; ++k) {
            if (k < n_chunks) {   // pF[k & 1] was emptied by the copy of chunk k-2, one trip ago
                ICNV_CUDA(cudaMemcpyAsync(pF[k & 1], dFu + G * slab * k, chunk_bytes(k), cudaMemcpyDeviceToHost, sd));
                ICNV_CUDA(cudaEventRecord(ev_f[k & 1], sd));
            }
            if (k >= 1) {
                ICNV_CUDA(cudaEventSynchronize(ev_f[(k - 1) & 1]));
                pool->copy2(F0 + G * slab * (k - 1), pF[(k - 1) & 1], chunk_bytes(k - 1), nullptr, nullptr, 0);
            }
        }
        ICNV_CUDA(cudaEventRecord(ev_f[0], sd));
        return ICNV_OK;
    };

    if (stage_in) {   // the first slab enters the ring while the reference pre-passes run on the device
        if ((rc = host_copies(0, -1))) return rc;
    }
    for (int64_t i = 0; i < n_slabs; ++i) {
        const int b = (int)(i & 1);
        const int64_t c0 = c_lo + s_at[(size_t)i], nc = slab_cells_of(i);
        const size_t bytes = sizeof(double) * (size_t)G * (size_t)nc;
        // the unit buffer: slab i writes its own columns of it; the first slab of a unit also overwrites what the previous
        // unit's last slab (i-1) has to have left through D2H
        double *d_out = mf ? dYu + G * (s_at[(size_t)i] - unit_lo[(size_t)i]) : dOut[b];
        if (mf && i >= 1 && unit_lo[(size_t)i] != unit_lo[(size_t)i - 1]) ICNV_CUDA(cudaStreamWaitEvent(sc, c.ev_d2h[b ^ 1], 0));
        if (stage_in) {
            if (h2d_issued <= i && (rc = issue_h2d(h2d_issued++))) return rc;
        } else {
            for (; h2d_issued <= std::min<int64_t>(i + 1, n_slabs - 1); ++h2d_issued)
                if ((rc = issue_h2d(h2d_issued))) return rc;
        }
        // kernels: need the slab on the device and the output buffers of slab i-2 drained
        ICNV_CUDA(cudaStreamWaitEvent(sc, c.ev_h2d[b], 0));
        if (i >= 2) ICNV_CUDA(cudaStreamWaitEvent(sc, c.ev_d2h[b], 0));
        const double *hmm_in = dIn[b];
        if (do_smooth) {
            rc = icnv_dev_cell_pipeline_f64(dIn[b], G, G, nullptr, nc, d_out, G, chr_start, chr_len, K, apply_log, lo1, hi1,
                                            mid1, threshold, window, 1, lo2, hi2, mid2, 1, d_flag, sc);
            if (rc) return rc;
            hmm_in = d_out;
        }
        if (grp) {
            rc = slab_group_sums(d_out, G, G, d_chunks + 2 * ch_at[(size_t)i], ch_at[(size_t)i + 1] - ch_at[(size_t)i],
                                 d_segs + 6 * sg_at[(size_t)i], sg_at[(size_t)i + 1] - sg_at[(size_t)i], d_part + 2 * G,
                                 d_part + G * (i & 1), d_part + G * ((i + 1) & 1), d_gm, sc);
            if (rc) return rc;
        }
        if (has_hmm) {
            rc = icnv_dev_viterbi_f64(hmm_in, G, nc, chr_start, chr_len, K, hmm->m, hmm->Pi, hmm->delta, hmm->mean, hmm->sd,
                                      0, dSt[b], nullptr, d_flag, sc);
            if (rc) return rc;
            if (states && (rc = icnv_dev_widen_states(dSt[b], dW[b], (int64_t)G * nc, sc))) return rc;
        }
        ICNV_CUDA(cudaEventRecord(c.ev_comp[b], sc));
        // D2H (staged: the ring slot of slab i-2 was emptied by host_copies(.., i-2) below, two iterations ago)
        ICNV_CUDA(cudaStreamWaitEvent(sd, c.ev_comp[b], 0));
        if (do_smooth && Y && grp && !stage_out) {   // page-locked Y: one copy per run of owned consecutive columns
            rc = col_runs(i, true, [&](int64_t r, int64_t col, int64_t n) -> int {
                ICNV_CUDA(cudaMemcpyAsync(Y + G * col, d_out + G * r, sizeof(double) * (size_t)(G * n), cudaMemcpyDeviceToHost, sd));
                return ICNV_OK;
            });
            if (rc) return rc;
        } else if (do_smooth && Y) {
            ICNV_CUDA(cudaMemcpyAsync(stage_out ? pOut[b] : Y + G * c0, d_out, bytes, cudaMemcpyDeviceToHost, sd));
        }
        if (hmm && states)
            ICNV_CUDA(cudaMemcpyAsync(stage_out ? (int32_t *)pSt[b] : states + G * c0, dW[b],
                                      sizeof(int32_t) * (size_t)G * (size_t)nc, cudaMemcpyDeviceToHost, sd));
        if (hmm && states8)
            ICNV_CUDA(cudaMemcpyAsync(stage_out ? (uint8_t *)pSt[b] : states8 + G * c0, dSt[b], (size_t)G * (size_t)nc,
                                      cudaMemcpyDeviceToHost, sd));
        ICNV_CUDA(cudaEventRecord(c.ev_d2h[b], sd));
        if (mf && unit_end[(size_t)i] && (rc = unit_median_filter(i))) return rc;
        // host side of the ring while the device works on slab i: slab i+1 in, slab i-1 out
        if (stage_in || stage_out)
            if ((rc = host_copies(stage_in ? i + 1 : -1, stage_out ? i - 1 : -1))) return rc;
    }
    if (stage_out && (rc = host_copies(-1, n_slabs - 1))) return rc;
    ICNV_CUDA(cudaStreamSynchronize(sh));
    ICNV_CUDA(cudaStreamSynchronize(sd));
    if (!grp) return check_flag(d_flag, sc);

    // group mode: the Viterbi of this range's groups (viterbi_impl's per-group median sd; i3: sigma), then every column its
    // positions own takes its group's trace, 255 for the cells in no list
    std::vector<uint8_t> h_st((size_t)G * (size_t)n_loc);
    std::vector<double> sdl((size_t)n_loc);
    if (n_loc > 0) {
        for (int64_t j = 0; j < n_loc; ++j) sdl[(size_t)j] = grp->sd_med.empty() ? hmm->sd[0] : grp->sd_med[(size_t)(k_lo + j)];
        ICNV_CUDA(cudaMemcpyAsync(d_gsd, sdl.data(), sizeof(double) * (size_t)n_loc, cudaMemcpyHostToDevice, sc));
        rc = icnv_dev_viterbi_f64(d_gm, G, n_loc, chr_start, chr_len, K, hmm->m, hmm->Pi, hmm->delta, hmm->mean, d_gsd, 1, d_gst,
                                  nullptr, d_flag, sc);
        if (rc) return rc;
        ICNV_CUDA(cudaMemcpyAsync(h_st.data(), d_gst, h_st.size(), cudaMemcpyDeviceToHost, sc));
    }
    if ((rc = check_flag(d_flag, sc))) return rc;
    const std::vector<uint8_t> none((size_t)G, 255);
    std::vector<CopyPool::Job> jobs;
    for (int64_t p = c_lo; p < c_hi; ++p) {
        if (!grp->owns[(size_t)p]) continue;
        const uint8_t *src = p < grp->n_listed ? h_st.data() + (size_t)G * (size_t)(grp->grp_at[(size_t)p] - k_lo) : none.data();
        jobs.push_back({(char *)(grp->states + G * grp->col(p)), (const char *)src, (size_t)G});
    }
    pool->copyv(jobs);
    return ICNV_OK;
}

// The cells are cut into one contiguous range per device context; each range is driven by its own host thread (a CUDA
// context per thread, its own streams, scratch and ring).  One context: the calling thread does the work itself.
static int host_pipeline(Ctx &c0, const double *X, double *Y, int32_t *states, uint8_t *states8, int64_t G, int64_t C,
                         const int32_t *chr_start, const int32_t *chr_len, int K, int do_smooth, const int32_t *grp_off,
                         const int32_t *grp_idx, int n_grp, int apply_log, double threshold, int window, int use_bounds,
                         const HmmModel *hmm, const I3Fused *i3 = nullptr, const GroupHmm *grp = nullptr) {
    // (group mode: C counts pipeline positions, see GroupHmm)
    const int n_dev = (int)std::min<int64_t>(std::max(1, device_slots()), std::max<int64_t>(1, C / 64));
    const bool pageable = !is_pinned(X) || (Y && !is_pinned(Y)) || (states && !is_pinned(states)) || (states8 && !is_pinned(states8)) ||
                          (i3 && i3->F && !is_pinned(i3->F));
    const int nt = pool_threads_per_device();
    if (n_dev <= 1) {   // (group mode: the copy threads also place the traces)
        std::unique_ptr<CopyPool> pool(pageable || grp ? new CopyPool(nt) : nullptr);
        return host_pipeline_range(c0, X, Y, states, states8, G, 0, C, chr_start, chr_len, K, do_smooth, grp_off, grp_idx, n_grp,
                                   apply_log, threshold, window, use_bounds, hmm, pool.get(), i3, nullptr, grp);
    }
    // even shares; with the median filter each cut moves to the nearest column no list's span crosses, in group mode to the
    // nearest group boundary (each group's means and trace come from one device)
    std::vector<int64_t> cut((size_t)n_dev + 1);
    for (int d = 0; d <= n_dev; ++d) {
        cut[(size_t)d] = C * d / n_dev;
        if (i3 && i3->F) cut[(size_t)d] = std::max(d ? cut[(size_t)d - 1] : 0, i3->cut_near(cut[(size_t)d]));
        if (grp) cut[(size_t)d] = std::max(d ? cut[(size_t)d - 1] : 0, grp->group_cut_near(cut[(size_t)d]));
    }
    int reporter = 0;   // the first device with cells reports the i3 model (every device computes the same bits)
    while (reporter < n_dev - 1 && cut[(size_t)reporter] == cut[(size_t)reporter + 1]) ++reporter;
    std::vector<I3Fused> i3d;
    if (i3) {
        i3d.assign((size_t)n_dev, *i3);
        for (int d = 0; d < n_dev; ++d)
            if (d != reporter) i3d[(size_t)d].model = nullptr;
    }
    std::vector<int> rcs((size_t)n_dev, ICNV_OK);
    std::vector<std::string> msgs((size_t)n_dev);
    std::vector<std::thread> th;
    const int caller_slot = current_slot();
    int n_busy = 0;
    for (int d = 0; d < n_dev; ++d) n_busy += cut[(size_t)d] < cut[(size_t)d + 1];
    // the fused i3 call promises that a unit that does not fit is refused before any output is written
    std::unique_ptr<StartGate> gate((i3 && i3->F) || grp ? new StartGate(n_dev, n_busy) : nullptr);
    for (int d = 0; d < n_dev; ++d) {
        const int64_t lo = cut[(size_t)d], hi = cut[(size_t)d + 1];
        if (lo == hi) continue;
        th.emplace_back([&, d, lo, hi] {
            set_current_slot(d);
            Ctx &c = ctx();
            std::unique_lock<std::mutex> lk(c.mu, std::defer_lock);
            if (d != caller_slot) lk.lock();   // the caller already holds its own context's lock
            int rc = ICNV_OK;
            if (cudaSetDevice(c.device) != cudaSuccess) rc = set_error(ICNV_E_CUDA, "cudaSetDevice(%d) failed", c.device);
            if (!rc) {
                std::unique_ptr<CopyPool> pool(pageable || grp ? new CopyPool(nt) : nullptr);
                rc = host_pipeline_range(c, X, Y, states, states8, G, lo, hi, chr_start, chr_len, K, do_smooth, grp_off, grp_idx,
                                         n_grp, apply_log, threshold, window, use_bounds, hmm, pool.get(),
                                         i3 ? &i3d[(size_t)d] : nullptr, gate.get(), grp);
            }
            if (gate) gate->arrive(d, rc == ICNV_OK);   // a range that failed before the gate still has to open it
            rcs[(size_t)d] = rc;
            if (rc) msgs[(size_t)d] = icnv_last_error();   // the message is per thread: carry it to the caller
        });
    }
    for (auto &t : th) t.join();
    cudaSetDevice(c0.device);
    if (gate && gate->first_fail >= 0) {   // report the device that could not start, not the ones it stopped
        const int d = gate->first_fail;
        return set_error(rcs[(size_t)d], "device %d: %s", ctx_of(d).device, msgs[(size_t)d].c_str());
    }
    for (int d = 0; d < n_dev; ++d)
        if (rcs[(size_t)d]) return set_error(rcs[(size_t)d], "device %d: %s", ctx_of(d).device, msgs[(size_t)d].c_str());
    return ICNV_OK;
}

int icnv_smooth_block_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *chr_start,
                          const int32_t *chr_len, int K, const int32_t *grp_off, const int32_t *grp_idx, int n_grp,
                          int apply_log, double threshold, int window, int use_bounds) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || G <= 0 || C <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_smooth_block_f64: bad argument");
    int rc = validate_chr(G, chr_start, chr_len, K);
    if (rc) return rc;
    if ((rc = validate_groups(C, grp_off, grp_idx, n_grp, false))) return rc;
    return host_pipeline(c, X, Y, nullptr, nullptr, G, C, chr_start, chr_len, K, 1, grp_off, grp_idx, n_grp, apply_log,
                         threshold, window, use_bounds, nullptr);
}

/* Fused smooth block + per-cell HMM in one pass over the matrix: run() steps 4..14 and step 17 for
 * analysis_mode = "cells" with prune_outliers = FALSE (the defaults between them do not touch expr.data).
 * Saves the second upload of the matrix that two separate calls need. */
static int smooth_hmm_impl(const double *X, double *Y, int32_t *states, uint8_t *states8, int64_t G, int64_t C,
                           const int32_t *chr_start, const int32_t *chr_len, int K, const int32_t *grp_off,
                           const int32_t *grp_idx, int n_grp, int apply_log, double threshold, int window, int use_bounds,
                           int m, const double *Pi, const double *delta, const double *mean, const double *sd) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || (!states && !states8) || G <= 0 || C <= 0 || !Pi || !delta || !mean || !sd)
        return set_error(ICNV_E_BAD_ARG, "icnv_smooth_hmm_f64: bad argument");
    if (m != 6 && m != 3) return set_error(ICNV_E_BAD_ARG, "m must be 6 or 3");
    int rc = validate_chr(G, chr_start, chr_len, K);
    if (rc) return rc;
    if ((rc = validate_groups(C, grp_off, grp_idx, n_grp, false))) return rc;
    HmmModel hm{m, Pi, delta, mean, sd};
    return host_pipeline(c, X, Y, states, states8, G, C, chr_start, chr_len, K, 1, grp_off, grp_idx, n_grp, apply_log,
                         threshold, window, use_bounds, &hm);
}

int icnv_smooth_hmm_f64(const double *X, double *Y, int32_t *states, int64_t G, int64_t C, const int32_t *chr_start,
                        const int32_t *chr_len, int K, const int32_t *grp_off, const int32_t *grp_idx, int n_grp,
                        int apply_log, double threshold, int window, int use_bounds, int m, const double *Pi,
                        const double *delta, const double *mean, const double *sd) {
    return smooth_hmm_impl(X, Y, states, nullptr, G, C, chr_start, chr_len, K, grp_off, grp_idx, n_grp, apply_log, threshold,
                           window, use_bounds, m, Pi, delta, mean, sd);
}

int icnv_smooth_hmm_u8_f64(const double *X, double *Y, uint8_t *states, int64_t G, int64_t C, const int32_t *chr_start,
                           const int32_t *chr_len, int K, const int32_t *grp_off, const int32_t *grp_idx, int n_grp,
                           int apply_log, double threshold, int window, int use_bounds, int m, const double *Pi,
                           const double *delta, const double *mean, const double *sd) {
    return smooth_hmm_impl(X, Y, nullptr, states, G, C, chr_start, chr_len, K, grp_off, grp_idx, n_grp, apply_log, threshold,
                           window, use_bounds, m, Pi, delta, mean, sd);
}

/* Fused i3 pass (see the header): smooth block, the i3 model of its reference cells, per-cell i3 HMM and
 * apply_median_filtering over the lists mf_*, one read of X and one write of each output. */
int icnv_smooth_i3_hmm_u8_f64(const double *X, double *Y, uint8_t *states, double *F, int64_t G, int64_t C,
                              const int32_t *chr_start, const int32_t *chr_len, int K, const int32_t *grp_off,
                              const int32_t *grp_idx, int n_grp, int apply_log, double threshold, int window, int use_bounds,
                              double i3_p_val, double t, const int32_t *mf_off, const int32_t *mf_idx, int n_mf,
                              int mf_window, double *model) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || !states || !model || G <= 1 || C <= 0)
        return set_error(ICNV_E_BAD_ARG, "icnv_smooth_i3_hmm_u8_f64: bad argument");
    if (!(i3_p_val > 0.0 && i3_p_val < 1.0)) return set_error(ICNV_E_BAD_ARG, "i3_p_val must lie in (0, 1)");
    if (window >= 2 && (window & 1) == 0)
        return set_error(ICNV_E_BAD_ARG, "window_length %d is even: the reference's behaviour is accidental there", window);
    int rc = validate_chr(G, chr_start, chr_len, K);
    if (rc) return rc;
    if ((rc = validate_groups(C, grp_off, grp_idx, n_grp, false))) return rc;
    I3Fused i3{i3_p_val, t, model, nullptr, mf_off, mf_idx, n_mf, mf_window, {}};
    if (F) {   // no lists: every cell is in none, so F is a copy of Y, as icnv_median_filter_f64 makes it
        if (mf_window < 3 || (mf_window & 1) == 0)
            return set_error(ICNV_E_BAD_ARG, "window_size must be an odd number >= 3 (noise_reduction.R:48-50)");
        if (n_mf < 0) return set_error(ICNV_E_BAD_ARG, "n_mf < 0");
        if (n_mf > 0 && (rc = validate_groups(C, mf_off, mf_idx, n_mf, false))) return rc;
        std::vector<std::pair<int64_t, int64_t>> sp((size_t)n_mf);
        for (int k = 0; k < n_mf; ++k) {
            const auto mm = std::minmax_element(mf_idx + mf_off[k], mf_idx + mf_off[k + 1]);
            sp[(size_t)k] = {*mm.first, (int64_t)*mm.second + 1};
        }
        std::sort(sp.begin(), sp.end());
        for (const auto &v : sp) {
            if (!i3.spans.empty() && v.first < i3.spans.back().second) i3.spans.back().second = std::max(i3.spans.back().second, v.second);
            else i3.spans.push_back(v);
        }
        i3.F = F;
    }
    return host_pipeline(c, X, Y, nullptr, states, G, C, chr_start, chr_len, K, 1, grp_off, grp_idx, n_grp, apply_log, threshold,
                         window, use_bounds, nullptr, &i3);
}

// The pipeline order of the group-mode calls (see GroupHmm) from the HMM lists; BAD_ARG for n_hmm == 0 or a bad list.
static int group_hmm_order(GroupHmm &gh, int64_t C, const int32_t *hmm_off, const int32_t *hmm_idx, int n_hmm, uint8_t *states) {
    if (n_hmm == 0) return set_error(ICNV_E_BAD_ARG, "n_hmm == 0: the per-cell calls run the HMM without groups");
    int rc = validate_groups(C, hmm_off, hmm_idx, n_hmm, false);
    if (rc) return rc;
    gh.off = hmm_off;
    gh.n_hmm = n_hmm;
    gh.n_listed = hmm_off[n_hmm];
    gh.states = states;
    std::vector<int32_t> last((size_t)C, -1);   // a cell's last listing writes it, as viterbi_impl's grp_of
    for (int32_t p = 0; p < hmm_off[n_hmm]; ++p) last[(size_t)hmm_idx[p]] = p;
    gh.order.assign(hmm_idx, hmm_idx + gh.n_listed);
    gh.grp_at.resize((size_t)gh.n_listed);
    gh.owns.resize((size_t)gh.n_listed);
    for (int k = 0; k < n_hmm; ++k)
        for (int32_t p = hmm_off[k]; p < hmm_off[k + 1]; ++p) {
            gh.grp_at[(size_t)p] = k;
            gh.owns[(size_t)p] = last[(size_t)hmm_idx[p]] == p;
        }
    for (int64_t c = 0; c < C; ++c)
        if (last[(size_t)c] < 0) {
            gh.order.push_back((int32_t)c);
            gh.owns.push_back(1);
        }
    return ICNV_OK;
}

/* Fused smooth block + group-mode HMM (see the header): run() steps 4..14 and 17 for analysis_mode "samples" and
 * "subclusters" (random_trees), one read of X and one write of Y and states. */
int icnv_smooth_hmm_groups_u8_f64(const double *X, double *Y, uint8_t *states, int64_t G, int64_t C, const int32_t *chr_start,
                                  const int32_t *chr_len, int K, const int32_t *grp_off, const int32_t *grp_idx, int n_grp,
                                  int apply_log, double threshold, int window, int use_bounds, const int32_t *hmm_off,
                                  const int32_t *hmm_idx, int n_hmm, int m, const double *Pi, const double *delta,
                                  const double *mean, const double *sd) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || !states || G <= 0 || C <= 0 || !Pi || !delta || !mean || !sd)
        return set_error(ICNV_E_BAD_ARG, "icnv_smooth_hmm_groups_u8_f64: bad argument");
    if (m != 6 && m != 3) return set_error(ICNV_E_BAD_ARG, "m must be 6 or 3");
    int rc = validate_chr(G, chr_start, chr_len, K);
    if (rc) return rc;
    if ((rc = validate_groups(C, grp_off, grp_idx, n_grp, false))) return rc;
    GroupHmm gh;
    if ((rc = group_hmm_order(gh, C, hmm_off, hmm_idx, n_hmm, states))) return rc;
    gh.sd_med.resize((size_t)n_hmm);
    for (int b = 0; b < n_hmm; ++b) {   // viterbi_impl's per-group median sd
        std::vector<double> v(sd + (size_t)m * b, sd + (size_t)m * (b + 1));
        std::sort(v.begin(), v.end());
        gh.sd_med[(size_t)b] = (m & 1) ? v[m / 2] : 0.5 * (v[m / 2 - 1] + v[m / 2]);
        if (!(gh.sd_med[(size_t)b] > 0.0)) return set_error(ICNV_E_BAD_ARG, "state sd must be positive (group %d)", b);
    }
    HmmModel hm{m, Pi, delta, mean, sd};
    return host_pipeline(c, X, Y, nullptr, nullptr, G, (int64_t)gh.order.size(), chr_start, chr_len, K, 1, grp_off, grp_idx,
                         n_grp, apply_log, threshold, window, use_bounds, &hm, nullptr, &gh);
}

/* The i3 twin: the i3 model fixed from the block's reference cells as in icnv_smooth_i3_hmm_u8_f64, then the group-mode
 * i3 HMM (sigma for every group).  No median filter. */
int icnv_smooth_i3_hmm_groups_u8_f64(const double *X, double *Y, uint8_t *states, int64_t G, int64_t C,
                                     const int32_t *chr_start, const int32_t *chr_len, int K, const int32_t *grp_off,
                                     const int32_t *grp_idx, int n_grp, int apply_log, double threshold, int window,
                                     int use_bounds, const int32_t *hmm_off, const int32_t *hmm_idx, int n_hmm,
                                     double i3_p_val, double t, double *model) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || !states || !model || G <= 1 || C <= 0)
        return set_error(ICNV_E_BAD_ARG, "icnv_smooth_i3_hmm_groups_u8_f64: bad argument");
    if (!(i3_p_val > 0.0 && i3_p_val < 1.0)) return set_error(ICNV_E_BAD_ARG, "i3_p_val must lie in (0, 1)");
    if (window >= 2 && (window & 1) == 0)
        return set_error(ICNV_E_BAD_ARG, "window_length %d is even: the reference's behaviour is accidental there", window);
    int rc = validate_chr(G, chr_start, chr_len, K);
    if (rc) return rc;
    if ((rc = validate_groups(C, grp_off, grp_idx, n_grp, false))) return rc;
    GroupHmm gh;
    if ((rc = group_hmm_order(gh, C, hmm_off, hmm_idx, n_hmm, states))) return rc;
    I3Fused i3{i3_p_val, t, model, nullptr, nullptr, nullptr, 0, 0, {}};
    return host_pipeline(c, X, Y, nullptr, nullptr, G, (int64_t)gh.order.size(), chr_start, chr_len, K, 1, grp_off, grp_idx,
                         n_grp, apply_log, threshold, window, use_bounds, nullptr, &i3, &gh);
}

static int viterbi_impl(const double *X, int64_t G, int64_t C, const int32_t *chr_start, const int32_t *chr_len, int K,
                        const int32_t *grp_off, const int32_t *grp_idx, int n_grp, int m, const double *Pi,
                        const double *delta, const double *mean, const double *sd, int32_t *states, uint8_t *states8,
                        double *margins) {
    ICNV_HOST_PROLOGUE();
    if (!X || (!states && !states8) || G <= 0 || C <= 0 || !Pi || !delta || !mean || !sd)
        return set_error(ICNV_E_BAD_ARG, "icnv_viterbi_f64: bad argument");
    if (m != 6 && m != 3) return set_error(ICNV_E_BAD_ARG, "m must be 6 or 3");
    int rc = validate_chr(G, chr_start, chr_len, K);
    if (rc) return rc;
    rc = validate_groups(C, grp_off, grp_idx, n_grp, true);
    if (rc) return rc;
    if (n_grp == 0 && !margins) {  // per-cell mode: slab pipeline (copies overlap the kernels)
        HmmModel hm{m, Pi, delta, mean, sd};
        return host_pipeline(c, X, nullptr, states, states8, G, C, chr_start, chr_len, K, 0, nullptr, nullptr, 0, 0, 0.0, 0, 0,
                             &hm);
    }
    double *dX;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    int *d_flag = (int *)scratch(SLOT_MISC, 64);
    if (!d_flag) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
    int32_t *d_out = (int32_t *)scratch(SLOT_OUT, sizeof(int32_t) * (size_t)(G * C));
    if (!d_out) return ICNV_E_NOMEM;

    if (n_grp == 0) {
        uint8_t *d_st = (uint8_t *)scratch(SLOT_STATES, (size_t)(G * C));
        double *d_mg = margins ? (double *)scratch(SLOT_TMP, sizeof(double) * (size_t)K * (size_t)C) : nullptr;
        if (!d_st || (margins && !d_mg)) return ICNV_E_NOMEM;
        rc = icnv_dev_viterbi_f64(dX, G, C, chr_start, chr_len, K, m, Pi, delta, mean, sd, 0, d_st, d_mg, d_flag, st);
        if (rc) return rc;
        if ((rc = icnv_dev_widen_states(d_st, d_out, G * C, st))) return rc;
        if (margins)
            ICNV_CUDA(cudaMemcpyAsync(margins, d_mg, sizeof(double) * (size_t)K * (size_t)C, cudaMemcpyDeviceToHost, st));
    } else {
        // group modes: x = rowMeans(X[chr, group]) (HMM.R:383), per-group median sd, trace broadcast
        const int64_t n_idx = grp_off[n_grp];
        int32_t *d_idx = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)(n_idx + C));
        double *d_xm = (double *)scratch(SLOT_MEANS, sizeof(double) * (size_t)G * (size_t)n_grp);
        double *d_sd = (double *)scratch(SLOT_BOUNDS, sizeof(double) * (size_t)std::max<int64_t>(n_grp, 6 * G));
        uint8_t *d_st = (uint8_t *)scratch(SLOT_STATES, (size_t)G * (size_t)n_grp);
        double *d_mg = margins ? (double *)scratch(SLOT_TMP, sizeof(double) * (size_t)K * (size_t)n_grp) : nullptr;
        if (!d_idx || !d_xm || !d_sd || !d_st || (margins && !d_mg)) return ICNV_E_NOMEM;
        std::vector<int32_t> grp_of((size_t)C, -1);
        std::vector<double> sdm((size_t)n_grp);
        for (int b = 0; b < n_grp; ++b) {
            for (int32_t i = grp_off[b]; i < grp_off[b + 1]; ++i) grp_of[grp_idx[i]] = b;
            std::vector<double> v(sd + (size_t)m * b, sd + (size_t)m * (b + 1));
            std::sort(v.begin(), v.end());
            sdm[b] = (m & 1) ? v[m / 2] : 0.5 * (v[m / 2 - 1] + v[m / 2]);
            if (!(sdm[b] > 0.0)) return set_error(ICNV_E_BAD_ARG, "state sd must be positive (group %d)", b);
        }
        ICNV_CUDA(cudaMemcpyAsync(d_idx, grp_idx, sizeof(int32_t) * (size_t)n_idx, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_idx + n_idx, grp_of.data(), sizeof(int32_t) * (size_t)C, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_sd, sdm.data(), sizeof(double) * (size_t)n_grp, cudaMemcpyHostToDevice, st));
        if ((rc = dev_group_means(dX, G, G, d_idx, grp_off, n_grp, 0, d_xm, st))) return rc;
        rc = icnv_dev_viterbi_f64(d_xm, G, n_grp, chr_start, chr_len, K, m, Pi, delta, mean, d_sd, 1, d_st, d_mg, d_flag, st);
        if (rc) return rc;
        if ((rc = icnv_dev_scatter_group_states(d_st, G, C, d_idx + n_idx, d_out, st))) return rc;
        if (margins)
            ICNV_CUDA(cudaMemcpyAsync(margins, d_mg, sizeof(double) * (size_t)K * (size_t)n_grp, cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaStreamSynchronize(st));  // grp_of / sdm are stack-lifetime host buffers
    }
    if (states) {
        ICNV_CUDA(cudaMemcpyAsync(states, d_out, sizeof(int32_t) * (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    } else {
        uint8_t *d_n = (uint8_t *)scratch(SLOT_SLAB_ST0, (size_t)(G * C));
        if (!d_n) return ICNV_E_NOMEM;
        if ((rc = icnv_dev_narrow_states(d_out, d_n, G * C, st))) return rc;
        ICNV_CUDA(cudaMemcpyAsync(states8, d_n, (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    }
    return check_flag(d_flag, st);
}

int icnv_viterbi_f64(const double *X, int64_t G, int64_t C, const int32_t *chr_start, const int32_t *chr_len, int K,
                     const int32_t *grp_off, const int32_t *grp_idx, int n_grp, int m, const double *Pi,
                     const double *delta, const double *mean, const double *sd, int32_t *states, double *margins) {
    return viterbi_impl(X, G, C, chr_start, chr_len, K, grp_off, grp_idx, n_grp, m, Pi, delta, mean, sd, states, nullptr,
                        margins);
}

int icnv_viterbi_u8_f64(const double *X, int64_t G, int64_t C, const int32_t *chr_start, const int32_t *chr_len, int K,
                        const int32_t *grp_off, const int32_t *grp_idx, int n_grp, int m, const double *Pi,
                        const double *delta, const double *mean, const double *sd, uint8_t *states, double *margins) {
    return viterbi_impl(X, G, C, chr_start, chr_len, K, grp_off, grp_idx, n_grp, m, Pi, delta, mean, sd, nullptr, states,
                        margins);
}

int icnv_median_filter_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *chr_start,
                           const int32_t *chr_len, int K, const int32_t *grp_off, const int32_t *grp_idx, int n_grp,
                           int window_size) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || G <= 0 || C <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_median_filter_f64: bad argument");
    int rc = validate_chr(G, chr_start, chr_len, K);
    if (rc) return rc;
    if ((rc = validate_groups(C, grp_off, grp_idx, n_grp, true))) return rc;
    double *dX, *dY;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(G * C));
    int *d_flag = (int *)scratch(SLOT_MISC, 64);
    if (!dY || !d_flag) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
    rc = icnv_dev_median_filter_f64(dX, dY, G, C, chr_start, chr_len, K, grp_off, grp_idx, n_grp, window_size, st);
    if (rc) return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    return check_flag(d_flag, st);
}

// ---- gene filters and counts ingest (run() steps 2-3; R/inferCNV_ops.R:2124-2209, 3064-3111) ------------------------

// rowMeans as R computes it: a long-double quotient rounded to double (the sums of count data are exact integers)
static void means_from_sums(const double *sums, int64_t G, int64_t C, double *means) {
    for (int64_t g = 0; g < G; ++g) means[g] = (double)((long double)sums[g] / (long double)C);
}

static int download_gene_stats(const double *d_sums, const int32_t *d_npos, int64_t G, int64_t C, double *sums,
                               int32_t *n_pos, double *means, cudaStream_t st) {
    std::vector<double> tmp;
    double *hs = sums;
    if (!hs) {
        tmp.resize((size_t)G);
        hs = tmp.data();
    }
    ICNV_CUDA(cudaMemcpyAsync(hs, d_sums, sizeof(double) * (size_t)G, cudaMemcpyDeviceToHost, st));
    if (n_pos) ICNV_CUDA(cudaMemcpyAsync(n_pos, d_npos, sizeof(int32_t) * (size_t)G, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    if (means) means_from_sums(hs, G, C, means);
    return ICNV_OK;
}

int icnv_gene_stats_f64(const double *X, int64_t G, int64_t C, double *sums, int32_t *n_pos, double *means) {
    ICNV_HOST_PROLOGUE();
    if (!X || G <= 0 || C <= 0 || (!sums && !n_pos && !means)) return set_error(ICNV_E_BAD_ARG, "icnv_gene_stats_f64: bad argument");
    double *dX;
    int rc;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    double *d_sums = (double *)scratch(SLOT_MEANS, sizeof(double) * (size_t)G);
    int32_t *d_npos = (int32_t *)scratch(SLOT_IDX2, sizeof(int32_t) * (size_t)G);
    if (!d_sums || !d_npos) return ICNV_E_NOMEM;
    if ((rc = icnv_dev_gene_stats_f64(dX, G, G, C, d_sums, d_npos, st))) return rc;
    return download_gene_stats(d_sums, d_npos, G, C, sums, n_pos, means, st);
}

/* scale_infercnv_expr, R/inferCNV_ops.R:3174-3186 (run() step 5 when scale_data = TRUE): every gene centred and scaled
 * to unit sd (n - 1) across the cells. */
int icnv_scale_infercnv_expr_f64(const double *X, double *Y, int64_t G, int64_t C) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || G <= 0 || C <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_scale_infercnv_expr_f64: bad argument");
    double *dX;
    int rc;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    double *dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(G * C));
    double *d_stat = (double *)scratch(SLOT_MEANS, sizeof(double) * 2 * (size_t)G);
    if (!dY || !d_stat) return ICNV_E_NOMEM;
    if ((rc = icnv_dev_scale_rows_f64(dX, dY, G, C, d_stat, d_stat + G, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

static int validate_keep(const int32_t *keep, int64_t n_keep, int64_t G) {
    if (!keep || n_keep <= 0 || n_keep > G) return set_error(ICNV_E_BAD_ARG, "the list of genes to keep is empty or too long");
    for (int64_t i = 0; i < n_keep; ++i)
        if (keep[i] < 0 || keep[i] >= G || (i > 0 && keep[i] <= keep[i - 1]))
            return set_error(ICNV_E_BAD_ARG, "genes to keep must be increasing row indices in [0, G)");
    return ICNV_OK;
}

int icnv_remove_genes_f64(const double *X, int64_t G, int64_t C, const int32_t *keep, int64_t n_keep, double *Y) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || G <= 0 || C <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_remove_genes_f64: bad argument");
    int rc = validate_keep(keep, n_keep, G);
    if (rc) return rc;
    double *dX;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    double *dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(n_keep * C));
    int32_t *d_keep = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)n_keep);
    if (!dY || !d_keep) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemcpyAsync(d_keep, keep, sizeof(int32_t) * (size_t)n_keep, cudaMemcpyHostToDevice, st));
    if ((rc = icnv_dev_gather_rows_f64(dX, G, d_keep, n_keep, dY, C, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)(n_keep * C), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

/* Row selection in any order (rows may repeat): Y (n x C) = X[idx, ].  The ingest step .order_reduce
 * (R/inferCNV.R:352-428) reorders the expression matrix to the genomic position table with it. */
int icnv_gather_genes_f64(const double *X, int64_t G, int64_t C, const int32_t *idx, int64_t n, double *Y) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || !idx || G <= 0 || C <= 0 || n <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_gather_genes_f64: bad argument");
    for (int64_t i = 0; i < n; ++i)
        if (idx[i] < 0 || idx[i] >= G) return set_error(ICNV_E_BAD_ARG, "row index %d out of range", idx[i]);
    double *dX;
    int rc;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    double *dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(n * C));
    int32_t *d_idx = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)n);
    if (!dY || !d_idx) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemcpyAsync(d_idx, idx, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, st));
    if ((rc = icnv_dev_gather_rows_f64(dX, G, d_idx, n, dY, C, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)(n * C), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

static int validate_csc(const int32_t *p, const int32_t *ri, const double *x, int64_t G, int64_t C) {
    if (!p || G <= 0 || C <= 0) return set_error(ICNV_E_BAD_ARG, "compressed-column matrix: bad argument");
    if (p[0] != 0) return set_error(ICNV_E_BAD_ARG, "compressed-column matrix: p[0] must be 0");
    for (int64_t c = 0; c < C; ++c)
        if (p[c + 1] < p[c]) return set_error(ICNV_E_BAD_ARG, "compressed-column matrix: p must be non-decreasing");
    const int64_t nnz = p[C];
    if (nnz > 0 && (!ri || !x)) return set_error(ICNV_E_BAD_ARG, "compressed-column matrix: i / x missing");
    for (int64_t k = 0; k < nnz; ++k)
        if (ri[k] < 0 || ri[k] >= G) return set_error(ICNV_E_BAD_ARG, "compressed-column matrix: row index out of range");
    return ICNV_OK;
}

// upload p / i / x into SLOT_IN (x first: 8-byte alignment)
static int upload_csc(const int32_t *p, const int32_t *ri, const double *x, int64_t C, const double **d_x,
                      const int32_t **d_i, const int32_t **d_p, cudaStream_t st) {
    const int64_t nnz = p[C];
    const size_t bx = sizeof(double) * (size_t)std::max<int64_t>(nnz, 1);
    const size_t bi = (sizeof(int32_t) * (size_t)std::max<int64_t>(nnz, 1) + 7) & ~(size_t)7;
    char *base = (char *)scratch(SLOT_IN, bx + bi + sizeof(int32_t) * (size_t)(C + 1));
    if (!base) return ICNV_E_NOMEM;
    if (nnz > 0) {
        ICNV_CUDA(cudaMemcpyAsync(base, x, sizeof(double) * (size_t)nnz, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(base + bx, ri, sizeof(int32_t) * (size_t)nnz, cudaMemcpyHostToDevice, st));
    }
    ICNV_CUDA(cudaMemcpyAsync(base + bx + bi, p, sizeof(int32_t) * (size_t)(C + 1), cudaMemcpyHostToDevice, st));
    *d_x = (const double *)base;
    *d_i = (const int32_t *)(base + bx);
    *d_p = (const int32_t *)(base + bx + bi);
    return ICNV_OK;
}

int icnv_csc_gene_stats_f64(const int32_t *p, const int32_t *ri, const double *x, int64_t G, int64_t C, double *sums,
                            int32_t *n_pos, double *means) {
    ICNV_HOST_PROLOGUE();
    int rc = validate_csc(p, ri, x, G, C);
    if (rc) return rc;
    if (!sums && !n_pos && !means) return set_error(ICNV_E_BAD_ARG, "icnv_csc_gene_stats_f64: no output requested");
    const double *d_x;
    const int32_t *d_i, *d_p;
    if ((rc = upload_csc(p, ri, x, C, &d_x, &d_i, &d_p, st))) return rc;
    double *d_sums = (double *)scratch(SLOT_MEANS, sizeof(double) * (size_t)G);
    int32_t *d_npos = (int32_t *)scratch(SLOT_IDX2, sizeof(int32_t) * (size_t)G);
    if (!d_sums || !d_npos) return ICNV_E_NOMEM;
    if ((rc = icnv_dev_csc_gene_stats_f64(d_i, d_x, p[C], G, d_sums, d_npos, st))) return rc;
    return download_gene_stats(d_sums, d_npos, G, C, sums, n_pos, means, st);
}

int icnv_csc_normalize_f64(const int32_t *p, const int32_t *ri, const double *x, int64_t G, int64_t C, const int32_t *keep,
                           int64_t n_keep, double normalize_factor, double *Y, double *col_sums) {
    ICNV_HOST_PROLOGUE();
    int rc = validate_csc(p, ri, x, G, C);
    if (rc) return rc;
    if (!Y) return set_error(ICNV_E_BAD_ARG, "icnv_csc_normalize_f64: bad argument");
    const int64_t G_out = keep ? n_keep : G;
    if (keep && (rc = validate_keep(keep, n_keep, G))) return rc;
    const double *d_x;
    const int32_t *d_i, *d_p;
    if ((rc = upload_csc(p, ri, x, C, &d_x, &d_i, &d_p, st))) return rc;
    int32_t *d_map = nullptr;
    std::vector<int32_t> map;
    if (keep) {
        map.assign((size_t)G, -1);
        for (int64_t i = 0; i < n_keep; ++i) map[(size_t)keep[i]] = (int32_t)i;
        d_map = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)G);
        if (!d_map) return ICNV_E_NOMEM;
        ICNV_CUDA(cudaMemcpyAsync(d_map, map.data(), sizeof(int32_t) * (size_t)G, cudaMemcpyHostToDevice, st));
    }
    double *d_cs = (double *)scratch(SLOT_PARTIAL, sizeof(double) * (size_t)C);
    double *dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(G_out * C));
    if (!d_cs || !dY) return ICNV_E_NOMEM;
    if ((rc = icnv_dev_csc_col_sums_f64(d_p, d_i, d_x, d_map, C, d_cs, st))) return rc;
    std::vector<double> cs((size_t)C);
    ICNV_CUDA(cudaMemcpyAsync(cs.data(), d_cs, sizeof(double) * (size_t)C, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    if (col_sums) std::copy(cs.begin(), cs.end(), col_sums);
    if (!(normalize_factor >= 0.0)) {   // NA: median of the library sizes (ops.R:3095-3097)
        std::sort(cs.begin(), cs.end());
        normalize_factor = (C & 1) ? cs[(size_t)(C / 2)] : 0.5 * (cs[(size_t)(C / 2 - 1)] + cs[(size_t)(C / 2)]);
    }
    if (!std::isfinite(normalize_factor)) return set_error(ICNV_E_NONFINITE, "Error, normalize factor not estimated");
    if ((rc = icnv_dev_csc_expand_f64(d_p, d_i, d_x, d_map, G_out, C, d_cs, normalize_factor, dY, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)(G_out * C), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

// ---- per-chromosome subcluster HMM (predict_CNV_via_HMM_on_tumor_subclusters_per_chr, HMM.R:412-487) --------------

int icnv_viterbi_per_chr_u8_f64(const double *X, int64_t G, int64_t C, const int32_t *chr_start, const int32_t *chr_len, int K,
                                const int32_t *chr_grp_off, const int32_t *grp_off, const int32_t *grp_idx, int m,
                                const double *Pi, const double *delta, const double *mean, const double *sd,
                                uint8_t *states) {
    ICNV_HOST_PROLOGUE();
    if (!X || !states || G <= 0 || C <= 0 || !Pi || !delta || !mean || !sd || !chr_grp_off)
        return set_error(ICNV_E_BAD_ARG, "icnv_viterbi_per_chr_u8_f64: bad argument");
    if (m != 6 && m != 3) return set_error(ICNV_E_BAD_ARG, "m must be 6 or 3");
    int rc = validate_chr(G, chr_start, chr_len, K);
    if (rc) return rc;
    if (chr_grp_off[0] != 0) return set_error(ICNV_E_BAD_ARG, "chr_grp_off[0] must be 0");
    for (int k = 0; k < K; ++k)
        if (chr_grp_off[k + 1] < chr_grp_off[k]) return set_error(ICNV_E_BAD_ARG, "chr_grp_off must be non-decreasing");
    const int n_tot = chr_grp_off[K];
    if (n_tot <= 0) return set_error(ICNV_E_BAD_ARG, "no subcluster given for any chromosome");
    if ((rc = validate_groups(C, grp_off, grp_idx, n_tot, false))) return rc;
    // group of every cell on every chromosome, per-group median sd (HMM.R:1122), chromosome of every gene
    std::vector<int32_t> grp_of((size_t)K * (size_t)C, -1), chr_id((size_t)G, 0);
    std::vector<double> sdm((size_t)n_tot);
    for (int k = 0; k < K; ++k) {
        for (int32_t g = chr_start[k]; g < chr_start[k] + chr_len[k]; ++g) chr_id[(size_t)g] = k;
        for (int b = chr_grp_off[k]; b < chr_grp_off[k + 1]; ++b)
            for (int32_t i = grp_off[b]; i < grp_off[b + 1]; ++i) {
                int32_t &slot = grp_of[(size_t)k * (size_t)C + (size_t)grp_idx[i]];
                if (slot >= 0) return set_error(ICNV_E_BAD_ARG, "cell %d is in two subclusters of chromosome %d", grp_idx[i], k);
                slot = b;
            }
    }
    for (int b = 0; b < n_tot; ++b) {
        std::vector<double> v(sd + (size_t)m * b, sd + (size_t)m * (b + 1));
        std::sort(v.begin(), v.end());
        sdm[(size_t)b] = (m & 1) ? v[m / 2] : 0.5 * (v[m / 2 - 1] + v[m / 2]);
        if (!(sdm[(size_t)b] > 0.0)) return set_error(ICNV_E_BAD_ARG, "state sd must be positive (group %d)", b);
    }
    double *dX;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    const int64_t n_idx = grp_off[n_tot];
    int32_t *d_idx = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)(n_idx + K * C + G));
    double *d_xm = (double *)scratch(SLOT_MEANS, sizeof(double) * (size_t)G * (size_t)n_tot);
    double *d_sd = (double *)scratch(SLOT_BOUNDS, sizeof(double) * (size_t)n_tot);
    uint8_t *d_st = (uint8_t *)scratch(SLOT_STATES, (size_t)G * (size_t)n_tot);
    uint8_t *d_out = (uint8_t *)scratch(SLOT_SLAB_ST0, (size_t)(G * C));
    int *d_flag = (int *)scratch(SLOT_MISC, 64);
    if (!d_idx || !d_xm || !d_sd || !d_st || !d_out || !d_flag) return ICNV_E_NOMEM;
    int32_t *d_grp_of = d_idx + n_idx, *d_chr_id = d_grp_of + (int64_t)K * C;
    ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
    ICNV_CUDA(cudaMemcpyAsync(d_idx, grp_idx, sizeof(int32_t) * (size_t)n_idx, cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaMemcpyAsync(d_grp_of, grp_of.data(), sizeof(int32_t) * grp_of.size(), cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaMemcpyAsync(d_chr_id, chr_id.data(), sizeof(int32_t) * (size_t)G, cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaMemcpyAsync(d_sd, sdm.data(), sizeof(double) * (size_t)n_tot, cudaMemcpyHostToDevice, st));
    // rowMeans of every (chromosome, subcluster) column over ALL genes - only its own chromosome's rows are used
    // below; the Viterbi of the other chromosomes' rows is redundant work on a G x n_tot matrix, small next to the
    // G x C upload
    if ((rc = dev_group_means(dX, G, G, d_idx, grp_off, n_tot, 0, d_xm, st))) return rc;
    rc = icnv_dev_viterbi_f64(d_xm, G, n_tot, chr_start, chr_len, K, m, Pi, delta, mean, d_sd, 1, d_st, nullptr, d_flag, st);
    if (rc) return rc;
    if ((rc = icnv_dev_scatter_states_per_chr_u8(d_st, G, C, d_chr_id, d_grp_of, d_out, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(states, d_out, (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    return check_flag(d_flag, st);   // synchronises: the host tables above outlive the copies
}

// ---- CNV region calling on the state matrix (R/inferCNV_HMM.R:706-1087) ----------------------------------------

static int check_state_flag(int *d_flag, cudaStream_t st) {
    int h = 0;
    ICNV_CUDA(cudaMemcpyAsync(&h, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    if (h & 4) return set_error(ICNV_E_BAD_ARG, "state outside 0..6 / 255 in the state matrix");
    return ICNV_OK;
}

// upload the states and the cell lists, run the consensus into SLOT_RG_CONS
static int host_consensus(const uint8_t *states, int64_t G, int64_t C, const int32_t *grp_off, const int32_t *grp_idx,
                          int n_grp, uint8_t **d_cons_out, cudaStream_t st) {
    uint8_t *dS = (uint8_t *)scratch(SLOT_STATES, (size_t)(G * C));
    int32_t *d_idx = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)grp_off[n_grp]);
    uint8_t *d_cons = (uint8_t *)scratch(SLOT_RG_CONS, (size_t)G * (size_t)n_grp);
    int *d_flag = (int *)scratch(SLOT_MISC, 64);
    if (!dS || !d_idx || !d_cons || !d_flag) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemcpyAsync(dS, states, (size_t)(G * C), cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaMemcpyAsync(d_idx, grp_idx, sizeof(int32_t) * (size_t)grp_off[n_grp], cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
    int rc = icnv_dev_state_consensus_u8(dS, G, G, d_idx, grp_off, n_grp, d_cons, d_flag, st);
    if (rc) return rc;
    if ((rc = check_state_flag(d_flag, st))) return rc;
    *d_cons_out = d_cons;
    return ICNV_OK;
}

int icnv_state_consensus_u8(const uint8_t *states, int64_t G, int64_t C, const int32_t *grp_off, const int32_t *grp_idx,
                            int n_grp, uint8_t *consensus) {
    ICNV_HOST_PROLOGUE();
    if (!states || !consensus || G <= 0 || C <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_state_consensus_u8: bad argument");
    int rc = validate_groups(C, grp_off, grp_idx, n_grp, false);
    if (rc) return rc;
    uint8_t *d_cons;
    if ((rc = host_consensus(states, G, C, grp_off, grp_idx, n_grp, &d_cons, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(consensus, d_cons, (size_t)G * (size_t)n_grp, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

/* get_predicted_CNV_regions(by = "subcluster") + the overwrite loop of HMM.R:472-483 as one pass */
int icnv_apply_state_consensus_u8(const uint8_t *states, int64_t G, int64_t C, const int32_t *chr_start,
                                  const int32_t *chr_len, int K, const int32_t *grp_off, const int32_t *grp_idx, int n_grp,
                                  uint8_t *out) {
    ICNV_HOST_PROLOGUE();
    if (!states || !out || G <= 0 || C <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_apply_state_consensus_u8: bad argument");
    int rc = validate_chr(G, chr_start, chr_len, K);
    if (rc) return rc;
    if ((rc = validate_groups(C, grp_off, grp_idx, n_grp, false))) return rc;
    std::vector<int32_t> tab((size_t)(G + C), -1);     // chr_of[G] (-1: chromosome with < 2 genes) | grp_of[C]
    for (int k = 0; k < K; ++k)
        for (int32_t g = chr_start[k]; g < chr_start[k] + chr_len[k]; ++g) tab[(size_t)g] = chr_len[k] >= 2 ? k : -1;
    for (int b = 0; b < n_grp; ++b)
        for (int32_t i = grp_off[b]; i < grp_off[b + 1]; ++i) {
            if (tab[(size_t)G + (size_t)grp_idx[i]] >= 0) return set_error(ICNV_E_BAD_ARG, "cell %d is in two groups", grp_idx[i]);
            tab[(size_t)G + (size_t)grp_idx[i]] = b;
        }
    uint8_t *d_cons;
    if ((rc = host_consensus(states, G, C, grp_off, grp_idx, n_grp, &d_cons, st))) return rc;   // states now in SLOT_STATES
    const uint8_t *dS = (const uint8_t *)ctx().slot_ptr[SLOT_STATES];
    int32_t *d_tab = (int32_t *)scratch(SLOT_IDX2, sizeof(int32_t) * tab.size());
    uint8_t *d_out = (uint8_t *)scratch(SLOT_SLAB_ST0, (size_t)(G * C));
    if (!d_tab || !d_out) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemcpyAsync(d_tab, tab.data(), sizeof(int32_t) * tab.size(), cudaMemcpyHostToDevice, st));
    if ((rc = icnv_dev_apply_consensus_u8(dS, d_cons, G, C, d_tab, d_tab + G, d_out, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(out, d_out, (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

static int validate_gene_positions(const double *gene_start, const double *gene_stop, int64_t G) {
    if (!gene_start || !gene_stop) return set_error(ICNV_E_BAD_ARG, "gene start / stop positions missing");
    for (int64_t g = 0; g < G; ++g)
        if (!std::isfinite(gene_start[g]) || !std::isfinite(gene_stop[g]))
            return set_error(ICNV_E_NONFINITE, "non-finite gene position at gene %lld", (long long)g);
    return ICNV_OK;
}

int icnv_cnv_regions_u8(const uint8_t *seqs, int64_t G, int64_t n_seq, const int32_t *chr_start, const int32_t *chr_len,
                        int K, const double *gene_start, const double *gene_stop, int64_t *n_regions) {
    ICNV_HOST_PROLOGUE();
    if (!seqs || !n_regions || G <= 0 || n_seq <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_cnv_regions_u8: bad argument");
    int rc = validate_chr(G, chr_start, chr_len, K);
    if (rc) return rc;
    if ((rc = validate_gene_positions(gene_start, gene_stop, G))) return rc;
    uint8_t *dS = (uint8_t *)scratch(SLOT_STATES, (size_t)(G * n_seq));
    if (!dS) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemcpyAsync(dS, seqs, (size_t)(G * n_seq), cudaMemcpyHostToDevice, st));
    return icnv_dev_cnv_regions_u8(dS, G, G, n_seq, nullptr, chr_start, chr_len, K, gene_start, gene_stop, n_regions, st);
}

int icnv_predicted_cnv_regions_u8(const uint8_t *states, int64_t G, int64_t C, const int32_t *chr_start,
                                  const int32_t *chr_len, int K, const double *gene_start, const double *gene_stop,
                                  const int32_t *grp_off, const int32_t *grp_idx, int n_grp, uint8_t *consensus,
                                  int64_t *n_regions) {
    ICNV_HOST_PROLOGUE();
    if (!states || !n_regions || G <= 0 || C <= 0)
        return set_error(ICNV_E_BAD_ARG, "icnv_predicted_cnv_regions_u8: bad argument");
    int rc = validate_chr(G, chr_start, chr_len, K);
    if (rc) return rc;
    if ((rc = validate_groups(C, grp_off, grp_idx, n_grp, false))) return rc;
    if ((rc = validate_gene_positions(gene_start, gene_stop, G))) return rc;
    bool singletons = !consensus;       // by = "cell": every group is one cell, its consensus is its own column
    for (int k = 0; k < n_grp && singletons; ++k) singletons = grp_off[k + 1] - grp_off[k] == 1;
    if (singletons) {
        uint8_t *dS = (uint8_t *)scratch(SLOT_STATES, (size_t)(G * C));
        int32_t *d_idx = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)n_grp);
        if (!dS || !d_idx) return ICNV_E_NOMEM;
        ICNV_CUDA(cudaMemcpyAsync(dS, states, (size_t)(G * C), cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_idx, grp_idx, sizeof(int32_t) * (size_t)n_grp, cudaMemcpyHostToDevice, st));
        return icnv_dev_cnv_regions_u8(dS, G, G, n_grp, d_idx, chr_start, chr_len, K, gene_start, gene_stop, n_regions, st);
    }
    uint8_t *d_cons;
    if ((rc = host_consensus(states, G, C, grp_off, grp_idx, n_grp, &d_cons, st))) return rc;
    if (consensus) ICNV_CUDA(cudaMemcpyAsync(consensus, d_cons, (size_t)G * (size_t)n_grp, cudaMemcpyDeviceToHost, st));
    return icnv_dev_cnv_regions_u8(d_cons, G, G, n_grp, nullptr, chr_start, chr_len, K, gene_start, gene_stop, n_regions, st);
}

int icnv_cnv_regions_fetch(int64_t n_regions, int32_t *seq, int32_t *chr, int32_t *first_gene, int32_t *last_gene,
                           int32_t *state, double *start, double *end) {
    ICNV_HOST_PROLOGUE();
    int64_t n = 0;
    const int32_t *d_seq, *d_chr, *d_first, *d_last, *d_state;
    const double *d_start, *d_end;
    int rc = icnv_dev_cnv_regions_records(&n, &d_seq, &d_chr, &d_first, &d_last, &d_state, &d_start, &d_end);
    if (rc) return rc;
    if (n_regions != n)
        return set_error(ICNV_E_BAD_ARG, "icnv_cnv_regions_fetch: %lld records asked for, the last region call produced %lld",
                         (long long)n_regions, (long long)n);
    if (n == 0) return ICNV_OK;
    const size_t bi = sizeof(int32_t) * (size_t)n, bd = sizeof(double) * (size_t)n;
    if (seq) ICNV_CUDA(cudaMemcpyAsync(seq, d_seq, bi, cudaMemcpyDeviceToHost, st));
    if (chr) ICNV_CUDA(cudaMemcpyAsync(chr, d_chr, bi, cudaMemcpyDeviceToHost, st));
    if (first_gene) ICNV_CUDA(cudaMemcpyAsync(first_gene, d_first, bi, cudaMemcpyDeviceToHost, st));
    if (last_gene) ICNV_CUDA(cudaMemcpyAsync(last_gene, d_last, bi, cudaMemcpyDeviceToHost, st));
    if (state) ICNV_CUDA(cudaMemcpyAsync(state, d_state, bi, cudaMemcpyDeviceToHost, st));
    if (start) ICNV_CUDA(cudaMemcpyAsync(start, d_start, bd, cudaMemcpyDeviceToHost, st));
    if (end) ICNV_CUDA(cudaMemcpyAsync(end, d_end, bd, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

/* normalize_counts_by_seq_depth, R/inferCNV_ops.R:3064-3111: x / colSums * normalize_factor; a negative or NaN
 * factor means "median of the column sums" (the reference's NA default). */
int icnv_normalize_counts_by_seq_depth_f64(const double *X, double *Y, int64_t G, int64_t C, double normalize_factor) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || G <= 1 || C <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_normalize_counts_by_seq_depth_f64: bad argument");
    double *dX;
    int rc;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    double *dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(G * C));
    double *d_sums = (double *)scratch(SLOT_PARTIAL, sizeof(double) * (size_t)C);
    if (!dY || !d_sums) return ICNV_E_NOMEM;
    if ((rc = icnv_dev_column_stats_f64(dX, G, nullptr, C, d_sums, nullptr, st))) return rc;
    if (!(normalize_factor >= 0.0)) {  // median of the C column sums: a C-vector, selected on the host
        std::vector<double> cs((size_t)C);
        ICNV_CUDA(cudaMemcpyAsync(cs.data(), d_sums, sizeof(double) * (size_t)C, cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        std::sort(cs.begin(), cs.end());
        normalize_factor = (C & 1) ? cs[C / 2] : 0.5 * (cs[C / 2 - 1] + cs[C / 2]);
    }
    if (!std::isfinite(normalize_factor)) return set_error(ICNV_E_NONFINITE, "Error, normalize factor not estimated");
    if ((rc = icnv_dev_scale_columns_f64(dX, dY, G, C, d_sums, normalize_factor, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

/* clear_noise_via_ref_mean_sd, R/inferCNV_ops.R:2302-2346 (noise_logistic = FALSE): mu = mean over all values of
 * the listed cells, s = sd_amplifier * mean over those cells of the per-cell sd; values strictly inside
 * (mu - s, mu + s) become mu.  idx = reference cells, or all observation cells when there are none. */
int icnv_clear_noise_via_ref_mean_sd_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *idx, int64_t n_idx,
                                         double sd_amplifier) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || !idx || G <= 1 || C <= 0 || n_idx <= 0)
        return set_error(ICNV_E_BAD_ARG, "icnv_clear_noise_via_ref_mean_sd_f64: bad argument");
    for (int64_t i = 0; i < n_idx; ++i)
        if (idx[i] < 0 || idx[i] >= C) return set_error(ICNV_E_BAD_ARG, "cell index out of range");
    double *dX;
    int rc;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    double *dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(G * C));
    int32_t *d_idx = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)n_idx);
    double *d_stats = (double *)scratch(SLOT_MEANS, sizeof(double) * 2 * (size_t)n_idx);
    if (!dY || !d_idx || !d_stats) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemcpyAsync(d_idx, idx, sizeof(int32_t) * (size_t)n_idx, cudaMemcpyHostToDevice, st));
    if ((rc = icnv_dev_column_stats_f64(dX, G, d_idx, n_idx, d_stats, d_stats + n_idx, st))) return rc;
    std::vector<double> h(2 * (size_t)n_idx);
    ICNV_CUDA(cudaMemcpyAsync(h.data(), d_stats, sizeof(double) * 2 * (size_t)n_idx, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    double tot = 0.0, sdsum = 0.0;   // n_idx-vectors: combined on the host in list order
    for (int64_t i = 0; i < n_idx; ++i) {
        tot += h[i];
        sdsum += h[n_idx + i];
    }
    const double mu = tot / ((double)G * (double)n_idx);
    const double s = (sdsum / (double)n_idx) * sd_amplifier;
    if ((rc = icnv_dev_clear_noise_f64(dX, dY, G * C, mu - s, mu + s, mu, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

// R's mean(): long-double sum, then one refinement pass (summary.c, real_mean)
static double r_mean_host(const double *x, int64_t n) {
    long double s = 0.0L;
    for (int64_t i = 0; i < n; ++i) s += x[i];
    s /= (long double)n;
    long double t = 0.0L;
    for (int64_t i = 0; i < n; ++i) t += (x[i] - s);
    s += t / (long double)n;
    return (double)s;
}

/* remove_outliers_norm / .remove_outliers_norm, R/inferCNV_ops.R:1969-2056 (run() step 16, prune_outliers): values
 * below lower_bound become lower_bound, values above upper_bound become upper_bound.  Both bounds given (not NaN):
 * hard thresholds.  Otherwise out_method "average_bound" (.get_average_bounds, ops.R:2734-2742): the mean over
 * the cells of each cell's smallest value, and of each cell's largest value.  bounds_out (may be NULL) receives the
 * two bounds used. */
int icnv_remove_outliers_norm_f64(const double *X, double *Y, int64_t G, int64_t C, double lower_bound, double upper_bound,
                                  double *bounds_out) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || G <= 0 || C <= 0)
        return set_error(ICNV_E_BAD_ARG, "Error, something is wrong with the data, either null or no rows or columns");
    double *dX;
    int rc;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    double *dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(G * C));
    if (!dY) return ICNV_E_NOMEM;
    if (!(lower_bound == lower_bound) || !(upper_bound == upper_bound)) {
        double *d_mm = (double *)scratch(SLOT_PARTIAL, sizeof(double) * 2 * (size_t)C);
        if (!d_mm) return ICNV_E_NOMEM;
        if ((rc = icnv_dev_column_minmax_f64(dX, G, C, d_mm, d_mm + C, st))) return rc;
        std::vector<double> mm(2 * (size_t)C);
        ICNV_CUDA(cudaMemcpyAsync(mm.data(), d_mm, sizeof(double) * 2 * (size_t)C, cudaMemcpyDeviceToHost, st));
        ICNV_CUDA(cudaStreamSynchronize(st));
        lower_bound = r_mean_host(mm.data(), C);
        upper_bound = r_mean_host(mm.data() + C, C);
    }
    if (bounds_out) {
        bounds_out[0] = lower_bound;
        bounds_out[1] = upper_bound;
    }
    if ((rc = icnv_dev_clamp_bounds_f64(dX, dY, G * C, lower_bound, upper_bound, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

// mean over all values of the listed cells (idx == NULL: all C cells) and mean of the per-cell sds
static int host_ref_mean_sd(const double *dX, int64_t G, int64_t C, const int32_t *idx, int64_t n_idx, double *mean,
                            double *mean_sd, cudaStream_t st) {
    const int64_t n = idx ? n_idx : C;
    int32_t *d_idx = nullptr;
    if (idx) {
        for (int64_t i = 0; i < n_idx; ++i)
            if (idx[i] < 0 || idx[i] >= C) return set_error(ICNV_E_BAD_ARG, "cell index out of range");
        d_idx = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)n_idx);
        if (!d_idx) return ICNV_E_NOMEM;
        ICNV_CUDA(cudaMemcpyAsync(d_idx, idx, sizeof(int32_t) * (size_t)n_idx, cudaMemcpyHostToDevice, st));
    }
    double *d_stats = (double *)scratch(SLOT_MEANS, sizeof(double) * 2 * (size_t)n);
    if (!d_stats) return ICNV_E_NOMEM;
    int rc = icnv_dev_column_stats_f64(dX, G, d_idx, n, d_stats, d_stats + n, st);
    if (rc) return rc;
    std::vector<double> h(2 * (size_t)n);
    ICNV_CUDA(cudaMemcpyAsync(h.data(), d_stats, sizeof(double) * 2 * (size_t)n, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    double tot = 0.0, sdsum = 0.0;   // n-vectors: combined on the host in list order
    for (int64_t i = 0; i < n; ++i) {
        tot += h[(size_t)i];
        sdsum += h[(size_t)(n + i)];
    }
    *mean = tot / ((double)G * (double)n);
    *mean_sd = sdsum / (double)n;
    return ICNV_OK;
}

/* clear_noise / .clear_noise, R/inferCNV_ops.R:2232-2275 (run() step 22 with a numeric noise_filter): centre = mean
 * over all values of the listed cells (reference cells; idx == NULL / n_idx == 0: all data, ops.R:2243-2247).
 * noise_logistic == 0: values strictly inside (centre - threshold, centre + threshold) become centre;
 * noise_logistic != 0: depress_log_signal_midpt_val(centre, threshold), slope 20 (R/inferCNV_heatmap.R:2783-2810).
 * threshold == 0: the matrix is returned unchanged (ops.R:2236-2238). */
int icnv_clear_noise_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *idx, int64_t n_idx, double threshold,
                         int noise_logistic) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || G <= 1 || C <= 0 || n_idx < 0) return set_error(ICNV_E_BAD_ARG, "icnv_clear_noise_f64: bad argument");
    if (threshold == 0.0) {
        if (Y != X) memcpy(Y, X, sizeof(double) * (size_t)(G * C));
        return ICNV_OK;
    }
    double *dX;
    int rc;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    double *dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(G * C));
    if (!dY) return ICNV_E_NOMEM;
    double mu, msd;
    if ((rc = host_ref_mean_sd(dX, G, C, n_idx > 0 ? idx : nullptr, n_idx, &mu, &msd, st))) return rc;
    if (noise_logistic)
        rc = icnv_dev_logistic_adj_f64(dX, dY, G * C, mu, threshold, 20.0, st);
    else
        rc = icnv_dev_clear_noise_f64(dX, dY, G * C, mu - threshold, mu + threshold, mu, st);
    if (rc) return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

/* clear_noise_via_ref_mean_sd with noise_logistic = TRUE, R/inferCNV_ops.R:2325-2329: the logistic depression around
 * the reference mean with midpoint sd_amplifier * mean(per-cell sd). */
int icnv_clear_noise_via_ref_mean_sd_logistic_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *idx,
                                                  int64_t n_idx, double sd_amplifier) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || !idx || G <= 1 || C <= 0 || n_idx <= 0)
        return set_error(ICNV_E_BAD_ARG, "icnv_clear_noise_via_ref_mean_sd_logistic_f64: bad argument");
    double *dX;
    int rc;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    double *dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(G * C));
    if (!dY) return ICNV_E_NOMEM;
    double mu, msd;
    if ((rc = host_ref_mean_sd(dX, G, C, idx, n_idx, &mu, &msd, st))) return rc;
    if ((rc = icnv_dev_logistic_adj_f64(dX, dY, G * C, mu, msd * sd_amplifier, 20.0, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

/* assign_HMM_states_to_proxy_expr_vals (HMM.R:1191-1206, m = 6) / i3HMM_assign_HMM_states_to_proxy_expr_vals
 * (i3HMM.R:405-417, m = 3) on a numeric state matrix of n entries. */
int icnv_assign_hmm_states_to_proxy_expr_vals_f64(const double *X, double *Y, int64_t n, int m) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || n <= 0 || (m != 6 && m != 3))
        return set_error(ICNV_E_BAD_ARG, "icnv_assign_hmm_states_to_proxy_expr_vals_f64: bad argument");
    double *dX;
    int rc;
    if ((rc = upload_matrix(X, n, &dX, SLOT_IN, st))) return rc;
    double *dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)n);
    if (!dY) return ICNV_E_NOMEM;
    if ((rc = icnv_dev_proxy_vals_f64(dX, dY, n, m, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

static int host_elementwise(const double *X, double *Y, int64_t n, int op, double param) {
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || n <= 0) return set_error(ICNV_E_BAD_ARG, "element-wise step: bad argument");
    double *dX;
    int rc;
    if ((rc = upload_matrix(X, n, &dX, SLOT_IN, st))) return rc;
    double *dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)n);
    int *d_flag = (int *)scratch(SLOT_MISC, 64);
    if (!dY || !d_flag) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
    if ((rc = icnv_dev_elementwise_f64(dX, dY, n, op, param, d_flag, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, st));
    return check_flag(d_flag, st);
}

int icnv_log2xplus1_f64(const double *X, double *Y, int64_t n) { return host_elementwise(X, Y, n, 0, 0.0); }
int icnv_invert_log2_f64(const double *X, double *Y, int64_t n) { return host_elementwise(X, Y, n, 1, 0.0); }
int icnv_apply_max_threshold_bounds_f64(const double *X, double *Y, int64_t n, double threshold) {
    if (!(threshold > 0.0)) return set_error(ICNV_E_BAD_ARG, "threshold must be positive");
    return host_elementwise(X, Y, n, 2, threshold);
}

int icnv_mean_sd_f64(const double *X, int64_t G, int64_t C, const int32_t *idx, int64_t n_idx, double *mu,
                     double *sigma) {
    ICNV_HOST_PROLOGUE();
    if (!X || !idx || !mu || !sigma || G <= 1 || C <= 0 || n_idx <= 0)
        return set_error(ICNV_E_BAD_ARG, "icnv_mean_sd_f64: bad argument");
    for (int64_t i = 0; i < n_idx; ++i)
        if (idx[i] < 0 || idx[i] >= C) return set_error(ICNV_E_BAD_ARG, "cell index out of range");
    // only the listed columns go to the device (the reference cells are a tenth of the matrix); the statistics then run over
    // the compact buffer's columns 0 .. n_idx-1
    int rc;
    double *dX = nullptr;
    int32_t *d_idx = nullptr;
    double *d_stats = (double *)scratch(SLOT_MEANS, sizeof(double) * 2 * (size_t)n_idx);
    if (!d_stats) return ICNV_E_NOMEM;
    if ((rc = upload_listed_columns(X, G, idx, n_idx, &dX, &d_idx, st))) return rc;
    // per-cell sum and sd on the device; the n_idx-vectors are combined in list order (the same
    // combination the multi-GPU driver applies to all-gathered per-cell statistics: identical bits)
    if ((rc = icnv_dev_column_stats_f64(dX, G, d_idx, n_idx, d_stats, d_stats + n_idx, st))) return rc;
    std::vector<double> h(2 * (size_t)n_idx);
    ICNV_CUDA(cudaMemcpyAsync(h.data(), d_stats, sizeof(double) * 2 * (size_t)n_idx, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    icnv_combine_cell_stats(h.data(), h.data() + n_idx, n_idx, G, mu, sigma);
    return ICNV_OK;
}

int icnv_pairwise_dist_f64(const double *X, int64_t G, int64_t C, const int32_t *cells, int64_t n, double *out) {
    ICNV_HOST_PROLOGUE();
    if (!cells) n = C;
    if (!X || G < 0 || C <= 0 || n < 0 || (n >= 2 && !out)) return set_error(ICNV_E_BAD_ARG, "icnv_pairwise_dist_f64: bad argument");
    for (int64_t i = 0; cells && i < n; ++i)
        if (cells[i] < 0 || cells[i] >= C) return set_error(ICNV_E_BAD_ARG, "cell index out of range");
    if (n < 2) return ICNV_OK;
    const size_t n_out = (size_t)n * (size_t)(n - 1) / 2;
    double *dX = nullptr, *d_out = (double *)scratch(SLOT_OUT, sizeof(double) * n_out);
    int32_t *d_idx = cells ? (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)n) : nullptr;
    int rc;
    if (!d_out || (cells && !d_idx)) return ICNV_E_NOMEM;
    if (G > 0 && (rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    if (G == 0) dX = d_out;   // never read
    if (cells) ICNV_CUDA(cudaMemcpyAsync(d_idx, cells, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, st));
    if ((rc = icnv_dev_pairwise_dist_f64(dX, G, G, d_idx, n, d_out, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(out, d_out, sizeof(double) * n_out, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

int icnv_pairwise_dist_rows_f64(const double *x, int64_t n, int64_t G, double *out) {
    ICNV_HOST_PROLOGUE();
    if (!x || G < 0 || n < 0 || (n >= 2 && !out)) return set_error(ICNV_E_BAD_ARG, "icnv_pairwise_dist_rows_f64: bad argument");
    if (n < 2) return ICNV_OK;
    const size_t n_out = (size_t)n * (size_t)(n - 1) / 2;
    double *dX = nullptr, *d_out = (double *)scratch(SLOT_OUT, sizeof(double) * n_out);
    int rc;
    if (!d_out) return ICNV_E_NOMEM;
    if (G > 0 && (rc = upload_matrix(x, G * n, &dX, SLOT_IN, st))) return rc;
    if (G == 0) dX = d_out;   // never read
    if ((rc = icnv_dev_pairwise_dist_rows_f64(dX, n, n, G, d_out, st))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(out, d_out, sizeof(double) * n_out, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

// k nearest neighbours: the input goes up whole (it is all K12 holds besides O(n k)), the n x k results come back
static int knn_host(const double *X, int64_t G, int64_t C, const int32_t *cells, int64_t n, int k, int32_t *idx, double *dist,
                    int rows, const char *who) {
    ICNV_HOST_PROLOGUE();
    if (!X || G < 0 || n < 0 || (!rows && C < 0) || (n > 0 && (!idx || !dist))) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    for (int64_t i = 0; cells && i < n; ++i)
        if (cells[i] < 0 || cells[i] >= C) return set_error(ICNV_E_BAD_ARG, "%s: cell index out of range", who);
    if (n == 0) return ICNV_OK;
    if (k < 1 || k > n) return set_error(ICNV_E_BAD_ARG, "%s: k = %d for %lld cells (1 <= k <= n)", who, k, (long long)n);
    if (k > ICNV_KNN_MAX_K) return set_error(ICNV_E_UNSUPPORTED, "%s: k = %d (limit %d)", who, k, ICNV_KNN_MAX_K);
    const size_t nk = (size_t)n * (size_t)k;
    double *d_dist = (double *)scratch(SLOT_OUT, (sizeof(double) + sizeof(int32_t)) * nk);
    int32_t *d_idx = (int32_t *)(d_dist + nk);
    int32_t *d_cells = cells ? (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)n) : nullptr;
    double *dX = nullptr;
    int rc;
    if (!d_dist || (cells && !d_cells)) return ICNV_E_NOMEM;
    if (G > 0 && (rc = upload_matrix(X, G * (rows ? n : C), &dX, SLOT_IN, st))) return rc;
    if (G == 0) dX = d_dist;   // never read
    if (cells) ICNV_CUDA(cudaMemcpyAsync(d_cells, cells, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, st));
    if ((rc = knn_launch(dX, G, rows ? n : G, d_cells, n, k, d_idx, d_dist, rows, st, who))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(idx, d_idx, sizeof(int32_t) * nk, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaMemcpyAsync(dist, d_dist, sizeof(double) * nk, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

int icnv_knn_f64(const double *X, int64_t G, int64_t C, const int32_t *cells, int64_t n, int k, int32_t *idx, double *dist) {
    if (!cells) n = C;
    return knn_host(X, G, C, cells, n, k, idx, dist, 0, "icnv_knn_f64");
}

int icnv_knn_rows_f64(const double *x, int64_t n, int64_t G, int k, int32_t *idx, double *dist) {
    return knn_host(x, G, n, nullptr, n, k, idx, dist, 1, "icnv_knn_rows_f64");
}

/* mu, sigma (n-1) over all values of n cells from the cells' own (sum, sd): sum of squares about mu of a cell =
 * sd_c^2 (G-1) + G (mean_c - mu)^2.  Plain host arithmetic on 2n numbers, in list order. */
void icnv_combine_cell_stats(const double *sums, const double *sds, int64_t n, int64_t G, double *mu, double *sigma) {
    double tot = 0.0;
    for (int64_t i = 0; i < n; ++i) tot += sums[i];
    const double N = (double)G * (double)n;
    const double m = tot / N;
    double ss = 0.0;
    for (int64_t i = 0; i < n; ++i) {
        const double d = sums[i] / (double)G - m;
        ss += sds[i] * sds[i] * (double)(G - 1) + (double)G * d * d;
    }
    *mu = m;
    *sigma = std::sqrt(ss / (N - 1.0));
}

}  // extern "C"

// ---- hclust (kernels and bodies in icnv_hclust.cu) ---------------------------------------------------------------------
// Weak references: a library built without icnv_hclust.cu - the host emulation of the other kernels' source - still loads
// and exports every entry point of the header; there the linkage entry points report ICNV_E_UNSUPPORTED.
namespace icnv {
int hclust_host(const double *d, int64_t n, int method, int32_t *merge, double *height, int32_t *order) __attribute__((weak));
int hclust_dev(const double *d_dist, int64_t n, int method, int32_t *merge, double *height, void *stream) __attribute__((weak));
}  // namespace icnv

extern "C" {

int icnv_hclust_f64(const double *d, int64_t n, int method, int32_t *merge, double *height, int32_t *order) {
    if (!icnv::hclust_host) return set_error(ICNV_E_UNSUPPORTED, "icnv_hclust_f64: this build has no linkage kernel");
    return icnv::hclust_host(d, n, method, merge, height, order);
}

int icnv_dev_hclust_f64(const double *d_dist, int64_t n, int method, int32_t *merge, double *height, void *stream) {
    if (!icnv::hclust_dev) return set_error(ICNV_E_UNSUPPORTED, "icnv_dev_hclust_f64: this build has no linkage kernel");
    return icnv::hclust_dev(d_dist, n, method, merge, height, stream);
}

// R's order: hcass2's traversal - start from the last merge, expand the first column before the second.
int icnv_hclust_order(const int32_t *merge, int64_t n, int32_t *order) {
    if (!merge || !order || n < 1) return set_error(ICNV_E_BAD_ARG, "icnv_hclust_order: bad argument");
    if (n == 1) {
        order[0] = 1;
        return ICNV_OK;
    }
    const int64_t nm = n - 1;
    std::vector<int32_t> stack;
    stack.reserve((size_t)n);
    stack.push_back((int32_t)nm);   // 1-based merge number
    int64_t out = 0;
    while (!stack.empty()) {
        const int32_t v = stack.back();
        stack.pop_back();
        if (v < 0) {
            if (out >= n || -v > n) return set_error(ICNV_E_BAD_ARG, "icnv_hclust_order: merge is not a tree");
            order[out++] = -v;
            continue;
        }
        if (v < 1 || v > nm) return set_error(ICNV_E_BAD_ARG, "icnv_hclust_order: merge is not a tree");
        stack.push_back(merge[nm + v - 1]);
        stack.push_back(merge[v - 1]);
    }
    if (out != n) return set_error(ICNV_E_BAD_ARG, "icnv_hclust_order: merge is not a tree");
    return ICNV_OK;
}

}  // extern "C"

// ---- running means and the random-trees null (kernels and the device body in icnv_random_trees.cu) -------------------------
// Weak references, as for the linkage: a build without icnv_random_trees.cu reports them as unsupported.
namespace icnv {
int runmean_launch(const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t G, int64_t ncols, const int32_t *d_rs,
                   const int32_t *d_rl, int K, int k, int *flag, cudaStream_t st) __attribute__((weak));
int random_trees_dev(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n, int window, int method,
                     int n_perm, unsigned long long seed, int32_t *merge, double *height, double *perm_max, void *stream,
                     const char *who) __attribute__((weak));
void random_trees_stats(double *out5) __attribute__((weak));
}  // namespace icnv

extern "C" {

int icnv_runmean_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *chr_start, const int32_t *chr_len,
                     int K, int k) {
    if (!icnv::runmean_launch) return set_error(ICNV_E_UNSUPPORTED, "icnv_runmean_f64: this build has no running-mean kernel");
    ICNV_HOST_PROLOGUE();
    if (!X || !Y || G <= 0 || C <= 0 || (chr_start && (!chr_len || K < 0)))
        return set_error(ICNV_E_BAD_ARG, "icnv_runmean_f64: bad argument");
    if (!chr_start) K = 1;
    for (int r = 0; chr_start && r < K; ++r) {   // ranges in order, disjoint, inside [0, G)
        const int64_t prev_end = r ? (int64_t)chr_start[r - 1] + chr_len[r - 1] : 0;
        if (chr_len[r] < 0 || chr_start[r] < prev_end || (int64_t)chr_start[r] + chr_len[r] > G)
            return set_error(ICNV_E_BAD_ARG, "icnv_runmean_f64: range %d [%d, +%d) is not ordered and disjoint inside [0, %lld)",
                             r, chr_start[r], chr_len[r], (long long)G);
    }
    int rc;
    double *dX = nullptr, *dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(G * C));
    int32_t *d_r = (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * 2 * (size_t)K + 16);
    int *d_flag = (int *)scratch(SLOT_MISC, 64);
    if (!dY || !d_r || !d_flag) return ICNV_E_NOMEM;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    ICNV_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
    if (chr_start) {
        ICNV_CUDA(cudaMemcpyAsync(d_r, chr_start, sizeof(int32_t) * (size_t)K, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaMemcpyAsync(d_r + K, chr_len, sizeof(int32_t) * (size_t)K, cudaMemcpyHostToDevice, st));
    }
    if ((rc = icnv::runmean_launch(dX, G, dY, G, G, C, chr_start ? d_r : nullptr, chr_start ? d_r + K : nullptr, K, k, d_flag, st)))
        return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    return check_flag(d_flag, st);
}

int icnv_dev_random_tree_heights_f64(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n, int window,
                                     int method, int n_perm, uint64_t seed, int32_t *merge, double *height, double *perm_max,
                                     void *stream) {
    if (!icnv::random_trees_dev)
        return set_error(ICNV_E_UNSUPPORTED, "icnv_dev_random_tree_heights_f64: this build has no random-trees kernels");
    return icnv::random_trees_dev(X, G, ldx, d_cells, n, window, method, n_perm, seed, merge, height, perm_max, stream,
                                  "icnv_dev_random_tree_heights_f64");
}

int icnv_random_tree_heights_f64(const double *X, int64_t G, int64_t C, const int32_t *cells, int64_t n, int window,
                                 int method, int n_perm, uint64_t seed, int32_t *merge, double *height, int32_t *order,
                                 double *perm_max) {
    if (!icnv::random_trees_dev)
        return set_error(ICNV_E_UNSUPPORTED, "icnv_random_tree_heights_f64: this build has no random-trees kernels");
    ICNV_HOST_PROLOGUE();
    if (!cells) n = C;
    if (!X || G <= 0 || C <= 0 || !merge || !height || !order || (n_perm > 0 && !perm_max))
        return set_error(ICNV_E_BAD_ARG, "icnv_random_tree_heights_f64: bad argument");
    for (int64_t i = 0; cells && i < n; ++i)
        if (cells[i] < 0 || cells[i] >= C) return set_error(ICNV_E_BAD_ARG, "icnv_random_tree_heights_f64: cell index out of range");
    const int64_t nm = n > 1 ? n - 1 : 0, np = n_perm > 0 ? n_perm : 0;
    int rc;
    double *dX = nullptr, *d_out = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(nm + np) + sizeof(int32_t) * 2 * (size_t)nm);
    int32_t *d_idx = cells ? (int32_t *)scratch(SLOT_IDX, sizeof(int32_t) * (size_t)std::max<int64_t>(n, 1)) : nullptr;
    if (!d_out || (cells && !d_idx)) return ICNV_E_NOMEM;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    if (cells && n > 0) ICNV_CUDA(cudaMemcpyAsync(d_idx, cells, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, st));
    double *d_height = d_out, *d_perm = d_out + nm;
    int32_t *d_merge = (int32_t *)(d_perm + np);
    if ((rc = icnv::random_trees_dev(dX, G, G, d_idx, n, window, method, n_perm, seed, d_merge, d_height, d_perm, st,
                                     "icnv_random_tree_heights_f64")))
        return rc;
    ICNV_CUDA(cudaMemcpyAsync(height, d_height, sizeof(double) * (size_t)nm, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaMemcpyAsync(merge, d_merge, sizeof(int32_t) * 2 * (size_t)nm, cudaMemcpyDeviceToHost, st));
    if (np) ICNV_CUDA(cudaMemcpyAsync(perm_max, d_perm, sizeof(double) * (size_t)np, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return icnv_hclust_order(merge, n, order);
}

int icnv_debug_random_trees(double *out5) {
    if (!out5) return set_error(ICNV_E_BAD_ARG, "icnv_debug_random_trees: out5 is NULL");
    for (int i = 0; i < 5; ++i) out5[i] = 0.0;
    if (icnv::random_trees_stats) icnv::random_trees_stats(out5);
    return ICNV_OK;
}

}  // extern "C"

// ---- masking of non-DE genes (kernels and the device body in icnv_de.cu) ---------------------------------------------------
// Weak references, as for the linkage: a build without icnv_de.cu reports it as unsupported.
namespace icnv {
int de_mask_dev(const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t G, int64_t C, const int32_t *ref_off,
                const int32_t *ref_idx, int n_ref, const int32_t *sub_off, const int32_t *sub_idx, int n_sub, int test,
                double p_thresh, int rule, double mask_val, double jitter_mean, double jitter_sd, unsigned long long seed,
                double *p_raw, double *p_adj, void *stream, const char *who) __attribute__((weak));
void de_mask_stats(double *out7) __attribute__((weak));
void de_mask_set_stats(const double *in7) __attribute__((weak));
int de_pack_dev(const double *X, int64_t ldx, const int32_t *d_cols, int64_t m, int n_dst, const int64_t *gene_lo,
                const int64_t *gene_hi, double *out, int *flag, void *stream, const char *who) __attribute__((weak));
int de_place_dev(const double *R, int64_t n, int n_src, const int64_t *src_m, const int32_t *d_tags, int64_t T, double *Z,
                 void *stream, const char *who) __attribute__((weak));
int de_slab_tests_dev(const double *Z, int64_t T, int64_t g0, int64_t n, const int32_t *ref_off, int n_ref,
                      const int32_t *sub_off, int n_sub, int test, double jitter_mean, double jitter_sd,
                      unsigned long long seed, double *p_raw, int64_t ldp, void *stream, double *times,
                      const char *who) __attribute__((weak));
int de_bh_mask_dev(const double *p_raw, int64_t G, int n_ref, int n_sub, const int32_t *sub_size, double p_thresh,
                   double *p_adj, const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t C, const int32_t *ref_idx,
                   int64_t n_ref_cells, const int32_t *sub_off, const int32_t *sub_idx, int rule, double mask_val,
                   void *stream, double *times, const char *who) __attribute__((weak));
// several device slots (icnv_de_multi.cu)
int de_mask_multi(int n_dev, const double *X, double *Y, int64_t G, int64_t C, const int32_t *ref_off, const int32_t *ref_idx,
                  int n_ref, const int32_t *sub_off, const int32_t *sub_idx, int n_sub, int test, double p_thresh, int rule,
                  double mask_val, double jitter_mean, double jitter_sd, uint64_t seed, double *p_raw,
                  double *p_adj) __attribute__((weak));

}  // namespace icnv

extern "C" {

int icnv_dev_mask_non_de_f64(const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t G, int64_t C,
                             const int32_t *ref_off, const int32_t *ref_idx, int n_ref, const int32_t *sub_off,
                             const int32_t *sub_idx, int n_sub, int test, double p_thresh, int rule, double mask_val,
                             double jitter_mean, double jitter_sd, uint64_t seed, double *p_raw, double *p_adj, void *stream) {
    if (!icnv::de_mask_dev) return set_error(ICNV_E_UNSUPPORTED, "icnv_dev_mask_non_de_f64: this build has no DE kernels");
    return icnv::de_mask_dev(X, ldx, Y, ldy, G, C, ref_off, ref_idx, n_ref, sub_off, sub_idx, n_sub, test, p_thresh, rule,
                             mask_val, jitter_mean, jitter_sd, seed, p_raw, p_adj, stream, "icnv_dev_mask_non_de_f64");
}

int icnv_mask_non_de_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *ref_off, const int32_t *ref_idx,
                         int n_ref, const int32_t *sub_off, const int32_t *sub_idx, int n_sub, int test, double p_thresh,
                         int rule, double mask_val, double jitter_mean, double jitter_sd, uint64_t seed, double *p_raw,
                         double *p_adj) {
    if (!icnv::de_mask_dev) return set_error(ICNV_E_UNSUPPORTED, "icnv_mask_non_de_f64: this build has no DE kernels");
    ICNV_HOST_PROLOGUE();
    if (!X || G <= 0 || C <= 0 || n_ref < 1 || n_sub < 0) return set_error(ICNV_E_BAD_ARG, "icnv_mask_non_de_f64: bad argument");
    if (device_slots() > 1) {
        if (!icnv::de_mask_multi) return set_error(ICNV_E_UNSUPPORTED, "icnv_mask_non_de_f64: this build has no multi-device DE path");
        return icnv::de_mask_multi(device_slots(), X, Y, G, C, ref_off, ref_idx, n_ref, sub_off, sub_idx, n_sub, test, p_thresh, rule,
                                   mask_val, jitter_mean, jitter_sd, seed, p_raw, p_adj);
    }
    const int64_t npair = (int64_t)n_sub * n_ref;
    int rc;
    double *dX = nullptr;
    double *d_p = (p_raw || p_adj) && npair > 0 ? (double *)scratch(SLOT_OUT, sizeof(double) * 2 * (size_t)(G * npair)) : nullptr;
    if ((p_raw || p_adj) && npair > 0 && !d_p) return ICNV_E_NOMEM;
    if ((rc = upload_matrix(X, G * C, &dX, SLOT_IN, st))) return rc;
    // the mask is written in place over the device copy (each entry is read and written by the same thread)
    if ((rc = icnv::de_mask_dev(dX, G, Y ? dX : nullptr, G, G, C, ref_off, ref_idx, n_ref, sub_off, sub_idx, n_sub, test,
                                p_thresh, rule, mask_val, jitter_mean, jitter_sd, seed, d_p, d_p ? d_p + G * npair : nullptr,
                                st, "icnv_mask_non_de_f64")))
        return rc;
    if (Y) ICNV_CUDA(cudaMemcpyAsync(Y, dX, sizeof(double) * (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    if (p_raw && d_p) ICNV_CUDA(cudaMemcpyAsync(p_raw, d_p, sizeof(double) * (size_t)(G * npair), cudaMemcpyDeviceToHost, st));
    if (p_adj && d_p)
        ICNV_CUDA(cudaMemcpyAsync(p_adj, d_p + G * npair, sizeof(double) * (size_t)(G * npair), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

int icnv_dev_de_pack_f64(const double *X, int64_t ldx, const int32_t *d_cols, int64_t m, int n_dst, const int64_t *gene_lo,
                         const int64_t *gene_hi, double *out, int *err_flag, void *stream) {
    if (!icnv::de_pack_dev) return set_error(ICNV_E_UNSUPPORTED, "icnv_dev_de_pack_f64: this build has no DE kernels");
    return icnv::de_pack_dev(X, ldx, d_cols, m, n_dst, gene_lo, gene_hi, out, err_flag, stream, "icnv_dev_de_pack_f64");
}

int icnv_dev_de_place_f64(const double *R, int64_t n, int n_src, const int64_t *src_m, const int32_t *d_tags, int64_t T,
                          double *Z, void *stream) {
    if (!icnv::de_place_dev) return set_error(ICNV_E_UNSUPPORTED, "icnv_dev_de_place_f64: this build has no DE kernels");
    return icnv::de_place_dev(R, n, n_src, src_m, d_tags, T, Z, stream, "icnv_dev_de_place_f64");
}

int icnv_dev_de_slab_tests_f64(const double *Z, int64_t T, int64_t g0, int64_t n, const int32_t *ref_off, int n_ref,
                               const int32_t *sub_off, int n_sub, int test, double jitter_mean, double jitter_sd, uint64_t seed,
                               double *p_raw, int64_t ldp, void *stream) {
    if (!icnv::de_slab_tests_dev) return set_error(ICNV_E_UNSUPPORTED, "icnv_dev_de_slab_tests_f64: this build has no DE kernels");
    return icnv::de_slab_tests_dev(Z, T, g0, n, ref_off, n_ref, sub_off, n_sub, test, jitter_mean, jitter_sd, seed, p_raw, ldp,
                                   stream, nullptr, "icnv_dev_de_slab_tests_f64");
}

int icnv_dev_de_bh_mask_f64(const double *p_raw, int64_t G, int n_ref, int n_sub, const int32_t *sub_size, double p_thresh,
                            double *p_adj, const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t C,
                            const int32_t *ref_idx, int64_t n_ref_cells, const int32_t *sub_off, const int32_t *sub_idx,
                            int rule, double mask_val, void *stream) {
    if (!icnv::de_bh_mask_dev) return set_error(ICNV_E_UNSUPPORTED, "icnv_dev_de_bh_mask_f64: this build has no DE kernels");
    return icnv::de_bh_mask_dev(p_raw, G, n_ref, n_sub, sub_size, p_thresh, p_adj, X, ldx, Y, ldy, C, ref_idx, n_ref_cells,
                                sub_off, sub_idx, rule, mask_val, stream, nullptr, "icnv_dev_de_bh_mask_f64");
}

int icnv_debug_mask_non_de(double *out7) {
    if (!out7) return set_error(ICNV_E_BAD_ARG, "icnv_debug_mask_non_de: out7 is NULL");
    for (int i = 0; i < 7; ++i) out7[i] = 0.0;
    if (icnv::de_mask_stats) icnv::de_mask_stats(out7);
    return ICNV_OK;
}

}  // extern "C"

// ---- Bayesian network filter (kernels and the device body in icnv_bayes.cu) -------------------------------------------------
// Weak references, as for the linkage: a build without icnv_bayes.cu reports it as unsupported.
namespace icnv {
int bayesnet_dev(const double *X, int64_t ldx, int64_t G, int64_t C, const int32_t *gene_off, const int32_t *gene_idx,
                 const int32_t *cell_off, const int32_t *cell_idx, const uint8_t *pooled, int n_reg, int m, const double *mu,
                 const double *tau, int n_chains, int n_burn, int n_keep, unsigned long long seed, double *theta,
                 int32_t *state_counts, double *loglik, void *stream, const char *who) __attribute__((weak));
void bayesnet_stats(double *out4) __attribute__((weak));
int bayesnet_check(int64_t G, int64_t C, const int32_t *gene_off, const int32_t *gene_idx, const int32_t *cell_off,
                   const int32_t *cell_idx, const uint8_t *pooled, int n_reg, int m, const double *mu, const double *tau,
                   int n_chains, int n_burn, int n_keep, int64_t *n_cols, const char *who) __attribute__((weak));

// The G x C host matrix into SLOT_IN.  Page-locked memory goes over PCIe directly; pageable memory (an R matrix) goes through
// the two pinned ring slots in chunks, the copy threads filling one slot while the other one's DMA runs.
static int upload_matrix_ring(const double *X, int64_t n, double **dX, cudaStream_t st) {
    Ctx &c = ctx();
    *dX = (double *)scratch(SLOT_IN, sizeof(double) * (size_t)n);
    if (!*dX) return ICNV_E_NOMEM;
    if (is_pinned(X)) {
        ICNV_CUDA(cudaMemcpyAsync(*dX, X, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice, st));
        return ICNV_OK;
    }
    const int64_t chunk = std::min<int64_t>(n, (int64_t)40 << 20);   // 320 MB per ring slot
    double *p[2];
    for (int b = 0; b < 2; ++b)
        if (!(p[b] = (double *)pinned(b, sizeof(double) * (size_t)chunk))) return ICNV_E_NOMEM;
    CopyPool pool(pool_threads_per_device());
    int64_t i = 0;
    for (int64_t q = 0; q < n; q += chunk, ++i) {
        const int b = (int)(i & 1);
        const int64_t nq = std::min<int64_t>(chunk, n - q);
        ICNV_CUDA(cudaEventSynchronize(c.ev_h2d[b]));   // the slot's previous DMA is done (a recorded-never event is complete)
        pool.copy2(p[b], X + q, sizeof(double) * (size_t)nq, nullptr, nullptr, 0);
        ICNV_CUDA(cudaMemcpyAsync(*dX + q, p[b], sizeof(double) * (size_t)nq, cudaMemcpyHostToDevice, st));
        ICNV_CUDA(cudaEventRecord(c.ev_h2d[b], st));
    }
    return ICNV_OK;
}
}  // namespace icnv

extern "C" {

int icnv_dev_bayesnet_f64(const double *X, int64_t ldx, int64_t G, int64_t C, const int32_t *gene_off, const int32_t *gene_idx,
                          const int32_t *cell_off, const int32_t *cell_idx, const uint8_t *pooled, int n_reg, int m,
                          const double *mu, const double *tau, int n_chains, int n_burn, int n_keep, uint64_t seed,
                          double *theta, int32_t *state_counts, double *loglik, void *stream) {
    if (!icnv::bayesnet_dev) return set_error(ICNV_E_UNSUPPORTED, "icnv_dev_bayesnet_f64: this build has no Bayesian network kernels");
    return icnv::bayesnet_dev(X, ldx, G, C, gene_off, gene_idx, cell_off, cell_idx, pooled, n_reg, m, mu, tau, n_chains, n_burn,
                              n_keep, seed, theta, state_counts, loglik, stream, "icnv_dev_bayesnet_f64");
}

int icnv_bayesnet_f64(const double *X, int64_t G, int64_t C, const int32_t *gene_off, const int32_t *gene_idx,
                      const int32_t *cell_off, const int32_t *cell_idx, const uint8_t *pooled, int n_reg, int m,
                      const double *mu, const double *tau, int n_chains, int n_burn, int n_keep, uint64_t seed, double *theta,
                      int32_t *state_counts, double *loglik) {
    if (!icnv::bayesnet_dev) return set_error(ICNV_E_UNSUPPORTED, "icnv_bayesnet_f64: this build has no Bayesian network kernels");
    ICNV_HOST_PROLOGUE();
    if (!X || !theta || !state_counts) return set_error(ICNV_E_BAD_ARG, "icnv_bayesnet_f64: bad argument");
    // every host-side check before the matrix goes up
    int64_t n_cols = 0;
    int rc = icnv::bayesnet_check(G, C, gene_off, gene_idx, cell_off, cell_idx, pooled, n_reg, m, mu, tau, n_chains, n_burn,
                                  n_keep, &n_cols, "icnv_bayesnet_f64");
    if (rc || n_reg == 0) return rc;
    const int64_t mm = m;
    const size_t b_theta = sizeof(double) * (size_t)n_reg * (size_t)n_chains * (size_t)n_keep * (size_t)mm,
                 b_counts = sizeof(int32_t) * (size_t)(n_cols * mm), b_ll = loglik ? sizeof(double) * (size_t)(n_cols * mm) : 0;
    double *dX = nullptr;
    if ((rc = upload_matrix_ring(X, G * C, &dX, st))) return rc;
    char *d_out = nullptr;
    if (cudaMalloc((void **)&d_out, b_theta + b_counts + b_ll + 512) != cudaSuccess) {
        cudaGetLastError();
        return set_error(ICNV_E_NOMEM, "icnv_bayesnet_f64: no room for the %zu-byte theta draws", b_theta);
    }
    double *d_theta = (double *)d_out;
    int32_t *d_counts = (int32_t *)(d_out + ((b_theta + 255) & ~(size_t)255));
    double *d_ll = loglik ? (double *)(d_out + ((b_theta + 255) & ~(size_t)255) + ((b_counts + 255) & ~(size_t)255)) : nullptr;
    rc = icnv::bayesnet_dev(dX, G, G, C, gene_off, gene_idx, cell_off, cell_idx, pooled, n_reg, m, mu, tau, n_chains, n_burn,
                            n_keep, seed, d_theta, d_counts, d_ll, st, "icnv_bayesnet_f64");
    if (!rc) {
        cudaError_t e = cudaMemcpyAsync(theta, d_theta, b_theta, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(state_counts, d_counts, b_counts, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess && loglik) e = cudaMemcpyAsync(loglik, d_ll, b_ll, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) rc = set_error(ICNV_E_CUDA, "icnv_bayesnet_f64: copy back failed: %s", cudaGetErrorString(e));
    }
    cudaStreamSynchronize(st);
    cudaFree(d_out);
    return rc;
}

int icnv_debug_bayesnet(double *out4) {
    if (!out4) return set_error(ICNV_E_BAD_ARG, "icnv_debug_bayesnet: out4 is NULL");
    for (int i = 0; i < 4; ++i) out4[i] = 0.0;
    if (icnv::bayesnet_stats) icnv::bayesnet_stats(out4);
    return ICNV_OK;
}

}  // extern "C"

// ---- coordinate-weighted smoothing (the kernel and the device body in icnv_smooth_coords.cu) --------------------------------
// Weak reference, as for the linkage: a build without icnv_smooth_coords.cu reports it as unsupported.
namespace icnv {
int smooth_coords_dev(const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t G, int64_t C, const int32_t *chr_start,
                      const int32_t *chr_len, int K, const double *gene_start, const double *gene_stop, double W,
                      cudaStream_t st, const char *who) __attribute__((weak));

// Ranges ordered and disjoint inside [0, G); finite coordinates for every gene of a range; a finite window.
static int smooth_coords_check(int64_t G, int64_t C, const int32_t *chr_start, const int32_t *chr_len, int K,
                               const double *gene_start, const double *gene_stop, double W, const char *who) {
    if (G <= 0 || C <= 0 || K < 0 || (K > 0 && (!chr_start || !chr_len)) || !gene_start || !gene_stop)
        return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    if (G > (int64_t)65535 * 32 || G > INT32_MAX)
        return set_error(ICNV_E_UNSUPPORTED, "%s: %lld genes (at most %d)", who, (long long)G, 65535 * 32);
    if (!std::isfinite(W)) return set_error(ICNV_E_BAD_ARG, "%s: window_length is not finite", who);
    for (int r = 0; r < K; ++r) {
        const int64_t prev_end = r ? (int64_t)chr_start[r - 1] + chr_len[r - 1] : 0;
        if (chr_len[r] < 0 || chr_start[r] < prev_end || (int64_t)chr_start[r] + chr_len[r] > G)
            return set_error(ICNV_E_BAD_ARG, "%s: range %d [%d, +%d) is not ordered and disjoint inside [0, %lld)", who, r,
                             chr_start[r], chr_len[r], (long long)G);
        for (int64_t g = chr_start[r]; g < (int64_t)chr_start[r] + chr_len[r]; ++g)
            if (!std::isfinite(gene_start[g]) || !std::isfinite(gene_stop[g]))
                return set_error(ICNV_E_BAD_ARG, "%s: gene %lld has a non-finite start or stop", who, (long long)g);
    }
    return ICNV_OK;
}
}  // namespace icnv

extern "C" {

int icnv_smooth_coordinates_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *chr_start,
                                const int32_t *chr_len, int K, const double *gene_start, const double *gene_stop,
                                double window_length) {
    static const char *who = "icnv_smooth_coordinates_f64";
    if (!icnv::smooth_coords_dev) return set_error(ICNV_E_UNSUPPORTED, "%s: this build has no coordinate-smoothing kernel", who);
    ICNV_HOST_PROLOGUE();
    if (!X || !Y) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    int rc = icnv::smooth_coords_check(G, C, chr_start, chr_len, K, gene_start, gene_stop, window_length, who);
    if (rc) return rc;
    double *dX = nullptr, *dY = (double *)scratch(SLOT_OUT, sizeof(double) * (size_t)(G * C));
    if (!dY) return ICNV_E_NOMEM;
    if ((rc = upload_matrix_ring(X, G * C, &dX, st))) return rc;
    if ((rc = icnv::smooth_coords_dev(dX, G, dY, G, G, C, chr_start, chr_len, K, gene_start, gene_stop, window_length, st, who)))
        return rc;
    ICNV_CUDA(cudaMemcpyAsync(Y, dY, sizeof(double) * (size_t)(G * C), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

int icnv_dev_smooth_coordinates_f64(const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t G, int64_t C,
                                    const int32_t *chr_start, const int32_t *chr_len, int K, const double *gene_start,
                                    const double *gene_stop, double window_length, void *stream) {
    static const char *who = "icnv_dev_smooth_coordinates_f64";
    if (!icnv::smooth_coords_dev) return set_error(ICNV_E_UNSUPPORTED, "%s: this build has no coordinate-smoothing kernel", who);
    ICNV_REQUIRE_READY();
    if (!X || !Y || ldx < G || ldy < G) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    int rc = icnv::smooth_coords_check(G, C, chr_start, chr_len, K, gene_start, gene_stop, window_length, who);
    if (rc) return rc;
    return icnv::smooth_coords_dev(X, ldx, Y, ldy, G, C, chr_start, chr_len, K, gene_start, gene_stop, window_length,
                                   pick_stream(stream), who);
}

}  // extern "C"

// ---- subclustering trees, K17 (kernels and device bodies in icnv_subclusters.cu) -------------------------------------------
// Weak references, as for the linkage: a build without icnv_subclusters.cu reports them as unsupported.
namespace icnv {
int zscore_outlier_dev(const double *X, int64_t G, const int32_t *d_cells, int64_t n, uint8_t *outlier, void *stream,
                       const char *who) __attribute__((weak));
int cluster_groups_check(int64_t G, const int32_t *keep, int64_t n_keep, const int32_t *grp_off, int n_grp, int method,
                         const char *who) __attribute__((weak));
int64_t cluster_groups_rows(const int32_t *grp_off, int n_grp) __attribute__((weak));
int cluster_groups_dev(const double *X, int64_t G, int64_t ldx, int64_t C, const int32_t *d_keep, int64_t n_keep,
                       const int32_t *grp_off, const int32_t *d_idx, int n_grp, int method, int32_t *merge, double *height,
                       void *stream, const char *who) __attribute__((weak));
void cluster_groups_stats(double *out5) __attribute__((weak));

}  // namespace icnv

extern "C" {

int icnv_zscore_outlier_genes_f64(const double *X, int64_t G, int64_t C, const int32_t *ref_idx, int64_t n_ref,
                                  uint8_t *outlier) {
    static const char *who = "icnv_zscore_outlier_genes_f64";
    if (!icnv::zscore_outlier_dev) return set_error(ICNV_E_UNSUPPORTED, "%s: this build has no z-score filter kernel", who);
    ICNV_HOST_PROLOGUE();
    if (!X || !ref_idx || !outlier || G <= 1 || C <= 0 || n_ref <= 0) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    for (int64_t i = 0; i < n_ref; ++i)
        if (ref_idx[i] < 0 || ref_idx[i] >= C) return set_error(ICNV_E_BAD_ARG, "%s: cell index out of range", who);
    double *dX = nullptr;
    int32_t *d_idx = nullptr;
    uint8_t *d_out = (uint8_t *)scratch(SLOT_OUT, (size_t)G);
    if (!d_out) return ICNV_E_NOMEM;
    int rc = upload_listed_columns(X, G, ref_idx, n_ref, &dX, &d_idx, st);
    if (rc) return rc;
    if ((rc = icnv::zscore_outlier_dev(dX, G, d_idx, n_ref, d_out, st, who))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(outlier, d_out, (size_t)G, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return ICNV_OK;
}

int icnv_dev_zscore_outlier_genes_f64(const double *X, int64_t G, const int32_t *d_ref_idx, int64_t n_ref, uint8_t *outlier,
                                      void *stream) {
    static const char *who = "icnv_dev_zscore_outlier_genes_f64";
    if (!icnv::zscore_outlier_dev) return set_error(ICNV_E_UNSUPPORTED, "%s: this build has no z-score filter kernel", who);
    return icnv::zscore_outlier_dev(X, G, d_ref_idx, n_ref, outlier, stream, who);
}

int icnv_cluster_groups_f64(const double *X, int64_t G, int64_t C, const int32_t *keep, int64_t n_keep, const int32_t *grp_off,
                            const int32_t *grp_idx, int n_grp, int method, int32_t *merge, double *height, int32_t *order) {
    static const char *who = "icnv_cluster_groups_f64";
    if (!icnv::cluster_groups_dev) return set_error(ICNV_E_UNSUPPORTED, "%s: this build has no group-tree kernels", who);
    int rc = icnv::cluster_groups_check(G, keep, n_keep, grp_off, n_grp, method, who);
    if (rc) return rc;
    ICNV_HOST_PROLOGUE();
    const int64_t n_list = n_grp > 0 ? grp_off[n_grp] : 0, rows = icnv::cluster_groups_rows(grp_off, n_grp);
    if (!X || C <= 0 || (n_list > 0 && (!grp_idx || !order)) || (rows > 0 && (!merge || !height)))
        return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    for (int64_t i = 0; i < n_list; ++i)
        if (grp_idx[i] < 0 || grp_idx[i] >= C) return set_error(ICNV_E_BAD_ARG, "%s: cell index out of range", who);
    for (int64_t i = 0; keep && i < n_keep; ++i)
        if (keep[i] < 0 || keep[i] >= G) return set_error(ICNV_E_BAD_ARG, "%s: gene index out of range", who);
    for (int k = 0; k < n_grp; ++k)
        if (grp_off[k + 1] - grp_off[k] == 1) order[grp_off[k]] = 1;
    if (rows == 0) return ICNV_OK;
    double *dX = nullptr;
    int32_t *d_idx = nullptr, *d_keep = nullptr;
    double *d_height = (double *)scratch(SLOT_OUT, (sizeof(double) + 2 * sizeof(int32_t)) * (size_t)rows);
    if (!d_height) return ICNV_E_NOMEM;
    int32_t *d_merge = (int32_t *)(d_height + rows);
    if ((rc = upload_listed_columns(X, G, grp_idx, n_list, &dX, &d_idx, st))) return rc;
    if (keep) {   // an empty list still means "no genes": any non-NULL device pointer stands for it
        d_keep = n_keep > 0 ? (int32_t *)scratch(SLOT_IDX2, sizeof(int32_t) * (size_t)n_keep) : d_idx;
        if (!d_keep) return ICNV_E_NOMEM;
        if (n_keep > 0) ICNV_CUDA(cudaMemcpyAsync(d_keep, keep, sizeof(int32_t) * (size_t)n_keep, cudaMemcpyHostToDevice, st));
    }
    if ((rc = icnv::cluster_groups_dev(dX, G, G, n_list, d_keep, n_keep, grp_off, d_idx, n_grp, method, d_merge, d_height, st,
                                       who)))
        return rc;
    ICNV_CUDA(cudaMemcpyAsync(merge, d_merge, sizeof(int32_t) * 2 * (size_t)rows, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaMemcpyAsync(height, d_height, sizeof(double) * (size_t)rows, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    int64_t r = 0;
    for (int k = 0; k < n_grp; ++k) {
        const int64_t n = (int64_t)grp_off[k + 1] - grp_off[k];
        if (n < 2) continue;
        if ((rc = icnv_hclust_order(merge + 2 * r, n, order + grp_off[k]))) return rc;
        r += n - 1;
    }
    return ICNV_OK;
}

int icnv_dev_cluster_groups_f64(const double *X, int64_t G, int64_t ldx, int64_t C, const int32_t *d_keep, int64_t n_keep,
                                const int32_t *grp_off, const int32_t *d_grp_idx, int n_grp, int method, int32_t *merge,
                                double *height, void *stream) {
    static const char *who = "icnv_dev_cluster_groups_f64";
    if (!icnv::cluster_groups_dev) return set_error(ICNV_E_UNSUPPORTED, "%s: this build has no group-tree kernels", who);
    return icnv::cluster_groups_dev(X, G, ldx, C, d_keep, n_keep, grp_off, d_grp_idx, n_grp, method, merge, height, stream,
                                    who);
}

int icnv_debug_cluster_groups(double *out5) {
    if (!out5) return set_error(ICNV_E_BAD_ARG, "icnv_debug_cluster_groups: out5 is NULL");
    for (int i = 0; i < 5; ++i) out5[i] = 0.0;
    if (icnv::cluster_groups_stats) icnv::cluster_groups_stats(out5);
    return ICNV_OK;
}

}  // extern "C"

// ---- hclust on the packed triangle, K19 (kernels and device bodies in icnv_hclust_tri.cu) -----------------------------------
// Weak references, as for the linkage: a build without icnv_hclust_tri.cu reports them as unsupported.
namespace icnv {
int hclust_tri_check(int64_t n, int method, const char *who) __attribute__((weak));
int hclust_tri_room(int64_t n, size_t extra, const char *who) __attribute__((weak));
int hclust_tri_host(const double *d, int64_t n, int method, int32_t *merge, double *height, int32_t *order,
                    const char *who) __attribute__((weak));
int hclust_tri_dev(const double *d_dist, int64_t n, int method, int32_t *merge, double *height, void *stream,
                   const char *who) __attribute__((weak));
int cluster_cells_dev(const double *X, int64_t G, int64_t ldx, int64_t C, const int32_t *d_keep, int64_t n_keep,
                      const int32_t *d_cells, int64_t n, int method, int32_t *merge, double *height, void *stream,
                      const char *who) __attribute__((weak));
}  // namespace icnv

extern "C" {

int icnv_hclust_tri_f64(const double *d, int64_t n, int method, int32_t *merge, double *height, int32_t *order) {
    static const char *who = "icnv_hclust_tri_f64";
    if (!icnv::hclust_tri_host) return set_error(ICNV_E_UNSUPPORTED, "%s: this build has no packed-triangle linkage", who);
    return icnv::hclust_tri_host(d, n, method, merge, height, order, who);
}

int icnv_dev_hclust_tri_f64(const double *d_dist, int64_t n, int method, int32_t *merge, double *height, void *stream) {
    static const char *who = "icnv_dev_hclust_tri_f64";
    if (!icnv::hclust_tri_dev) return set_error(ICNV_E_UNSUPPORTED, "%s: this build has no packed-triangle linkage", who);
    return icnv::hclust_tri_dev(d_dist, n, method, merge, height, stream, who);
}

int icnv_cluster_cells_f64(const double *X, int64_t G, int64_t C, const int32_t *keep, int64_t n_keep, const int32_t *cells,
                           int64_t n, int method, int32_t *merge, double *height, int32_t *order) {
    static const char *who = "icnv_cluster_cells_f64";
    if (!icnv::cluster_cells_dev) return set_error(ICNV_E_UNSUPPORTED, "%s: this build has no packed-triangle linkage", who);
    if (!cells) n = C;
    int rc = icnv::hclust_tri_check(n, method, who);
    if (rc) return rc;
    if (!X || G < 0 || C < 1 || n_keep < 0 || !merge || !height || !order || (keep && n_keep > 0 && G < 1))
        return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    for (int64_t i = 0; cells && i < n; ++i)
        if (cells[i] < 0 || cells[i] >= C) return set_error(ICNV_E_BAD_ARG, "%s: cell index out of range", who);
    for (int64_t i = 0; keep && i < n_keep; ++i)
        if (keep[i] < 0 || keep[i] >= G) return set_error(ICNV_E_BAD_ARG, "%s: gene index out of range", who);
    ICNV_HOST_PROLOGUE();
    // everything this call will hold on the device besides the triangle, before any of it is allocated
    const int64_t Gk = keep ? n_keep : G, nm = n - 1;
    const size_t x_bytes = sizeof(double) * (size_t)std::max<int64_t>(G * n, 1);
    const size_t out_bytes = (sizeof(double) + 2 * sizeof(int32_t)) * (size_t)nm;
    const size_t extra = (x_bytes > c.slot_bytes[SLOT_IN] ? x_bytes : 0) + (out_bytes > c.slot_bytes[SLOT_OUT] ? out_bytes : 0) +
                         (keep && Gk > 0 ? sizeof(double) * (size_t)Gk * (size_t)n : 0) + 256;
    if ((rc = icnv::hclust_tri_room(n, extra, who))) return rc;
    double *dX = nullptr;
    int32_t *d_idx = nullptr, *d_keep = nullptr;
    double *d_height = (double *)scratch(SLOT_OUT, out_bytes);
    if (!d_height) return ICNV_E_NOMEM;
    int32_t *d_merge = (int32_t *)(d_height + nm);
    if (cells) {
        if ((rc = upload_listed_columns(X, G, cells, n, &dX, &d_idx, st))) return rc;
    } else if ((rc = upload_matrix_ring(X, G * C, &dX, st))) {
        return rc;
    }
    if (keep) {   // an empty list still means "no genes": any non-NULL device pointer stands for it
        d_keep = n_keep > 0 ? (int32_t *)scratch(SLOT_IDX2, sizeof(int32_t) * (size_t)n_keep) : d_merge;
        if (!d_keep) return ICNV_E_NOMEM;
        if (n_keep > 0) ICNV_CUDA(cudaMemcpyAsync(d_keep, keep, sizeof(int32_t) * (size_t)n_keep, cudaMemcpyHostToDevice, st));
    }
    if ((rc = icnv::cluster_cells_dev(dX, G, G, n, d_keep, n_keep, nullptr, n, method, d_merge, d_height, st, who))) return rc;
    ICNV_CUDA(cudaMemcpyAsync(merge, d_merge, sizeof(int32_t) * 2 * (size_t)nm, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaMemcpyAsync(height, d_height, sizeof(double) * (size_t)nm, cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    return icnv_hclust_order(merge, n, order);
}

int icnv_dev_cluster_cells_f64(const double *X, int64_t G, int64_t ldx, int64_t C, const int32_t *d_keep, int64_t n_keep,
                               const int32_t *d_cells, int64_t n, int method, int32_t *merge, double *height, void *stream) {
    static const char *who = "icnv_dev_cluster_cells_f64";
    if (!icnv::cluster_cells_dev) return set_error(ICNV_E_UNSUPPORTED, "%s: this build has no packed-triangle linkage", who);
    if (!d_cells) n = C;
    return icnv::cluster_cells_dev(X, G, ldx, C, d_keep, n_keep, d_cells, n, method, merge, height, stream, who);
}

}  // extern "C"

// ---- Seurat's SNN graph, K18 (kernels and the device body in icnv_snn.cu) ---------------------------------------------------
// Weak references, as for the linkage: a build without icnv_snn.cu reports them as unsupported.
namespace icnv {
int seurat_snn_check(int64_t G, int64_t n, int n_features, int npcs, int k, const char *who) __attribute__((weak));
int seurat_snn_room(int64_t G, int64_t n, const char *who) __attribute__((weak));
int seurat_snn_dev(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n, int n_features, int npcs,
                   int k, int64_t *nnz, void *stream, const char *who) __attribute__((weak));
int seurat_snn_fetch(int64_t *row_ptr, int32_t *col, double *w, int32_t *features, double *emb, int32_t *idx,
                     cudaStream_t st, const char *who) __attribute__((weak));
void seurat_snn_stats(double *out16) __attribute__((weak));
}  // namespace icnv

extern "C" {

int icnv_seurat_snn_f64(const double *X, int64_t G, int64_t C, const int32_t *cells, int64_t n, int n_features, int npcs,
                        int k, int64_t *nnz) {
    static const char *who = "icnv_seurat_snn_f64";
    if (!icnv::seurat_snn_dev) return set_error(ICNV_E_UNSUPPORTED, "%s: this build has no SNN kernels", who);
    if (!cells) n = C;
    if (!X || C < 1 || !nnz) return set_error(ICNV_E_BAD_ARG, "%s: bad argument", who);
    for (int64_t i = 0; cells && i < n; ++i)
        if (cells[i] < 0 || cells[i] >= C) return set_error(ICNV_E_BAD_ARG, "%s: cell index out of range", who);
    int rc = icnv::seurat_snn_check(G, n, n_features, npcs, k, who);
    if (rc) return rc;
    ICNV_HOST_PROLOGUE();
    if ((rc = icnv::seurat_snn_room(G, n, who))) return rc;
    double *dX = nullptr;
    int32_t *d_idx = nullptr;
    if (cells) {
        if ((rc = upload_listed_columns(X, G, cells, n, &dX, &d_idx, st))) return rc;
    } else if ((rc = upload_matrix_ring(X, G * C, &dX, st))) {
        return rc;
    }
    return icnv::seurat_snn_dev(dX, G, G, nullptr, n, n_features, npcs, k, nnz, st, who);
}

int icnv_dev_seurat_snn_f64(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n, int n_features,
                            int npcs, int k, int64_t *nnz, void *stream) {
    static const char *who = "icnv_dev_seurat_snn_f64";
    if (!icnv::seurat_snn_dev) return set_error(ICNV_E_UNSUPPORTED, "%s: this build has no SNN kernels", who);
    return icnv::seurat_snn_dev(X, G, ldx, d_cells, n, n_features, npcs, k, nnz, stream, who);
}

int icnv_seurat_snn_fetch(int64_t *row_ptr, int32_t *col, double *w, int32_t *features, double *emb, int32_t *idx) {
    static const char *who = "icnv_seurat_snn_fetch";
    if (!icnv::seurat_snn_fetch) return set_error(ICNV_E_UNSUPPORTED, "%s: this build has no SNN kernels", who);
    ICNV_HOST_PROLOGUE();
    return icnv::seurat_snn_fetch(row_ptr, col, w, features, emb, idx, st, who);
}

int icnv_debug_seurat_snn(double *out16) {
    if (!out16) return set_error(ICNV_E_BAD_ARG, "icnv_debug_seurat_snn: out16 is NULL");
    for (int i = 0; i < 16; ++i) out16[i] = 0.0;
    if (icnv::seurat_snn_stats) icnv::seurat_snn_stats(out16);
    return ICNV_OK;
}

}  // extern "C"
