// icnv_common.cuh - context, error plumbing and small device helpers shared by the kernels of
// libinfercnv_b200.so (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/infercnv_b200.h"

namespace icnv {

// ---- per-process context -----------------------------------------------------------------------

enum ScratchSlot {
    SLOT_IN = 0,      // staged input matrix (host API)
    SLOT_OUT,         // staged output matrix (host API)
    SLOT_TMP,         // centred/smoothed reference columns (smooth block pass 1)
    SLOT_PARTIAL,     // partial sums for group means
    SLOT_MEANS,       // G x n_grp means
    SLOT_BOUNDS,      // lo1,hi1,mid1,lo2,hi2,mid2 (6 x G)
    SLOT_IDX,         // device copies of index lists
    SLOT_SEGS,        // segment table of the cell pipeline
    SLOT_BP,          // Viterbi backpointer scratch
    SLOT_STATES,      // uint8 states
    SLOT_MISC,        // flags, margins, small things
    SLOT_MISC2,
    SLOT_IDX2,
    SLOT_SYNTH,
    SLOT_MF,          // median-filter tile tables
    SLOT_TABLE,       // emission polynomial table
    SLOT_LIST,        // sequences to re-run exactly
    SLOT_LE,          // per-warp emission rows of the exact re-run
    SLOT_SLAB_IN0, SLOT_SLAB_IN1,     // double-buffered cell slabs of the pipelined host entry points
    SLOT_SLAB_OUT0, SLOT_SLAB_OUT1,
    SLOT_SLAB_ST0, SLOT_SLAB_ST1,     // uint8 states per slab
    SLOT_SLAB_W0, SLOT_SLAB_W1,       // int32 states per slab
    SLOT_REFX,                        // compact copy of the reference cells' columns
    SLOT_RG_COUNTS,                   // region calling: per (group, gene) state counts
    SLOT_RG_CONS,                     // consensus sequences (uint8, G x n_grp)
    SLOT_RG_CHUNKS,                   // cell chunks of the counting kernel
    SLOT_RG_GENE,                     // chromosome id per gene, chromosome ranges, gene start / stop
    SLOT_RG_TILES,                    // per-tile region counts and their scanned offsets
    SLOT_RG_REC,                      // region records of the last call (kept until fetched)
    SLOT_VIT_ITEMS,                   // chromosome work items of the Viterbi launch (cached: Ctx::up_items)
    SLOT_MF_PRE,                      // median filter: range of the matrix and the value sample of its pre-pass
    SLOT_KNN,                         // k nearest neighbours: per-split partial lists and the non-finite flag
    SLOT_GRP_MEANS,                   // fused group-mode HMM: G x n_hmm group means, then the per-group sds
    SLOT_GRP_PART,                    // ... chunk sums of one slab and the two sums of a group left open between slabs
    SLOT_GRP_TAB,                     // ... chunk and segment tables of every slab
    SLOT_GRP_ST,                      // ... uint8 G x n_hmm traces
    SLOT_COUNT
};

struct Ctx {
    bool ready = false;
    int device = -1;
    int sm_count = 0;
    int smem_optin = 0;      // max dynamic shared memory per block (opt-in), bytes
    cudaStream_t stream = nullptr;
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;   // copy streams of the pipelined host entry points
    cudaEvent_t ev_h2d[2] = {}, ev_comp[2] = {}, ev_d2h[2] = {};
    void *slot_ptr[SLOT_COUNT] = {};
    size_t slot_bytes[SLOT_COUNT] = {};
    std::atomic<int64_t> launches{0};
    int hmm_mode = 1;                 // 0 reference-order arithmetic, 1 certified FP64 pass (default)
    bool table_uploaded = false;
    bool math_tables_uploaded = false;
    unsigned int *hmm_list_count = nullptr;  // device counter of the last Viterbi call's re-run list
    int64_t rg_n = 0;                 // number of region records held in SLOT_RG_REC
    // what the small per-launch tables (thread segments of the cell pipeline, chromosome items of the Viterbi) held when
    // they were last uploaded: an unchanged table is not copied again, so the slab loop of the host pipeline enqueues
    // nothing from pageable host memory (such a copy may synchronise the host with the stream)
    std::vector<unsigned char> up_segs, up_items;
    cudaStream_t up_segs_stream = nullptr, up_items_stream = nullptr;   // an upload orders only the stream it was issued on
    // pinned staging ring of the host-pointer entry points (pageable caller memory, e.g. an R matrix): two slabs in, two out,
    // two for the states and two for the median-filtered chunks of the fused i3 call
    void *pin_ptr[8] = {};
    size_t pin_bytes[8] = {};
    // tuning switches, read from the environment ONCE in icnv_init (never at launch time); -1 / 0 = library default
    int opt_cell_kernel = 0, opt_cell_nt = 0, opt_cell_variant = -1, opt_cell_padq = 1, opt_cell_lfix = 1;
    long opt_slab_cells = 0;
    // the cell-pipeline instantiation the last icnv_dev_cell_pipeline_f64 call launched: family (3 / 4), NT, MINB, PADQ, LFIX,
    // slice length L; all zero when that call launched nothing (refused, or no columns)
    int cell_kernel[6] = {};
    std::mutex mu;
};

constexpr int ICNV_MAX_DEVICES = 16;
int current_slot();            // which of the library's device contexts this host thread works on
void set_current_slot(int s);
int device_slots();            // contexts initialised by icnv_init (1) or icnv_init_devices (n)
Ctx &ctx_of(int slot);

// upload `bytes` of `src` to `dst` on `st` unless `cache` says the device copy already holds them and the upload that put
// them there was ordered on the same stream
inline cudaError_t upload_if_changed(std::vector<unsigned char> &cache, cudaStream_t &last, void *dst, const void *src,
                                     size_t bytes, cudaStream_t st) {
    if (last == st && cache.size() == bytes && memcmp(cache.data(), src, bytes) == 0) return cudaSuccess;
    cache.assign(static_cast<const unsigned char *>(src), static_cast<const unsigned char *>(src) + bytes);
    last = st;
    return cudaMemcpyAsync(dst, cache.data(), bytes, cudaMemcpyHostToDevice, st);
}

// One linkage of a member-table launch (K17: trees of groups of different sizes side by side).  Its cells are the list
// entries cell_off .. cell_off + n - 1, its n x ld distance matrix starts at M + m_off (ld = n rounded up to even), its
// linkage scratch at w8 + s8_off (n + P doubles) and w4 + s4_off (6 n + P int32; P = the power of two >= n - 1), and its
// merge / height at merge + 2 out_off / height + out_off.  dist_square_kernel and hclust_nn_chain_kernel both read it.
struct HcMember {
    int64_t cell_off, n, ld, m_off, s8_off, s4_off, out_off;
    int32_t P, pad;
};

Ctx &ctx();
int set_error(int code, const char *fmt, ...);
// grow-only device scratch; returns nullptr (and sets the error) on failure
void *scratch(int slot, size_t bytes);
inline cudaStream_t pick_stream(void *s) { return s ? reinterpret_cast<cudaStream_t>(s) : ctx().stream; }
inline void count_launch(int n = 1) { ctx().launches.fetch_add(n, std::memory_order_relaxed); }

#define ICNV_REQUIRE_READY()                                                                   \
    do {                                                                                       \
        if (!icnv::ctx().ready) {                                                              \
            int rc__ = icnv_init(-1);                                                          \
            if (rc__ != ICNV_OK) return rc__;                                                  \
        }                                                                                      \
    } while (0)

#define ICNV_CUDA(call)                                                                        \
    do {                                                                                       \
        cudaError_t e__ = (call);                                                              \
        if (e__ != cudaSuccess)                                                                \
            return icnv::set_error(ICNV_E_CUDA, "%s failed at %s:%d: %s", #call, __FILE__,     \
                                   __LINE__, cudaGetErrorString(e__));                         \
    } while (0)

#define ICNV_CHECK_LAUNCH(name)                                                                \
    do {                                                                                       \
        cudaError_t e__ = cudaGetLastError();                                                  \
        if (e__ != cudaSuccess)                                                                \
            return icnv::set_error(ICNV_E_CUDA, "launch of %s failed: %s", name,               \
                                   cudaGetErrorString(e__));                                   \
        icnv::count_launch();                                                                  \
    } while (0)

// ---- device helpers ----------------------------------------------------------------------------

#ifdef __CUDACC__

__device__ __forceinline__ bool is_finite_d(double v) {
    // exponent all ones <=> inf / nan
    return ((__double2hiint(v) >> 20) & 0x7ff) != 0x7ff;
}

// order-preserving map double -> uint64 (and back), for bisection in "key space"
__device__ __forceinline__ unsigned long long key_of(double v) {
    unsigned long long u = (unsigned long long)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double double_of_key(unsigned long long k) {
    unsigned long long u = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
    return __longlong_as_double((long long)u);
}

// Counter-based splitmix64 generator: a pure function of its arguments (the synthetic workload, the permutations of the
// random-trees null).  oracle/infercnv_oracle.c (syn_hash3) and tests/runmean_reference.py restate it.
__device__ __forceinline__ uint64_t mix64(uint64_t z) {  // splitmix64 finaliser
    z += 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ uint64_t hash3(uint64_t seed, uint64_t a, uint64_t b, uint64_t c) {
    return mix64(mix64(mix64(seed ^ 0x243f6a8885a308d3ull) + a) * 0x9fb21c651e98df25ull + b) ^ mix64(c + 0x13198a2e03707344ull);
}
// a (0, 1] uniform and a Box-Muller standard normal from generator words (the synthetic workload, the Gibbs sampler)
__device__ __forceinline__ double u01(uint64_t h) {  // (0, 1]
    return ((double)(h >> 11) + 1.0) * (1.0 / 9007199254740992.0);
}
__device__ __forceinline__ double std_normal(uint64_t h1, uint64_t h2) {
    return sqrt(-2.0 * log(u01(h1))) * cospi(2.0 * u01(h2));
}
// Error-free transformations (the running mean, the DE means and variances, the coordinate smoother).
// (s + e) == a + b exactly (no branch, no assumption on magnitudes)
__device__ __forceinline__ void two_sum(double a, double b, double &s, double &e) {
    s = a + b;
    const double bp = s - a;
    e = (a - (s - bp)) + (b - bp);
}
// (hi, lo) += x
__device__ __forceinline__ void dd_add(double &hi, double &lo, double x) {
    double s, e;
    two_sum(hi, x, s, e);
    two_sum(s, lo + e, hi, lo);
}
// (hi + lo) / c, c a positive integer: the quotient of hi and its exact remainder, corrected once
__device__ __forceinline__ double dd_div(double hi, double lo, double c) {
    const double q = hi / c;
    const double r = fma(-q, c, hi);
    return q + (r + lo) / c;
}
__device__ __forceinline__ double warp_min_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

#endif  // __CUDACC__

}  // namespace icnv
