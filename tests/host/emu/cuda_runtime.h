// cuda_runtime.h - TEST INFRASTRUCTURE: a host emulation of the CUDA execution model, just large enough to run the
// byte / index kernels of libinfercnv_b200 (icnv_regions.cu, icnv_ingest.cu, icnv_reduce.cu) and the host entry points
// of icnv_api.cu on a machine without a GPU, from the SAME source text.  It shadows <cuda_runtime.h> on the include
// path of tests/host/build_emu.py only; nothing in the package refers to it and the library it produces is never
// loaded by infercnv_b200/ (the product has no CPU path - see tests/test_capi_symbols.py).
//
// Model: a launch runs its blocks one after another on the calling thread; the threads of a block are fibers
// (ucontext) scheduled round-robin, each running until it finishes or reaches a synchronisation point:
//   __syncthreads()            - released when every live thread of the block waits there
//   __shfl_*_sync / __reduce_* - released when every live lane of the warp waits at a warp collective
// A block in which some live threads wait at the block barrier and others (of a not yet complete warp) at a warp
// collective for ever is reported as a divergence error and aborts: the emulation doubles as a barrier-divergence check.
// Atomics are plain operations (one OS thread).  "Device memory" is host memory; streams and events are no-ops.
#pragma once

#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>
#include <execinfo.h>
#include <signal.h>
#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <functional>
#include <type_traits>
#include <vector>

// ---- language extensions ------------------------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__ __attribute__((noinline))
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))
#define __constant__

struct uint3 { unsigned x = 0, y = 0, z = 0; };
struct dim3 {
    unsigned x = 1, y = 1, z = 1;
    dim3() {}
    dim3(unsigned x_, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct uint4 { unsigned x, y, z, w; };
struct int2 { int x, y; };
struct double2 { double x, y; };
struct alignas(16) float4 { float x, y, z, w; };
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline int2 make_int2(int x, int y) { return int2{x, y}; }
static inline double2 make_double2(double x, double y) { return double2{x, y}; }

inline uint3 threadIdx, blockIdx;
inline dim3 blockDim, gridDim;

template <class A, class B> constexpr std::common_type_t<A, B> min(A a, B b) { return b < a ? (std::common_type_t<A, B>)b : (std::common_type_t<A, B>)a; }
template <class A, class B> constexpr std::common_type_t<A, B> max(A a, B b) { return a < b ? (std::common_type_t<A, B>)b : (std::common_type_t<A, B>)a; }

struct int4 {
    int x, y, z, w;
};
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
static inline unsigned __double2uint_rd(double v) { return v > 0.0 ? (v >= 4294967295.0 ? 4294967295u : (unsigned)v) : 0u; }

// ---- runtime API --------------------------------------------------------------------------------------------------
typedef int cudaError_t;
typedef struct emuStream *cudaStream_t;
typedef struct emuEvent *cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorNoDevice = 100 };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2 };
struct cudaDeviceProp {
    int major, minor, multiProcessorCount;
    size_t sharedMemPerBlockOptin;
};

static inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) {
    p->major = 9; p->minor = 0; p->multiProcessorCount = 4; p->sharedMemPerBlockOptin = 227 * 1024;
    return cudaSuccess;
}
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = (cudaStream_t)malloc(8); return cudaSuccess; }
static inline cudaError_t cudaStreamCreate(cudaStream_t *s) { return cudaStreamCreateWithFlags(s, 0); }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { *e = (cudaEvent_t)malloc(8); return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
static inline cudaError_t cudaMalloc(void **p, size_t n) {
    // poison fresh "device" memory so a kernel that reads what it never wrote is noticed
    *p = malloc(n);
    if (!*p) return cudaErrorMemoryAllocation;
    memset(*p, 0xA5, n);
    return cudaSuccess;
}
template <class T> static inline cudaError_t cudaMalloc(T **p, size_t n) { return cudaMalloc((void **)p, n); }
static inline cudaError_t cudaFree(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) {
    if (n) memmove(d, s, n);
    return cudaSuccess;
}
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = nullptr) {
    if (n) memset(d, v, n);
    return cudaSuccess;
}
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) {
    if (n) memmove(d, s, n);
    return cudaSuccess;
}
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
// page-locked host memory: plain allocations; every caller pointer reports as pageable, so the host pipeline's staging
// ring (pageable caller memory -> pinned slab -> device) is the path the emulated tests take
enum { cudaHostAllocPortable = 1 };
enum cudaMemoryType { cudaMemoryTypeUnregistered = 0, cudaMemoryTypeHost = 1, cudaMemoryTypeDevice = 2, cudaMemoryTypeManaged = 3 };
struct cudaPointerAttributes {
    cudaMemoryType type;
};
static inline cudaError_t cudaHostAlloc(void **p, size_t n, unsigned) {
    *p = malloc(n);
    if (!*p) return cudaErrorMemoryAllocation;
    memset(*p, 0xA5, n);
    return cudaSuccess;
}
static inline cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaPointerGetAttributes(cudaPointerAttributes *a, const void *) { a->type = cudaMemoryTypeUnregistered; return cudaSuccess; }
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
template <class K> static inline cudaError_t cudaFuncSetAttribute(K, cudaFuncAttribute, int) { return cudaSuccess; }
template <class K> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *n, K, int, size_t) { *n = 1; return cudaSuccess; }
template <class T> static inline cudaError_t cudaMemcpyToSymbol(T &sym, const void *src, size_t n, size_t off = 0, cudaMemcpyKind = cudaMemcpyHostToDevice) {
    memcpy((char *)&sym + off, src, n);
    return cudaSuccess;
}
template <class T> static inline cudaError_t cudaMemcpyFromSymbol(void *dst, const T &sym, size_t n, size_t off = 0, cudaMemcpyKind = cudaMemcpyDeviceToHost) {
    memcpy(dst, (const char *)&sym + off, n);
    return cudaSuccess;
}
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline const char *cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated CUDA error"; }

// ---- execution model ----------------------------------------------------------------------------------------------
namespace emu {

enum State { RUN = 0, WAIT_BLOCK, WAIT_WARP, DONE };
struct Fiber {
    ucontext_t ctx;
    State state = DONE;
    unsigned gen = 0;          // number of warp collectives this thread has entered
    bool spun = false;         // came back from a spin-wait iteration (made no progress of its own)
};
constexpr size_t STACK_BYTES = 64 * 1024;
constexpr int MAX_THREADS = 1024;

inline std::vector<Fiber> fibers;
inline std::vector<char> stacks;
inline ucontext_t sched_ctx;
inline Fiber *cur = nullptr;
inline const std::function<void()> *body = nullptr;
inline uint64_t warp_slot[2][MAX_THREADS / 32][32];
inline unsigned warp_posted[2][MAX_THREADS / 32][32];   // collective number (gen + 1) the slot was written for
constexpr size_t DYN_SMEM_MAX = 227 * 1024;
alignas(128) inline unsigned char dyn_smem[DYN_SMEM_MAX];
inline size_t dyn_smem_bytes = 0;
inline unsigned long long launches = 0, blocks_run = 0;
inline int order_mode = -1;                 // 0 forward, 1 reverse, 2 random
inline unsigned long long order_rng = 1;
inline void read_order_mode() {
    if (order_mode >= 0) return;
    const char *e = getenv("EMU_ORDER");
    order_mode = 0;
    if (e && !strncmp(e, "reverse", 7)) order_mode = 1;
    if (e && !strncmp(e, "random", 6)) {
        order_mode = 2;
        order_rng = e[6] == ':' ? strtoull(e + 7, nullptr, 10) * 2 + 1 : 12345;
    }
}

inline void yield_to_scheduler() { swapcontext(&cur->ctx, &sched_ctx); }
// one iteration of a spin-wait on memory another thread (or an asynchronous copy) will write: stay runnable, let the
// others run.  A block in which every runnable thread only spins, pass after pass, is reported as a dead-lock.
inline void spin_yield() {
    cur->spun = true;
    yield_to_scheduler();
}
// The rules of cp.async.bulk and of the mbarrier's transaction count, for the synchronous stand-ins of
// tests/host/build_emu.py: source and destination 16-byte aligned, a size that is a non-zero multiple of 16, and a phase
// completed only when the bytes announced by expect_tx (kept in the word behind the phase word) have all arrived.  On the
// GPU a short count leaves the barrier waiting forever and an excess completes the phase early; here both abort.
inline void bulk_copy_check(const void *dst, const void *src, unsigned bytes) {
    if (((uintptr_t)dst & 15u) || ((uintptr_t)src & 15u) || (bytes & 15u) || bytes == 0) {
        fprintf(stderr, "emu: cp.async.bulk of %u bytes from %p to %p breaks the 16-byte alignment / size rule\n", bytes, src, dst);
        abort();
    }
}
inline void tx_complete_check(const unsigned long long *bar) {
    if (bar[1] != 0ull) {
        fprintf(stderr, "emu: mbarrier phase completed with %lld transaction bytes not matched by copies\n", (long long)bar[1]);
        abort();
    }
}
inline void trampoline() {
    (*body)();
    cur->state = DONE;
    swapcontext(&cur->ctx, &sched_ctx);
}

inline void run_block(unsigned nt, const std::function<void()> &fn) {
    if (nt == 0 || nt > MAX_THREADS || (nt & 31)) {
        fprintf(stderr, "emu: block size %u not supported (multiple of 32, <= 1024)\n", nt);
        abort();
    }
    body = &fn;
    if (fibers.size() < nt) fibers.resize(nt);
    if (stacks.size() < (size_t)nt * STACK_BYTES) stacks.resize((size_t)nt * STACK_BYTES);
    for (unsigned t = 0; t < nt; ++t) {
        Fiber &f = fibers[t];
        getcontext(&f.ctx);
        f.ctx.uc_stack.ss_sp = stacks.data() + (size_t)t * STACK_BYTES;
        f.ctx.uc_stack.ss_size = STACK_BYTES;
        f.ctx.uc_link = &sched_ctx;
        makecontext(&f.ctx, trampoline, 0);
        f.state = RUN;
        f.gen = 0;
    }
    memset(warp_posted, 0, sizeof(warp_posted));
    if (dyn_smem_bytes) memset(dyn_smem, 0xA5, dyn_smem_bytes);     // shared memory starts undefined in every block
    unsigned alive = nt;
    unsigned long long passes = 0, idle_passes = 0;
    while (alive > 0) {
        if (++passes == 200000000ull) {     // no kernel of this library synchronises this often: a live-lock
            unsigned st[4] = {0, 0, 0, 0};
            for (unsigned t = 0; t < nt; ++t) st[fibers[t].state]++;
            fprintf(stderr, "emu: block (%u,%u) still running after 2e8 scheduler passes (run %u, block-wait %u, warp-wait %u, done %u)\n",
                    blockIdx.x, blockIdx.y, st[0], st[1], st[2], st[3]);
            abort();
        }
        bool ran = false, progress = false;
        // EMU_ORDER: the order in which the runnable threads of a block are resumed within a scheduler pass -
        // "forward" (default), "reverse", or "random[:seed]" (a fresh odd-stride permutation every pass).  A kernel
        // whose results depend on it has a data race (a missing barrier, an unsynchronised hand-off).
        unsigned start = 0, step = 1;
        if (order_mode == 1) { start = nt - 1; step = nt - 1; }
        else if (order_mode == 2) {
            order_rng = order_rng * 6364136223846793005ull + 1442695040888963407ull;
            start = (unsigned)(order_rng >> 33) % nt;
            step = ((unsigned)(order_rng >> 13) % nt) | 1u;          // odd stride: a permutation for power-of-two-multiple sizes
            if (std::__gcd(step, nt) != 1) step = 1;
        }
        for (unsigned i = 0, t = start; i < nt; ++i, t = (t + step) % nt) {
            Fiber &f = fibers[t];
            if (f.state != RUN) continue;
            cur = &f;
            threadIdx.x = t;
            f.spun = false;
            swapcontext(&sched_ctx, &f.ctx);
            ran = true;
            progress |= !f.spun;
            if (f.state == DONE) --alive;
        }
        if (alive == 0) break;
        bool released = false;
        for (unsigned w = 0; w < nt / 32; ++w) {      // warp collectives first
            unsigned live = 0, waiting = 0;
            for (unsigned l = 0; l < 32; ++l) {
                const State s = fibers[w * 32 + l].state;
                live += s != DONE;
                waiting += s == WAIT_WARP;
            }
            if (live && waiting == live) {
                for (unsigned l = 0; l < 32; ++l)
                    if (fibers[w * 32 + l].state == WAIT_WARP) fibers[w * 32 + l].state = RUN;
                released = true;
            }
        }
        if (!released) {
            unsigned waiting = 0;
            for (unsigned t = 0; t < nt; ++t) waiting += fibers[t].state == WAIT_BLOCK;
            if (waiting == alive) {
                for (unsigned t = 0; t < nt; ++t)
                    if (fibers[t].state == WAIT_BLOCK) fibers[t].state = RUN;
                released = true;
            }
        }
        idle_passes = (progress || released) ? 0 : idle_passes + 1;
        if (idle_passes > 1000000) {
            fprintf(stderr, "emu: block (%u,%u): every runnable thread spins on a condition nobody satisfies\n", blockIdx.x, blockIdx.y);
            abort();
        }
        if (!released && !ran) {
            fprintf(stderr, "emu: divergent synchronisation in block (%u,%u): the live threads wait at different barriers\n",
                    blockIdx.x, blockIdx.y);
            abort();
        }
    }
    ++blocks_run;
}

struct Cfg {
    dim3 grid, block;
    size_t smem;
    Cfg(dim3 g, dim3 b, size_t s = 0, cudaStream_t = nullptr) : grid(g), block(b), smem(s) {}
};

// EMU_WATCHDOG=<seconds>: print a native backtrace of wherever the emulation is when the alarm fires, then abort
inline void watchdog_handler(int) {
    void *frames[64];
    const int n = backtrace(frames, 64);
    const char msg[] = "emu: watchdog fired; native backtrace:\n";
    (void)!write(2, msg, sizeof(msg) - 1);
    backtrace_symbols_fd(frames, n, 2);
    _exit(99);
}
inline void arm_watchdog() {
    static bool armed = false;
    const char *e = getenv("EMU_WATCHDOG");      // also turns an abort() anywhere into a native backtrace
    if (armed || !e) return;
    armed = true;
    signal(SIGABRT, watchdog_handler);
    signal(SIGALRM, watchdog_handler);
    alarm((unsigned)atoi(e));
}

inline void launch(const Cfg &cfg, const std::function<void()> &fn) {
    arm_watchdog();
    read_order_mode();
    if (cfg.block.y != 1 || cfg.block.z != 1 || cfg.grid.z != 1) {
        fprintf(stderr, "emu: only (x, y) grids of 1-D blocks are supported\n");
        abort();
    }
    if (cfg.smem > DYN_SMEM_MAX) {
        fprintf(stderr, "emu: %zu bytes of dynamic shared memory exceed the 227 KB of a CTA\n", cfg.smem);
        abort();
    }
    gridDim = cfg.grid;
    blockDim = cfg.block;
    dyn_smem_bytes = cfg.smem;
    ++launches;
    // canary behind the dynamic shared memory the launch asked for: a store past the end (a size formula in a launcher that
    // forgot a table) is caught here; a load past the end reads the canary and shows up as a parity failure
    const size_t guard = DYN_SMEM_MAX - cfg.smem < 4096 ? DYN_SMEM_MAX - cfg.smem : 4096;
    for (unsigned by = 0; by < cfg.grid.y; ++by)
        for (unsigned bx = 0; bx < cfg.grid.x; ++bx) {
            blockIdx.x = bx;
            blockIdx.y = by;
            memset(dyn_smem + cfg.smem, 0x5C, guard);
            run_block(cfg.block.x, fn);
            for (size_t i = 0; i < guard; ++i)
                if (dyn_smem[cfg.smem + i] != 0x5C) {
                    fprintf(stderr, "emu: block (%u,%u) wrote %zu bytes past its %zu bytes of dynamic shared memory\n", bx, by,
                            i + 1, cfg.smem);
                    abort();
                }
        }
}

template <class T>
inline T warp_exchange(T v, int src_lane) {
    static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
    Fiber *f = cur;
    const unsigned tid = threadIdx.x, w = tid >> 5, lane = tid & 31, n = ++f->gen, g = n & 1u;
    uint64_t bits = 0;
    memcpy(&bits, &v, sizeof(T));
    warp_slot[g][w][lane] = bits;
    warp_posted[g][w][lane] = n;
    f->state = WAIT_WARP;
    yield_to_scheduler();
    // a lane that left the kernel before this collective never posted: the result is undefined on the GPU, own value here
    if (src_lane < 0 || src_lane > 31 || warp_posted[g][w][src_lane] != n) return v;
    T out;
    memcpy(&out, &warp_slot[g][w][src_lane], sizeof(T));
    return out;
}

}  // namespace emu

#define EMU_LAUNCH(kernel, cfg, args) emu::launch(emu::Cfg cfg, [&]() { kernel args; })

static inline void __syncthreads() {
    emu::cur->state = emu::WAIT_BLOCK;
    emu::yield_to_scheduler();
}
static inline void __syncwarp(unsigned = 0xffffffffu) { (void)emu::warp_exchange<int>(0, 0); }
template <class T> static inline T __shfl_sync(unsigned, T v, int src) { return emu::warp_exchange(v, src & 31); }
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int m) { return emu::warp_exchange(v, (int)((threadIdx.x & 31) ^ (unsigned)m)); }
template <class T> static inline T __shfl_up_sync(unsigned, T v, unsigned d) {
    const int lane = (int)(threadIdx.x & 31);
    return emu::warp_exchange(v, lane >= (int)d ? lane - (int)d : lane);
}
template <class T> static inline T __shfl_down_sync(unsigned, T v, unsigned d) {
    const int lane = (int)(threadIdx.x & 31);
    return emu::warp_exchange(v, lane + (int)d <= 31 ? lane + (int)d : lane);
}

namespace emu {
// every live lane posts a value; after the release each lane folds the posted values of the live lanes
template <class T, class F>
inline T warp_fold(T v, F f) {
    Fiber *fb = cur;
    const unsigned tid = threadIdx.x, w = tid >> 5, lane = tid & 31, n = ++fb->gen, g = n & 1u;
    uint64_t bits = 0;
    memcpy(&bits, &v, sizeof(T));
    warp_slot[g][w][lane] = bits;
    warp_posted[g][w][lane] = n;
    fb->state = WAIT_WARP;
    yield_to_scheduler();
    T acc = v;
    for (unsigned l = 0; l < 32; ++l) {
        if (l == lane || warp_posted[g][w][l] != n) continue;     // lanes that have left the kernel do not take part
        T o;
        memcpy(&o, &warp_slot[g][w][l], sizeof(T));
        acc = f(acc, o);
    }
    return acc;
}
}  // namespace emu
static inline int __reduce_add_sync(unsigned, int v) { return emu::warp_fold(v, [](int a, int b) { return a + b; }); }
static inline unsigned __reduce_add_sync(unsigned, unsigned v) { return emu::warp_fold(v, [](unsigned a, unsigned b) { return a + b; }); }
static inline unsigned __reduce_or_sync(unsigned, unsigned v) { return emu::warp_fold(v, [](unsigned a, unsigned b) { return a | b; }); }
static inline int __reduce_max_sync(unsigned, int v) { return emu::warp_fold(v, [](int a, int b) { return a > b ? a : b; }); }
static inline int __reduce_min_sync(unsigned, int v) { return emu::warp_fold(v, [](int a, int b) { return a < b ? a : b; }); }
static inline unsigned __ballot_sync(unsigned, int pred) {
    return emu::warp_fold(pred ? 1u << (threadIdx.x & 31) : 0u, [](unsigned a, unsigned b) { return a | b; });
}

// ---- intrinsics ---------------------------------------------------------------------------------------------------
// IEEE operations that must not be contracted into an FMA: out of line, so the host compiler cannot fuse them either
__attribute__((noinline)) static double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }
__attribute__((noinline)) static double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }
__attribute__((noinline)) static double __ddiv_rn(double a, double b) { volatile double r = a / b; return r; }
static inline float __frcp_rn(float a) { return 1.0f / a; }
static inline double cospi(double x) { return cos(M_PI * x); }
static inline double sinpi(double x) { return sin(M_PI * x); }
static inline double rsqrt(double x) { return 1.0 / sqrt(x); }
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
static inline double __hiloint2double(int hi, int lo) {
    const uint64_t u = ((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo;
    double v;
    memcpy(&v, &u, 8);
    return v;
}
static inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
static inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned sh) {
    sh &= 31;
    return sh ? (hi << sh) | (lo >> (32 - sh)) : hi;
}
static inline size_t __cvta_generic_to_shared(const void *p) { return (size_t)p; }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __double2hiint(double v) { uint64_t u; memcpy(&u, &v, 8); return (int)(u >> 32); }
static inline int __double2loint(double v) { uint64_t u; memcpy(&u, &v, 8); return (int)(u & 0xffffffffu); }
static inline long long __double_as_longlong(double v) { long long u; memcpy(&u, &v, 8); return u; }
static inline double __longlong_as_double(long long u) { double v; memcpy(&v, &u, 8); return v; }

static inline double atomicAdd(double *p, double v) { const double o = *p; *p = o + v; return o; }
static inline unsigned atomicAdd(unsigned *p, unsigned v) { const unsigned o = *p; *p = o + v; return o; }
static inline int atomicAdd(int *p, int v) { const int o = *p; *p = o + v; return o; }
static inline unsigned long long atomicAdd(unsigned long long *p, unsigned long long v) { const unsigned long long o = *p; *p = o + v; return o; }
static inline unsigned long long atomicMin(unsigned long long *p, unsigned long long v) { const unsigned long long o = *p; if (v < o) *p = v; return o; }
static inline unsigned long long atomicMax(unsigned long long *p, unsigned long long v) { const unsigned long long o = *p; if (v > o) *p = v; return o; }
static inline unsigned atomicOr(unsigned *p, unsigned v) { const unsigned o = *p; *p = o | v; return o; }
static inline unsigned atomicExch(unsigned *p, unsigned v) { const unsigned o = *p; *p = v; return o; }
static inline unsigned long long atomicExch(unsigned long long *p, unsigned long long v) { const unsigned long long o = *p; *p = v; return o; }
static inline int atomicOr(int *p, int v) { const int o = *p; *p = o | v; return o; }
static inline int atomicExch(int *p, int v) { const int o = *p; *p = v; return o; }
