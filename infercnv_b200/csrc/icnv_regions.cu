// icnv_regions.cu - CNV region calling on the HMM state matrix (SURVEY section 8(f), rank 1): the step right
// after the Viterbi kernels on the same G x C one-byte state matrix.
//
//   .get_state_consensus        R/inferCNV_HMM.R:977-988    state_counts_kernel + consensus_from_counts_kernel
//   .define_cnv_gene_regions    R/inferCNV_HMM.R:1006-1058  region_count_kernel -> tile_scan_kernel -> region_emit_kernel
//   .get_cnv_gene_region_bounds R/inferCNV_HMM.R:1071-1087  region_finish_kernel
//
// Byte / index work, HBM-bound by construction: the consensus reads every state byte of the listed cells once
// (1 B per cell-gene, 32-bit loads of four consecutive genes, counts kept as byte-wide packed counters in registers
// and merged with integer atomics, so the result does not depend on how the cells are chunked or on the GPU
// count); region calling reads each sequence twice (count, then emit at the scanned offsets) and writes one
// 28-byte record per region in (sequence, chromosome, position) order - the order get_predicted_CNV_regions
// numbers its regions in (HMM.R:735-760), so the region counter is simply the record index + 1.
#include <algorithm>
#include <cmath>
#include <vector>

#include "icnv_common.cuh"
#include "icnv_regions_core.h"

namespace icnv {

struct RgChunk {       // entries [begin, end) of the flattened cell list, all of group `grp`
    int32_t grp, begin, end, pad;
};

constexpr int RG_CT = 128;                 // threads per CTA, counting kernel
constexpr int RG_GPT = 4;                  // genes per thread (one 32-bit load)
constexpr int RG_RT = 256;                 // threads per CTA, region kernels
constexpr int RG_TILE = RG_RT * RG_GPT;    // genes per tile of a sequence
constexpr int RG_CHUNK_CELLS = 256;        // cells per counting chunk

template <bool ALIGNED>
__device__ __forceinline__ uint32_t rg_load4(const uint8_t *__restrict__ col, int64_t g0, int64_t G) {
    if (ALIGNED && g0 + RG_GPT <= G) return *reinterpret_cast<const uint32_t *>(col + g0);
    uint32_t w = 0;
#pragma unroll
    for (int k = 0; k < RG_GPT; ++k) {
        const uint32_t b = (g0 + k < G) ? (uint32_t)col[g0 + k] : 0u;
        w |= b << (8 * k);
    }
    return w;
}

// counts[((grp - grp0) * G + g) * 8 + slot] += number of listed cells of `grp` whose state at gene g has that slot
template <bool ALIGNED>
__global__ void __launch_bounds__(RG_CT) state_counts_kernel(const uint8_t *__restrict__ S, int64_t G, int64_t lds,
                                                             const int32_t *__restrict__ cells,
                                                             const RgChunk *__restrict__ chunks, int gene_blocks, int grp0,
                                                             uint32_t *__restrict__ counts, int *__restrict__ flag) {
    const int gb = (int)(blockIdx.x % (unsigned)gene_blocks);
    const RgChunk ch = chunks[blockIdx.x / (unsigned)gene_blocks];
    const int64_t g0 = ((int64_t)gb * RG_CT + threadIdx.x) * RG_GPT;
    if (g0 >= G) return;
    uint32_t tot[RG_GPT][RG_SLOTS];
#pragma unroll
    for (int k = 0; k < RG_GPT; ++k)
#pragma unroll
        for (int s = 0; s < RG_SLOTS; ++s) tot[k][s] = 0u;
    uint64_t acc[RG_GPT] = {0ull, 0ull, 0ull, 0ull};
    bool bad = false;
    int pending = 0;
    auto flush = [&]() {     // byte-wide counters: emptied into the 32-bit totals before they can wrap
#pragma unroll
        for (int k = 0; k < RG_GPT; ++k) {
#pragma unroll
            for (int s = 0; s < RG_SLOTS; ++s) tot[k][s] += rg_packed_get(acc[k], s);
            acc[k] = 0ull;
        }
        pending = 0;
    };
    // eight listed cells per round: their (index, state word) loads are issued back to back before any of them is
    // used - one cell at a time the loop is a chain of two dependent loads per 4 bytes.  Past the chunk's end the last
    // cell is re-read and not counted.
    constexpr int RG_BATCH = 8;
    const bool whole_word = ALIGNED && g0 + RG_GPT <= G;
    for (int i = ch.begin; i < ch.end; i += RG_BATCH) {
        uint32_t w[RG_BATCH];
        int32_t cidx[RG_BATCH];
#pragma unroll
        for (int u = 0; u < RG_BATCH; ++u) cidx[u] = cells[min(i + u, ch.end - 1)];
        if (whole_word) {   // the usual case: eight independent 32-bit loads, nothing between them
#pragma unroll
            for (int u = 0; u < RG_BATCH; ++u) w[u] = *reinterpret_cast<const uint32_t *>(S + (int64_t)cidx[u] * lds + g0);
        } else {            // last genes of the matrix or an unaligned layout: byte loads
#pragma unroll
            for (int u = 0; u < RG_BATCH; ++u) w[u] = rg_load4<false>(S + (int64_t)cidx[u] * lds, g0, G);
        }
        if (pending + RG_BATCH > 255) flush();
#pragma unroll
        for (int u = 0; u < RG_BATCH; ++u) {
            if (i + u < ch.end) {
#pragma unroll
                for (int k = 0; k < RG_GPT; ++k) {
                    const int s = rg_slot((w[u] >> (8 * k)) & 0xffu);
                    bad |= (s < 0) && (g0 + k < G);
                    acc[k] += rg_packed_one(s < 0 ? 0 : s);
                }
                ++pending;
            }
        }
    }
    flush();
    uint32_t *out = counts + ((int64_t)(ch.grp - grp0) * G + g0) * RG_SLOTS;
#pragma unroll
    for (int k = 0; k < RG_GPT; ++k) {
        if (g0 + k < G) {
#pragma unroll
            for (int s = 0; s < RG_SLOTS; ++s)
                if (tot[k][s]) atomicAdd(out + k * RG_SLOTS + s, tot[k][s]);
        }
    }
    if (bad) atomicOr(flag, 4);
}

// cons[i] = modal state of counts[i*8 .. i*8+8), ties to the smallest state; i = gene + G * group
__global__ void __launch_bounds__(256) consensus_from_counts_kernel(const uint32_t *__restrict__ counts, int64_t n,
                                                                    uint8_t *__restrict__ cons) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const uint4 a = reinterpret_cast<const uint4 *>(counts)[2 * i];
    const uint4 b = reinterpret_cast<const uint4 *>(counts)[2 * i + 1];
    const uint32_t c[RG_SLOTS] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    cons[i] = rg_state_of_slot(rg_argmax_first(c));
}

struct RgParams {
    const uint8_t *seqs;      // sequence s = column (cols ? cols[s] : s), lds bytes apart
    int64_t G, lds;
    const int32_t *cols;
    const int32_t *chr_of;    // chromosome id per gene, -1 for chromosomes with < 2 genes (HMM.R:1012-1014)
    int tiles_per_seq;
};

// region-start flags of this thread's four genes in tile `tile` (bit k = gene g0 + k), plus what the emit pass needs
template <bool ALIGNED>
__device__ __forceinline__ unsigned rg_thread_flags(const RgParams &p, unsigned tile, int64_t &g0, uint32_t &w) {
    const int64_t s = tile / (unsigned)p.tiles_per_seq;
    const int t = (int)(tile % (unsigned)p.tiles_per_seq);
    const uint8_t *col = p.seqs + (p.cols ? (int64_t)p.cols[s] : s) * p.lds;
    g0 = ((int64_t)t * RG_RT + threadIdx.x) * RG_GPT;
    w = 0u;
    if (g0 >= p.G) return 0u;
    w = rg_load4<ALIGNED>(col, g0, p.G);
    unsigned s_prev = g0 > 0 ? (unsigned)col[g0 - 1] : 0u;
    int chr_prev = g0 > 0 ? p.chr_of[g0 - 1] : -1;
    unsigned flags = 0u;
#pragma unroll
    for (int k = 0; k < RG_GPT; ++k) {
        if (g0 + k < p.G) {
            const unsigned v = (w >> (8 * k)) & 0xffu;
            const int c = p.chr_of[g0 + k];
            if (rg_opens_region(g0 + k, chr_prev, c, s_prev, v)) flags |= 1u << k;
            s_prev = v;
            chr_prev = c;
        }
    }
    return flags;
}

template <bool ALIGNED>
__global__ void __launch_bounds__(RG_RT) region_count_kernel(RgParams p, uint32_t *__restrict__ tile_counts) {
    __shared__ int wsum[RG_RT / 32];
    int64_t g0;
    uint32_t w;
    int n = __popc(rg_thread_flags<ALIGNED>(p, blockIdx.x, g0, w));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int i = 0; i < RG_RT / 32; ++i) t += wsum[i];
        tile_counts[blockIdx.x] = (uint32_t)t;
    }
}

// exclusive scan of n tile counts into offsets[0..n] (offsets[n] = total); one CTA, contiguous slice per thread
__global__ void __launch_bounds__(1024) tile_scan_kernel(const uint32_t *__restrict__ counts, int64_t n,
                                                         int64_t *__restrict__ offsets) {
    __shared__ int64_t part[1024];
    const int64_t per = (n + 1023) / 1024;
    const int64_t b = min(n, (int64_t)threadIdx.x * per);
    const int64_t e = min(n, b + per);
    int64_t s = 0;
    for (int64_t i = b; i < e; ++i) s += counts[i];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {
        const int64_t v = (int)threadIdx.x >= off ? part[threadIdx.x - off] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    int64_t run = part[threadIdx.x] - s;
    for (int64_t i = b; i < e; ++i) {
        offsets[i] = run;
        run += counts[i];
    }
    if (threadIdx.x == 1023) offsets[n] = part[1023];
}

template <bool ALIGNED>
__global__ void __launch_bounds__(RG_RT) region_emit_kernel(RgParams p, const int64_t *__restrict__ tile_off,
                                                            int32_t *__restrict__ r_seq, int32_t *__restrict__ r_chr,
                                                            int32_t *__restrict__ r_first, int32_t *__restrict__ r_state) {
    __shared__ int wsum[RG_RT / 32];
    int64_t g0;
    uint32_t w;
    const unsigned f = rg_thread_flags<ALIGNED>(p, blockIdx.x, g0, w);
    const int n = __popc(f);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    int base = 0;
    for (int i = 0; i < warp; ++i) base += wsum[i];
    if (f) {
        int64_t pos = tile_off[blockIdx.x] + base + incl - n;
        const int32_t s = (int32_t)(blockIdx.x / (unsigned)p.tiles_per_seq);
#pragma unroll
        for (int k = 0; k < RG_GPT; ++k) {
            if ((f >> k) & 1u) {
                const unsigned v = (w >> (8 * k)) & 0xffu;
                r_seq[pos] = s;
                r_chr[pos] = p.chr_of[g0 + k];
                r_first[pos] = (int32_t)(g0 + k);
                r_state[pos] = v == RG_UNASSIGNED ? -1 : (int32_t)v;
                ++pos;
            }
        }
    }
}

// one warp per region: last gene (the gene before the next region of the same sequence and chromosome, else the
// chromosome's last gene), min(start), max(stop) over the region's genes
__global__ void __launch_bounds__(256) region_finish_kernel(int64_t n, const int32_t *__restrict__ r_seq,
                                                            const int32_t *__restrict__ r_chr,
                                                            const int32_t *__restrict__ r_first,
                                                            const int32_t *__restrict__ chr_start,
                                                            const int32_t *__restrict__ chr_len,
                                                            const double *__restrict__ gene_start,
                                                            const double *__restrict__ gene_stop,
                                                            int32_t *__restrict__ r_last, double *__restrict__ r_start,
                                                            double *__restrict__ r_end) {
    const int64_t r = ((int64_t)blockIdx.x * 256 + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n) return;     // warp-uniform
    const int first = r_first[r], c = r_chr[r];
    int last = chr_start[c] + chr_len[c] - 1;
    if (r + 1 < n && r_seq[r + 1] == r_seq[r] && r_chr[r + 1] == c) last = r_first[r + 1] - 1;
    double lo = INFINITY, hi = -INFINITY;
    for (int g = first + lane; g <= last; g += 32) {
        lo = fmin(lo, gene_start[g]);
        hi = fmax(hi, gene_stop[g]);
    }
    lo = warp_min_d(lo);
    hi = warp_max_d(hi);
    if (lane == 0) {
        r_last[r] = last;
        r_start[r] = lo;
        r_end[r] = hi;
    }
}

// predict_CNV_via_HMM_on_tumor_subclusters_per_chr (HMM.R:412-487): every chromosome has its own partition of the
// cells.  gs holds one state sequence per (chromosome, group) column; cell c takes, on the genes of chromosome k,
// the sequence of its group on that chromosome: out[g, c] = gs[g, grp_of[chr(g) * C + c]], 255 (R's -1) if it has none.
__global__ void __launch_bounds__(256) scatter_states_per_chr_kernel(const uint8_t *__restrict__ gs, int64_t G, int64_t C,
                                                                     const int32_t *__restrict__ chr_id,
                                                                     const int32_t *__restrict__ grp_of,
                                                                     uint8_t *__restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < G * C; i += stride) {
        const int64_t c = i / G, g = i - c * G;
        const int grp = grp_of[(int64_t)chr_id[g] * C + c];
        out[i] = grp < 0 ? (uint8_t)RG_UNASSIGNED : gs[g + G * grp];
    }
}

// the consensus step that ends that driver (HMM.R:472-483): every cell of a group takes the group's consensus state
// on the genes region calling covers (chromosomes with >= 2 genes, chr_of >= 0); everything else keeps its state
__global__ void __launch_bounds__(256) apply_consensus_kernel(const uint8_t *__restrict__ S, const uint8_t *__restrict__ cons,
                                                              int64_t G, int64_t C, const int32_t *__restrict__ chr_of,
                                                              const int32_t *__restrict__ grp_of,
                                                              uint8_t *__restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < G * C; i += stride) {
        const int64_t c = i / G, g = i - c * G;
        const int grp = grp_of[c];
        out[i] = (grp >= 0 && chr_of[g] >= 0) ? cons[g + G * grp] : S[i];
    }
}

static inline int64_t round_up4(int64_t n) { return (n + 3) & ~(int64_t)3; }

// record arrays inside SLOT_RG_REC for n regions
struct RgRecords {
    int32_t *seq, *chr, *first, *last, *state;
    double *start, *end;
};
static RgRecords records_at(void *base, int64_t n) {
    const int64_t n4 = std::max<int64_t>(4, round_up4(n));
    RgRecords r;
    r.seq = (int32_t *)base;
    r.chr = r.seq + n4;
    r.first = r.chr + n4;
    r.last = r.first + n4;
    r.state = r.last + n4;
    r.start = (double *)(r.state + n4);   // 20 * n4 bytes in: a multiple of 16
    r.end = r.start + n4;
    return r;
}
static size_t records_bytes(int64_t n) { return (size_t)std::max<int64_t>(4, round_up4(n)) * 36; }

}  // namespace icnv

using namespace icnv;

extern "C" {

/* counts (uint32, n_grp x G x 8, zeroed here) of the listed cells' states; see include/infercnv_b200.h */
int icnv_dev_state_counts_u8(const uint8_t *S, int64_t G, int64_t lds, const int32_t *d_cells, const int32_t *h_grp_off,
                             int n_grp, uint32_t *d_counts, int *d_flag, void *stream) {
    cudaStream_t st = pick_stream(stream);
    if (!S || !d_cells || !h_grp_off || !d_counts || !d_flag || G <= 0 || lds < G || n_grp <= 0)
        return set_error(ICNV_E_BAD_ARG, "icnv_dev_state_counts_u8: bad argument");
    std::vector<RgChunk> chunks;
    for (int k = 0; k < n_grp; ++k)
        for (int32_t b = h_grp_off[k]; b < h_grp_off[k + 1]; b += RG_CHUNK_CELLS)
            chunks.push_back(RgChunk{k, b, std::min<int32_t>(b + RG_CHUNK_CELLS, h_grp_off[k + 1]), 0});
    ICNV_CUDA(cudaMemsetAsync(d_counts, 0, sizeof(uint32_t) * (size_t)n_grp * (size_t)G * RG_SLOTS, st));
    if (chunks.empty()) return ICNV_OK;
    RgChunk *d_chunks = (RgChunk *)scratch(SLOT_RG_CHUNKS, sizeof(RgChunk) * chunks.size());
    if (!d_chunks) return ICNV_E_NOMEM;
    ICNV_CUDA(cudaMemcpyAsync(d_chunks, chunks.data(), sizeof(RgChunk) * chunks.size(), cudaMemcpyHostToDevice, st));
    const int gene_blocks = (int)((G + RG_CT * RG_GPT - 1) / (RG_CT * RG_GPT));
    const int64_t grid = (int64_t)gene_blocks * (int64_t)chunks.size();
    if (grid > 0x7fffffffLL) return set_error(ICNV_E_UNSUPPORTED, "icnv_dev_state_counts_u8: too many cell chunks");
    const bool aligned = (lds % 4 == 0) && (((uintptr_t)S) % 4 == 0);
    if (aligned)
        state_counts_kernel<true><<<(unsigned)grid, RG_CT, 0, st>>>(S, G, lds, d_cells, d_chunks, gene_blocks, 0, d_counts, d_flag);
    else
        state_counts_kernel<false><<<(unsigned)grid, RG_CT, 0, st>>>(S, G, lds, d_cells, d_chunks, gene_blocks, 0, d_counts, d_flag);
    ICNV_CHECK_LAUNCH("state_counts_kernel");
    ICNV_CUDA(cudaStreamSynchronize(st));   // `chunks` is a stack-lifetime host buffer
    return ICNV_OK;
}

int icnv_dev_consensus_from_counts(const uint32_t *d_counts, int64_t G, int n_grp, uint8_t *d_cons, void *stream) {
    cudaStream_t st = pick_stream(stream);
    if (!d_counts || !d_cons || G <= 0 || n_grp <= 0)
        return set_error(ICNV_E_BAD_ARG, "icnv_dev_consensus_from_counts: bad argument");
    const int64_t n = G * (int64_t)n_grp;
    consensus_from_counts_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_counts, n, d_cons);
    ICNV_CHECK_LAUNCH("consensus_from_counts_kernel");
    return ICNV_OK;
}

/* .get_state_consensus for n_grp index lists over a device-resident state matrix; groups are processed in batches so
 * the count buffer stays below 512 MB */
int icnv_dev_state_consensus_u8(const uint8_t *S, int64_t G, int64_t lds, const int32_t *d_cells, const int32_t *h_grp_off,
                                int n_grp, uint8_t *d_cons, int *d_flag, void *stream) {
    if (n_grp <= 0 || G <= 0) return set_error(ICNV_E_BAD_ARG, "icnv_dev_state_consensus_u8: bad argument");
    const int64_t per_grp = G * RG_SLOTS * (int64_t)sizeof(uint32_t);
    const int batch = (int)std::max<int64_t>(1, std::min<int64_t>(n_grp, (512LL << 20) / per_grp));
    uint32_t *d_counts = (uint32_t *)scratch(SLOT_RG_COUNTS, (size_t)per_grp * (size_t)batch);
    if (!d_counts) return ICNV_E_NOMEM;
    std::vector<int32_t> off((size_t)batch + 1);
    for (int g0 = 0; g0 < n_grp; g0 += batch) {
        const int nb = std::min(batch, n_grp - g0);
        // the kernel indexes the cell list by absolute position, so the batch keeps the global offsets
        for (int k = 0; k <= nb; ++k) off[k] = h_grp_off[g0 + k];
        int rc = icnv_dev_state_counts_u8(S, G, lds, d_cells, off.data(), nb, d_counts, d_flag, stream);
        if (rc) return rc;
        if ((rc = icnv_dev_consensus_from_counts(d_counts, G, nb, d_cons + (int64_t)g0 * G, stream))) return rc;
    }
    return ICNV_OK;
}

/* .define_cnv_gene_regions + .get_cnv_gene_region_bounds for n_seq device-resident sequences (columns of d_seqs, or
 * the columns d_cols[] of it).  Synchronises `stream`; the records stay in the library until icnv_cnv_regions_fetch. */
int icnv_dev_cnv_regions_u8(const uint8_t *d_seqs, int64_t G, int64_t lds, int64_t n_seq, const int32_t *d_cols,
                            const int32_t *chr_start, const int32_t *chr_len, int K, const double *gene_start,
                            const double *gene_stop, int64_t *n_regions, void *stream) {
    Ctx &c = ctx();
    cudaStream_t st = pick_stream(stream);
    if (!d_seqs || G <= 0 || lds < G || n_seq < 0 || !chr_start || !chr_len || K <= 0 || !gene_start || !gene_stop || !n_regions)
        return set_error(ICNV_E_BAD_ARG, "icnv_dev_cnv_regions_u8: bad argument");
    c.rg_n = 0;
    *n_regions = 0;
    if (n_seq == 0) return ICNV_OK;
    // gene tables: chr_of[G] | chr_start[K] | chr_len[K] (int32), then gene_start[G] | gene_stop[G] (double)
    const size_t n_i32 = (size_t)round_up4(G + 2 * (int64_t)K);
    const size_t bytes = n_i32 * 4 + (size_t)G * 16;
    char *d_tab = (char *)scratch(SLOT_RG_GENE, bytes);
    if (!d_tab) return ICNV_E_NOMEM;
    std::vector<int32_t> tab(n_i32, 0);
    for (int k = 0; k < K; ++k) {
        for (int32_t g = chr_start[k]; g < chr_start[k] + chr_len[k]; ++g) tab[(size_t)g] = chr_len[k] >= 2 ? k : -1;
        tab[(size_t)G + k] = chr_start[k];
        tab[(size_t)G + K + k] = chr_len[k];
    }
    int32_t *d_chr_of = (int32_t *)d_tab;
    double *d_gs = (double *)(d_tab + n_i32 * 4), *d_ge = d_gs + G;
    ICNV_CUDA(cudaMemcpyAsync(d_chr_of, tab.data(), n_i32 * 4, cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaMemcpyAsync(d_gs, gene_start, sizeof(double) * (size_t)G, cudaMemcpyHostToDevice, st));
    ICNV_CUDA(cudaMemcpyAsync(d_ge, gene_stop, sizeof(double) * (size_t)G, cudaMemcpyHostToDevice, st));

    RgParams p;
    p.seqs = d_seqs;
    p.G = G;
    p.lds = lds;
    p.cols = d_cols;
    p.chr_of = d_chr_of;
    p.tiles_per_seq = (int)((G + RG_TILE - 1) / RG_TILE);
    const int64_t n_tiles = n_seq * (int64_t)p.tiles_per_seq;
    if (n_tiles > 0x7fffffffLL) return set_error(ICNV_E_UNSUPPORTED, "icnv_dev_cnv_regions_u8: too many sequences");
    // tile counts (uint32, padded to 8 bytes) then offsets (int64, n_tiles + 1)
    const size_t cnt_bytes = (size_t)((n_tiles + 1) & ~(int64_t)1) * 4;
    char *d_tiles = (char *)scratch(SLOT_RG_TILES, cnt_bytes + (size_t)(n_tiles + 1) * 8);
    if (!d_tiles) return ICNV_E_NOMEM;
    uint32_t *d_cnt = (uint32_t *)d_tiles;
    int64_t *d_off = (int64_t *)(d_tiles + cnt_bytes);
    const bool aligned = (lds % 4 == 0) && (((uintptr_t)d_seqs) % 4 == 0);
    if (aligned)
        region_count_kernel<true><<<(unsigned)n_tiles, RG_RT, 0, st>>>(p, d_cnt);
    else
        region_count_kernel<false><<<(unsigned)n_tiles, RG_RT, 0, st>>>(p, d_cnt);
    ICNV_CHECK_LAUNCH("region_count_kernel");
    tile_scan_kernel<<<1, 1024, 0, st>>>(d_cnt, n_tiles, d_off);
    ICNV_CHECK_LAUNCH("tile_scan_kernel");
    int64_t n = 0;
    ICNV_CUDA(cudaMemcpyAsync(&n, d_off + n_tiles, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    ICNV_CUDA(cudaStreamSynchronize(st));
    if (n < 0 || n > n_seq * G) return set_error(ICNV_E_CUDA, "icnv_dev_cnv_regions_u8: inconsistent region count");
    void *d_rec = scratch(SLOT_RG_REC, records_bytes(n));
    if (!d_rec) return ICNV_E_NOMEM;
    if (n > 0) {
        RgRecords r = records_at(d_rec, n);
        if (aligned)
            region_emit_kernel<true><<<(unsigned)n_tiles, RG_RT, 0, st>>>(p, d_off, r.seq, r.chr, r.first, r.state);
        else
            region_emit_kernel<false><<<(unsigned)n_tiles, RG_RT, 0, st>>>(p, d_off, r.seq, r.chr, r.first, r.state);
        ICNV_CHECK_LAUNCH("region_emit_kernel");
        region_finish_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(n, r.seq, r.chr, r.first, d_chr_of + G, d_chr_of + G + K,
                                                                     d_gs, d_ge, r.last, r.start, r.end);
        ICNV_CHECK_LAUNCH("region_finish_kernel");
    }
    ICNV_CUDA(cudaStreamSynchronize(st));
    c.rg_n = n;
    *n_regions = n;
    return ICNV_OK;
}

int icnv_dev_scatter_states_per_chr_u8(const uint8_t *gs, int64_t G, int64_t C, const int32_t *d_chr_id, const int32_t *d_grp_of,
                                       uint8_t *out, void *stream) {
    ICNV_REQUIRE_READY();
    if (!gs || !d_chr_id || !d_grp_of || !out || G <= 0 || C <= 0)
        return set_error(ICNV_E_BAD_ARG, "icnv_dev_scatter_states_per_chr_u8: bad argument");
    const int64_t blocks = std::min<int64_t>((G * C + 255) / 256, (int64_t)ctx().sm_count * 32);
    scatter_states_per_chr_kernel<<<(unsigned)blocks, 256, 0, pick_stream(stream)>>>(gs, G, C, d_chr_id, d_grp_of, out);
    ICNV_CHECK_LAUNCH("scatter_states_per_chr_kernel");
    return ICNV_OK;
}

int icnv_dev_apply_consensus_u8(const uint8_t *S, const uint8_t *cons, int64_t G, int64_t C, const int32_t *d_chr_of,
                                const int32_t *d_grp_of, uint8_t *out, void *stream) {
    ICNV_REQUIRE_READY();
    if (!S || !cons || !d_chr_of || !d_grp_of || !out || G <= 0 || C <= 0)
        return set_error(ICNV_E_BAD_ARG, "icnv_dev_apply_consensus_u8: bad argument");
    const int64_t blocks = std::min<int64_t>((G * C + 255) / 256, (int64_t)ctx().sm_count * 32);
    apply_consensus_kernel<<<(unsigned)blocks, 256, 0, pick_stream(stream)>>>(S, cons, G, C, d_chr_of, d_grp_of, out);
    ICNV_CHECK_LAUNCH("apply_consensus_kernel");
    return ICNV_OK;
}

/* device pointers of the records of the last region call (valid until the next one); any output may be NULL */
int icnv_dev_cnv_regions_records(int64_t *n, const int32_t **seq, const int32_t **chr, const int32_t **first_gene,
                                 const int32_t **last_gene, const int32_t **state, const double **start,
                                 const double **end) {
    Ctx &c = ctx();
    if (!c.slot_ptr[SLOT_RG_REC]) return set_error(ICNV_E_BAD_ARG, "no region call has been made");
    RgRecords r = records_at(c.slot_ptr[SLOT_RG_REC], c.rg_n);
    if (n) *n = c.rg_n;
    if (seq) *seq = r.seq;
    if (chr) *chr = r.chr;
    if (first_gene) *first_gene = r.first;
    if (last_gene) *last_gene = r.last;
    if (state) *state = r.state;
    if (start) *start = r.start;
    if (end) *end = r.end;
    return ICNV_OK;
}

}  // extern "C"
