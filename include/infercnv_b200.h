/*
 * infercnv_b200.h - C ABI of libinfercnv_b200.so: the H100 (sm_90a) drop-in for the
 * smoothing + HMM hot path of broadinstitute/infercnv.
 *
 * The reference is pure R (DESCRIPTION: "NeedsCompilation: no"; NAMESPACE has no useDynLib), so it
 * has no native interface to bind to.  The boundary is the set of internal R functions that
 * infercnv::run() calls on this path; each entry point below replaces the body of one of them
 * (file:line of the reference given per function) and is what a `.Call()` shim binds
 * (see INTEGRATION.md and infercnv_b200/r/).
 *
 * Conventions
 *   layout   R column-major, X[g + G*c]: g = gene (row, chromosome-ordered), c = cell (column).
 *            A cell's gene vector is contiguous.  Sizes are int64 (R long vectors).
 *   dtype    float64 across the ABI (R `double`); states are int32 (1..m, -1 = not assigned), or one byte each
 *            (1..m, 255 = not assigned) from the *_u8 variants - a quarter of the bytes over PCIe.
 *   indices  0-based everywhere (the R shim subtracts 1).  Index lists are CSR style:
 *            group k owns grp_idx[grp_off[k] .. grp_off[k+1]).
 *   chromosomes  K contiguous row ranges [chr_start[k], chr_start[k]+chr_len[k]) - the reference
 *            pre-sorts rows by chr,start,stop (R/inferCNV.R:407-413).
 *   ownership  caller owns every buffer it passes; inputs are never modified; outputs may alias
 *            inputs only where stated.  The library owns all device memory, streams and a pinned
 *            staging ring (two slabs in, two out per GPU): caller memory that is not page-locked -
 *            an R matrix, a NumPy array - is moved through that ring by the library's copy threads,
 *            page-locked caller memory is used directly.  Everything is freed in icnv_shutdown().
 *   errors   every entry returns 0 or a negative icnv_status and records a per-thread message
 *            readable through icnv_last_error().  Nothing throws across the ABI.  There is no CPU
 *            fallback: without a usable CUDA device every compute entry returns ICNV_E_NO_DEVICE.
 *   threading  calls are synchronous (result resident in the caller's buffer at return) and
 *            serialised internally; call from one host thread at a time per process.
 *
 * Two families:
 *   icnv_*      host pointers in / host pointers out (what R binds).  H2D / D2H inside.
 *   icnv_dev_*  device pointers on the library's current device + a cudaStream_t (as void*);
 *               asynchronous on that stream.  Used by the multi-GPU driver and the benchmark.
 */
#ifndef INFERCNV_B200_H
#define INFERCNV_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define ICNV_API __attribute__((visibility("default")))
#else
#define ICNV_API
#endif

typedef enum icnv_status {
    ICNV_OK = 0,
    ICNV_E_NO_DEVICE = -1,   /* no CUDA device / driver, or icnv_init failed */
    ICNV_E_CUDA = -2,        /* a CUDA runtime call or kernel failed */
    ICNV_E_BAD_ARG = -3,     /* NULL pointer, negative size, inconsistent ranges, even window, ... */
    ICNV_E_UNSUPPORTED = -4, /* outside the kernels' envelope (e.g. G too large for shared memory) */
    ICNV_E_NONFINITE = -5,   /* NA/NaN/Inf in the input where the reference would stop() */
    ICNV_E_UNDERFLOW = -6,   /* "Problems With Underflow" (R/inferCNV_HMM.R:1165-1166) */
    ICNV_E_NOMEM = -7
} icnv_status;

/* ---- lifecycle ------------------------------------------------------------------------------ */

/* Select `device` (cudaSetDevice), create the library's stream and scratch pools.  Idempotent for
 * the same device; re-initialises when called with another one.  device < 0 -> keep the current
 * set-up, or device 0 when there is none.  Tuning switches (ICNV_* environment variables, DESIGN.md
 * section 8) are read here, once, and the ones that are set are reported on stderr. */
ICNV_API int icnv_init(int device);
/* Multi-GPU for a single host process - the form the R shim uses (infercnv::run() is one R process;
 * its num_threads, R/inferCNV_ops.R:388, never reaches this path): initialise n_devices GPUs
 * (device_ids == NULL: devices 0 .. n-1; n_devices <= 0: every device present).  Afterwards the
 * host-pointer entry points that stream cells (icnv_smooth_block_f64, icnv_smooth_hmm_*_f64, the
 * per-cell icnv_viterbi_*_f64) cut the cells into one contiguous range per GPU, driven by one host
 * thread each; every GPU reduces ALL reference cells itself in list order (they are <= ~10 % of the
 * matrix and cross PCIe once per GPU), so no inter-GPU exchange is needed and the result is bit-identical
 * for any device count (SURVEY section 8e, "broadcast the ref-cell columns").  All other entry points use
 * the first device.  icnv_dev_* calls address the device of the calling thread's context (the first). */
ICNV_API int icnv_init_devices(int n_devices, const int *device_ids);
ICNV_API int icnv_devices_in_use(void);        /* 0 before initialisation */
/* Host threads that move the caller's (pageable) matrix into / out of the pinned staging ring; they are
 * split over the GPUs in use.  0 = default: half the hardware threads, at most 16. */
ICNV_API int icnv_set_host_threads(int n);
ICNV_API void icnv_shutdown(void);
ICNV_API int icnv_device_count(void);          /* >= 0, or a negative icnv_status */
ICNV_API const char *icnv_last_error(void);    /* never NULL */
ICNV_API const char *icnv_version(void);
/* Number of kernel launches issued by this library since icnv_init (for bench `gpu_launches`). */
ICNV_API int64_t icnv_launch_count(void);

/* HMM arithmetic.  mode 0: reference-order IEEE arithmetic for every sequence.  mode 1 (default): certified FP64 pass -
 * table emission + structured recursion, every arg-max margin checked, and each sequence whose smallest margin is below
 * 1e-7 recomputed in mode-0 arithmetic.  The state calls are the same in both modes.  Any other mode is refused with
 * ICNV_E_BAD_ARG.  Also settable with the environment variable ICNV_HMM_MODE (read at icnv_init: "0" or "e..." selects
 * mode 0, anything else mode 1). */
ICNV_API int icnv_set_hmm_mode(int mode);
/* Number of sequences the last Viterbi call recomputed in reference-order arithmetic (syncs). */
ICNV_API int64_t icnv_hmm_rerun_count(void);
/* Always 0: no HMM mode hands sequences to a second pass.  Kept so that existing callers still link. */
ICNV_API int64_t icnv_hmm_second_pass_count(void);

/* ---- host-pointer entry points (what the R shim binds) ---------------------------------------- */

/* .get_normal_gene_mean_bounds, R/inferCNV_ops.R:1708-1735.
 * means[g + G*k] = mean(X[g, group k]);  inv_log != 0: log2(mean(2^x - 1) + 1). */
ICNV_API int icnv_ref_means_f64(const double *X, int64_t G, int64_t C, const int32_t *grp_off,
                                const int32_t *grp_idx, int n_grp, int inv_log, double *means);

/* .subtract_expr, R/inferCNV_ops.R:1742-1786 (body of subtract_ref_expr_from_obs, :1678-1702).
 * use_bounds: y = x-max_k(means) if x>max; x-min_k(means) if x<min; else 0.  Otherwise x-mean_k(means).
 * Y may alias X. */
ICNV_API int icnv_subtract_ref_f64(const double *X, double *Y, int64_t G, int64_t C, const double *means,
                                   int n_grp, int use_bounds);

/* smooth_by_chromosome -> .smooth_window -> .smooth_helper, R/inferCNV_ops.R:2406-2532, 2640-2661.
 * Truncated, renormalised triangular ("pyramidinal") moving average per cell per chromosome.
 * window < 2: copy.  Even window: ICNV_E_BAD_ARG (the reference's behaviour is accidental there).
 * Chromosomes with < 2 genes are left untouched (:2417).  NA input: ICNV_E_NONFINITE. */
ICNV_API int icnv_smooth_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *chr_start,
                             const int32_t *chr_len, int K, int window);

/* .center_columns, R/inferCNV_ops.R:2094-2109 (center_cell_expr_across_chromosome, :2074-2088).
 * use_median != 0: subtract the per-cell median over all G genes; else the per-cell mean. */
ICNV_API int icnv_center_f64(const double *X, double *Y, int64_t G, int64_t C, int use_median);

/* The two steps either side of the path (SURVEY section 8f), so the reference's bundled example runs
 * count.data -> expr.data on the GPU end to end:
 * normalize_counts_by_seq_depth (R/inferCNV_ops.R:3064-3111; normalize_factor < 0 or NaN = median of colSums) and
 * clear_noise_via_ref_mean_sd (R/inferCNV_ops.R:2302-2346, noise_logistic = FALSE). */
ICNV_API int icnv_normalize_counts_by_seq_depth_f64(const double *X, double *Y, int64_t G, int64_t C,
                                                    double normalize_factor);
ICNV_API int icnv_clear_noise_via_ref_mean_sd_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *idx,
                                                  int64_t n_idx, double sd_amplifier);

/* remove_outliers_norm / .remove_outliers_norm, R/inferCNV_ops.R:1969-2056 (run() step 16): clamp to
 * [lower_bound, upper_bound].  A NaN bound (R's NA) selects out_method "average_bound" (.get_average_bounds,
 * ops.R:2734-2742): lower = mean over cells of each cell's smallest value, upper = mean of each cell's largest.
 * bounds_out: optional double[2] receiving the bounds used. */
ICNV_API int icnv_remove_outliers_norm_f64(const double *X, double *Y, int64_t G, int64_t C, double lower_bound,
                                           double upper_bound, double *bounds_out);

/* clear_noise / .clear_noise, R/inferCNV_ops.R:2232-2275 (run() step 22 with a numeric noise_filter): centre = mean
 * over all values of the listed cells (n_idx == 0: all data); values strictly inside centre +- threshold become
 * centre, or - noise_logistic != 0 - are pulled towards it by depress_log_signal_midpt_val (slope 20,
 * R/inferCNV_heatmap.R:2783-2810).  threshold == 0: unchanged copy. */
ICNV_API int icnv_clear_noise_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *idx, int64_t n_idx,
                                  double threshold, int noise_logistic);

/* clear_noise_via_ref_mean_sd(noise_logistic = TRUE), R/inferCNV_ops.R:2325-2329. */
ICNV_API int icnv_clear_noise_via_ref_mean_sd_logistic_f64(const double *X, double *Y, int64_t G, int64_t C,
                                                           const int32_t *idx, int64_t n_idx, double sd_amplifier);

/* Element-wise steps as stand-alone calls (inside icnv_smooth_block_f64 they are fused into the loads
 * and stores): log2xplus1 (R/inferCNV_ops.R:2756-2769), invert_log2 (:2814-2826),
 * apply_max_threshold_bounds (:2970-2983).  n = G*C elements, Y may alias X. */
ICNV_API int icnv_log2xplus1_f64(const double *X, double *Y, int64_t n);
ICNV_API int icnv_invert_log2_f64(const double *X, double *Y, int64_t n);
ICNV_API int icnv_apply_max_threshold_bounds_f64(const double *X, double *Y, int64_t n, double threshold);

/* Fused run() steps 4, 8, 9, 10, 11, 12, 14 (R/inferCNV_ops.R:614, 771, 817, 865, 911, 952, 1031):
 * [log2(x+1)] -> subtract ref (bounds) -> clamp +-threshold -> smooth(window) -> centre by
 * median -> subtract ref again -> 2^x.  X is the depth-normalised matrix (after step 3).
 * n_grp == 0 is BAD_ARG (callers pass the proxy group of all observation cells when there are no
 * references, as the reference does at ops.R:1686-1689).  threshold <= 0 disables the clamp. */
ICNV_API int icnv_smooth_block_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *chr_start,
                                   const int32_t *chr_len, int K, const int32_t *grp_off, const int32_t *grp_idx,
                                   int n_grp, int apply_log, double threshold, int window, int use_bounds);

/* Fused icnv_smooth_block_f64 + per-cell icnv_viterbi_f64 in ONE pass over the matrix: run() steps
 * 4..14 followed by step 17 for analysis_mode = "cells" (R/inferCNV_ops.R:614-1031, :1235-1309); with
 * the default prune_outliers = FALSE nothing between those steps touches expr.data.  Y receives the
 * smoothed matrix (what run() keeps as the preliminary object), states the HMM calls on it. */
ICNV_API int icnv_smooth_hmm_f64(const double *X, double *Y, int32_t *states, int64_t G, int64_t C,
                                 const int32_t *chr_start, const int32_t *chr_len, int K, const int32_t *grp_off,
                                 const int32_t *grp_idx, int n_grp, int apply_log, double threshold, int window,
                                 int use_bounds, int m, const double *Pi, const double *delta, const double *mean,
                                 const double *sd);
/* same, states as one byte each (1..m): the host-pointer calls are PCIe-bound, and int32 states are a third of
 * the bytes this call returns.  This is the variant the R shim binds (it widens to R doubles either way). */
ICNV_API int icnv_smooth_hmm_u8_f64(const double *X, double *Y, uint8_t *states, int64_t G, int64_t C,
                                    const int32_t *chr_start, const int32_t *chr_len, int K, const int32_t *grp_off,
                                    const int32_t *grp_idx, int n_grp, int apply_log, double threshold, int window,
                                    int use_bounds, int m, const double *Pi, const double *delta, const double *mean,
                                    const double *sd);

/* The i3 counterpart, with the median filter on the same pass: run() steps 4..14, the i3 model, step 17 per cell and
 * apply_median_filtering, for HMM_type = "i3", analysis_mode = "cells", use_KS = FALSE.  The matrix is read once and
 * every output written once.
 *   Y       = icnv_smooth_block_f64 with the same arguments (bit-identical).
 *   model   = {mu, sigma, mean_delta}: mu and sigma over every value of the reference cells in Y
 *             (.i3HMM_get_sd_trend_by_num_cells_fit, R/inferCNV_i3HMM.R:17-80; bit-identical to icnv_mean_sd_f64(Y,
 *             grp_idx)), mean_delta = |qnorm(i3_p_val, 0, sigma)| (Wichura's AS241, as R's qnorm).  They are fixed
 *             from the reference cells before the first observation cell is processed.
 *   states  = per-cell icnv_viterbi_u8_f64 of Y under .i3HMM_get_HMM (i3HMM.R:99-156): transition diagonal 1 - 5t,
 *             off-diagonal t, delta (t, 1 - 5t, t), means (mu - d, mu, mu + d), sd sigma.
 *   F       = icnv_median_filter_f64(Y, mf lists, mf_window) (noise_reduction.R:43-113; cells in no list are copied,
 *             so n_mf == 0 gives F = Y); F == NULL: no filter, mf_* and mf_window are not read.  The cells are cut
 *             into runs no list's span crosses; one run's Y and F (2 x 8 x G bytes per cell of it) stay on the device
 *             at a time, and a run that does not fit is ICNV_E_NOMEM before any output is written.  The two buffers
 *             stay allocated at the largest run's size until icnv_shutdown / icnv_init, like the library's other
 *             scratch: lists whose spans overlap across a large group make that run, and the buffers, large.  Lists
 *             may be arbitrary column sets.
 * Several devices (icnv_init_devices): the cells are cut at the run boundaries nearest to even shares; every device
 * allocates its buffers before any device starts, so the ICNV_E_NOMEM above still leaves every output unwritten;
 * every device reduces all reference cells itself, so every output is independent of the device count.
 * BAD_ARG: an even window, an even mf_window or mf_window < 3 (with F), an index out of range, i3_p_val outside
 * (0, 1), G < 2. */
ICNV_API int icnv_smooth_i3_hmm_u8_f64(const double *X, double *Y, uint8_t *states, double *F, int64_t G, int64_t C,
                                       const int32_t *chr_start, const int32_t *chr_len, int K, const int32_t *grp_off,
                                       const int32_t *grp_idx, int n_grp, int apply_log, double threshold, int window,
                                       int use_bounds, double i3_p_val, double t, const int32_t *mf_off,
                                       const int32_t *mf_idx, int n_mf, int mf_window, double *model);

/* Group-mode twins of the two fused calls: run() steps 4..14 and step 17 for analysis_mode = "samples" and "subclusters"
 * (tumor_subcluster_partition_method = "random_trees", whose partition is made before the block), prune_outliers = FALSE.
 * The HMM runs on the group means of Y over the lists hmm_off / hmm_idx (CSR, n_hmm groups), as icnv_viterbi_u8_f64
 * with those lists does.
 *   Y       = icnv_smooth_block_f64 with the same arguments (bit-identical).
 *   states  = icnv_viterbi_u8_f64(Y, hmm lists, m, Pi, delta, mean, sd) (bit-identical): sd[m * n_hmm] holds every
 *             group's state sds and each group's trace uses their median.  A cell in no list gets 255; a cell in several
 *             lists gets the trace of the last one (R's <<- overwrite does the same).
 *   i3:       model = {mu, sigma, mean_delta} exactly as icnv_smooth_i3_hmm_u8_f64 returns it; states = the same group
 *             Viterbi under .i3HMM_get_HMM(model) with sd sigma for every group.  No median filter: callers run
 *             icnv_median_filter_f64 on Y.
 * The cells stream through the device in list order (every list entry, then the cells in no list), so a group's means are
 * summed in dev_group_means' fixed 32-entry chunks; the device holds the slabs, G x n_hmm means and traces, and the sums of
 * the group open at a slab boundary - never the matrix.  Page-locked X and Y are copied one run of consecutive columns at a
 * time; pageable ones are gathered into and scattered from the pinned ring by the copy threads.
 * Several devices (icnv_init_devices): the list order is cut at the group boundaries nearest to even shares, each group's
 * means and trace are computed on one device, and every device reduces all reference cells itself, so every output is
 * independent of the device count and of ICNV_SLAB_CELLS.
 * BAD_ARG (nothing written): n_hmm == 0 (the per-cell calls cover it), an empty group, an index out of range, a
 * non-positive median sd; for i3 also an even window, i3_p_val outside (0, 1), G < 2.  Buffers that do not fit are
 * ICNV_E_NOMEM before any output is written, on every device. */
ICNV_API int icnv_smooth_hmm_groups_u8_f64(const double *X, double *Y, uint8_t *states, int64_t G, int64_t C,
                                           const int32_t *chr_start, const int32_t *chr_len, int K, const int32_t *grp_off,
                                           const int32_t *grp_idx, int n_grp, int apply_log, double threshold, int window,
                                           int use_bounds, const int32_t *hmm_off, const int32_t *hmm_idx, int n_hmm, int m,
                                           const double *Pi, const double *delta, const double *mean, const double *sd);
ICNV_API int icnv_smooth_i3_hmm_groups_u8_f64(const double *X, double *Y, uint8_t *states, int64_t G, int64_t C,
                                              const int32_t *chr_start, const int32_t *chr_len, int K,
                                              const int32_t *grp_off, const int32_t *grp_idx, int n_grp, int apply_log,
                                              double threshold, int window, int use_bounds, const int32_t *hmm_off,
                                              const int32_t *hmm_idx, int n_hmm, double i3_p_val, double t,
                                              double *model);

/* Viterbi.dthmm.adj, R/inferCNV_HMM.R:1101-1176, batched over the drivers
 * predict_CNV_via_HMM_on_indiv_cells (HMM.R:284-324), ..._on_tumor_subclusters (:345-408),
 * ..._on_whole_tumor_samples (:509-567) and the i3 twins (R/inferCNV_i3HMM.R:180-389).
 * m = 6 (i6) or 3 (i3).  Pi: m x m column-major, Pi[j + m*k] = P(j -> k); delta[m]; mean[m].
 * n_grp == 0: one sequence per (cell, chromosome), sd[m].
 * n_grp  > 0: one sequence per (group, chromosome) on rowMeans(X[chr, group]); sd[m*n_grp]
 *             (per-group sds as .get_state_emission_params, HMM.R:586-614, computes them);
 *             the trace is written to every cell of the group, other cells get -1.
 * states: int32 G x C.  margins: optional (may be NULL) K x (C or n_grp) doubles receiving, per
 * sequence, the smallest winner/runner-up gap over the traceback decisions (diagnostic).
 * Sequences with < 2 genes get state 3 (HMM.R:1104-1107). */
ICNV_API int icnv_viterbi_f64(const double *X, int64_t G, int64_t C, const int32_t *chr_start,
                              const int32_t *chr_len, int K, const int32_t *grp_off, const int32_t *grp_idx,
                              int n_grp, int m, const double *Pi, const double *delta, const double *mean,
                              const double *sd, int32_t *states, double *margins);
/* same, states as uint8 G x C (1..m, 255 where the int32 variant writes -1) */
ICNV_API int icnv_viterbi_u8_f64(const double *X, int64_t G, int64_t C, const int32_t *chr_start,
                                 const int32_t *chr_len, int K, const int32_t *grp_off, const int32_t *grp_idx,
                                 int n_grp, int m, const double *Pi, const double *delta, const double *mean,
                                 const double *sd, uint8_t *states, double *margins);

/* assign_HMM_states_to_proxy_expr_vals, R/inferCNV_HMM.R:1191-1206 (m = 6: states 1..6 -> 0, 0.5, 1, 1.5, 2, 3) and
 * i3HMM_assign_HMM_states_to_proxy_expr_vals, R/inferCNV_i3HMM.R:405-417 (m = 3: 1..3 -> 0.5, 1, 1.5) on the numeric
 * state matrix (n entries); any other value (e.g. -1) passes through.  Y may alias X. */
ICNV_API int icnv_assign_hmm_states_to_proxy_expr_vals_f64(const double *X, double *Y, int64_t n, int m);

/* predict_CNV_via_HMM_on_tumor_subclusters_per_chr, R/inferCNV_HMM.R:412-471: every chromosome k has its own list of
 * subclusters - groups chr_grp_off[k] .. chr_grp_off[k+1]) of the CSR lists (grp_off, grp_idx); one Viterbi sequence
 * per (chromosome, subcluster) on rowMeans(X[chr, cells]) with that group's sds (sd: m per group, the median is used,
 * HMM.R:1122); the trace is written to the subcluster's cells on that chromosome's genes, cells in no subcluster of a
 * chromosome get 255 (R's -1, HMM.R:436) there.  A cell in two subclusters of one chromosome: ICNV_E_BAD_ARG. */
ICNV_API int icnv_viterbi_per_chr_u8_f64(const double *X, int64_t G, int64_t C, const int32_t *chr_start,
                                         const int32_t *chr_len, int K, const int32_t *chr_grp_off,
                                         const int32_t *grp_off, const int32_t *grp_idx, int m, const double *Pi,
                                         const double *delta, const double *mean, const double *sd, uint8_t *states);

/* apply_median_filtering / .median_filter, R/noise_reduction.R:43-113.  Blocks = chromosome x one
 * index list (a subcluster for observations, a whole group for references), cells in list order.
 * Window radius is (window_size+1)/2 as in the reference (noise_reduction.R:102-106).
 * Cells in no list are copied.  window_size even or < 3: ICNV_E_BAD_ARG. */
ICNV_API int icnv_median_filter_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *chr_start,
                                    const int32_t *chr_len, int K, const int32_t *grp_off, const int32_t *grp_idx,
                                    int n_grp, int window_size);

/* .i3HMM_get_sd_trend_by_num_cells_fit, R/inferCNV_i3HMM.R:17-30: mean and sd (n-1) over all
 * values of the listed cells. */
ICNV_API int icnv_mean_sd_f64(const double *X, int64_t G, int64_t C, const int32_t *idx, int64_t n_idx, double *mu,
                              double *sigma);

/* parallelDist(t(expr.data[, cells])) with its default method "euclidean" - the distance matrix behind every hclust() of
 * the reference: R/inferCNV_tumor_subclusters.R:191,411,472,582,609, R/inferCNV_ops.R:1930,3242,
 * R/inferCNV_heatmap.R:719,755,1062,1079 (SURVEY section 8(f) row 4).  cells: n 0-based columns (NULL: all C columns in
 * order, n is then ignored).  out: R's "dist" vector, n (n - 1) / 2 doubles, the strict lower triangle by columns -
 * out[n a - a (a + 1) / 2 + (b - a - 1)] for list positions a < b.  Difference form, genes in order, one fused
 * multiply-add per term (no cancellation for near-identical cells).  n < 2: nothing is written. */
ICNV_API int icnv_pairwise_dist_f64(const double *X, int64_t G, int64_t C, const int32_t *cells, int64_t n, double *out);
/* The same distances from the matrix AS parallelDist() RECEIVES IT - observations x variables, column-major, i.e. the
 * t(expr.data[, cells]) the reference builds at every call site (n cells x G genes, cell a / gene g at x[a + n g]): the R
 * closure passes its argument through without transposing it back. */
ICNV_API int icnv_pairwise_dist_rows_f64(const double *x, int64_t n, int64_t G, double *out);

/* RANN::nn2(data, k = k) with the query set = the data set - the kNN graph of .leiden_simple_snn,
 * R/inferCNV_tumor_subclusters.R:725-741 (NAMESPACE: importFrom(RANN, nn2)): for each of the n cells its k nearest cells
 * under the Euclidean distance over the genes, itself included.  Exact (no approximation, no n x n buffer: device memory is
 * the input plus O(n k)).  idx / dist: n x k column-major, as R's nn.idx / nn.dists; idx holds 0-based list positions (the
 * R shim adds 1).  Row i is ordered by ascending squared distance, then ascending position - a total order, so the result
 * does not depend on the launch geometry, and cell i comes first in its row unless a duplicate of it has a lower position.
 * ANN orders ties by its tree traversal, so among equally near cells the choice can differ from RANN's; only ties that
 * straddle the k-th place change the neighbour set.  Distances are the square roots of the same sums as
 * icnv_pairwise_dist_f64 (difference form, genes in order, one fused multiply-add each): every dist[i, j] has the bits of
 * that pair's "dist" entry.  k < 1 or k > n: ICNV_E_BAD_ARG; k > ICNV_KNN_MAX_K: ICNV_E_UNSUPPORTED; NaN / Inf in a listed
 * cell: ICNV_E_NONFINITE; n = 0: nothing is written; G = 0: every distance is 0, row i is 0 .. k-1.
 * This entry takes the matrix as nn2() receives it: observations x variables, cell a / gene g at x[a + n g]. */
#define ICNV_KNN_MAX_K 64
ICNV_API int icnv_knn_rows_f64(const double *x, int64_t n, int64_t G, int k, int32_t *idx, double *dist);
/* The same from the genes x cells matrix X (G x C, column-major) and a list of n 0-based columns (NULL: all C columns in
 * order, n is then ignored), as icnv_pairwise_dist_f64 takes them. */
ICNV_API int icnv_knn_f64(const double *X, int64_t G, int64_t C, const int32_t *cells, int64_t n, int k, int32_t *idx,
                          double *dist);

/* hclust(d, method) - fastcluster::hclust, which infercnv imports - on R's "dist" vector d of n observations (the layout
 * above).  Nearest-neighbour chain with Lance-Williams updates on an n x n FP64 matrix on the device (n^2 * 8 bytes; the
 * host vector goes in slab by slab).  method, coded as fastcluster orders them: 0 single, 1 complete, 2 average,
 * 3 mcquitty, 4 ward.D, 7 ward.D2 (ward.D on the squared input, heights rooted).  5 centroid / 6 median and n > 65536:
 * ICNV_E_UNSUPPORTED; NaN / Inf in d: ICNV_E_NONFINITE; n < 2 or another code: ICNV_E_BAD_ARG; no room: ICNV_E_NOMEM.
 * Output in R's convention: merge (n - 1) x 2 column-major (singleton -(i + 1), cluster of step s +s, the smaller node
 * first), height (n - 1, non-decreasing), order (n, 1-based).  Tie rules: see icnv_hclust.cu. */
ICNV_API int icnv_hclust_f64(const double *d, int64_t n, int method, int32_t *merge, double *height, int32_t *order);
/* R's order from merge: hcass2's traversal (start from the last merge, expand the first column before the second).
 * Host only, no GPU. */
ICNV_API int icnv_hclust_order(const int32_t *merge, int64_t n, int32_t *order);
/* icnv_hclust_f64 past its 65536 limit: the same linkage on the packed strict lower triangle - R's "dist" vector itself,
 * 4 n (n - 1) bytes on the device instead of 8 n^2 - so n is bounded by memory alone (about 130 000 observations on an
 * 80 GB device).  Same methods, arithmetic, tie rules and output convention: wherever both run, merge / height / order
 * equal icnv_hclust_f64's bit for bit.  The host vector goes up in 64 MB pieces through two page-locked slabs straight into
 * the device triangle.  Before anything is allocated, the triangle plus the linkage's scratch (8 (n + P) + 4 (6 n + P)
 * bytes, P the power of two >= n - 1) plus 256 MB is checked against the free device memory: ICNV_E_NOMEM if it does not
 * fit.  Centroid / median: ICNV_E_UNSUPPORTED; NaN / Inf in d: ICNV_E_NONFINITE; n < 2 or another code: ICNV_E_BAD_ARG. */
ICNV_API int icnv_hclust_tri_f64(const double *d, int64_t n, int method, int32_t *merge, double *height, int32_t *order);
/* hclust(parallelDist(t(X[keep, cells])), method) in one call, for one group of any size that fits: the distances of the
 * listed columns of the G x C matrix X (cells: n 0-based columns, NULL: all C in order, n is then ignored) over the genes
 * keep (n_keep 0-based rows; NULL: all G; an empty list, keep != NULL and n_keep = 0: none, so every distance is 0) are
 * written by K10's tiles straight into the device triangle and linked there - no distance vector crosses PCIe.
 * merge / height / order equal icnv_pairwise_dist_f64 -> icnv_hclust_tri_f64 bit for bit (and icnv_cluster_groups_f64 for
 * a group it accepts).  Only the listed columns go to the device.  Errors as icnv_hclust_tri_f64 (the memory check also
 * counts the uploaded columns and the gathered genes); an index out of range: ICNV_E_BAD_ARG; NaN / Inf in a used column
 * (or an infinite distance): ICNV_E_NONFINITE. */
ICNV_API int icnv_cluster_cells_f64(const double *X, int64_t G, int64_t C, const int32_t *keep, int64_t n_keep,
                                    const int32_t *cells, int64_t n, int method, int32_t *merge, double *height,
                                    int32_t *order);

/* caTools::runmean(x, k) with its defaults (alg "C", endrule "mean", align "center") down every column of the G x C matrix X,
 * per row range - smooth_by_chromosome_runmeans (R/inferCNV_ops.R:2679-2704) with the chromosomes as ranges.  For a range
 * of L genes, k' = min(k, L), k2 = k' / 2, k1 = k' - 1 - k2: Y[p] = mean(X[max(0, p - k1) .. min(L - 1, p + k2)]) (positions
 * within the range).  k <= 1, ranges of fewer than 2 genes and the genes outside every range are copied.  The K ranges
 * (chr_start, chr_len; chr_start NULL: the single range [0, G), K ignored) must be ordered and disjoint inside [0, G).
 * An even k is computed by the rule above.  Double-double running sum: |Y[p] - m| <= 2 u |m| + 8 L u^2 T / cnt
 * (m the exact window mean, cnt its count, T the sum of |x| over the range, u = 2^-53), independent of the launch geometry.
 * NaN / Inf anywhere in X: ICNV_E_NONFINITE (caTools skips NaNs; the R wrapper falls back). */
ICNV_API int icnv_runmean_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *chr_start,
                              const int32_t *chr_len, int K, int k);

/* The permutation null of random-trees subclustering, .parameterize_random_cluster_heights_smoothed_trees
 * (R/inferCNV_tumor_subclusters.random_smoothed_trees.R:217-304), for one clade in one call.  The clade is the list of n
 * 0-based columns `cells` of the G x C matrix X (NULL: all C columns, n is then ignored).
 *   Observed tree: icnv_runmean_f64(window) over [0, G) -> icnv_center_f64 (median) -> icnv_pairwise_dist_f64 ->
 *   icnv_hclust_f64(method): merge / height / order exactly as that composition returns them, bit for bit.
 *   perm_max_height[p], p < n_perm: the largest height of the tree built the same way on permutation p, which shuffles
 *   every gene independently across the cells: key(p, g, i) = mix64(hash3(seed, p, g, i)) (the splitmix generator of
 *   icnv_synth.cu, finalised once more so that the keys of one (p, g) order the positions uniformly),
 *   pi_{p,g} = the stable ascending argsort of the keys over the list positions i, and
 *   X_p[g, i] = X[g, cells[pi_{p,g}(i)]].  Member p depends only on (data, seed, p): the first m maxima of a call equal an
 *   m-permutation call with the same seed.
 * The members run in waves of B = min(n_perm + 1, SM count, members that fit the free device memory) linkages, one SM each;
 * the result does not depend on B.  Device memory: the input, two G x n working copies and one n x n matrix per member of a
 * wave.  Methods as icnv_hclust_f64.  n < 2, another method code or n_perm < 0: ICNV_E_BAD_ARG; centroid / median or
 * n > 65536: ICNV_E_UNSUPPORTED; NaN / Inf in the clade: ICNV_E_NONFINITE; not even one member fits: ICNV_E_NOMEM. */
ICNV_API int icnv_random_tree_heights_f64(const double *X, int64_t G, int64_t C, const int32_t *cells, int64_t n, int window,
                                          int method, int n_perm, uint64_t seed, int32_t *merge, double *height,
                                          int32_t *order, double *perm_max_height);
/* What the last random-trees call did: out5 = {B, waves, ms of shuffle + runmean + centring, ms of distances, ms of
 * linkages} (device time summed over the waves); zeros before any call. */
ICNV_API int icnv_debug_random_trees(double *out5);

/* The z-score gene filter of define_signif_tumor_subclusters (R/inferCNV_tumor_subclusters.R:45-68) on the G x C matrix X:
 *   ref = X[, ref_idx] (n_ref 0-based columns, unlist(reference_grouped_cell_indices) in that order),
 *   z = (ref - mean(ref)) / sd(ref),   outlier[g] = 1 when mean(|z[g, ]|) >= 0.8, else 0.
 * mean(ref) / sd(ref) are icnv_mean_sd_f64's bits for the same list; each z is |__ddiv_rn(x - mu, sigma)|, and the row mean
 * is the correctly rounded mean of those values (R's long-double mean() with its refinement pass, restated with
 * double-double sums).  The threshold is the literal 0.8; a constant reference (sigma = 0, every z NaN) flags no gene.
 * G < 2, n_ref < 1 or an index outside [0, C): ICNV_E_BAD_ARG; NaN / Inf in a listed column: ICNV_E_NONFINITE. */
ICNV_API int icnv_zscore_outlier_genes_f64(const double *X, int64_t G, int64_t C, const int32_t *ref_idx, int64_t n_ref,
                                           uint8_t *outlier);

/* Every tree of define_signif_tumor_subclusters in one call: for each group k (CSR: 0-based columns
 * grp_idx[grp_off[k] .. grp_off[k+1]) of the G x C matrix X) with n_k >= 2 cells,
 *   hclust(parallelDist(t(X[keep, cells_k])), method) - icnv_pairwise_dist_f64 -> icnv_hclust_f64 on that group, bit for bit.
 * keep: n_keep 0-based genes (any order); NULL means all G genes, and an empty list (n_keep = 0, keep != NULL) means none,
 * so every distance is 0 (expr.data[-integer(0), ] keeps no row).  Outputs are packed in group order: the trees of the groups
 * before k take R_k = sum of (n_j - 1) over those of them with n_j >= 2 rows, and group k's merge ((n_k - 1) x 2,
 * column-major) is at merge + 2 R_k, its height at height + R_k, its order (1-based) at order + grp_off[k].  A group of one
 * cell gets order 1 and no row; an empty group gets nothing.  Only the listed columns go to the device.  The groups run as
 * the linkages of waves of at most one group per SM (largest first, as many as fit the free device memory); the result does
 * not depend on the waves.  Methods as icnv_hclust_f64.  Centroid / median or a group of more than 65536 cells:
 * ICNV_E_UNSUPPORTED, before anything is allocated; another method code, an index out of range or descending offsets:
 * ICNV_E_BAD_ARG; NaN / Inf in a used column (or an infinite distance): ICNV_E_NONFINITE. */
ICNV_API int icnv_cluster_groups_f64(const double *X, int64_t G, int64_t C, const int32_t *keep, int64_t n_keep,
                                     const int32_t *grp_off, const int32_t *grp_idx, int n_grp, int method, int32_t *merge,
                                     double *height, int32_t *order);
/* What the last group-trees call did: out5 = {waves, groups in the largest wave, ms of the gene gather, ms of distances,
 * ms of linkages} (device time summed over the waves); zeros before any call and after a call without a tree. */
ICNV_API int icnv_debug_cluster_groups(double *out5);

/* The shared-nearest-neighbour graph of .leiden_seurat_preprocess_routine (R/inferCNV_tumor_subclusters.R:699-723; Seurat 5's
 * FindVariableFeatures(vst) -> ScaleData -> RunPCA(npcs) -> FindNeighbors(k.param), prune.SNN 1/15) on the group matrix
 * X[, cells] (G x C, 0-based columns; cells NULL: all C):
 *   1. mu_g and v_g (denominator n - 1) over the n cells;
 *   2. the vst trend: direct local quadratic loess (span 0.3, tricube weights on the q = floor(0.3 m) nearest) of log10 v on
 *      log10 mu over the m genes with v > 0; expected variance 10^fit, 0 for constant genes;
 *   3. standardised variance sum_c min((x - mu) / s, sqrt(n))^2 / (n - 1), s = sqrt(expected variance) (0 where s = 0),
 *      ranked decreasing, ties by lower index: the first min(n_features, G) genes are the variable features;
 *   4. z = min((x - mu) / sqrt(v), 10) on the F non-constant variable features;
 *   5. the top npcs eigenvectors V of Z Z^T (exact to ||C v - l v|| <= 1e-12 l_1), each signed so that its largest |entry| is
 *      positive (ties: lower feature rank); embeddings E = Z^T V;
 *   6. K12's exact k nearest cells in E (self included; distance, then position), and for every pair with
 *      s = |N(i) & N(j)| >= 1, w = s / (k + (k - s)), dropped when w < 1/15.  Symmetric, diagonal kept (w = 1).
 * The result stays in the library until the next call; *nnz is its number of graph entries and icnv_seurat_snn_fetch
 * copies it out.  Bad sizes or an index out of range: ICNV_E_BAD_ARG; NaN / Inf in a listed column: ICNV_E_NONFINITE;
 * k > 64, npcs > 16, n <= npcs, fewer than 3 genes in the loess window, F <= npcs, a non-constant gene with mean <= 0 (vst's
 * log10 warns there), no convergence of the eigenpairs, or a group larger than the free device memory: ICNV_E_UNSUPPORTED. */
ICNV_API int icnv_seurat_snn_f64(const double *X, int64_t G, int64_t C, const int32_t *cells, int64_t n, int n_features,
                                 int npcs, int k, int64_t *nnz);
/* Copies out the last SNN call's result; any pointer may be NULL.  row_ptr: n + 1; col (0-based, ascending per row) and w:
 * nnz; features: min(n_features, G) 0-based gene indices in rank order; emb: npcs x n column-major (K12's layout);
 * idx: n x k column-major, 0-based positions.  No result held: ICNV_E_BAD_ARG. */
ICNV_API int icnv_seurat_snn_fetch(int64_t *row_ptr, int32_t *col, double *w, int32_t *features, double *emb, int32_t *idx);
/* What the last SNN call did: out16 = {F, npcs used, eigen-iterations, largest ||C v_j - l_j v_j|| / l_1, l_npcs / l_npcs+1
 * (inf when the block has no npcs+1-th value), standardised-variance gap between ranks n_features and n_features + 1 (inf
 * when G <= n_features), local trend fits that were singular (where R's loess warns and the routine falls back), device ms
 * of: statistics, trend, standardised variance + ranking, Gram matrix, eigenpairs, embeddings, kNN, SNN; hub rows that took
 * the global-memory path}; zeros before any call. */
ICNV_API int icnv_debug_seurat_snn(double *out16);

/* mask_non_DE_genes_basic (R/inferCNV_mask_non_DE.R:28-52; run() step 21, R/inferCNV_ops.R:1509-1524) on the G x C matrix X:
 * get_DE_genes_basic's tests, BH and .mask_DE_genes' mask in one call.
 *   Groups (CSR, 0-based columns): n_ref >= 1 reference groups; n_sub >= 0 TESTED subclusters in R's loop order (observation
 *   group by group, its subclusters in names() order - a group whose subclusters are not a named list is tested by R for
 *   nothing and is simply not listed).  Pair column s * n_ref + j: x = reference group j, y = subcluster s.
 *   test 0 (wilcoxon, :191-203): each side jittered (below), then wilcox.test(x, y) with R's defaults - exact when n_x < 50,
 *        n_y < 50 and no ties in x u y, else the normal approximation with continuity and tie corrections (NaN when every
 *        value of the pair is tied).  test 1 (t, :166-176): Welch's t.test(x, y) on the unjittered values; NaN where R's
 *        try() catches an error (n < 2, or stderr < 10 eps max(|mean x|, |mean y|)).
 *   p_adj: p.adjust(method = "BH") per pair over the genes in R's operation order, n = the non-NaN count; NaN stays NaN.
 *   DE: p_adj < p_thresh.  Mask: per cell and gene a count - reference cells and the cells of a tested subcluster of < 5
 *   list entries start at n_ref, each cell of a tested subcluster of >= 5 entries adds 1 per reference group where the gene
 *   is DE for that subcluster (once per subcluster), other cells start at 0; rule 0 "any" masks count == 0, 1 "most"
 *   count < n_ref / 2, 2 "all" count != n_ref.  Masked entries of Y are mask_val (R's center_val), the others X's.
 *   Generator (Wilcoxon): jitter = jitter_mean + jitter_sd z (no contraction), z Box-Muller on two (0, 1] uniforms
 *   ((mix64(hash3(seed, a, g, 2 i + k)) >> 11) + 1) 2^-53 (k = 0, 1), z = sqrt(-2 log u_0) cospi(2 u_1); g the gene, i the
 *   list position within the group, a = j for reference group j, a = 2^32 + pair for a subcluster.  Reference-side draws
 *   are keyed by (j, gene, position) and shared by all subclusters, so each reference row is jittered and sorted once per
 *   gene: the joint law of one subcluster's columns equals R's (it uses each reference group once), but the columns of
 *   different subclusters are dependent through the shared draws, where R's are conditionally independent.  R's closure
 *   passes 1e-4 / 1e-4; jitter_sd = 0 keeps every tie and makes the statistic deterministic.
 * Y (G x C; may be X), p_raw and p_adj (G x (n_sub n_ref), column-major, column s * n_ref + j) are each nullable.
 * An empty group, an index out of range, an unknown test or rule code, jitter_sd < 0: ICNV_E_BAD_ARG; NaN / Inf in a listed
 * cell: ICNV_E_NONFINITE; not enough device memory: ICNV_E_NOMEM.
 * Several device slots (icnv_init_devices): the genes are cut into one contiguous range per device, each device uploads only
 * its genes of the listed columns (in sub-slabs sized from its free memory) and tests them; the p rows are gathered on the
 * host, every device runs BH on all of them and masks its own range of cells, streamed through it in chunks.  The output
 * bytes are those of one device, and X need not fit on any one of them. */
ICNV_API int icnv_mask_non_de_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *ref_off,
                                  const int32_t *ref_idx, int n_ref, const int32_t *sub_off, const int32_t *sub_idx, int n_sub,
                                  int test, double p_thresh, int rule, double mask_val, double jitter_mean, double jitter_sd,
                                  uint64_t seed, double *p_raw, double *p_adj);
/* What the last mask call did: out7 = {gene tiles, genes per tile, ms of (a) gather, (b) reference sorts / group statistics,
 * (c) pair tests, (d) BH, (e) mask} (device time summed over the tiles); zeros before any call.  With several device slots:
 * the tiles summed over the devices, the largest tile, and each stage's time on the device where it took longest (the
 * gather is the transposition of the uploaded columns; BH and the mask are summed over a device's cell chunks). */
ICNV_API int icnv_debug_mask_non_de(double *out7);

/* Gibbs sampling of inferCNVBayesNet (R/inferCNV_BayesNet.R run_gibb_sampling, :1054-1107; run() step 18) for n_reg CNV
 * regions of the G x C matrix X in one call - the posterior JAGS samples, not its draws.
 *   Regions (CSR, 0-based): genes gene_idx[gene_off[r] .. gene_off[r+1]), cells cell_idx[cell_off[r] .. cell_off[r+1]), both
 *   non-empty.  pooled (nullable u8 per region): R's one-gene quirk - the region is ONE pseudo-cell whose "genes" are all its
 *   entries (cells in list order, within a cell its genes in list order); C'_r = 1 for a pooled region, C_r otherwise.
 *   Model: x ~ dnorm(mu[eps], tau[eps]) (tau a precision), eps_j ~ dcat(theta), theta ~ ddirich(1, ..., 1), m = 2..8 states.
 *   L[j, k] = sum over the region's entries of column j of (1/2 log tau_k - 1/2 tau_k (x - mu_k)^2), FP64 in list order.
 *   n_chains chains (chain c starts from eps = c mod m, as R's inits rep(c, C)), n_burn discarded sweeps, then n_keep kept,
 *   thin 1; a sweep draws theta | eps ~ Dirichlet(1 + n) (Marsaglia-Tsang gammas, FP64), then eps_j | theta with weights
 *   theta_k exp(L[j, k]): FP64 log-weights less their maximum, exp and cumulative sum in FP32 (each normalised weight within
 *   1e-6 absolute: expf's 2 ulp, the FP32 rounding of the argument and of the sum stay under 8e-7).  Every draw is keyed
 *   by (seed, region, chain, sweep, state or column, rejection attempt) through mix64 / hash3, so the result is a pure
 *   function of (seed, inputs), whatever the launch shape or the thread order.
 *   Device memory besides the outputs: L (when loglik is NULL) and one private count buffer per sampler CTA of
 *   ceil(max_r C'_r / 256) * 256 * m int32 - (2 x SM count) CTAs, e.g. 634 MB for 264 CTAs at 100 000 cells and m = 6.
 * theta: per region r at offset r n_chains n_keep m, a column-major (n_chains n_keep) x m block, chains stacked in order (R's
 * do.call(rbind, chains)).  state_counts (int32) and loglik (nullable): per region an m x C'_r column-major block at offset
 * m sum_{s<r} C'_s; state_counts[k, j] = kept draws of column j in state k over all chains (sums to n_chains n_keep).
 * An empty gene or cell list, an index out of range, m outside 2..8, tau <= 0, a non-finite mu or tau, n_chains < 1,
 * n_keep < 1 or n_burn < 0: ICNV_E_BAD_ARG; NaN / Inf in a listed entry: ICNV_E_NONFINITE; not enough device memory:
 * ICNV_E_NOMEM.  Pageable X goes up through the pinned staging ring. */
ICNV_API int icnv_bayesnet_f64(const double *X, int64_t G, int64_t C, const int32_t *gene_off, const int32_t *gene_idx,
                               const int32_t *cell_off, const int32_t *cell_idx, const uint8_t *pooled, int n_reg, int m,
                               const double *mu, const double *tau, int n_chains, int n_burn, int n_keep, uint64_t seed,
                               double *theta, int32_t *state_counts, double *loglik);
/* What the last Bayesian network call did: out4 = {regions, sampler CTAs, ms of (a) the log-likelihood pass, (b) the
 * sampler}; zeros before any call. */
ICNV_API int icnv_debug_bayesnet(double *out4);

/* smooth_by_chromosome_coordinates (R/inferCNV_ops.R:2534-2622; run() step 10, smooth_method = "coordinates") on the G x C
 * matrix X, the K ranges (chr_start, chr_len) as its chromosomes.  For gene i of a range of n >= 2 genes with starts s and
 * stops e (gene_start / gene_stop, indexed by row of X) and W = window_length >= 2:
 *   pos = (s[i] + e[i]) / 2, around = {j : s[j] > pos - W and e[j] < pos + W} ({i} if empty; need not be contiguous),
 *   w_j = 1 - |(e[j] + s[j]) / 2 - pos| / W, to_add = floor(|around| / 2), lo = max(0, min(around) - to_add),
 *   hi = min(n - 1, max(around) + to_add), wv = (0.1 x (min(around) - lo), w_around, 0.1 x (hi - max(around))),
 *   Y[i] = sum_k X[lo + k] wv[k mod |wv|] / sum(wv),  k = 0 .. hi - lo   (R's recycling where `around` has holes).
 * W < 2, ranges of one gene and the genes outside every range are copied.  Genes need not be sorted by start.  Ranges
 * must be ordered and disjoint inside [0, G); the coordinates of every gene of a range finite; W finite (else
 * ICNV_E_BAD_ARG); G <= 2 097 120 (else ICNV_E_UNSUPPORTED).  NaN / Inf in X: ICNV_E_NONFINITE (the R wrapper falls back).
 * The host builds the weights of every row (O(n^2) per range; sum over rows of (hi - lo + 1) doubles of device memory, up
 * to the sum of n^2 when W spans whole ranges: ICNV_E_NOMEM if it does not fit).
 * Arithmetic: t_k = fl(x_k w_k) as R's `*` (no contraction); den = sum(wv) in sequential long double, rounded (= R's on
 * x86-64); the numerator N is Sum2 (cascaded two-sum) of the t_k in increasing k, and Y = fl(N / den).  With S = sum t_k,
 * A = sum |t_k|, L = hi - lo + 1, u = 2^-53 and g_n = n u / (1 - n u):
 *   |Y - S / den| <= ((2 u + u^2) |S| + (1 + u) g_{L-1}^2 A) / den,
 * independent of the launch geometry; R's own value (80-bit partial sums, u' = 2^-64, g'_n = n u' / (1 - n u')) satisfies
 * |Y_R - S / den| <= ((2 u + u^2) |S| + (1 + u)^2 g'_{L-1} A) / den.
 * The dev variant takes X / Y on the device (leading dimensions ldx, ldy >= G; Y must not overlap X), the ranges and
 * coordinates on the host; it returns once the result is complete. */
ICNV_API int icnv_smooth_coordinates_f64(const double *X, double *Y, int64_t G, int64_t C, const int32_t *chr_start,
                                         const int32_t *chr_len, int K, const double *gene_start, const double *gene_stop,
                                         double window_length);
ICNV_API int icnv_dev_smooth_coordinates_f64(const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t G, int64_t C,
                                             const int32_t *chr_start, const int32_t *chr_len, int K, const double *gene_start,
                                             const double *gene_stop, double window_length, void *stream);

/* Combine per-cell (sum, sd) pairs - e.g. all-gathered from several GPUs - into mu / sigma over all values
 * of those cells, in list order (what icnv_mean_sd_f64 does internally). */
ICNV_API void icnv_combine_cell_stats(const double *sums, const double *sds, int64_t n, int64_t G, double *mu,
                                      double *sigma);

/* ---- gene filters and counts ingest: the steps in front of the path (run() steps 2-3) ------------------------
 * Per-gene statistics of a dense G x C matrix for the two gene filters of run() step 2:
 *   sums[g]  = sum over all cells; means[g] = rowMeans as R rounds it (long-double quotient -> double), what
 *              .below_min_mean_expr_cutoff compares with the cutoff (R/inferCNV_ops.R:2149-2158);
 *   n_pos[g] = number of cells with x > 0 (NaN counts as not expressed), what require_above_min_cells_ref compares
 *              with min_cells_per_gene (ops.R:2177-2209).
 * Any of the three outputs may be NULL. */
ICNV_API int icnv_gene_stats_f64(const double *X, int64_t G, int64_t C, double *sums, int32_t *n_pos, double *means);

/* scale_infercnv_expr, R/inferCNV_ops.R:3174-3186 (run() step 5, scale_data = TRUE): t(scale(t(expr))) - every gene
 * (row) centred at its mean over the cells and divided by its sd (n - 1).  A constant gene gives NaN, as in R. */
ICNV_API int icnv_scale_infercnv_expr_f64(const double *X, double *Y, int64_t G, int64_t C);

/* remove_genes, R/inferCNV.R:445-457: Y (n_keep x C) = X[keep, ]; keep = increasing 0-based row indices. */
ICNV_API int icnv_remove_genes_f64(const double *X, int64_t G, int64_t C, const int32_t *keep, int64_t n_keep,
                                   double *Y);

/* Rows in any order, repeats allowed: Y (n x C) = X[idx, ] - the reordering of the expression matrix to the genomic
 * position table in .order_reduce (R/inferCNV.R:352-428; CreateInfercnvObject's ingest). */
ICNV_API int icnv_gather_genes_f64(const double *X, int64_t G, int64_t C, const int32_t *idx, int64_t n, double *Y);

/* The same statistics for a compressed-sparse-column counts matrix (a dgCMatrix's @p, @i, @x; the reference accepts
 * one as raw_counts_matrix, R/inferCNV.R:158-160): p[C+1] column pointers, i[nnz] 0-based row indices, x[nnz]. */
ICNV_API int icnv_csc_gene_stats_f64(const int32_t *p, const int32_t *i, const double *x, int64_t G, int64_t C,
                                     double *sums, int32_t *n_pos, double *means);

/* Gene removal + normalize_counts_by_seq_depth (ops.R:3064-3111) straight from the compressed columns: Y, dense
 * G_out x C (G_out = n_keep, or G when keep == NULL), = (x / colSums over the kept genes) * normalize_factor; a
 * negative or NaN factor means "median of the column sums" (the reference's NA default).  The matrix crosses PCIe
 * as 12 bytes per stored count instead of 8 bytes per cell-gene.  col_sums: optional C doubles. */
ICNV_API int icnv_csc_normalize_f64(const int32_t *p, const int32_t *i, const double *x, int64_t G, int64_t C,
                                    const int32_t *keep, int64_t n_keep, double normalize_factor, double *Y,
                                    double *col_sums);

/* ---- CNV region calling on the HMM state matrix (the step after the Viterbi kernels) ---------------------
 * States use the one-byte wire format of the *_u8 Viterbi variants: 0..6 = state, 255 = unassigned (R's -1).
 *
 * .get_state_consensus, R/inferCNV_HMM.R:977-988: consensus[g + G*k] = the most frequent state of gene g over
 * the cells of group k; ties go to the smallest state, 255 (-1) ordering before every state, as
 * table() / order(decreasing=TRUE)[1] do.  A byte outside {0..6, 255}: ICNV_E_BAD_ARG. */
ICNV_API int icnv_state_consensus_u8(const uint8_t *states, int64_t G, int64_t C, const int32_t *grp_off,
                                     const int32_t *grp_idx, int n_grp, uint8_t *consensus);

/* The step that ends predict_CNV_via_HMM_on_tumor_subclusters_per_chr (HMM.R:470-483: get_predicted_CNV_regions by
 * "subcluster", then every region's state written to all cells of its group): out[g, c] = consensus state of c's
 * group at gene g, for the genes region calling covers (chromosomes with >= 2 genes); other genes and cells in no
 * group keep their state.  out may alias states. */
ICNV_API int icnv_apply_state_consensus_u8(const uint8_t *states, int64_t G, int64_t C, const int32_t *chr_start,
                                           const int32_t *chr_len, int K, const int32_t *grp_off,
                                           const int32_t *grp_idx, int n_grp, uint8_t *out);

/* .define_cnv_gene_regions + .get_cnv_gene_region_bounds, R/inferCNV_HMM.R:1006-1087, for n_seq state sequences
 * (the columns of seqs, G x n_seq): within every chromosome of >= 2 genes (shorter ones are skipped, :1012-1014)
 * each run of equal states is one region.  Regions are produced in (sequence, chromosome, position) order - the
 * order get_predicted_CNV_regions numbers them in (:735-760), so region i (0-based) of a call is "region_<i+1>".
 * gene_start / gene_stop: gene_order$start / $stop as doubles (exact for integer positions below 2^53).
 * The call leaves the records in the library and reports their number; icnv_cnv_regions_fetch copies them out. */
ICNV_API int icnv_cnv_regions_u8(const uint8_t *seqs, int64_t G, int64_t n_seq, const int32_t *chr_start,
                                 const int32_t *chr_len, int K, const double *gene_start, const double *gene_stop,
                                 int64_t *n_regions);

/* get_predicted_CNV_regions, R/inferCNV_HMM.R:706-764, in one upload of the state matrix: consensus of every
 * cell group (reference groups + observation groups for by = "consensus", the subclusters for by = "subcluster",
 * one single-cell group per cell for by = "cell"; the caller orders the groups as the reference does) followed
 * by region calling on the n_grp consensus sequences.  consensus: optional G x n_grp output (may be NULL). */
ICNV_API int icnv_predicted_cnv_regions_u8(const uint8_t *states, int64_t G, int64_t C, const int32_t *chr_start,
                                           const int32_t *chr_len, int K, const double *gene_start,
                                           const double *gene_stop, const int32_t *grp_off, const int32_t *grp_idx,
                                           int n_grp, uint8_t *consensus, int64_t *n_regions);

/* Records of the last icnv_cnv_regions_u8 / icnv_predicted_cnv_regions_u8 call; n_regions must be the number that
 * call reported.  Per region: seq (0-based sequence / group), chr (0-based chromosome), first_gene .. last_gene
 * (0-based, inclusive), state (0..6, -1 = unassigned), start = min(gene_start), end = max(gene_stop) over its
 * genes (:1078-1079).  Any output pointer may be NULL. */
ICNV_API int icnv_cnv_regions_fetch(int64_t n_regions, int32_t *seq, int32_t *chr, int32_t *first_gene,
                                    int32_t *last_gene, int32_t *state, double *start, double *end);

/* ---- device-pointer entry points ------------------------------------------------------------- */
/* All pointers are device pointers on the icnv_init() device unless marked host.  `stream` is a
 * cudaStream_t; NULL = the library's own (non-blocking) stream - pass cudaStreamLegacy ((void*)1) to
 * run on the legacy default stream.  Asynchronous: the caller synchronises. */

/* Partial sums for group means, fixed summation order so results do not depend on the number of
 * GPUs: cells[0..n_cells) (device, column indices into X) are cut into chunks of `chunk` list
 * entries; partial[g + G*q] = sum over chunk q, in list order, of f(X[g, cell]) with
 * f = identity, or log2(x+1) when apply_log.  n_chunks = ceil(n_cells/chunk). */
ICNV_API int icnv_dev_group_partial_sums_f64(const double *X, int64_t G, int64_t ldx, const int32_t *cells,
                                             int64_t n_cells, int chunk, int apply_log, double *partial,
                                             void *stream);
/* Reference bounds (min / max / mean over the groups of the per-gene group means) from chunk sums laid out
 * [world][tot_rows][G] - what an all-gather of every rank's icnv_dev_group_partial_sums_f64 rows gives; group k owns rows
 * row_off[k] .. row_off[k+1] of each rank's block, counts[k] is its global size.  Replaces .get_normal_gene_mean_bounds'
 * per-group mean() (R/inferCNV_ops.R:1708-1735) + the min / max of .subtract_expr (:1742-1786) in one launch. */
ICNV_API int icnv_dev_bounds_from_partials_f64(const double *partials, int64_t G, int world, int64_t tot_rows, int n_grp,
                                               const int32_t *row_off, const int64_t *counts, double *lo, double *hi,
                                               double *mid, void *stream);
/* The group means themselves from the same layout of chunk sums: means[g + G*k] (rowMeans of a group spread over ranks -
 * the group modes of the HMM, R/inferCNV_HMM.R:383 - in the fixed chunk order, so the rank count does not matter). */
ICNV_API int icnv_dev_means_from_partials_f64(const double *partials, int64_t G, int world, int64_t tot_rows, int n_grp,
                                              const int32_t *row_off, const int64_t *counts, double *means, void *stream);
/* Group-mode broadcast on the device: out[g + G*c] = group_states[g + G*grp_of[c]], 255 where grp_of[c] < 0
 * (R/inferCNV_HMM.R:368, 399: every cell of a group gets the group's trace, cells in no group stay unassigned). */
ICNV_API int icnv_dev_scatter_group_states_u8(const uint8_t *group_states, int64_t G, int64_t C, const int32_t *grp_of,
                                              uint8_t *out, void *stream);
/* means[g] = (sum_q partial[g + G*q], q ascending) / count */
ICNV_API int icnv_dev_combine_partials_f64(const double *partial, int64_t G, int64_t n_chunks, int64_t count,
                                           double *means, void *stream);
/* lo/hi/mid over the n_grp columns of means (each length G). */
ICNV_API int icnv_dev_bounds_from_means_f64(const double *means, int64_t G, int n_grp, double *lo, double *hi,
                                            double *mid, void *stream);

/* The fused per-cell kernel.  For every listed column (cols == NULL: columns 0..n_cols-1 of X):
 *   v = X[:, col]; [v = log2(v+1)]; [v = dead-band subtract (lo1, hi1) or v - mid1];
 *   [clamp +-threshold]; [smooth(window) per chromosome]; [v -= median(v) | mean(v)];
 *   [dead-band subtract (lo2, hi2) or v - mid2]; [v = 2^v]; Y[:, i] = v   (output column i, ld = ldy)
 * Stage selection: lo1/hi1 NULL -> skip; mid1 used when lo1 == NULL && mid1 != NULL; threshold <= 0
 * -> skip; window < 2 -> skip; center: 0 none, 1 median, 2 mean; lo2/hi2/mid2 likewise; apply_exp2.
 * err_flag (device int*, may be NULL) is set to 1 when a non-finite value is seen. */
ICNV_API int icnv_dev_cell_pipeline_f64(const double *X, int64_t G, int64_t ldx, const int32_t *cols, int64_t n_cols,
                                        double *Y, int64_t ldy, const int32_t *chr_start /*host*/,
                                        const int32_t *chr_len /*host*/, int K, int apply_log, const double *lo1,
                                        const double *hi1, const double *mid1, double threshold, int window,
                                        int center, const double *lo2, const double *hi2, const double *mid2,
                                        int apply_exp2, int *err_flag, void *stream);
/* Which instantiation of the fused kernel the last icnv_dev_cell_pipeline_f64 call on this device launched (read-only;
 * the host entry points go through it too): out6 = {family (3: two-buffer kernel, 4: single-buffer kernel), threads per
 * CTA, minimum CTAs per SM of its launch bounds, padded-Q layout (0 / 1), fully unrolled slice length (0: generic loops),
 * slice length L of the segment table}.  All zero when that call launched nothing (refused, or no columns). */
ICNV_API int icnv_debug_cell_kernel(int *out6);

/* Whole smooth block on device-resident data (single GPU): X, Y are G x C (ld = G). */
ICNV_API int icnv_dev_smooth_block_f64(const double *X, double *Y, int64_t G, int64_t C,
                                       const int32_t *chr_start /*host*/, const int32_t *chr_len /*host*/, int K,
                                       const int32_t *grp_off /*host*/, const int32_t *grp_idx /*host*/, int n_grp,
                                       int apply_log, double threshold, int window, int use_bounds, void *stream);

/* Per-sequence Viterbi on device-resident X (G x C, ld = G), one sequence per (column, chromosome).
 * states_u8: uint8 G x C (1..m).  margins: device K x C doubles or NULL.  Model arrays are host.
 * sd has m entries (sd_per_col == 0) or m per column (sd_per_col != 0, device-order = column). */
ICNV_API int icnv_dev_viterbi_f64(const double *X, int64_t G, int64_t C, const int32_t *chr_start /*host*/,
                                  const int32_t *chr_len /*host*/, int K, int m, const double *Pi /*host*/,
                                  const double *delta /*host*/, const double *mean /*host*/,
                                  const double *sd /*host*/, int sd_per_col, uint8_t *states_u8, double *margins,
                                  int *err_flag, void *stream);

/* Per-cell sum and sd (n-1) of the listed columns (cells == NULL: columns 0..n_cells-1); sums / sds may be NULL. */
ICNV_API int icnv_dev_column_stats_f64(const double *X, int64_t G, const int32_t *cells, int64_t n_cells, double *sums,
                                       double *sds, void *stream);

/* Median filter on device-resident data; index lists are host arrays. */
ICNV_API int icnv_dev_median_filter_f64(const double *X, double *Y, int64_t G, int64_t C,
                                        const int32_t *chr_start /*host*/, const int32_t *chr_len /*host*/, int K,
                                        const int32_t *grp_off /*host*/, const int32_t *grp_idx /*host*/, int n_grp,
                                        int window_size, void *stream);

/* icnv_pairwise_dist_f64 on device pointers: columns X + ldx * (d_cells ? d_cells[a] : a), a < n; out: n (n - 1) / 2
 * doubles (device).  Asynchronous on `stream`. */
ICNV_API int icnv_dev_pairwise_dist_f64(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n,
                                        double *out, void *stream);
ICNV_API int icnv_dev_pairwise_dist_rows_f64(const double *x, int64_t n, int64_t ldx, int64_t G, double *out, void *stream);
/* icnv_knn_f64 on device pointers: columns X + ldx * (d_cells ? d_cells[a] : a), a < n (a gene range - one chromosome - is
 * X offset by its first gene, ldx unchanged); idx / dist: n x k column-major (device).  Both kernels are enqueued on
 * `stream`, which is then synchronised once to report non-finite input. */
ICNV_API int icnv_dev_knn_f64(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n, int k,
                              int32_t *idx, double *dist, void *stream);
/* icnv_seurat_snn_f64 on device pointers: columns X + ldx * (d_cells ? d_cells[a] : a), a < n (a chromosome is X offset by
 * its first gene, ldx unchanged).  Synchronises `stream`; the result stays in the library (icnv_seurat_snn_fetch). */
ICNV_API int icnv_dev_seurat_snn_f64(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n,
                                     int n_features, int npcs, int k, int64_t *nnz, void *stream);
/* icnv_hclust_f64 on a device "dist" vector: merge / height (device) as above, no order (icnv_hclust_order on the host
 * copy of merge).  Synchronises the stream once, after filling the matrix, to report non-finite input; the linkage itself
 * is enqueued on `stream`. */
ICNV_API int icnv_dev_hclust_f64(const double *d_dist, int64_t n, int method, int32_t *merge, double *height, void *stream);
/* icnv_random_tree_heights_f64 on device pointers: columns X + ldx * (d_cells ? d_cells[i] : i), i < n; merge / height /
 * perm_max_height (device), no order (icnv_hclust_order on the host copy of merge).  Synchronises `stream` once, after the
 * first wave's distances, to report non-finite input, and once at the end. */
ICNV_API int icnv_dev_random_tree_heights_f64(const double *X, int64_t G, int64_t ldx, const int32_t *d_cells, int64_t n,
                                              int window, int method, int n_perm, uint64_t seed, int32_t *merge,
                                              double *height, double *perm_max_height, void *stream);
/* icnv_zscore_outlier_genes_f64 on device pointers: X is G x (columns) with ld G, d_ref_idx n_ref device indices, outlier
 * G bytes (device).  Synchronises `stream` twice: the per-cell statistics are combined on the host, then the non-finite check. */
ICNV_API int icnv_dev_zscore_outlier_genes_f64(const double *X, int64_t G, const int32_t *d_ref_idx, int64_t n_ref,
                                               uint8_t *outlier, void *stream);
/* icnv_cluster_groups_f64 on device pointers: X (column stride ldx >= G, C columns), d_keep (device; NULL: all genes),
 * grp_off (HOST), d_grp_idx (device), merge / height (device, packed as above), no order (icnv_hclust_order on the host
 * copy of each group's merge).  With a keep list the kept rows of all C columns are gathered once (n_keep x C doubles).
 * Synchronises `stream` once to check the indices, once per wave after its distances (non-finite check) and at the end. */
ICNV_API int icnv_dev_cluster_groups_f64(const double *X, int64_t G, int64_t ldx, int64_t C, const int32_t *d_keep,
                                         int64_t n_keep, const int32_t *grp_off /*host*/, const int32_t *d_grp_idx, int n_grp,
                                         int method, int32_t *merge, double *height, void *stream);
/* icnv_hclust_tri_f64 on a device "dist" vector (left unchanged: the linkage works on its own copy): merge / height
 * (device), no order (icnv_hclust_order on the host copy of merge).  Synchronises `stream` once, after preparing the
 * triangle, to report non-finite input; the linkage itself is enqueued on `stream`. */
ICNV_API int icnv_dev_hclust_tri_f64(const double *d_dist, int64_t n, int method, int32_t *merge, double *height, void *stream);
/* icnv_cluster_cells_f64 on device pointers: X (column stride ldx >= G, C columns), d_keep (device; NULL: all genes),
 * d_cells (device, n columns; NULL: all C columns, n is then ignored; a gene range - one chromosome - is X offset by its
 * first gene with G its length), merge / height (device), no order.  With a keep list the kept rows of all C columns are
 * gathered once (n_keep x C doubles).  Synchronises `stream` to check the indices and the distances. */
ICNV_API int icnv_dev_cluster_cells_f64(const double *X, int64_t G, int64_t ldx, int64_t C, const int32_t *d_keep,
                                        int64_t n_keep, const int32_t *d_cells, int64_t n, int method, int32_t *merge,
                                        double *height, void *stream);
/* icnv_mask_non_de_f64 on device pointers: X (column stride ldx >= G), Y (ldy >= G; may be X, nullable), p_raw / p_adj
 * (G x (n_sub n_ref), nullable); the group lists are HOST arrays.  Synchronises `stream` after each gene tile (non-finite
 * check) and at the end. */
ICNV_API int icnv_dev_mask_non_de_f64(const double *X, int64_t ldx, double *Y, int64_t ldy, int64_t G, int64_t C,
                                      const int32_t *ref_off /*host*/, const int32_t *ref_idx /*host*/, int n_ref,
                                      const int32_t *sub_off /*host*/, const int32_t *sub_idx /*host*/, int n_sub, int test,
                                      double p_thresh, int rule, double mask_val, double jitter_mean, double jitter_sd,
                                      uint64_t seed, double *p_raw, double *p_adj, void *stream);
/* The stages of icnv_dev_mask_non_de_f64 on their own, for a caller that splits the genes over devices or ranks (Engine.
 * mask_non_de_sharded): each rank packs the listed cells it holds for every rank's gene range, the blocks are exchanged
 * (all-to-all), each rank places what it received into slab rows and tests its genes, the p rows are all-gathered, and every
 * rank runs BH on all of them and masks its own cells.  Every stage depends on a gene only through its absolute index and
 * on a cell only through its global list position, so the bytes equal one device's for any split.
 * icnv_dev_de_pack_f64: per destination d, the gene-major block out_d[gl * m + k] = X[gene_lo[d] + gl + ldx * d_cols[k]]
 *   (gene_hi[d] - gene_lo[d] genes x m cells, d_cols on the device, each in [0, C)), the blocks back to back in destination
 *   order; *err_flag |= 1 (device int) on a non-finite value.  Asynchronous on `stream`.
 * icnv_dev_de_place_f64: R holds one gene-major block of n genes x src_m[q] cells per source q, back to back in source order;
 *   d_tags (device, T entries in the same order) is each received cell's global list position (references in group order,
 *   then the subclusters, as icnv_mask_non_de_f64 lists them).  Z[gl * T + d_tags[e]] = the value: the n x T slab rows.
 *   sum(src_m) must be T.  Asynchronous on `stream`.
 * icnv_dev_de_slab_tests_f64: stages (b) and (c) on the slab rows Z (n x T, gene-major) of the absolute genes g0 .. g0 + n:
 *   p of pair s * n_ref + j and gene g0 + gl into p_raw[(s * n_ref + j) * ldp + gl].  Group sizes as the CSR offsets of
 *   icnv_mask_non_de_f64 (HOST arrays; their total must be T).  Z must be finite (the pack or gather reports it).
 *   Synchronises `stream`.
 * icnv_dev_de_bh_mask_f64: BH of every pair over the whole p_raw (rows of G), into p_adj (nullable), then the mask of the C
 *   columns of X into Y (nullable: BH only; may be X).  sub_size[s]: subcluster s's whole list length (the < 5 rule);
 *   ref_idx / sub_off / sub_idx (HOST, 0-based columns of this block): its reference cells and, per subcluster, its cells
 *   (possibly none).  Synchronises `stream`. */
ICNV_API int icnv_dev_de_pack_f64(const double *X, int64_t ldx, const int32_t *d_cols, int64_t m, int n_dst,
                                  const int64_t *gene_lo /*host*/, const int64_t *gene_hi /*host*/, double *out, int *err_flag,
                                  void *stream);
ICNV_API int icnv_dev_de_place_f64(const double *R, int64_t n, int n_src, const int64_t *src_m /*host*/, const int32_t *d_tags,
                                   int64_t T, double *Z, void *stream);
ICNV_API int icnv_dev_de_slab_tests_f64(const double *Z, int64_t T, int64_t g0, int64_t n, const int32_t *ref_off /*host*/,
                                        int n_ref, const int32_t *sub_off /*host*/, int n_sub, int test, double jitter_mean,
                                        double jitter_sd, uint64_t seed, double *p_raw, int64_t ldp, void *stream);
ICNV_API int icnv_dev_de_bh_mask_f64(const double *p_raw, int64_t G, int n_ref, int n_sub, const int32_t *sub_size /*host*/,
                                     double p_thresh, double *p_adj, const double *X, int64_t ldx, double *Y, int64_t ldy,
                                     int64_t C, const int32_t *ref_idx /*host*/, int64_t n_ref_cells,
                                     const int32_t *sub_off /*host*/, const int32_t *sub_idx /*host*/, int rule, double mask_val,
                                     void *stream);
/* icnv_bayesnet_f64 on device pointers: X (column stride ldx >= G), theta, state_counts, loglik (nullable); the region lists,
 * pooled, mu and tau are HOST arrays.  Synchronises `stream` after the log-likelihood pass (non-finite check) and at the end. */
ICNV_API int icnv_dev_bayesnet_f64(const double *X, int64_t ldx, int64_t G, int64_t C, const int32_t *gene_off /*host*/,
                                   const int32_t *gene_idx /*host*/, const int32_t *cell_off /*host*/,
                                   const int32_t *cell_idx /*host*/, const uint8_t *pooled /*host*/, int n_reg, int m,
                                   const double *mu /*host*/, const double *tau /*host*/, int n_chains, int n_burn, int n_keep,
                                   uint64_t seed, double *theta, int32_t *state_counts, double *loglik, void *stream);
/* Region calling on device-resident states (uint8, column stride lds >= G).
 * icnv_dev_state_counts_u8: counts[(k*G + g)*8 + slot] = number of cells of group k (d_cells[h_grp_off[k] ..
 * h_grp_off[k+1]), device) whose state at gene g falls in `slot` (0: unassigned, v+1: state v); integer counts, so
 * ranks holding different cells of a group can add theirs (all-reduce) before icnv_dev_consensus_from_counts.
 * err_flag |= 4 on a byte outside {0..6, 255}.  Synchronises the stream. */
ICNV_API int icnv_dev_state_counts_u8(const uint8_t *S, int64_t G, int64_t lds, const int32_t *d_cells,
                                      const int32_t *h_grp_off /*host*/, int n_grp, uint32_t *d_counts, int *err_flag,
                                      void *stream);
ICNV_API int icnv_dev_consensus_from_counts(const uint32_t *d_counts, int64_t G, int n_grp, uint8_t *d_cons,
                                            void *stream);
ICNV_API int icnv_dev_state_consensus_u8(const uint8_t *S, int64_t G, int64_t lds, const int32_t *d_cells,
                                         const int32_t *h_grp_off /*host*/, int n_grp, uint8_t *d_cons, int *err_flag,
                                         void *stream);
/* Regions of the n_seq sequences d_seqs[:, d_cols ? d_cols[s] : s]; synchronises; records stay in the library. */
ICNV_API int icnv_dev_cnv_regions_u8(const uint8_t *d_seqs, int64_t G, int64_t lds, int64_t n_seq,
                                     const int32_t *d_cols, const int32_t *chr_start /*host*/,
                                     const int32_t *chr_len /*host*/, int K, const double *gene_start /*host*/,
                                     const double *gene_stop /*host*/, int64_t *n_regions /*host*/, void *stream);
/* Device pointers of the last call's records (valid until the next region call); any output may be NULL. */
ICNV_API int icnv_dev_cnv_regions_records(int64_t *n, const int32_t **seq, const int32_t **chr,
                                          const int32_t **first_gene, const int32_t **last_gene,
                                          const int32_t **state, const double **start, const double **end);

/* Gene filters / ingest / outlier clamp on device-resident data (see the host entry points of the same names):
 * per-gene sum and number of values > 0 over the C columns (column stride ldx); row gather Y[i + n_keep*c] =
 * X[keep[i] + ldx*c]; per-cell min / max (NaN skipped); clamp to [lower, upper]. */
ICNV_API int icnv_dev_gene_stats_f64(const double *X, int64_t G, int64_t ldx, int64_t C, double *sums, int32_t *n_pos,
                                     void *stream);
ICNV_API int icnv_dev_gather_rows_f64(const double *X, int64_t ldx, const int32_t *keep, int64_t n_keep, double *Y,
                                      int64_t C, void *stream);
ICNV_API int icnv_dev_column_minmax_f64(const double *X, int64_t G, int64_t C, double *mins, double *maxs, void *stream);
ICNV_API int icnv_dev_clamp_bounds_f64(const double *X, double *Y, int64_t n, double lower, double upper, void *stream);

/* Deterministic synthetic workload of SURVEY section 8(d) written straight into HBM: counter-based
 * generator keyed by (seed, global cell, gene), so any sharding of the cells yields identical data.
 * Fills X (G x n_cells, ld = G) for global cells [cell0, cell0 + n_cells). */
ICNV_API int icnv_dev_synth_f64(double *X, int64_t G, int64_t cell0, int64_t n_cells, int64_t C_total,
                                const int32_t *chr_start /*host*/, const int32_t *chr_len /*host*/, int K,
                                uint64_t seed, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* INFERCNV_B200_H */
