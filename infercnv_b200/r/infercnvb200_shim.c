/*
 * infercnvb200_shim.c - the `.Call()` glue between R and libinfercnv_b200.so.
 *
 * Build on a machine with R:   R CMD SHLIB infercnvb200_shim.c -L<dir> -linfercnv_b200 -I<repo>/include
 * (tests/test_r_shim_compiles.py compile-checks this file against a minimal mock of Rinternals.h,
 *  because R is not installable in the build image.)
 *
 * Every entry: extract plain vectors from the SEXPs, allocate the result with allocMatrix, make ONE
 * call into the C ABI, and turn a non-zero status into an R error AFTER all locals are dead
 * (Rf_error longjmps).  Index vectors arrive 1-based from R and are shifted here.
 */
#include <R.h>
#include <Rinternals.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "infercnv_b200.h"

/* list of integer vectors (1-based) -> CSR (0-based); caller frees *off and *idx */
static int list_to_csr(SEXP groups, int32_t **off, int32_t **idx) {
    int n = Rf_length(groups);
    int64_t total = 0;
    for (int k = 0; k < n; ++k) total += Rf_length(VECTOR_ELT(groups, k));
    *off = (int32_t *)malloc(sizeof(int32_t) * (size_t)(n + 1));
    *idx = (int32_t *)malloc(sizeof(int32_t) * (size_t)(total > 0 ? total : 1));
    if (!*off || !*idx) return -1;
    int32_t pos = 0;
    (*off)[0] = 0;
    for (int k = 0; k < n; ++k) {
        SEXP v = VECTOR_ELT(groups, k);
        const int *p = INTEGER(v);
        for (int i = 0; i < Rf_length(v); ++i) (*idx)[pos++] = p[i] - 1;
        (*off)[k + 1] = pos;
    }
    return n;
}

/* as.integer(gene_order$chr) (rows pre-sorted by chr) -> contiguous ranges */
static int chr_to_ranges(SEXP chr_codes, int32_t **start, int32_t **len) {
    int G = Rf_length(chr_codes);
    const int *c = INTEGER(chr_codes);
    int K = 0;
    for (int g = 0; g < G; ++g)
        if (g == 0 || c[g] != c[g - 1]) ++K;
    *start = (int32_t *)malloc(sizeof(int32_t) * (size_t)(K > 0 ? K : 1));
    *len = (int32_t *)malloc(sizeof(int32_t) * (size_t)(K > 0 ? K : 1));
    if (!*start || !*len) return -1;
    int k = -1;
    for (int g = 0; g < G; ++g) {
        if (g == 0 || c[g] != c[g - 1]) {
            ++k;
            (*start)[k] = g;
            (*len)[k] = 0;
        }
        (*len)[k] += 1;
    }
    return K;
}

static void fail_if(int rc) {
    if (rc != 0) Rf_error("infercnv_b200: %s (status %d)", icnv_last_error(), rc);
}

/* subtract_ref_expr_from_obs: .get_normal_gene_mean_bounds + .subtract_expr (ops.R:1678-1786) */
SEXP icnvR_subtract_ref(SEXP expr, SEXP ref_groups, SEXP inv_log, SEXP use_bounds) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int32_t *off = NULL, *idx = NULL;
    int n_grp = list_to_csr(ref_groups, &off, &idx);
    double *means = (double *)malloc(sizeof(double) * (size_t)(G * (n_grp > 0 ? n_grp : 1)));
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = (n_grp < 0 || !means) ? ICNV_E_NOMEM
                                   : icnv_ref_means_f64(REAL(expr), G, C, off, idx, n_grp, Rf_asLogical(inv_log), means);
    if (rc == 0) rc = icnv_subtract_ref_f64(REAL(expr), REAL(ans), G, C, means, n_grp, Rf_asLogical(use_bounds));
    free(off); free(idx); free(means);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* smooth_by_chromosome (ops.R:2406-2434) */
SEXP icnvR_smooth(SEXP expr, SEXP chr_codes, SEXP window_length) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int32_t *cs = NULL, *cl = NULL;
    int K = chr_to_ranges(chr_codes, &cs, &cl);
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = K < 0 ? ICNV_E_NOMEM : icnv_smooth_f64(REAL(expr), REAL(ans), G, C, cs, cl, K, Rf_asInteger(window_length));
    free(cs); free(cl);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* center_cell_expr_across_chromosome (ops.R:2074-2109) */
SEXP icnvR_center(SEXP expr, SEXP use_median) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = icnv_center_f64(REAL(expr), REAL(ans), G, C, Rf_asLogical(use_median));
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* fused run() steps 4, 8-12, 14 */
SEXP icnvR_smooth_block(SEXP expr, SEXP chr_codes, SEXP ref_groups, SEXP apply_log, SEXP threshold, SEXP window_length,
                        SEXP use_bounds) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int32_t *cs = NULL, *cl = NULL, *off = NULL, *idx = NULL;
    int K = chr_to_ranges(chr_codes, &cs, &cl);
    int n_grp = list_to_csr(ref_groups, &off, &idx);
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = (K < 0 || n_grp < 0) ? ICNV_E_NOMEM
                                  : icnv_smooth_block_f64(REAL(expr), REAL(ans), G, C, cs, cl, K, off, idx, n_grp,
                                                          Rf_asLogical(apply_log), Rf_asReal(threshold),
                                                          Rf_asInteger(window_length), Rf_asLogical(use_bounds));
    free(cs); free(cl); free(off); free(idx);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* fused run() steps 4, 8-12, 14 AND step 17 for analysis_mode = "cells" (per-cell i6 / i3 HMM on the block's output):
 * ONE upload of the matrix, the smoothed matrix and one byte per state back.  Returns list(expr, states). */
SEXP icnvR_smooth_hmm(SEXP expr, SEXP chr_codes, SEXP ref_groups, SEXP apply_log, SEXP threshold, SEXP window_length,
                      SEXP use_bounds, SEXP Pi, SEXP delta, SEXP mean, SEXP sd) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int m = Rf_length(delta);
    int32_t *cs = NULL, *cl = NULL, *off = NULL, *idx = NULL;
    int K = chr_to_ranges(chr_codes, &cs, &cl);
    int n_grp = list_to_csr(ref_groups, &off, &idx);
    uint8_t *st = (uint8_t *)malloc((size_t)(G * C));
    SEXP ans = PROTECT(Rf_allocVector(VECSXP, 2));
    SEXP y = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    SEXP states = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = (K < 0 || n_grp < 0 || !st) ? ICNV_E_NOMEM
                                         : icnv_smooth_hmm_u8_f64(REAL(expr), REAL(y), st, G, C, cs, cl, K, off, idx, n_grp,
                                                                  Rf_asLogical(apply_log), Rf_asReal(threshold),
                                                                  Rf_asInteger(window_length), Rf_asLogical(use_bounds), m, REAL(Pi),
                                                                  REAL(delta), REAL(mean), REAL(sd));
    if (rc == 0) {
        double *out = REAL(states);   /* the reference keeps states as doubles (HMM.R:320) */
        for (int64_t i = 0; i < G * C; ++i) out[i] = (st[i] == 255) ? -1.0 : (double)st[i];
    }
    SET_VECTOR_ELT(ans, 0, y);
    SET_VECTOR_ELT(ans, 1, states);
    free(cs); free(cl); free(off); free(idx); free(st);
    UNPROTECT(3);
    fail_if(rc);
    return ans;
}

/* the i3 counterpart (icnv_smooth_i3_hmm_u8_f64): run() steps 4, 8-12, 14, the i3 model of the reference cells, step 17 per
 * cell and, with median_lists non-NULL, apply_median_filtering (noise_reduction.R:43-113) in one pass.
 * Returns list(expr, states, median_filtered or NULL, c(mu, sigma, mean_delta)). */
SEXP icnvR_smooth_i3_hmm(SEXP expr, SEXP chr_codes, SEXP ref_groups, SEXP apply_log, SEXP threshold, SEXP window_length,
                         SEXP use_bounds, SEXP i3_p_val, SEXP t, SEXP median_lists, SEXP median_window) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int32_t *cs = NULL, *cl = NULL, *off = NULL, *idx = NULL, *moff = NULL, *midx = NULL;
    int K = chr_to_ranges(chr_codes, &cs, &cl);
    int n_grp = list_to_csr(ref_groups, &off, &idx);
    const int filter = !Rf_isNull(median_lists);
    int n_mf = filter ? list_to_csr(median_lists, &moff, &midx) : 0;
    uint8_t *st = (uint8_t *)malloc((size_t)(G * C));
    SEXP ans = PROTECT(Rf_allocVector(VECSXP, 4));
    SEXP y = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    SEXP states = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    SEXP f = PROTECT(filter ? Rf_allocMatrix(REALSXP, (int)G, (int)C) : R_NilValue);
    SEXP model = PROTECT(Rf_allocVector(REALSXP, 3));
    int rc = (K < 0 || n_grp < 0 || n_mf < 0 || !st)
                 ? ICNV_E_NOMEM
                 : icnv_smooth_i3_hmm_u8_f64(REAL(expr), REAL(y), st, filter ? REAL(f) : NULL, G, C, cs, cl, K, off, idx, n_grp,
                                             Rf_asLogical(apply_log), Rf_asReal(threshold), Rf_asInteger(window_length),
                                             Rf_asLogical(use_bounds), Rf_asReal(i3_p_val), Rf_asReal(t), moff, midx, n_mf,
                                             filter ? Rf_asInteger(median_window) : 0, REAL(model));
    if (rc == 0) {
        double *out = REAL(states);   /* the reference keeps states as doubles (i3HMM.R:222) */
        for (int64_t i = 0; i < G * C; ++i) out[i] = (st[i] == 255) ? -1.0 : (double)st[i];
    }
    SET_VECTOR_ELT(ans, 0, y);
    SET_VECTOR_ELT(ans, 1, states);
    SET_VECTOR_ELT(ans, 2, f);
    SET_VECTOR_ELT(ans, 3, model);
    free(cs); free(cl); free(off); free(idx); free(moff); free(midx); free(st);
    UNPROTECT(5);
    fail_if(rc);
    return ans;
}

/* the group-mode twins (icnv_smooth_hmm_groups_u8_f64, icnv_smooth_i3_hmm_groups_u8_f64): run() steps 4, 8-12, 14 and
 * step 17 for analysis_mode "samples" / "subclusters" on the HMM lists hmm_groups.  i6: Pi, delta, mean and sd (m entries
 * per group); i3: i3_p_val and t.  Returns list(expr, states) (i6) or list(expr, states, c(mu, sigma, mean_delta)). */
static SEXP smooth_hmm_groups(SEXP expr, SEXP chr_codes, SEXP ref_groups, SEXP apply_log, SEXP threshold, SEXP window_length,
                              SEXP use_bounds, SEXP hmm_groups, int i3, SEXP Pi, SEXP delta, SEXP mean, SEXP sd, SEXP i3_p_val,
                              SEXP t) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int32_t *cs = NULL, *cl = NULL, *off = NULL, *idx = NULL, *hoff = NULL, *hidx = NULL;
    int K = chr_to_ranges(chr_codes, &cs, &cl);
    int n_grp = list_to_csr(ref_groups, &off, &idx);
    int n_hmm = list_to_csr(hmm_groups, &hoff, &hidx);
    uint8_t *st = (uint8_t *)malloc((size_t)(G * C));
    SEXP ans = PROTECT(Rf_allocVector(VECSXP, i3 ? 3 : 2));
    SEXP y = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    SEXP states = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    SEXP model = PROTECT(Rf_allocVector(REALSXP, 3));
    int rc;
    if (K < 0 || n_grp < 0 || n_hmm < 0 || !st)
        rc = ICNV_E_NOMEM;
    else if (i3)
        rc = icnv_smooth_i3_hmm_groups_u8_f64(REAL(expr), REAL(y), st, G, C, cs, cl, K, off, idx, n_grp, Rf_asLogical(apply_log),
                                              Rf_asReal(threshold), Rf_asInteger(window_length), Rf_asLogical(use_bounds), hoff,
                                              hidx, n_hmm, Rf_asReal(i3_p_val), Rf_asReal(t), REAL(model));
    else
        rc = icnv_smooth_hmm_groups_u8_f64(REAL(expr), REAL(y), st, G, C, cs, cl, K, off, idx, n_grp, Rf_asLogical(apply_log),
                                           Rf_asReal(threshold), Rf_asInteger(window_length), Rf_asLogical(use_bounds), hoff, hidx,
                                           n_hmm, Rf_length(delta), REAL(Pi), REAL(delta), REAL(mean), REAL(sd));
    if (rc == 0) {
        double *out = REAL(states);   /* the reference keeps states as doubles; -1 for cells in no group */
        for (int64_t i = 0; i < G * C; ++i) out[i] = (st[i] == 255) ? -1.0 : (double)st[i];
    }
    SET_VECTOR_ELT(ans, 0, y);
    SET_VECTOR_ELT(ans, 1, states);
    if (i3) SET_VECTOR_ELT(ans, 2, model);
    free(cs); free(cl); free(off); free(idx); free(hoff); free(hidx); free(st);
    UNPROTECT(4);
    fail_if(rc);
    return ans;
}

SEXP icnvR_smooth_hmm_groups(SEXP expr, SEXP chr_codes, SEXP ref_groups, SEXP apply_log, SEXP threshold, SEXP window_length,
                             SEXP use_bounds, SEXP hmm_groups, SEXP Pi, SEXP delta, SEXP mean, SEXP sd) {
    return smooth_hmm_groups(expr, chr_codes, ref_groups, apply_log, threshold, window_length, use_bounds, hmm_groups, 0, Pi,
                             delta, mean, sd, R_NilValue, R_NilValue);
}

SEXP icnvR_smooth_i3_hmm_groups(SEXP expr, SEXP chr_codes, SEXP ref_groups, SEXP apply_log, SEXP threshold,
                                SEXP window_length, SEXP use_bounds, SEXP hmm_groups, SEXP i3_p_val, SEXP t) {
    return smooth_hmm_groups(expr, chr_codes, ref_groups, apply_log, threshold, window_length, use_bounds, hmm_groups, 1,
                             R_NilValue, R_NilValue, R_NilValue, R_NilValue, i3_p_val, t);
}

/* icnv_init_devices: single-process multi-GPU (infercnv::run() is one R process).  ids = NULL: every GPU present. */
SEXP icnvR_init_devices(SEXP ids) {
    int rc = Rf_isNull(ids) ? icnv_init_devices(0, NULL) : icnv_init_devices(Rf_length(ids), INTEGER(ids));
    fail_if(rc);
    return Rf_ScalarInteger(icnv_devices_in_use());
}

/* predict_CNV_via_HMM_on_* / i3HMM_predict_* (HMM.R:284-567, i3HMM.R:180-389): groups = NULL -> per cell */
SEXP icnvR_viterbi(SEXP expr, SEXP chr_codes, SEXP groups, SEXP Pi, SEXP delta, SEXP mean, SEXP sd) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int m = Rf_length(delta);
    int32_t *cs = NULL, *cl = NULL, *off = NULL, *idx = NULL;
    int K = chr_to_ranges(chr_codes, &cs, &cl);
    int n_grp = Rf_isNull(groups) ? 0 : list_to_csr(groups, &off, &idx);
    /* one byte per state over PCIe (255 = cell in no group); the reference keeps states as doubles (HMM.R:320) */
    uint8_t *st = (uint8_t *)malloc((size_t)(G * C));
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = (K < 0 || n_grp < 0 || !st) ? ICNV_E_NOMEM
                                         : icnv_viterbi_u8_f64(REAL(expr), G, C, cs, cl, K, off, idx, n_grp, m, REAL(Pi),
                                                               REAL(delta), REAL(mean), REAL(sd), st, NULL);
    if (rc == 0) {
        double *out = REAL(ans);
        for (int64_t i = 0; i < G * C; ++i) out[i] = (st[i] == 255) ? -1.0 : (double)st[i];
    }
    free(cs); free(cl); free(off); free(idx); free(st);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* apply_median_filtering (noise_reduction.R:43-89) */
SEXP icnvR_median_filter(SEXP expr, SEXP chr_codes, SEXP index_lists, SEXP window_size) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int32_t *cs = NULL, *cl = NULL, *off = NULL, *idx = NULL;
    int K = chr_to_ranges(chr_codes, &cs, &cl);
    int n_grp = list_to_csr(index_lists, &off, &idx);
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = (K < 0 || n_grp < 0) ? ICNV_E_NOMEM
                                  : icnv_median_filter_f64(REAL(expr), REAL(ans), G, C, cs, cl, K, off, idx, n_grp,
                                                           Rf_asInteger(window_size));
    free(cs); free(cl); free(off); free(idx);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* .i3HMM_get_sd_trend_by_num_cells_fit: mu, sigma over the listed cells (i3HMM.R:17-30) */
SEXP icnvR_mean_sd(SEXP expr, SEXP cells) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int n = Rf_length(cells);
    int32_t *idx = (int32_t *)malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
    double mu = 0, sg = 0;
    int rc = ICNV_E_NOMEM;
    if (idx) {
        for (int i = 0; i < n; ++i) idx[i] = INTEGER(cells)[i] - 1;
        rc = icnv_mean_sd_f64(REAL(expr), G, C, idx, n, &mu, &sg);
    }
    free(idx);
    fail_if(rc);
    SEXP ans = PROTECT(Rf_allocVector(REALSXP, 2));
    REAL(ans)[0] = mu;
    REAL(ans)[1] = sg;
    UNPROTECT(1);
    return ans;
}

/* parallelDist(x) (method "euclidean") for x = observations x variables, the t(expr.data[, cells]) every hclust() call site
 * of the reference builds (R/inferCNV_tumor_subclusters.R:191, R/inferCNV_ops.R:1930, ...): the bare "dist" vector, the R
 * closure attaches Size / Labels / class */
SEXP icnvR_pairwise_dist(SEXP x) {
    SEXP dim = Rf_getAttrib(x, R_DimSymbol);
    int64_t n = INTEGER(dim)[0], G = INTEGER(dim)[1];
    SEXP ans = PROTECT(Rf_allocVector(REALSXP, (R_xlen_t)(n * (n - 1) / 2)));
    int rc = icnv_pairwise_dist_rows_f64(REAL(x), n, G, REAL(ans));
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* hclust(d, method) (fastcluster::hclust, an import of infercnv) on a "dist" vector d: method_code as in
 * icnv_hclust_f64 (0 single, 1 complete, 2 average, 3 mcquitty, 4 ward.D, 7 ward.D2).  Returns list(merge (n-1) x 2
 * INTSXP, height REALSXP, order INTSXP); the R closure adds labels / method / call / dist.method and the class. */
SEXP icnvR_hclust(SEXP d, SEXP method_code) {
    R_xlen_t len = Rf_xlength(d);
    int64_t n = (int64_t)((1.0 + sqrt(1.0 + 8.0 * (double)len)) / 2.0 + 0.5);
    if (n * (n - 1) / 2 != (int64_t)len || n < 2) Rf_error("infercnv_b200: not a \"dist\" vector of at least 2 observations");
    SEXP ans = PROTECT(Rf_allocVector(VECSXP, 3));
    SEXP merge = Rf_allocMatrix(INTSXP, (int)(n - 1), 2);
    SET_VECTOR_ELT(ans, 0, merge);
    SEXP height = Rf_allocVector(REALSXP, (R_xlen_t)(n - 1));
    SET_VECTOR_ELT(ans, 1, height);
    SEXP order = Rf_allocVector(INTSXP, (R_xlen_t)n);
    SET_VECTOR_ELT(ans, 2, order);
    int rc = icnv_hclust_f64(REAL(d), n, Rf_asInteger(method_code), INTEGER(merge), REAL(height), INTEGER(order));
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* hclust(d, method) past 65 536 observations: the packed-triangle linkage on R's "dist" vector as it is. */
SEXP icnvR_hclust_tri(SEXP d, SEXP method_code) {
    R_xlen_t len = Rf_xlength(d);
    int64_t n = (int64_t)((1.0 + sqrt(1.0 + 8.0 * (double)len)) / 2.0 + 0.5);
    if (n * (n - 1) / 2 != (int64_t)len || n < 2) Rf_error("infercnv_b200: not a \"dist\" vector of at least 2 observations");
    SEXP ans = PROTECT(Rf_allocVector(VECSXP, 3));
    SEXP merge = Rf_allocMatrix(INTSXP, (int)(n - 1), 2);
    SET_VECTOR_ELT(ans, 0, merge);
    SEXP height = Rf_allocVector(REALSXP, (R_xlen_t)(n - 1));
    SET_VECTOR_ELT(ans, 1, height);
    SEXP order = Rf_allocVector(INTSXP, (R_xlen_t)n);
    SET_VECTOR_ELT(ans, 2, order);
    int rc = icnv_hclust_tri_f64(REAL(d), n, Rf_asInteger(method_code), INTEGER(merge), REAL(height), INTEGER(order));
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* apply(m, 2, caTools::runmean, k = k) per row range - smooth_by_chromosome_runmeans (ops.R:2679-2704) with the ranges the
 * R closure computed (0-based starts, lengths; genes outside them are copied). */
SEXP icnvR_runmean(SEXP expr, SEXP chr_start, SEXP chr_len, SEXP k) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int K = Rf_length(chr_start);
    if (Rf_length(chr_len) != K) Rf_error("infercnv_b200: runmean ranges differ in length");
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = icnv_runmean_f64(REAL(expr), REAL(ans), G, C, (const int32_t *)INTEGER(chr_start),
                              (const int32_t *)INTEGER(chr_len), K, Rf_asInteger(k));
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* smooth_by_chromosome_coordinates (ops.R:2534-2622) with the ranges the R closure computed (0-based starts, lengths) and
 * gene_order's start / stop as doubles, one per row of expr. */
SEXP icnvR_smooth_coordinates(SEXP expr, SEXP chr_start, SEXP chr_len, SEXP gene_start, SEXP gene_stop, SEXP window_length) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int K = Rf_length(chr_start);
    if (Rf_length(chr_len) != K) Rf_error("infercnv_b200: coordinate-smoothing ranges differ in length");
    if (Rf_length(gene_start) != G || Rf_length(gene_stop) != G)
        Rf_error("infercnv_b200: coordinate smoothing needs one start and stop per gene");
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = icnv_smooth_coordinates_f64(REAL(expr), REAL(ans), G, C, (const int32_t *)INTEGER(chr_start),
                                         (const int32_t *)INTEGER(chr_len), K, REAL(gene_start), REAL(gene_stop),
                                         Rf_asReal(window_length));
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* .parameterize_random_cluster_heights_smoothed_trees (random_smoothed_trees.R:217-304) on the clade matrix expr (genes x
 * cells): list(merge, height, order, rand_max_height_dist); the closure builds the "hclust" object.  seed: two whole numbers
 * in [0, 2^31) drawn from R's RNG, combined as hi * 2^32 + lo. */
SEXP icnvR_random_tree_heights(SEXP expr, SEXP window, SEXP method_code, SEXP n_perm, SEXP seed) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], n = INTEGER(dim)[1];
    int np = Rf_asInteger(n_perm);
    if (n < 2 || np < 0 || Rf_length(seed) != 2) Rf_error("infercnv_b200: random trees need 2 cells, n_perm >= 0, two seeds");
    uint64_t sd = ((uint64_t)REAL(seed)[0] << 32) | (uint64_t)REAL(seed)[1];
    SEXP ans = PROTECT(Rf_allocVector(VECSXP, 4));
    SEXP merge = Rf_allocMatrix(INTSXP, (int)(n - 1), 2);
    SET_VECTOR_ELT(ans, 0, merge);
    SEXP height = Rf_allocVector(REALSXP, (R_xlen_t)(n - 1));
    SET_VECTOR_ELT(ans, 1, height);
    SEXP order = Rf_allocVector(INTSXP, (R_xlen_t)n);
    SET_VECTOR_ELT(ans, 2, order);
    SEXP pm = Rf_allocVector(REALSXP, (R_xlen_t)np);
    SET_VECTOR_ELT(ans, 3, pm);
    int rc = icnv_random_tree_heights_f64(REAL(expr), G, n, NULL, n, Rf_asInteger(window), Rf_asInteger(method_code), np, sd,
                                          INTEGER(merge), REAL(height), INTEGER(order), np > 0 ? REAL(pm) : NULL);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* nn2(data, k = k) (RANN::nn2, an import of infercnv) with the query set = the data set, data = observations x variables
 * (.leiden_simple_snn, R/inferCNV_tumor_subclusters.R:725-741).  Returns list(nn.idx n x k INTSXP, 1-based, nn.dists n x k
 * REALSXP); the R closure names the fields. */
SEXP icnvR_knn(SEXP x, SEXP k_) {
    SEXP dim = Rf_getAttrib(x, R_DimSymbol);
    int64_t n = INTEGER(dim)[0], G = INTEGER(dim)[1];
    int k = Rf_asInteger(k_);
    if (k < 1 || (int64_t)k > n) Rf_error("infercnv_b200: nn2() needs 1 <= k <= nrow(data)");
    SEXP ans = PROTECT(Rf_allocVector(VECSXP, 2));
    SEXP idx = Rf_allocMatrix(INTSXP, (int)n, k);
    SET_VECTOR_ELT(ans, 0, idx);
    SEXP dist = Rf_allocMatrix(REALSXP, (int)n, k);
    SET_VECTOR_ELT(ans, 1, dist);
    int rc = icnv_knn_rows_f64(REAL(x), n, G, k, INTEGER(idx), REAL(dist));
    if (rc == 0) {
        int *p = INTEGER(idx);
        for (int64_t e = 0; e < n * (int64_t)k; ++e) p[e] += 1;
    }
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* .leiden_seurat_preprocess_routine's graph (R/inferCNV_tumor_subclusters.R:699-723) on the genes x cells expr: Seurat's
 * infercnv_snn with n_features 2000, npcs 10, k.param = k.  Returns list(p (n + 1, 0-based), i (nnz, 0-based), x (nnz),
 * singular local trend fits); the graph is symmetric, so the CSR arrays are the dgCMatrix's CSC arrays. */
SEXP icnvR_seurat_snn(SEXP expr, SEXP k_) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], n = INTEGER(dim)[1], nnz = 0;
    int k = Rf_asInteger(k_);
    int rc = icnv_seurat_snn_f64(REAL(expr), G, n, NULL, n, 2000, 10, k, &nnz);
    fail_if(rc);
    if (nnz > 2147483647) Rf_error("infercnv_b200: the SNN graph has more entries than a dgCMatrix holds");
    SEXP ans = PROTECT(Rf_allocVector(VECSXP, 4));
    SEXP p = Rf_allocVector(INTSXP, (R_xlen_t)(n + 1));
    SET_VECTOR_ELT(ans, 0, p);
    SEXP i = Rf_allocVector(INTSXP, (R_xlen_t)nnz);
    SET_VECTOR_ELT(ans, 1, i);
    SEXP x = Rf_allocVector(REALSXP, (R_xlen_t)nnz);
    SET_VECTOR_ELT(ans, 2, x);
    int64_t *rp = (int64_t *)malloc(sizeof(int64_t) * (size_t)(n + 1));
    double st[16];
    rc = rp ? icnv_seurat_snn_fetch(rp, INTEGER(i), REAL(x), NULL, NULL, NULL) : -7;
    if (rc == 0) {
        for (int64_t e = 0; e <= n; ++e) INTEGER(p)[e] = (int)rp[e];
        rc = icnv_debug_seurat_snn(st);
    }
    free(rp);
    SET_VECTOR_ELT(ans, 3, Rf_ScalarInteger(rc == 0 ? (int)st[6] : 0));
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* normalize_counts_by_seq_depth (ops.R:3064-3111); normalize_factor NA -> median of colSums */
SEXP icnvR_normalize(SEXP expr, SEXP normalize_factor) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    double nf = Rf_asReal(normalize_factor);
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = icnv_normalize_counts_by_seq_depth_f64(REAL(expr), REAL(ans), G, C, (nf == nf) ? nf : -1.0);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* clear_noise_via_ref_mean_sd (ops.R:2302-2346), noise_logistic = FALSE */
SEXP icnvR_clear_noise(SEXP expr, SEXP cells, SEXP sd_amplifier) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int n = Rf_length(cells);
    int32_t *idx = (int32_t *)malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = ICNV_E_NOMEM;
    if (idx) {
        for (int i = 0; i < n; ++i) idx[i] = INTEGER(cells)[i] - 1;
        rc = icnv_clear_noise_via_ref_mean_sd_f64(REAL(expr), REAL(ans), G, C, idx, n, Rf_asReal(sd_amplifier));
    }
    free(idx);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* get_predicted_CNV_regions (HMM.R:706-764): consensus state per cell group, run-length regions per chromosome and
 * their bounds in one call.  `states` is the numeric state matrix of the HMM object (-1 = unassigned); it crosses
 * PCIe as one byte per entry.  Returns list(seq, chr, first_gene, last_gene, state, start, end), one entry per
 * region in the reference's numbering order, indices 1-based. */
SEXP icnvR_cnv_regions(SEXP states, SEXP chr_codes, SEXP gene_start, SEXP gene_stop, SEXP groups) {
    SEXP dim = Rf_getAttrib(states, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int32_t *cs = NULL, *cl = NULL, *off = NULL, *idx = NULL;
    int K = chr_to_ranges(chr_codes, &cs, &cl);
    int n_grp = list_to_csr(groups, &off, &idx);
    uint8_t *st = (uint8_t *)malloc((size_t)(G * C));
    int64_t n = 0;
    int not_states = 0;
    int rc = (K < 0 || n_grp < 0 || !st) ? ICNV_E_NOMEM : 0;
    if (rc == 0) {
        const double *x = REAL(states);
        for (int64_t i = 0; i < G * C && !not_states; ++i) {
            if (x[i] == -1.0) st[i] = 255;
            else if (x[i] >= 0.0 && x[i] <= 6.0 && x[i] == (double)(int)x[i]) st[i] = (uint8_t)x[i];
            else not_states = 1;            /* not a state matrix: the R wrapper falls back to the reference code */
        }
    }
    if (rc == 0 && !not_states)
        rc = icnv_predicted_cnv_regions_u8(st, G, C, cs, cl, K, REAL(gene_start), REAL(gene_stop), off, idx, n_grp, NULL, &n);
    free(cs); free(cl); free(off); free(idx); free(st);
    if (not_states) Rf_error("infercnv_b200: expr.data does not hold HMM states (-1, 0..6)");
    fail_if(rc);
    SEXP ans = PROTECT(Rf_allocVector(VECSXP, 7));
    SEXP v[7];
    for (int k = 0; k < 7; ++k) {
        v[k] = Rf_allocVector(k < 4 ? INTSXP : REALSXP, (long)n);
        SET_VECTOR_ELT(ans, k, v[k]);
    }
    int32_t *state = (int32_t *)malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
    rc = !state ? ICNV_E_NOMEM
                : icnv_cnv_regions_fetch(n, INTEGER(v[0]), INTEGER(v[1]), INTEGER(v[2]), INTEGER(v[3]), state, REAL(v[5]),
                                         REAL(v[6]));
    if (rc == 0) {
        for (int64_t i = 0; i < n; ++i) {
            for (int k = 0; k < 4; ++k) INTEGER(v[k])[i] += 1;      /* R is 1-based */
            REAL(v[4])[i] = (double)state[i];                      /* states stay numeric, as in @expr.data */
        }
    }
    free(state);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* normalize_counts_by_seq_depth on a dgCMatrix (R/inferCNV.R:158-160 accepts one): @p, @i, @x (0-based, as the
 * Matrix package stores them) -> dense depth-normalised G x C matrix; 12 bytes per stored count over PCIe. */
SEXP icnvR_csc_normalize(SEXP p, SEXP i, SEXP x, SEXP dims, SEXP normalize_factor) {
    int64_t G = INTEGER(dims)[0], C = INTEGER(dims)[1];
    double nf = Rf_asReal(normalize_factor);
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = (Rf_length(p) != C + 1) ? ICNV_E_BAD_ARG
                                     : icnv_csc_normalize_f64(INTEGER(p), INTEGER(i), REAL(x), G, C, NULL, 0,
                                                              (nf == nf) ? nf : -1.0, REAL(ans), NULL);
    UNPROTECT(1);
    if (rc == ICNV_E_BAD_ARG && Rf_length(p) != C + 1) Rf_error("infercnv_b200: @p does not match the matrix dimensions");
    fail_if(rc);
    return ans;
}

/* remove_outliers_norm (ops.R:1969-2056): NA bounds select "average_bound" */
SEXP icnvR_remove_outliers(SEXP expr, SEXP lower_bound, SEXP upper_bound) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = icnv_remove_outliers_norm_f64(REAL(expr), REAL(ans), G, C, Rf_asReal(lower_bound), Rf_asReal(upper_bound), NULL);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* clear_noise (ops.R:2232-2263): cells = reference cells (1-based) or NULL for "all data" */
SEXP icnvR_clear_noise_threshold(SEXP expr, SEXP cells, SEXP threshold, SEXP noise_logistic) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int n = Rf_isNull(cells) ? 0 : Rf_length(cells);
    int32_t *idx = (int32_t *)malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = ICNV_E_NOMEM;
    if (idx) {
        for (int i = 0; i < n; ++i) idx[i] = INTEGER(cells)[i] - 1;
        rc = icnv_clear_noise_f64(REAL(expr), REAL(ans), G, C, idx, n, Rf_asReal(threshold), Rf_asLogical(noise_logistic));
    }
    free(idx);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* predict_CNV_via_HMM_on_tumor_subclusters_per_chr (HMM.R:412-487): groups = the subclusters of all chromosomes, one
 * after the other (list of 1-based integer vectors), chr_grp_off = where each chromosome's subclusters start (0-based
 * offsets into that list, K + 1 entries), sds = m values per subcluster.  The per-chromosome traces and the final
 * per-subcluster consensus (consensus_groups: the tumour subclusters) are both done in the library. */
SEXP icnvR_viterbi_per_chr(SEXP expr, SEXP chr_codes, SEXP groups, SEXP chr_grp_off, SEXP Pi, SEXP delta, SEXP mean, SEXP sds,
                           SEXP consensus_groups) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int m = Rf_length(delta);
    int32_t *cs = NULL, *cl = NULL, *off = NULL, *idx = NULL, *coff = NULL, *cidx = NULL;
    int K = chr_to_ranges(chr_codes, &cs, &cl);
    int n_grp = list_to_csr(groups, &off, &idx);
    int n_cons = list_to_csr(consensus_groups, &coff, &cidx);
    uint8_t *st = (uint8_t *)malloc((size_t)(G * C));
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = (K < 0 || n_grp < 0 || n_cons < 0 || !st || Rf_length(chr_grp_off) != K + 1) ? ICNV_E_NOMEM : 0;
    if (rc == 0)
        rc = icnv_viterbi_per_chr_u8_f64(REAL(expr), G, C, cs, cl, K, INTEGER(chr_grp_off), off, idx, m, REAL(Pi), REAL(delta),
                                         REAL(mean), REAL(sds), st);
    if (rc == 0 && n_cons > 0) rc = icnv_apply_state_consensus_u8(st, G, C, cs, cl, K, coff, cidx, n_cons, st);
    if (rc == 0) {
        double *out = REAL(ans);
        for (int64_t i = 0; i < G * C; ++i) out[i] = st[i] == 255 ? -1.0 : (double)st[i];
    }
    free(cs); free(cl); free(off); free(idx); free(coff); free(cidx); free(st);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* scale_infercnv_expr (ops.R:3174-3186) */
SEXP icnvR_scale(SEXP expr) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    SEXP ans = PROTECT(Rf_allocMatrix(REALSXP, (int)G, (int)C));
    int rc = icnv_scale_infercnv_expr_f64(REAL(expr), REAL(ans), G, C);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* mask_non_DE_genes_basic (R/inferCNV_mask_non_DE.R:28-52): the masked matrix and p_adj (G x n_sub n_ref) of the tested
 * subclusters (lists of 1-based columns, R's loop order) against the reference groups.  test 0 wilcoxon / 1 t, rule
 * 0 any / 1 most / 2 all; seed: two whole numbers in [0, 2^31) drawn from R's RNG, combined as hi * 2^32 + lo. */
SEXP icnvR_mask_non_de(SEXP expr, SEXP ref_groups, SEXP subclusters, SEXP test, SEXP p_thresh, SEXP rule, SEXP center_val,
                       SEXP seed) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    if (Rf_length(seed) != 2) Rf_error("infercnv_b200: the mask needs two seeds");
    uint64_t sd = ((uint64_t)REAL(seed)[0] << 32) | (uint64_t)REAL(seed)[1];
    int32_t *roff = NULL, *ridx = NULL, *soff = NULL, *sidx = NULL;
    int n_ref = list_to_csr(ref_groups, &roff, &ridx), n_sub = list_to_csr(subclusters, &soff, &sidx);
    SEXP ans = PROTECT(Rf_allocVector(VECSXP, 2));
    SEXP y = Rf_allocMatrix(REALSXP, (int)G, (int)C);
    SET_VECTOR_ELT(ans, 0, y);
    SEXP padj = Rf_allocMatrix(REALSXP, (int)G, n_sub > 0 && n_ref > 0 ? n_sub * n_ref : 0);
    SET_VECTOR_ELT(ans, 1, padj);
    int rc = (n_ref < 0 || n_sub < 0) ? ICNV_E_NOMEM
             : icnv_mask_non_de_f64(REAL(expr), REAL(y), G, C, roff, ridx, n_ref, soff, sidx, n_sub, Rf_asInteger(test),
                                    Rf_asReal(p_thresh), Rf_asInteger(rule), Rf_asReal(center_val), 1e-4, 1e-4, sd, NULL,
                                    n_sub > 0 ? REAL(padj) : NULL);
    free(roff); free(ridx); free(soff); free(sidx);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* inferCNVBayesNet's sampling: list(theta per region ((chains x n_keep) x m), cell frequencies per region (m x C')) */
SEXP icnvR_bayesnet(SEXP expr, SEXP genes, SEXP cells, SEXP pooled, SEXP mu, SEXP tau, SEXP n_chains, SEXP n_burn, SEXP n_keep,
                    SEXP seed) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    if (Rf_length(seed) != 2) Rf_error("infercnv_b200: the Bayesian network needs two seeds");
    uint64_t sd = ((uint64_t)REAL(seed)[0] << 32) | (uint64_t)REAL(seed)[1];
    int32_t *goff = NULL, *gidx = NULL, *coff = NULL, *cidx = NULL;
    int n_reg = list_to_csr(genes, &goff, &gidx), n_reg2 = list_to_csr(cells, &coff, &cidx);
    int m = Rf_length(mu), nc = Rf_asInteger(n_chains), nb = Rf_asInteger(n_burn), nk = Rf_asInteger(n_keep);
    int rc = ICNV_OK;
    if (n_reg < 0 || n_reg2 < 0) rc = ICNV_E_NOMEM;
    else if (n_reg != n_reg2 || Rf_length(pooled) != n_reg || Rf_length(tau) != m || m < 2 || m > 8 || nc < 1 || nk < 1)
        rc = ICNV_E_BAD_ARG;
    int64_t n_cols = 0;
    uint8_t *pool = (uint8_t *)calloc((size_t)(n_reg > 0 ? n_reg : 1), 1);
    if (!pool && rc == ICNV_OK) rc = ICNV_E_NOMEM;
    for (int r = 0; rc == ICNV_OK && r < n_reg; ++r) {
        pool[r] = (uint8_t)(INTEGER(pooled)[r] == 1);
        n_cols += pool[r] ? 1 : coff[r + 1] - coff[r];
    }
    const int64_t rows = (int64_t)nc * nk;
    double *theta = rc == ICNV_OK ? (double *)malloc(sizeof(double) * (size_t)(n_reg * rows * m + 1)) : NULL;
    int32_t *counts = rc == ICNV_OK ? (int32_t *)malloc(sizeof(int32_t) * (size_t)(n_cols * m + 1)) : NULL;
    if (rc == ICNV_OK && (!theta || !counts)) rc = ICNV_E_NOMEM;
    if (rc == ICNV_OK)
        rc = icnv_bayesnet_f64(REAL(expr), G, C, goff, gidx, coff, cidx, pool, n_reg, m, REAL(mu), REAL(tau), nc, nb, nk, sd,
                               theta, counts, NULL);
    SEXP ans = PROTECT(Rf_allocVector(VECSXP, 2));
    if (rc == ICNV_OK) {
        SEXP th_l = Rf_allocVector(VECSXP, n_reg);
        SET_VECTOR_ELT(ans, 0, th_l);
        SEXP cp_l = Rf_allocVector(VECSXP, n_reg);
        SET_VECTOR_ELT(ans, 1, cp_l);
        int64_t off = 0;
        for (int r = 0; r < n_reg; ++r) {
            SEXP th = Rf_allocMatrix(REALSXP, (int)rows, m);
            SET_VECTOR_ELT(th_l, r, th);
            memcpy(REAL(th), theta + (int64_t)r * rows * m, sizeof(double) * (size_t)(rows * m));
            const int ncr = pool[r] ? 1 : coff[r + 1] - coff[r];
            SEXP cp = Rf_allocMatrix(REALSXP, m, ncr);
            SET_VECTOR_ELT(cp_l, r, cp);
            for (int64_t i = 0; i < (int64_t)ncr * m; ++i) REAL(cp)[i] = (double)counts[off * m + i] / (double)rows;
            off += ncr;
        }
    }
    free(goff); free(gidx); free(coff); free(cidx); free(pool); free(theta); free(counts);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

/* The z-score gene filter of define_signif_tumor_subclusters (R/inferCNV_tumor_subclusters.R:45-68): a logical vector of
 * nrow(expr), TRUE where mean(abs(z)) >= 0.8 over the reference columns ref (1-based, unlist(reference_grouped_cell_indices)
 * in that order).  The closure takes which() of it. */
SEXP icnvR_zscore_outlier_genes(SEXP expr, SEXP ref) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int n = Rf_length(ref);
    int32_t *idx = (int32_t *)malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
    uint8_t *out = (uint8_t *)malloc((size_t)(G > 0 ? G : 1));
    int rc = ICNV_E_NOMEM;
    if (idx && out) {
        for (int i = 0; i < n; ++i) idx[i] = INTEGER(ref)[i] - 1;
        rc = icnv_zscore_outlier_genes_f64(REAL(expr), G, C, idx, n, out);
    }
    free(idx);
    SEXP ans = R_NilValue;
    if (rc == 0) {
        ans = PROTECT(Rf_allocVector(LGLSXP, (R_xlen_t)G));
        for (int64_t g = 0; g < G; ++g) LOGICAL(ans)[g] = out[g] != 0;
        UNPROTECT(1);
    }
    free(out);
    fail_if(rc);
    return ans;
}

/* hclust(parallelDist(t(expr[keep, g])), method) for every group g of `groups` (a list of 1-based column vectors) in one
 * call: keep is NULL (every gene) or 1-based genes (integer(0): none).  Returns, per group, list(merge, height, order) or NULL
 * for a group of fewer than 2 cells; the closure builds the "hclust" objects. */
SEXP icnvR_cluster_groups(SEXP expr, SEXP keep, SEXP groups, SEXP method_code) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int32_t *off = NULL, *idx = NULL, *kp = NULL, *merge = NULL, *order = NULL;
    double *height = NULL;
    int n_grp = list_to_csr(groups, &off, &idx);
    int64_t rows = 0, n_keep = Rf_isNull(keep) ? 0 : Rf_length(keep);
    int rc = ICNV_E_NOMEM;
    if (n_grp >= 0) {
        for (int k = 0; k < n_grp; ++k) rows += off[k + 1] - off[k] >= 2 ? off[k + 1] - off[k] - 1 : 0;
        kp = (int32_t *)malloc(sizeof(int32_t) * (size_t)(n_keep > 0 ? n_keep : 1));
        merge = (int32_t *)malloc(sizeof(int32_t) * (size_t)(rows > 0 ? 2 * rows : 1));
        height = (double *)malloc(sizeof(double) * (size_t)(rows > 0 ? rows : 1));
        order = (int32_t *)malloc(sizeof(int32_t) * (size_t)(off[n_grp] > 0 ? off[n_grp] : 1));
        if (kp && merge && height && order) {
            for (int64_t i = 0; i < n_keep; ++i) kp[i] = INTEGER(keep)[i] - 1;
            rc = icnv_cluster_groups_f64(REAL(expr), G, C, Rf_isNull(keep) ? NULL : kp, n_keep, off, idx, n_grp,
                                         Rf_asInteger(method_code), merge, height, order);
        }
    }
    SEXP ans = R_NilValue;
    if (rc == 0) {
        ans = PROTECT(Rf_allocVector(VECSXP, n_grp));
        int64_t r = 0;
        for (int k = 0; k < n_grp; ++k) {
            const int64_t n = off[k + 1] - off[k];
            if (n < 2) continue;
            SEXP t = Rf_allocVector(VECSXP, 3);
            SET_VECTOR_ELT(ans, k, t);
            SEXP m = Rf_allocMatrix(INTSXP, (int)(n - 1), 2);
            SET_VECTOR_ELT(t, 0, m);
            memcpy(INTEGER(m), merge + 2 * r, sizeof(int32_t) * 2 * (size_t)(n - 1));
            SEXP h = Rf_allocVector(REALSXP, (R_xlen_t)(n - 1));
            SET_VECTOR_ELT(t, 1, h);
            memcpy(REAL(h), height + r, sizeof(double) * (size_t)(n - 1));
            SEXP o = Rf_allocVector(INTSXP, (R_xlen_t)n);
            SET_VECTOR_ELT(t, 2, o);
            memcpy(INTEGER(o), order + off[k], sizeof(int32_t) * (size_t)n);
            r += n - 1;
        }
        UNPROTECT(1);
    }
    free(off);
    free(idx);
    free(kp);
    free(merge);
    free(height);
    free(order);
    fail_if(rc);
    return ans;
}

SEXP icnvR_available(void) { return Rf_ScalarLogical(icnv_device_count() > 0 && icnv_init(-1) == 0); }

/* hclust(parallelDist(t(expr[keep, cells])), method) for one group of any size that fits the device: keep (1-based rows or
 * NULL = all; integer(0) = none), cells (1-based columns) -> list(merge, height, order). */
SEXP icnvR_cluster_cells(SEXP expr, SEXP keep, SEXP cells, SEXP method_code) {
    SEXP dim = Rf_getAttrib(expr, R_DimSymbol);
    int64_t G = INTEGER(dim)[0], C = INTEGER(dim)[1];
    int64_t n = Rf_length(cells), n_keep = Rf_isNull(keep) ? 0 : Rf_length(keep);
    if (n < 2) Rf_error("infercnv_b200: a tree needs at least 2 cells");
    int32_t *kp = (int32_t *)malloc(sizeof(int32_t) * (size_t)(n_keep > 0 ? n_keep : 1));
    int32_t *cl = (int32_t *)malloc(sizeof(int32_t) * (size_t)n);
    if (!kp || !cl) {
        free(kp);
        free(cl);
        Rf_error("infercnv_b200: out of host memory");
    }
    for (int64_t i = 0; i < n_keep; ++i) kp[i] = INTEGER(keep)[i] - 1;
    for (int64_t i = 0; i < n; ++i) cl[i] = INTEGER(cells)[i] - 1;
    SEXP ans = PROTECT(Rf_allocVector(VECSXP, 3));
    SEXP merge = Rf_allocMatrix(INTSXP, (int)(n - 1), 2);
    SET_VECTOR_ELT(ans, 0, merge);
    SEXP height = Rf_allocVector(REALSXP, (R_xlen_t)(n - 1));
    SET_VECTOR_ELT(ans, 1, height);
    SEXP order = Rf_allocVector(INTSXP, (R_xlen_t)n);
    SET_VECTOR_ELT(ans, 2, order);
    int rc = icnv_cluster_cells_f64(REAL(expr), G, C, Rf_isNull(keep) ? NULL : kp, n_keep, cl, n, Rf_asInteger(method_code),
                                    INTEGER(merge), REAL(height), INTEGER(order));
    free(kp);
    free(cl);
    UNPROTECT(1);
    fail_if(rc);
    return ans;
}

static const R_CallMethodDef call_methods[] = {
    {"icnvR_subtract_ref", (DL_FUNC)&icnvR_subtract_ref, 4}, {"icnvR_smooth", (DL_FUNC)&icnvR_smooth, 3},
    {"icnvR_center", (DL_FUNC)&icnvR_center, 2},             {"icnvR_smooth_block", (DL_FUNC)&icnvR_smooth_block, 7},
    {"icnvR_viterbi", (DL_FUNC)&icnvR_viterbi, 7},           {"icnvR_median_filter", (DL_FUNC)&icnvR_median_filter, 4},
    {"icnvR_mean_sd", (DL_FUNC)&icnvR_mean_sd, 2},           {"icnvR_available", (DL_FUNC)&icnvR_available, 0},
    {"icnvR_normalize", (DL_FUNC)&icnvR_normalize, 2},       {"icnvR_clear_noise", (DL_FUNC)&icnvR_clear_noise, 3},
    {"icnvR_cnv_regions", (DL_FUNC)&icnvR_cnv_regions, 5},   {"icnvR_csc_normalize", (DL_FUNC)&icnvR_csc_normalize, 5},
    {"icnvR_remove_outliers", (DL_FUNC)&icnvR_remove_outliers, 3},
    {"icnvR_viterbi_per_chr", (DL_FUNC)&icnvR_viterbi_per_chr, 9}, {"icnvR_scale", (DL_FUNC)&icnvR_scale, 1},
    {"icnvR_clear_noise_threshold", (DL_FUNC)&icnvR_clear_noise_threshold, 4},
    {"icnvR_smooth_hmm", (DL_FUNC)&icnvR_smooth_hmm, 11},   {"icnvR_init_devices", (DL_FUNC)&icnvR_init_devices, 1},
    {"icnvR_smooth_i3_hmm", (DL_FUNC)&icnvR_smooth_i3_hmm, 11},
    {"icnvR_smooth_hmm_groups", (DL_FUNC)&icnvR_smooth_hmm_groups, 12},
    {"icnvR_smooth_i3_hmm_groups", (DL_FUNC)&icnvR_smooth_i3_hmm_groups, 10},
    {"icnvR_pairwise_dist", (DL_FUNC)&icnvR_pairwise_dist, 1}, {"icnvR_hclust", (DL_FUNC)&icnvR_hclust, 2},
    {"icnvR_knn", (DL_FUNC)&icnvR_knn, 2},
    {"icnvR_runmean", (DL_FUNC)&icnvR_runmean, 4},
    {"icnvR_random_tree_heights", (DL_FUNC)&icnvR_random_tree_heights, 5},
    {"icnvR_mask_non_de", (DL_FUNC)&icnvR_mask_non_de, 8},
    {"icnvR_bayesnet", (DL_FUNC)&icnvR_bayesnet, 10},
    {"icnvR_smooth_coordinates", (DL_FUNC)&icnvR_smooth_coordinates, 6},
    {"icnvR_zscore_outlier_genes", (DL_FUNC)&icnvR_zscore_outlier_genes, 2},
    {"icnvR_cluster_groups", (DL_FUNC)&icnvR_cluster_groups, 4},
    {"icnvR_hclust_tri", (DL_FUNC)&icnvR_hclust_tri, 2},
    {"icnvR_cluster_cells", (DL_FUNC)&icnvR_cluster_cells, 4},
    {"icnvR_seurat_snn", (DL_FUNC)&icnvR_seurat_snn, 2},
    {NULL, NULL, 0}};

void R_init_infercnvb200_shim(DllInfo *dll) {
    R_registerRoutines(dll, NULL, call_methods, NULL, NULL);
    R_useDynamicSymbols(dll, FALSE);
}

void R_unload_infercnvb200_shim(DllInfo *dll) {
    (void)dll;
    icnv_shutdown();
}
