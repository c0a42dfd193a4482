## infercnv_b200.R - drop-in GPU replacements for inferCNV's smoothing + HMM hot path.
##
## Usage (on a box with R, the infercnv package and an H100):
##   R CMD SHLIB infercnvb200_shim.c -I<repo>/include -L<repo>/infercnv_b200 -linfercnv_b200
##   dyn.load("<repo>/infercnv_b200/libinfercnv_b200.so"); dyn.load("infercnvb200_shim.so")
##   source("infercnv_b200.R"); infercnvb200_install()
##   infercnv::run(...)            # unchanged call; steps 8, 10, 11, 12, 17 now run on the GPU
##
## Each replacement has the SAME name and signature as the internal infercnv function it replaces
## (reference file:line in the comments) and keeps a handle to the original, which it calls whenever
## the input is outside the validated envelope (see .icnv_ok) or the library reports an error.
## The S4 object, run() and every other step are untouched.  GPU use can be switched off with
## options(infercnv.b200 = FALSE).

.icnv_env <- new.env()

## STATUS: experimental.  The shim is compile-checked against a mock of Rinternals.h and the same C entry points are
## exercised through ctypes by the repository's GPU tests, but this R layer has not been executed under R yet (no R in the
## build image); see INTEGRATION.md for the check list of a first run.

.icnv_enabled <- function() {
    if (!isTRUE(getOption("infercnv.b200", TRUE))) return(FALSE)
    ok <- .icnv_try(.Call("icnvR_available"), error = function(e) {
        if (is.null(.icnv_env$warned_unavailable)) {     # once per session: a broken GPU install must not be invisible
            .icnv_env$warned_unavailable <- TRUE
            futile.logger::flog.warn(sprintf("infercnv_b200: GPU path unavailable (%s); every step runs the R implementation", conditionMessage(e)))
        }
        FALSE
    })
    if (!isTRUE(ok) && is.null(.icnv_env$warned_unavailable)) {
        .icnv_env$warned_unavailable <- TRUE
        futile.logger::flog.warn("infercnv_b200: no usable CUDA device; every step runs the R implementation")
    }
    isTRUE(ok)
}

## one .Call into the library; an error is LOGGED (never swallowed silently) and turned into NULL = "use the R original"
.icnv_try <- function(expr, what) {
    tryCatch(expr, error = function(e) {
        futile.logger::flog.warn(sprintf("infercnv_b200: %s failed on the GPU (%s); falling back to the R implementation (hours at scale)",
                                         what, conditionMessage(e)))
        NULL
    })
}

## Single-process multi-GPU: infercnv::run() is one R process and its num_threads never reaches this path
## (R/inferCNV_ops.R:388); after this call the library shards the cells of the streaming entry points over the devices.
infercnvb200_init_devices <- function(device_ids = NULL) {
    .Call("icnvR_init_devices", if (is.null(device_ids)) NULL else as.integer(device_ids))
}

## envelope: base dense double matrix without NA/NaN/Inf (the R smoother strips NAs per cell,
## ops.R:2487-2489; expr.data may also be a dgCMatrix, R/inferCNV.R:40)
.icnv_ok <- function(m) {
    is.matrix(m) && is.double(m) && !anyNA(m) && all(is.finite(range(m)))
}

.icnv_chr_codes <- function(infercnv_obj) {
    chr <- infercnv_obj@gene_order[["chr"]]
    codes <- as.integer(factor(chr, levels = unique(chr)))   # rows are pre-sorted by chr (R/inferCNV.R:407-413)
    if (is.unsorted(codes)) return(NULL)
    codes
}

.icnv_ref_groups <- function(infercnv_obj) {
    if (length(infercnv_obj@reference_grouped_cell_indices) > 0) {
        lapply(infercnv_obj@reference_grouped_cell_indices, as.integer)
    } else {                                               # ops.R:1686-1689: proxy group of all observations
        list(proxyNormal = as.integer(unlist(infercnv_obj@observation_grouped_cell_indices)))
    }
}

.icnv_keep_names <- function(new, old) { dimnames(new) <- dimnames(old); new }

## subtract_ref_expr_from_obs, R/inferCNV_ops.R:1678
b200_subtract_ref_expr_from_obs <- function(infercnv_obj, inv_log=FALSE, use_bounds=TRUE) {
    orig <- .icnv_env$orig$subtract_ref_expr_from_obs
    m <- infercnv_obj@expr.data
    if (!.icnv_enabled() || !.icnv_ok(m)) return(orig(infercnv_obj, inv_log=inv_log, use_bounds=use_bounds))
    futile.logger::flog.info(sprintf("::subtract_ref_expr_from_obs:Start inv_log=%s, use_bounds=%s (GPU)", inv_log, use_bounds))
    res <- tryCatch(.Call("icnvR_subtract_ref", m, .icnv_ref_groups(infercnv_obj), inv_log, use_bounds), "available")
    if (is.null(res)) return(orig(infercnv_obj, inv_log=inv_log, use_bounds=use_bounds))
    infercnv_obj@expr.data <- .icnv_keep_names(res, m)
    if (!is.null(infercnv_obj@.hspike)) {
        futile.logger::flog.info("-mirroring for hspike")
        infercnv_obj@.hspike <- b200_subtract_ref_expr_from_obs(infercnv_obj@.hspike, inv_log=inv_log, use_bounds=use_bounds)
    }
    infercnv_obj
}

## smooth_by_chromosome, R/inferCNV_ops.R:2406
b200_smooth_by_chromosome <- function(infercnv_obj, window_length, smooth_ends=TRUE) {
    orig <- .icnv_env$orig$smooth_by_chromosome
    m <- infercnv_obj@expr.data
    codes <- .icnv_chr_codes(infercnv_obj)
    ## even or < 2 windows: the reference's behaviour is accidental / identity - leave it to R
    if (!.icnv_enabled() || !.icnv_ok(m) || is.null(codes) || window_length < 2 || window_length %% 2 == 0)
        return(orig(infercnv_obj, window_length, smooth_ends))
    res <- .icnv_try(.Call("icnvR_smooth", m, codes, as.integer(window_length)), "smooth")
    if (is.null(res)) return(orig(infercnv_obj, window_length, smooth_ends))
    infercnv_obj@expr.data <- .icnv_keep_names(res, m)
    if (!is.null(infercnv_obj@.hspike)) {
        futile.logger::flog.info("-mirroring for hspike")
        infercnv_obj@.hspike <- b200_smooth_by_chromosome(infercnv_obj@.hspike, window_length, smooth_ends)
    }
    infercnv_obj
}

## center_cell_expr_across_chromosome, R/inferCNV_ops.R:2074
b200_center_cell_expr_across_chromosome <- function(infercnv_obj, method="mean") {
    orig <- .icnv_env$orig$center_cell_expr_across_chromosome
    m <- infercnv_obj@expr.data
    if (!.icnv_enabled() || !.icnv_ok(m)) return(orig(infercnv_obj, method))
    futile.logger::flog.info("::center_smooth across chromosomes per cell (GPU)")
    res <- .icnv_try(.Call("icnvR_center", m, identical(method, "median")), "center")
    if (is.null(res)) return(orig(infercnv_obj, method))
    infercnv_obj@expr.data <- .icnv_keep_names(res, m)
    if (!is.null(infercnv_obj@.hspike)) {
        futile.logger::flog.info("-mirroring for hspike")
        infercnv_obj@.hspike <- b200_center_cell_expr_across_chromosome(infercnv_obj@.hspike, method)
    }
    infercnv_obj
}

## Viterbi for a set of (group or cell) sequences; used by the six drivers below
.icnv_hmm <- function(infercnv_obj, HMM_info, groups = NULL, sds = NULL) {
    m <- infercnv_obj@expr.data
    codes <- .icnv_chr_codes(infercnv_obj)
    if (!.icnv_enabled() || !.icnv_ok(m) || is.null(codes)) return(NULL)
    sd <- if (is.null(sds)) HMM_info[["state_emission_params"]]$sd else sds
    res <- .icnv_try(.Call("icnvR_viterbi", m, codes, groups, HMM_info[["state_transitions"]], HMM_info[["delta"]],
                          HMM_info[["state_emission_params"]]$mean, as.double(sd)), "viterbi")
    if (is.null(res)) return(NULL)
    .icnv_keep_names(res, m)
}

## predict_CNV_via_HMM_on_indiv_cells, R/inferCNV_HMM.R:284
b200_predict_CNV_via_HMM_on_indiv_cells <- function(infercnv_obj, cnv_mean_sd=infercnv:::get_spike_dists(infercnv_obj@.hspike), t=1e-6) {
    res <- .icnv_hmm(infercnv_obj, infercnv:::.get_HMM(cnv_mean_sd, t))
    if (is.null(res)) return(.icnv_env$orig$predict_CNV_via_HMM_on_indiv_cells(infercnv_obj, cnv_mean_sd, t))
    infercnv_obj@expr.data <- res
    infercnv_obj
}

## predict_CNV_via_HMM_on_tumor_subclusters, R/inferCNV_HMM.R:345
b200_predict_CNV_via_HMM_on_tumor_subclusters <- function(infercnv_obj,
        cnv_mean_sd=infercnv:::get_spike_dists(infercnv_obj@.hspike),
        cnv_level_to_mean_sd_fit=infercnv:::get_hspike_cnv_mean_sd_trend_by_num_cells_fit(infercnv_obj@.hspike), t=1e-6) {
    orig <- .icnv_env$orig$predict_CNV_via_HMM_on_tumor_subclusters
    if (is.null(infercnv_obj@tumor_subclusters)) return(orig(infercnv_obj, cnv_mean_sd, cnv_level_to_mean_sd_fit, t))
    groups <- lapply(unlist(infercnv_obj@tumor_subclusters[["subclusters"]], recursive=FALSE), as.integer)
    sds <- unlist(lapply(groups, function(g)                       # .get_state_emission_params, HMM.R:586-614
        infercnv:::.get_state_emission_params(length(g), cnv_mean_sd, cnv_level_to_mean_sd_fit)$sd))
    res <- .icnv_hmm(infercnv_obj, infercnv:::.get_HMM(cnv_mean_sd, t), groups, sds)
    if (is.null(res)) return(orig(infercnv_obj, cnv_mean_sd, cnv_level_to_mean_sd_fit, t))
    infercnv_obj@expr.data <- res
    infercnv_obj
}

## predict_CNV_via_HMM_on_whole_tumor_samples, R/inferCNV_HMM.R:509
b200_predict_CNV_via_HMM_on_whole_tumor_samples <- function(infercnv_obj, cluster_by_groups,
        cnv_mean_sd=infercnv:::get_spike_dists(infercnv_obj@.hspike),
        cnv_level_to_mean_sd_fit=infercnv:::get_hspike_cnv_mean_sd_trend_by_num_cells_fit(infercnv_obj@.hspike), t=1e-6) {
    obs <- infercnv_obj@observation_grouped_cell_indices
    ## cluster_by_groups = FALSE: the reference writes c(all_observations = unlist(obs), <list of reference groups>)
    ## (R/inferCNV_HMM.R:531, R/inferCNV_i3HMM.R:356); c() of an integer vector and a list makes every observation cell a
    ## list element of its own, i.e. each observation cell is a one-cell "sample" (rowMeans = the cell, sd for num_cells = 1)
    groups <- c(if (isTRUE(cluster_by_groups)) obs else as.list(unlist(obs, use.names=FALSE)),
                infercnv_obj@reference_grouped_cell_indices)
    groups <- lapply(groups, as.integer)
    sds <- unlist(lapply(groups, function(g)
        infercnv:::.get_state_emission_params(length(g), cnv_mean_sd, cnv_level_to_mean_sd_fit)$sd))
    res <- .icnv_hmm(infercnv_obj, infercnv:::.get_HMM(cnv_mean_sd, t), groups, sds)
    if (is.null(res))
        return(.icnv_env$orig$predict_CNV_via_HMM_on_whole_tumor_samples(infercnv_obj, cluster_by_groups, cnv_mean_sd,
                                                                         cnv_level_to_mean_sd_fit, t))
    infercnv_obj@expr.data <- res
    infercnv_obj
}

## i3HMM_predict_CNV_via_HMM_on_indiv_cells, R/inferCNV_i3HMM.R:180 (sd_trend stays R's; group twins below)
b200_i3HMM_predict_CNV_via_HMM_on_indiv_cells <- function(infercnv_obj, i3_p_val=0.05,
        sd_trend=infercnv:::.i3HMM_get_sd_trend_by_num_cells_fit(infercnv_obj, i3_p_val), t=1e-6, use_KS=TRUE) {
    res <- .icnv_hmm(infercnv_obj, infercnv:::.i3HMM_get_HMM(sd_trend, t=t, i3_p_val=i3_p_val, use_KS=use_KS))
    if (is.null(res)) return(.icnv_env$orig$i3HMM_predict_CNV_via_HMM_on_indiv_cells(infercnv_obj, i3_p_val, sd_trend, t, use_KS))
    infercnv_obj@expr.data <- res
    infercnv_obj
}

## i3HMM_predict_CNV_via_HMM_on_tumor_subclusters, R/inferCNV_i3HMM.R:249: one trace per subcluster on rowMeans, the
## same three-state parameters for every group (no group-size dependent sd in the i3 model)
b200_i3HMM_predict_CNV_via_HMM_on_tumor_subclusters <- function(infercnv_obj, i3_p_val=0.05,
        sd_trend=infercnv:::.i3HMM_get_sd_trend_by_num_cells_fit(infercnv_obj, i3_p_val), t=1e-6, use_KS=TRUE) {
    orig <- .icnv_env$orig$i3HMM_predict_CNV_via_HMM_on_tumor_subclusters
    if (is.null(infercnv_obj@tumor_subclusters)) return(orig(infercnv_obj, i3_p_val, sd_trend, t, use_KS))
    groups <- lapply(unlist(infercnv_obj@tumor_subclusters[["subclusters"]], recursive=FALSE), as.integer)
    HMM_info <- infercnv:::.i3HMM_get_HMM(sd_trend, t=t, i3_p_val=i3_p_val, use_KS=use_KS)
    res <- .icnv_hmm(infercnv_obj, HMM_info, groups, rep(HMM_info[["state_emission_params"]]$sd, length(groups)))
    if (is.null(res)) return(orig(infercnv_obj, i3_p_val, sd_trend, t, use_KS))
    infercnv_obj@expr.data <- res
    infercnv_obj
}

## i3HMM_predict_CNV_via_HMM_on_whole_tumor_samples, R/inferCNV_i3HMM.R:332
b200_i3HMM_predict_CNV_via_HMM_on_whole_tumor_samples <- function(infercnv_obj, cluster_by_groups, i3_p_val=0.05,
        sd_trend=infercnv:::.i3HMM_get_sd_trend_by_num_cells_fit(infercnv_obj, i3_p_val), t=1e-6, use_KS=TRUE) {
    obs <- infercnv_obj@observation_grouped_cell_indices
    ## cluster_by_groups = FALSE: the reference writes c(all_observations = unlist(obs), <list of reference groups>)
    ## (R/inferCNV_HMM.R:531, R/inferCNV_i3HMM.R:356); c() of an integer vector and a list makes every observation cell a
    ## list element of its own, i.e. each observation cell is a one-cell "sample" (rowMeans = the cell, sd for num_cells = 1)
    groups <- c(if (isTRUE(cluster_by_groups)) obs else as.list(unlist(obs, use.names=FALSE)),
                infercnv_obj@reference_grouped_cell_indices)
    groups <- lapply(groups, as.integer)
    HMM_info <- infercnv:::.i3HMM_get_HMM(sd_trend, t=t, i3_p_val=i3_p_val, use_KS=use_KS)
    res <- .icnv_hmm(infercnv_obj, HMM_info, groups, rep(HMM_info[["state_emission_params"]]$sd, length(groups)))
    if (is.null(res))
        return(.icnv_env$orig$i3HMM_predict_CNV_via_HMM_on_whole_tumor_samples(infercnv_obj, cluster_by_groups, i3_p_val,
                                                                               sd_trend, t, use_KS))
    infercnv_obj@expr.data <- res
    infercnv_obj
}

## apply_median_filtering, R/noise_reduction.R:43 (exported)
b200_apply_median_filtering <- function(infercnv_obj, window_size=7, on_observations=TRUE, on_references=TRUE) {
    orig <- .icnv_env$orig$apply_median_filtering
    m <- infercnv_obj@expr.data
    codes <- .icnv_chr_codes(infercnv_obj)
    if (!.icnv_enabled() || !.icnv_ok(m) || is.null(codes) || window_size %% 2 != 1 || window_size < 3)
        return(orig(infercnv_obj, window_size, on_observations, on_references))
    lists <- list()
    if (on_observations) for (tt in names(infercnv_obj@observation_grouped_cell_indices))
        lists <- c(lists, lapply(infercnv_obj@tumor_subclusters[["subclusters"]][[tt]], as.integer))
    if (on_references) lists <- c(lists, lapply(infercnv_obj@reference_grouped_cell_indices, as.integer))
    res <- .icnv_try(.Call("icnvR_median_filter", m, codes, lists, as.integer(window_size)), "median_filter")
    if (is.null(res)) return(orig(infercnv_obj, window_size, on_observations, on_references))
    infercnv_obj@expr.data <- .icnv_keep_names(res, m)
    infercnv_obj
}

## normalize_counts_by_seq_depth, R/inferCNV_ops.R:3064
b200_normalize_counts_by_seq_depth <- function(infercnv_obj, normalize_factor=NA) {
    m <- infercnv_obj@expr.data
    if (.icnv_enabled() && methods::is(m, "dgCMatrix") && !anyNA(m@x)) {
        ## sparse counts (R/inferCNV.R:158-160): the compressed columns cross PCIe, the dense normalised matrix comes back
        res <- .icnv_try(.Call("icnvR_csc_normalize", m@p, m@i, as.double(m@x), dim(m), as.double(normalize_factor)), "csc_normalize")
        if (!is.null(res)) {
            futile.logger::flog.info("normalizing counts matrix by depth (GPU, sparse input)")
            infercnv_obj@expr.data <- .icnv_keep_names(res, m)
            return(infercnv_obj)
        }
    }
    if (!.icnv_enabled() || !.icnv_ok(m)) return(.icnv_env$orig$normalize_counts_by_seq_depth(infercnv_obj, normalize_factor))
    res <- .icnv_try(.Call("icnvR_normalize", m, as.double(normalize_factor)), "normalize")
    if (is.null(res)) return(.icnv_env$orig$normalize_counts_by_seq_depth(infercnv_obj, normalize_factor))
    infercnv_obj@expr.data <- .icnv_keep_names(res, m)
    infercnv_obj
}

## clear_noise_via_ref_mean_sd, R/inferCNV_ops.R:2302 (noise_logistic=TRUE stays in R)
b200_clear_noise_via_ref_mean_sd <- function(infercnv_obj, sd_amplifier=1.5, noise_logistic=FALSE) {
    orig <- .icnv_env$orig$clear_noise_via_ref_mean_sd
    m <- infercnv_obj@expr.data
    if (!.icnv_enabled() || !.icnv_ok(m) || isTRUE(noise_logistic)) return(orig(infercnv_obj, sd_amplifier, noise_logistic))
    cells <- if (length(infercnv_obj@reference_grouped_cell_indices) > 0)
        unlist(infercnv_obj@reference_grouped_cell_indices) else unlist(infercnv_obj@observation_grouped_cell_indices)
    res <- .icnv_try(.Call("icnvR_clear_noise", m, as.integer(cells), as.double(sd_amplifier)), "clear_noise")
    if (is.null(res)) return(orig(infercnv_obj, sd_amplifier, noise_logistic))
    infercnv_obj@expr.data <- .icnv_keep_names(res, m)
    infercnv_obj
}

## predict_CNV_via_HMM_on_tumor_subclusters_per_chr, R/inferCNV_HMM.R:412 (Leiden + per_chr_hmm_subclusters)
b200_predict_CNV_via_HMM_on_tumor_subclusters_per_chr <- function(infercnv_obj, subclusters_per_chr,
        cnv_mean_sd=infercnv:::get_spike_dists(infercnv_obj@.hspike),
        cnv_level_to_mean_sd_fit=infercnv:::get_hspike_cnv_mean_sd_trend_by_num_cells_fit(infercnv_obj@.hspike), t=1e-6) {
    orig <- .icnv_env$orig$predict_CNV_via_HMM_on_tumor_subclusters_per_chr
    m <- infercnv_obj@expr.data
    codes <- .icnv_chr_codes(infercnv_obj)
    if (is.null(subclusters_per_chr) || !.icnv_enabled() || !.icnv_ok(m) || is.null(codes))
        return(orig(infercnv_obj, subclusters_per_chr, cnv_mean_sd, cnv_level_to_mean_sd_fit, t))
    futile.logger::flog.info("predict_CNV_via_HMM_on_tumor_subclusters_per_chr (GPU)")
    chrs <- unique(infercnv_obj@gene_order$chr)
    per <- lapply(chrs, function(chr) lapply(subclusters_per_chr[[chr]], as.integer))
    flat <- unlist(per, recursive=FALSE)
    sds <- unlist(lapply(flat, function(g)
        infercnv:::.get_state_emission_params(length(g), cnv_mean_sd, cnv_level_to_mean_sd_fit)$sd))
    HMM_info <- infercnv:::.get_HMM(cnv_mean_sd, t)
    tumor_subclusters <- lapply(unlist(infercnv_obj@tumor_subclusters[["subclusters"]], recursive=FALSE), as.integer)
    res <- .icnv_try(.Call("icnvR_viterbi_per_chr", m, codes, flat, as.integer(cumsum(c(0L, lengths(per)))),
                          HMM_info[["state_transitions"]], HMM_info[["delta"]], HMM_info[["state_emission_params"]]$mean,
                          as.double(sds), tumor_subclusters), "viterbi_per_chr")
    if (is.null(res)) return(orig(infercnv_obj, subclusters_per_chr, cnv_mean_sd, cnv_level_to_mean_sd_fit, t))
    infercnv_obj@expr.data <- .icnv_keep_names(res, m)
    infercnv_obj
}

## scale_infercnv_expr, R/inferCNV_ops.R:3174 (run() step 5 when scale_data = TRUE)
b200_scale_infercnv_expr <- function(infercnv_obj) {
    orig <- .icnv_env$orig$scale_infercnv_expr
    m <- infercnv_obj@expr.data
    if (!.icnv_enabled() || !.icnv_ok(m)) return(orig(infercnv_obj))
    futile.logger::flog.info("-scaling expr data (GPU)")
    res <- .icnv_try(.Call("icnvR_scale", m), "scale")
    if (is.null(res)) return(orig(infercnv_obj))
    infercnv_obj@expr.data <- .icnv_keep_names(res, m)
    if (!is.null(infercnv_obj@.hspike)) {
        futile.logger::flog.info("-mirroring for hspike")
        infercnv_obj@.hspike <- b200_scale_infercnv_expr(infercnv_obj@.hspike)
    }
    infercnv_obj
}

## remove_outliers_norm, R/inferCNV_ops.R:1969 (run() step 16)
b200_remove_outliers_norm <- function(infercnv_obj, out_method="average_bound", lower_bound=NA, upper_bound=NA) {
    orig <- .icnv_env$orig$remove_outliers_norm
    m <- infercnv_obj@expr.data
    hard <- !is.na(lower_bound) & !is.na(upper_bound)
    ## anything but hard bounds / "average_bound" ends in the reference's stop(991) / stop(992): leave it to R
    if (!.icnv_enabled() || !.icnv_ok(m) || !(hard || identical(out_method, "average_bound")))
        return(orig(infercnv_obj, out_method, lower_bound, upper_bound))
    futile.logger::flog.info(paste("::remove_outlier_norm:Start (GPU)", "out_method:", out_method, "lower_bound:", lower_bound,
                                   "upper_bound:", upper_bound))
    res <- .icnv_try(.Call("icnvR_remove_outliers", m, as.double(if (hard) lower_bound else NA),
                          as.double(if (hard) upper_bound else NA)), "remove_outliers")
    if (is.null(res)) return(orig(infercnv_obj, out_method, lower_bound, upper_bound))
    infercnv_obj@expr.data <- .icnv_keep_names(res, m)
    if (!is.null(infercnv_obj@.hspike)) {
        futile.logger::flog.info("-mirroring for hspike")
        infercnv_obj@.hspike <- b200_remove_outliers_norm(infercnv_obj@.hspike, out_method, lower_bound, upper_bound)
    }
    infercnv_obj
}

## clear_noise, R/inferCNV_ops.R:2232 (run() step 22 with a numeric noise_filter)
b200_clear_noise <- function(infercnv_obj, threshold, noise_logistic=FALSE) {
    orig <- .icnv_env$orig$clear_noise
    m <- infercnv_obj@expr.data
    if (!.icnv_enabled() || !.icnv_ok(m) || threshold == 0) return(orig(infercnv_obj, threshold, noise_logistic))
    cells <- if (length(infercnv_obj@reference_grouped_cell_indices) > 0)
        as.integer(unlist(infercnv_obj@reference_grouped_cell_indices)) else NULL
    res <- .icnv_try(.Call("icnvR_clear_noise_threshold", m, cells, as.double(threshold), isTRUE(noise_logistic)), "clear_noise_threshold")
    if (is.null(res)) return(orig(infercnv_obj, threshold, noise_logistic))
    infercnv_obj@expr.data <- .icnv_keep_names(res, m)
    infercnv_obj
}

## get_predicted_CNV_regions, R/inferCNV_HMM.R:706-764: consensus state per cell group, run-length regions per
## chromosome and their bounds from ONE library call; the returned list has the reference's shape
## (cell_group_name, cells, gene_regions = named list of per-gene data.frames, cnv_ranges = data.frame), so
## generate_cnv_region_reports (HMM.R:790-869) and everything downstream of its files run unchanged.
b200_get_predicted_CNV_regions <- function(infercnv_obj, by=c("consensus", "subcluster", "cell")) {
    by <- match.arg(by)
    orig <- .icnv_env$orig$get_predicted_CNV_regions
    m <- infercnv_obj@expr.data
    codes <- .icnv_chr_codes(infercnv_obj)
    go <- infercnv_obj@gene_order
    if (!.icnv_enabled() || !.icnv_ok(m) || is.null(codes) || anyNA(go$start) || anyNA(go$stop)) return(orig(infercnv_obj, by))
    futile.logger::flog.info(sprintf("get_predicted_CNV_regions(%s) (GPU)", by))
    if (is.null(infercnv_obj@tumor_subclusters)) {
        futile.logger::flog.warn("get_predicted_CNV_regions() - no subclusters defined, resetting reporting mode to consensus")
        by <- "consensus"
    }
    if (by == "consensus") {                                                      # HMM.R:721-723
        cell_groups <- c(infercnv_obj@reference_grouped_cell_indices, infercnv_obj@observation_grouped_cell_indices)
    } else if (by == "subcluster") {                                              # HMM.R:724-725
        cell_groups <- unlist(infercnv_obj@tumor_subclusters[["subclusters"]], recursive=FALSE)
    } else {                                                                      # HMM.R:726-729
        cells <- c(unlist(infercnv_obj@reference_grouped_cell_indices, use.names=FALSE),
                   unlist(infercnv_obj@observation_grouped_cell_indices, use.names=FALSE))
        cell_groups <- as.list(cells)
        names(cell_groups) <- colnames(m)[cells]
    }
    res <- .icnv_try(.Call("icnvR_cnv_regions", m, codes, as.double(go$start), as.double(go$stop),
                          lapply(cell_groups, as.integer)), "cnv_regions")
    if (is.null(res)) return(orig(infercnv_obj, by))
    names(res) <- c("seq", "chr", "first_gene", "last_gene", "state", "start", "end")
    chr_levels <- unique(go$chr)                       # order of appearance = the order of the chromosome ranges
    gene_names <- rownames(go)
    cnv_name <- sprintf("%s-region_%d", as.character(chr_levels[res$chr]), seq_along(res$seq))   # running counter, :758
    if (is.integer(go$start) && is.integer(go$stop)) { res$start <- as.integer(res$start); res$end <- as.integer(res$end) }
    by_group <- split(seq_along(res$seq), factor(res$seq, levels = seq_along(cell_groups)))
    lapply(seq_along(cell_groups), function(k) {
        sel <- by_group[[k]]
        futile.logger::flog.info(sprintf("-processing cell_group_name: %s, size: %d", names(cell_groups)[k], length(cell_groups[[k]])))
        gene_regions <- lapply(sel, function(i) {
            g <- res$first_gene[i]:res$last_gene[i]
            data.frame(state = res$state[i], gene = gene_names[g], chr = go$chr[g], start = go$start[g], end = go$stop[g])
        })
        names(gene_regions) <- cnv_name[sel]
        list(cell_group_name = names(cell_groups)[k],
             cells = colnames(m)[cell_groups[[k]]],
             gene_regions = gene_regions,
             cnv_ranges = data.frame(cnv_name = cnv_name[sel], state = res$state[sel], chr = chr_levels[res$chr[sel]],
                                     start = res$start[sel], end = res$end[sel]))
    })
}

## run() steps 4, 8 .. 12, 14 (and step 17 for analysis_mode = "cells") as ONE library call: one upload of the matrix instead
## of four round trips through the per-step closures above.  infercnv::run() itself calls the steps one by one
## (R/inferCNV_ops.R:771, 865, 911, 952, 1031), so this is for callers that drive the steps themselves, or for a maintainer's
## three-line change in run() (INTEGRATION.md, "fused block").  Input: the object after step 3 (depth-normalised counts, before
## log2) when apply_log = TRUE, after step 4 otherwise; use_bounds / max_centered_threshold / window_length as in run().
## HMM_info (optional): the list .get_HMM() returns (i6, a fixed model) -> per-cell states are predicted on the block's output
## in the same pass.  An i3 model cannot be passed in: .i3HMM_get_HMM() is built from this block's own output (mu and sigma
## of the reference cells after step 14).  For i3 leave HMM_info NULL and set i3_p_val (t and use_KS as in run()): the
## library fixes the model from the reference cells inside the pass.  median_filter_window (optional, i3 path): also
## apply_median_filtering(window_size = median_filter_window) on the block's output, over the lists
## b200_apply_median_filtering builds from THIS object: its tumor_subclusters and its reference groups.  run() defines
## tumor_subclusters only at step 15, after the block, so on an object straight from step 3 they are absent and the
## observation cells come back unfiltered (copied, as apply_median_filtering itself leaves them on that object); a caller
## who wants run()'s step-22 result sets tumor_subclusters first (with partition_method = "none": one subcluster per
## observation group).  use_KS = TRUE needs R's KS delta before the HMM: NULL is returned.
## Returns list(infercnv_obj = <after step 14>, hmm_obj = <states object or NULL>), on the i3 path also median_obj (the
## median-filtered object or NULL) and sd_trend (.i3HMM_get_sd_trend_by_num_cells_fit's list); NULL when the input is outside
## the GPU path's envelope (the caller then runs the R steps).
## analysis_mode = "samples" or "subclusters" (cluster_by_groups and tumor_subcluster_partition_method as in run()) runs
## step 17 in group mode instead: i6 when i3_p_val is NULL (HMM_info is not read: the model and every group's sds come from
## the smoothed hspike, as predict_CNV_via_HMM_on_whole_tumor_samples / _on_tumor_subclusters build them), i3 otherwise.
## "subclusters" needs the random_trees partition, which run() makes at step 7, before the block; without subclusters on the
## object the groups are the whole samples, as in R.  Leiden and the other partitions are made from the block's output: NULL.
## The group-mode call has no median filter (median_obj is NULL; run b200_apply_median_filtering on infercnv_obj).
infercnvb200_run_smooth_block <- function(infercnv_obj, window_length=101, max_centered_threshold=3, use_bounds=TRUE,
                                          apply_log=TRUE, HMM_info=NULL, i3_p_val=NULL, t=1e-6, use_KS=FALSE,
                                          median_filter_window=NULL, analysis_mode="cells", cluster_by_groups=TRUE,
                                          tumor_subcluster_partition_method="random_trees") {
    m <- infercnv_obj@expr.data
    codes <- .icnv_chr_codes(infercnv_obj)
    i3 <- is.null(HMM_info) && !is.null(i3_p_val)
    if (!.icnv_enabled() || !.icnv_ok(m) || is.null(codes) || window_length < 2 || window_length %% 2 == 0 ||
        is.na(max_centered_threshold) || !is.numeric(max_centered_threshold)) return(NULL)
    if (i3 && (isTRUE(use_KS) || !is.numeric(i3_p_val) || !(i3_p_val > 0 && i3_p_val < 1) ||
               (!is.null(median_filter_window) && (median_filter_window %% 2 != 1 || median_filter_window < 3)))) return(NULL)
    futile.logger::flog.info(sprintf("::smooth block (steps 4, 8-12, 14%s) in one pass (GPU)",
                                     if (i3) paste0(" + i3 model + per-cell HMM", if (is.null(median_filter_window)) "" else " + median filter")
                                     else if (is.null(HMM_info)) "" else " + per-cell HMM"))
    refs <- .icnv_ref_groups(infercnv_obj)
    if (!identical(analysis_mode, "cells")) {
        if (!(analysis_mode %in% c("samples", "subclusters")) || (!i3 && is.null(infercnv_obj@.hspike)) ||
            (analysis_mode == "subclusters" && !identical(tumor_subcluster_partition_method, "random_trees"))) return(NULL)
        return(.icnv_smooth_block_groups(infercnv_obj, m, codes, refs, window_length, max_centered_threshold, use_bounds,
                                         apply_log, i3, i3_p_val, t, analysis_mode, cluster_by_groups))
    }
    hmm_obj <- NULL
    median_obj <- NULL
    sd_trend <- NULL
    if (i3) {
        lists <- NULL
        if (!is.null(median_filter_window)) {   # as b200_apply_median_filtering builds them
            lists <- list()
            for (tt in names(infercnv_obj@observation_grouped_cell_indices))
                lists <- c(lists, lapply(infercnv_obj@tumor_subclusters[["subclusters"]][[tt]], as.integer))
            lists <- c(lists, lapply(infercnv_obj@reference_grouped_cell_indices, as.integer))
        }
        res <- .icnv_try(.Call("icnvR_smooth_i3_hmm", m, codes, refs, isTRUE(apply_log), as.double(max_centered_threshold),
                               as.integer(window_length), isTRUE(use_bounds), as.double(i3_p_val), as.double(t), lists,
                               as.integer(if (is.null(median_filter_window)) 7L else median_filter_window)), "smooth_i3_hmm")
        if (is.null(res)) return(NULL)
        infercnv_obj@expr.data <- .icnv_keep_names(res[[1]], m)
        hmm_obj <- infercnv_obj
        hmm_obj@expr.data <- .icnv_keep_names(res[[2]], m)
        if (!is.null(res[[3]])) {
            median_obj <- infercnv_obj
            median_obj@expr.data <- .icnv_keep_names(res[[3]], m)
        }
        mu <- res[[4]][1]; sigma <- res[[4]][2]; mean_delta <- res[[4]][3]
        message("mean_delta: ", mean_delta, ", at sigma: ", sigma, ", and pval: ", i3_p_val)
        ## the reference draws the KS delta even with use_KS = FALSE (rnorm + ks.test, i3HMM.R:68); drawing it here keeps R's
        ## random stream where every later RNG-dependent step expects it
        KS_delta <- infercnv:::get_HoneyBADGER_setGexpDev(gexp.sd=sigma, alpha=i3_p_val, k_cells=length(unlist(refs)))
        message("KS_delta: ", KS_delta, ", at sigma: ", sigma, ", and pval: ", i3_p_val)
        sd_trend <- list(mu=mu, sigma=sigma, mean_delta=mean_delta, KS_delta=KS_delta)
    } else if (is.null(HMM_info)) {
        res <- .icnv_try(.Call("icnvR_smooth_block", m, codes, refs, isTRUE(apply_log), as.double(max_centered_threshold),
                               as.integer(window_length), isTRUE(use_bounds)), "smooth_block")
        if (is.null(res)) return(NULL)
        infercnv_obj@expr.data <- .icnv_keep_names(res, m)
    } else {
        res <- .icnv_try(.Call("icnvR_smooth_hmm", m, codes, refs, isTRUE(apply_log), as.double(max_centered_threshold),
                               as.integer(window_length), isTRUE(use_bounds), HMM_info[["state_transitions"]], HMM_info[["delta"]],
                               HMM_info[["state_emission_params"]]$mean, as.double(HMM_info[["state_emission_params"]]$sd)),
                         "smooth_hmm")
        if (is.null(res)) return(NULL)
        infercnv_obj@expr.data <- .icnv_keep_names(res[[1]], m)
        hmm_obj <- infercnv_obj
        hmm_obj@expr.data <- .icnv_keep_names(res[[2]], m)
    }
    if (!is.null(infercnv_obj@.hspike)) {
        futile.logger::flog.info("-mirroring for hspike")
        h <- infercnvb200_run_smooth_block(infercnv_obj@.hspike, window_length, max_centered_threshold, use_bounds, apply_log, NULL)
        if (is.null(h)) return(NULL)
        infercnv_obj@.hspike <- h$infercnv_obj
    }
    if (i3) return(list(infercnv_obj = infercnv_obj, hmm_obj = hmm_obj, median_obj = median_obj, sd_trend = sd_trend))
    list(infercnv_obj = infercnv_obj, hmm_obj = hmm_obj)
}

## The HMM lists of predict_CNV_via_HMM_on_tumor_subclusters (unlist(tumor_subclusters$subclusters)) and
## predict_CNV_via_HMM_on_whole_tumor_samples (observation groups - one cell each when cluster_by_groups is FALSE - then the
## reference groups), R/inferCNV_HMM.R:345-567.
.icnv_hmm_groups <- function(infercnv_obj, analysis_mode, cluster_by_groups) {
    if (analysis_mode == "subclusters" && !is.null(infercnv_obj@tumor_subclusters))
        return(lapply(unlist(infercnv_obj@tumor_subclusters[["subclusters"]], recursive=FALSE), as.integer))
    if (analysis_mode == "subclusters") cluster_by_groups <- TRUE
    obs <- if (isTRUE(cluster_by_groups)) infercnv_obj@observation_grouped_cell_indices
           else as.list(unlist(infercnv_obj@observation_grouped_cell_indices))
    lapply(c(obs, infercnv_obj@reference_grouped_cell_indices), as.integer)
}

## infercnvb200_run_smooth_block's group-mode path.  The hspike is smoothed first (its own small call), because the i6 sds
## are fitted on the smoothed hspike: get_spike_dists, get_hspike_cnv_mean_sd_trend_by_num_cells_fit (which draws from R's
## RNG), .get_HMM and .get_state_emission_params run here in the order the reference's drivers evaluate them at step 17 -
## nothing between steps 14 and 17 draws in these modes - and the fused call follows.  The i3 path draws the KS delta as
## the per-cell path does.
.icnv_smooth_block_groups <- function(infercnv_obj, m, codes, refs, window_length, max_centered_threshold, use_bounds,
                                      apply_log, i3, i3_p_val, t, analysis_mode, cluster_by_groups) {
    futile.logger::flog.info(sprintf("::smooth block (steps 4, 8-12, 14) + %s HMM on %s in one pass (GPU)",
                                     if (i3) "i3" else "i6", analysis_mode))
    hmm_groups <- .icnv_hmm_groups(infercnv_obj, analysis_mode, cluster_by_groups)
    if (!is.null(infercnv_obj@.hspike)) {
        futile.logger::flog.info("-mirroring for hspike")
        h <- infercnvb200_run_smooth_block(infercnv_obj@.hspike, window_length, max_centered_threshold, use_bounds, apply_log, NULL)
        if (is.null(h)) return(NULL)
        infercnv_obj@.hspike <- h$infercnv_obj
    }
    sd_trend <- NULL
    if (i3) {
        res <- .icnv_try(.Call("icnvR_smooth_i3_hmm_groups", m, codes, refs, isTRUE(apply_log), as.double(max_centered_threshold),
                               as.integer(window_length), isTRUE(use_bounds), hmm_groups, as.double(i3_p_val), as.double(t)),
                         "smooth_i3_hmm_groups")
        if (is.null(res)) return(NULL)
        mu <- res[[3]][1]; sigma <- res[[3]][2]; mean_delta <- res[[3]][3]
        message("mean_delta: ", mean_delta, ", at sigma: ", sigma, ", and pval: ", i3_p_val)
        KS_delta <- infercnv:::get_HoneyBADGER_setGexpDev(gexp.sd=sigma, alpha=i3_p_val, k_cells=length(unlist(refs)))
        message("KS_delta: ", KS_delta, ", at sigma: ", sigma, ", and pval: ", i3_p_val)
        sd_trend <- list(mu=mu, sigma=sigma, mean_delta=mean_delta, KS_delta=KS_delta)
    } else {
        cnv_mean_sd <- infercnv:::get_spike_dists(infercnv_obj@.hspike)
        HMM_info <- infercnv:::.get_HMM(cnv_mean_sd, t)
        fit <- infercnv:::get_hspike_cnv_mean_sd_trend_by_num_cells_fit(infercnv_obj@.hspike)
        sds <- unlist(lapply(hmm_groups, function(g)
            as.double(infercnv:::.get_state_emission_params(length(g), cnv_mean_sd, fit)$sd)))
        res <- .icnv_try(.Call("icnvR_smooth_hmm_groups", m, codes, refs, isTRUE(apply_log), as.double(max_centered_threshold),
                               as.integer(window_length), isTRUE(use_bounds), hmm_groups, HMM_info[["state_transitions"]],
                               HMM_info[["delta"]], HMM_info[["state_emission_params"]]$mean, sds), "smooth_hmm_groups")
        if (is.null(res)) return(NULL)
    }
    infercnv_obj@expr.data <- .icnv_keep_names(res[[1]], m)
    hmm_obj <- infercnv_obj
    hmm_obj@expr.data <- .icnv_keep_names(res[[2]], m)
    if (i3) return(list(infercnv_obj = infercnv_obj, hmm_obj = hmm_obj, median_obj = NULL, sd_trend = sd_trend))
    list(infercnv_obj = infercnv_obj, hmm_obj = hmm_obj)
}

## parallelDist::parallelDist as the reference calls it before every hclust() - parallelDist(t(expr[, cells]), threads = n)
## (R/inferCNV_tumor_subclusters.R:191,411,472,582,609; R/inferCNV_ops.R:1930,3242; R/inferCNV_heatmap.R:719,755,1062,1079).
## Same signature as parallelDist::parallelDist(x, method = "euclidean", diag = FALSE, upper = FALSE, threads = NULL, ...); any
## method but the default one, a non-matrix / non-double / NA-holding x, or a GPU error goes to the original.  `threads` never
## reaches the GPU path.  infercnv imports the function (R/inferCNV_constants.R:27), so the replacement is bound in the
## package's IMPORTS environment (infercnvb200_install); the "dist" object it returns is what hclust() and as.matrix() expect.
b200_parallelDist <- function(x, method = "euclidean", diag = FALSE, upper = FALSE, threads = NULL, ...) {
    orig <- .icnv_env$orig_parallelDist
    ok <- .icnv_enabled() && identical(method, "euclidean") && is.matrix(x) && is.double(x) && !anyNA(x) && nrow(x) >= 2 &&
        nrow(x) <= 65535 * 128    # the distance kernel's tile grid; hclust() past 65 536 takes the packed-triangle linkage
    if (ok) {
        d <- .icnv_try(.Call("icnvR_pairwise_dist", x), "parallelDist (euclidean)")
        if (!is.null(d)) {
            attributes(d) <- list(Size = nrow(x), Labels = rownames(x), Diag = diag, Upper = upper, method = "euclidean",
                                  call = match.call(), class = "dist")
            return(d)
        }
    }
    orig(x, method = method, diag = diag, upper = upper, threads = threads, ...)
}

## fastcluster::hclust as infercnv calls it on every parallelDist() result - hclust(d, method = hclust_method), default
## "ward.D2" (R/inferCNV_ops.R:262; R/inferCNV_tumor_subclusters.R:191,411,474,498,582,609; R/inferCNV_ops.R:1930,3242;
## R/inferCNV_heatmap.R:719,755,1062,1079).  Same signature as fastcluster::hclust(d, method = "complete", members = NULL)
## and the same "hclust" object.  The six reducible methods run as a nearest-neighbour chain on the GPU: up to 65 536
## observations on the square matrix (icnvR_hclust), beyond that on the packed triangle (icnvR_hclust_tri, the same tree
## bit for bit, bounded by the free device memory: 4 n (n - 1) bytes plus scratch).  Anything else - not a "dist", non-NULL
## members, centroid / median / the alias "ward", fewer than 2 observations, NA in d, or a library error (a triangle that
## does not fit is ICNV_E_NOMEM) - goes to the original, with the error logged.
b200_hclust <- function(d, method = "complete", members = NULL) {
    orig <- .icnv_env$orig_hclust
    codes <- c(single = 0L, complete = 1L, average = 2L, mcquitty = 3L, ward.D = 4L, ward.D2 = 7L)
    n <- if (inherits(d, "dist")) attr(d, "Size") else NA
    ok <- .icnv_enabled() && inherits(d, "dist") && is.null(members) && is.character(method) && length(method) == 1 &&
        method %in% names(codes) && !is.null(n) && !is.na(n) && n >= 2 && !anyNA(d)
    if (ok) {
        code <- codes[[method]]
        res <- if (n <= 65536) .icnv_try(.Call("icnvR_hclust", d, code), "hclust") else
            .icnv_try(.Call("icnvR_hclust_tri", d, code), "hclust (packed triangle)")
        if (!is.null(res)) {
            return(structure(list(merge = res[[1]], height = res[[2]], order = res[[3]], labels = attr(d, "Labels"),
                                  method = method, call = match.call(), dist.method = attr(d, "method")),
                             class = "hclust"))
        }
    }
    if (is.null(orig)) orig <- fastcluster::hclust
    orig(d, method = method, members = members)
}

## RANN::nn2 as .leiden_simple_snn calls it - nn2(t(expr_data), k = k_nn)$nn.idx (R/inferCNV_tumor_subclusters.R:725-741),
## the kNN graph of the default per-chromosome Leiden subclustering.  Same signature as RANN::nn2(data, query = data,
## k = min(10, nrow(data)), treetype = c("kd", "bd"), searchtype = c("standard", "priority", "radius"), radius = 0, eps = 0)
## and the same list(nn.idx, nn.dists).  The exact search runs on the GPU when query is the data itself, data is a double
## matrix without NA, searchtype is not "radius", eps is 0 and 1 <= k <= min(nrow(data), 64); anything else, or a library
## error, goes to the original.  Among equally near cells the GPU takes the lowest row (ANN: its tree traversal).
b200_nn2 <- function(data, query = data, k = min(10, nrow(data)), treetype = c("kd", "bd"),
                     searchtype = c("standard", "priority", "radius"), radius = 0, eps = 0) {
    orig <- .icnv_env$orig_nn2
    st <- tryCatch(match.arg(searchtype), error = function(e) NA_character_)
    ok <- .icnv_enabled() && (missing(query) || identical(query, data)) && is.matrix(data) && is.double(data) &&
        !anyNA(data) && !is.na(st) && st != "radius" && is.numeric(eps) && length(eps) == 1 && isTRUE(eps == 0) &&
        is.numeric(k) && length(k) == 1 && !is.na(k) && k == round(k) && k >= 1 && k <= min(nrow(data), 64)
    if (ok) {
        res <- .icnv_try(.Call("icnvR_knn", data, as.integer(k)), "nn2")
        if (!is.null(res)) return(list(nn.idx = res[[1]], nn.dists = res[[2]]))
    }
    if (is.null(orig)) orig <- RANN::nn2
    orig(data, query = query, k = k, treetype = treetype, searchtype = searchtype, radius = radius, eps = eps)
}

## smooth_by_chromosome_runmeans (R/inferCNV_ops.R:2679-2704), run()'s step 10 for smooth_method = "runmeans":
## apply(chr_data, 2, caTools::runmean, k = window_length) per chromosome, chromosomes of one gene left alone, hspike
## mirrored.  Falls back for NA, an even window, a non-double / non-matrix slot, genes of a chromosome not contiguous, or a
## library error.
b200_smooth_by_chromosome_runmeans <- function(infercnv_obj, window_length) {
    orig <- .icnv_env$orig$smooth_by_chromosome_runmeans
    m <- infercnv_obj@expr.data
    codes <- .icnv_chr_codes(infercnv_obj)
    if (!.icnv_enabled() || !.icnv_ok(m) || is.null(codes) || !is.numeric(window_length) || length(window_length) != 1 ||
        is.na(window_length) || window_length %% 2 == 0)
        return(orig(infercnv_obj, window_length))
    r <- rle(codes)
    lens <- as.integer(r$lengths)
    starts <- as.integer(c(0L, cumsum(lens)[-length(lens)]))
    for (chr in unique(infercnv_obj@gene_order[["chr"]])) futile.logger::flog.info(paste0("smooth_by_chromosome: chr: ", chr))
    res <- .icnv_try(.Call("icnvR_runmean", m, starts, lens, as.integer(window_length)), "smooth_by_chromosome_runmeans")
    if (is.null(res)) return(orig(infercnv_obj, window_length))
    dimnames(res) <- dimnames(m)
    infercnv_obj@expr.data <- res
    if (!is.null(infercnv_obj@.hspike)) {
        futile.logger::flog.info("-mirroring for hspike")
        infercnv_obj@.hspike <- b200_smooth_by_chromosome_runmeans(infercnv_obj@.hspike, window_length)
    }
    infercnv_obj
}

## smooth_by_chromosome_coordinates (R/inferCNV_ops.R:2534-2622), run()'s step 10 for smooth_method = "coordinates": every
## chromosome's genes smoothed by the genomic-distance weights of .smooth_helper_by_coordinates in one GPU call, chromosomes
## of one gene left alone, hspike mirrored with window_length = 51 as in the original.  Falls back for NA, a non-double /
## non-matrix slot, genes of a chromosome not contiguous, NA or non-finite start / stop, a window_length that is not one
## finite number, window_length < 2 (the original's warnings), or a library error.
b200_smooth_by_chromosome_coordinates <- function(infercnv_obj, window_length) {
    orig <- .icnv_env$orig$smooth_by_chromosome_coordinates
    m <- infercnv_obj@expr.data
    codes <- .icnv_chr_codes(infercnv_obj)
    gs <- infercnv_obj@gene_order[["start"]]
    ge <- infercnv_obj@gene_order[["stop"]]
    if (!.icnv_enabled() || !.icnv_ok(m) || is.null(codes) || !is.numeric(gs) || !is.numeric(ge) ||
        length(gs) != nrow(m) || length(ge) != nrow(m) || !all(is.finite(gs)) || !all(is.finite(ge)) ||
        !is.numeric(window_length) || length(window_length) != 1 || !is.finite(window_length) || window_length < 2)
        return(orig(infercnv_obj, window_length))
    r <- rle(codes)
    lens <- as.integer(r$lengths)
    starts <- as.integer(c(0L, cumsum(lens)[-length(lens)]))
    for (chr in unique(infercnv_obj@gene_order[["chr"]])) futile.logger::flog.info(paste0("smooth_by_chromosome: chr: ", chr))
    res <- .icnv_try(.Call("icnvR_smooth_coordinates", m, starts, lens, as.double(gs), as.double(ge), as.double(window_length)),
                     "smooth_by_chromosome_coordinates")
    if (is.null(res)) return(orig(infercnv_obj, window_length))
    dimnames(res) <- dimnames(m)
    infercnv_obj@expr.data <- res
    if (!is.null(infercnv_obj@.hspike)) {
        futile.logger::flog.info("-mirroring for hspike")
        infercnv_obj@.hspike <- b200_smooth_by_chromosome_coordinates(infercnv_obj@.hspike, window_length = 51)
    }
    infercnv_obj
}

## .parameterize_random_cluster_heights_smoothed_trees (R/inferCNV_tumor_subclusters.random_smoothed_trees.R:217-304): the
## observed tree and the 100 permuted maxima of one clade in one GPU call, the same list(h_obs, max_h,
## rand_max_height_dist, ecdf).  h_obs is the "hclust" object b200_hclust returns (labels = colnames(expr_matrix)).  The
## permutations come from the library's generator, seeded by two draws of R's RNG, so set.seed() before run() makes the
## null reproducible; the distribution is R's sample(), the draws are not.  Falls back for methods outside the six,
## n outside [2, 65536], NA, or a library error.
b200_.parameterize_random_cluster_heights_smoothed_trees <- function(expr_matrix, hclust_method, window_size, plot = FALSE) {
    orig <- .icnv_env$orig$.parameterize_random_cluster_heights_smoothed_trees
    codes <- c(single = 0L, complete = 1L, average = 2L, mcquitty = 3L, ward.D = 4L, ward.D2 = 7L)
    n <- if (is.matrix(expr_matrix)) ncol(expr_matrix) else NA
    ok <- .icnv_enabled() && .icnv_ok(expr_matrix) && is.character(hclust_method) && length(hclust_method) == 1 &&
        hclust_method %in% names(codes) && !is.na(n) && n >= 2 && n <= 65536 && is.numeric(window_size) &&
        length(window_size) == 1 && !is.na(window_size)
    if (ok) {
        seed <- as.double(c(sample.int(2^31 - 1, 1), sample.int(2^31 - 1, 1)))
        res <- .icnv_try(.Call("icnvR_random_tree_heights", expr_matrix, as.integer(window_size), codes[[hclust_method]],
                               100L, seed), "random trees")
        if (!is.null(res)) {
            h_obs <- structure(list(merge = res[[1]], height = res[[2]], order = res[[3]], labels = colnames(expr_matrix),
                                    method = hclust_method, call = match.call(), dist.method = "euclidean"),
                               class = "hclust")
            max_rand_heights <- res[[4]]
            max_height <- max(h_obs$height)
            message(sprintf("Lengths for original tree branches (h): %s", paste(h_obs$height, sep = ",", collapse = ",")))
            message(sprintf("Max height: %g", max_height))
            message(sprintf("Lengths for max heights: %s", paste(max_rand_heights, sep = ",", collapse = ",")))
            e <- stats::ecdf(max_rand_heights)
            message(sprintf("pval: %g", 1 - e(max_height)))
            params_list <- list(h_obs = h_obs, max_h = max_height, rand_max_height_dist = max_rand_heights, ecdf = e)
            if (plot) infercnv:::.plot_tree_height_dist(params_list)
            return(params_list)
        }
    }
    orig(expr_matrix, hclust_method, window_size, plot)
}

## .leiden_seurat_preprocess_routine (R/inferCNV_tumor_subclusters.R:699-723), the Leiden graph of step 15's default
## leiden_method = "PCA" (per group, and per (chromosome, group) for leiden_method_per_chr = "PCA"): Seurat's
## FindVariableFeatures(vst) -> ScaleData -> RunPCA(npcs = 10) -> FindNeighbors(k.param = k_nn) in one GPU call
## (icnv_seurat_snn_f64), then igraph's graph_from_adjacency_matrix(mode = "min", weighted = TRUE) and cluster_leiden
## exactly as the original calls them.  Deviations from the original:
##  - irlba and annoy are approximate; the device computes what they approximate (exact eigenpairs, the exact kNN), so the
##    graph can differ where annoy misses a neighbour or irlba's 1e-5 tolerance moves a near-tie;
##  - vst's loess is the direct local fit; R's default surface = "interpolate" interpolates it on a kd-tree, so genes whose
##    standardised variances lie within that interpolation error of the 2000th can be chosen differently
##    (icnv_debug_seurat_snn reports the gap at the cut);
##  - set.seed(42) is called where RunPCA(seed.use = 42) calls it, so the partition does not depend on the user's seed, as
##    in the original; partitions are not claimed equal to R's draw for draw (irlba's draws are not replayed).
## Falls back to the original for a matrix that is not double or holds NA, k_nn > 64, any library error (a non-constant
## gene with mean <= 0 among them: vst's log10 warns there), or a singular local trend fit - where R's loess warns and the
## original falls back to .leiden_simple_snn, which stays R's.
b200_.leiden_seurat_preprocess_routine <- function(expr_data, k_nn, resolution_parameter, objective_function) {
    orig <- .icnv_env$orig$.leiden_seurat_preprocess_routine
    ok <- .icnv_enabled() && .icnv_ok(expr_data) && is.numeric(k_nn) && length(k_nn) == 1 && !is.na(k_nn) && k_nn >= 1 &&
        k_nn <= 64 && k_nn <= ncol(expr_data)
    if (ok) {
        res <- .icnv_try(.Call("icnvR_seurat_snn", expr_data, as.integer(k_nn)), "the Seurat SNN graph")
        if (!is.null(res) && res[[4]] == 0L) {
            n <- ncol(expr_data)
            snn <- Matrix::sparseMatrix(i = res[[2]], p = res[[1]], x = res[[3]], dims = c(n, n), index1 = FALSE,
                                        dimnames = list(colnames(expr_data), colnames(expr_data)))
            set.seed(42)
            graph_obj <- igraph::graph_from_adjacency_matrix(snn, mode = "min", weighted = TRUE)
            partition_obj <- igraph::cluster_leiden(graph_obj, resolution_parameter = resolution_parameter,
                                                    objective_function = objective_function)
            return(partition_obj$membership)
        }
    }
    orig(expr_data, k_nn, resolution_parameter, objective_function)
}

## mask_non_DE_genes_basic (R/inferCNV_mask_non_DE.R:28-52), run()'s step 21: every (subcluster, reference group) test,
## BH and the mask in one GPU call, with the original's two messages per pair.  The Wilcoxon jitter comes from the
## library's generator (rnorm's law, mean 1e-4, sd 1e-4), seeded by two draws of R's RNG; reference-side draws are shared by
## all subclusters (INTEGRATION.md section 4).  Falls back for test.use = "perm", a non-double or NA-holding matrix, NULL or
## duplicated rownames, duplicated pair names, an unknown require_DE_all_normals (the original's stop()), or a library error.
b200_mask_non_DE_genes_basic <- function(infercnv_obj, p_val_thresh = 0.05, test.use = "wilcoxon",
                                         center_val = mean(infercnv_obj@expr.data), require_DE_all_normals = "any") {
    orig <- .icnv_env$orig$mask_non_DE_genes_basic
    m <- infercnv_obj@expr.data
    rules <- c(any = 0L, most = 1L, all = 2L)
    tests <- c(wilcoxon = 0L, t = 1L)
    refs <- infercnv_obj@reference_grouped_cell_indices
    ok <- .icnv_enabled() && is.matrix(m) && is.double(m) && !anyNA(m) && !is.null(rownames(m)) &&
        !anyDuplicated(rownames(m)) && is.character(test.use) && length(test.use) == 1 && test.use %in% names(tests) &&
        is.character(require_DE_all_normals) && length(require_DE_all_normals) == 1 &&
        require_DE_all_normals %in% names(rules) && length(refs) > 0 && is.numeric(center_val) && length(center_val) == 1
    if (ok) {
        ## get_DE_genes_basic's loop (:213-224): a group whose subclusters are not a (named) list is tested for nothing
        sub_names <- character(0)
        subs <- list()
        for (tumor_type in names(infercnv_obj@observation_grouped_cell_indices)) {
            indices <- infercnv_obj@tumor_subclusters[["subclusters"]][[tumor_type]]
            if (is.list(indices)) for (nm in names(indices)) {
                sub_names <- c(sub_names, nm)
                subs[[length(subs) + 1]] <- as.integer(indices[[nm]])
            }
        }
        pairs <- as.vector(t(outer(sub_names, names(refs), paste, sep = ",")))
        ok <- !anyDuplicated(pairs)
    }
    if (ok) {
        seed <- as.double(c(sample.int(2^31 - 1, 1), sample.int(2^31 - 1, 1)))
        res <- .icnv_try(.Call("icnvR_mask_non_de", m, lapply(refs, as.integer), subs, tests[[test.use]],
                               as.double(p_val_thresh), rules[[require_DE_all_normals]], as.double(center_val), seed),
                         "mask_non_DE_genes_basic")
        if (!is.null(res)) {
            p_adj <- res[[2]]
            k <- 0L
            for (s in seq_along(subs)) for (normal_type in names(refs)) {
                k <- k + 1L
                futile.logger::flog.info(sprintf("Finding DE genes between %s and %s", sub_names[[s]], normal_type))
                p <- p_adj[, k]
                futile.logger::flog.info(sprintf("Found %d genes / %d total as DE", sum(p < p_val_thresh, na.rm = TRUE) +
                                                 sum(is.na(p)), length(p)))
            }
            dimnames(res[[1]]) <- dimnames(m)
            infercnv_obj@expr.data <- res[[1]]
            return(infercnv_obj)
        }
    }
    orig(infercnv_obj, p_val_thresh = p_val_thresh, test.use = test.use, center_val = center_val,
         require_DE_all_normals = require_DE_all_normals)
}

## inferCNVBayesNet (R/inferCNV_BayesNet.R:1237-1364; run() step 18) with every region's Gibbs sampling in one library call
## (icnv_bayesnet_f64) in place of runMCMC's one JAGS model per region: the same posterior, not JAGS's draws.  The chains
## (6 for i6, 3 for i3, chain c from state c), 500 + 200 discarded and 1000 kept sweeps, and the outputs' shapes and dimnames
## are the original's; a region of one gene and several cells is JAGS's single pseudo-cell (INTEGRATION.md section 4).  The
## generator is seeded by two draws of R's RNG.  The whole original runs for diagnostics = TRUE when no_plot does not turn
## them off (coda needs the raw chains), a model file that is not the bundled one, or a non-double or NA-holding matrix -
## all decided before anything is logged; the original's runMCMC runs on the initialised object, with R's RNG stream as it
## was, for a region without cells or a library error.
b200_inferCNVBayesNet <- function( file_dir,
                              infercnv_obj,
                              HMM_states,
                              out_dir,
                              resume_file_token,
                              model_file        = NULL,
                              CORES             = 1,
                              postMcmcMethod    = NULL,
                              plotingProbs      = TRUE,
                              quietly           = TRUE,
                              diagnostics       = FALSE,
                              HMM_type          = HMM_type,
                              k_obs_groups      = k_obs_groups,
                              cluster_by_groups = cluster_by_groups,
                              reassignCNVs      = TRUE,
                              no_plot           = no_plot,
                              useRaster) {
    orig <- .icnv_env$orig$inferCNVBayesNet
    fallback <- function() orig(file_dir = file_dir, infercnv_obj = infercnv_obj, HMM_states = HMM_states, out_dir = out_dir,
                                resume_file_token = resume_file_token, model_file = model_file, CORES = CORES,
                                postMcmcMethod = postMcmcMethod, plotingProbs = plotingProbs, quietly = quietly,
                                diagnostics = diagnostics, HMM_type = HMM_type, k_obs_groups = k_obs_groups,
                                cluster_by_groups = cluster_by_groups, reassignCNVs = reassignCNVs, no_plot = no_plot,
                                useRaster = useRaster)
    bundled <- ifelse(HMM_type == "i6", system.file("BUGS_Mixture_Model", package = "infercnv"),
                      system.file("BUGS_Mixture_Model_i3", package = "infercnv"))
    ## no_plot overrides the plotting options first, as in the original
    diag_on <- if (no_plot == TRUE) FALSE else isTRUE(diagnostics)
    x <- infercnv_obj@expr.data
    if (!.icnv_enabled() || diag_on || !is.matrix(x) || !is.double(x) || anyNA(x) ||
        (!is.null(model_file) && !identical(normalizePath(model_file, mustWork = FALSE), normalizePath(bundled, mustWork = FALSE))))
        return(fallback())
    ## the original's input checks
    if (!is.null(model_file) && !file.exists(model_file)){
        error_message <- paste("Cannot find the model file.",
                               "Please supply the correct path for the model file.")
        futile.logger::flog.error(error_message)
        stop(error_message)
    }
    if (!(CORES == 1)){
        if (is.na(parallel::detectCores())){
            futile.logger::flog.warn(paste("Unable to detect number of cores available through parallel:detectCores(), using the provided number", CORES))
        } else if (as.integer(CORES) > parallel::detectCores()){
            error_message <- paste("Too many cores previded. The following system has ", parallel::detectCores(), " cores.",
                                   "Please select an appropriate amount.")
            futile.logger::flog.error(error_message)
            stop(error_message)
        }
    }
    if(out_dir != "." & !file.exists(out_dir)){
        dir.create(file.path(out_dir))
        futile.logger::flog.info(paste("Creating the following Directory: ", out_dir))
    }
    if (is.null(model_file)) model_file <- bundled
    if (no_plot == TRUE) {
        plotingProbs <- FALSE
        diagnostics <- FALSE
    }
    args_parsed <- list("file_dir" = file_dir, "model_file" = model_file, "CORES" = CORES, "out_dir"= out_dir,
                        "resume_file_token" = resume_file_token, "plotingProbs" = plotingProbs,
                        "postMcmcMethod"= postMcmcMethod, "quietly" = quietly, "BayesMaxPNormal" = 0, "HMM_type" = HMM_type,
                        "k_obs_groups" = k_obs_groups, "cluster_by_groups" = cluster_by_groups,
                        "reassignCNVs" = reassignCNVs, "diagnostics" = diagnostics)
    obj <- methods::new("MCMC_inferCNV")
    obj <- infercnv:::initializeObject(obj, args_parsed, infercnv_obj)
    obj <- infercnv:::MeanSD(obj = obj, HMM_states = HMM_states, infercnv_obj = infercnv_obj)
    m <- obj@expr.data
    cg <- obj@cell_gene
    n_states <- ifelse(HMM_type == "i6", 6L, 3L)
    n_chains <- n_states
    start_time <- Sys.time()
    res <- NULL
    if (length(cg) > 0 && !any(vapply(cg, function(i) length(i$Cells) == 0 || length(i$Genes) == 0, logical(1)))) {
        ## the seeds are the last thing drawn before the call; a library error puts R's RNG stream back
        had_seed <- exists(".Random.seed", envir = globalenv(), inherits = FALSE)
        old_seed <- if (had_seed) get(".Random.seed", envir = globalenv(), inherits = FALSE) else NULL
        seed <- as.double(c(sample.int(2^31 - 1, 1), sample.int(2^31 - 1, 1)))
        genes <- lapply(cg, function(i) as.integer(if (is.character(i$Genes)) match(i$Genes, rownames(m)) else i$Genes))
        cells <- lapply(cg, function(i) as.integer(if (is.character(i$Cells)) match(i$Cells, colnames(m)) else i$Cells))
        pooled <- vapply(cg, function(i) length(i$Genes) == 1 && length(i$Cells) > 1, logical(1))
        res <- .icnv_try(.Call("icnvR_bayesnet", m, genes, cells, as.integer(pooled), as.double(obj@mu), as.double(obj@sig),
                               n_chains, 700L, 1000L, seed), "inferCNVBayesNet")
        if (is.null(res)) {
            if (had_seed) assign(".Random.seed", old_seed, envir = globalenv())
            else if (exists(".Random.seed", envir = globalenv(), inherits = FALSE)) rm(".Random.seed", envir = globalenv())
        }
    }
    if (is.null(res)) {
        ## the original's own sampling on the object it would have built
        obj <- infercnv:::runMCMC(obj, diagnostics)
        res <- list(NULL, NULL)
    }
    if (!is.null(res[[1]])) {
        obj@cnv_probabilities <- lapply(res[[1]], function(th) {
            colnames(th) <- sprintf("theta[%d]", seq_len(n_states))
            th
        })
        ## cell_prob's names: one epsilon column drops to a vector, which as.data.frame names "epsilons"
        obj@cell_probabilities <- lapply(res[[2]], function(p) {
            dimnames(p) <- list(as.character(seq_len(n_states)),
                                if (ncol(p) == 1) "epsilons" else sprintf("epsilon[%d]", seq_len(ncol(p))))
            p
        })
    }
    end_time <- Sys.time()
    futile.logger::flog.info(paste("Gibbs sampling time: ", difftime(end_time, start_time, units = "min")[[1]], " Minutes"))
    saveRDS(obj, file = file.path(obj@args$out_dir, "MCMC_inferCNV_obj.rds"))
    if (obj@args$postMcmcMethod == "removeCNV" || obj@args$reassignCNVs == TRUE ){
        title <- sprintf(" (1 - Probabilities of Normal) Before Filtering")
        output_filename <- "infercnv.NormalProbabilities.PreFiltering"
    } else {
        title <- sprintf(" 1 - Probabilities of Normal ")
        output_filename <- "infercnv.NormalProbabilities"
    }
    infercnv:::postProbNormal(obj, PNormal = NULL, title = title, output_filename = output_filename, useRaster = useRaster)
    obj
}

## define_signif_tumor_subclusters (R/inferCNV_tumor_subclusters.R:2-177), run() step 15, and its hidden-spike mirror: the
## z-score gene filter (:45-68) and every hclust() tree of the step in GPU calls - one icnvR_zscore_outlier_genes, then one
## icnvR_cluster_groups for all groups (and, with Leiden, all partitions), so no distance vector passes through R.  Same
## signature and result as the original.  The filter keeps the original's quirk: which() never returns NULL, so with no outlier
## gene expr.data[-outliers, ] keeps no gene and every distance is 0.
##   qnorm / pheight / qgamma / none: cut heights and cutree() are R's own on the returned trees.
##   leiden: the partition of every group is computed first, in group order, by the original's own
##   .leiden_seurat_preprocess_routine / .leiden_simple_snn, so R's RNG is consumed as the original consumes it (the trees use
##   none of it); then one call builds every partition's tree (and the whole group when k_nn >= its size), and the phylo
##   assembly runs in the original's partition order.  The per-chromosome part stays the original's
##   .whole_dataset_leiden_subclustering_per_chr on the filtered data (its nn2() is b200_nn2).
## Falls back to the original for restrict_to_DE_genes = TRUE, a method outside the six, an unknown partition_method, a
## non-double or NA-holding matrix, a group of more than 65 536 cells, or a library error.
b200_define_signif_tumor_subclusters <- function(infercnv_obj, p_val = 0.1, k_nn = 20, leiden_method = c("PCA", "simple"),
                                                 leiden_function = c("CPM", "modularity"), leiden_resolution = "auto",
                                                 leiden_method_per_chr = c("simple", "PCA"),
                                                 leiden_function_per_chr = c("modularity", "CPM"),
                                                 leiden_resolution_per_chr = 1, hclust_method = "ward.D2",
                                                 cluster_by_groups = TRUE, partition_method = "leiden",
                                                 per_chr_hmm_subclusters = FALSE,
                                                 per_chr_hmm_subclusters_references = FALSE, z_score_filter = 0.8,
                                                 restrict_to_DE_genes = FALSE) {
    orig <- .icnv_env$orig$define_signif_tumor_subclusters
    call_orig <- function() orig(infercnv_obj, p_val = p_val, k_nn = k_nn, leiden_method = leiden_method,
                                 leiden_function = leiden_function, leiden_resolution = leiden_resolution,
                                 leiden_method_per_chr = leiden_method_per_chr, leiden_function_per_chr = leiden_function_per_chr,
                                 leiden_resolution_per_chr = leiden_resolution_per_chr, hclust_method = hclust_method,
                                 cluster_by_groups = cluster_by_groups, partition_method = partition_method,
                                 per_chr_hmm_subclusters = per_chr_hmm_subclusters,
                                 per_chr_hmm_subclusters_references = per_chr_hmm_subclusters_references,
                                 z_score_filter = z_score_filter, restrict_to_DE_genes = restrict_to_DE_genes)
    codes <- c(single = 0L, complete = 1L, average = 2L, mcquitty = 3L, ward.D = 4L, ward.D2 = 7L)
    m <- infercnv_obj@expr.data
    refs <- infercnv_obj@reference_grouped_cell_indices
    obs <- infercnv_obj@observation_grouped_cell_indices
    if (cluster_by_groups) {
        tumor_groups <- c(obs, refs)
    } else {
        tumor_groups <- c(list(all_observations = unlist(obs, use.names = FALSE)), refs)
    }
    ok <- .icnv_enabled() && !isTRUE(restrict_to_DE_genes) && .icnv_ok(m) && nrow(m) >= 2 && is.character(hclust_method) &&
        length(hclust_method) == 1 && hclust_method %in% names(codes) && is.character(partition_method) &&
        length(partition_method) == 1 && partition_method %in% c("leiden", "qnorm", "pheight", "qgamma", "none")
    if (!ok) return(call_orig())
    leiden_method <- match.arg(leiden_method)
    leiden_method_per_chr <- match.arg(leiden_method_per_chr)
    leiden_function <- match.arg(leiden_function)
    leiden_function_per_chr <- match.arg(leiden_function_per_chr)
    futile.logger::flog.info(sprintf("define_signif_tumor_subclusters(p_val=%g", p_val))

    ## the filter: keep = NULL (every gene) or the kept rows, 1-based
    keep <- NULL
    gene_order <- infercnv_obj@gene_order
    if (z_score_filter > 0 && length(refs) > 0) {
        flags <- .icnv_try(.Call("icnvR_zscore_outlier_genes", m, as.integer(unlist(refs, use.names = FALSE))), "z-score filter")
        if (is.null(flags)) return(call_orig())
        outliers <- which(flags)
        keep <- seq_len(nrow(m))[-outliers]        # integer(0) when there is no outlier, as expr.data[-outliers, ] is
        gene_order <- gene_order[-outliers, , drop = FALSE]
    }
    mk_hclust <- function(tr, cols) {
        structure(list(merge = tr[[1]], height = tr[[2]], order = tr[[3]], labels = colnames(m)[cols], method = hclust_method,
                       call = match.call(), dist.method = "euclidean"), class = "hclust")
    }
    ## groups of up to 65 536 cells in one icnvR_cluster_groups call; each larger one through icnvR_cluster_cells (the
    ## packed-triangle linkage, bounded by the free device memory); the same trees either way
    trees_of <- function(lists) {
        if (length(lists) == 0) return(list())
        kp <- if (is.null(keep)) NULL else as.integer(keep)
        big <- lengths(lists) > 65536
        out <- vector("list", length(lists))
        if (any(!big)) {
            small <- .icnv_try(.Call("icnvR_cluster_groups", m, kp, lapply(lists[!big], as.integer), codes[[hclust_method]]),
                               "subcluster trees")
            if (is.null(small)) return(NULL)
            out[!big] <- small
        }
        for (i in which(big)) {
            tr <- .icnv_try(.Call("icnvR_cluster_cells", m, kp, as.integer(lists[[i]]), codes[[hclust_method]]),
                            "subcluster tree (more than 65 536 cells)")
            if (is.null(tr)) return(NULL)
            out[[i]] <- tr
        }
        out
    }

    res <- list()
    if (partition_method != "leiden") {
        big <- names(tumor_groups)[lengths(tumor_groups) > 2]
        trees <- trees_of(unname(tumor_groups[big]))
        if (is.null(trees)) return(call_orig())
        names(trees) <- big
        for (tumor_group in names(tumor_groups)) {
            futile.logger::flog.info(sprintf("define_signif_tumor_subclusters(), tumor: %s", tumor_group))
            tumor_group_idx <- tumor_groups[[tumor_group]]
            names(tumor_group_idx) <- colnames(m)[tumor_group_idx]
            info <- list()
            if (length(tumor_group_idx) > 2) {
                hc <- mk_hclust(trees[[tumor_group]], tumor_group_idx)
                info$hc <- hc
                heights <- hc$height
                if (partition_method == "pheight") {
                    cut_height <- p_val * max(heights)
                } else if (partition_method == "qnorm") {
                    cut_height <- stats::qnorm(p = 1 - p_val, mean = mean(heights), sd = stats::sd(heights))
                } else if (partition_method == "qgamma") {
                    gamma_fit <- fitdistrplus::fitdist(heights, "gamma")
                    cut_height <- stats::qgamma(p = 1 - p_val, shape = gamma_fit$estimate[1], rate = gamma_fit$estimate[2])
                }
                if (partition_method == "none") {
                    grps <- stats::cutree(hc, k = 1)
                } else {
                    futile.logger::flog.info(sprintf("cut height based on p_val(%g) = %g and partition_method: %s", p_val,
                                                     cut_height, partition_method))
                    grps <- stats::cutree(hc, h = cut_height)
                }
                info$subclusters <- list()
                s <- split(grps, grps)
                futile.logger::flog.info(sprintf("cut tree into: %g groups", length(s)))
                start_idx <- 1
                for (g in names(s)) {
                    split_subcluster <- paste0(tumor_group, "_s", g)
                    futile.logger::flog.info(sprintf("-processing %s,%s", tumor_group, split_subcluster))
                    end_idx <- start_idx + length(s[[g]]) - 1
                    info$subclusters[[split_subcluster]] <- tumor_group_idx[hc$order[start_idx:end_idx]]
                    start_idx <- end_idx + 1
                }
            } else {
                info$hc <- NULL
                info$subclusters[[paste0(tumor_group, "_s1")]] <- tumor_group_idx
            }
            res$hc[[tumor_group]] <- info$hc
            res$subclusters[[tumor_group]] <- info$subclusters
        }
    } else {
        ## every group's partition first, in group order (the RNG draws of the original's order)
        expr_kept <- if (is.null(keep)) m else m[keep, , drop = FALSE]
        parts <- list()
        lists <- list()
        for (tumor_group in names(tumor_groups)) {
            futile.logger::flog.info(sprintf("define_signif_tumor_subclusters(), tumor: %s", tumor_group))
            idx <- tumor_groups[[tumor_group]]
            if (length(idx) < 3) {
                futile.logger::flog.info(paste0("Too few cells in group ", tumor_group, " for any (sub)clustering. Keeping as is."))
                next
            }
            if (k_nn >= length(idx)) {
                futile.logger::flog.info(paste0("Less cells in group ", tumor_group, " than k_nn setting. Keeping as a single subcluster."))
                lists[[length(lists) + 1]] <- idx
                next
            }
            res_used <- if (identical(leiden_resolution, "auto")) (11.98 / length(idx))^(1 / 1.165) else leiden_resolution
            if (identical(leiden_resolution, "auto"))
                futile.logger::flog.info(sprintf("Setting auto leiden resolution for %s to %g", tumor_group, res_used))
            tumor_expr_data <- expr_kept[, idx, drop = FALSE]
            if (leiden_method == "PCA") {
                partition <- infercnv:::.leiden_seurat_preprocess_routine(expr_data = tumor_expr_data, k_nn = k_nn,
                                                                          resolution_parameter = res_used,
                                                                          objective_function = leiden_function)
            } else {
                partition <- infercnv:::.leiden_simple_snn(tumor_expr_data, k_nn, res_used, leiden_function)
            }
            parts[[tumor_group]] <- partition
            for (i in names(sort(table(partition), decreasing = TRUE))) {
                w <- which(partition == i)
                if (length(w) >= 2) lists[[length(lists) + 1]] <- idx[w]
            }
        }
        trees <- trees_of(lists)
        if (is.null(trees)) return(call_orig())
        next_tree <- 0
        for (tumor_group in names(tumor_groups)) {
            idx <- tumor_groups[[tumor_group]]
            names(idx) <- colnames(m)[idx]
            if (length(idx) < 3) {
                res$hc[[tumor_group]] <- NULL
                res$subclusters[[tumor_group]] <- list()
                res$subclusters[[tumor_group]][[paste0(tumor_group, "_s1")]] <- idx
                next
            }
            if (k_nn >= length(idx)) {
                next_tree <- next_tree + 1
                res$subclusters[[tumor_group]] <- list()
                res$subclusters[[tumor_group]][[tumor_group]] <- idx
                res$hc[[tumor_group]] <- mk_hclust(trees[[next_tree]], idx)
                next
            }
            partition <- parts[[tumor_group]]
            subs <- list()
            full <- NULL
            for (i in names(sort(table(partition), decreasing = TRUE))) {
                w <- which(partition == i)
                subs[[paste(tumor_group, i, sep = "_s")]] <- idx[w]
                if (length(w) >= 2) {
                    next_tree <- next_tree + 1
                    tmp <- ape::as.phylo(mk_hclust(trees[[next_tree]], idx[w]))
                    if (is.null(full)) {
                        full <- tmp
                    } else {
                        h1 <- phytools::get.rooted.tree.height(tmp)
                        h2 <- phytools::get.rooted.tree.height(full)
                        if (h1 == h2) {
                            tmp$root.edge <- 1
                            full$root.edge <- 1
                        } else if (h1 > h2) {
                            tmp$root.edge <- 1
                            full$root.edge <- h1 - h2 + 1
                        } else {
                            tmp$root.edge <- h2 - h1 + 1
                            full$root.edge <- 1
                        }
                        full <- tmp + full
                    }
                } else {
                    full <- infercnv:::add_single_branch_to_phylo(full, colnames(m)[idx[w]])
                }
            }
            res$hc[[tumor_group]] <- ape::as.hclust.phylo(full)
            res$subclusters[[tumor_group]] <- subs
        }
    }
    infercnv_obj@tumor_subclusters <- res

    subclusters_per_chr <- NULL
    if (per_chr_hmm_subclusters && partition_method == "leiden") {
        if (!per_chr_hmm_subclusters_references) {
            tumor_groups <- if (cluster_by_groups) obs else list(all_observations = unlist(obs, use.names = FALSE))
        }
        expr_kept <- if (is.null(keep)) m else m[keep, , drop = FALSE]
        subclusters_per_chr <- infercnv:::.whole_dataset_leiden_subclustering_per_chr(
            expr_data = expr_kept, tumor_groups = tumor_groups, chrs = gene_order$chr, k_nn = k_nn,
            leiden_resolution = leiden_resolution_per_chr, leiden_method = leiden_method_per_chr,
            leiden_function = leiden_function_per_chr)
        if (!per_chr_hmm_subclusters_references) {
            for (i in names(subclusters_per_chr)) subclusters_per_chr[[i]] <- c(subclusters_per_chr[[i]], refs)
        }
    }
    if (!is.null(infercnv_obj@.hspike)) {
        futile.logger::flog.info("-mirroring for hspike")
        infercnv_obj@.hspike <- b200_define_signif_tumor_subclusters(infercnv_obj@.hspike, cluster_by_groups = TRUE,
                                                                     partition_method = "none")[[1]]
    }
    list(infercnv_obj, subclusters_per_chr)
}

infercnvb200_install <- function() {
    fns <- c("subtract_ref_expr_from_obs", "smooth_by_chromosome", "center_cell_expr_across_chromosome",
             "predict_CNV_via_HMM_on_indiv_cells", "predict_CNV_via_HMM_on_tumor_subclusters",
             "predict_CNV_via_HMM_on_whole_tumor_samples", "i3HMM_predict_CNV_via_HMM_on_indiv_cells",
             "apply_median_filtering", "normalize_counts_by_seq_depth", "clear_noise_via_ref_mean_sd",
             "get_predicted_CNV_regions", "remove_outliers_norm", "clear_noise",
             "predict_CNV_via_HMM_on_tumor_subclusters_per_chr", "i3HMM_predict_CNV_via_HMM_on_tumor_subclusters",
             "i3HMM_predict_CNV_via_HMM_on_whole_tumor_samples", "scale_infercnv_expr", "smooth_by_chromosome_runmeans",
             "mask_non_DE_genes_basic", "inferCNVBayesNet", "smooth_by_chromosome_coordinates",
             "define_signif_tumor_subclusters",
             ## internal, dot-prefixed names: their closures are b200_.parameterize... and b200_.leiden..., which the get()
             ## below finds as they are
             ".parameterize_random_cluster_heights_smoothed_trees", ".leiden_seurat_preprocess_routine")
    ns <- asNamespace("infercnv")
    .icnv_env$orig <- lapply(stats::setNames(fns, fns), function(f) get(f, envir = ns))
    for (f in fns) utils::assignInNamespace(f, get(paste0("b200_", f)), ns = "infercnv")
    ## parallelDist is an IMPORT of infercnv: its binding lives in the parent of the namespace ("imports:infercnv")
    imp <- parent.env(ns)
    if (exists("parallelDist", envir = imp, inherits = FALSE)) {
        .icnv_env$orig_parallelDist <- get("parallelDist", envir = imp)
        unlockBinding("parallelDist", imp)
        assign("parallelDist", b200_parallelDist, envir = imp)
        lockBinding("parallelDist", imp)
    }
    ## hclust is an import too (NAMESPACE: importFrom(fastcluster, hclust))
    if (exists("hclust", envir = imp, inherits = FALSE)) {
        .icnv_env$orig_hclust <- get("hclust", envir = imp)
        unlockBinding("hclust", imp)
        assign("hclust", b200_hclust, envir = imp)
        lockBinding("hclust", imp)
    }
    ## and nn2 (NAMESPACE: importFrom(RANN, nn2))
    if (exists("nn2", envir = imp, inherits = FALSE)) {
        .icnv_env$orig_nn2 <- get("nn2", envir = imp)
        unlockBinding("nn2", imp)
        assign("nn2", b200_nn2, envir = imp)
        lockBinding("nn2", imp)
    }
    invisible(TRUE)
}

infercnvb200_uninstall <- function() {
    for (f in names(.icnv_env$orig)) utils::assignInNamespace(f, .icnv_env$orig[[f]], ns = "infercnv")
    imp <- parent.env(asNamespace("infercnv"))
    if (!is.null(.icnv_env$orig_parallelDist)) {
        unlockBinding("parallelDist", imp)
        assign("parallelDist", .icnv_env$orig_parallelDist, envir = imp)
        lockBinding("parallelDist", imp)
    }
    if (!is.null(.icnv_env$orig_hclust)) {
        unlockBinding("hclust", imp)
        assign("hclust", .icnv_env$orig_hclust, envir = imp)
        lockBinding("hclust", imp)
    }
    if (!is.null(.icnv_env$orig_nn2)) {
        unlockBinding("nn2", imp)
        assign("nn2", .icnv_env$orig_nn2, envir = imp)
        lockBinding("nn2", imp)
    }
    invisible(TRUE)
}
