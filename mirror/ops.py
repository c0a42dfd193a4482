"""Host-side mirror of the reference's R interface for the hot path: same function names, argument
meaning and error behaviour as the R functions whose bodies the GPU library replaces, so the parity
tests read like the reference's own tests.  Every function is `f(infercnv_obj, ...) -> infercnv_obj`
that rewrites `expr_data` and mirrors itself onto `hspike` when that slot is set, exactly like
the R originals (e.g. R/inferCNV_ops.R:1695-1698, 2081-2084, 2427-2430).

All numerics happen in libinfercnv_b200.so (CUDA); nothing here computes on the CPU beyond
argument marshalling.  R is 1-based, this mirror is 0-based.
"""
from __future__ import annotations

import copy
import logging
import os
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from infercnv_b200 import api

log = logging.getLogger("infercnv_b200")  # the R functions log through futile.logger's flog.info



@dataclass
class Infercnv:
    """The slots of the S4 class `infercnv` (R/inferCNV.R:37-47) the hot path touches."""
    expr_data: np.ndarray                                   # genes x cells, float64 (Fortran order)
    gene_order_chr: np.ndarray                              # gene_order$chr as codes, rows pre-sorted by chr
    reference_grouped_cell_indices: dict = field(default_factory=dict)     # name -> 0-based cell indices
    observation_grouped_cell_indices: dict = field(default_factory=dict)
    tumor_subclusters: Optional[dict] = None                # {"subclusters": {group: {name: indices}}}
    count_data: Optional[np.ndarray] = None
    options: dict = field(default_factory=dict)
    hspike: Optional["Infercnv"] = None                     # @.hspike
    # the rest of @gene_order and the dimnames of @expr.data: only the region reports read them
    gene_names: Optional[list] = None                       # rownames(gene_order)
    gene_order_start: Optional[np.ndarray] = None           # gene_order$start
    gene_order_stop: Optional[np.ndarray] = None            # gene_order$stop
    cell_names: Optional[list] = None                       # colnames(expr.data)
    chr_names: Optional[dict] = None                        # label of each gene_order_chr code (default: str(code))

    def __post_init__(self):
        self.expr_data = np.asfortranarray(self.expr_data, dtype=np.float64)

    def chr_ranges(self):
        return api.chr_ranges(self.gene_order_chr)


def has_reference_cells(obj: Infercnv) -> bool:
    """R/inferCNV.R has_reference_cells: length(reference_grouped_cell_indices) != 0."""
    return len(obj.reference_grouped_cell_indices) != 0


def _ref_groups(obj: Infercnv):
    # subtract_ref_expr_from_obs, R/inferCNV_ops.R:1683-1689
    if has_reference_cells(obj):
        log.info("subtracting mean(normal) per gene per cell across all data")
        return [np.asarray(v) for v in obj.reference_grouped_cell_indices.values()]
    log.info("-no reference cells specified... using mean of all cells as proxy")
    return [np.concatenate([np.asarray(v) for v in obj.observation_grouped_cell_indices.values()])]


def subtract_ref_expr_from_obs(infercnv_obj: Infercnv, inv_log: bool = False, use_bounds: bool = True) -> Infercnv:
    """R/inferCNV_ops.R:1678-1702."""
    log.info("::subtract_ref_expr_from_obs:Start inv_log=%s, use_bounds=%s", inv_log, use_bounds)
    obj = copy.copy(infercnv_obj)
    means = api.ref_means(obj.expr_data, _ref_groups(obj), inv_log=inv_log)        # .get_normal_gene_mean_bounds
    log.info("-subtracting expr per gene, use_bounds=%s", use_bounds)
    obj.expr_data = api.subtract_ref(obj.expr_data, means, use_bounds=use_bounds)  # .subtract_expr
    if obj.hspike is not None:
        log.info("-mirroring for hspike")
        obj.hspike = subtract_ref_expr_from_obs(obj.hspike, inv_log=inv_log, use_bounds=use_bounds)
    return obj


def normalize_counts_by_seq_depth(infercnv_obj: Infercnv, normalize_factor=None) -> Infercnv:
    """R/inferCNV_ops.R:3064-3111 (no hspike mirroring in the reference: the spike is built after this step)."""
    log.info("normalizing counts matrix by depth")
    obj = copy.copy(infercnv_obj)
    obj.expr_data = api.normalize_counts_by_seq_depth(obj.expr_data, normalize_factor)
    return obj


def clear_noise_via_ref_mean_sd(infercnv_obj: Infercnv, sd_amplifier: float = 1.5, noise_logistic: bool = False) -> Infercnv:
    """R/inferCNV_ops.R:2302-2346 (hspike mirroring is commented out in the reference)."""
    if has_reference_cells(infercnv_obj):
        log.info("denoising using mean(normal) +- sd_amplifier * sd(normal) per gene per cell across all data")
        cells = np.concatenate([np.asarray(v) for v in infercnv_obj.reference_grouped_cell_indices.values()])
    else:
        log.info("-no reference cells specified... using mean and sd of all cells as proxy for denoising")
        cells = np.concatenate([np.asarray(v) for v in infercnv_obj.observation_grouped_cell_indices.values()])
    obj = copy.copy(infercnv_obj)
    if noise_logistic:
        obj.expr_data = api.clear_noise_via_ref_mean_sd_logistic(obj.expr_data, cells, sd_amplifier)
    else:
        obj.expr_data = api.clear_noise_via_ref_mean_sd(obj.expr_data, cells, sd_amplifier)
    return obj


def clear_noise(infercnv_obj: Infercnv, threshold: float, noise_logistic: bool = False) -> Infercnv:
    """R/inferCNV_ops.R:2232-2263: noise around the mean of the reference cells (or of all data) within +- threshold."""
    log.info("********* ::clear_noise:Start. threshold: %s", threshold)
    if threshold == 0:
        return infercnv_obj                       # nothing to do
    cells = (np.concatenate([np.asarray(v) for v in infercnv_obj.reference_grouped_cell_indices.values()])
             if has_reference_cells(infercnv_obj) else None)
    obj = copy.copy(infercnv_obj)
    obj.expr_data = api.clear_noise(obj.expr_data, cells, threshold, noise_logistic)
    return obj


def remove_outliers_norm(infercnv_obj: Infercnv, out_method: Optional[str] = "average_bound", lower_bound=None,
                         upper_bound=None) -> Infercnv:
    """R/inferCNV_ops.R:1969-2056 (run() step 16): hard bounds when both are given, else "average_bound"."""
    log.info("::remove_outlier_norm:Start out_method: %s lower_bound: %s upper_bound: %s", out_method, lower_bound, upper_bound)
    obj = copy.copy(infercnv_obj)
    if lower_bound is not None and upper_bound is not None:
        log.info("::remove_outlier_norm: using hard thresholds:  lower_bound: %s upper_bound: %s", lower_bound, upper_bound)
        obj.expr_data = api.remove_outliers_norm(obj.expr_data, lower_bound, upper_bound)
    elif out_method is not None:
        log.info("::remove_outlier_norm using method: %s for defining outliers.", out_method)
        if out_method != "average_bound":
            log.error("::remove_outlier_norm:Error, please provide an approved method for outlier removal for visualization.")
            raise RuntimeError("991")                                    # stop(991)
        obj.expr_data, (lo, hi) = api.remove_outliers_norm(obj.expr_data, want_bounds=True)
        log.info("outlier bounds defined between: %g - %g", lo, hi)
    else:
        log.error("::remove_outlier_norm:Error, must specify outmethod or define exact bounds")
        raise RuntimeError("992")                                        # stop(992)
    if obj.hspike is not None:
        log.info("-mirroring for hspike")
        obj.hspike = remove_outliers_norm(obj.hspike, out_method, lower_bound, upper_bound)
    return obj


def log2xplus1(infercnv_obj: Infercnv) -> Infercnv:
    """R/inferCNV_ops.R:2756-2769."""
    log.info("transforming log2xplus1()")
    obj = copy.copy(infercnv_obj)
    obj.expr_data = api.log2xplus1(obj.expr_data)
    if obj.hspike is not None:
        log.info("-mirroring for hspike")
        obj.hspike = log2xplus1(obj.hspike)
    return obj


def invert_log2(infercnv_obj: Infercnv) -> Infercnv:
    """R/inferCNV_ops.R:2814-2826."""
    log.info("invert_log2(), computing 2^x")
    obj = copy.copy(infercnv_obj)
    obj.expr_data = api.invert_log2(obj.expr_data)
    if obj.hspike is not None:
        log.info("-mirroring for hspike")
        obj.hspike = invert_log2(obj.hspike)
    return obj


def apply_max_threshold_bounds(infercnv_obj: Infercnv, threshold: float) -> Infercnv:
    """R/inferCNV_ops.R:2970-2983."""
    log.info("::process_data:setting max centered expr, threshold set to: +/-: %s", threshold)
    obj = copy.copy(infercnv_obj)
    obj.expr_data = api.apply_max_threshold_bounds(obj.expr_data, threshold)
    if obj.hspike is not None:
        log.info("-mirroring for hspike")
        obj.hspike = apply_max_threshold_bounds(obj.hspike, threshold)
    return obj


def smooth_by_chromosome(infercnv_obj: Infercnv, window_length: int, smooth_ends: bool = True) -> Infercnv:
    """R/inferCNV_ops.R:2406-2434 (`smooth_ends` is accepted and ignored there too, SURVEY Q13)."""
    obj = copy.copy(infercnv_obj)
    if window_length < 2:
        log.warning("window length < 2, returning original unmodified data")      # ops.R:2444-2447
    cs, cl = obj.chr_ranges()
    obj.expr_data = api.smooth(obj.expr_data, cs, cl, window_length)
    if obj.hspike is not None:
        log.info("-mirroring for hspike")
        obj.hspike = smooth_by_chromosome(obj.hspike, window_length, smooth_ends)
    return obj


def smooth_by_chromosome_coordinates(infercnv_obj: Infercnv, window_length: float) -> Infercnv:
    """R/inferCNV_ops.R:2534-2622: every gene's value becomes the weighted mean over the genes of its chromosome within
    window_length of its midpoint (gene_order_start / gene_order_stop), with R's padding and recycling; the hidden spike is
    mirrored with window_length = 51 as in the original."""
    obj = copy.copy(infercnv_obj)
    if obj.gene_order_start is None or obj.gene_order_stop is None:
        raise ValueError("smooth_by_chromosome_coordinates needs gene_order_start and gene_order_stop")
    cs, cl = obj.chr_ranges()
    for s, n in zip(cs, cl):
        log.info("smooth_by_chromosome: chr: %s", _chr_label(obj, obj.gene_order_chr[s]))
        if n > 1 and window_length < 2:
            log.warning("window length < 2, returning original unmodified data")      # ops.R:2568-2571
    obj.expr_data = api.smooth_coordinates(obj.expr_data, cs, cl, obj.gene_order_start, obj.gene_order_stop, window_length)
    if obj.hspike is not None:
        log.info("-mirroring for hspike")
        obj.hspike = smooth_by_chromosome_coordinates(obj.hspike, window_length=51)
    return obj


def center_cell_expr_across_chromosome(infercnv_obj: Infercnv, method: str = "mean") -> Infercnv:
    """R/inferCNV_ops.R:2074-2088; any method other than "median" centres by the mean (:2096-2107)."""
    log.info("::center_smooth across chromosomes per cell")
    obj = copy.copy(infercnv_obj)
    obj.expr_data = api.center(obj.expr_data, "median" if method == "median" else "mean")
    if obj.hspike is not None:
        log.info("-mirroring for hspike")
        obj.hspike = center_cell_expr_across_chromosome(obj.hspike, method)
    return obj


def smooth_block(infercnv_obj: Infercnv, window_length: int = 101, max_centered_threshold: float = 3.0,
                 apply_log: bool = True, use_bounds: bool = True) -> Infercnv:
    """run() steps 4, 8, 9, 10, 11, 12, 14 in one library call (R/inferCNV_ops.R:614-1031), for the
    default option set (smooth_method="pyramidinal", ref_subtract_use_mean_bounds=TRUE)."""
    obj = copy.copy(infercnv_obj)
    cs, cl = obj.chr_ranges()
    obj.expr_data = api.smooth_block(obj.expr_data, cs, cl, _ref_groups(obj), apply_log=apply_log,
                                     threshold=max_centered_threshold, window_length=window_length,
                                     use_bounds=use_bounds)
    if obj.hspike is not None:
        obj.hspike = smooth_block(obj.hspike, window_length, max_centered_threshold, apply_log, use_bounds)
    return obj


def _hmm_groups(obj: Infercnv, analysis_mode: str, cluster_by_groups: bool) -> list:
    """The HMM lists of the group-mode drivers: unlist(tumor_subclusters$subclusters) for "subclusters"
    (predict_CNV_via_HMM_on_tumor_subclusters, HMM.R:345-408; without subclusters R falls back to whole samples with
    cluster_by_groups = TRUE), else the observation groups - one-cell groups when cluster_by_groups is FALSE - then the
    reference groups (..._on_whole_tumor_samples, HMM.R:509-567)."""
    if analysis_mode not in ("samples", "subclusters"):
        raise ValueError(f"analysis_mode {analysis_mode!r} has no HMM groups")
    if analysis_mode == "subclusters":
        if obj.tumor_subclusters is not None:
            return [np.asarray(idx) for sub in obj.tumor_subclusters["subclusters"].values() for idx in sub.values()]
        cluster_by_groups = True
    obs = [np.asarray(v) for v in obj.observation_grouped_cell_indices.values()]
    refs = [np.asarray(v) for v in obj.reference_grouped_cell_indices.values()]
    return (obs if cluster_by_groups else [np.asarray([c]) for c in np.concatenate(obs)]) + refs


def _states_object(obj: Infercnv, S: np.ndarray) -> Infercnv:
    out = copy.copy(obj)
    st = S.astype(np.float64)
    st[S == 255] = -1.0                          # the wire format's "unassigned" back to R's -1 (marshalling)
    out.expr_data = np.asfortranarray(st)
    return out


def smooth_block_hmm(infercnv_obj: Infercnv, analysis_mode: str, cnv_mean_sd: dict, cnv_level_to_mean_sd_fit: dict,
                     cluster_by_groups: bool = True, t: float = 1e-6, window_length: int = 101,
                     max_centered_threshold: float = 3.0, apply_log: bool = True, use_bounds: bool = True):
    """run() steps 4, 8-12, 14 and the i6 group-mode HMM of step 17 (predict_CNV_via_HMM_on_whole_tumor_samples or
    ..._on_tumor_subclusters on the block's output) in one library call, for analysis_mode "samples" and "subclusters"
    (random_trees subclusters, made before the block).  Returns (obj after step 14, states object); the hspike goes through
    the plain block."""
    obj = copy.copy(infercnv_obj)
    cs, cl = obj.chr_ranges()
    groups = _hmm_groups(obj, analysis_mode, cluster_by_groups)
    Pi, delta, mean, _ = get_HMM(cnv_mean_sd, t)
    sds = np.concatenate([_state_emission_sds(len(g), cnv_mean_sd, cnv_level_to_mean_sd_fit) for g in groups])
    Y, S = api.smooth_hmm(obj.expr_data, cs, cl, _ref_groups(obj), Pi, delta, mean, sds, apply_log=apply_log,
                          threshold=max_centered_threshold, window_length=window_length, use_bounds=use_bounds,
                          groups=groups)
    obj.expr_data = Y
    hmm_obj = _states_object(obj, S)
    if obj.hspike is not None:
        obj.hspike = smooth_block(obj.hspike, window_length, max_centered_threshold, apply_log, use_bounds)
    return obj, hmm_obj


def smooth_block_i3_hmm(infercnv_obj: Infercnv, window_length: int = 101, max_centered_threshold: float = 3.0,
                        apply_log: bool = True, use_bounds: bool = True, i3_p_val: float = 0.05, t: float = 1e-6,
                        median_filter_window: Optional[int] = None, analysis_mode: str = "cells",
                        cluster_by_groups: bool = True):
    """The i3 counterpart of smooth_block: run() steps 4, 8-12, 14, .i3HMM_get_sd_trend_by_num_cells_fit on the block's
    reference cells, the i3 HMM (i3HMM.R:180-389, use_KS = FALSE) and, with median_filter_window, the
    apply_median_filtering of that window (noise_reduction.R:43-113, the lists of apply_median_filtering below) - one library
    call.  analysis_mode "samples" / "subclusters" runs the group-mode HMM over the lists of smooth_block_hmm; the median
    filter is then a second call on the block's output.  Returns (obj after step 14, states object, median-filtered object
    or None, sd_trend); sd_trend's KS_delta is None (it comes from R's RNG)."""
    obj = copy.copy(infercnv_obj)
    cs, cl = obj.chr_ranges()
    lists = None
    if median_filter_window is not None:   # without tumor_subclusters (run() sets them at step 15) only references are listed
        subs = (obj.tumor_subclusters or {}).get("subclusters", {})
        lists = [np.asarray(idx) for tt in obj.observation_grouped_cell_indices for idx in subs.get(tt, {}).values()]
        lists += [np.asarray(idx) for idx in obj.reference_grouped_cell_indices.values()]
    if analysis_mode != "cells":
        Y, S, _, model = api.smooth_i3_hmm(obj.expr_data, cs, cl, _ref_groups(obj), i3_p_val=i3_p_val, t=t,
                                           apply_log=apply_log, threshold=max_centered_threshold,
                                           window_length=window_length, use_bounds=use_bounds,
                                           groups=_hmm_groups(obj, analysis_mode, cluster_by_groups))
        F = api.median_filter(Y, cs, cl, lists, median_filter_window) if lists is not None else None
    else:
        Y, S, F, model = api.smooth_i3_hmm(obj.expr_data, cs, cl, _ref_groups(obj), i3_p_val=i3_p_val, t=t,
                                           median_lists=lists, median_window=median_filter_window or 7,
                                           apply_log=apply_log, threshold=max_centered_threshold,
                                           window_length=window_length, use_bounds=use_bounds)
    obj.expr_data = Y
    hmm_obj = _states_object(obj, S)
    med_obj = None
    if F is not None:
        med_obj = copy.copy(obj)
        med_obj.expr_data = F
    if obj.hspike is not None:
        obj.hspike = smooth_block(obj.hspike, window_length, max_centered_threshold, apply_log, use_bounds)
    return obj, hmm_obj, med_obj, dict(model, KS_delta=None)


def apply_median_filtering(infercnv_obj: Infercnv, window_size: int = 7, on_observations: bool = True,
                           on_references: bool = True) -> Infercnv:
    """R/noise_reduction.R:43-89.  Observations are filtered per tumour subcluster, references per
    whole reference group, each in the order of its index list."""
    if window_size % 2 != 1 or window_size < 2:
        raise ValueError("::apply_median_filtering: Error, window_size is an even or < 2. "
                         "Please specify an odd number >= 3.")
    obj = copy.copy(infercnv_obj)
    lists = []
    if on_observations:
        for tumor_type in obj.observation_grouped_cell_indices:
            for idx in obj.tumor_subclusters["subclusters"][tumor_type].values():
                lists.append(np.asarray(idx))
    if on_references:
        for idx in obj.reference_grouped_cell_indices.values():
            lists.append(np.asarray(idx))
    cs, cl = obj.chr_ranges()
    obj.expr_data = api.median_filter(obj.expr_data, cs, cl, lists, window_size)
    return obj


# ---- HMM -----------------------------------------------------------------------------------------------

from infercnv_b200.hmm import CNV_LEVELS, get_HMM, i3HMM_get_HMM  # noqa: E402,F401  (parameter tables live in hmm.py)


def i3HMM_get_sd_trend_by_num_cells_fit(infercnv_obj: Infercnv, i3_p_val: float = 0.05) -> dict:
    """.i3HMM_get_sd_trend_by_num_cells_fit, R/inferCNV_i3HMM.R:17-80: mu / sigma over the
    reference cells (or all observation cells) on the GPU; mean_delta = |qnorm(p, 0, sigma)|.
    KS_delta (RNG-driven KS tests, :469-493) stays in R and is not provided."""
    from statistics import NormalDist
    groups = infercnv_obj.reference_grouped_cell_indices or infercnv_obj.observation_grouped_cell_indices
    cells = np.concatenate([np.asarray(v) for v in groups.values()])
    mu, sigma = api.mean_sd(infercnv_obj.expr_data, cells)
    mean_delta = abs(NormalDist(0.0, sigma).inv_cdf(i3_p_val))        # determine_mean_delta_via_Z, :435-445
    return {"mu": mu, "sigma": sigma, "mean_delta": mean_delta, "KS_delta": None}


def _state_emission_sds(num_cells: int, cnv_mean_sd: dict, cnv_level_to_mean_sd_fit: dict) -> np.ndarray:
    """.get_state_emission_params, R/inferCNV_HMM.R:586-614: sd = exp(predict(lm(log(sd) ~ log(num_cells)))).
    A fit is given as (intercept, slope) of that regression."""
    out = []
    for lvl in CNV_LEVELS:
        a, b = cnv_level_to_mean_sd_fit[lvl]
        out.append(np.exp(a + b * np.log(num_cells)))
    return np.array(out)


def _run_hmm(obj: Infercnv, Pi, delta, mean, sd, groups=None) -> Infercnv:
    cs, cl = obj.chr_ranges()
    states = api.viterbi(obj.expr_data, cs, cl, Pi, delta, mean, sd, groups=groups)
    out = copy.copy(obj)
    out.expr_data = np.asfortranarray(states, dtype=np.float64)   # the reference stores states as doubles
    return out


def predict_CNV_via_HMM_on_indiv_cells(infercnv_obj: Infercnv, cnv_mean_sd: dict, t: float = 1e-6) -> Infercnv:
    """R/inferCNV_HMM.R:284-324."""
    log.info("predict_CNV_via_HMM_on_indiv_cells()")
    Pi, delta, mean, sd = get_HMM(cnv_mean_sd, t)
    return _run_hmm(infercnv_obj, Pi, delta, mean, sd)


def predict_CNV_via_HMM_on_tumor_subclusters(infercnv_obj: Infercnv, cnv_mean_sd: dict,
                                             cnv_level_to_mean_sd_fit: dict, t: float = 1e-6) -> Infercnv:
    """R/inferCNV_HMM.R:345-408."""
    log.info("predict_CNV_via_HMM_on_tumor_subclusters")
    if infercnv_obj.tumor_subclusters is None:
        log.warning("No subclusters defined, so instead running on whole samples")
        return predict_CNV_via_HMM_on_whole_tumor_samples(infercnv_obj, True, cnv_mean_sd, cnv_level_to_mean_sd_fit, t)
    Pi, delta, mean, _ = get_HMM(cnv_mean_sd, t)
    groups = [np.asarray(idx) for sub in infercnv_obj.tumor_subclusters["subclusters"].values() for idx in sub.values()]
    sds = np.concatenate([_state_emission_sds(len(g), cnv_mean_sd, cnv_level_to_mean_sd_fit) for g in groups])
    return _run_hmm(infercnv_obj, Pi, delta, mean, sds, groups)


def predict_CNV_via_HMM_on_tumor_subclusters_per_chr(infercnv_obj: Infercnv, subclusters_per_chr, cnv_mean_sd: dict,
                                                     cnv_level_to_mean_sd_fit: dict, t: float = 1e-6) -> Infercnv:
    """R/inferCNV_HMM.R:412-487.  subclusters_per_chr: {chromosome code: [cell index arrays]} - a partition of the
    cells per chromosome (Leiden per chromosome in the reference).  One trace per (chromosome, subcluster) on its
    rowMeans, then every tumour subcluster takes its consensus state per gene (get_predicted_CNV_regions by
    "subcluster" + the overwrite loop, :470-483)."""
    log.info("predict_CNV_via_HMM_on_tumor_subclusters_per_chr")
    if subclusters_per_chr is None:
        log.warning("No subclusters defined, so instead running on whole samples")
        return predict_CNV_via_HMM_on_whole_tumor_samples(infercnv_obj, True, cnv_mean_sd, cnv_level_to_mean_sd_fit, t)
    Pi, delta, mean, _ = get_HMM(cnv_mean_sd, t)
    cs, cl = infercnv_obj.chr_ranges()
    per = [[np.asarray(g) for g in subclusters_per_chr[infercnv_obj.gene_order_chr[s]]] for s in cs]
    sds = np.concatenate([_state_emission_sds(len(g), cnv_mean_sd, cnv_level_to_mean_sd_fit) for p_ in per for g in p_])
    states = api.viterbi_per_chr(infercnv_obj.expr_data, cs, cl, per, Pi, delta, mean, sds)
    log.info("-done predicting CNV based on per chromosome subclusters")
    log.info("-calculating initial tumor subclusters CNV consensus based on per chromosome predictions")
    groups = [np.asarray(idx) for sub in infercnv_obj.tumor_subclusters["subclusters"].values() for idx in sub.values()]
    states = api.apply_state_consensus(states, cs, cl, groups)
    out = copy.copy(infercnv_obj)
    st = states.astype(np.float64)
    st[states == 255] = -1.0                     # the wire format's "unassigned" back to R's -1 (marshalling)
    out.expr_data = np.asfortranarray(st)
    return out


def predict_CNV_via_HMM_on_whole_tumor_samples(infercnv_obj: Infercnv, cluster_by_groups: bool, cnv_mean_sd: dict,
                                               cnv_level_to_mean_sd_fit: dict, t: float = 1e-6) -> Infercnv:
    """R/inferCNV_HMM.R:509-567."""
    log.info("predict_CNV_via_HMM_on_whole_tumor_samples")
    Pi, delta, mean, _ = get_HMM(cnv_mean_sd, t)
    obs = [np.asarray(v) for v in infercnv_obj.observation_grouped_cell_indices.values()]
    refs = [np.asarray(v) for v in infercnv_obj.reference_grouped_cell_indices.values()]
    # cluster_by_groups = FALSE: the reference's c(all_observations = unlist(obs), <reference list>) makes every observation
    # cell a list element of its own (R coerces the integer vector into the list): one-cell "samples"
    groups = (obs if cluster_by_groups else [np.asarray([c]) for c in np.concatenate(obs)]) + refs
    sds = np.concatenate([_state_emission_sds(len(g), cnv_mean_sd, cnv_level_to_mean_sd_fit) for g in groups])
    return _run_hmm(infercnv_obj, Pi, delta, mean, sds, groups)


def i3HMM_predict_CNV_via_HMM_on_indiv_cells(infercnv_obj: Infercnv, i3_p_val: float = 0.05,
                                             sd_trend: Optional[dict] = None, t: float = 1e-6,
                                             use_KS: bool = False) -> Infercnv:
    """R/inferCNV_i3HMM.R:180-225 (run() passes use_KS = HMM_i3_use_KS = FALSE, ops.R:274)."""
    if sd_trend is None:
        sd_trend = i3HMM_get_sd_trend_by_num_cells_fit(infercnv_obj, i3_p_val)
    Pi, delta, mean, sd = i3HMM_get_HMM(sd_trend, t, i3_p_val, use_KS)
    return _run_hmm(infercnv_obj, Pi, delta, mean, sd)


def i3HMM_predict_CNV_via_HMM_on_tumor_subclusters(infercnv_obj: Infercnv, i3_p_val: float = 0.05,
                                                   sd_trend: Optional[dict] = None, t: float = 1e-6,
                                                   use_KS: bool = False) -> Infercnv:
    """R/inferCNV_i3HMM.R:249-308: one trace per subcluster on rowMeans, shared sigma."""
    if sd_trend is None:
        sd_trend = i3HMM_get_sd_trend_by_num_cells_fit(infercnv_obj, i3_p_val)
    Pi, delta, mean, sd = i3HMM_get_HMM(sd_trend, t, i3_p_val, use_KS)
    groups = [np.asarray(idx) for sub in infercnv_obj.tumor_subclusters["subclusters"].values() for idx in sub.values()]
    return _run_hmm(infercnv_obj, Pi, delta, mean, np.tile(sd, len(groups)), groups)


def i3HMM_predict_CNV_via_HMM_on_whole_tumor_samples(infercnv_obj: Infercnv, cluster_by_groups: bool = True,
                                                     i3_p_val: float = 0.05, sd_trend: Optional[dict] = None,
                                                     t: float = 1e-6, use_KS: bool = False) -> Infercnv:
    """R/inferCNV_i3HMM.R:332-389."""
    if sd_trend is None:
        sd_trend = i3HMM_get_sd_trend_by_num_cells_fit(infercnv_obj, i3_p_val)
    Pi, delta, mean, sd = i3HMM_get_HMM(sd_trend, t, i3_p_val, use_KS)
    obs = [np.asarray(v) for v in infercnv_obj.observation_grouped_cell_indices.values()]
    refs = [np.asarray(v) for v in infercnv_obj.reference_grouped_cell_indices.values()]
    # cluster_by_groups = FALSE: the reference's c(all_observations = unlist(obs), <reference list>) makes every observation
    # cell a list element of its own (R coerces the integer vector into the list): one-cell "samples"
    groups = (obs if cluster_by_groups else [np.asarray([c]) for c in np.concatenate(obs)]) + refs
    return _run_hmm(infercnv_obj, Pi, delta, mean, np.tile(sd, len(groups)), groups)


def assign_HMM_states_to_proxy_expr_vals(infercnv_obj: Infercnv) -> Infercnv:
    """R/inferCNV_HMM.R:1191-1206 (i6): state -> {0, 0.5, 1, 1.5, 2, 3}; other values (-1) are left as they are."""
    obj = copy.copy(infercnv_obj)
    obj.expr_data = api.assign_hmm_states_to_proxy_expr_vals(obj.expr_data, 6)
    return obj


def i3HMM_assign_HMM_states_to_proxy_expr_vals(infercnv_obj: Infercnv) -> Infercnv:
    """R/inferCNV_i3HMM.R:405-417: state -> {0.5, 1, 1.5}."""
    obj = copy.copy(infercnv_obj)
    obj.expr_data = api.assign_hmm_states_to_proxy_expr_vals(obj.expr_data, 3)
    return obj


# ---- CNV region reports (R/inferCNV_HMM.R:706-1087) ---------------------------------------------------------------

def _chr_label(obj: Infercnv, code) -> str:
    if obj.chr_names is not None:
        return str(obj.chr_names[code])
    return str(code)


def _cell_groups(obj: Infercnv, by: str):
    """get_predicted_CNV_regions, HMM.R:709-733: ordered (name, cell indices) pairs."""
    names = obj.cell_names if obj.cell_names is not None else [str(i) for i in range(obj.expr_data.shape[1])]
    refs, obs = obj.reference_grouped_cell_indices, obj.observation_grouped_cell_indices
    if by == "consensus":
        return [(n, np.asarray(v)) for n, v in list(refs.items()) + list(obs.items())]
    if by == "subcluster":          # unlist(tumor_subclusters[["subclusters"]], recursive=FALSE) -> "group.subcluster"
        return [("%s.%s" % (g, n), np.asarray(v)) for g, sub in obj.tumor_subclusters["subclusters"].items()
                for n, v in sub.items()]
    cells = [int(i) for v in list(refs.values()) + list(obs.values()) for i in v]
    return [(names[i], np.array([i])) for i in cells]


def get_predicted_CNV_regions(infercnv_obj: Infercnv, by: str = "consensus") -> list:
    """R/inferCNV_HMM.R:706-764 on an object whose expr_data holds the HMM states.  One entry per cell group:
    {"cell_group_name", "cells" (names), "cnv_ranges": {cnv_name, state, chr, start, end} (one row per region,
    .get_cnv_gene_region_bounds), "gene_regions": {first_gene, last_gene} (0-based inclusive gene ranges of the same
    regions; the per-gene data.frames of .define_cnv_gene_regions are these ranges of gene_order)}.
    Consensus, segmentation and bounds run in libinfercnv_b200 (icnv_predicted_cnv_regions_u8)."""
    if by not in ("consensus", "subcluster", "cell"):
        raise ValueError("'arg' should be one of 'consensus', 'subcluster', 'cell'")      # match.arg
    log.info("get_predicted_CNV_regions(%s)", by)
    obj = infercnv_obj
    if obj.tumor_subclusters is None:
        log.warning("get_predicted_CNV_regions() - no subclusters defined, resetting reporting mode to consensus")
        by = "consensus"
    if obj.gene_order_start is None or obj.gene_order_stop is None:
        raise ValueError("gene_order start / stop are needed for the region bounds")
    groups = _cell_groups(obj, by)
    names = obj.cell_names if obj.cell_names is not None else [str(i) for i in range(obj.expr_data.shape[1])]
    cs, cl = obj.chr_ranges()
    chr_labels = [_chr_label(obj, obj.gene_order_chr[s]) if n > 0 else "" for s, n in zip(cs, cl)]
    for name, cells in groups:
        log.info("-processing cell_group_name: %s, size: %d", name, len(cells))
    reg = api.predicted_cnv_regions(obj.expr_data, cs, cl, obj.gene_order_start, obj.gene_order_stop,
                                    [c for _, c in groups])
    bounds = np.searchsorted(reg["seq"], np.arange(len(groups) + 1))      # records are ordered by group
    out = []
    for k, (name, cells) in enumerate(groups):
        a, b = int(bounds[k]), int(bounds[k + 1])
        chrs = [chr_labels[c] for c in reg["chr"][a:b]]
        out.append({
            "cell_group_name": name,
            "cells": [names[i] for i in cells],
            "cnv_ranges": {"cnv_name": ["%s-region_%d" % (ch, i + 1) for ch, i in zip(chrs, range(a, b))],
                           "state": reg["state"][a:b], "chr": chrs, "start": reg["start"][a:b], "end": reg["end"][a:b]},
            "gene_regions": {"first_gene": reg["first_gene"][a:b], "last_gene": reg["last_gene"][a:b]},
        })
    return out


def _num(v) -> str:
    """write.table: integer-valued numbers print without a decimal point, others with 15 significant digits."""
    return "%d" % v if float(v) == int(v) else "%.15g" % v


def generate_cnv_region_reports(infercnv_obj: Infercnv, output_filename_prefix: str, out_dir: str,
                                ignore_neutral_state=None, by: str = "consensus") -> None:
    """R/inferCNV_HMM.R:790-869: writes <prefix>.cell_groupings, .pred_cnv_regions.dat, .pred_cnv_genes.dat and
    .genes_used.dat as write.table(quote=FALSE, sep="\t") lays them out (the gene order file keeps its row names)."""
    cnv_regions = get_predicted_CNV_regions(infercnv_obj, by)
    obj = infercnv_obj
    G = obj.expr_data.shape[0]
    gene_names = obj.gene_names if obj.gene_names is not None else [str(i) for i in range(G)]
    gchr = [_chr_label(obj, c) for c in obj.gene_order_chr]
    gs, ge = [_num(v) for v in obj.gene_order_start], [_num(v) for v in obj.gene_order_stop]
    keep = (lambda st: True) if ignore_neutral_state is None else (lambda st: st != ignore_neutral_state)

    path = os.path.join(out_dir, output_filename_prefix + ".cell_groupings")
    log.info("-writing cell clusters file: %s", path)
    with open(path, "w") as f:
        f.write("cell_group_name\tcell\n")
        for g in cnv_regions:
            f.writelines("%s\t%s\n" % (g["cell_group_name"], c) for c in g["cells"])

    path = os.path.join(out_dir, output_filename_prefix + ".pred_cnv_regions.dat")
    log.info("-writing cnv regions file: %s", path)
    with open(path, "w") as f:
        f.write("cell_group_name\tcnv_name\tstate\tchr\tstart\tend\n")
        for g in cnv_regions:
            r = g["cnv_ranges"]
            f.writelines("%s\t%s\t%s\t%s\t%s\t%s\n" % (g["cell_group_name"], n, _num(st), ch, _num(a), _num(b))
                         for n, st, ch, a, b in zip(r["cnv_name"], r["state"], r["chr"], r["start"], r["end"]) if keep(st))

    if by == "cell":
        log.warning("Note, HMM reporting is being done by 'cell', so this may use more memory, write more info to disk, "
                    "take more time, ...")
    path = os.path.join(out_dir, output_filename_prefix + ".pred_cnv_genes.dat")
    log.info("-writing per-gene cnv report: %s", path)
    with open(path, "w") as f:
        f.write("cell_group_name\tgene_region_name\tstate\tgene\tchr\tstart\tend\n")
        for g in cnv_regions:
            r, gr = g["cnv_ranges"], g["gene_regions"]
            for n, st, a, b in zip(r["cnv_name"], r["state"], gr["first_gene"], gr["last_gene"]):
                if keep(st):
                    head = "%s\t%s\t%s\t" % (g["cell_group_name"], n, _num(st))
                    f.writelines(head + "%s\t%s\t%s\t%s\n" % (gene_names[i], gchr[i], gs[i], ge[i])
                                 for i in range(int(a), int(b) + 1))

    path = os.path.join(out_dir, output_filename_prefix + ".genes_used.dat")
    log.info("-writing gene ordering info: %s", path)
    with open(path, "w") as f:
        f.write("chr\tstart\tstop\n")
        f.writelines("%s\t%s\t%s\t%s\n" % (gene_names[i], gchr[i], gs[i], ge[i]) for i in range(G))


# ---- gene filters on the raw counts (run() step 2) ------------------------------------------------------------------

def below_min_mean_expr_cutoff(expr_data, min_mean_expr) -> np.ndarray:
    """.below_min_mean_expr_cutoff, R/inferCNV_ops.R:2149-2158: (0-based) indices of the genes whose mean over all
    cells is below the cutoff."""
    _, _, means = api.gene_stats(expr_data)
    return np.flatnonzero(means < min_mean_expr)


def remove_genes(infercnv_obj: Infercnv, gene_indices_to_remove) -> Infercnv:
    """remove_genes, R/inferCNV.R:445-457: drops the rows from expr.data, count.data and gene_order."""
    obj = copy.copy(infercnv_obj)
    G = obj.expr_data.shape[0]
    mask = np.ones(G, dtype=bool)
    mask[np.asarray(gene_indices_to_remove, dtype=np.int64)] = False
    keep = np.flatnonzero(mask)
    obj.expr_data = api.remove_genes(obj.expr_data, keep)
    if obj.count_data is not None:
        obj.count_data = api.remove_genes(obj.count_data, keep)
    obj.gene_order_chr = np.asarray(obj.gene_order_chr)[keep]
    if obj.gene_names is not None:
        obj.gene_names = [obj.gene_names[i] for i in keep]
    if obj.gene_order_start is not None:
        obj.gene_order_start = np.asarray(obj.gene_order_start)[keep]
    if obj.gene_order_stop is not None:
        obj.gene_order_stop = np.asarray(obj.gene_order_stop)[keep]
    return obj


def require_above_min_mean_expr_cutoff(infercnv_obj: Infercnv, min_mean_expr_cutoff: float) -> Infercnv:
    """R/inferCNV_ops.R:2124-2144."""
    log.info("::above_min_mean_expr_cutoff:Start")
    indices = below_min_mean_expr_cutoff(infercnv_obj.expr_data, min_mean_expr_cutoff)
    if len(indices) > 0:
        log.info("Removing %d genes from matrix as below mean expr threshold: %g", len(indices), min_mean_expr_cutoff)
        infercnv_obj = remove_genes(infercnv_obj, indices)
        log.info("There are %d genes and %d cells remaining in the expr matrix.", *infercnv_obj.expr_data.shape)
    return infercnv_obj


def require_above_min_cells_ref(infercnv_obj: Infercnv, min_cells_per_gene: int) -> Infercnv:
    """R/inferCNV_ops.R:2177-2209: keeps the genes expressed (x > 0) in at least min_cells_per_gene cells."""
    _, n_pos, _ = api.gene_stats(infercnv_obj.expr_data)
    passed = np.flatnonzero(n_pos >= min_cells_per_gene)
    G = infercnv_obj.expr_data.shape[0]
    num_removed = G - len(passed)
    if num_removed > 0:
        log.info("Removed %d genes having fewer than %d min cells per gene = %g %% genes removed here", num_removed,
                 min_cells_per_gene, num_removed / G * 100)
        if num_removed == G:
            log.warning("::All genes removed! Must revisit your data..., cannot continue here.")
            raise RuntimeError("998")                                   # stop(998)
        mask = np.ones(G, dtype=bool)
        mask[passed] = False
        infercnv_obj = remove_genes(infercnv_obj, np.flatnonzero(mask))
    else:
        log.info("no genes removed due to min cells/gene filter")
    return infercnv_obj


def ingest_sparse_counts(p, i, x, n_genes, gene_order_chr, min_mean_expr_cutoff=None, min_cells_per_gene=None,
                         normalize_factor=None):
    """run() steps 2-3 on a compressed-sparse-column counts matrix (dgCMatrix @p / @i / @x, 0-based) without ever
    building the dense counts on the host: the mean-expression filter, then the min-cells filter on what is left
    (the order run() applies them in, ops.R:560-564), then depth normalisation over the kept genes.  Returns
    (expr_data dense kept-genes x cells, kept gene indices, chromosome codes of the kept genes)."""
    G = int(n_genes)
    _, n_pos, means = api.csc_gene_stats(p, i, x, G)
    keep = np.ones(G, dtype=bool)
    if min_mean_expr_cutoff is not None:
        keep &= ~(means < min_mean_expr_cutoff)
    if min_cells_per_gene is not None:        # per-gene statistic: removing other genes first does not change it
        passed = n_pos >= min_cells_per_gene
        if not np.any(keep & passed):
            raise RuntimeError("998")
        keep &= passed
    kept = np.flatnonzero(keep)
    expr = api.csc_normalize(p, i, x, G, keep=kept, normalize_factor=normalize_factor)
    return expr, kept, np.asarray(gene_order_chr)[kept]


# ---- optional steps inside the path: scaling (step 5) and chromosome-end removal (step 13) -----------------------------

def scale_infercnv_expr(infercnv_obj: Infercnv) -> Infercnv:
    """R/inferCNV_ops.R:3174-3186: t(scale(t(expr.data))), mirrored onto the hidden spike."""
    log.info("-scaling expr data")
    obj = copy.copy(infercnv_obj)
    obj.expr_data = api.scale_infercnv_expr(obj.expr_data)
    if obj.hspike is not None:
        log.info("-mirroring for hspike")
        obj.hspike = scale_infercnv_expr(obj.hspike)
    return obj


def _remove_tails(chr_idx, tail_length):
    """.remove_tails, R/inferCNV_ops.R:2370-2385: the indices of the first and last tail_length genes of a chromosome
    (a third of it each when the chromosome is shorter than two tails); nothing for tails or chromosomes below 3."""
    chr_idx = np.asarray(chr_idx)
    n = len(chr_idx)
    if tail_length < 3 or n < 3:
        return np.zeros(0, dtype=np.int64)
    if n < tail_length * 2:
        tail_length = n // 3
    tail_length = int(tail_length)
    return np.concatenate([chr_idx[:tail_length], chr_idx[n - tail_length:]])


def remove_genes_at_ends_of_chromosomes(infercnv_obj: Infercnv, window_length: int) -> Infercnv:
    """R/inferCNV_ops.R:3000-3045 (run() step 13 when remove_genes_at_chr_ends = TRUE): drops (window_length - 1) / 2
    genes at both ends of every chromosome from expr.data, count.data and gene_order."""
    contig_tail = (window_length - 1) / 2
    cs, cl = infercnv_obj.chr_ranges()
    remove = np.concatenate([_remove_tails(np.arange(s, s + n), contig_tail) for s, n in zip(cs, cl)] or [np.zeros(0, np.int64)])
    if len(remove) == 0:
        log.error("No genes removed at chr ends.... something wrong here")
        raise RuntimeError("1234")                                   # stop(1234)
    obj = remove_genes(infercnv_obj, remove)
    log.info("::process_data:Remove genes at chr ends, new dimensions (r,c) = %s", ",".join(map(str, obj.expr_data.shape)))
    if obj.hspike is not None:
        log.info("-mirroring for hspike")
        obj.hspike = remove_genes_at_ends_of_chromosomes(obj.hspike, window_length)
    return obj


# ---- ingest: CreateInfercnvObject's gene ordering (R/inferCNV.R:352-428) ----------------------------------------------

def order_reduce(data, data_gene_names, position_gene_names, chr, start, stop):
    """.order_reduce: keep the genes present both in the expression matrix and in the genomic position table, order
    them by (chromosome in order of first appearance in the table, start, stop), and reorder the matrix rows to match.
    The name matching and the sort are index bookkeeping on the host; the matrix rows are gathered by the library.
    Returns {"expr", "gene_names", "chr", "start", "stop"} or None values when nothing matches (the reference returns
    list(expr=NULL, order=NULL, chr_order=NULL))."""
    log.info("::order_reduce:Start.")
    none = {"expr": None, "gene_names": None, "chr": None, "start": None, "stop": None}
    if data is None or position_gene_names is None:
        return none
    chr, start, stop = np.asarray(chr), np.asarray(start), np.asarray(stop)
    pos_names = list(position_gene_names)
    ok = (start + stop) != 0                                             # drop entries at position 0 (:364-370)
    pos_index = {}
    for i, n in enumerate(pos_names):
        if ok[i] and n not in pos_index:
            pos_index[n] = i
    data_index = {}
    for i, n in enumerate(data_gene_names):
        data_index.setdefault(n, i)
    keep = [n for n in dict.fromkeys(data_gene_names) if n in pos_index]  # intersect(): order of the first argument
    if not keep:
        log.info("::process_data:order_reduce:The position file and the expression file row (gene) names do not match.")
        return none
    levels = {c: k for k, c in enumerate(dict.fromkeys(chr[ok].tolist()))}     # factor levels = unique(chr), :398-400
    p_idx = np.array([pos_index[n] for n in keep])
    order = np.lexsort((stop[p_idx], start[p_idx], np.array([levels[c] for c in chr[p_idx].tolist()])))   # order(chr,start,stop)
    sel = p_idx[order]
    rows = np.array([data_index[keep[i]] for i in order], dtype=np.int32)
    return {"expr": api.gather_genes(data, rows), "gene_names": [keep[i] for i in order], "chr": chr[sel],
            "start": start[sel], "stop": stop[sel]}


# ---- distances for hclust() (parallelDist::parallelDist, an import of the reference: R/inferCNV_constants.R:27) -------------

def parallelDist(x, method: str = "euclidean", threads=None) -> np.ndarray:
    """`parallelDist(t(expr.data[, cells]), threads=...)` as the reference calls it before every hclust()
    (R/inferCNV_tumor_subclusters.R:191, R/inferCNV_ops.R:1930, ...): x is observations x variables (cells x genes), the
    result R's "dist" vector (strict lower triangle by columns).  Only the default method is on the GPU; `threads` is accepted
    and ignored like every other thread count on this path."""
    if method != "euclidean":
        raise NotImplementedError(f"parallelDist(method={method!r}): only 'euclidean' (the reference never passes another)")
    x = np.asarray(x, dtype=np.float64)
    if x.ndim != 2:
        raise ValueError("x must be a matrix (observations x variables)")
    return api.pairwise_dist_rows(x)


def nn2(data, k=None) -> dict:
    """`nn2(data, k = k)` as .leiden_simple_snn calls it (RANN::nn2, imported by the reference;
    R/inferCNV_tumor_subclusters.R:725-741) on observations x variables `data`, the query set being the data set: RANN's
    result, {"nn.idx": n x k 1-based, "nn.dists": n x k}, exact.  k defaults to min(10, nrow(data)) as in RANN."""
    data = np.asarray(data, dtype=np.float64)
    if data.ndim != 2:
        raise ValueError("data must be a matrix (observations x variables)")
    if k is None:
        k = min(10, data.shape[0])
    idx, dist = api.knn_rows(data, k)
    return {"nn.idx": idx + 1, "nn.dists": dist}


def leiden_seurat_preprocess_routine_graph(expr_data, k_nn=20):
    """The graph .leiden_seurat_preprocess_routine hands to cluster_leiden (R/inferCNV_tumor_subclusters.R:699-723):
    Seurat's infercnv_snn of the genes x cells `expr_data` (vst features, ScaleData, RunPCA(npcs = 10),
    FindNeighbors(k.param = k_nn)), exact, as a symmetric scipy.sparse.csr_matrix.  Leiden itself stays igraph's."""
    from scipy.sparse import csr_matrix
    r = api.seurat_snn(expr_data, k=k_nn)
    n = len(r.indptr) - 1
    return csr_matrix((r.data, r.indices, r.indptr), shape=(n, n))


def hclust(d, method: str = "complete", members=None) -> dict:
    """`hclust(d, method)` as infercnv calls it (fastcluster::hclust, imported by the reference; R/inferCNV_ops.R:262 passes
    "ward.D2" by default) on a "dist" vector such as parallelDist()'s.  Returns a dict shaped like R's "hclust" object:
    merge ((n - 1) x 2), height, order (1-based), labels, method, dist.method.  centroid / median and `members` are not
    on the GPU."""
    if members is not None:
        raise NotImplementedError("hclust(members=...) is not on the GPU path")
    d = np.ascontiguousarray(d, dtype=np.float64).ravel()
    big = d.size > api.HCLUST_NMAX * (api.HCLUST_NMAX - 1) // 2   # past the square matrix: the packed-triangle linkage
    merge, height, order = (api.hclust_tri if big else api.hclust)(d, method)
    return {"merge": merge, "height": height, "order": order, "labels": None, "method": method, "dist.method": "euclidean"}


def cluster_groups(expr_data, groups, method: str = "ward.D2", keep=None) -> list:
    """`hclust(parallelDist(t(expr_data[keep, g])), method)` for every cell list g of `groups`, as (merge, height, order) in
    group order: the groups of at most api.HCLUST_NMAX cells in one api.cluster_groups call, each larger one through
    api.cluster_cells (the packed-triangle linkage, bounded by device memory).  Both return the same bits where both run."""
    big = [len(g) > api.HCLUST_NMAX for g in groups]
    small = [g for g, b in zip(groups, big) if not b]
    small = api.cluster_groups(expr_data, small, method=method, keep=keep) if small else []
    it = iter(small)
    return [api.cluster_cells(expr_data, g, method=method, keep=keep) if b else next(it) for g, b in zip(groups, big)]


def runmean(x, k) -> np.ndarray:
    """`caTools::runmean(x, k)` with its defaults (endrule "mean", align "center") as infercnv applies it, column by
    column (`apply(m, 2, caTools::runmean, k = k)`): a vector or a genes x cells matrix (icnv_runmean_f64)."""
    x = np.asarray(x, dtype=np.float64)
    if x.ndim == 1:
        return api.runmean(x[:, None], k)[:, 0]
    return api.runmean(x, k)


def parameterize_random_cluster_heights_smoothed_trees(expr_matrix, hclust_method, window_size, n_perm=100, seed=0) -> dict:
    """`.parameterize_random_cluster_heights_smoothed_trees(expr_matrix, hclust_method, window_size)`
    (R/inferCNV_tumor_subclusters.random_smoothed_trees.R:217-304) on the genes x cells clade matrix: the reference's list
    fields h_obs (as hclust() returns it), max_h and rand_max_height_dist (n_perm maxima, 100 in the reference).  The
    permutations come from the library's own generator at `seed` - the same distribution as R's sample(), not its draws."""
    merge, height, order, perm_max = api.random_tree_heights(expr_matrix, window=window_size, method=hclust_method,
                                                             n_perm=n_perm, seed=seed)
    h_obs = {"merge": merge, "height": height, "order": order, "labels": None, "method": hclust_method,
             "dist.method": "euclidean"}
    return {"h_obs": h_obs, "max_h": float(height.max()), "rand_max_height_dist": perm_max}


def cutree(merge, height, k=None, h=None) -> np.ndarray:
    """stats::cutree(tree, k = k, h = h) on a tree as hclust() returns it: the group (1-based) of every observation.  With h,
    the merges of height <= h are applied (k = n + 1 - which.max(c(height, Inf) > h)); with k, the first n - k merges.  Groups
    are numbered by first appearance in observation order."""
    merge = np.asarray(merge)
    n = merge.shape[0] + 1
    if h is not None:
        k = n - int(np.argmax(np.append(np.asarray(height, dtype=np.float64), np.inf) > h))
    if k is None or not 1 <= k <= n:
        raise ValueError(f"cutree: k = {k} for {n} observations")
    lab = np.arange(n)                     # the observations' cluster representative, relabelled wholesale per merge
    rep = np.zeros(n, dtype=np.int64)      # merge s + 1 -> its representative
    for s in range(n - k):
        a, b = (int(v) for v in merge[s])
        ra = lab[-a - 1] if a < 0 else rep[a - 1]
        rb = lab[-b - 1] if b < 0 else rep[b - 1]
        lab[lab == ra] = rb
        rep[s] = rb
    _, first, inv = np.unique(lab, return_index=True, return_inverse=True)
    return np.argsort(np.argsort(first))[inv] + 1


def _assemble_subclusters(tumor_name: str, tumor_group_idx, order, grps) -> dict:
    # .single_tumor_subclustering (R/inferCNV_tumor_subclusters.R:236-257): tumor_group_idx[hc$order] cut into consecutive
    # runs, one per group of split(grps, grps) in group-id order, as long as that group
    ordered = np.asarray(tumor_group_idx)[np.asarray(order) - 1]
    ids, counts = np.unique(grps, return_counts=True)
    ends = np.cumsum(counts)
    return {f"{tumor_name}_s{g}": ordered[e - c:e] for g, c, e in zip(ids.tolist(), counts.tolist(), ends.tolist())}


def _r_mean_sd(x):
    # mean(x), sd(x) as R computes them: long-double sums with the refinement pass of mean() (summary.c, cov.c)
    x = np.asarray(x, dtype=np.float64).astype(np.longdouble)
    n = len(x)
    m = np.cumsum(x)[-1] / n
    m = m + np.cumsum(x - m)[-1] / n
    d = x - m
    return float(m), float(np.sqrt(np.float64(np.cumsum(d * d)[-1] / (n - 1))))


def define_signif_tumor_subclusters(infercnv_obj: Infercnv, p_val: float = 0.1, k_nn: int = 20, leiden_method="PCA",
                                    leiden_function="CPM", leiden_resolution="auto", leiden_method_per_chr="simple",
                                    leiden_function_per_chr="modularity", leiden_resolution_per_chr=1,
                                    hclust_method: str = "ward.D2", cluster_by_groups: bool = True,
                                    partition_method: str = "leiden", per_chr_hmm_subclusters: bool = False,
                                    per_chr_hmm_subclusters_references: bool = False, z_score_filter: float = 0.8,
                                    restrict_to_DE_genes: bool = False):
    """define_signif_tumor_subclusters (R/inferCNV_tumor_subclusters.R:2-177) for partition_method "none", "pheight" and
    "qnorm": returns (infercnv_obj with tumor_subclusters = {"hc": {group: hclust dict or None}, "subclusters": {group:
    {"<group>_s<id>": indices}}}, None), the hidden spike mirrored with partition_method "none".  The z-score gene filter
    (icnv_zscore_outlier_genes_f64) and every group's tree (icnv_cluster_groups_f64; a group above 65 536 cells through
    icnv_cluster_cells_f64) are GPU calls; the cut heights and
    cutree() are host arithmetic on the returned trees, as in R.  "qgamma" (fitdistrplus) and "leiden" (igraph's RNG) are not
    on this path, nor is restrict_to_DE_genes."""
    if partition_method in ("leiden", "qgamma"):
        raise NotImplementedError(f"partition_method={partition_method!r} is not on the GPU path")
    if partition_method not in ("none", "pheight", "qnorm"):
        raise ValueError("Error, not recognizing parition_method")
    if restrict_to_DE_genes:
        raise NotImplementedError("restrict_to_DE_genes is not on the GPU path")
    log.info("define_signif_tumor_subclusters(p_val=%g", p_val)
    obj = copy.copy(infercnv_obj)
    refs = obj.reference_grouped_cell_indices
    obs = obj.observation_grouped_cell_indices
    if cluster_by_groups:
        tumor_groups = {**obs, **refs}
    else:
        allobs = np.concatenate([np.asarray(v) for v in obs.values()]) if obs else np.zeros(0, np.int64)
        tumor_groups = {"all_observations": allobs, **refs}
    keep = None
    if z_score_filter > 0 and len(refs) > 0:
        ref_cells = np.concatenate([np.asarray(v) for v in refs.values()])
        outliers = api.zscore_outlier_genes(obj.expr_data, ref_cells)
        keep = np.flatnonzero(~outliers)   # expr.data[-which(...), ]: no outlier gene keeps no gene at all
        if not outliers.any():
            keep = keep[:0]
    names = list(tumor_groups)
    treed = [g for g in names if len(tumor_groups[g]) > 2]
    trees = dict(zip(treed, cluster_groups(obj.expr_data, [tumor_groups[g] for g in treed], method=hclust_method, keep=keep)))
    res = {"hc": {}, "subclusters": {}}
    for g in names:
        log.info("define_signif_tumor_subclusters(), tumor: %s", g)
        idx = np.asarray(tumor_groups[g])
        if g not in trees:
            res["hc"][g] = None
            res["subclusters"][g] = {f"{g}_s1": idx}
            continue
        merge, height, order = trees[g]
        labels = [obj.cell_names[i] for i in idx] if obj.cell_names is not None else None
        res["hc"][g] = {"merge": merge, "height": height, "order": order, "labels": labels, "method": hclust_method,
                        "dist.method": "euclidean"}
        if partition_method == "none":
            grps = cutree(merge, height, k=1)
        else:
            if partition_method == "pheight":
                cut = p_val * float(height.max())
            else:
                from scipy.stats import norm
                mu, sigma = _r_mean_sd(height)
                cut = float(norm.ppf(1 - p_val, loc=mu, scale=sigma))
            log.info("cut height based on p_val(%g) = %g and partition_method: %s", p_val, cut, partition_method)
            grps = cutree(merge, height, h=cut)
        res["subclusters"][g] = _assemble_subclusters(g, idx, order, grps)
        log.info("cut tree into: %d groups", len(res["subclusters"][g]))
    obj.tumor_subclusters = res
    if obj.hspike is not None:
        log.info("-mirroring for hspike")
        obj.hspike = define_signif_tumor_subclusters(obj.hspike, cluster_by_groups=True, partition_method="none")[0]
    return obj, None


def _tested_subclusters(infercnv_obj: Infercnv):
    """get_DE_genes_basic's loop (R/inferCNV_mask_non_DE.R:213-224): per observation group in order, its subclusters when
    they are a named list (a dict here), nothing when they are a plain index vector (R wraps it in an unnamed list)."""
    subs = (infercnv_obj.tumor_subclusters or {}).get("subclusters", {})
    names, lists = [], []
    for group in infercnv_obj.observation_grouped_cell_indices:
        v = subs.get(group)
        if isinstance(v, dict):
            for name, idx in v.items():
                names.append(name)
                lists.append(np.asarray(idx, dtype=np.int32))
    return names, lists


def get_DE_genes_basic(infercnv_obj: Infercnv, p_val_thresh: float = 0.05, test_use: str = "wilcoxon", seed: int = 0) -> dict:
    """`get_DE_genes_basic` (R/inferCNV_mask_non_DE.R:158-259): {"<subcluster>,<reference group>": {tumor_indices, normal,
    pvals (BH-adjusted), de_genes (gene indices with pvals < p_val_thresh)}} in R's pair order, with R's two messages per
    pair.  The Wilcoxon jitter comes from the library's generator at `seed`."""
    refs = list(infercnv_obj.reference_grouped_cell_indices.items())
    names, lists = _tested_subclusters(infercnv_obj)
    _, _, p_adj = api.mask_non_de_genes(infercnv_obj.expr_data, [np.asarray(v) for _, v in refs], lists, test=test_use,
                                        p_val_thresh=p_val_thresh, seed=seed, want_y=False)
    out = {}
    for s, (name, idx) in enumerate(zip(names, lists)):
        for j, (normal, _) in enumerate(refs):
            log.info("Finding DE genes between %s and %s", name, normal)
            p = p_adj[:, s * len(refs) + j]
            genes = np.flatnonzero(p < p_val_thresh)
            log.info("Found %d genes / %d total as DE", len(genes) + int(np.isnan(p).sum()), len(p))
            out[f"{name},{normal}"] = {"tumor_indices": idx, "normal": normal, "pvals": p, "de_genes": genes}
    return out


def mask_non_DE_genes_basic(infercnv_obj: Infercnv, p_val_thresh: float = 0.05, test_use: str = "wilcoxon",
                            center_val: Optional[float] = None, require_DE_all_normals: str = "any",
                            seed: int = 0) -> Infercnv:
    """`mask_non_DE_genes_basic` (R/inferCNV_mask_non_DE.R:28-52): entries of genes not DE against the reference groups (by
    require_DE_all_normals) set to center_val (default: the mean of expr.data), one GPU call (icnv_mask_non_de_f64)."""
    if require_DE_all_normals not in api.DE_RULES:
        raise ValueError(f"Error, not recognizing require_DE_all_normals={require_DE_all_normals}")
    refs = [np.asarray(v) for v in infercnv_obj.reference_grouped_cell_indices.values()]
    names, lists = _tested_subclusters(infercnv_obj)
    Y, _, p_adj = api.mask_non_de_genes(infercnv_obj.expr_data, refs, lists, test=test_use, p_val_thresh=p_val_thresh,
                                        rule=require_DE_all_normals, center_val=center_val, seed=seed)
    for s, name in enumerate(names):
        for j, normal in enumerate(infercnv_obj.reference_grouped_cell_indices):
            p = p_adj[:, s * len(refs) + j]
            log.info("Finding DE genes between %s and %s", name, normal)
            log.info("Found %d genes / %d total as DE", int((p < p_val_thresh).sum() + np.isnan(p).sum()), len(p))
    out = copy.copy(infercnv_obj)
    out.expr_data = Y
    return out


def cell_gene_from_regions(regions: list, cell_names=None, HMM_type: str = "i6") -> list:
    """inferCNVBayesNet's @cell_gene (initializeObject / getGenesCells, R/inferCNV_BayesNet.R:245-339) from
    get_predicted_CNV_regions' report, as R reads it back from the step-17 files: the per-gene file is written with
    ignore_neutral_state (R/inferCNV_ops.R:1316), so regions in the neutral state (3 for i6, 2 for i3) are not there; the
    remaining regions in file order, group by group.  Per region {"cnv_regions": name, "Genes": 0-based rows of the
    region's genes in ascending order (which(rownames %in% genes)), "Cells": 0-based columns whose name is one of the
    group's cells, ascending (which(colnames %in% cells)), "State": the HMM state}.  Without cell_names the report's cell
    labels are the column indices."""
    if HMM_type not in ("i6", "i3"):
        raise ValueError("HMM_type must be 'i6' or 'i3'")
    neutral = 3 if HMM_type == "i6" else 2
    out = []
    for grp in regions:
        if cell_names is not None:
            cells = np.flatnonzero(np.isin(np.asarray(cell_names, dtype=object), np.asarray(list(grp["cells"]), dtype=object)))
        else:
            cells = np.unique(np.asarray([int(c) for c in grp["cells"]], dtype=np.int64))
        cells = cells.astype(np.int32)
        cr, gr = grp["cnv_ranges"], grp["gene_regions"]
        for i, name in enumerate(cr["cnv_name"]):
            if int(cr["state"][i]) == neutral:
                continue
            out.append({"cnv_regions": name, "Genes": np.arange(gr["first_gene"][i], gr["last_gene"][i] + 1, dtype=np.int32),
                        "Cells": cells, "State": int(cr["state"][i])})
    return out


def inferCNVBayesNet_sampling(expr_data, cell_gene: list, mu, sig, HMM_type: str = "i6", n_burn: int = 700,
                              n_keep: int = 1000, seed: int = 0) -> dict:
    """run_gibb_sampling for every region of `cell_gene` and getProbabilities (R/inferCNV_BayesNet.R:362-388, 1054-1107) in
    one GPU call (icnv_bayesnet_f64): {"cell_gene", "cnv_probabilities": per region the (chains x 1000) x m theta draws,
    "cell_probabilities": per region m x C' state frequencies, "HMM_type"}.  6 chains for i6, 3 for i3, chain c starting
    from state c; a region of one gene and several cells is R's single pseudo-cell.  Same posterior as JAGS, not its
    draws: they come from the library's generator at `seed`."""
    if HMM_type not in ("i6", "i3"):
        raise ValueError("HMM_type must be 'i6' or 'i3'")
    n_chains = 6 if HMM_type == "i6" else 3
    pooled = [len(r["Genes"]) == 1 and len(r["Cells"]) > 1 for r in cell_gene]
    res = api.bayesnet(expr_data, [r["Genes"] for r in cell_gene], [r["Cells"] for r in cell_gene], mu, sig, n_chains,
                       n_burn=n_burn, n_keep=n_keep, seed=seed, pooled=pooled)
    return {"cell_gene": list(cell_gene), "cnv_probabilities": res["theta"], "cell_probabilities": res["cell_probabilities"],
            "HMM_type": HMM_type}


def removeCNV(mcmc: dict, HMM_states: np.ndarray, BayesMaxPNormal: float):
    """removeCNV (R/inferCNV_BayesNet.R:562-629): every region whose mean theta of the normal state (3 for i6, 2 for i3)
    exceeds BayesMaxPNormal is set to the normal state over its genes x cells and dropped.  Returns (mcmc, HMM_states)."""
    normal = 3 if mcmc["HMM_type"] == "i6" else 2
    means = [np.asarray(t).mean(axis=0) for t in mcmc["cnv_probabilities"]]
    remove = [i for i, mt in enumerate(means) if mt[normal - 1] > BayesMaxPNormal]
    log.info("Attempting to removing CNV(s) with a probability of being normal above  %s", BayesMaxPNormal)
    log.info("Removing  %d  CNV(s) identified by the HMM.", len(remove))
    if not remove:
        return mcmc, HMM_states
    S = HMM_states.copy()
    for i in remove:
        cg = mcmc["cell_gene"][i]
        S[np.ix_(cg["Genes"], cg["Cells"])] = normal
    keep = [i for i in range(len(means)) if i not in set(remove)]
    out = dict(mcmc)
    for k in ("cell_gene", "cnv_probabilities", "cell_probabilities"):
        out[k] = [mcmc[k][i] for i in keep]
    log.info("Total CNV's after removing:  %d", len(out["cell_gene"]))
    return out, S


def reassignCNV(mcmc: dict, HMM_states: np.ndarray):
    """reassignCNV (R/inferCNV_BayesNet.R:491-539): each region's state becomes the first arg-max of its mean theta,
    written over its genes x cells.  Returns (mcmc, HMM_states)."""
    log.info("Reassigning CNVs based on state probabilities.")
    S = HMM_states.copy()
    out = dict(mcmc)
    out["cell_gene"] = []
    for cg, th in zip(mcmc["cell_gene"], mcmc["cnv_probabilities"]):
        mt = np.asarray(th).mean(axis=0)
        state = int(np.flatnonzero(mt == mt.max())[0]) + 1
        S[np.ix_(cg["Genes"], cg["Cells"])] = state
        out["cell_gene"].append(dict(cg, State=state))
    return out, S
