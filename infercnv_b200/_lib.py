"""ctypes loader for libinfercnv_b200.so (the C ABI of include/infercnv_b200.h).

There is no CPU fallback anywhere in this package: if the shared library is missing, or no
CUDA device is usable, the calls raise.
"""
from __future__ import annotations

import ctypes as ct
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libinfercnv_b200.so")

c_d_p = ct.c_void_p   # pointers are passed as integers (numpy .ctypes.data / torch .data_ptr())
c_i64 = ct.c_int64
c_int = ct.c_int

# name -> (restype, argtypes); mirrors include/infercnv_b200.h one to one
_P = ct.c_void_p
SIGNATURES = {
    "icnv_init": (c_int, [c_int]),
    "icnv_init_devices": (c_int, [c_int, _P]),
    "icnv_devices_in_use": (c_int, []),
    "icnv_set_host_threads": (c_int, [c_int]),
    "icnv_shutdown": (None, []),
    "icnv_device_count": (c_int, []),
    "icnv_last_error": (ct.c_char_p, []),
    "icnv_version": (ct.c_char_p, []),
    "icnv_launch_count": (c_i64, []),
    "icnv_set_hmm_mode": (c_int, [c_int]),
    "icnv_hmm_rerun_count": (c_i64, []),
    "icnv_hmm_second_pass_count": (c_i64, []),
    "icnv_ref_means_f64": (c_int, [_P, c_i64, c_i64, _P, _P, c_int, c_int, _P]),
    "icnv_subtract_ref_f64": (c_int, [_P, _P, c_i64, c_i64, _P, c_int, c_int]),
    "icnv_smooth_f64": (c_int, [_P, _P, c_i64, c_i64, _P, _P, c_int, c_int]),
    "icnv_center_f64": (c_int, [_P, _P, c_i64, c_i64, c_int]),
    "icnv_normalize_counts_by_seq_depth_f64": (c_int, [_P, _P, c_i64, c_i64, ct.c_double]),
    "icnv_clear_noise_via_ref_mean_sd_f64": (c_int, [_P, _P, c_i64, c_i64, _P, c_i64, ct.c_double]),
    "icnv_log2xplus1_f64": (c_int, [_P, _P, c_i64]),
    "icnv_invert_log2_f64": (c_int, [_P, _P, c_i64]),
    "icnv_apply_max_threshold_bounds_f64": (c_int, [_P, _P, c_i64, ct.c_double]),
    "icnv_smooth_block_f64": (c_int, [_P, _P, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, c_int, ct.c_double, c_int,
                                      c_int]),
    "icnv_smooth_hmm_f64": (c_int, [_P, _P, _P, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, c_int, ct.c_double, c_int, c_int,
                                    c_int, _P, _P, _P, _P]),
    "icnv_smooth_hmm_u8_f64": (c_int, [_P, _P, _P, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, c_int, ct.c_double, c_int,
                                       c_int, c_int, _P, _P, _P, _P]),
    "icnv_smooth_i3_hmm_u8_f64": (c_int, [_P, _P, _P, _P, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, c_int, ct.c_double,
                                          c_int, c_int, ct.c_double, ct.c_double, _P, _P, c_int, c_int, _P]),
    "icnv_smooth_hmm_groups_u8_f64": (c_int, [_P, _P, _P, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, c_int, ct.c_double,
                                              c_int, c_int, _P, _P, c_int, c_int, _P, _P, _P, _P]),
    "icnv_smooth_i3_hmm_groups_u8_f64": (c_int, [_P, _P, _P, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, c_int, ct.c_double,
                                                 c_int, c_int, _P, _P, c_int, ct.c_double, ct.c_double, _P]),
    "icnv_viterbi_f64": (c_int, [_P, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, c_int, _P, _P, _P, _P, _P, _P]),
    "icnv_viterbi_u8_f64": (c_int, [_P, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, c_int, _P, _P, _P, _P, _P, _P]),
    "icnv_median_filter_f64": (c_int, [_P, _P, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, c_int]),
    "icnv_mean_sd_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, _P, _P]),
    "icnv_pairwise_dist_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, _P]),
    "icnv_dev_pairwise_dist_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, _P, _P]),
    "icnv_pairwise_dist_rows_f64": (c_int, [_P, c_i64, c_i64, _P]),
    "icnv_dev_pairwise_dist_rows_f64": (c_int, [_P, c_i64, c_i64, c_i64, _P, _P]),
    "icnv_knn_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, c_int, _P, _P]),
    "icnv_knn_rows_f64": (c_int, [_P, c_i64, c_i64, c_int, _P, _P]),
    "icnv_dev_knn_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, c_int, _P, _P, _P]),
    "icnv_hclust_f64": (c_int, [_P, c_i64, c_int, _P, _P, _P]),
    "icnv_dev_hclust_f64": (c_int, [_P, c_i64, c_int, _P, _P, _P]),
    "icnv_hclust_order": (c_int, [_P, c_i64, _P]),
    "icnv_hclust_tri_f64": (c_int, [_P, c_i64, c_int, _P, _P, _P]),
    "icnv_dev_hclust_tri_f64": (c_int, [_P, c_i64, c_int, _P, _P, _P]),
    "icnv_cluster_cells_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, _P, c_i64, c_int, _P, _P, _P]),
    "icnv_dev_cluster_cells_f64": (c_int, [_P, c_i64, c_i64, c_i64, _P, c_i64, _P, c_i64, c_int, _P, _P, _P]),
    "icnv_runmean_f64": (c_int, [_P, _P, c_i64, c_i64, _P, _P, c_int, c_int]),
    "icnv_random_tree_heights_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, c_int, c_int, c_int, ct.c_uint64, _P, _P, _P, _P]),
    "icnv_dev_random_tree_heights_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, c_int, c_int, c_int, ct.c_uint64, _P, _P, _P, _P]),
    "icnv_debug_random_trees": (c_int, [_P]),
    "icnv_zscore_outlier_genes_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, _P]),
    "icnv_dev_zscore_outlier_genes_f64": (c_int, [_P, c_i64, _P, c_i64, _P, _P]),
    "icnv_cluster_groups_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, _P, _P, c_int, c_int, _P, _P, _P]),
    "icnv_dev_cluster_groups_f64": (c_int, [_P, c_i64, c_i64, c_i64, _P, c_i64, _P, _P, c_int, c_int, _P, _P, _P]),
    "icnv_debug_cluster_groups": (c_int, [_P]),
    "icnv_seurat_snn_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, c_int, c_int, c_int, _P]),
    "icnv_dev_seurat_snn_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, c_int, c_int, c_int, _P, _P]),
    "icnv_seurat_snn_fetch": (c_int, [_P, _P, _P, _P, _P, _P]),
    "icnv_debug_seurat_snn": (c_int, [_P]),
    "icnv_mask_non_de_f64": (c_int, [_P, _P, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, c_int, ct.c_double, c_int,
                                     ct.c_double, ct.c_double, ct.c_double, ct.c_uint64, _P, _P]),
    "icnv_dev_mask_non_de_f64": (c_int, [_P, c_i64, _P, c_i64, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, c_int, ct.c_double,
                                         c_int, ct.c_double, ct.c_double, ct.c_double, ct.c_uint64, _P, _P, _P]),
    "icnv_debug_mask_non_de": (c_int, [_P]),
    "icnv_dev_de_pack_f64": (c_int, [_P, c_i64, _P, c_i64, c_int, _P, _P, _P, _P, _P]),
    "icnv_dev_de_place_f64": (c_int, [_P, c_i64, c_int, _P, _P, c_i64, _P, _P]),
    "icnv_dev_de_slab_tests_f64": (c_int, [_P, c_i64, c_i64, c_i64, _P, c_int, _P, c_int, c_int, ct.c_double, ct.c_double,
                                           ct.c_uint64, _P, c_i64, _P]),
    "icnv_dev_de_bh_mask_f64": (c_int, [_P, c_i64, c_int, c_int, _P, ct.c_double, _P, _P, c_i64, _P, c_i64, c_i64, _P, c_i64,
                                        _P, _P, c_int, ct.c_double, _P]),
    "icnv_bayesnet_f64": (c_int, [_P, c_i64, c_i64, _P, _P, _P, _P, _P, c_int, c_int, _P, _P, c_int, c_int, c_int, ct.c_uint64,
                                  _P, _P, _P]),
    "icnv_dev_bayesnet_f64": (c_int, [_P, c_i64, c_i64, c_i64, _P, _P, _P, _P, _P, c_int, c_int, _P, _P, c_int, c_int, c_int,
                                      ct.c_uint64, _P, _P, _P, _P]),
    "icnv_debug_bayesnet": (c_int, [_P]),
    "icnv_smooth_coordinates_f64": (c_int, [_P, _P, c_i64, c_i64, _P, _P, c_int, _P, _P, ct.c_double]),
    "icnv_dev_smooth_coordinates_f64": (c_int, [_P, c_i64, _P, c_i64, c_i64, c_i64, _P, _P, c_int, _P, _P, ct.c_double, _P]),
    "icnv_dev_group_partial_sums_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, c_int, c_int, _P, _P]),
    "icnv_dev_combine_partials_f64": (c_int, [_P, c_i64, c_i64, c_i64, _P, _P]),
    "icnv_dev_bounds_from_partials_f64": (c_int, [_P, c_i64, c_int, c_i64, c_int, _P, _P, _P, _P, _P, _P]),
    "icnv_dev_means_from_partials_f64": (c_int, [_P, c_i64, c_int, c_i64, c_int, _P, _P, _P, _P]),
    "icnv_dev_scatter_group_states_u8": (c_int, [_P, c_i64, c_i64, _P, _P, _P]),
    "icnv_dev_bounds_from_means_f64": (c_int, [_P, c_i64, c_int, _P, _P, _P, _P]),
    "icnv_dev_cell_pipeline_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, _P, c_i64, _P, _P, c_int, c_int, _P, _P, _P,
                                           ct.c_double, c_int, c_int, _P, _P, _P, c_int, _P, _P]),
    "icnv_debug_cell_kernel": (c_int, [_P]),
    "icnv_dev_smooth_block_f64": (c_int, [_P, _P, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, c_int, ct.c_double,
                                          c_int, c_int, _P]),
    "icnv_dev_viterbi_f64": (c_int, [_P, c_i64, c_i64, _P, _P, c_int, c_int, _P, _P, _P, _P, c_int, _P, _P, _P, _P]),
    "icnv_combine_cell_stats": (None, [_P, _P, c_i64, c_i64, _P, _P]),
    "icnv_dev_column_stats_f64": (c_int, [_P, c_i64, _P, c_i64, _P, _P, _P]),
    "icnv_dev_median_filter_f64": (c_int, [_P, _P, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, c_int, _P]),
    "icnv_assign_hmm_states_to_proxy_expr_vals_f64": (c_int, [_P, _P, c_i64, c_int]),
    "icnv_remove_outliers_norm_f64": (c_int, [_P, _P, c_i64, c_i64, ct.c_double, ct.c_double, _P]),
    "icnv_clear_noise_f64": (c_int, [_P, _P, c_i64, c_i64, _P, c_i64, ct.c_double, c_int]),
    "icnv_clear_noise_via_ref_mean_sd_logistic_f64": (c_int, [_P, _P, c_i64, c_i64, _P, c_i64, ct.c_double]),
    "icnv_gene_stats_f64": (c_int, [_P, c_i64, c_i64, _P, _P, _P]),
    "icnv_scale_infercnv_expr_f64": (c_int, [_P, _P, c_i64, c_i64]),
    "icnv_gather_genes_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, _P]),
    "icnv_remove_genes_f64": (c_int, [_P, c_i64, c_i64, _P, c_i64, _P]),
    "icnv_csc_gene_stats_f64": (c_int, [_P, _P, _P, c_i64, c_i64, _P, _P, _P]),
    "icnv_csc_normalize_f64": (c_int, [_P, _P, _P, c_i64, c_i64, _P, c_i64, ct.c_double, _P, _P]),
    "icnv_viterbi_per_chr_u8_f64": (c_int, [_P, c_i64, c_i64, _P, _P, c_int, _P, _P, _P, c_int, _P, _P, _P, _P, _P]),
    "icnv_apply_state_consensus_u8": (c_int, [_P, c_i64, c_i64, _P, _P, c_int, _P, _P, c_int, _P]),
    "icnv_state_consensus_u8": (c_int, [_P, c_i64, c_i64, _P, _P, c_int, _P]),
    "icnv_cnv_regions_u8": (c_int, [_P, c_i64, c_i64, _P, _P, c_int, _P, _P, _P]),
    "icnv_predicted_cnv_regions_u8": (c_int, [_P, c_i64, c_i64, _P, _P, c_int, _P, _P, _P, _P, c_int, _P, _P]),
    "icnv_cnv_regions_fetch": (c_int, [c_i64, _P, _P, _P, _P, _P, _P, _P]),
    "icnv_dev_gene_stats_f64": (c_int, [_P, c_i64, c_i64, c_i64, _P, _P, _P]),
    "icnv_dev_gather_rows_f64": (c_int, [_P, c_i64, _P, c_i64, _P, c_i64, _P]),
    "icnv_dev_column_minmax_f64": (c_int, [_P, c_i64, c_i64, _P, _P, _P]),
    "icnv_dev_clamp_bounds_f64": (c_int, [_P, _P, c_i64, ct.c_double, ct.c_double, _P]),
    "icnv_dev_state_counts_u8": (c_int, [_P, c_i64, c_i64, _P, _P, c_int, _P, _P, _P]),
    "icnv_dev_consensus_from_counts": (c_int, [_P, c_i64, c_int, _P, _P]),
    "icnv_dev_state_consensus_u8": (c_int, [_P, c_i64, c_i64, _P, _P, c_int, _P, _P, _P]),
    "icnv_dev_cnv_regions_u8": (c_int, [_P, c_i64, c_i64, c_i64, _P, _P, _P, c_int, _P, _P, _P, _P]),
    "icnv_dev_cnv_regions_records": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P]),
    "icnv_dev_synth_f64": (c_int, [_P, c_i64, c_i64, c_i64, c_i64, _P, _P, c_int, ct.c_uint64, _P]),
}

_lib = None


class InfercnvB200Error(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"libinfercnv_b200 error {code}: {message}")
        self.code = code


def load() -> ct.CDLL:
    """dlopen the library and declare every prototype.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -m infercnv_b200.build` "
            "(needs nvcc; there is no CPU fallback)")
    lib = ct.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        raise InfercnvB200Error(rc, load().icnv_last_error().decode("utf-8", "replace"))
