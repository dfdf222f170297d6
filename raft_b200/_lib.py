"""ctypes binding of include/raft_b200.h.  No fallback: a missing library is an error."""
from __future__ import annotations

import ctypes
import os

from . import _build

_lib = None

# every symbol include/raft_b200.h declares
SYMBOLS = [
    "b2d_version", "b2d_last_error", "b2d_set_option", "b2d_debug_nn_stats", "b2d_pairwise_workspace_bytes", "b2d_pairwise_distance",
    "b2d_fused_l2_nn_workspace_bytes", "b2d_fused_l2_nn", "b2d_fused_distance_nn", "b2d_fused_l2_nn_keys",
    "b2d_fused_l2_nn_finalize", "b2d_row_norm", "b2d_knn_l2_workspace_bytes", "b2d_knn_l2", "b2d_knn",
    "b2d_silhouette_score_workspace_bytes", "b2d_silhouette_score",
    "b2d_trustworthiness_score_workspace_bytes", "b2d_trustworthiness_score", "b2d_profile_begin", "b2d_profile_end",
    "b2d_row_argmin", "b2d_fused_l2_nn_multi", "b2d_masked_l2_nn_workspace_bytes", "b2d_masked_l2_nn",
    "b2d_select_k_workspace_bytes", "b2d_select_k", "b2d_eps_neighbors_l2sq_workspace_bytes", "b2d_eps_neighbors_l2sq",
    "b2d_gram_matrix_workspace_bytes", "b2d_gram_matrix", "b2d_kmeans_workspace_bytes", "b2d_kmeans_fit",
    "b2d_kmeans_predict", "b2d_kmeans_update_centroids", "b2d_kmeans_init_plus_plus", "b2d_kmeans_scalable_workspace_bytes",
    "b2d_kmeans_init_scalable", "b2d_kmeans_fit_scalable", "b2d_kmeans_balanced_workspace_bytes",
    "b2d_kmeans_balanced_fit", "b2d_debug_kmeans_balanced_fine_assign",
    "b2d_mst_workspace_bytes", "b2d_mst",
    "b2d_single_linkage_workspace_bytes", "b2d_single_linkage", "b2d_debug_single_linkage_plan",
    "b2d_dbscan_workspace_bytes", "b2d_dbscan_fit",
    "b2d_debug_pairwise_plan", "b2d_radius_neighbors_workspace_bytes", "b2d_radius_neighbors_count",
    "b2d_radius_neighbors_fill", "b2d_kde_workspace_bytes", "b2d_kde_score_samples",
    "b2d_mean_shift_fit_workspace_bytes", "b2d_mean_shift_fit", "b2d_debug_mean_shift_sums",
    "b2d_ball_cover_index_bytes", "b2d_ball_cover_build_workspace_bytes", "b2d_ball_cover_build", "b2d_ball_cover_knn",
    "b2d_ball_cover_eps_workspace_bytes", "b2d_ball_cover_eps_count", "b2d_ball_cover_eps_fill",
    "b2d_dbscan_rbc_workspace_bytes", "b2d_dbscan_rbc_fit",
    "b2d_emst_rbc_workspace_bytes", "b2d_emst_rbc", "b2d_single_linkage_rbc_workspace_bytes", "b2d_single_linkage_rbc",
    "b2d_hdbscan_rbc_workspace_bytes", "b2d_hdbscan_rbc_fit", "b2d_hdbscan_rbc_model_bytes", "b2d_hdbscan_rbc_fit_model",
    "b2d_hdbscan_rbc_approximate_predict",
]

B2D_OK, B2D_ERR_INVALID_ARG, B2D_ERR_CUDA, B2D_ERR_UNSUPPORTED, B2D_ERR_WORKSPACE = range(5)
B2D_F32, B2D_F16, B2D_F64 = 0, 1, 2
B2D_HDBSCAN_EOM, B2D_HDBSCAN_LEAF = range(2)
B2D_KERNEL_LINEAR, B2D_KERNEL_POLYNOMIAL, B2D_KERNEL_RBF, B2D_KERNEL_TANH = range(4)
B2D_KMEANS_INIT_PLUS_PLUS, B2D_KMEANS_INIT_RANDOM, B2D_KMEANS_INIT_ARRAY = range(3)
(B2D_KDE_GAUSSIAN, B2D_KDE_TOPHAT, B2D_KDE_EPANECHNIKOV, B2D_KDE_EXPONENTIAL, B2D_KDE_LINEAR,
 B2D_KDE_COSINE) = range(6)


class RaftB200Error(RuntimeError):
    """Mirrors raft::exception (cpp/include/raft/core/error.hpp:37-58)."""


class LogicError(RaftB200Error, ValueError):
    """raft::logic_error (RAFT_EXPECTS failures), error.hpp:218-239."""


class CudaError(RaftB200Error):
    """raft::cuda_error, cpp/include/raft/util/cuda_rt_essentials.hpp:23-52."""


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("RAFT_B200_LIB", _build.SO_PATH)   # developer hook: an experimental build of the same ABI
    if not os.path.exists(path):
        if os.environ.get("RAFT_B200_NO_AUTOBUILD"):
            raise ImportError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        _build.build()
    L = ctypes.CDLL(path)
    i64, vp, sz, ci, cf = ctypes.c_int64, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_float
    L.b2d_version.restype = ci
    L.b2d_last_error.restype = ctypes.c_char_p
    L.b2d_set_option.restype = ci
    L.b2d_set_option.argtypes = [ctypes.c_char_p, ctypes.c_double]
    L.b2d_debug_nn_stats.restype = ci
    L.b2d_debug_nn_stats.argtypes = [vp, vp, i64, i64, i64, vp]
    L.b2d_pairwise_workspace_bytes.restype = sz
    L.b2d_pairwise_workspace_bytes.argtypes = [ci, ci, i64, i64, i64]
    L.b2d_pairwise_distance.restype = ci
    L.b2d_pairwise_distance.argtypes = [vp, ci, ci, vp, i64, vp, i64, vp, i64, i64, i64, i64, ci, cf, vp, sz]
    L.b2d_debug_pairwise_plan.restype = ci
    L.b2d_debug_pairwise_plan.argtypes = [ci, ci, vp, i64, vp, i64, vp, i64, i64, i64, i64, ci, vp, ci]
    L.b2d_fused_l2_nn_workspace_bytes.restype = sz
    L.b2d_fused_l2_nn_workspace_bytes.argtypes = [i64, i64, i64]
    L.b2d_fused_l2_nn.restype = ci
    L.b2d_fused_l2_nn.argtypes = [vp, vp, vp, i64, vp, i64, vp, vp, i64, i64, i64, ci, ci, vp, sz]
    L.b2d_fused_distance_nn.restype = ci
    L.b2d_fused_distance_nn.argtypes = [vp, vp, ci, vp, i64, vp, i64, vp, vp, i64, i64, i64, ci, vp, sz]
    L.b2d_masked_l2_nn_workspace_bytes.restype = sz
    L.b2d_masked_l2_nn_workspace_bytes.argtypes = [i64, i64, i64, i64]
    L.b2d_masked_l2_nn.restype = ci
    L.b2d_masked_l2_nn.argtypes = [vp, vp, vp, i64, vp, i64, vp, vp, vp, i64, vp, i64, i64, i64, i64, ci, ci, vp, sz]
    L.b2d_fused_l2_nn_keys.restype = ci
    L.b2d_fused_l2_nn_keys.argtypes = [vp, vp, vp, i64, vp, i64, vp, vp, i64, i64, i64, i64, ci, vp, sz]
    L.b2d_fused_l2_nn_finalize.restype = ci
    L.b2d_fused_l2_nn_finalize.argtypes = [vp, vp, vp, i64, ci, vp, sz]
    L.b2d_knn_l2_workspace_bytes.restype = sz
    L.b2d_knn_l2_workspace_bytes.argtypes = [i64, i64, i64, i64]
    L.b2d_knn.restype = ci
    L.b2d_knn.argtypes = [vp, vp, vp, ci, vp, i64, vp, i64, i64, i64, i64, i64, vp, sz]
    L.b2d_knn_l2.restype = ci
    L.b2d_knn_l2.argtypes = [vp, vp, vp, vp, i64, vp, i64, i64, i64, i64, i64, ci, vp, sz]
    L.b2d_silhouette_score_workspace_bytes.restype = sz
    L.b2d_silhouette_score_workspace_bytes.argtypes = [i64, i64, ci, ci, i64]
    L.b2d_silhouette_score.restype = ci
    L.b2d_silhouette_score.argtypes = [vp, vp, vp, vp, i64, vp, i64, i64, ci, ci, cf, i64, vp, sz]
    L.b2d_trustworthiness_score_workspace_bytes.restype = sz
    L.b2d_trustworthiness_score_workspace_bytes.argtypes = [i64, i64, i64, ci, ci, i64]
    L.b2d_trustworthiness_score.restype = ci
    L.b2d_trustworthiness_score.argtypes = [vp, vp, vp, i64, vp, i64, i64, i64, i64, ci, ci, i64, vp, sz]
    L.b2d_profile_begin.restype = ci
    L.b2d_profile_begin.argtypes = [ci]
    L.b2d_profile_end.restype = ci
    L.b2d_profile_end.argtypes = [vp, ci, vp]
    L.b2d_row_argmin.restype = ci
    L.b2d_row_argmin.argtypes = [vp, vp, vp, i64, i64, i64]
    L.b2d_select_k_workspace_bytes.restype = sz
    L.b2d_select_k_workspace_bytes.argtypes = [i64, i64, i64]
    L.b2d_select_k.restype = ci
    L.b2d_select_k.argtypes = [vp, vp, i64, vp, i64, i64, i64, ci, vp, vp, vp, sz]
    L.b2d_eps_neighbors_l2sq_workspace_bytes.restype = sz
    L.b2d_eps_neighbors_l2sq_workspace_bytes.argtypes = [i64, i64, i64]
    L.b2d_eps_neighbors_l2sq.restype = ci
    L.b2d_eps_neighbors_l2sq.argtypes = [vp, vp, i64, vp, ci, ci, vp, i64, vp, i64, i64, i64, i64, cf, vp, sz]
    L.b2d_gram_matrix_workspace_bytes.restype = sz
    L.b2d_gram_matrix_workspace_bytes.argtypes = [ci, ci, i64, i64, i64]
    L.b2d_gram_matrix.restype = ci
    L.b2d_gram_matrix.argtypes = [vp, ci, ci, ctypes.c_double, ctypes.c_double, ci, vp, i64, vp, i64, vp, i64, i64, i64, i64,
                                  ci, vp, sz]
    u64, cd = ctypes.c_uint64, ctypes.c_double
    L.b2d_kmeans_workspace_bytes.restype = sz
    L.b2d_kmeans_workspace_bytes.argtypes = [i64, i64, i64]
    L.b2d_kmeans_fit.restype = ci
    L.b2d_kmeans_fit.argtypes = [vp, ci, ci, cd, ci, ci, u64, ci, vp, i64, vp, i64, i64, vp, vp, vp, vp, sz]
    L.b2d_kmeans_predict.restype = ci
    L.b2d_kmeans_predict.argtypes = [vp, vp, i64, vp, i64, i64, vp, ci, vp, vp, ci, vp, sz]
    L.b2d_kmeans_update_centroids.restype = ci
    L.b2d_kmeans_update_centroids.argtypes = [vp, vp, i64, vp, vp, i64, i64, vp, ci, vp, vp, vp, sz]
    L.b2d_kmeans_init_plus_plus.restype = ci
    L.b2d_kmeans_init_plus_plus.argtypes = [vp, vp, i64, vp, i64, i64, ci, u64, vp, vp, sz]
    L.b2d_kmeans_scalable_workspace_bytes.restype = sz
    L.b2d_kmeans_scalable_workspace_bytes.argtypes = [i64, i64, i64, cd]
    L.b2d_kmeans_init_scalable.restype = ci
    L.b2d_kmeans_init_scalable.argtypes = [vp, vp, i64, vp, i64, i64, ci, cd, u64, vp, vp, vp, vp, sz]
    L.b2d_kmeans_fit_scalable.restype = ci
    L.b2d_kmeans_fit_scalable.argtypes = [vp, ci, ci, cd, cd, ci, u64, ci, vp, i64, vp, i64, i64, vp, vp, vp, vp, sz]
    L.b2d_kmeans_balanced_workspace_bytes.restype = sz
    L.b2d_kmeans_balanced_workspace_bytes.argtypes = [i64, i64, i64]
    L.b2d_kmeans_balanced_fit.restype = ci
    L.b2d_kmeans_balanced_fit.argtypes = [vp, ci, ci, u64, vp, i64, i64, i64, vp, vp, vp, vp, sz]
    L.b2d_debug_kmeans_balanced_fine_assign.restype = ci
    L.b2d_debug_kmeans_balanced_fine_assign.argtypes = [vp, vp, i64, i64, i64, vp, vp, ci, vp, i64, vp, vp, sz]
    L.b2d_mst_workspace_bytes.restype = sz
    L.b2d_mst_workspace_bytes.argtypes = [i64, i64]
    L.b2d_mst.restype = ci
    L.b2d_mst.argtypes = [vp, vp, vp, vp, i64, i64, vp, vp, vp, vp, vp, vp, sz]
    L.b2d_single_linkage_workspace_bytes.restype = sz
    L.b2d_single_linkage_workspace_bytes.argtypes = [i64, i64, ci]
    L.b2d_single_linkage.restype = ci
    L.b2d_single_linkage.argtypes = [vp, ci, vp, i64, i64, i64, ci, ci, vp, vp, vp, vp, vp, vp, sz]
    L.b2d_debug_single_linkage_plan.restype = ci
    L.b2d_debug_single_linkage_plan.argtypes = [i64, i64, vp]
    L.b2d_dbscan_workspace_bytes.restype = sz
    L.b2d_dbscan_workspace_bytes.argtypes = [i64, i64, i64]
    L.b2d_dbscan_fit.restype = ci
    L.b2d_dbscan_fit.argtypes = [vp, ci, vp, i64, i64, i64, cd, i64, i64, vp, vp, vp, vp, sz]
    L.b2d_dbscan_rbc_workspace_bytes.restype = sz
    L.b2d_dbscan_rbc_workspace_bytes.argtypes = [i64, i64, i64]
    L.b2d_dbscan_rbc_fit.restype = ci
    L.b2d_dbscan_rbc_fit.argtypes = [vp, ci, vp, i64, i64, i64, cd, i64, i64, u64, vp, vp, vp, vp, sz]
    L.b2d_emst_rbc_workspace_bytes.restype = sz
    L.b2d_emst_rbc_workspace_bytes.argtypes = [i64, i64, i64]
    L.b2d_emst_rbc.restype = ci
    L.b2d_emst_rbc.argtypes = [vp, ci, vp, i64, i64, i64, i64, u64, vp, vp, vp, vp, sz]
    L.b2d_single_linkage_rbc_workspace_bytes.restype = sz
    L.b2d_single_linkage_rbc_workspace_bytes.argtypes = [i64, i64, i64]
    L.b2d_single_linkage_rbc.restype = ci
    L.b2d_single_linkage_rbc.argtypes = [vp, ci, vp, i64, i64, i64, i64, u64, ci, vp, vp, vp, vp, vp, sz]
    L.b2d_hdbscan_rbc_workspace_bytes.restype = sz
    L.b2d_hdbscan_rbc_workspace_bytes.argtypes = [i64, i64, i64]
    L.b2d_hdbscan_rbc_fit.restype = ci
    L.b2d_hdbscan_rbc_fit.argtypes = [vp, ci, vp, i64, i64, i64, ci, ci, cd, ci, ci, i64, u64, vp, vp, vp, vp, vp, vp,
                                      vp, sz]
    L.b2d_hdbscan_rbc_model_bytes.restype = sz
    L.b2d_hdbscan_rbc_model_bytes.argtypes = [i64, i64, i64]
    L.b2d_hdbscan_rbc_fit_model.restype = ci
    L.b2d_hdbscan_rbc_fit_model.argtypes = [vp, ci, vp, i64, i64, i64, ci, ci, cd, ci, ci, i64, u64, vp, vp, vp, vp, vp,
                                            vp, vp, sz, vp]
    L.b2d_hdbscan_rbc_approximate_predict.restype = ci
    L.b2d_hdbscan_rbc_approximate_predict.argtypes = [vp, vp, i64, i64, ci, i64, ci, vp, i64, i64, vp, vp, vp, vp]
    L.b2d_radius_neighbors_workspace_bytes.restype = sz
    L.b2d_radius_neighbors_workspace_bytes.argtypes = [i64, i64, i64, i64]
    L.b2d_radius_neighbors_count.restype = ci
    L.b2d_radius_neighbors_count.argtypes = [vp, vp, ci, vp, i64, vp, i64, i64, i64, i64, cf, vp, sz]
    L.b2d_radius_neighbors_fill.restype = ci
    L.b2d_radius_neighbors_fill.argtypes = [vp, vp, i64, vp, vp, ci, vp, i64, vp, i64, i64, i64, i64, cf, vp, sz]
    L.b2d_kde_workspace_bytes.restype = sz
    L.b2d_kde_workspace_bytes.argtypes = [i64, i64, i64, i64]
    L.b2d_kde_score_samples.restype = ci
    L.b2d_kde_score_samples.argtypes = [vp, ci, cd, vp, i64, vp, vp, i64, i64, i64, i64, i64, vp, vp, sz]
    L.b2d_mean_shift_fit_workspace_bytes.restype = sz
    L.b2d_mean_shift_fit_workspace_bytes.argtypes = [i64, i64, i64, i64]
    L.b2d_mean_shift_fit.restype = ci
    L.b2d_mean_shift_fit.argtypes = [vp, vp, i64, i64, i64, cd, vp, i64, i64, ci, i64, ci, ci, i64, vp, vp, vp, vp, vp, sz]
    L.b2d_debug_mean_shift_sums.restype = ci
    L.b2d_debug_mean_shift_sums.argtypes = [vp, vp, i64, i64, vp, i64, i64, i64, vp, vp, vp, vp, vp, sz]
    L.b2d_ball_cover_index_bytes.restype = sz
    L.b2d_ball_cover_index_bytes.argtypes = [i64, i64, i64]
    L.b2d_ball_cover_build_workspace_bytes.restype = sz
    L.b2d_ball_cover_build_workspace_bytes.argtypes = [i64, i64, i64]
    L.b2d_ball_cover_build.restype = ci
    L.b2d_ball_cover_build.argtypes = [vp, vp, vp, i64, i64, i64, ci, i64, u64, vp, sz]
    L.b2d_ball_cover_knn.restype = ci
    L.b2d_ball_cover_knn.argtypes = [vp, vp, vp, vp, i64, i64, ci, i64, vp, i64, i64, i64]
    L.b2d_ball_cover_eps_workspace_bytes.restype = sz
    L.b2d_ball_cover_eps_workspace_bytes.argtypes = [i64, i64]
    L.b2d_ball_cover_eps_count.restype = ci
    L.b2d_ball_cover_eps_count.argtypes = [vp, vp, vp, i64, i64, ci, i64, vp, i64, i64, cf, vp, sz]
    L.b2d_ball_cover_eps_fill.restype = ci
    L.b2d_ball_cover_eps_fill.argtypes = [vp, vp, i64, vp, vp, vp, i64, i64, ci, i64, vp, i64, i64, cf, vp, sz]
    L.b2d_row_norm.restype = ci
    L.b2d_row_norm.argtypes = [vp, vp, vp, i64, i64, i64, ci, ci]
    _lib = L
    return L


def check(status: int) -> None:
    if status == B2D_OK:
        return
    msg = lib().b2d_last_error().decode("utf-8", "replace")
    if status in (B2D_ERR_INVALID_ARG, B2D_ERR_UNSUPPORTED, B2D_ERR_WORKSPACE):
        raise LogicError(msg)
    raise CudaError(msg)
