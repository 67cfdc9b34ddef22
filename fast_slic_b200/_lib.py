"""ctypes binding of libfslic_b200.so (the C ABI declared in include/fslic_b200.h).

The library is built in-tree by ``fast_slic_b200/csrc/build.sh`` (see ``__graft_entry__.build``).
There is no CPU fallback: if the shared library is missing the import fails loudly.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfslic_b200.so")

# every symbol include/fslic_b200.h declares
EXPORTED_SYMBOLS = (
    "fslic_b200_last_error", "fslic_b200_version", "fslic_b200_sizeof_cluster", "fslic_b200_create",
    "fslic_b200_destroy", "fslic_b200_initialize_clusters", "fslic_b200_iterate", "fslic_b200_iterate_host",
    "fslic_b200_initialize_clusters_host", "fslic_b200_enforce_connectivity", "fslic_b200_debug_stages",
    "fslic_b200_rgb_to_quad", "fslic_b200_debug_heap_select", "fslic_b200_stage_ms", "fslic_b200_get_S",
    "fslic_b200_launches_last_iterate", "fslic_b200_assign_kernel_time", "fslic_b200_debug_cca_counters",
    "fslic_b200_iterate_host_async", "fslic_b200_wait", "fslic_b200_create_cca",
    "fslic_b200_debug_assign_impl", "fslic_b200_debug_dispatch", "fslic_b200_debug_cca_dispatch", "fslic_b200_connectivity_scratch_bytes", "fslic_b200_get_connectivity",
    "fslic_b200_get_mask_density", "fslic_b200_cluster_density_to_mask", "fslic_b200_cca_stage_ms",
    "fslic_b200_iterate_real", "fslic_b200_iterate_preemptive", "fslic_b200_set_manhattan_spatial_dist",
    "fslic_b200_iterate_lsc", "fslic_b200_debug_lsc_stages",
    "fslic_b200_crf_create", "fslic_b200_crf_destroy", "fslic_b200_crf_get_params", "fslic_b200_crf_set_params",
    "fslic_b200_crf_times", "fslic_b200_crf_push_frame", "fslic_b200_crf_pop_frame", "fslic_b200_crf_set_clusters",
    "fslic_b200_crf_get_clusters", "fslic_b200_crf_set_connectivity", "fslic_b200_crf_get_connectivity",
    "fslic_b200_crf_set_unary", "fslic_b200_crf_get_unary", "fslic_b200_crf_set_unbiased", "fslic_b200_crf_set_mask",
    "fslic_b200_crf_set_proba", "fslic_b200_crf_get_inferred", "fslic_b200_crf_reset_inferred",
    "fslic_b200_crf_initialize", "fslic_b200_crf_inference", "fslic_b200_crf_spatial_pairwise_energy",
    "fslic_b200_crf_temporal_pairwise_energy", "fslic_b200_debug_expf_host", "fslic_b200_debug_expf_device",
    "fslic_b200_set_trace", "fslic_b200_trace_info", "fslic_b200_trace_snapshots", "fslic_b200_format_report",
    "fslic_b200_free_report", "fslic_b200_debug_graph_counts",
    "fslic_b200_connectivity_batch_scratch_bytes", "fslic_b200_get_connectivity_batch",
    "fslic_b200_get_mask_density_batch", "fslic_b200_cluster_density_to_mask_batch",
    "fslic_b200_crfdev_push_scratch_bytes", "fslic_b200_crfdev_push_label_frames", "fslic_b200_crfdev_set_unary",
    "fslic_b200_crfdev_set_proba", "fslic_b200_crfdev_set_mask", "fslic_b200_crfdev_get_inferred",
    "fslic_b200_debug_logf_host", "fslic_b200_debug_logf_device",
    "fslic_b200_crfgroup_inference", "fslic_b200_crfdev_group_push_label_frames", "fslic_b200_crfdev_group_set_proba",
    "fslic_b200_crfdev_group_reset_inferred", "fslic_b200_crfdev_group_get_inferred", "fslic_b200_crfgroup_pop_frame",
    "fslic_b200_pool_batch_scratch_bytes", "fslic_b200_pool_batch", "fslic_b200_pool_unpool_batch",
    "fslic_b200_pool_paint_argmax_batch", "fslic_b200_pool_paint_batch",
    "fslic_b200_rag_batch_scratch_bytes", "fslic_b200_rag_batch_count", "fslic_b200_rag_fill_scratch_bytes",
    "fslic_b200_rag_batch_fill", "fslic_b200_rag3d_batch_scratch_bytes", "fslic_b200_rag3d_batch_count",
    "fslic_b200_rag3d_batch_fill",
    "fslic_b200_gt_histogram_batch", "fslic_b200_gt_scores_scratch_bytes", "fslic_b200_gt_scores_batch",
    "fslic_b200_gt_boundaries_batch", "fslic_b200_gt_scores3d_scratch_bytes", "fslic_b200_gt_scores3d_batch",
    "fslic_b200_gt_boundaries3d_batch",
    "fslic_b200_props_batch", "fslic_b200_props3d_batch",
    "fslic_b200_merge_scratch_bytes", "fslic_b200_merge_batch",
    "fslic_b200_boundary_select_scratch_bytes", "fslic_b200_boundary_select_batch",
    "fslic_b200_boundary_stats_scratch_bytes", "fslic_b200_boundary_stats_batch",
    "fslic_b200_boundary3d_select_scratch_bytes", "fslic_b200_boundary3d_select_batch",
    "fslic_b200_boundary3d_stats_scratch_bytes", "fslic_b200_boundary3d_stats_batch",
    "fslic_b200_knn_scratch_bytes", "fslic_b200_knn_count", "fslic_b200_knn_fill",
    "fslic_b200_feature_slic_scratch_bytes", "fslic_b200_feature_slic",
    "fslic_b200_soft_assign", "fslic_b200_soft_assign_backward", "fslic_b200_soft_pool",
    "fslic_b200_soft_pool_backward", "fslic_b200_soft_unpool", "fslic_b200_soft_unpool_backward",
    "fslic_b200_soft_labels",
    "fslic_b200_mp_gather", "fslic_b200_mp_gather_backward_scratch_bytes", "fslic_b200_mp_gather_backward",
    "fslic_b200_mp_softmax", "fslic_b200_mp_softmax_backward", "fslic_b200_mp_aggregate",
    "fslic_b200_mp_aggregate_backward_scratch_bytes", "fslic_b200_mp_aggregate_backward",
    "fslic_b200_sv_enforce_scratch_bytes", "fslic_b200_sv_enforce", "fslic_b200_sv_slic_scratch_bytes",
    "fslic_b200_sv_slic",
)

STAGE_NAMES = ("cielab_conversion", "assign", "update", "full_assign", "enforce_connectivity", "iterate")
LSC_STAGE_NAMES = ("before_iteration", "after_update")  # FSLIC_T_BEFORE_ITERATION, FSLIC_T_AFTER_UPDATE
DISPATCH_COUNT = 15  # FSLIC_DISPATCH_COUNT
PASS_FIELDS = ("kernel", "tps", "grid", "workers", "items", "trips")  # one pass of fslic_b200_debug_dispatch
CCA_DISPATCH_FIELDS = ("heap_smem", "heap_smem_max_k", "sub_batches", "split", "number_nb")  # fslic_b200_debug_cca_dispatch
CCA_DISPATCH_COUNT = len(CCA_DISPATCH_FIELDS)  # FSLIC_CCA_DISPATCH_COUNT
CCA_STAGE_NAMES =("build_disjoint_set", "flatten", "threshold_by_area", "sort", "substitute", "output")  # cca.cpp:194-263


class Params(C.Structure):
    """== fslic_params (include/fslic_b200.h)."""
    _fields_ = [("compactness", C.c_float), ("min_size_factor", C.c_float), ("subsample_stride", C.c_int32),
                ("convert_to_lab", C.c_int32), ("max_iter", C.c_int32), ("collect_timing", C.c_int32)]


class FslicError(RuntimeError):
    pass


_lib = None


def build_library(verbose=False):
    import subprocess
    script = os.path.join(_HERE, "csrc", "build.sh")
    subprocess.check_call(["bash", script], stdout=None if verbose else subprocess.DEVNULL)


def lib():
    """Load (once) and return the C-ABI library."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "fast_slic_b200: %s is missing -- build it with fast_slic_b200/csrc/build.sh "
            "(there is no CPU fallback)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, i32 = C.c_void_p, C.c_int
    L.fslic_b200_last_error.restype = C.c_char_p
    L.fslic_b200_version.restype = C.c_char_p
    L.fslic_b200_create.argtypes = [i32, i32, i32, i32, i32, C.POINTER(vp)]
    L.fslic_b200_create_cca.argtypes = [i32, i32, i32, i32, C.POINTER(vp)]
    L.fslic_b200_destroy.argtypes = [vp]
    L.fslic_b200_initialize_clusters.argtypes = [vp, vp, vp, i32, vp]
    L.fslic_b200_iterate.argtypes = [vp, vp, vp, vp, i32, C.POINTER(Params), vp]
    L.fslic_b200_iterate_real.argtypes = [vp, i32, vp, vp, vp, i32, C.POINTER(Params), vp]
    L.fslic_b200_iterate_preemptive.argtypes = [vp, vp, vp, vp, i32, C.POINTER(Params), C.c_float, vp]
    L.fslic_b200_set_manhattan_spatial_dist.argtypes = [vp, i32]
    L.fslic_b200_iterate_lsc.argtypes = [vp, vp, vp, vp, i32, C.POINTER(Params), vp]
    L.fslic_b200_debug_lsc_stages.argtypes = [vp, vp, vp, vp, i32, vp]
    L.fslic_b200_iterate_host.argtypes = [vp, vp, vp, vp, i32, C.POINTER(Params)]
    L.fslic_b200_iterate_host_async.argtypes = [vp, vp, vp, vp, i32, C.POINTER(Params)]
    L.fslic_b200_wait.argtypes = [vp]
    L.fslic_b200_initialize_clusters_host.argtypes = [vp, vp, vp, i32]
    L.fslic_b200_enforce_connectivity.argtypes = [vp, vp, i32, i32, i32, vp]
    L.fslic_b200_debug_stages.argtypes = [vp, vp, vp, i32, vp]
    L.fslic_b200_rgb_to_quad.argtypes = [vp, vp, vp, i32, i32, vp]
    L.fslic_b200_debug_heap_select.argtypes = [vp, vp, i32, i32, vp, vp]
    L.fslic_b200_stage_ms.argtypes = [vp, C.POINTER(C.c_float), i32]
    L.fslic_b200_cca_stage_ms.argtypes = [vp, C.POINTER(C.c_float), i32]
    L.fslic_b200_get_S.argtypes = [vp]
    L.fslic_b200_launches_last_iterate.argtypes = [vp]
    L.fslic_b200_debug_assign_impl.argtypes = [vp]
    L.fslic_b200_debug_dispatch.argtypes = [vp, C.POINTER(C.c_int32), i32]
    L.fslic_b200_debug_cca_dispatch.argtypes = [vp, C.POINTER(C.c_int32), i32]
    L.fslic_b200_connectivity_scratch_bytes.argtypes = [i32]
    L.fslic_b200_connectivity_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_get_connectivity.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp, C.c_size_t, vp]
    L.fslic_b200_get_mask_density.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp]
    L.fslic_b200_cluster_density_to_mask.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp]
    L.fslic_b200_connectivity_batch_scratch_bytes.argtypes = [i32, i32]
    L.fslic_b200_connectivity_batch_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_get_connectivity_batch.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, C.c_size_t, vp]
    L.fslic_b200_get_mask_density_batch.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp]
    L.fslic_b200_cluster_density_to_mask_batch.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp]
    L.fslic_b200_pool_batch_scratch_bytes.argtypes = [i32, i32, i32, i32]
    L.fslic_b200_pool_batch_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_pool_batch.argtypes = [i32, i32, i32, i32, i32, i32, vp, vp, i32, vp, vp, vp, C.c_size_t, vp]
    L.fslic_b200_pool_unpool_batch.argtypes = [i32, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp]
    L.fslic_b200_pool_paint_argmax_batch.argtypes = [i32, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp]
    L.fslic_b200_pool_paint_batch.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp]
    i64 = C.c_longlong
    L.fslic_b200_rag_batch_scratch_bytes.argtypes = [i32, i32, i32, i32, i32, i32]
    L.fslic_b200_rag_batch_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_rag_batch_count.argtypes = [i32, i32, i32, i32, i32, i32, i32, vp, i64, vp, vp, vp, C.c_size_t, vp]
    L.fslic_b200_rag_fill_scratch_bytes.argtypes = [i32, i32, i64]
    L.fslic_b200_rag_fill_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_rag_batch_fill.argtypes = [i32, i32, i32, i32, i32, i32, i32, i64, i64, vp, C.c_size_t, vp, C.c_size_t,
                                            vp, vp, vp, vp]
    L.fslic_b200_rag3d_batch_scratch_bytes.argtypes = [i32] * 7
    L.fslic_b200_rag3d_batch_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_rag3d_batch_count.argtypes = [i32] * 8 + [vp, i64, vp, vp, vp, C.c_size_t, vp]
    L.fslic_b200_rag3d_batch_fill.argtypes = [i32] * 8 + [i64, i64, vp, C.c_size_t, vp, C.c_size_t, vp, vp, vp, vp]
    L.fslic_b200_gt_histogram_batch.argtypes = [i32, i32, i32, i32, i32, i32, i32, vp, vp, vp, vp]
    L.fslic_b200_gt_scores_scratch_bytes.argtypes = [i32, i32, i32, i32]
    L.fslic_b200_gt_scores_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_gt_scores_batch.argtypes = [i32, i32, i32, i32, i32, i32, i32, vp, vp, i32, i64, vp, vp, C.c_size_t,
                                             vp]
    L.fslic_b200_gt_boundaries_batch.argtypes = [i32, i32, i32, i32, vp, vp, vp]
    L.fslic_b200_gt_scores3d_scratch_bytes.argtypes = [i32] * 5
    L.fslic_b200_gt_scores3d_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_gt_scores3d_batch.argtypes = [i32] * 10 + [vp, vp, i32, i64, vp, vp, C.c_size_t, vp]
    L.fslic_b200_gt_boundaries3d_batch.argtypes = [i32] * 5 + [vp] * 3
    L.fslic_b200_props_batch.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.fslic_b200_props3d_batch.argtypes = [i32] * 6 + [vp] * 9
    L.fslic_b200_merge_scratch_bytes.argtypes = [i32, i32]
    L.fslic_b200_merge_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_merge_batch.argtypes = [i32, i32, i32, i32, i32, vp, i64, vp, vp, vp, i32, C.c_double, i32, vp, vp, vp,
                                         vp, C.c_size_t, vp]
    L.fslic_b200_boundary_select_scratch_bytes.argtypes = [i32, i32, i32, i32, i32]
    L.fslic_b200_boundary_select_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_boundary_select_batch.argtypes = [i32, i32, i32, i32, i32, i32, vp, vp, vp, C.c_size_t, vp]
    L.fslic_b200_boundary_stats_scratch_bytes.argtypes = [i64, i64]
    L.fslic_b200_boundary_stats_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_boundary_stats_batch.argtypes = [i32, i32, i32, i32, i32, i32, i32, vp, vp, i64, vp, C.c_size_t, i64,
                                                  i64, i64, vp, vp, i32, vp, vp, vp, vp, vp, C.c_size_t, vp]
    L.fslic_b200_boundary3d_select_scratch_bytes.argtypes = [i32] * 6
    L.fslic_b200_boundary3d_select_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_boundary3d_select_batch.argtypes = [i32] * 7 + [vp, vp, vp, C.c_size_t, vp]
    L.fslic_b200_boundary3d_stats_scratch_bytes.argtypes = [i64] * 3
    L.fslic_b200_boundary3d_stats_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_boundary3d_stats_batch.argtypes = [i32] * 8 + [vp, vp, i64, i64, vp, C.c_size_t, i64, i64, i64, vp, vp,
                                                                i32, vp, vp, vp, vp, vp, C.c_size_t, vp]
    L.fslic_b200_knn_scratch_bytes.argtypes = [i32, i32, i32, i32, i32]
    L.fslic_b200_knn_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_knn_count.argtypes = [i32, i32, i32, i32, i32, i32, vp, vp, i64, vp, vp, vp, C.c_size_t, vp]
    L.fslic_b200_knn_fill.argtypes = [i32, i32, i32, i32, i32, i32, i64, i64, vp, C.c_size_t, vp, vp, vp, vp]
    L.fslic_b200_feature_slic_scratch_bytes.argtypes = [i32, i32, i32, i32, i32, i32, i32]
    L.fslic_b200_feature_slic_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_feature_slic.argtypes = [i32, i32, i32, i32, i32, i32, C.c_float, i32, i32, vp, vp, vp, vp, vp, vp, vp,
                                          vp, vp, C.c_size_t, vp]
    soft = [i32] * 7  # device, batch, H, W, C, nh, nw
    L.fslic_b200_soft_assign.argtypes = soft + [vp] * 4
    L.fslic_b200_soft_assign_backward.argtypes = soft + [vp] * 8
    L.fslic_b200_soft_pool.argtypes = soft + [vp] * 5
    L.fslic_b200_soft_pool_backward.argtypes = soft + [vp] * 10
    L.fslic_b200_soft_unpool.argtypes = soft + [vp] * 4
    L.fslic_b200_soft_unpool_backward.argtypes = soft + [vp] * 6
    L.fslic_b200_soft_labels.argtypes = [i32] * 6 + [vp] * 3
    L.fslic_b200_mp_gather.argtypes = [i32, i64, i64, i32, i32] + [vp] * 5
    L.fslic_b200_mp_gather_backward_scratch_bytes.argtypes = [i64, i64]
    L.fslic_b200_mp_gather_backward_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_mp_gather_backward.argtypes = [i32, i64, i64, i32, i32] + [vp] * 5 + [C.c_size_t, vp]
    L.fslic_b200_mp_softmax.argtypes = [i32, i64, i64, i32] + [vp] * 5
    L.fslic_b200_mp_softmax_backward.argtypes = [i32, i64, i64, i32] + [vp] * 6
    L.fslic_b200_mp_aggregate.argtypes = [i32, i64, i64, i32, i32, i32] + [vp] * 8
    L.fslic_b200_mp_aggregate_backward_scratch_bytes.argtypes = [i64, i64, i32, i32]
    L.fslic_b200_mp_aggregate_backward_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_mp_aggregate_backward.argtypes = [i32, i64, i64, i32, i32, i32] + [vp] * 10 + [C.c_size_t, vp]
    L.fslic_b200_sv_enforce_scratch_bytes.argtypes = [i32] * 4
    L.fslic_b200_sv_enforce_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_sv_enforce.argtypes = [i32] * 7 + [vp] * 3 + [C.c_size_t, vp]
    L.fslic_b200_sv_slic_scratch_bytes.argtypes = [i32] * 10
    L.fslic_b200_sv_slic_scratch_bytes.restype = C.c_size_t
    L.fslic_b200_sv_slic.argtypes = [i32] * 9 + [C.c_float] * 3 + [i32] * 3 + [vp] * 7 + [C.c_size_t, vp]
    L.fslic_b200_assign_kernel_time.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_int)]
    L.fslic_b200_debug_cca_counters.argtypes = [vp, C.POINTER(C.c_int32), i32]
    L.fslic_b200_set_trace.argtypes = [vp, i32]
    L.fslic_b200_debug_graph_counts.argtypes = [vp, C.POINTER(i32), C.POINTER(i32)]
    L.fslic_b200_trace_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    L.fslic_b200_trace_snapshots.argtypes = [vp, i32, vp, vp, vp, C.POINTER(C.c_uint32)]
    L.fslic_b200_format_report.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, C.POINTER(C.c_void_p),
                                           C.POINTER(C.c_size_t)]
    L.fslic_b200_free_report.argtypes = [vp]
    L.fslic_b200_free_report.restype = None
    assert L.fslic_b200_sizeof_cluster() == 32
    _lib = L
    return L


def check(rc):
    if rc != 0:
        msg = lib().fslic_b200_last_error().decode("utf-8", "replace")
        if rc == -1:
            raise ValueError(msg)
        if rc == -3:
            raise MemoryError(msg)
        raise FslicError("fslic_b200 error %d: %s" % (rc, msg))


def format_recorder_report(H, W, assignment, min_dists, clusters):
    """The reference's debug_mode report (recorder.h) as bytes, from snapshot arrays laid out like
    Engine.trace_snapshots returns them: assignment u16[T, H*W], min_dists u16 or float32 [T, H*W], clusters [T, K]
    32-byte records.  Formatted by fslic_b200_format_report (host code, no device needed)."""
    import numpy as np
    assignment = np.ascontiguousarray(assignment, np.uint16)
    min_dists = np.ascontiguousarray(min_dists)
    clusters = np.ascontiguousarray(clusters)
    if min_dists.dtype not in (np.uint16, np.float32):
        raise ValueError("min_dists must be uint16 or float32")
    T = clusters.shape[0] if clusters.ndim == 2 else 0
    K = clusters.shape[1] if clusters.ndim == 2 else 0
    if clusters.dtype.itemsize != 32 or assignment.size != T * H * W or min_dists.size != T * H * W:
        raise ValueError("snapshot arrays do not match T=%d, H=%d, W=%d" % (T, H, W))
    L = lib()
    out, n = C.c_void_p(), C.c_size_t()
    check(L.fslic_b200_format_report(int(H), int(W), K, T, int(min_dists.dtype == np.float32), assignment.ctypes.data,
                                     min_dists.ctypes.data, clusters.ctypes.data, C.byref(out), C.byref(n)))
    try:
        return C.string_at(out, n.value)
    finally:
        L.fslic_b200_free_report(out)
