"""ctypes binding of libdemon_b200.so (include/demon_b200.h).

There is no CPU fallback: if the library is missing or no CUDA device is present the ops raise.
The library path can be overridden with DEMON_B200_LIB, like LMBSPECIALOPS_LIB in the reference
(lmbspecialops/python/lmbspecialops/__init__.py:23-39).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_DEFAULT = os.path.join(_HERE, "lib", "libdemon_b200.so")

c_void_p, c_int, c_int64, c_float, c_double, c_char_p = (
    ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_double, ctypes.c_char_p)


class PipelineArgs(ctypes.Structure):
    """demon_pipeline_args: one fused-pipeline call, every field 64 bits wide (include/demon_b200.h)."""
    _fields_ = [("input", c_int64), ("images", c_void_p), ("image2_2", c_void_p), ("image2_2_mode", c_int64),
                ("sn", c_int64), ("si", c_int64), ("sy", c_int64), ("h", c_int64), ("w", c_int64), ("resample", c_int64),
                ("K", c_void_p), ("status", c_void_p), ("iterations", c_int64), ("snapshots", c_int64),
                ("depth0", c_void_p), ("normal0", c_void_p), ("rotation", c_void_p), ("translation", c_void_p),
                ("flow2", c_void_p), ("depth2", c_void_p), ("normal2", c_void_p)]


# PipelineArgs.input (DEMON_INPUT_*)
INPUT_F32, INPUT_U8, INPUT_RESIZE_U8, INPUT_VIEWS_U8 = range(4)

# name -> argtypes; every function returns int unless listed in _RESTYPES
_P = c_void_p
PROTOTYPES = {
    "demon_warp2d_f32": [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_float, _P],
    "demon_warp2d_f64": [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_double, _P],
    "demon_depth_to_flow_f32": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P],
    "demon_depth_to_flow_f64": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P],
    "demon_flow_to_depth_f32": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P],
    "demon_flow_to_depth_f64": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P],
    "demon_leaky_relu_f32": [_P, _P, c_int64, c_float, _P],
    "demon_leaky_relu_f64": [_P, _P, c_int64, c_double, _P],
    "demon_median3x3_downsample_f32": [_P, _P, c_int64, c_int, c_int, _P],
    "demon_median3x3_downsample_f64": [_P, _P, c_int64, c_int, c_int, _P],
    "demon_scale_invariant_gradient_f32": [_P, _P, c_int64, c_int, c_int, _P, _P, c_int, c_float, _P],
    "demon_scale_invariant_gradient_f64": [_P, _P, c_int64, c_int, c_int, _P, _P, c_int, c_double, _P],
    "demon_scale_invariant_gradient_grad_f32": [_P, _P, _P, c_int64, c_int, c_int, _P, _P, c_int, c_float, _P],
    "demon_scale_invariant_gradient_grad_f64": [_P, _P, _P, c_int64, c_int, c_int, _P, _P, c_int, c_double, _P],
    "demon_leaky_relu_grad_f32": [_P, _P, _P, c_int64, c_float, _P],
    "demon_leaky_relu_grad_f64": [_P, _P, _P, c_int64, c_double, _P],
    "demon_replace_nonfinite_f32": [_P, _P, c_int64, c_float, _P],
    "demon_replace_nonfinite_f64": [_P, _P, c_int64, c_double, _P],
    "demon_replace_nonfinite_grad_f32": [_P, _P, _P, c_int64, _P],
    "demon_replace_nonfinite_grad_f64": [_P, _P, _P, c_int64, _P],
    "demon_depth_to_normals_f32": [_P, _P, _P, c_int64, c_int, c_int, c_int, _P],
    "demon_depth_to_normals_f64": [_P, _P, _P, c_int64, c_int, c_int, c_int, _P],
    "demon_correlation_f32": [_P, _P, _P] + [c_int] * 11 + [_P],
    "demon_correlation_grad_f32": [_P] * 5 + [c_int] * 11 + [_P],
    "demon_correlation_1d_f32": [_P, _P, _P] + [c_int] * 12 + [_P],
    "demon_correlation_1d_grad_f32": [_P] * 5 + [c_int] * 12 + [_P],
    "demon_flow_warp_f32": [_P, _P, _P] + [c_int] * 5 + [_P],
    "demon_flow_warp_grad_workspace_bytes": [c_int, c_int, c_int],
    "demon_flow_warp_grad_f32": [_P] * 5 + [c_int] * 4 + [_P, c_int64, _P],
    "demon_flow_out_of_frame_f32": [_P, _P, _P, c_int, c_int, c_int, _P],
    "demon_resample_f32": [_P, _P] + [c_int] * 8 + [_P],
    "demon_resample_f64": [_P, _P] + [c_int] * 8 + [_P],
    "demon_loss_workspace_bytes": [_P, c_int, c_int, c_int],
    "demon_loss_forward_f32": [_P, c_int, _P, c_int64, _P],
    "demon_loss_forward_f64": [_P, c_int, _P, c_int64, _P],
    "demon_loss_backward_f32": [_P, c_int, _P, c_int64, _P],
    "demon_loss_backward_f64": [_P, c_int, _P, c_int64, _P],
    "demon_confidence_map_f32": [_P, _P, _P, c_int64, c_double, _P],
    "demon_confidence_map_f64": [_P, _P, _P, c_int64, c_double, _P],
    "demon_loss_ground_truth_workspace_bytes": [c_int, c_int, c_int, c_int],
    "demon_loss_ground_truth_f32": [_P] * 4 + [c_int] * 3 + [_P] * 9 + [_P, c_int64, _P],
    "demon_loss_ground_truth_f64": [_P] * 4 + [c_int] * 3 + [_P] * 9 + [_P, c_int64, _P],
    "demon_metric_workspace_bytes": [c_int, c_int64],
    "demon_depth_error_sums_f32": [_P, _P, c_int, c_int64, c_int, c_int, _P, _P, _P, _P, _P],
    "demon_depth_scale_factor": [_P, c_int, c_int, _P, _P],
    "demon_flow_epe_sums_f32": [_P, _P, c_int, c_int64, _P, _P, _P],
    "demon_depth_error_sums_resampled_f32": [_P, c_int, c_int, _P, _P] + [c_int] * 7 + [_P, _P, c_int, c_int] + [_P] * 5,
    "demon_flow_epe_sums_resampled_f32": [_P, c_int, c_int, _P] + [c_int] * 7 + [_P] * 5,
    "demon_motion_errors": [_P, _P, _P, c_int, _P, _P, _P],
    "demon_visible_points_mask_f32": [_P] * 5 + [c_int] * 7 + [_P, _P],
    "demon_visible_points_mask_inverse_f32": [_P] * 5 + [c_int] * 7 + [_P, _P],
    "demon_point_cloud_scratch_bytes": [c_int, c_int, c_int],
    "demon_point_cloud_f32": [_P] * 7 + [c_int] * 3 + [_P] * 6,
    "demon_point_cloud_inverse_f32": [_P] * 7 + [c_int] * 3 + [_P] * 6,
    "demon_tsdf_integrate_f32": [_P] * 3 + [c_int] * 3 + [_P, c_float, c_float] + [_P] * 5 + [c_int] * 3 + [_P],
    "demon_marching_cubes_scratch_bytes": [c_int, c_int, c_int],
    "demon_marching_cubes_count_f32": [_P, _P, c_int, c_int, c_int, _P, _P, _P],
    "demon_marching_cubes_f32": [_P] * 3 + [c_int] * 3 + [_P, c_float] + [_P] * 5,
    "demon_sparse_tsdf_rehash": [_P, _P, c_int64, _P, _P, c_int64, _P, _P],
    "demon_sparse_tsdf_allocate_f32": [_P, _P, c_int64, _P, _P, c_float, c_float] + [_P] * 4 + [c_int] * 3 + [_P],
    "demon_sparse_tsdf_gather_new": [_P, _P, c_int64, _P, _P, _P],
    "demon_sparse_tsdf_commit": [_P, _P, c_int64, _P, c_int, c_int, _P, _P],
    "demon_sparse_tsdf_integrate_f32": [_P] * 4 + [c_int, _P, c_float, c_float] + [_P] * 5 + [c_int] * 3 + [_P],
    "demon_sparse_tsdf_mesh_scratch_bytes": [c_int],
    "demon_sparse_tsdf_mesh_count_f32": [_P] * 3 + [c_int, _P, _P, c_int64, _P, _P, _P],
    "demon_sparse_tsdf_mesh_f32": [_P] * 4 + [c_int, _P, c_float] + [_P] * 5,
    "demon_tsdf_raycast_f32": [_P] * 3 + [c_int] * 3 + [_P, c_float] + [_P] * 5 + [c_float] + [c_int] * 3 + [_P] * 4,
    "demon_sparse_tsdf_raycast_scratch_bytes": [c_int],
    "demon_sparse_tsdf_far_f32": [_P, c_int, _P, c_float, _P, _P, c_int, _P, _P],
    "demon_sparse_tsdf_raycast_f32": [_P] * 4 + [c_int, _P, _P, c_int64, _P, _P, c_float] + [_P] * 5 + [c_float] + [c_int] * 3 + [_P] * 4,
    "demon_sparse_tsdf_mesh_range_count_f32": [_P] * 3 + [c_int] * 3 + [_P, _P, c_int64, _P, _P, _P],
    "demon_sparse_tsdf_mesh_range_f32": [_P] * 4 + [c_int] * 3 + [_P, c_float] + [_P] * 5,
    "demon_sparse_tsdf_depth_tiles_f32": [_P] + [c_int] * 3 + [_P, _P],
    "demon_sparse_tsdf_reach_f32": [_P, c_int, _P, c_float, c_float] + [_P] * 4 + [c_int] * 3 + [_P, c_int, _P],
    "demon_sparse_tsdf_evict": [_P] * 7 + [c_int64, _P, _P, c_int] + [_P] * 5 + [_P],
    "demon_sparse_tsdf_restore": [_P] * 6 + [c_int] + [_P] * 5 + [c_int, _P, _P, c_int64, _P],
    "demon_sparse_tsdf_index": [_P, _P, c_int64, _P, c_int, c_int, _P],
    "demon_tsdf_indexed_mesh_scratch_bytes": [c_int, c_int, c_int],
    "demon_tsdf_indexed_mesh_count_f32": [_P, _P, c_int, c_int, c_int, _P, _P, _P],
    "demon_tsdf_indexed_mesh_f32": [_P] * 3 + [c_int] * 3 + [_P, c_float] + [_P] * 6,
    "demon_sparse_tsdf_edge_mark_f32": [_P] * 3 + [c_int] * 3 + [_P, _P, c_int64] + [_P] * 4,
    "demon_sparse_tsdf_edge_scan_bytes": [c_int],
    "demon_sparse_tsdf_edge_scan": [_P, c_int] + [_P] * 4,
    "demon_sparse_tsdf_indexed_mesh_range_count_f32": [_P] * 3 + [c_int] * 3 + [_P, _P, _P, c_int64, _P, _P, _P],
    "demon_sparse_tsdf_indexed_mesh_range_f32": [_P] * 4 + [c_int] * 3 + [_P, _P, _P, c_int64] + [_P] * 4 + [c_float] + [_P] * 6,
    "demon_mesh_components_scratch_bytes": [c_int, c_int64],
    "demon_mesh_components_count": [_P, c_int64, c_int, _P, _P, _P, _P],
    "demon_mesh_component_sizes": [_P, c_int64, _P, c_int, c_int64, _P, _P, _P],
    "demon_mesh_filter_count": [_P, c_int64, _P, c_int, _P, c_int64, _P, _P, _P, _P],
    "demon_mesh_filter": [_P, c_int64, _P, c_int, _P, c_int64] + [_P] * 10,
    "demon_net_create": [ctypes.POINTER(c_void_p), c_int, c_int, c_int, c_int],
    "demon_net_destroy": [_P],
    "demon_net_set_weight": [_P, c_char_p, _P, _P, c_int],
    "demon_net_num_variables": [_P],
    "demon_net_variable_name": [_P, c_int],
    "demon_net_finalize": [_P],
    "demon_bootstrap_forward": [_P] + [_P] * 8 + [c_int, _P],
    "demon_iterative_forward": [_P] + [_P] * 12 + [c_int, _P],
    "demon_refine_forward": [_P, _P, _P, _P, c_int, _P],
    "demon_net_create_v2": [ctypes.POINTER(c_void_p), c_int, c_int, c_int, c_int],
    "demon_net_variant": [_P],
    "demon_bootstrap_forward_v2": [_P] + [_P] * 8 + [c_int, _P],
    "demon_iterative_forward_v2": [_P] + [_P] * 12 + [c_int, _P],
    "demon_refine_forward_v2": [_P] * 6 + [c_int, _P],
    "demon_flow_block_forward_v2": [_P, c_char_p] + [_P] * 9 + [c_int, _P],
    "demon_depthmotion_block_forward_v2": [_P, c_char_p] + [_P] * 12 + [c_int, _P],
    "demon_pipeline_run": [_P, ctypes.POINTER(PipelineArgs), _P],
    "demon_pipeline_run_host": [_P, ctypes.POINTER(PipelineArgs), c_int, _P],
    "demon_debug_describe_plan": [c_int] * 5 + [_P, c_int],
    "demon_resize_u8": [_P, c_int64, c_int64, c_int, c_int, c_int, _P, c_int, c_int, c_int, _P],
    "demon_adjust_intrinsics_u8": [_P, c_int64, c_int64, c_int, c_int, c_int, _P] + [c_double] * 4 + [_P, c_int, c_int, _P, _P],
    "demon_resize_area_f32": [_P, c_int64, _P] + [c_int] * 6 + [_P],
    "demon_sharpness_u8": [_P, c_int64, c_int64, c_int, c_int, c_int, _P, _P],
    "demon_sun3d_depth_u16": [_P, c_int, c_int, c_int, _P, _P, _P],
    "demon_depth_ratios_f32": [_P] * 5 + [c_int] * 3 + [_P, c_int, _P, _P],
    "demon_depth_consistency_counts_f32": [_P] * 5 + [c_int] * 3 + [_P, c_int, c_float, c_float, _P, _P],
    "demon_datareader_prepare": [_P, _P, c_int, c_int, c_int, _P, _P, _P],
    "demon_datareader_batch": [_P, _P, c_int, c_int, _P, c_int, c_int] + [c_float] * 4 + [c_int] * 4 + [_P] * 5,
    "demon_net_batch": [_P],
    "demon_net_workspace_bytes": [_P],
    "demon_net_pipeline_launches": [_P, c_int],
    "demon_net_snapshot_launches": [_P, c_int],
    "demon_net_layer_uses_tensor_cores": [_P, c_char_p],
    "demon_net_profile_begin": [_P],
    "demon_net_profile_end": [_P],
    "demon_net_num_layers": [_P],
    "demon_net_layer_name": [_P, c_int],
    "demon_net_layer_profile": [_P, c_int, _P, _P, _P, _P],
    "demon_debug_tc_timeouts": [],
    "demon_check_errors": [],
    "demon_debug_describe_layers": [_P, _P, c_int],
    "demon_debug_trace_layers": [_P, _P, _P],
    "demon_debug_describe_conv": [c_int] * 13 + [_P, c_int],
    "demon_debug_last_conv_ms": [],
    "demon_debug_tc_timing": [c_int, _P, c_int],
    "demon_conv_slice_nhwc": [_P, c_int, _P] + [c_int] * 11 + [_P, _P, c_int, c_int, _P],
    "demon_conv_slice_nhwc_same": [_P, c_int, _P] + [c_int] * 10 + [_P, _P, c_int, c_int, _P],
    "demon_conv2d_nhwc": [_P, _P] + [c_int] * 9 + [_P, _P, c_int, c_int, _P],
    "demon_deconv4x4s2_nhwc": [_P, _P] + [c_int] * 5 + [_P, _P, c_int, c_int, _P],
    "demon_last_error": [],
    "demon_version": [],
    "demon_launch_count": [],
}
_RESTYPES = {
    "demon_net_destroy": None,
    "demon_net_variable_name": c_char_p,
    "demon_net_layer_name": c_char_p,
    "demon_net_workspace_bytes": c_int64,
    "demon_metric_workspace_bytes": c_int64,
    "demon_loss_workspace_bytes": c_int64,
    "demon_loss_ground_truth_workspace_bytes": c_int64,
    "demon_flow_warp_grad_workspace_bytes": c_int64,
    "demon_point_cloud_scratch_bytes": c_int64,
    "demon_marching_cubes_scratch_bytes": c_int64,
    "demon_sparse_tsdf_mesh_scratch_bytes": c_int64,
    "demon_sparse_tsdf_raycast_scratch_bytes": c_int64,
    "demon_tsdf_indexed_mesh_scratch_bytes": c_int64,
    "demon_sparse_tsdf_edge_scan_bytes": c_int64,
    "demon_mesh_components_scratch_bytes": c_int64,
    "demon_last_error": c_char_p,
    "demon_version": c_char_p,
    "demon_launch_count": c_int64,
    "demon_debug_last_conv_ms": c_double,
}

_lib = None


def lib_path():
    return os.environ.get("DEMON_B200_LIB", _DEFAULT)


def load():
    """Load the shared library (no CUDA call is made by loading)."""
    global _lib
    if _lib is None:
        path = lib_path()
        if not os.path.isfile(path):
            raise ValueError(
                "Cannot find libdemon_b200.so at %s. Build it with `python -m demon_b200.build` or set the "
                "environment variable DEMON_B200_LIB." % path)
        lib = ctypes.CDLL(path)
        for name, args in PROTOTYPES.items():
            fn = getattr(lib, name)   # AttributeError if the library does not export a declared symbol
            fn.argtypes = args
            fn.restype = _RESTYPES.get(name, c_int)
        _lib = lib
    return _lib


def check_errors():
    """Synchronise the current device and raise if a tensor-core kernel's bounded pipeline wait timed out since the last
    check (its outputs are garbage) or a CUDA error is pending.  Cheap enough to call once per batch."""
    check(load().demon_check_errors())


def check(rc):
    """Turn a DEMON_E_* return code into the exception the reference's Python layer would raise."""
    if rc == 0:
        return
    msg = load().demon_last_error().decode("utf-8", "replace")
    if rc == -1:
        raise ValueError(msg)
    raise RuntimeError("demon_b200 error %d: %s" % (rc, msg))
