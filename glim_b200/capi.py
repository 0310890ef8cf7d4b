"""ctypes binding of libglim_b200.so (the C-ABI of include/glim_b200.h).

There is no fallback of any kind: if the shared library is missing, or a call fails, this module
raises.  The product path never touches oracle/.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libglim_b200.so")

# every symbol include/glim_b200.h declares (tests check the library exports exactly these)
SYMBOLS = [
    "gb_status_string", "gb_last_error", "gb_device_count", "gb_mem_info",
    "gb_ctx_create", "gb_ctx_create_on_stream", "gb_ctx_destroy", "gb_ctx_synchronize", "gb_ctx_stream", "gb_ctx_kernel_launches",
    "gb_cloud_upload", "gb_cloud_size", "gb_cloud_download", "gb_cloud_device_ptrs", "gb_cloud_destroy",
    "gb_hessian_blocks", "gb_slab_row_hessian_blocks",
    "gb_voxelmap_build", "gb_voxelmap_info", "gb_voxelmap_download", "gb_voxelmap_destroy",
    "gb_voxelmap_create_incremental", "gb_voxelmap_insert",
    "gb_vgicp_factor_create", "gb_vgicp_factor_destroy", "gb_vgicp_linearize", "gb_vgicp_error",
    "gb_factor_set_linearize", "gb_factor_set_error",
    "gb_sweep_create", "gb_sweep_destroy", "gb_sweep_attach_slab", "gb_sweep_set_poses", "gb_sweep_launch", "gb_sweep_fetch", "gb_sweep_linearize",
    "gb_sweep_results_device", "gb_sweep_stats",
    "gb_peer_slab_create", "gb_peer_slab_export", "gb_peer_slab_connect", "gb_peer_slab_destroy", "gb_sweep_attach_peer_slab",
    "gb_peer_slab_signal_wait", "gb_peer_slab_device_ptr", "gb_peer_slab_fetch", "gb_peer_slab_fetch_async",
    "gb_overlap", "gb_covariances", "gb_find_neighbors", "gb_voxelgrid_sampling", "gb_preprocess_default_params", "gb_preprocess", "gb_merge_frames",
    "gb_deskew_pose_table", "gb_deskew",
    "gb_align_default_params", "gb_vgicp_align",
    "gb_ivox_create", "gb_ivox_insert", "gb_ivox_info", "gb_ivox_download", "gb_ivox_destroy", "gb_gicp_factor_create",
    "gb_cloud_add_times", "gb_cloud_time_table", "gb_ct_gicp_factor_create", "gb_ct_gicp_linearize", "gb_ct_gicp_error",
    "gb_ct_default_params", "gb_ct_gicp_align", "gb_ct_deskew",
    "gb_point_grid_build", "gb_point_grid_info", "gb_point_grid_download", "gb_point_grid_destroy", "gb_gicp_grid_factor_create",
    "gb_gicp_grid_factor_half_width",
    "gb_cloud_estimate_fpfh", "gb_cloud_fpfh", "gb_fpfh_match", "gb_ransac_default_params", "gb_ransac_align",
    "gb_gnc_default_params", "gb_gnc_align",
]

GB_SLAB_STRIDE = 96
GB_IPC_HANDLE_BYTES = 64
GB_FACTOR_SURFACE_VALIDATION = 1


class GlimB200Error(RuntimeError):
    pass


class PreprocessParams(C.Structure):
    """gb_preprocess_params (include/glim_b200.h)."""
    _fields_ = [("distance_near_thresh", C.c_double), ("distance_far_thresh", C.c_double), ("use_random_grid_downsampling", C.c_int), ("downsample_resolution", C.c_double),
                ("downsample_target", C.c_int), ("downsample_rate", C.c_double), ("seed", C.c_uint64), ("global_shutter", C.c_int), ("crop_bbox_frame", C.c_int),
                ("crop_bbox_min", C.c_double * 3), ("crop_bbox_max", C.c_double * 3), ("T_imu_lidar", C.c_double * 16), ("enable_outlier_removal", C.c_int), ("outlier_removal_k", C.c_int), ("outlier_std_mul_factor", C.c_double),
                ("k_correspondences", C.c_int), ("estimate_covariances", C.c_int), ("k_neighbors_cov", C.c_int), ("knn_cell_size", C.c_double)]


class Preprocessed(C.Structure):
    """gb_preprocessed (include/glim_b200.h)."""
    _fields_ = [("num_points", C.c_size_t), ("last_time", C.c_double), ("times", C.c_void_p), ("xyzw", C.c_void_p), ("intensities", C.c_void_p), ("neighbors", C.c_void_p),
                ("normals4", C.c_void_p), ("cov4x4", C.c_void_p), ("cloud", C.c_void_p)]


class AlignParams(C.Structure):
    """gb_align_params (include/glim_b200.h)."""
    _fields_ = [("max_iterations", C.c_int), ("lambda_initial", C.c_double), ("lambda_factor", C.c_double), ("lambda_upper_bound", C.c_double),
                ("relative_error_tol", C.c_double), ("absolute_error_tol", C.c_double), ("step_translation_tol", C.c_double), ("step_rotation_tol", C.c_double)]


class AlignResult(C.Structure):
    """gb_align_result (include/glim_b200.h)."""
    _fields_ = [("T_target_source", C.c_double * 16), ("error", C.c_double), ("num_inliers", C.c_double), ("lambda_", C.c_double),
                ("iterations", C.c_int), ("trials", C.c_int), ("status", C.c_int)]


class CtParams(C.Structure):
    """gb_ct_params (include/glim_b200.h)."""
    _fields_ = [("lm", AlignParams), ("location_consistency_inf_scale", C.c_double), ("constant_velocity_inf_scale", C.c_double)]


class CtResult(C.Structure):
    """gb_ct_result (include/glim_b200.h)."""
    _fields_ = [("X", C.c_double * 16), ("Y", C.c_double * 16), ("error", C.c_double), ("num_inliers", C.c_double), ("lambda_", C.c_double),
                ("iterations", C.c_int), ("trials", C.c_int), ("status", C.c_int)]


class RansacParams(C.Structure):
    """gb_ransac_params (include/glim_b200.h)."""
    _fields_ = [("max_iterations", C.c_int), ("early_stop_inlier_rate", C.c_double), ("inlier_voxel_resolution", C.c_double), ("dof", C.c_int), ("seed", C.c_uint64)]


class RansacResult(C.Structure):
    """gb_ransac_result (include/glim_b200.h)."""
    _fields_ = [("T_target_source", C.c_double * 16), ("inlier_rate", C.c_double), ("inliers", C.c_int), ("best_hypothesis", C.c_int), ("evaluated", C.c_int),
                ("status", C.c_int)]


class GncParams(C.Structure):
    """gb_gnc_params (include/glim_b200.h)."""
    _fields_ = [("max_init_samples", C.c_int), ("dof", C.c_int), ("seed", C.c_uint64)]


class GncResult(C.Structure):
    """gb_gnc_result (include/glim_b200.h)."""
    _fields_ = [("T_target_source", C.c_double * 16), ("inlier_rate", C.c_double), ("inliers", C.c_int), ("samples", C.c_int), ("correspondences", C.c_int),
                ("iterations", C.c_int), ("status", C.c_int)]


# gb_ransac_result::status
RANSAC_FOUND, RANSAC_EARLY_STOP, RANSAC_DEGENERATE = 0, 1, 2
RANSAC_STATUS_NAMES = {0: "FOUND", 1: "EARLY_STOP", 2: "DEGENERATE"}
FPFH_DIM = 33

# gb_gnc_result::status
GNC_FOUND, GNC_DEGENERATE = 0, 1
GNC_STATUS_NAMES = {0: "FOUND", 1: "DEGENERATE"}

# gb_align_result::status
ALIGN_CONVERGED, ALIGN_MAX_ITERATIONS, ALIGN_LAMBDA_EXCEEDED, ALIGN_DEGENERATE = 0, 1, 2, 3
ALIGN_STATUS_NAMES = {0: "CONVERGED", 1: "MAX_ITERATIONS", 2: "LAMBDA_EXCEEDED", 3: "DEGENERATE"}

_lib = None


def lib():
    """Load libglim_b200.so (raises if it is not built -- run `python -c 'import __graft_entry__ as g; g.build()'`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise GlimB200Error(f"{SO_PATH} is missing: the CUDA extension is not built (python __graft_entry__.py build); there is no CPU fallback")
    L = C.CDLL(SO_PATH)
    vp, i32, f32, f64, sz, u64 = C.c_void_p, C.c_int, C.c_float, C.c_double, C.c_size_t, C.c_uint64
    L.gb_status_string.restype = C.c_char_p
    L.gb_status_string.argtypes = [i32]
    L.gb_last_error.restype = C.c_char_p
    L.gb_device_count.restype = i32
    L.gb_mem_info.argtypes = [i32, vp, vp]
    L.gb_ctx_create.argtypes = [i32, vp]
    L.gb_ctx_create_on_stream.argtypes = [i32, vp, vp]
    L.gb_ctx_destroy.argtypes = [vp]
    L.gb_ctx_synchronize.argtypes = [vp]
    L.gb_ctx_stream.restype = vp
    L.gb_ctx_stream.argtypes = [vp]
    L.gb_ctx_kernel_launches.restype = u64
    L.gb_ctx_kernel_launches.argtypes = [vp]
    L.gb_cloud_upload.argtypes = [vp, sz, vp, vp, vp, vp]
    L.gb_cloud_size.argtypes = [vp, vp]
    L.gb_cloud_download.argtypes = [vp, vp, vp]
    L.gb_cloud_destroy.argtypes = [vp]
    L.gb_cloud_device_ptrs.argtypes = [vp, vp, vp, vp, vp]
    L.gb_sweep_linearize.argtypes = [vp, vp, vp]
    L.gb_preprocess_default_params.argtypes = [vp]
    L.gb_preprocess.argtypes = [vp, sz, vp, vp, vp, vp, vp]
    L.gb_merge_frames.argtypes = [vp, sz, vp, vp, f64, i32, u64, vp, vp, vp, vp]
    L.gb_hessian_blocks.argtypes = [vp, f64, vp, vp, vp, vp, vp, vp]
    L.gb_slab_row_hessian_blocks.argtypes = [vp, f64, vp, vp, vp, vp, vp, vp, vp]
    L.gb_voxelmap_build.argtypes = [vp, vp, f32, i32, i32, f64, vp]
    L.gb_voxelmap_info.argtypes = [vp, vp, vp, vp]
    L.gb_voxelmap_download.argtypes = [vp, vp, vp, vp, vp]
    L.gb_voxelmap_destroy.argtypes = [vp]
    L.gb_voxelmap_create_incremental.argtypes = [vp, f32, i32, i32, f64, i32, i32, vp]
    L.gb_voxelmap_insert.argtypes = [vp, vp, vp, vp, f64, u64]
    L.gb_vgicp_factor_create.argtypes = [vp, vp, vp, i32, vp]
    L.gb_vgicp_factor_destroy.argtypes = [vp]
    L.gb_vgicp_linearize.argtypes = [vp, vp, vp]
    L.gb_vgicp_error.argtypes = [vp, vp, vp, vp]
    L.gb_factor_set_linearize.argtypes = [vp, sz, vp, vp, vp]
    L.gb_factor_set_error.argtypes = [vp, sz, vp, vp, vp, vp]
    L.gb_sweep_create.argtypes = [vp, sz, vp, vp, vp]
    L.gb_sweep_destroy.argtypes = [vp]
    L.gb_sweep_attach_slab.argtypes = [vp, vp, sz]
    L.gb_sweep_set_poses.argtypes = [vp, vp]
    L.gb_sweep_launch.argtypes = [vp]
    L.gb_sweep_fetch.argtypes = [vp, vp]
    L.gb_sweep_results_device.argtypes = [vp, vp]
    L.gb_sweep_stats.argtypes = [vp, vp, vp, vp, vp]
    L.gb_peer_slab_create.argtypes = [vp, sz, i32, i32, vp]
    L.gb_peer_slab_export.argtypes = [vp, vp]
    L.gb_peer_slab_connect.argtypes = [vp, vp]
    L.gb_peer_slab_destroy.argtypes = [vp]
    L.gb_sweep_attach_peer_slab.argtypes = [vp, vp]
    L.gb_peer_slab_signal_wait.argtypes = [vp]
    L.gb_peer_slab_device_ptr.argtypes = [vp, vp]
    L.gb_peer_slab_fetch.argtypes = [vp, vp]
    L.gb_peer_slab_fetch_async.argtypes = [vp, vp]
    L.gb_overlap.argtypes = [vp, sz, vp, vp, vp, vp]
    L.gb_covariances.argtypes = [vp, sz, vp, vp, i32, i32, vp, vp]
    L.gb_find_neighbors.argtypes = [vp, sz, vp, i32, vp]
    L.gb_voxelgrid_sampling.argtypes = [vp, sz, vp, vp, vp, f64, vp, vp, vp, vp]
    L.gb_deskew_pose_table.argtypes = [vp, vp, vp, sz, vp, vp, f64, sz, vp, vp, vp, vp]
    L.gb_deskew.argtypes = [vp, vp, vp, vp, sz, vp, vp, f64, sz, vp, vp, vp, vp]
    L.gb_align_default_params.argtypes = [vp]
    L.gb_vgicp_align.argtypes = [vp, sz, vp, vp, vp, vp, vp]
    L.gb_ivox_create.argtypes = [vp, f64, f64, i32, i32, i32, i32, vp]
    L.gb_ivox_insert.argtypes = [vp, vp, vp, vp, f64, u64]
    L.gb_ivox_info.argtypes = [vp, vp, vp, vp]
    L.gb_ivox_download.argtypes = [vp, vp, vp, vp, vp]
    L.gb_ivox_destroy.argtypes = [vp]
    L.gb_gicp_factor_create.argtypes = [vp, vp, vp, f64, vp]
    L.gb_cloud_add_times.argtypes = [vp, vp, sz, vp]
    L.gb_cloud_time_table.argtypes = [vp, vp, vp, vp, vp, vp]
    L.gb_ct_gicp_factor_create.argtypes = [vp, vp, vp, f64, vp]
    L.gb_ct_gicp_linearize.argtypes = [vp, vp, vp, vp]
    L.gb_ct_gicp_error.argtypes = [vp, vp, vp, vp, vp, vp]
    L.gb_ct_default_params.argtypes = [vp]
    L.gb_ct_gicp_align.argtypes = [vp, sz, vp, vp, vp, vp, vp, vp]
    L.gb_ct_deskew.argtypes = [vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp]
    L.gb_point_grid_build.argtypes = [vp, vp, f64, vp]
    L.gb_point_grid_info.argtypes = [vp, vp, vp, vp]
    L.gb_point_grid_download.argtypes = [vp, vp, vp, vp, vp, vp]
    L.gb_point_grid_destroy.argtypes = [vp]
    L.gb_gicp_grid_factor_create.argtypes = [vp, vp, vp, f64, vp]
    L.gb_gicp_grid_factor_half_width.argtypes = [vp, vp]
    L.gb_cloud_estimate_fpfh.argtypes = [vp, vp, f64]
    L.gb_cloud_fpfh.argtypes = [vp, vp]
    L.gb_fpfh_match.argtypes = [vp, vp, vp, vp]
    L.gb_ransac_default_params.argtypes = [vp]
    L.gb_ransac_align.argtypes = [vp, vp, vp, vp, vp, vp]
    L.gb_gnc_default_params.argtypes = [vp]
    L.gb_gnc_align.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    for name in SYMBOLS:
        getattr(L, name)  # AttributeError here means the library and include/glim_b200.h are out of sync
    _lib = L
    return L


def check(status):
    if status != 0:
        L = lib()
        raise GlimB200Error(f"{L.gb_status_string(status).decode()}: {L.gb_last_error().decode()}")


def ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def pose16(T):
    """4x4 (or ...x4x4) numpy pose(s) -> column-major 16-double rows (Eigen::Isometry3d::data())."""
    T = np.asarray(T, dtype=np.float64)
    return np.ascontiguousarray(np.swapaxes(T, -1, -2)).reshape(T.shape[:-2] + (16,))
