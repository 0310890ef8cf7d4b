"""ctypes binding of libglim_b200.so (the C-ABI of include/glim_b200.h).

There is no fallback of any kind: if the shared library is missing, or a call fails, this module
raises.  The product path never touches oracle/.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libglim_b200.so")

# every function include/glim_b200.h declares -> (argtypes, restype): pointers and arrays are c_void_p, and st is the gb_status
# code (tests/test_binding_host.py checks the table against the header's prototypes)
vp, i32, f32, f64, sz, u64, st = C.c_void_p, C.c_int, C.c_float, C.c_double, C.c_size_t, C.c_uint64, C.c_int
_SIGNATURES = {
    "gb_status_string": ([i32], C.c_char_p),
    "gb_last_error": ([], C.c_char_p),
    "gb_device_count": ([], i32),
    "gb_mem_info": ([i32, vp, vp], st),
    "gb_ctx_create": ([i32, vp], st),
    "gb_ctx_create_on_stream": ([i32, vp, vp], st),
    "gb_ctx_destroy": ([vp], st),
    "gb_ctx_synchronize": ([vp], st),
    "gb_ctx_stream": ([vp], vp),
    "gb_ctx_kernel_launches": ([vp], u64),
    "gb_cloud_upload": ([vp, sz, vp, vp, vp, vp], st),
    "gb_cloud_size": ([vp, vp], st),
    "gb_cloud_download": ([vp, vp, vp], st),
    "gb_cloud_device_ptrs": ([vp, vp, vp, vp, vp], st),
    "gb_cloud_destroy": ([vp], st),
    "gb_hessian_blocks": ([vp, f64, vp, vp, vp, vp, vp, vp], st),
    "gb_slab_row_hessian_blocks": ([vp, f64, vp, vp, vp, vp, vp, vp, vp], st),
    "gb_voxelmap_build": ([vp, vp, f32, i32, i32, f64, vp], st),
    "gb_voxelmap_info": ([vp, vp, vp, vp], st),
    "gb_voxelmap_download": ([vp, vp, vp, vp, vp], st),
    "gb_voxelmap_destroy": ([vp], st),
    "gb_voxelmap_create_incremental": ([vp, f32, i32, i32, f64, i32, i32, vp], st),
    "gb_voxelmap_insert": ([vp, vp, vp, vp, f64, u64], st),
    "gb_vgicp_factor_create": ([vp, vp, vp, i32, vp], st),
    "gb_vgicp_factor_destroy": ([vp], st),
    "gb_vgicp_linearize": ([vp, vp, vp], st),
    "gb_vgicp_error": ([vp, vp, vp, vp], st),
    "gb_factor_set_linearize": ([vp, sz, vp, vp, vp], st),
    "gb_factor_set_error": ([vp, sz, vp, vp, vp, vp], st),
    "gb_sweep_create": ([vp, sz, vp, vp, vp], st),
    "gb_sweep_destroy": ([vp], st),
    "gb_sweep_attach_slab": ([vp, vp, sz], st),
    "gb_sweep_set_poses": ([vp, vp], st),
    "gb_sweep_launch": ([vp], st),
    "gb_sweep_fetch": ([vp, vp], st),
    "gb_sweep_linearize": ([vp, vp, vp], st),
    "gb_sweep_results_device": ([vp, vp], st),
    "gb_sweep_stats": ([vp, vp, vp, vp, vp], st),
    "gb_peer_slab_create": ([vp, sz, i32, i32, vp], st),
    "gb_peer_slab_export": ([vp, vp], st),
    "gb_peer_slab_connect": ([vp, vp], st),
    "gb_peer_slab_destroy": ([vp], st),
    "gb_sweep_attach_peer_slab": ([vp, vp], st),
    "gb_peer_slab_signal_wait": ([vp], st),
    "gb_peer_slab_device_ptr": ([vp, vp], st),
    "gb_peer_slab_fetch": ([vp, vp], st),
    "gb_peer_slab_fetch_async": ([vp, vp], st),
    "gb_overlap": ([vp, sz, vp, vp, vp, vp], st),
    "gb_find_overlapping_submaps": ([vp, sz, vp, vp, vp, sz, sz, vp, f64, f64, sz, vp, vp, vp], st),
    "gb_covariances": ([vp, sz, vp, vp, i32, i32, vp, vp], st),
    "gb_find_neighbors": ([vp, sz, vp, i32, vp], st),
    "gb_voxelgrid_sampling": ([vp, sz, vp, vp, vp, f64, vp, vp, vp, vp], st),
    "gb_preprocess_default_params": ([vp], st),
    "gb_preprocess": ([vp, sz, vp, vp, vp, vp, vp], st),
    "gb_merge_frames": ([vp, sz, vp, vp, f64, i32, u64, vp, vp, vp, vp], st),
    "gb_deskew_pose_table": ([vp, vp, vp, sz, vp, vp, f64, sz, vp, vp, vp, vp], st),
    "gb_deskew": ([vp, vp, vp, vp, sz, vp, vp, f64, sz, vp, vp, vp, vp], st),
    "gb_align_default_params": ([vp], st),
    "gb_vgicp_align": ([vp, sz, vp, vp, vp, vp, vp], st),
    "gb_graph_optimize": ([vp, sz, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp], st),
    "gb_pose_graph_optimize": ([vp, sz, vp, sz, vp, vp, sz, vp, vp, vp, sz, vp, vp, vp, vp], st),
    "gb_imu_default_params": ([vp], st),
    "gb_imu_preintegrate": ([vp, sz, vp, sz, vp, vp, vp, vp], st),
    "gb_nav_graph_optimize": ([vp, sz, vp, sz, vp, sz, vp, sz, vp, vp, sz, vp, vp, vp, sz, vp, sz, vp, sz, vp, vp, vp, vp, vp, vp], st),
    "gb_ivox_create": ([vp, f64, f64, i32, i32, i32, i32, vp], st),
    "gb_ivox_insert": ([vp, vp, vp, vp, f64, u64], st),
    "gb_ivox_info": ([vp, vp, vp, vp], st),
    "gb_ivox_download": ([vp, vp, vp, vp, vp], st),
    "gb_ivox_destroy": ([vp], st),
    "gb_ivox_extract": ([vp, vp, vp, i32, u64, vp], st),
    "gb_gicp_factor_create": ([vp, vp, vp, f64, vp], st),
    "gb_cloud_add_times": ([vp, vp, sz, vp], st),
    "gb_cloud_time_table": ([vp, vp, vp, vp, vp, vp], st),
    "gb_ct_gicp_factor_create": ([vp, vp, vp, f64, vp], st),
    "gb_ct_gicp_linearize": ([vp, vp, vp, vp], st),
    "gb_ct_gicp_error": ([vp, vp, vp, vp, vp, vp], st),
    "gb_ct_default_params": ([vp], st),
    "gb_ct_gicp_align": ([vp, sz, vp, vp, vp, vp, vp, vp], st),
    "gb_ct_deskew": ([vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp], st),
    "gb_point_grid_build": ([vp, vp, f64, vp], st),
    "gb_point_grid_info": ([vp, vp, vp, vp], st),
    "gb_point_grid_download": ([vp, vp, vp, vp, vp, vp], st),
    "gb_point_grid_destroy": ([vp], st),
    "gb_gicp_grid_factor_create": ([vp, vp, vp, f64, vp], st),
    "gb_gicp_grid_factor_half_width": ([vp, vp], st),
    "gb_icp_grid_factor_create": ([vp, vp, vp, f64, vp], st),
    "gb_cloud_estimate_normals": ([vp, vp], st),
    "gb_cloud_normals": ([vp, vp], st),
    "gb_cloud_estimate_covariances": ([vp, vp, i32, i32], st),
    "gb_cloud_estimate_fpfh": ([vp, vp, f64], st),
    "gb_cloud_fpfh": ([vp, vp], st),
    "gb_fpfh_match": ([vp, vp, vp, vp], st),
    "gb_ransac_default_params": ([vp], st),
    "gb_ransac_align": ([vp, vp, vp, vp, vp, vp], st),
    "gb_gnc_default_params": ([vp], st),
    "gb_gnc_align": ([vp, vp, vp, vp, vp, vp, vp], st),
    "gb_concat_frames": ([vp, sz, vp, vp, vp, vp, vp, vp], st),
    "gb_region_growing_default_params": ([vp], st),
    "gb_region_growing": ([vp, vp, vp, vp, vp, vp, vp], st),
    "gb_min_cut_default_params": ([vp], st),
    "gb_min_cut": ([vp, vp, vp, vp, vp, vp, vp, vp], st),
    "gb_select_gizmo": ([vp, sz, vp, vp, vp, i32, vp, vp], st),
    "gb_select_radius_default_params": ([vp], st),
    "gb_select_radius": ([vp, vp, vp, vp, vp, vp], st),
    "gb_remove_points": ([vp, sz, vp, sz, vp, vp, vp, vp], st),
    "gb_plane_patch_default_params": ([vp], st),
    "gb_plane_patch": ([vp, sz, vp, vp, vp, vp, vp], st),
    "gb_plane_auto_radius": ([vp, sz, vp, vp, vp, vp], st),
    "gb_plane_evm_factor_create": ([vp, sz, vp, vp, vp, vp], st),
    "gb_plane_evm_factor_info": ([vp, vp, vp, vp, vp], st),
    "gb_plane_evm_linearize": ([vp, sz, vp, vp, vp, vp, vp, vp], st),
    "gb_plane_evm_error": ([vp, sz, vp, vp, vp], st),
}
del vp, i32, f32, f64, sz, u64, st
SYMBOLS = tuple(_SIGNATURES)  # tests check the library exports exactly these

GB_SLAB_STRIDE = 96
GB_IPC_HANDLE_BYTES = 64
GB_FACTOR_SURFACE_VALIDATION = 1
# gb_cloud_estimate_covariances' outputs
GB_CLOUD_COVARIANCES, GB_CLOUD_NORMALS = 1, 2


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


GB_GRAPH_MAX_KEYS = 32
GB_POSE_GRAPH_MAX_KEYS = 1024
# gb_between_term (include/glim_b200.h): Z and information column-major
BETWEEN_DTYPE = np.dtype([("key_i", "<i4"), ("key_j", "<i4"), ("Z", "<f8", 16), ("information", "<f8", 36), ("huber_width", "<f8")], align=True)


GB_NAV_GRAPH_MAX_SLOTS = 2048
GB_OVERLAP_SEARCH_MAX_SUBMAPS = 4096


class ImuParams(C.Structure):
    """gb_imu_params (include/glim_b200.h)."""
    _fields_ = [("acc_noise", C.c_double), ("gyro_noise", C.c_double), ("int_noise", C.c_double), ("gravity", C.c_double * 3)]


# gb_imu_preintegrated (include/glim_b200.h): 9 x 3 and 9 x 9 matrices row-major
PREINTEGRATED_DTYPE = np.dtype([("delta_t", "<f8"), ("preintegrated", "<f8", 9), ("H_bias_acc", "<f8", (9, 3)), ("H_bias_omega", "<f8", (9, 3)),
                                ("covariance", "<f8", (9, 9)), ("bias_hat", "<f8", 6), ("gravity", "<f8", 3), ("num_integrated", "<i4"), ("pad", "<i4")], align=True)
IMU_TERM_DTYPE = np.dtype([("pose_i", "<i4"), ("vel_i", "<i4"), ("pose_j", "<i4"), ("vel_j", "<i4"), ("bias_i", "<i4"), ("pad", "<i4"),
                           ("pim", PREINTEGRATED_DTYPE)], align=True)
VECTOR_TERM_DTYPE = np.dtype([("kind", "<i4"), ("key_a", "<i4"), ("key_b", "<i4"), ("pad", "<i4"), ("z", "<f8", 6), ("precision", "<f8")], align=True)
# gb_vector_term kinds (GB_VECTOR_*)
VECTOR_KINDS = {"velocity_prior": 0, "bias_prior": 1, "velocity_between": 2, "bias_between": 3, "rotate_velocity": 4}


class GraphResult(C.Structure):
    """gb_graph_result (include/glim_b200.h)."""
    _fields_ = [("error", C.c_double), ("num_inliers", C.c_double), ("lambda_", C.c_double), ("iterations", C.c_int), ("trials", C.c_int), ("status", C.c_int)]


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


class CellWindow(C.Structure):
    """gb_cell_window (include/glim_b200.h)."""
    _fields_ = [("cell_size", C.c_double), ("lo", C.c_int32 * 3), ("hi", C.c_int32 * 3)]


class RegionGrowingParams(C.Structure):
    """gb_region_growing_params (include/glim_b200.h)."""
    _fields_ = [("distance_threshold", C.c_double), ("angle_threshold", C.c_double), ("dilation_radius", C.c_double)]


class RegionGrowingResult(C.Structure):
    """gb_region_growing_result (include/glim_b200.h)."""
    _fields_ = [("seed", C.c_int32), ("status", C.c_int32), ("num_region", C.c_size_t), ("num_selected", C.c_size_t), ("num_components", C.c_size_t)]


# gb_region_growing_result::status
REGION_FOUND, REGION_NO_SEED = 0, 1
REGION_STATUS_NAMES = {0: "FOUND", 1: "NO_SEED"}


class MinCutParams(C.Structure):
    """gb_min_cut_params (include/glim_b200.h)."""
    _fields_ = [("distance_sigma", C.c_double), ("angle_sigma", C.c_double), ("foreground_mask_radius", C.c_double),
                ("background_mask_radius", C.c_double), ("foreground_weight", C.c_double), ("k_neighbors", C.c_int)]


class MinCutResult(C.Structure):
    """gb_min_cut_result (include/glim_b200.h)."""
    _fields_ = [("seed", C.c_int32), ("status", C.c_int32), ("num_points", C.c_size_t), ("num_foreground", C.c_size_t),
                ("num_background", C.c_size_t), ("num_edges", C.c_size_t), ("num_selected", C.c_size_t), ("cut_value", C.c_int64),
                ("rounds", C.c_int32)]


# gb_min_cut_result::status
MINCUT_FOUND, MINCUT_NO_SEED, MINCUT_NOT_CONVERGED = 0, 1, 2
MINCUT_STATUS_NAMES = {0: "FOUND", 1: "NO_SEED", 2: "NOT_CONVERGED"}

# gb_select_gizmo's shape
GIZMO_BOX, GIZMO_SPHERE = 0, 1


class SelectRadiusParams(C.Structure):
    """gb_select_radius_params (include/glim_b200.h)."""
    _fields_ = [("radius", C.c_double), ("radius_offset", C.c_double), ("stddev_thresh", C.c_double), ("mode", C.c_int32), ("k", C.c_int32)]


class SelectRadiusResult(C.Structure):
    """gb_select_radius_result (include/glim_b200.h)."""
    _fields_ = [("status", C.c_int32), ("num_participants", C.c_size_t), ("num_selected", C.c_size_t), ("threshold", C.c_double)]


# gb_select_radius_params::mode and gb_select_radius_result::status
RADIUS_INSIDE, RADIUS_OUTLIERS = 0, 1
RADIUS_OK, RADIUS_NOT_ENOUGH_POINTS = 0, 1
RADIUS_STATUS_NAMES = {0: "OK", 1: "NOT_ENOUGH_POINTS"}


class RemovePointsResult(C.Structure):
    """gb_remove_points_result (include/glim_b200.h)."""
    _fields_ = [("num_removed", C.c_size_t), ("num_ignored", C.c_size_t), ("num_changed", C.c_size_t)]


class PlanePatchParams(C.Structure):
    """gb_plane_patch_params (include/glim_b200.h)."""
    _fields_ = [("center", C.c_double * 3), ("radius", C.c_double), ("max_frame_distance", C.c_double), ("min_radius", C.c_double),
                ("max_radius", C.c_double), ("plane_eps", C.c_double)]


PLANE_MAX_TRIALS = 10


class PlanePatchResult(C.Structure):
    """gb_plane_patch_result (include/glim_b200.h)."""
    _fields_ = [("radius", C.c_double), ("num_points", C.c_size_t), ("eigenvalues", C.c_double * 3), ("num_trials", C.c_int32),
                ("trial_radius", C.c_double * PLANE_MAX_TRIALS), ("trial_points", C.c_size_t * PLANE_MAX_TRIALS)]


# gb_plane_evm_linearize's status
PLANE_EVM_OK, PLANE_EVM_DEGENERATE = 0, 1
PLANE_EVM_STATUS_NAMES = {0: "OK", 1: "DEGENERATE"}

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
    for name, (argtypes, restype) in _SIGNATURES.items():
        fn = getattr(L, name)  # AttributeError here means the library and include/glim_b200.h are out of sync
        fn.argtypes, fn.restype = argtypes, restype
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
