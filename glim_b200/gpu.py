"""Host-side mirror (Python) of the gtsam_points GPU class surface GLIM constructs (SURVEY.md 8(b) 'inner'
boundary), forwarding to the C-ABI of libglim_b200.so.  Same names, argument meaning and defaults as
the reference call sites; used by the parity tests and the bench.  The C++ twin of this file is
include/glim_b200/gtsam_points_compat.hpp.

    PointCloudGPU.clone(points, covs)                       odometry_estimation_gpu.cpp:96
    GaussianVoxelMapGPU(resolution, 8192*2, 10, 1e-3).insert(cloud)   odometry_estimation_gpu.cpp:103-104
    IncrementalVoxelMapGPU(resolution, lru_horizon).insert(cloud, T, rate)   GaussianVoxelMapCPU::insert, odometry_estimation_cpu.cpp:177-191
    IntegratedVGICPFactorGPU(target_key | fixed_target_pose, source_key, voxelmap, source)   :144, :161
    NonlinearFactorSetGPU.add(...) / .linearize(values)     odometry_estimation_gpu.cpp:383-386
    overlap_gpu(voxelmap(s), source, delta(s))              odometry_estimation_gpu.cpp:231, :248
    IVoxGPU(resolution, min_dist, ...).insert(cloud, T, rate)   gtsam_points::iVox, odometry_estimation_cpu.cpp:57-61, :177-191
    IntegratedGICPFactorGPU(target, source_key, ivox, source, max_corr)   odometry_estimation_cpu.cpp:95-104
    PointGridGPU(cloud, cell_size)                          the target frame's KdTree (global_mapping_pose_graph.cpp:273)
    IntegratedGICPFactorGPU(target, source_key, grid, source, max_corr)   IntegratedGICPFactor between frames: sub_mapping.cpp:189-211,
                                                            global_mapping.cpp:379-428, global_mapping_pose_graph.cpp:391-405
    IntegratedICPFactorGPU(target, source_key, grid, source, max_corr)   IntegratedICPFactor, manual_loop_close_modal.cpp:479-492
    align_vgicp(problems, T_init, params)                   the LM loop of odometry_estimation_cpu.cpp:105-150 /
                                                            global_mapping_pose_graph.cpp:405-417, many problems per call
    PointCloudGPU.add_times(times)                          PointCloud::add_times, odometry_estimation_ct.cpp:101
    IntegratedCT_GICPFactorGPU(key_X, key_Y, ivox, source, max_corr)   odometry_estimation_ct.cpp:159-163
    align_ct_gicp(factors, X_init, Y_init, X_prior, params) the CT LM solve with its motion priors, odometry_estimation_ct.cpp:166-182
    deskew_ct(cloud, X, Y, neighbors, k_neighbors)          deskewed_source_points + covariances, odometry_estimation_ct.cpp:199-204
    PointCloudGPU.estimate_normals() / .normals()           gtsam_points::estimate_normals, manual_loop_close_modal.cpp:391, :410
    PointCloudGPU.estimate_fpfh(radius) / .fpfh()           gtsam_points::estimate_fpfh, manual_loop_close_modal.cpp:382-397, :415
    fpfh_match(target, source)                              the target's KdTreeX over FPFH features, manual_loop_close_modal.cpp:402
    estimate_pose_ransac(target, source, **params)          gtsam_points::estimate_pose_ransac, manual_loop_close_modal.cpp:435-443
    estimate_pose_gnc(target, source, **params)             gtsam_points::estimate_pose_gnc, manual_loop_close_modal.cpp:446-458
    concat_frames(poses, frames, window)                    the map editor's world-frame cloud, points_selector.cpp:85-177;
                                                            GlobalMapping::export_points, global_mapping.cpp:638-680
    region_growing(cloud, seed_point, **params)             gtsam_points::region_growing_init / _update, points_selector.cpp:798-810
    min_cut(cloud, picked_point, **params)                  gtsam_points::min_cut, points_selector.cpp:774-796
    plane_patch(frames, poses, center, **params)            the bundle adjustment modal's Update, bundle_adjustment_modal.cpp:137-184
    plane_auto_radius(frames, poses, center, **params)      its Auto Radius, bundle_adjustment_modal.cpp:186-227
    PlaneEVMFactorGPU(frames, poses, center, **params)      gtsam_points::PlaneEVMFactor of its Create Factor, :229-245
    linearize_plane_evm(factors, poses_per_factor)          many PlaneEVMFactors relinearized in one launch
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi
from .capi import check, f64, lib, pose16, ptr

LIN_DTYPE = np.dtype([("H_tt", "f8", (36,)), ("H_ss", "f8", (36,)), ("H_ts", "f8", (36,)), ("b_t", "f8", (6,)), ("b_s", "f8", (6,)), ("error", "f8"), ("num_inliers", "f8")])
assert LIN_DTYPE.itemsize == 122 * 8


class _Handle:
    """An object holding one C-ABI handle `h`, which the class's `_destroy` function releases exactly once: on close() or when
    the object is collected.  The release does not depend on the Context being open: clouds and maps keep no context, and
    factors, sweeps and peer slabs hold a reference to theirs that their destroy function drops."""

    _destroy = ""  # the gb_*_destroy entry point of the class
    h = None

    @staticmethod
    def _create(create, *args) -> C.c_void_p:
        """create(*args, &handle) -> handle; raises if the call fails"""
        h = C.c_void_p()
        check(create(*args, C.byref(h)))
        return h

    def close(self):
        h, self.h = self.h, None
        if h:
            getattr(lib(), self._destroy)(h)

    def __del__(self):
        try:
            self.close()
        except Exception:  # at interpreter shutdown the module globals may already be gone
            pass


class Context(_Handle):
    """gtsam_points::CUDAStream + StreamTempBufferRoundRobin (odometry_estimation_gpu.cpp:76-77)."""

    _destroy = "gb_ctx_destroy"

    def __init__(self, device: int = 0, cuda_stream: int | None = None):
        if cuda_stream is None:
            self.h = self._create(lib().gb_ctx_create, device)
        else:
            self.h = self._create(lib().gb_ctx_create_on_stream, device, C.c_void_p(cuda_stream))
        self.device = device

    def synchronize(self):
        check(lib().gb_ctx_synchronize(self.h))

    @property
    def stream(self) -> int:
        return lib().gb_ctx_stream(self.h) or 0

    @property
    def kernel_launches(self) -> int:
        return lib().gb_ctx_kernel_launches(self.h)


_default_ctx = {}


def default_context(device: int = 0) -> Context:
    if device not in _default_ctx:
        _default_ctx[device] = Context(device)
    return _default_ctx[device]


class PointCloudGPU(_Handle):
    """gtsam_points::PointCloudGPU (device copy of points / covs / normals in fp32)."""

    _destroy = "gb_cloud_destroy"

    def __init__(self, ctx: Context, handle, n: int):
        self.ctx, self.h, self.n = ctx, handle, n

    @staticmethod
    def clone(points, covs=None, normals=None, ctx: Context | None = None) -> "PointCloudGPU":
        """points (N,4) fp64 with w = 1; covs (N,4,4) fp64 [i,row,col] (symmetric); normals (N,4) or None."""
        ctx = ctx or default_context()
        points = f64(points)
        n = points.shape[0]
        c16 = None
        if covs is not None:
            covs = np.asarray(covs, dtype=np.float64)
            # [i,row,col] -> column-major 4x4 per point
            c16 = np.ascontiguousarray(np.swapaxes(covs.reshape(n, 4, 4), 1, 2)).reshape(n, 16)
        nr = f64(normals) if normals is not None else None
        return PointCloudGPU(ctx, PointCloudGPU._create(lib().gb_cloud_upload, ctx.h, n, ptr(points), ptr(c16), ptr(nr)), n)

    def size(self) -> int:
        return self.n

    def download(self):
        xyz = np.empty((self.n, 3), np.float32)
        cov6 = np.empty((self.n, 6), np.float32)
        check(lib().gb_cloud_download(self.h, ptr(xyz), ptr(cov6)))
        return xyz, cov6

    def add_times(self, times):
        """PointCloud::add_times (odometry_estimation_ct.cpp:101): the cloud's time table (gb_cloud_add_times); times (n,) in
        the original point order, finite and non-decreasing."""
        t = f64(times).reshape(-1)
        check(lib().gb_cloud_add_times(self.ctx.h, self.h, t.shape[0], ptr(t)))
        return self

    def time_table(self):
        """-> (starts (B+1,) int32, tau (B,) float64, t_first, t_last); B = 0 without times"""
        B = C.c_int()
        check(lib().gb_cloud_time_table(self.h, C.byref(B), None, None, None, None))
        starts, tau = np.empty(B.value + 1, np.int32), np.empty(B.value, np.float64)
        t0, t1 = C.c_double(), C.c_double()
        check(lib().gb_cloud_time_table(self.h, None, ptr(starts), ptr(tau), C.byref(t0), C.byref(t1)))
        return (starts if B.value else np.zeros(0, np.int32)), tau, t0.value, t1.value

    def estimate_normals(self):
        """gtsam_points::estimate_normals(points, covs, n) (manual_loop_close_modal.cpp:391, :410): every point's normal from its
        own covariance, sign-ruled away from the origin, into the cloud's normals (gb_cloud_estimate_normals); the cloud must
        carry covariances.  Discards FPFH features computed earlier."""
        check(lib().gb_cloud_estimate_normals(self.ctx.h, self.h))
        return self

    def normals(self) -> np.ndarray:
        """-> (n, 3) float32 normals in the original point order"""
        out = np.empty((self.n, 3), np.float32)
        check(lib().gb_cloud_normals(self.h, ptr(out)))
        return out

    def estimate_fpfh(self, radius: float):
        """gtsam_points::estimate_fpfh with search_radius = radius (manual_loop_close_modal.cpp:382-397): the cloud's FPFH features,
        kept on the device with it (gb_cloud_estimate_fpfh); the cloud must carry normals.  A second call replaces them."""
        check(lib().gb_cloud_estimate_fpfh(self.ctx.h, self.h, float(radius)))
        return self

    def fpfh(self) -> np.ndarray:
        """-> (n, 33) float32 features in the original point order"""
        out = np.empty((self.n, capi.FPFH_DIM), np.float32)
        check(lib().gb_cloud_fpfh(self.h, ptr(out)))
        return out


class GaussianVoxelMapGPU(_Handle):
    """gtsam_points::GaussianVoxelMapGPU(resolution, init_num_buckets, max_bucket_scan_count, target_points_drop_rate)."""

    _destroy = "gb_voxelmap_destroy"

    def __init__(self, resolution: float, init_num_buckets: int = 8192 * 2, max_bucket_scan_count: int = 10, target_points_drop_rate: float = 1e-3, ctx: Context | None = None):
        self.resolution = float(resolution)
        self.init_num_buckets = init_num_buckets
        self.max_bucket_scan_count = max_bucket_scan_count
        self.target_points_drop_rate = target_points_drop_rate
        self.ctx = ctx
        self.num_voxels = 0
        self.num_buckets = 0
        self._cloud = None

    def insert(self, cloud: PointCloudGPU):
        if self.h is not None:
            raise capi.GlimB200Error("GaussianVoxelMapGPU::insert may be called once (as every GLIM call site does)")
        self.ctx = self.ctx or cloud.ctx
        self.h = self._create(lib().gb_voxelmap_build, self.ctx.h, cloud.h, self.resolution, self.init_num_buckets, self.max_bucket_scan_count, self.target_points_drop_rate)
        self._info()
        return self

    def _info(self):
        nv, nb, res = C.c_int(), C.c_int(), C.c_float()
        check(lib().gb_voxelmap_info(self.h, C.byref(nv), C.byref(nb), C.byref(res)))
        self.num_voxels, self.num_buckets = nv.value, nb.value

    def voxel_resolution(self) -> float:
        return self.resolution

    def download(self):
        buckets = np.empty((self.num_buckets, 4), np.int32)
        vnum = np.empty((self.num_voxels,), np.int32)
        vmean = np.empty((self.num_voxels, 3), np.float32)
        vcov = np.empty((self.num_voxels, 6), np.float32)
        check(lib().gb_voxelmap_download(self.h, ptr(buckets), ptr(vnum), ptr(vmean), ptr(vcov)))
        return buckets, vnum, vmean, vcov


class IncrementalVoxelMapGPU(_Handle):
    """A Gaussian voxel map kept on the device across frames (gb_voxelmap_create_incremental / gb_voxelmap_insert): the
    GaussianVoxelMapCPU::insert + set_lru_horizon target of GLIM's odometry (odometry_estimation_cpu.cpp:67, :177-191).  Accepted
    wherever a GaussianVoxelMapGPU is (factors, align_vgicp, overlap_gpu); factors and sweeps follow its inserts."""

    _destroy = "gb_voxelmap_destroy"

    def __init__(self, resolution: float, lru_horizon: int = 0, lru_clear_cycle: int = 10, init_num_buckets: int = 16384, max_bucket_scan_count: int = 10,
                 target_points_drop_rate: float = 1e-3, ctx: Context | None = None):
        self.ctx = ctx or default_context()
        self.resolution = float(resolution)
        self.h = self._create(lib().gb_voxelmap_create_incremental, self.ctx.h, self.resolution, init_num_buckets, max_bucket_scan_count,
                              target_points_drop_rate, int(lru_horizon), int(lru_clear_cycle))
        self._info()

    _info = GaussianVoxelMapGPU._info

    def insert(self, cloud: PointCloudGPU, T=None, sampling_rate: float = 1.0, seed: int = 0):
        """Insert `cloud` at T_map_cloud (4x4, None = identity), keeping a sampling_rate share of its points."""
        Tc = pose16(np.asarray(T, dtype=np.float64).reshape(4, 4)) if T is not None else None
        check(lib().gb_voxelmap_insert(self.ctx.h, self.h, cloud.h, ptr(Tc), float(sampling_rate), int(seed)))
        self._info()
        return self

    def voxel_resolution(self) -> float:
        return self.resolution

    download = GaussianVoxelMapGPU.download


def unpack_linearized(rec) -> dict:
    """gb_linearized6 record -> numpy blocks indexed [row, col]."""
    return {
        "H_tt": np.asarray(rec["H_tt"]).reshape(6, 6).T.copy(),
        "H_ss": np.asarray(rec["H_ss"]).reshape(6, 6).T.copy(),
        "H_ts": np.asarray(rec["H_ts"]).reshape(6, 6).T.copy(),
        "b_t": np.asarray(rec["b_t"]).copy(),
        "b_s": np.asarray(rec["b_s"]).copy(),
        "error": float(rec["error"]),
        "num_inliers": float(rec["num_inliers"]),
    }


class IntegratedVGICPFactorGPU(_Handle):
    """gtsam_points::IntegratedVGICPFactorGPU.

    Binary form: (target_key, source_key, voxelmap, source); unary form: (fixed_target_pose 4x4, source_key, ...).
    `values` is a dict key -> 4x4 pose.  delta = T_target^-1 T_source (SURVEY A.1).  The handle is created on first use.
    """

    _destroy = "gb_vgicp_factor_destroy"

    def __init__(self, target, source_key, voxelmap: GaussianVoxelMapGPU, source: PointCloudGPU, ctx: Context | None = None):
        self.ctx = ctx or source.ctx
        if isinstance(target, np.ndarray):
            self.fixed_target_pose = np.asarray(target, dtype=np.float64).reshape(4, 4)
            self.target_key = None
        else:
            self.fixed_target_pose = None
            self.target_key = target
        self.source_key = source_key
        self.voxelmap, self.source = voxelmap, source  # keep alive, as the reference factor's shared_ptrs do
        self.flags = 0
        self._lin_point = None

    def set_enable_surface_validation(self, enable: bool):
        if self.h is not None:
            raise capi.GlimB200Error("set_enable_surface_validation must precede the first linearize")
        self.flags = capi.GB_FACTOR_SURFACE_VALIDATION if enable else 0

    def _handle(self):
        if self.h is None:
            self.h = self._create(lib().gb_vgicp_factor_create, self.ctx.h, self.voxelmap.h, self.source.h, self.flags)
        return self.h

    def keys(self):
        return [self.source_key] if self.target_key is None else [self.target_key, self.source_key]

    def dim(self):
        return 6

    def is_binary(self):
        return self.target_key is not None

    def get_fixed_target_pose(self):
        return self.fixed_target_pose

    def delta(self, values) -> np.ndarray:
        Tt = self.fixed_target_pose if self.target_key is None else np.asarray(values[self.target_key], dtype=np.float64)
        Ts = np.asarray(values[self.source_key], dtype=np.float64)
        Tti = np.eye(4)
        Tti[:3, :3] = Tt[:3, :3].T
        Tti[:3, 3] = -Tt[:3, :3].T @ Tt[:3, 3]
        return Tti @ Ts

    def linearize(self, values) -> dict:
        d = self.delta(values)
        self._lin_point = d
        out = np.zeros(1, LIN_DTYPE)
        check(lib().gb_vgicp_linearize(self._handle(), ptr(pose16(d)), ptr(out)))
        return unpack_linearized(out[0])

    def error(self, values) -> float:
        """error at `values` with the inlier set of the last linearization point (SURVEY A.2 / A.5)."""
        d = self.delta(values)
        lin = self._lin_point if self._lin_point is not None else d
        e = C.c_double()
        check(lib().gb_vgicp_error(self._handle(), ptr(pose16(lin)), ptr(pose16(d)), C.byref(e)))
        return e.value


class IVoxGPU(_Handle):
    """gtsam_points::iVox kept on the device (gb_ivox_create / gb_ivox_insert): the GICP target of GLIM's CPU odometry
    (odometry_estimation_cpu.cpp:57-61, update_target :177-191).  Factors and sweeps on it follow its inserts."""

    _destroy = "gb_ivox_destroy"

    def __init__(self, resolution: float, min_dist_in_cell: float = 0.1, max_points_in_cell: int = 10, neighbor_voxel_mode: int = 1,
                 lru_horizon: int = 100, lru_clear_cycle: int = 10, ctx: Context | None = None):
        self.ctx = ctx or default_context()
        self.resolution = float(resolution)
        self.h = self._create(lib().gb_ivox_create, self.ctx.h, self.resolution, float(min_dist_in_cell), int(max_points_in_cell), int(neighbor_voxel_mode),
                              int(lru_horizon), int(lru_clear_cycle))
        self.info()

    def info(self):
        """-> (num_voxels, num_points, resolution)"""
        nv, npt, res = C.c_int(), C.c_size_t(), C.c_double()
        check(lib().gb_ivox_info(self.h, C.byref(nv), C.byref(npt), C.byref(res)))
        self.num_voxels, self.num_points = nv.value, npt.value
        return nv.value, npt.value, res.value

    def insert(self, cloud: PointCloudGPU, T=None, sampling_rate: float = 1.0, seed: int = 0):
        """Insert `cloud` at T_map_cloud (4x4, None = identity), keeping a sampling_rate share of its points."""
        Tc = pose16(np.asarray(T, dtype=np.float64).reshape(4, 4)) if T is not None else None
        check(lib().gb_ivox_insert(self.ctx.h, self.h, cloud.h, ptr(Tc), float(sampling_rate), int(seed)))
        self.info()
        return self

    def voxel_resolution(self) -> float:
        return self.resolution

    def download(self):
        """-> voxel coords (V,3) int32 in ascending key order, counts (V,) int32, points (P,3) f32 and covariances (P,6) f32
        voxel-major in slot order"""
        V, P = self.num_voxels, self.num_points
        coords, counts = np.empty((V, 3), np.int32), np.empty(V, np.int32)
        xyz, cov6 = np.empty((P, 3), np.float32), np.empty((P, 6), np.float32)
        check(lib().gb_ivox_download(self.h, ptr(coords), ptr(counts), ptr(xyz), ptr(cov6)))
        return coords, counts, xyz, cov6


class PointGridGPU(_Handle):
    """A whole frame's points on the device, grouped in cubic cells (gb_point_grid_build): the target of a GICP factor between
    two frames, where gtsam_points builds a KdTree (global_mapping_pose_graph.cpp:273).  Built once from a PointCloudGPU, which
    may be released afterwards."""

    _destroy = "gb_point_grid_destroy"

    def __init__(self, cloud: PointCloudGPU, cell_size: float, ctx: Context | None = None):
        self.ctx = ctx or cloud.ctx
        self.cell_size = float(cell_size)
        self.h = self._create(lib().gb_point_grid_build, self.ctx.h, cloud.h, self.cell_size)
        nc, npt = C.c_int(), C.c_size_t()
        check(lib().gb_point_grid_info(self.h, C.byref(nc), C.byref(npt), None))
        self.num_cells, self.num_points = nc.value, npt.value

    def download(self):
        """-> cell coords (C,3) int32 in ascending key order, counts (C,) int32, original indices (P,) int32, points (P,3) f32 and
        covariances (P,6) f32 in record order"""
        Cn, P = self.num_cells, self.num_points
        coords, counts, idx = np.empty((Cn, 3), np.int32), np.empty(Cn, np.int32), np.empty(P, np.int32)
        xyz, cov6 = np.empty((P, 3), np.float32), np.empty((P, 6), np.float32)
        check(lib().gb_point_grid_download(self.h, ptr(coords), ptr(counts), ptr(idx), ptr(xyz), ptr(cov6)))
        return coords, counts, idx, xyz, cov6


class IntegratedGICPFactorGPU(IntegratedVGICPFactorGPU):
    """IntegratedGICPFactor_<iVox, PointCloud>(target, source_key, ivox, source) + set_max_correspondence_distance
    (odometry_estimation_cpu.cpp:95-104) on the device, or, with a PointGridGPU target, IntegratedGICPFactor between two frames
    (sub_mapping.cpp:189-211, global_mapping.cpp:379-428, global_mapping_pose_graph.cpp:391-405): a gb_factor like the VGICP one,
    so NonlinearFactorSetGPU, Sweep and align_vgicp take it (one target class per set, sweep or call)."""

    def __init__(self, target, source_key, ivox: "IVoxGPU | PointGridGPU", source: PointCloudGPU, max_correspondence_distance: float, ctx: Context | None = None):
        super().__init__(target, source_key, ivox, source, ctx=ctx)
        self.ivox = ivox
        self.max_correspondence_distance = float(max_correspondence_distance)

    def set_enable_surface_validation(self, enable: bool):
        if enable:
            raise capi.GlimB200Error("surface validation is a VGICP factor option")

    def _handle(self):
        if self.h is None:
            create = lib().gb_gicp_grid_factor_create if isinstance(self.ivox, PointGridGPU) else lib().gb_gicp_factor_create
            self.h = self._create(create, self.ctx.h, self.ivox.h, self.source.h, self.max_correspondence_distance)
        return self.h

    def search_half_width(self) -> int:
        """the search half-width m of a factor on a point grid (cells c + [-m, m]^3 are searched); 0 on an iVox"""
        m = C.c_int()
        check(lib().gb_gicp_grid_factor_half_width(self._handle(), C.byref(m)))
        return m.value


class IntegratedICPFactorGPU(IntegratedGICPFactorGPU):
    """IntegratedICPFactor(target, source_key, target_frame, source_frame) + set_max_correspondence_distance
    (manual_loop_close_modal.cpp:479-492, the fine registration of clouds without covariances) with the target's KdTree a
    PointGridGPU: point-to-point residuals on the grid factor's correspondences, no covariances needed.  NonlinearFactorSetGPU,
    Sweep and align_vgicp take it (ICP factors only per set, sweep or call)."""

    def __init__(self, target, source_key, grid: PointGridGPU, source: PointCloudGPU, max_correspondence_distance: float, ctx: Context | None = None):
        super().__init__(target, source_key, grid, source, max_correspondence_distance, ctx=ctx)

    def _handle(self):
        if self.h is None:
            self.h = self._create(lib().gb_icp_grid_factor_create, self.ctx.h, self.ivox.h, self.source.h, self.max_correspondence_distance)
        return self.h


class IntegratedCT_GICPFactorGPU(_Handle):
    """IntegratedCT_GICPFactor_<iVox, PointCloud>(X, Y, ivox, frame, ivox) + max_correspondence_distance
    (odometry_estimation_ct.cpp:159-163) on the device.  Its two keys are the poses at the scan's first and last time-table
    entries; the source must carry times (PointCloudGPU.add_times).  linearize(values) returns the usual dict with X in the
    target slot (H_tt = H_XX, b_t = b_X) and Y in the source slot (H_ss = H_YY, b_s = b_Y), H_ts = H_XY."""

    _destroy = "gb_vgicp_factor_destroy"

    def __init__(self, key_X, key_Y, ivox: IVoxGPU, source: PointCloudGPU, max_correspondence_distance: float, ctx: Context | None = None):
        self.ctx = ctx or source.ctx
        self.key_X, self.key_Y = key_X, key_Y
        self.ivox, self.source = ivox, source  # keep alive
        self.max_correspondence_distance = float(max_correspondence_distance)
        self._lin_point = None
        self.h = self._create(lib().gb_ct_gicp_factor_create, self.ctx.h, ivox.h, source.h, self.max_correspondence_distance)

    def keys(self):
        return [self.key_X, self.key_Y]

    def _handle(self):
        return self.h

    def poses(self, values):
        return np.asarray(values[self.key_X], dtype=np.float64).reshape(4, 4), np.asarray(values[self.key_Y], dtype=np.float64).reshape(4, 4)

    def linearize(self, values) -> dict:
        X, Y = self.poses(values)
        self._lin_point = (X, Y)
        out = np.zeros(1, LIN_DTYPE)
        check(lib().gb_ct_gicp_linearize(self.h, ptr(pose16(X)), ptr(pose16(Y)), ptr(out)))
        return unpack_linearized(out[0])

    def error(self, values) -> float:
        """error at `values` with the correspondences of the last linearization point"""
        X, Y = self.poses(values)
        Xl, Yl = self._lin_point if self._lin_point is not None else (X, Y)
        e = C.c_double()
        check(lib().gb_ct_gicp_error(self.h, ptr(pose16(Xl)), ptr(pose16(Yl)), ptr(pose16(X)), ptr(pose16(Y)), C.byref(e)))
        return e.value


def _params(p, fill, name, overrides):
    """p as fill (a gb_*_default_params) leaves it, with the given fields replaced; the fields of a nested gb_align_params `lm`
    may be given by name"""
    check(fill(C.byref(p)))
    for k, v in overrides.items():
        if hasattr(p, "lm") and k in dict(capi.AlignParams._fields_):
            setattr(p.lm, k, v)
        elif k in dict(type(p)._fields_) and k != "lm":
            setattr(p, k, v)
        else:
            raise capi.GlimB200Error(f"{name} has no field {k!r}")
    return p


def _pose(col16) -> np.ndarray:
    """a result struct's 16 column-major doubles -> (4,4)"""
    return np.array(col16[:]).reshape(4, 4).T.copy()


def _result(r, *poses) -> dict:
    """a gb_align_result / gb_ct_result as a dict: the named poses (4,4), then the fields the two share"""
    out = {k: _pose(getattr(r, k)) for k in poses}
    out.update({"error": r.error, "num_inliers": r.num_inliers, "lambda": r.lambda_, "iterations": r.iterations, "trials": r.trials,
                "status": r.status, "status_name": capi.ALIGN_STATUS_NAMES.get(r.status, "?")})
    return out


def ct_params(**overrides) -> capi.CtParams:
    """gb_ct_default_params (GLIM's shipped CT settings) with the given fields replaced; fields of gb_align_params may be
    given by name as well (max_iterations=..., ...)."""
    return _params(capi.CtParams(), lib().gb_ct_default_params, "gb_ct_params", overrides)


def align_ct_gicp(factors: list[IntegratedCT_GICPFactorGPU], X_init, Y_init, X_prior, params=None, ctx: Context | None = None) -> list[dict]:
    """gb_ct_gicp_align: the per-frame LM solve of GLIM's CT odometry (odometry_estimation_ct.cpp:159-182) for every problem
    in one call.  factors[p] is problem p's CT factor; X_init, Y_init, X_prior: (P,4,4); params: None (defaults), a dict of
    overrides or a capi.CtParams.  -> per problem {X, Y (4,4), error, num_inliers, lambda, iterations, trials, status, status_name}"""
    P = len(factors)
    if P == 0:
        return []
    if params is None or isinstance(params, dict):
        params = ct_params(**(params or {}))
    ctx = ctx or factors[0].ctx
    arr = (C.c_void_p * P)(*[f._handle() for f in factors])
    X0, Y0, Xp = (pose16(np.asarray(a, dtype=np.float64).reshape(P, 4, 4)) for a in (X_init, Y_init, X_prior))
    res = (capi.CtResult * P)()
    check(lib().gb_ct_gicp_align(ctx.h, P, C.cast(arr, C.c_void_p), ptr(X0), ptr(Y0), ptr(Xp), C.byref(params), C.cast(res, C.c_void_p)))
    return [_result(r, "X", "Y") for r in res]


def deskew_ct(cloud: PointCloudGPU, X, Y, neighbors, k_neighbors: int, host_outputs: bool = True, ctx: Context | None = None):
    """gb_ct_deskew: the deskewed frame of GLIM's CT odometry (deskewed_source_points(values, true) + covariance re-estimation
    with the same neighbour indices, odometry_estimation_ct.cpp:199-204).  cloud carries times; neighbors (n, k_correspondences)
    int32 in the original order.  -> (points (n,4), covs (n,4,4) [i,row,col], normals (n,4), PointCloudGPU); the host arrays are
    None unless host_outputs."""
    ctx = ctx or cloud.ctx
    nb = np.ascontiguousarray(neighbors, dtype=np.int32)
    n = cloud.n
    kc = nb.shape[1] if nb.ndim == 2 else 0
    pts = np.empty((n, 4)) if host_outputs else None
    cov = np.empty((n, 16)) if host_outputs else None
    nrm = np.empty((n, 4)) if host_outputs else None
    h = PointCloudGPU._create(lib().gb_ct_deskew, ctx.h, cloud.h, ptr(pose16(np.asarray(X, dtype=np.float64).reshape(4, 4))), ptr(pose16(np.asarray(Y, dtype=np.float64).reshape(4, 4))),
                              ptr(nb), int(kc), int(k_neighbors), ptr(pts), ptr(cov), ptr(nrm))
    out = PointCloudGPU(ctx, h, n)
    if not host_outputs:
        return None, None, None, out
    return pts, cov.reshape(n, 4, 4).transpose(0, 2, 1).copy(), nrm, out


def fpfh_match(target: PointCloudGPU, source: PointCloudGPU, ctx: Context | None = None) -> np.ndarray:
    """gb_fpfh_match: for every source feature the index of the nearest target feature (exact, ties to the smaller index),
    -> (n_source,) int32"""
    ctx = ctx or source.ctx
    out = np.empty(source.n, np.int32)
    check(lib().gb_fpfh_match(ctx.h, target.h, source.h, ptr(out)))
    return out


def ransac_params(**overrides) -> capi.RansacParams:
    """gb_ransac_default_params (the manual loop-closure modal's values) with the given fields replaced."""
    return _params(capi.RansacParams(), lib().gb_ransac_default_params, "gb_ransac_params", overrides)


def estimate_pose_ransac(target: PointCloudGPU, source: PointCloudGPU, ctx: Context | None = None, hypothesis_inliers: bool = False, **params) -> dict:
    """gtsam_points::estimate_pose_ransac (manual_loop_close_modal.cpp:435-443) on the device (gb_ransac_align): both clouds carry
    FPFH features; params are fields of gb_ransac_params (max_iterations, early_stop_inlier_rate, inlier_voxel_resolution, dof,
    seed).  -> {T_target_source (4,4), inliers, inlier_rate, best_hypothesis, evaluated, status, status_name} and, with
    hypothesis_inliers, the per-hypothesis counts (max_iterations,) int32 (-1 invalid sample, -2 not evaluated)."""
    ctx = ctx or source.ctx
    p = ransac_params(**params)
    r = capi.RansacResult()
    counts = np.empty(p.max_iterations, np.int32) if hypothesis_inliers else None
    check(lib().gb_ransac_align(ctx.h, target.h, source.h, C.byref(p), C.byref(r), ptr(counts)))
    out = {"T_target_source": _pose(r.T_target_source), "inliers": r.inliers, "inlier_rate": r.inlier_rate,
           "best_hypothesis": r.best_hypothesis, "evaluated": r.evaluated, "status": r.status, "status_name": capi.RANSAC_STATUS_NAMES.get(r.status, "?")}
    if counts is not None:
        out["hypothesis_inliers"] = counts
    return out


class NonlinearFactorSetGPU:
    """gtsam_points::NonlinearFactorSetGPU: batch linearization of every GPU factor of a graph."""

    def __init__(self, ctx: Context | None = None):
        self.ctx = ctx
        self.factors: list[IntegratedVGICPFactorGPU] = []

    def add(self, factors):
        for f in (factors if isinstance(factors, (list, tuple)) else [factors]):
            if isinstance(f, IntegratedVGICPFactorGPU):
                self.factors.append(f)
                self.ctx = self.ctx or f.ctx
        return self

    def size(self):
        return len(self.factors)

    def _handles(self):
        return (C.c_void_p * len(self.factors))(*[f._handle() for f in self.factors])

    def linearize(self, values) -> list[dict]:
        F = len(self.factors)
        if F == 0:
            return []
        deltas = np.stack([f.delta(values) for f in self.factors])
        for f, d in zip(self.factors, deltas):
            f._lin_point = d
        return [unpack_linearized(r) for r in self.linearize_deltas(deltas)]

    def linearize_deltas(self, deltas) -> np.ndarray:
        F = len(self.factors)
        out = np.zeros(F, LIN_DTYPE)
        if F:
            check(lib().gb_factor_set_linearize(self.ctx.h, F, C.cast(self._handles(), C.c_void_p), ptr(pose16(deltas)), ptr(out)))
        return out

    def error_deltas(self, deltas_lin, deltas_eval) -> np.ndarray:
        F = len(self.factors)
        out = np.zeros(F)
        if F:
            check(lib().gb_factor_set_error(self.ctx.h, F, C.cast(self._handles(), C.c_void_p), ptr(pose16(deltas_lin)), ptr(pose16(deltas_eval)), ptr(out)))
        return out


class Sweep(_Handle):
    """A prepared, device-resident batch (gb_sweep): upload poses / launch / fetch are separate steps."""

    _destroy = "gb_sweep_destroy"

    def __init__(self, ctx: Context, factors: list[IntegratedVGICPFactorGPU], pair_index=None):
        self.ctx = ctx
        self.factors = list(factors)
        F = len(factors)
        arr = (C.c_void_p * F)(*[f._handle() for f in factors])
        pi = np.ascontiguousarray(pair_index, dtype=np.int32) if pair_index is not None else None
        self.h = self._create(lib().gb_sweep_create, ctx.h, F, C.cast(arr, C.c_void_p), ptr(pi))
        self.F = F
        pf, ab, nt, gs = C.c_uint64(), C.c_uint64(), C.c_uint32(), C.c_uint32()
        check(lib().gb_sweep_stats(self.h, C.byref(pf), C.byref(ab), C.byref(nt), C.byref(gs)))
        self.point_factors, self.algorithmic_bytes, self.num_tiles, self.grid = pf.value, ab.value, nt.value, gs.value

    def attach_peer_slab(self, peer_slab: "PeerSlab | None"):
        self._peer = peer_slab  # keep alive
        check(lib().gb_sweep_attach_peer_slab(self.h, peer_slab.h if peer_slab is not None else None))

    def attach_slab(self, device_ptr: int, num_pairs: int):
        check(lib().gb_sweep_attach_slab(self.h, C.c_void_p(device_ptr), num_pairs))

    def set_poses(self, deltas):
        self._poses = pose16(deltas)  # keep the host array alive until the copy was staged
        check(lib().gb_sweep_set_poses(self.h, ptr(self._poses)))

    def launch(self):
        check(lib().gb_sweep_launch(self.h))

    def fetch(self) -> np.ndarray:
        out = np.zeros(self.F, LIN_DTYPE)
        check(lib().gb_sweep_fetch(self.h, ptr(out)))
        return out

    def linearize(self, deltas) -> np.ndarray:
        """gb_sweep_linearize: poses up, one launch (a CUDA graph for small sweeps), records down."""
        out = np.zeros(self.F, LIN_DTYPE)
        self._poses = pose16(deltas)
        check(lib().gb_sweep_linearize(self.h, ptr(self._poses), ptr(out)))
        return out

    def linearize_raw(self, poses16: np.ndarray, out: np.ndarray) -> np.ndarray:
        """The same call with caller-owned buffers (poses16: (F,16) float64 column-major, out: (F,) LIN_DTYPE): no Python-side
        array work around the C entry point."""
        check(lib().gb_sweep_linearize(self.h, poses16.ctypes.data, out.ctypes.data))
        return out

    def results_device_ptr(self) -> int:
        p = C.c_void_p()
        check(lib().gb_sweep_results_device(self.h, C.byref(p)))
        return p.value or 0


class PeerSlab(_Handle):
    """gb_peer_slab: ping-pong fp32 [num_pairs][96] result buffers shared with the other ranks of the box through CUDA
    IPC; the sweep's epilogue stores finished pair rows straight into every rank's buffer (multi-GPU exchange fused into
    the kernel, SURVEY 8(e)).  `exchange(handle_bytes) -> list[bytes]` must all-gather the 64-byte handles in rank order
    (torch.distributed in the bench); with world == 1 nothing is exchanged."""

    _destroy = "gb_peer_slab_destroy"

    def __init__(self, ctx: Context, num_pairs: int, world: int = 1, rank: int = 0, exchange=None):
        self.ctx, self.num_pairs, self.world, self.rank = ctx, num_pairs, world, rank
        self.h = self._create(lib().gb_peer_slab_create, ctx.h, num_pairs, world, rank)
        if world > 1:
            buf = (C.c_ubyte * capi.GB_IPC_HANDLE_BYTES)()
            check(lib().gb_peer_slab_export(self.h, C.cast(buf, C.c_void_p)))
            handles = exchange(bytes(buf))
            assert len(handles) == world and all(len(x) == capi.GB_IPC_HANDLE_BYTES for x in handles)
            blob = (C.c_ubyte * (capi.GB_IPC_HANDLE_BYTES * world)).from_buffer_copy(b"".join(handles))
            check(lib().gb_peer_slab_connect(self.h, C.cast(blob, C.c_void_p)))

    def signal_wait(self):
        check(lib().gb_peer_slab_signal_wait(self.h))

    def fetch(self) -> np.ndarray:
        out = np.empty((self.num_pairs, capi.GB_SLAB_STRIDE), np.float32)
        check(lib().gb_peer_slab_fetch(self.h, ptr(out)))
        return out

    def fetch_async(self) -> np.ndarray:
        """Enqueue the D2H into the slab's pinned buffer; the returned view is valid after the next stream sync."""
        p = C.POINTER(C.c_float)()
        check(lib().gb_peer_slab_fetch_async(self.h, C.byref(p)))
        return np.ctypeslib.as_array(p, shape=(self.num_pairs, capi.GB_SLAB_STRIDE))

    def device_ptr(self) -> int:
        p = C.c_void_p()
        check(lib().gb_peer_slab_device_ptr(self.h, C.byref(p)))
        return p.value or 0


def align_params(**overrides) -> capi.AlignParams:
    """gb_align_default_params (the odometry_estimation_cpu values) with the given fields replaced."""
    return _params(capi.AlignParams(), lib().gb_align_default_params, "gb_align_params", overrides)


def align_vgicp(problems: list[list[IntegratedVGICPFactorGPU]], T_init, params=None, ctx: Context | None = None) -> list[dict]:
    """gb_vgicp_align: Levenberg-Marquardt registration of every problem in one call (odometry_estimation_cpu.cpp:105-150,
    global_mapping_pose_graph.cpp:405-417).  problems[p] = the factors (levels) of problem p, used as unary factors on
    T_target_source with the target fixed at identity (their keys are not read); T_init: (P,4,4) or one (4,4) per problem;
    params: None (defaults), a dict of field overrides or a capi.AlignParams.
    -> per problem {T_target_source (4,4), error, num_inliers, lambda, iterations, trials, status, status_name}"""
    P = len(problems)
    if P == 0:
        return []
    if params is None or isinstance(params, dict):
        params = align_params(**(params or {}))
    flat = [f for prob in problems for f in prob]
    ctx = ctx or (flat[0].ctx if flat else default_context())
    off = np.zeros(P + 1, np.uint64)
    off[1:] = np.cumsum([len(prob) for prob in problems])
    T0 = pose16(np.asarray(T_init, dtype=np.float64).reshape(P, 4, 4))
    arr = (C.c_void_p * max(1, len(flat)))(*[f._handle() for f in flat])
    res = (capi.AlignResult * P)()
    check(lib().gb_vgicp_align(ctx.h, P, ptr(off), C.cast(arr, C.c_void_p), ptr(T0), C.byref(params), C.cast(res, C.c_void_p)))
    return [_result(r, "T_target_source") for r in res]


def overlap_gpu(voxelmaps, source: PointCloudGPU, deltas, ctx: Context | None = None) -> float:
    """gtsam_points::overlap_gpu: single (voxelmap, delta) or lists (odometry_estimation_gpu.cpp:231, :248)."""
    if isinstance(voxelmaps, (GaussianVoxelMapGPU, IncrementalVoxelMapGPU)):
        voxelmaps, deltas = [voxelmaps], [deltas]
    ctx = ctx or source.ctx
    T = len(voxelmaps)
    arr = (C.c_void_p * T)(*[m.h for m in voxelmaps])
    d = pose16(np.stack([np.asarray(x, dtype=np.float64) for x in deltas])) if T else np.zeros((0, 16))
    out = C.c_double()
    check(lib().gb_overlap(ctx.h, T, C.cast(arr, C.c_void_p), source.h, ptr(d), C.byref(out)))
    return out.value


def merge_frames_gpu(poses, frames, downsample_resolution: float, target_num_points: int = 0, seed: int = 0, ctx: Context | None = None, host_outputs: bool = True):
    """gtsam_points::merge_frames(poses, frames, downsample_resolution, target_num_points) on the device (sub_mapping.cpp:481-497).
    poses: K x (4,4) T_origin_frame; frames: K PointCloudGPU.  -> (points (M,4), covs (M,4,4) [i,row,col], PointCloudGPU)"""
    ctx = ctx or frames[0].ctx
    K, arr, T = _frames(frames, poses)
    cap = sum(f.n for f in frames)
    pts = np.empty((cap, 4)) if host_outputs else None
    cov = np.empty((cap, 16)) if host_outputs else None
    m = C.c_size_t()
    h = PointCloudGPU._create(lib().gb_merge_frames, ctx.h, K, arr, ptr(T), float(downsample_resolution), int(target_num_points), int(seed), ptr(pts), ptr(cov),
                              C.byref(m))
    cloud = PointCloudGPU(ctx, h, m.value) if h.value else None
    if not host_outputs:
        return None, None, cloud
    return pts[: m.value].copy(), cov[: m.value].reshape(-1, 4, 4).transpose(0, 2, 1).copy(), cloud


overlap_auto = overlap_gpu  # gtsam_points::overlap_auto dispatches to the GPU version for GPU voxel maps (sub_mapping.cpp:252)


def median_distance(points, max_scan_count: int = 256) -> float:
    """gtsam_points::median_distance(frame, 256) (odometry_estimation_gpu.cpp:91): strided sample of <= max_scan_count
    points, median of their norms.  256 points: stays on the host (SURVEY K6)."""
    points = np.asarray(points)
    n = points.shape[0]
    if n == 0:
        return 0.0
    step = max(1, n // max_scan_count)
    d = np.linalg.norm(points[::step, :3], axis=1)
    d = np.sort(d)
    return float(d[len(d) // 2])


def gnc_params(**overrides) -> capi.GncParams:
    """gb_gnc_default_params (the manual loop-closure modal's values) with the given fields replaced."""
    return _params(capi.GncParams(), lib().gb_gnc_default_params, "gb_gnc_params", overrides)


def estimate_pose_gnc(target: PointCloudGPU, source: PointCloudGPU, ctx: Context | None = None, correspondences: bool = False, **params) -> dict:
    """gtsam_points::estimate_pose_gnc as the modal runs it (manual_loop_close_modal.cpp:446-458: reciprocal matches, no tuple
    check) on the device (gb_gnc_align): both clouds carry FPFH features; params are fields of gb_gnc_params (max_init_samples,
    dof, seed).  -> {T_target_source (4,4), inliers, inlier_rate, samples, correspondences, iterations, status, status_name} and,
    with correspondences, pairs (K,2) int32 (source index, target index) and their final weights (K,)."""
    ctx = ctx or source.ctx
    p = gnc_params(**params)
    r = capi.GncResult()
    m = min(source.n, p.max_init_samples)
    pairs = np.empty((m, 2), np.int32) if correspondences else None
    weights = np.empty(m) if correspondences else None
    check(lib().gb_gnc_align(ctx.h, target.h, source.h, C.byref(p), C.byref(r), ptr(pairs), ptr(weights)))
    out = {"T_target_source": _pose(r.T_target_source), "inliers": r.inliers, "inlier_rate": r.inlier_rate,
           "samples": r.samples, "correspondences": r.correspondences, "iterations": r.iterations, "status": r.status,
           "status_name": capi.GNC_STATUS_NAMES.get(r.status, "?")}
    if correspondences:
        out["pairs"] = pairs[:r.correspondences].copy()
        out["weights"] = weights[:r.correspondences].copy()
    return out


def concat_frames(poses, frames, window=None, ctx: Context | None = None):
    """The submaps' device clouds in one world-frame device cloud (gb_concat_frames): poses K x (4,4) T_world_frame, frames K
    PointCloudGPU, window None (every point) or (cell_size, lo (3,), hi (3,)) inclusive cell bounds.  -> (PointCloudGPU, ids
    (M,) uint64 = (frame << 32) | original index, the map editor's point ids)"""
    ctx = ctx or (frames[0].ctx if len(frames) else default_context())
    K, arr, T = _frames(frames, poses)
    w = None
    if window is not None:
        cell, lo, hi = window
        w = capi.CellWindow(float(cell), (C.c_int32 * 3)(*[int(v) for v in lo]), (C.c_int32 * 3)(*[int(v) for v in hi]))
    ids = np.empty(sum(f.n for f in frames), np.uint64)
    h, m = C.c_void_p(), C.c_size_t()
    check(lib().gb_concat_frames(ctx.h, K, arr, ptr(T), C.byref(w) if w is not None else None, C.byref(h), ptr(ids), C.byref(m)))
    return PointCloudGPU(ctx, h, m.value), ids[: m.value].copy()


def region_growing_params(**overrides) -> capi.RegionGrowingParams:
    """gb_region_growing_default_params (this library's choice, not gtsam_points') with the given fields replaced."""
    return _params(capi.RegionGrowingParams(), lib().gb_region_growing_default_params, "gb_region_growing_params", overrides)


def region_growing(cloud: PointCloudGPU, seed_point, ctx: Context | None = None, labels: bool = False, **params) -> dict:
    """gtsam_points::region_growing_init + region_growing_update (points_selector.cpp:798-810) on the device
    (gb_region_growing): the connected surface of `cloud` (with normals) through the point nearest seed_point, dilated by
    dilation_radius.  params are fields of gb_region_growing_params (distance_threshold, angle_threshold in radians,
    dilation_radius).  -> {seed, status, status_name, num_region, num_selected, num_components, selected (num_selected,) int32
    in ascending original index} and, with labels, labels (n,) int32 (the component's smallest index, -1 for non-finite points)."""
    ctx = ctx or cloud.ctx
    p = region_growing_params(**params)
    r = capi.RegionGrowingResult()
    q = f64(np.asarray(seed_point, dtype=np.float64).reshape(-1)[:3])
    sel = np.empty(cloud.n, np.int32)
    lab = np.empty(cloud.n, np.int32) if labels else None
    check(lib().gb_region_growing(ctx.h, cloud.h, ptr(q), C.byref(p), C.byref(r), ptr(sel), ptr(lab)))
    out = {"seed": r.seed, "status": r.status, "status_name": capi.REGION_STATUS_NAMES.get(r.status, "?"), "num_region": r.num_region,
           "num_selected": r.num_selected, "num_components": r.num_components, "selected": sel[: r.num_selected].copy()}
    if lab is not None:
        out["labels"] = lab
    return out


def min_cut_params(**overrides) -> capi.MinCutParams:
    """gb_min_cut_default_params (the editor's radii and weight; this library's sigmas and k) with the given fields replaced."""
    return _params(capi.MinCutParams(), lib().gb_min_cut_default_params, "gb_min_cut_params", overrides)


def min_cut(cloud: PointCloudGPU, picked_point, ctx: Context | None = None, graph: bool = False, **params) -> dict:
    """gtsam_points::min_cut (points_selector.cpp:774-796) on the device (gb_min_cut): the object of `cloud` (with normals)
    around picked_point, cut from the background shell by a minimum s-t cut.  params are fields of gb_min_cut_params
    (distance_sigma, angle_sigma in radians, foreground_mask_radius, background_mask_radius, foreground_weight,
    k_neighbors).  -> {seed, status, status_name, num_points, num_foreground, num_background, num_edges, num_selected,
    cut_value (units of 2^-16), rounds, selected (num_selected,) int32 in ascending original index} and, with graph, edges
    (num_edges, 2) int32 original indices i < j ascending and capacities (num_edges,) int32: the graph the cut was taken on."""
    ctx = ctx or cloud.ctx
    p = min_cut_params(**params)
    r = capi.MinCutResult()
    q = f64(np.asarray(picked_point, dtype=np.float64).reshape(-1)[:3])
    sel = np.empty(cloud.n, np.int32)
    cap = cloud.n * max(int(p.k_neighbors), 0) if graph else 0
    e = np.empty((cap, 2), np.int32) if graph else None
    w = np.empty(cap, np.int32) if graph else None
    check(lib().gb_min_cut(ctx.h, cloud.h, ptr(q), C.byref(p), C.byref(r), ptr(sel), ptr(e), ptr(w)))
    out = {"seed": r.seed, "status": r.status, "status_name": capi.MINCUT_STATUS_NAMES.get(r.status, "?"), "num_points": r.num_points,
           "num_foreground": r.num_foreground, "num_background": r.num_background, "num_edges": r.num_edges, "num_selected": r.num_selected,
           "cut_value": r.cut_value, "rounds": r.rounds, "selected": sel[: r.num_selected].copy()}
    if graph:
        out["edges"] = e[: r.num_edges].copy()
        out["capacities"] = w[: r.num_edges].copy()
    return out


def plane_patch_params(center=(0.0, 0.0, 0.0), **overrides) -> capi.PlanePatchParams:
    """gb_plane_patch_default_params (the bundle adjustment modal's) at `center`, with the given fields replaced."""
    p = _params(capi.PlanePatchParams(), lib().gb_plane_patch_default_params, "gb_plane_patch_params", overrides)
    p.center = (C.c_double * 3)(*[float(v) for v in np.asarray(center, dtype=np.float64).reshape(-1)[:3]])
    return p


def _frames(frames, poses):
    """(K, handle array, K x 16 column-major poses) of a frame list and its T_world_frame poses"""
    K = len(frames)
    arr = (C.c_void_p * max(K, 1))(*[f.h for f in frames])
    T = pose16(np.stack([np.asarray(p, dtype=np.float64) for p in poses])) if K else np.zeros((0, 16))
    return K, C.cast(arr, C.c_void_p), T


def _patch(r: capi.PlanePatchResult) -> dict:
    t = r.num_trials
    return {"radius": r.radius, "num_points": r.num_points, "eigenvalues": np.array(r.eigenvalues[:]),
            "trials": [(r.trial_radius[i], r.trial_points[i]) for i in range(t)]}


def plane_patch(frames, poses, center, ids: bool = False, ctx: Context | None = None, **params) -> dict:
    """The bundle adjustment modal's Update (gb_plane_patch): the points of the submaps within max_frame_distance of `center`
    that lie within `radius` of it, their count and covariance eigenvalues (ascending).  frames K PointCloudGPU, poses K x (4,4)
    T_world_submap; params are fields of gb_plane_patch_params.  -> {radius, num_points, eigenvalues (3,), trials []} and, with
    ids, ids (num_points,) uint64 = (frame << 32) | original index, frame-major and ascending."""
    ctx = ctx or (frames[0].ctx if len(frames) else default_context())
    K, arr, T = _frames(frames, poses)
    p = plane_patch_params(center, **params)
    r = capi.PlanePatchResult()
    buf = np.empty(sum(f.n for f in frames), np.uint64) if ids else None
    check(lib().gb_plane_patch(ctx.h, K, arr, ptr(T), C.byref(p), C.byref(r), ptr(buf)))
    out = _patch(r)
    if ids:
        out["ids"] = buf[: r.num_points].copy()
    return out


def plane_auto_radius(frames, poses, center, ctx: Context | None = None, **params) -> dict:
    """The bundle adjustment modal's Auto Radius (gb_plane_auto_radius): the radius its loop settles on, with the count and
    eigenvalues there, and trials [(radius, count)] of every evaluated trial in order."""
    ctx = ctx or (frames[0].ctx if len(frames) else default_context())
    K, arr, T = _frames(frames, poses)
    p = plane_patch_params(center, **params)
    r = capi.PlanePatchResult()
    check(lib().gb_plane_auto_radius(ctx.h, K, arr, ptr(T), C.byref(p), C.byref(r)))
    return _patch(r)


class PlaneEVMFactorGPU(_Handle):
    """gtsam_points::PlaneEVMFactor of the bundle adjustment modal's Create Factor (gb_plane_evm_factor_create): the submap
    points within `radius` of `center`, keyed by their submap.  keys: the frame indices (in the creating list) that hold
    selected points; key_points: their counts.  linearize(poses) / error(poses) take the keys' T_world_submap poses, as a
    (K, 4, 4) array in key order or a dict {frame index: (4, 4)}.  The factor keeps its moments on the host: its frames may be
    destroyed after creation."""

    _destroy = "gb_vgicp_factor_destroy"

    def __init__(self, frames, poses, center, ctx: Context | None = None, **params):
        self.ctx = ctx or (frames[0].ctx if len(frames) else default_context())
        K, arr, T = _frames(frames, poses)
        p = plane_patch_params(center, **params)
        self.h = self._create(lib().gb_plane_evm_factor_create, self.ctx.h, K, arr, ptr(T), C.byref(p))
        nk, npts = C.c_size_t(), C.c_size_t()
        check(lib().gb_plane_evm_factor_info(self.h, C.byref(nk), C.byref(npts), None, None))
        self.keys = np.empty(nk.value, np.int32)
        self.key_points = np.empty(nk.value, np.uint64)
        check(lib().gb_plane_evm_factor_info(self.h, None, None, ptr(self.keys), ptr(self.key_points)))
        self.num_points = npts.value

    def _handle(self):
        return self.h

    def key_poses(self, poses) -> np.ndarray:
        if isinstance(poses, dict):
            poses = [poses[int(k)] for k in self.keys]
        return np.asarray(poses, dtype=np.float64).reshape(len(self.keys), 4, 4)

    def linearize(self, poses) -> dict:
        """{H (6K, 6K), b (6K,), error, status, status_name}: e(xi) ~ error + 2 b^T xi + xi^T H xi along X_k Exp(xi_k)"""
        return linearize_plane_evm([self], [poses], ctx=self.ctx)[0]

    def error(self, poses) -> float:
        e = np.zeros(1)
        arr = (C.c_void_p * 1)(self.h)
        check(lib().gb_plane_evm_error(self.ctx.h, 1, C.cast(arr, C.c_void_p), ptr(pose16(self.key_poses(poses))), ptr(e)))
        return float(e[0])


def linearize_plane_evm(factors: list[PlaneEVMFactorGPU], poses_per_factor, ctx: Context | None = None) -> list[dict]:
    """Linearize many PlaneEVMFactorGPU in one call (gb_plane_evm_linearize: one upload, one launch, one download)."""
    F = len(factors)
    ctx = ctx or (factors[0].ctx if F else default_context())
    X = [f.key_poses(p) for f, p in zip(factors, poses_per_factor)]
    Ks = [len(f.keys) for f in factors]
    T = pose16(np.concatenate(X)) if F else np.zeros((0, 16))
    H = np.zeros(sum(36 * k * k for k in Ks))
    b = np.zeros(sum(6 * k for k in Ks))
    e = np.zeros(F)
    s = np.zeros(F, np.int32)
    arr = (C.c_void_p * max(F, 1))(*[f.h for f in factors])
    check(lib().gb_plane_evm_linearize(ctx.h, F, C.cast(arr, C.c_void_p), ptr(T), ptr(H), ptr(b), ptr(e), ptr(s)))
    out, h0, b0 = [], 0, 0
    for f, K in enumerate(Ks):
        n6 = 6 * K
        out.append({"H": H[h0:h0 + n6 * n6].reshape(n6, n6).T.copy(), "b": b[b0:b0 + n6].copy(), "error": float(e[f]), "status": int(s[f]),
                    "status_name": capi.PLANE_EVM_STATUS_NAMES.get(int(s[f]), "?")})
        h0 += n6 * n6
        b0 += n6
    return out
