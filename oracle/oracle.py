"""ctypes wrapper around oracle/libglim_oracle.so (the CPU oracle, see glim_oracle.c).

TEST INFRASTRUCTURE ONLY -- parity unpinned (see the header of glim_oracle.c).  Only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this module;
nothing under glim_b200/ does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libglim_oracle.so")


def build(force=False):
    src = os.path.join(_HERE, "glim_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        vp, i32, f32, f64 = C.c_void_p, C.c_int, C.c_float, C.c_double
        L.go_voxel_hash.restype = C.c_uint64
        L.go_voxel_hash.argtypes = [i32, i32, i32]
        L.go_gpumap_build.restype = vp
        L.go_gpumap_build.argtypes = [i32, vp, vp, f32, i32, i32, f64]
        L.go_gpumap_free.argtypes = [vp]
        L.go_gpumap_info.argtypes = [vp, vp, vp, vp]
        L.go_gpumap_get.argtypes = [vp, vp, vp, vp, vp, vp]
        L.go_gpumap_correspondences.argtypes = [vp, i32, vp, vp, vp]
        L.go_vgicp_linearize_gpumap.argtypes = [vp, i32, vp, vp, vp, i32, vp, vp]
        L.go_vgicp_linearize_gpumap_sv.argtypes = [vp, i32, vp, vp, vp, vp, i32, vp, vp]
        L.go_vgicp_error_gpumap.restype = f64
        L.go_vgicp_error_gpumap.argtypes = [vp, i32, vp, vp, vp, vp]
        L.go_vgicp_error_gpumap_sv.restype = f64
        L.go_vgicp_error_gpumap_sv.argtypes = [vp, i32, vp, vp, vp, vp, vp]
        L.go_overlap_gpumap.restype = f64
        L.go_overlap_gpumap.argtypes = [i32, vp, i32, vp, vp]
        L.go_pack_cloud_f32.argtypes = [i32, vp, vp, vp, vp]
        L.go_cpumap_create.restype = vp
        L.go_cpumap_create.argtypes = [f64]
        L.go_cpumap_free.argtypes = [vp]
        L.go_cpumap_insert.argtypes = [vp, i32, vp, vp]
        L.go_cpumap_set_lru.argtypes = [vp, i32, i32]
        L.go_cpumap_num_voxels.restype = i32
        L.go_cpumap_num_voxels.argtypes = [vp]
        L.go_cpumap_lookup.restype = i32
        L.go_cpumap_lookup.argtypes = [vp, vp, vp, vp]
        L.go_cpu_cache_create.restype = vp
        L.go_cpu_cache_create.argtypes = [i32]
        L.go_cpu_cache_free.argtypes = [vp]
        L.go_vgicp_cpu_update_correspondences.argtypes = [vp, i32, vp, vp, vp, i32, vp]
        L.go_vgicp_cpu_evaluate.argtypes = [vp, i32, vp, vp, i32, i32, vp, vp]
        L.go_vgicp_cpu_linearize.argtypes = [vp, i32, vp, vp, vp, i32, vp, vp]
        L.go_eigen_sym3_direct.argtypes = [vp, vp, vp]
        L.go_covariance_estimate.argtypes = [i32, vp, vp, i32, i32, i32, vp, vp]
        L.go_knn_bruteforce.argtypes = [i32, vp, i32, i32, vp, vp]
        L.go_voxelgrid_sampling.restype = i32
        L.go_voxelgrid_sampling.argtypes = [i32, vp, vp, vp, f64, vp, vp, vp]
        L.go_merge_frames.restype = i32
        L.go_merge_frames.argtypes = [i32, vp, vp, vp, vp, f64, i32, C.c_uint64, vp, vp]
        L.go_randomgrid_sampling.restype = i32
        L.go_randomgrid_sampling.argtypes = [i32, vp, f64, f64, C.c_uint64, vp]
        L.go_deskew_const_vel.restype = i32
        L.go_deskew_const_vel.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp]
        L.go_deskew_imu.restype = i32
        L.go_deskew_imu.argtypes = [vp, i32, vp, vp, f64, i32, vp, vp, vp, vp]
        L.go_num_threads.restype = i32
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def pose_colmajor(T):
    """4x4 numpy pose -> 16 doubles column-major (the C-ABI / Eigen layout)."""
    return np.ascontiguousarray(np.asarray(T, dtype=np.float64).T).reshape(16)


def split122(o):
    """122-double linearized6 record -> dict of column-major 6x6 blocks as numpy [row, col]."""
    o = np.asarray(o, dtype=np.float64)
    return {
        "H_tt": o[0:36].reshape(6, 6).T.copy(),
        "H_ss": o[36:72].reshape(6, 6).T.copy(),
        "H_ts": o[72:108].reshape(6, 6).T.copy(),
        "b_t": o[108:114].copy(),
        "b_s": o[114:120].copy(),
        "error": float(o[120]),
        "num_inliers": float(o[121]),
    }


def num_threads():
    return lib().go_num_threads()


def pack_cloud(pts4, cov16=None):
    """PointCloudGPU::clone's host cast: fp64 Vector4d/Matrix4d -> fp32 xyz (N,3) + cov6 (N,6)."""
    pts4 = _f64(pts4)
    n = pts4.shape[0]
    xyz = np.empty((n, 3), np.float32)
    cov6 = None
    c16 = None
    if cov16 is not None:
        c16 = _f64(cov16).reshape(n, 16)
        cov6 = np.empty((n, 6), np.float32)
    lib().go_pack_cloud_f32(n, _p(pts4), _p(c16), _p(xyz), _p(cov6))
    return xyz, cov6


class GpuMap:
    """Deterministic restatement of gtsam_points::GaussianVoxelMapGPU (fp32, open addressing)."""

    def __init__(self, xyz, cov6, resolution, init_buckets=8192 * 2, max_scan=10, drop_rate=1e-3):
        self.xyz = _f32(xyz)
        self.cov6 = _f32(cov6)
        n = self.xyz.shape[0]
        self.h = lib().go_gpumap_build(n, _p(self.xyz), _p(self.cov6), float(resolution), init_buckets, max_scan, drop_rate)
        nv, nb, nd = C.c_int(), C.c_int(), C.c_int()
        lib().go_gpumap_info(self.h, C.byref(nv), C.byref(nb), C.byref(nd))
        self.num_voxels, self.num_buckets, self.num_dropped_points = nv.value, nb.value, nd.value
        self.resolution = float(np.float32(resolution))
        self.buckets = np.empty((self.num_buckets, 4), np.int32)
        self.vcoord = np.empty((self.num_voxels, 3), np.int32)
        self.vnum = np.empty((self.num_voxels,), np.int32)
        self.vmean = np.empty((self.num_voxels, 3), np.float32)
        self.vcov = np.empty((self.num_voxels, 6), np.float32)
        lib().go_gpumap_get(self.h, _p(self.buckets), _p(self.vcoord), _p(self.vnum), _p(self.vmean), _p(self.vcov))

    def __del__(self):
        if getattr(self, "h", None):
            lib().go_gpumap_free(self.h)
            self.h = None

    def correspondences(self, xyz, T):
        xyz = _f32(xyz)
        corr = np.empty((xyz.shape[0],), np.int32)
        Tc = pose_colmajor(T)
        lib().go_gpumap_correspondences(self.h, xyz.shape[0], _p(xyz), _p(Tc), _p(corr))
        return corr


def linearize_gpumap(m, xyz, cov6, T, with_derivs=True, normals=None):
    """normals: (n,3|4) source normals -> surface validation on (corr == -2 marks correspondences the gate rejected)."""
    xyz, cov6 = _f32(xyz), _f32(cov6)
    out = np.zeros(122)
    corr = np.empty((xyz.shape[0],), np.int32)
    Tc = pose_colmajor(T)
    nr = _f32(np.asarray(normals)[:, :3]) if normals is not None else None
    lib().go_vgicp_linearize_gpumap_sv(m.h, xyz.shape[0], _p(xyz), _p(cov6), _p(nr), _p(Tc), int(with_derivs), _p(out), _p(corr))
    return out, corr


def error_gpumap(m, xyz, cov6, T_lin, T_eval, normals=None):
    """error at T_eval with the correspondences of T_lin.  normals: (n,3|4) source normals -> surface validation on, the gate
    deciding at T_lin (where the correspondences are found)."""
    xyz, cov6 = _f32(xyz), _f32(cov6)
    nr = _f32(np.asarray(normals)[:, :3]) if normals is not None else None
    return lib().go_vgicp_error_gpumap_sv(m.h, xyz.shape[0], _p(xyz), _p(cov6), _p(nr), _p(pose_colmajor(T_lin)), _p(pose_colmajor(T_eval)))


def overlap_gpumap(maps, xyz, Ts):
    xyz = _f32(xyz)
    arr = (C.c_void_p * len(maps))(*[m.h for m in maps])
    Tc = np.concatenate([pose_colmajor(T) for T in Ts]) if len(maps) else np.zeros(0)
    return lib().go_overlap_gpumap(len(maps), C.cast(arr, C.c_void_p), xyz.shape[0], _p(xyz), _p(Tc))


class CpuMap:
    """Restatement of gtsam_points::GaussianVoxelMapCPU (fp64, node-based hash map)."""

    def __init__(self, resolution):
        self.h = lib().go_cpumap_create(float(resolution))
        self.resolution = float(resolution)

    def __del__(self):
        if getattr(self, "h", None):
            lib().go_cpumap_free(self.h)
            self.h = None

    def set_lru_horizon(self, horizon, clear_cycle=10):
        """GaussianVoxelMapCPU::set_lru_horizon (odometry_estimation_cpu.cpp:67)."""
        lib().go_cpumap_set_lru(self.h, int(horizon), int(clear_cycle))

    def insert(self, pts4, cov16):
        pts4 = _f64(pts4)
        cov16 = _f64(cov16).reshape(pts4.shape[0], 16)
        lib().go_cpumap_insert(self.h, pts4.shape[0], _p(pts4), _p(cov16))

    @property
    def num_voxels(self):
        return lib().go_cpumap_num_voxels(self.h)

    def lookup(self, p3):
        p3 = _f64(p3)
        mean = np.zeros(4)
        cov = np.zeros(16)
        j = lib().go_cpumap_lookup(self.h, _p(p3), _p(mean), _p(cov))
        return j, mean, cov.reshape(4, 4).T


class CpuFactor:
    """Restatement of gtsam_points::IntegratedVGICPFactor (CPU fp64, two-phase linearize)."""

    def __init__(self, cpumap, pts4, cov16, num_threads=1):
        self.m = cpumap
        self.pts4 = _f64(pts4)
        self.cov16 = _f64(cov16).reshape(self.pts4.shape[0], 16)
        self.n = self.pts4.shape[0]
        self.num_threads = num_threads
        self.cache = lib().go_cpu_cache_create(self.n)

    def __del__(self):
        if getattr(self, "cache", None):
            lib().go_cpu_cache_free(self.cache)
            self.cache = None

    def linearize(self, T):
        out = np.zeros(122)
        lib().go_vgicp_cpu_linearize(self.m.h, self.n, _p(self.pts4), _p(self.cov16), _p(pose_colmajor(T)), self.num_threads, self.cache, _p(out))
        return out

    def linearize_raw(self, Tc, out):
        """No-allocation variant for timing: Tc = 16 doubles column-major, out = 122 doubles."""
        lib().go_vgicp_cpu_linearize(self.m.h, self.n, _p(self.pts4), _p(self.cov16), _p(Tc), self.num_threads, self.cache, _p(out))

    def error(self, T_eval):
        """error() at a trial pose re-uses correspondences and Mahalanobis from the last linearize."""
        out = np.zeros(122)
        lib().go_vgicp_cpu_evaluate(self.m.h, self.n, _p(self.pts4), _p(pose_colmajor(T_eval)), 0, self.num_threads, self.cache, _p(out))
        return float(out[120])


def eigen_sym3(A):
    A = _f64(A).reshape(9)
    ev = np.zeros(3)
    V = np.zeros(9)
    lib().go_eigen_sym3_direct(_p(A), _p(ev), _p(V))
    return ev, V.reshape(3, 3)


def covariance_estimate(pts4, neighbors, k_neighbors=None, num_threads=1):
    pts4 = _f64(pts4)
    n = pts4.shape[0]
    neighbors = np.ascontiguousarray(neighbors, dtype=np.int32).reshape(n, -1) if n else np.zeros((0, 1), np.int32)
    kc = neighbors.shape[1]
    k = kc if k_neighbors is None else k_neighbors
    normals = np.zeros((n, 4))
    covs = np.zeros((n, 16))
    lib().go_covariance_estimate(n, _p(pts4), _p(neighbors), kc, k, num_threads, _p(normals), _p(covs))
    return normals, covs.reshape(n, 4, 4).transpose(0, 2, 1).copy()  # -> [i, row, col]


def knn_bruteforce(pts4, k, num_threads=0):
    pts4 = _f64(pts4)
    n = pts4.shape[0]
    nb = np.empty((n, k), np.int32)
    d = np.empty((n, k))
    lib().go_knn_bruteforce(n, _p(pts4), k, num_threads or num_threads or lib().go_num_threads(), _p(nb), _p(d))
    return nb, d


def voxelgrid_sampling(pts4, resolution, times=None, intensities=None):
    pts4 = _f64(pts4)
    n = pts4.shape[0]
    t = _f64(times) if times is not None else None
    it = _f64(intensities) if intensities is not None else None
    op = np.empty((n, 4))
    ot = np.empty((n,)) if t is not None else None
    oi = np.empty((n,)) if it is not None else None
    m = lib().go_voxelgrid_sampling(n, _p(pts4), _p(t), _p(it), float(resolution), _p(op), _p(ot), _p(oi))
    return op[:m].copy(), (ot[:m].copy() if ot is not None else None), (oi[:m].copy() if oi is not None else None)


def merge_frames(poses, clouds, resolution, target=0, seed=0):
    """clouds: list of (xyz f32 (n,3), cov6 f32 (n,6)) device-layout clouds; poses: list of 4x4.  -> points (M,4), covs (M,4,4) [i,row,col]"""
    n = np.array([len(c[0]) for c in clouds], np.int32)
    xyz = _f32(np.concatenate([c[0] for c in clouds]))
    cov6 = _f32(np.concatenate([c[1] for c in clouds]))
    T = np.concatenate([pose_colmajor(p) for p in poses])
    tot = int(n.sum())
    op, oc = np.empty((tot, 4)), np.empty((tot, 16))
    m = lib().go_merge_frames(len(clouds), _p(n), _p(xyz), _p(cov6), _p(T), float(resolution), int(target), int(seed), _p(op), _p(oc))
    return op[:m].copy(), oc[:m].reshape(m, 4, 4).transpose(0, 2, 1).copy()


def randomgrid_sampling(pts4, resolution, rate, seed=0):
    """-> bool mask of the survivors (original order is kept), see go_randomgrid_sampling."""
    pts4 = _f64(pts4)
    keep = np.zeros(pts4.shape[0], np.int32)
    lib().go_randomgrid_sampling(pts4.shape[0], _p(pts4), float(resolution), float(rate), int(seed), _p(keep))
    return keep.astype(bool)


def deskew_const_vel(T_imu_lidar, linear_vel, angular_vel, times, pts4, T_post=None):
    """CloudDeskewing::deskew (constant velocity), src/glim/common/cloud_deskewing.cpp:11-55."""
    pts4, times = _f64(pts4), _f64(times)
    out = np.empty_like(pts4)
    Tp = pose_colmajor(T_post) if T_post is not None else None
    lib().go_deskew_const_vel(_p(pose_colmajor(T_imu_lidar)), _p(_f64(linear_vel)), _p(_f64(angular_vel)), pts4.shape[0], _p(times), _p(pts4), _p(Tp), _p(out))
    return out


def deskew_imu(T_imu_lidar, imu_times, imu_poses, stamp, times, pts4, T_post=None):
    """CloudDeskewing::deskew (predicted IMU poses), src/glim/common/cloud_deskewing.cpp:57-133."""
    pts4, times, imu_times = _f64(pts4), _f64(times), _f64(imu_times)
    poses = np.ascontiguousarray(np.swapaxes(np.asarray(imu_poses, dtype=np.float64).reshape(-1, 4, 4), 1, 2)).reshape(-1, 16)
    out = np.empty_like(pts4)
    Tp = pose_colmajor(T_post) if T_post is not None else None
    lib().go_deskew_imu(_p(pose_colmajor(T_imu_lidar)), len(imu_times), _p(imu_times), _p(poses), float(stamp), pts4.shape[0], _p(times), _p(pts4), _p(Tp), _p(out))
    return out
