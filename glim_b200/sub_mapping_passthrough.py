"""GLIM's passthrough sub-mapping (glim::SubMappingPassthrough, src/glim/mapping/sub_mapping_passthrough.cpp) over a device iVox:
the sub-mapping module of the low-end configuration (config_odometry_cpu, config_sub_mapping_passthrough,
config_global_mapping_pose_graph).  Each keyframe is inserted whole into the iVox at T_world_sensor, the iVox's voxel count
decides where a submap is cut, and the submap's cloud is made on the device by IVoxGPU.voxel_data (gb_ivox_extract): the map's
points posed by T_world_origin^-1 and thinned to submap_target_num_points.  The host logic below mirrors the module statement
for statement; the frames' clouds never leave the device.

Differences from the reference, each recorded in DESIGN.md section 7:
  * which points a submap keeps when it is thinned: the hash pick of gb_ivox_extract in the map's key order, not an
    std::mt19937 draw in voxel_data()'s insertion order (the count is the reference's);
  * the map stores the fp32 rounding of the world-frame points (the reference keeps fp64);
  * the cell capacity is min(max_num_points_in_voxel, 64), the iVox's limit;
  * the map is created without eviction (lru_horizon 0) instead of lru_horizon INT_MAX, which would overflow stamp + horizon on
    the device; with lru_clear_cycle INT_MAX the reference never evicts either.
"""
from __future__ import annotations

import math
import sys
from dataclasses import dataclass, field

import numpy as np

from .gpu import Context, IVoxGPU

INT_MAX = 2**31 - 1
DBL_MAX = sys.float_info.max
IVOX_MAX_POINTS_IN_CELL = 64  # gb_ivox_create's limit


@dataclass
class SubMappingPassthroughParams:
    """SubMappingPassthroughParams (:16-35) with the shipped values of config/config_sub_mapping_passthrough.json, -1 converted
    as the constructor converts it."""

    keyframe_update_interval_rot: float = 0.01
    keyframe_update_interval_trans: float = 0.1
    max_num_keyframes: int = 50
    max_num_voxels: int = INT_MAX  # shipped -1
    adaptive_max_num_voxels: float = 2.5
    submap_target_num_points: int = 50000
    submap_voxel_resolution: float = 0.5
    min_dist_in_voxel: float = 0.2
    max_num_points_in_voxel: int = 100

    @classmethod
    def from_config(cls, sub_mapping: dict) -> "SubMappingPassthroughParams":
        """The constructor's reading of the "sub_mapping" section: its code defaults for missing keys, and a negative
        max_num_keyframes or max_num_voxels as INT_MAX, a negative adaptive_max_num_voxels as DBL_MAX."""
        g = sub_mapping.get
        max_kf = int(g("max_num_keyframes", 50))
        max_nv = int(g("max_num_voxels", 50000))
        adaptive = float(g("adaptive_max_num_voxels", 0.5))
        return cls(keyframe_update_interval_rot=float(g("keyframe_update_interval_rot", 0.01)),
                   keyframe_update_interval_trans=float(g("keyframe_update_interval_trans", 0.1)),
                   max_num_keyframes=INT_MAX if max_kf < 0 else max_kf,
                   max_num_voxels=INT_MAX if max_nv < 0 else max_nv,
                   adaptive_max_num_voxels=DBL_MAX if adaptive < 0 else adaptive,
                   submap_target_num_points=int(g("submap_target_num_points", 40000)),
                   submap_voxel_resolution=float(g("submap_voxel_resolution", 0.5)),
                   min_dist_in_voxel=float(g("min_dist_in_voxel", 0.1)),
                   max_num_points_in_voxel=int(g("max_num_points_in_voxel", 100)))


@dataclass
class SubMap:
    """The fields of glim::SubMap the module fills: id, the three poses (4x4 fp64), the odometry frames' ids (odom_frames and
    frames), the keyframes' ids and the submap's cloud in the origin frame."""

    id: int
    T_world_origin: np.ndarray
    T_origin_endpoint_L: np.ndarray
    T_origin_endpoint_R: np.ndarray
    odom_frame_ids: list
    keyframe_ids: list
    frame: object = field(repr=False)


def inverse(T: np.ndarray) -> np.ndarray:
    """Eigen::Isometry3d::inverse(): [R^T | -(R^T t)], each entry of R^T t as (a x + b y) + c z"""
    R, t = T[:3, :3], T[:3, 3]
    out = np.eye(4)
    out[:3, :3] = R.T
    out[:3, 3] = [-((R[0, r] * t[0] + R[1, r] * t[1]) + R[2, r] * t[2]) for r in range(3)]
    return out


def compose(A: np.ndarray, B: np.ndarray) -> np.ndarray:
    """Isometry3d A * B: R_A R_B and R_A t_B + t_A, each sum over k in ascending order, the translation added last"""
    out = np.eye(4)
    for r in range(3):
        for c in range(3):
            out[r, c] = (A[r, 0] * B[0, c] + A[r, 1] * B[1, c]) + A[r, 2] * B[2, c]
        out[r, 3] = ((A[r, 0] * B[0, 3] + A[r, 1] * B[1, 3]) + A[r, 2] * B[2, 3]) + A[r, 3]
    return out


def rotation_angle(R: np.ndarray) -> float:
    """Eigen::AngleAxisd(R).angle(): R to a quaternion by Eigen's trace / largest-diagonal rule, then 2 atan2(|v|, |w|)"""
    t = (R[0, 0] + R[1, 1]) + R[2, 2]
    q = [0.0, 0.0, 0.0]
    if t > 0:
        s = math.sqrt(t + 1.0)
        w = 0.5 * s
        s = 0.5 / s
        q = [(R[2, 1] - R[1, 2]) * s, (R[0, 2] - R[2, 0]) * s, (R[1, 0] - R[0, 1]) * s]
    else:
        i = 0
        if R[1, 1] > R[0, 0]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(((R[i, i] - R[j, j]) - R[k, k]) + 1.0)
        q[i] = 0.5 * s
        s = 0.5 / s
        w = (R[k, j] - R[j, k]) * s
        q[j] = (R[j, i] + R[i, j]) * s
        q[k] = (R[k, i] + R[i, k]) * s
    n = math.sqrt((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2])
    return 2.0 * math.atan2(n, abs(w)) if n != 0.0 else 0.0


def submap_seed(submap_count: int, num_points: int) -> int:
    """The module's seed submap_count * 643145 + frame->size() * 4312 (:150), as uint64; here it feeds rg_hash"""
    return (submap_count * 643145 + num_points * 4312) % 2**64


class SubMappingPassthroughGPU:
    """glim::SubMappingPassthrough with its map on the device.  insert_frame takes the odometry frame's id, its cloud (a
    PointCloudGPU with covariances, in the sensor frame) and T_world_sensor.  map_factory(resolution, min_dist_in_cell,
    max_points_in_cell, neighbor_voxel_mode, lru_horizon, lru_clear_cycle, ctx=...) makes the map; anything with insert(cloud, T),
    num_voxels, num_points, voxel_data(T_out_map, target_num_points, seed) and close() serves (IVoxGPU by default)."""

    def __init__(self, params: SubMappingPassthroughParams | None = None, ctx: Context | None = None, map_factory=IVoxGPU):
        self.params = params or SubMappingPassthroughParams()
        self.ctx = ctx
        self.map_factory = map_factory
        self.submap_count = 0
        self.odom_frames = []  # (frame id, T_world_sensor)
        self.keyframes = []
        self.num_voxels_history = []
        self.submap_queue = []
        self.voxelmap = self._create_map()

    def _create_map(self):
        p = self.params
        return self.map_factory(p.submap_voxel_resolution, p.min_dist_in_voxel, min(p.max_num_points_in_voxel, IVOX_MAX_POINTS_IN_CELL), 1, 0, INT_MAX, ctx=self.ctx)

    def insert_frame(self, frame_id, cloud, T_world_sensor):
        """:52-94"""
        T = np.array(T_world_sensor, dtype=np.float64).reshape(4, 4)
        self.odom_frames.append((frame_id, T))
        insert_as_keyframe = True
        if self.keyframes:
            T_last_current = compose(inverse(self.keyframes[-1][1]), T)
            t = T_last_current[:3, 3]
            dt = math.sqrt((t[0] * t[0] + t[1] * t[1]) + t[2] * t[2])
            dr = rotation_angle(T_last_current[:3, :3])
            insert_as_keyframe = dt > self.params.keyframe_update_interval_trans or dr > self.params.keyframe_update_interval_rot
        if insert_as_keyframe:
            self.keyframes.append((frame_id, T))
            self.voxelmap.insert(cloud, T)
            self.num_voxels_history.append(self.voxelmap.num_voxels)

        new_submap = self._create_submap()
        if new_submap is not None:
            new_submap.id = self.submap_count
            self.submap_count += 1
            self.submap_queue.append(new_submap)
            self.odom_frames, self.keyframes, self.num_voxels_history = [], [], []
            self.voxelmap.close()  # voxelmap->clear(): a new, empty map
            self.voxelmap = self._create_map()

    def get_submaps(self) -> list:
        """:96-100"""
        submaps, self.submap_queue = self.submap_queue, []
        return submaps

    def submit_end_of_sequence(self) -> list:
        """:102-114"""
        submaps = []
        if self.odom_frames:
            new_submap = self._create_submap(force_create=True)
            if new_submap is not None:
                new_submap.id = self.submap_count
                self.submap_count += 1
                submaps.append(new_submap)
        return submaps

    def _create_submap(self, force_create: bool = False) -> SubMap | None:
        """:116-156"""
        p = self.params
        num_voxels = self.voxelmap.num_voxels

        def check_adaptive_num_voxels():
            if len(self.num_voxels_history) < 3:
                return True
            return num_voxels < self.num_voxels_history[2] * p.adaptive_max_num_voxels

        if not force_create and len(self.keyframes) < p.max_num_keyframes and num_voxels < p.max_num_voxels and check_adaptive_num_voxels():
            return None

        center = len(self.odom_frames) // 2
        T_world_origin = self.odom_frames[center][1]
        T_origin_world = inverse(T_world_origin)
        T_origin_endpoint_L = compose(T_origin_world, self.odom_frames[0][1])
        T_origin_endpoint_R = compose(T_origin_world, self.odom_frames[-1][1])
        seed = submap_seed(self.submap_count, self.voxelmap.num_points)
        frame = self.voxelmap.voxel_data(T_origin_world, p.submap_target_num_points, seed)
        return SubMap(0, T_world_origin, T_origin_endpoint_L, T_origin_endpoint_R, [f for f, _ in self.odom_frames], [f for f, _ in self.keyframes], frame)
