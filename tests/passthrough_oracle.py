"""numpy restatement of GLIM's passthrough sub-mapping over a device iVox, written from include/glim_b200.h (gb_ivox_extract) and
the reference source (src/glim/mapping/sub_mapping_passthrough.cpp), independently of glim_b200/sub_mapping_passthrough.py:

  * extract: the extraction rule, over the map state of tests/ivox_oracle.IVox (map order = ascending key, slot order), the fp64
    transform of tests/voxelmap_oracle.transform and the hash of voxelmap_oracle.rg_hash;
  * run: the module's decisions over a list of frames (keyframe test, the three cut criteria, centre frame, poses, seeds), with
    the map an ivox_oracle.IVox, returning each submap with the criterion that cut it."""
import math

import numpy as np

from tests import ivox_oracle
from tests import voxelmap_oracle as vo

INT_MAX = 2**31 - 1


def thin_count(P, target):
    """m of the rule: P unless target > 0 and P > target, else (size_t)((double)P * ((double)target / (double)P))"""
    if target > 0 and P > target:
        return int(float(P) * (float(target) / float(P)))
    return P


def extract(xyz, cov6, T, target, seed):
    """(q, C' upper 6) fp64 of the kept points in map order, from the map's fp32 points in map order"""
    P = len(xyz)
    q, c6 = vo.transform(np.eye(4) if T is None else T, xyz, cov6)
    m = thin_count(P, target)
    if m == P:
        return q, c6
    keep = np.zeros(P, bool)
    keep[np.argsort(vo.rg_hash(seed, np.arange(P)), kind="stable")[:m]] = True
    return q[keep], c6[keep]


def extract_ivox(ivox, T, target, seed):
    return extract(ivox.xyz, ivox.cov6, T, target, seed)


def cov4x4(c6):
    """(n, 6) upper triangle -> (n, 4, 4) symmetric, zero last row / column (an upload's covariances)"""
    n = len(c6)
    C = np.zeros((n, 4, 4))
    for e, (r, c) in enumerate([(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]):
        C[:, r, c] = c6[:, e]
        C[:, c, r] = c6[:, e]
    return C


# ---------------------------------------------------------------------------------------------------------------------
# the module
# ---------------------------------------------------------------------------------------------------------------------
def iso_inv(T):
    """[R^T | -(R^T t)], R^T t row by row as (R_0r t_0 + R_1r t_1) + R_2r t_2"""
    out = np.eye(4)
    out[:3, :3] = T[:3, :3].T
    for r in range(3):
        out[r, 3] = -((T[0, r] * T[0, 3] + T[1, r] * T[1, 3]) + T[2, r] * T[2, 3])
    return out


def iso_mul(A, B):
    """A * B for isometries: each entry a sum over k = 0, 1, 2 in order, A's translation added last"""
    out = np.eye(4)
    out[:3, :] = [[(A[r, 0] * B[0, c] + A[r, 1] * B[1, c]) + A[r, 2] * B[2, c] + (A[r, 3] if c == 3 else 0.0) for c in range(4)] for r in range(3)]
    return out


def angle(R):
    """Eigen::AngleAxisd(R).angle() through Eigen's matrix-to-quaternion rule"""
    tr = (R[0, 0] + R[1, 1]) + R[2, 2]
    v = np.zeros(3)
    if tr > 0:
        s = math.sqrt(tr + 1.0)
        w, s = 0.5 * s, 0.5 / s
        v[:] = [(R[2, 1] - R[1, 2]) * s, (R[0, 2] - R[2, 0]) * s, (R[1, 0] - R[0, 1]) * s]
    else:
        i = int(R[1, 1] > R[0, 0])
        i = 2 if R[2, 2] > R[i, i] else i
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(((R[i, i] - R[j, j]) - R[k, k]) + 1.0)
        v[i], s = 0.5 * s, 0.5 / s
        w = (R[k, j] - R[j, k]) * s
        v[j] = (R[j, i] + R[i, j]) * s
        v[k] = (R[k, i] + R[i, k]) * s
    n = math.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])
    return 0.0 if n == 0.0 else 2.0 * math.atan2(n, abs(w))


def new_map(params):
    return ivox_oracle.IVox(params.submap_voxel_resolution, params.min_dist_in_voxel, min(params.max_num_points_in_voxel, 64), 1, 0, INT_MAX)


def run(params, frames, end_of_sequence=True):
    """frames: [(frame id, xyz (n,3) f32, cov6 (n,6) f32, T_world_sensor 4x4)] -> submaps, each a dict with id, the poses, the
    frame and keyframe ids, seed, P (points in the map), max_cell (the most points a cell holds), the extracted fp64 (q, c6), `reason` ("keyframes", "voxels",
    "adaptive" or "end") and `after` (the index in `frames` of the frame whose insertion cut it; len(frames) at the end)."""
    out = []
    count = 0
    odom, keys, hist = [], [], []
    ivox = new_map(params)

    def cut(reason, after):
        c = len(odom) // 2
        T_wo = odom[c][1]
        T_ow = iso_inv(T_wo)
        P = ivox.num_points
        seed = (count * 643145 + P * 4312) % 2**64
        q, c6 = extract_ivox(ivox, T_ow, params.submap_target_num_points, seed)
        return {"id": count, "T_world_origin": T_wo, "T_origin_endpoint_L": iso_mul(T_ow, odom[0][1]), "T_origin_endpoint_R": iso_mul(T_ow, odom[-1][1]),
                "odom_frame_ids": [f for f, _ in odom], "keyframe_ids": [f for f, _ in keys], "seed": seed, "P": P, "num_voxels": ivox.num_voxels,
                "max_cell": int(ivox.counts.max()) if ivox.num_voxels else 0, "q": q, "c6": c6, "reason": reason, "after": after, "center": c}

    for idx, (fid, xyz, cov6, T) in enumerate(frames):
        T = np.asarray(T, dtype=np.float64)
        odom.append((fid, T))
        is_key = True
        if keys:
            D = iso_mul(iso_inv(keys[-1][1]), T)
            t = D[:3, 3]
            is_key = math.sqrt((t[0] * t[0] + t[1] * t[1]) + t[2] * t[2]) > params.keyframe_update_interval_trans or angle(D[:3, :3]) > params.keyframe_update_interval_rot
        if is_key:
            keys.append((fid, T))
            ivox.insert(xyz, cov6, T)
            hist.append(ivox.num_voxels)
        nv = ivox.num_voxels
        reason = None
        if len(keys) >= params.max_num_keyframes:
            reason = "keyframes"
        elif nv >= params.max_num_voxels:
            reason = "voxels"
        elif len(hist) >= 3 and not nv < hist[2] * params.adaptive_max_num_voxels:
            reason = "adaptive"
        if reason:
            out.append(cut(reason, idx))
            count += 1
            odom, keys, hist = [], [], []
            ivox = new_map(params)
    if end_of_sequence and odom:
        out.append(cut("end", len(frames)))
    return out
