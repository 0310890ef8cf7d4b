"""numpy / scipy restatement of the map segmentation rules of include/glim_b200.h (gb_concat_frames, gb_region_growing).

numpy float32 operations round each operation and never fuse, which is the uncontracted fp32 rule of the device; float64
likewise for the fp64 parts.  Candidate pairs come from scipy's cKDTree at a slightly inflated fp64 radius and are then
filtered by the exact fp32 point_d2, so the sets are the brute-force ones."""
import math

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components
from scipy.spatial import cKDTree

F32, F64 = np.float32, np.float64
KEY_HALF = 1 << 20


def point_d2(p, q):
    """fp32 (ex^2 + ey^2) + ez^2 with e = p - q, rounded per operation"""
    e = np.asarray(p, F32) - np.asarray(q, F32)
    return (e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2]


def finite(xyz):
    return np.isfinite(xyz).all(axis=-1)


def keyed(xyz, cell):
    """the 21-bit key rule of a grid at fp64 cell size `cell`: finite, and floor(x * (float)(1 / cell)) (fp32) in [-2^20, 2^20)"""
    xyz = np.asarray(xyz, F32)
    inv = F32(1.0 / cell)
    with np.errstate(invalid="ignore", over="ignore"):
        k = np.floor(xyz * inv)
        ok = ((k >= -KEY_HALF) & (k < KEY_HALF)).all(axis=-1)
    return finite(xyz) & ok


def normals_join(a, b, cos_t):
    """(a_x b_x + a_y b_y) + a_z b_z in fp64 from fp32 normals, >= cos_t (NaN never)"""
    a, b = np.asarray(a, F32).astype(F64), np.asarray(b, F32).astype(F64)
    with np.errstate(invalid="ignore"):
        d = (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]
        return d >= cos_t


def pairs_within(xyz, idx_a, idx_b, max_d2):
    """every (i in idx_a, j in idx_b) with point_d2(i, j) < max_d2 (fp32), as two index arrays"""
    if len(idx_a) == 0 or len(idx_b) == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    r = math.sqrt(float(max_d2)) * (1 + 1e-5)
    P = np.asarray(xyz, F32).astype(F64)
    ta, tb = cKDTree(P[idx_a]), cKDTree(P[idx_b])
    m = ta.sparse_distance_matrix(tb, r, output_type="coo_matrix")
    i, j = idx_a[m.row], idx_b[m.col]
    ok = point_d2(xyz[i], xyz[j]) < max_d2
    return i[ok], j[ok]


def edges(xyz, nrm, distance_threshold, angle_threshold):
    """the joins (i < j) of gb_region_growing"""
    xyz = np.asarray(xyz, F32)
    max_d2 = F32(distance_threshold * distance_threshold)
    idx = np.flatnonzero(keyed(xyz, 1.05 * distance_threshold))
    if len(idx) == 0:
        return np.zeros((0, 2), np.int64)
    r = math.sqrt(float(max_d2)) * (1 + 1e-5)
    pr = cKDTree(xyz[idx].astype(F64)).query_pairs(r, output_type="ndarray")
    i, j = idx[pr[:, 0]], idx[pr[:, 1]]
    ok = (point_d2(xyz[i], xyz[j]) < max_d2) & normals_join(nrm[i], nrm[j], math.cos(angle_threshold))
    e = np.stack([np.minimum(i, j), np.maximum(i, j)], axis=1)[ok]
    return e


def component_labels(n, e, fin):
    """the smallest original index of each point's component; -1 for the points where fin is false"""
    if n == 0:
        return np.zeros(0, np.int64)
    g = coo_matrix((np.ones(len(e), np.int8), (e[:, 0], e[:, 1])), shape=(n, n))
    _, comp = connected_components(g, directed=False)
    low = np.full(comp.max() + 1, n, np.int64)
    np.minimum.at(low, comp, np.arange(n))
    lab = low[comp]
    lab[~fin] = -1
    return lab


def seed_of(xyz, seed_point):
    """the finite point with the smallest fp32 point_d2 to (float)seed_point, ties to the smaller index; -1 for none"""
    fin = finite(np.asarray(xyz, F32))
    if not fin.any():
        return -1
    with np.errstate(over="ignore"):
        d2 = point_d2(xyz, np.asarray(seed_point, F64).astype(F32))
    d2 = np.where(fin, d2, np.inf).astype(F64)
    cand = np.flatnonzero(fin)
    return int(cand[np.argmin(d2[cand])])


def region_growing(xyz, nrm, seed_point, distance_threshold, angle_threshold, dilation_radius=0.0):
    """-> dict(seed, status, num_region, num_selected, num_components, selected, labels) by the rule of gb_region_growing"""
    xyz, nrm = np.asarray(xyz, F32), np.asarray(nrm, F32)
    n = len(xyz)
    fin = finite(xyz)
    lab = component_labels(n, edges(xyz, nrm, distance_threshold, angle_threshold), fin)
    seed = seed_of(xyz, seed_point)
    R = (lab == lab[seed]) & (lab >= 0) if seed >= 0 else np.zeros(n, bool)
    sel = R.copy()
    if dilation_radius > 0 and R.any():
        cell = 1.05 * dilation_radius
        k = keyed(xyz, cell)
        i, j = pairs_within(xyz, np.flatnonzero(R & k), np.flatnonzero(~R & k), F32(dilation_radius * dilation_radius))
        sel[j] = True
    return {"seed": seed, "status": 0 if seed >= 0 else 1, "num_region": int(R.sum()), "num_selected": int(sel.sum()),
            "num_components": int(len(np.unique(lab[lab >= 0]))), "selected": np.flatnonzero(sel).astype(np.int32), "labels": lab.astype(np.int32)}


def transform_points(T, a):
    """q = R a + t in gb_transform_frames' order: ((T_r0 x + T_r1 y) + T_r2 z) + T_r3, fp64 from fp32 a"""
    a = np.asarray(a, F32).astype(F64)
    T = np.asarray(T, F64)
    return np.stack([((T[r, 0] * a[:, 0] + T[r, 1] * a[:, 1]) + T[r, 2] * a[:, 2]) + T[r, 3] for r in range(3)], axis=1)


def transform_covs(T, cov6):
    """R C R^T in gb_transform_frames' order, upper triangle (c00 c01 c02 c11 c12 c22), fp64 from the fp32 entries"""
    c = np.asarray(cov6, F32).astype(F64)
    C = [[c[:, 0], c[:, 1], c[:, 2]], [c[:, 1], c[:, 3], c[:, 4]], [c[:, 2], c[:, 4], c[:, 5]]]
    T = np.asarray(T, F64)
    RC = [[(T[r, 0] * C[0][k] + T[r, 1] * C[1][k]) + T[r, 2] * C[2][k] for k in range(3)] for r in range(3)]
    return np.stack([(RC[r][0] * T[k, 0] + RC[r][1] * T[k, 1]) + RC[r][2] * T[k, 2] for r in range(3) for k in range(r, 3)], axis=1)


def rotate_normals(T, nrm):
    """n' = R n, row r as (R_r0 nx + R_r1 ny) + R_r2 nz in fp64 from the fp32 normals"""
    v = np.asarray(nrm, F32).astype(F64)
    T = np.asarray(T, F64)
    return np.stack([(T[r, 0] * v[:, 0] + T[r, 1] * v[:, 1]) + T[r, 2] * v[:, 2] for r in range(3)], axis=1)


def in_window(q, cell_size, lo, hi):
    """floor(q * (1.0 / cell_size)) in [lo, hi] per axis (fp64); never for a non-finite q"""
    with np.errstate(invalid="ignore", over="ignore"):
        k = np.floor(q * (1.0 / cell_size))
        ok = (k >= np.asarray(lo, F64)) & (k <= np.asarray(hi, F64))
    return np.isfinite(q).all(axis=1) & ok.all(axis=1)


def concat_frames(poses, frames, window=None):
    """frames: list of (xyz fp32 (n,3), cov6 fp32 (n,6) or None, normals fp32 (n,3) or None) -> dict(xyz, cov6 or None,
    normals or None, ids) by the rule of gb_concat_frames (fp32 outputs)"""
    covs = len(frames) > 0 and all(f[1] is not None for f in frames)
    nrms = len(frames) > 0 and all(f[2] is not None for f in frames)
    xs, cs, ns, ids = [], [], [], []
    for k, (T, (xyz, cov6, nrm)) in enumerate(zip(poses, frames)):
        q = transform_points(T, xyz)
        keep = np.ones(len(q), bool) if window is None else in_window(q, *window)
        xs.append(q[keep].astype(F32))
        if covs:
            cs.append(transform_covs(T, cov6)[keep].astype(F32))
        if nrms:
            ns.append(rotate_normals(T, nrm)[keep].astype(F32))
        ids.append((np.uint64(k) << np.uint64(32)) | np.flatnonzero(keep).astype(np.uint64))
    cat = lambda a, w: np.concatenate(a) if a else np.zeros((0, w), F32)
    return {"xyz": cat(xs, 3), "cov6": cat(cs, 6) if covs else None, "normals": cat(ns, 3) if nrms else None,
            "ids": np.concatenate(ids) if ids else np.zeros(0, np.uint64)}
