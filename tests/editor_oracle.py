"""numpy restatement of the map editor's selection tools and point removal (gb_select_gizmo, gb_select_radius,
gb_remove_points; the rules of include/glim_b200.h), with scipy's cKDTree for the k-NN.  Every fp64 expression is written in
the header's association order; numpy's elementwise operations round each one."""
import numpy as np
from scipy.spatial import cKDTree

from tests import segment_oracle as so

F32, F64 = np.float32, np.float64


def compose(A, B):
    """M = A B of two 4x4 affine matrices: (A_r0 B_0c + A_r1 B_1c) + A_r2 B_2c, plus A_r3 in the translation column"""
    A, B = np.asarray(A, F64), np.asarray(B, F64)
    M = np.zeros((4, 4))
    for r in range(3):
        for c in range(4):
            s = (A[r, 0] * B[0, c] + A[r, 1] * B[1, c]) + A[r, 2] * B[2, c]
            M[r, c] = s + A[r, 3] if c == 3 else s
    M[3, 3] = 1.0
    return M


def in_box(q):
    q = np.asarray(q, F64)
    with np.errstate(invalid="ignore"):
        return np.all((q > -0.5) & (q < 0.5), axis=1)


def in_sphere(q, r2=1.0):
    q = np.asarray(q, F64)
    with np.errstate(invalid="ignore"):
        return ((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]) < r2


def select_gizmo(poses, frames_xyz, T_local_world, shape="box"):
    """ids (uint64) of the points of frames_xyz (K arrays (n_k, 3) fp32, local frames) inside the gizmo"""
    out = []
    for k, (T, a) in enumerate(zip(poses, frames_xyz)):
        if len(a) == 0:
            continue
        q = so.transform_points(compose(T_local_world, T), a)
        inside = in_box(q) if shape == "box" else in_sphere(q, 1.0)
        out.append((np.uint64(k) << np.uint64(32)) | np.flatnonzero(inside).astype(np.uint64))
    return np.concatenate(out) if out else np.zeros(0, np.uint64)


def d2(xyz, c):
    """fp64 (dx^2 + dy^2) + dz^2 of the widened fp32 points to c"""
    p = np.asarray(xyz, F32).astype(F64)
    dx, dy, dz = p[:, 0] - c[0], p[:, 1] - c[1], p[:, 2] - c[2]
    return (dx * dx + dy * dy) + dz * dz


def radius_flags(xyz, c, inner2, outer2):
    """(inside, participant) boolean arrays"""
    fin = np.all(np.isfinite(np.asarray(xyz, F32)), axis=1)
    with np.errstate(invalid="ignore"):
        e = d2(xyz, c)
        return fin & (e < inner2), fin & (e < outer2)


def threshold(S, S2, m, stddev_thresh):
    mean = S / m
    var = S2 / m - mean * mean
    return mean + stddev_thresh * np.sqrt(max(var, 0.0))


def mean_knn_dists(P, k):
    """d_i over the rows of fp64 points P (m, 3): the k nearest by exact fp64 d2, ties to the smaller index, the query included,
    their distances summed nearest first, over k"""
    m = len(P)
    kk = min(m, k + 8)
    _, idx = cKDTree(P).query(P, k=kk)
    idx = np.asarray(idx).reshape(m, kk)
    d = np.empty(m)
    for i in range(m):
        cand = np.unique(idx[i])
        e = P[cand] - P[i]
        dd = (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]
        order = np.lexsort((cand, dd))[:k]
        s = 0.0
        for v in np.sqrt(dd[order]):
            s = s + v
        d[i] = s / k
    return d


def select_radius(xyz, center, mode="inside", radius=2.0, radius_offset=1.0, k=10, stddev_thresh=2.0):
    """-> dict(status, num_participants, selected, threshold, d, nodes): the selection in ascending original index; for
    OUTLIERS also the participants' d_i and their original indices"""
    c = np.asarray(center, F64)
    inside, part = radius_flags(xyz, c, radius * radius, (radius + radius_offset) ** 2)
    if mode == "inside":
        return {"status": 0, "num_participants": 0, "selected": np.flatnonzero(inside).astype(np.int32), "threshold": np.nan}
    nodes = np.flatnonzero(part)
    m = len(nodes)
    if m < k:
        return {"status": 1, "num_participants": m, "selected": np.zeros(0, np.int32), "threshold": np.nan}
    P = np.asarray(xyz, F32)[nodes].astype(F64)
    d = mean_knn_dists(P, k)
    th = threshold(float(np.sum(d)), float(np.sum(d * d)), m, stddev_thresh)
    sel = inside[nodes] & ~(d < th)
    return {"status": 0, "num_participants": m, "selected": nodes[sel].astype(np.int32), "threshold": th, "d": d, "nodes": nodes}


def remove_points(sizes, ids):
    """-> (per-frame sorted survivor indices or None for an unchanged frame, num_removed, num_ignored)"""
    ids = np.asarray(ids, np.uint64).reshape(-1)
    f, i = (ids >> np.uint64(32)).astype(np.int64), (ids & np.uint64(0xFFFFFFFF)).astype(np.int64)
    K = len(sizes)
    ok = (f < K) & (i < np.asarray(list(sizes) + [0], np.int64)[np.minimum(f, K)])
    out, removed = [], 0
    for k in range(K):
        gone = np.unique(i[ok & (f == k)])
        removed += len(gone)
        out.append(np.setdiff1d(np.arange(sizes[k]), gone) if len(gone) else None)
    return out, removed, int((~ok).sum())
