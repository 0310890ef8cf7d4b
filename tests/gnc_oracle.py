"""Numpy restatement of GNC global registration (gb_gnc_align), written from the rule in include/glim_b200.h and independently
of the CUDA: the sample pick (the m smallest rg_hash), the reciprocal pair filter over the exact feature match of
tests/global_oracle.py, the weighted closed-form pose (Horn's estimator here by numpy's symmetric eigensolver) and the
Geman-McClure schedule."""
import math

import numpy as np

from tests.global_oracle import match
from tests.voxelmap_oracle import rg_hash

F32, F64 = np.float32, np.float64
GNC_FOUND, GNC_DEGENERATE = 0, 1
GNC_DIV_FACTOR, GNC_MIN_SCALE, GNC_MAX_SCALE = 1.4, 1.0, 1e3


def gnc_samples(seed, ns, max_init_samples):
    """every source index when ns <= max_init_samples, else the max_init_samples with the smallest rg_hash(seed, i); ascending"""
    if ns <= max_init_samples:
        return np.arange(ns)
    h = rg_hash(seed, np.arange(ns))
    return np.sort(np.argsort(h, kind="stable")[:max_init_samples])


def gnc_pairs(tgt_feat, src_feat, tgt_xyz, src_xyz, seed, max_init_samples):
    """(K, 2) [source index, target index]: the samples whose nearest target feature has them as its nearest source feature
    (over all source features), both positions finite; ascending source index"""
    s = gnc_samples(seed, len(src_feat), max_init_samples)
    src_feat = np.asarray(src_feat, dtype=F32)
    tgt_feat = np.asarray(tgt_feat, dtype=F32)
    j = match(tgt_feat, src_feat[s])
    back = match(src_feat, tgt_feat[np.maximum(j, 0)])
    sx = np.asarray(src_xyz, dtype=F32)[s]
    tx = np.asarray(tgt_xyz, dtype=F32)[np.maximum(j, 0)]
    ok = (j >= 0) & (back == s) & np.isfinite(sx).all(1) & np.isfinite(tx).all(1)
    return np.stack([s[ok], j[ok]], 1)


def gnc_pose(a, b, w, a_shift, b_shift, dof):
    """the weighted closed form about the shifts: T (4,4)"""
    A, B = a - a_shift, b - b_shift
    W = w.sum()
    p, q = (w[:, None] * A).sum(0), (w[:, None] * B).sum(0)
    S = (w[:, None] * A).T @ B - np.outer(p, q) / W
    ca, cb = a_shift + p / W, b_shift + q / W
    if dof == 4:
        yaw = math.atan2(S[0, 1] - S[1, 0], S[0, 0] + S[1, 1])
        R = np.array([[math.cos(yaw), -math.sin(yaw), 0], [math.sin(yaw), math.cos(yaw), 0], [0, 0, 1.0]])
    else:
        (sxx, sxy, sxz), (syx, syy, syz), (szx, szy, szz) = S
        N = np.array([[sxx + syy + szz, syz - szy, szx - sxz, sxy - syx],
                      [syz - szy, sxx - syy - szz, sxy + syx, szx + sxz],
                      [szx - sxz, sxy + syx, -sxx + syy - szz, syz + szy],
                      [sxy - syx, szx + sxz, syz + szy, -sxx - syy + szz]])
        qw, x, y, z = np.linalg.eigh(N)[1][:, -1]
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - qw * z), 2 * (x * z + qw * y)],
                      [2 * (x * y + qw * z), 1 - 2 * (x * x + z * z), 2 * (y * z - qw * x)],
                      [2 * (x * z - qw * y), 2 * (y * z + qw * x), 1 - 2 * (x * x + y * y)]])
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = cb - R @ ca
    return T


def gnc_residual2(T, a, b):
    e = b - (a @ T[:3, :3].T + T[:3, 3])
    return (e * e).sum(1)


def gnc_solve(a, b, dof):
    """the GNC Geman-McClure schedule on pairs (a source, b target; fp32 positions) -> (T (4,4), final weights (K,),
    iterations, status)"""
    a = np.asarray(a, dtype=F32).astype(F64)
    b = np.asarray(b, dtype=F32).astype(F64)
    K = len(a)
    if K < 3:
        return np.eye(4), np.zeros(K), 0, GNC_DEGENERATE
    a_shift, b_shift = a.sum(0) / K, b.sum(0) / K
    T = gnc_pose(a, b, np.ones(K), a_shift, b_shift, dof)
    mu = min(max(float(gnc_residual2(T, a, b).max()), GNC_MIN_SCALE), GNC_MAX_SCALE)
    iterations = 0
    while True:
        w = (mu / (mu + gnc_residual2(T, a, b))) ** 2
        T = gnc_pose(a, b, w, a_shift, b_shift, dof)
        iterations += 1
        if mu == GNC_MIN_SCALE:
            return T, w, iterations, GNC_FOUND
        mu = max(mu / GNC_DIV_FACTOR, GNC_MIN_SCALE)
