"""numpy restatement of the point-to-point ICP factor on a point grid (gb_icp_grid_factor_create), written from the rule in
include/glim_b200.h and independently of the CUDA: the correspondences are tests/grid_oracle.py's brute-force fp32 argmin, and
the per-point arithmetic is the GICP grid factor's with M = I, in fp64 at the fp32-cast pose the kernel uses."""
import numpy as np

from tests import grid_oracle as go
from tests import ivox_oracle as io
from tests import lm_oracle as lm

F32, F64 = np.float32, np.float64


def grid(xyz, cell_size):
    """the point grid of a cloud without covariances (its records hold zero covariances)"""
    xyz = np.asarray(xyz, dtype=F32).reshape(-1, 3)
    return go.PointGrid(xyz, np.zeros((len(xyz), 6), F32), cell_size)


def linearize(g: go.PointGrid, xyz, T, max_corr, corr=None):
    """fp64 blocks at T with the correspondences of T (or `corr`): r = p - q, error = sum r^T r.  -> (dict, corr)"""
    if corr is None:
        corr = go.correspondences(g, xyz, T, max_corr)
    Tf = np.asarray(T, dtype=F32).astype(F64)
    R, t = Tf[:3, :3], Tf[:3, 3]
    k = corr >= 0
    a = np.asarray(xyz, dtype=F32)[k].astype(F64)
    q = a @ R.T + t
    r = g.xyz[corr[k]].astype(F64) - q
    n = a.shape[0]
    Jt = np.concatenate([-io.hat(q), np.tile(np.eye(3), (n, 1, 1))], axis=2)
    Js = np.concatenate([R @ io.hat(a), np.tile(-R, (n, 1, 1))], axis=2)
    out = {
        "H_tt": np.einsum("nki,nkj->ij", Jt, Jt),
        "H_ss": np.einsum("nki,nkj->ij", Js, Js),
        "H_ts": np.einsum("nki,nkj->ij", Jt, Js),
        "b_t": np.einsum("nki,nk->i", Jt, r),
        "b_s": np.einsum("nki,nk->i", Js, r),
        "error": float(np.einsum("ni,ni->", r, r)),
        "num_inliers": float(n),
    }
    return out, corr


def error(g: go.PointGrid, xyz, T_lin, T_eval, max_corr):
    """error at T_eval with the correspondences of T_lin"""
    return linearize(g, xyz, T_eval, max_corr, corr=go.correspondences(g, xyz, T_lin, max_corr))[0]["error"]


def align(g: go.PointGrid, xyz, T0, max_corr, params=None):
    """gb_vgicp_align's rule (tests/lm_oracle.py) on one ICP factor, in fp64"""

    def lin(T):
        r, corr = linearize(g, xyz, T, max_corr)
        return r["H_ss"], r["b_s"], r["error"], r["num_inliers"], corr

    return lm.align_pose(lin, lambda corr, Tn: linearize(g, xyz, Tn, max_corr, corr=corr)[0]["error"], T0, params)


def hit(T, a, v):
    """one hit's accumulators as accumulate_icp_hit lays them out, in fp64 at the fp32-cast pose: the upper triangle of H_tt
    (row-major, 21), b_t (6), error, count"""
    Tf = np.asarray(T, dtype=F32).astype(F64)
    q = Tf[:3, :3] @ np.asarray(a, dtype=F32).astype(F64) + Tf[:3, 3]
    r = np.asarray(v, dtype=F32).astype(F64) - q
    J = np.concatenate([-io.hat(q[None])[0], np.eye(3)], axis=1)
    H = J.T @ J
    return np.concatenate([H[np.triu_indices(6)], J.T @ r, [r @ r, 1.0]])
