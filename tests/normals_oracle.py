"""numpy restatement of gb_cloud_estimate_normals (the rule in include/glim_b200.h): per point the eigenvector of the smallest
eigenvalue of its fp32 covariance widened to fp64 (numpy.linalg.eigh), turned away from the point when p . n > 0; zero for a
point whose position or covariance is not finite.  Also returns the relative eigen-gap, below which the direction is not
determined by the covariance."""
import numpy as np

F32, F64 = np.float32, np.float64


def normals(xyz, cov6):
    """xyz (n,3), cov6 (n,6: c00 c01 c02 c11 c12 c22) fp32 -> (normals (n,3) fp64, relative gap (n,): (l1 - l0) / max |l|)"""
    xyz = np.asarray(xyz, dtype=F32).astype(F64)
    c = np.asarray(cov6, dtype=F32).astype(F64)
    ok = np.isfinite(xyz).all(1) & np.isfinite(c).all(1)
    A = np.zeros((len(c), 3, 3))
    A[ok] = np.stack([c[ok][:, [0, 1, 2]], c[ok][:, [1, 3, 4]], c[ok][:, [2, 4, 5]]], 1)
    w, V = np.linalg.eigh(A)
    n = V[:, :, 0]
    flip = (xyz[:, 0] * n[:, 0] + xyz[:, 1] * n[:, 1]) + xyz[:, 2] * n[:, 2] > 0
    n[flip] = -n[flip]
    n[~ok] = 0.0
    scale = np.abs(w).max(1)
    gap = np.where(scale > 0, (w[:, 1] - w[:, 0]) / np.where(scale > 0, scale, 1.0), 0.0)
    gap[~ok] = 0.0
    return n, gap
