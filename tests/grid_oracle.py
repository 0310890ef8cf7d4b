"""numpy restatement of the device point grid and its GICP factor (gb_point_grid_build, gb_gicp_grid_factor_create), written
from the rules in include/glim_b200.h and independently of the CUDA: the build (fp32 keys, cell order, record order, the table
with drop rate 0), the correspondence as a brute-force fp32 argmin over every target point with the index tie, the search
half-width's bound, and linearize / error over them with the Levenberg-Marquardt rule of tests/lm_oracle.py.  The per-point fp64 arithmetic is
tests/ivox_oracle.py's (residuals, linearize), fed this module's correspondences."""
import numpy as np

from tests import ivox_oracle as io
from tests import lm_oracle as lm
from tests import voxelmap_oracle as vo

F32, F64 = np.float32, np.float64
INIT_BUCKETS, MAX_SCAN = 16384, 10
MAX_HALF_WIDTH = 8


class PointGrid:
    """Every point of a cloud (fp32 xyz (n,3) and cov6 (n,6) in the caller's order) grouped by its fp32 key."""

    def __init__(self, xyz, cov6, cell_size):
        xyz, cov6 = np.asarray(xyz, dtype=F32).reshape(-1, 3), np.asarray(cov6, dtype=F32).reshape(-1, 6)
        n = len(xyz)
        self.cell_size = float(cell_size)
        self.inv = F32(1.0 / self.cell_size)
        fin = np.isfinite(xyz).all(1)
        c = io.fp32_coords(np.where(fin[:, None], xyz, F32(0)), self.inv)
        ok = fin & (c >= -vo.KEY_OFFSET).all(1) & (c < vo.KEY_OFFSET).all(1)
        keys = np.full(n, np.iinfo(np.uint64).max, np.uint64)
        if ok.any():
            keys[ok] = vo.pack(c[ok])
        order = np.lexsort((np.arange(n), keys))  # ascending key, then original index; keyless points last
        self.index = order.astype(np.int64)
        self.xyz, self.cov6 = xyz[order], cov6[order]
        self.num_keyed = int(ok.sum())
        ks = keys[order][: self.num_keyed]
        self.keys, self.first, self.counts = np.unique(ks, return_index=True, return_counts=True)
        self.first, self.counts = self.first.astype(np.int64), self.counts.astype(np.int32)
        self.vcoord = vo.unpack(self.keys) if len(self.keys) else np.zeros((0, 3), np.int64)
        self.key_extent = int(np.maximum(-self.vcoord, self.vcoord + 1).max()) if len(self.keys) else 0
        self.buckets, dropped = vo.build_table(self.vcoord, self.counts, INIT_BUCKETS, MAX_SCAN, 0.0, float(n))
        assert dropped == 0

    @property
    def num_cells(self):
        return len(self.keys)

    @property
    def num_points(self):
        return len(self.xyz)


def half_width(inv, max_d2, key_extent):
    """grid_half_width of gb_grid_math.cuh: ceil(W) with W = D inv + u (A_p + A_q) (+ slack), D = sqrt(max_d2) / (1 - u),
    A_p = K / (1 - u), A_q = A_p + D inv; MAX_HALF_WIDTH + 1 when W exceeds MAX_HALF_WIDTH"""
    u = 2.0 ** -24
    D = np.sqrt(float(F32(max_d2))) / (1.0 - u)
    Ap = float(key_extent) / (1.0 - u)
    Aq = Ap + D * float(F32(inv))
    W = (D * float(F32(inv)) + u * (Ap + Aq) + 2.0 ** -148) * (1.0 + 2.0 ** -40)
    return int(np.ceil(W)) if W <= MAX_HALF_WIDTH else MAX_HALF_WIDTH + 1


def max_d2(max_corr):
    return F32(float(max_corr) * float(max_corr))


def d2_matrix(q, p):
    """fp32 (dx^2 + dy^2) + dz^2 of every (query, point) pair, d = p - q, each operation rounded to fp32"""
    d = p[None, :, :] - q[:, None, :]
    with np.errstate(invalid="ignore", over="ignore"):
        return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def nearest(g: PointGrid, q, thr, chunk=256):
    """record of the brute-force correspondence of every fp32 query q (n,3): the smallest d2 < thr over every keyed point,
    ties to the smaller original index; -1 for none"""
    q = np.asarray(q, dtype=F32)
    out = np.full(len(q), -1, np.int64)
    K = g.num_keyed
    if K == 0:
        return out
    p, idx = g.xyz[:K], g.index[:K]
    for a in range(0, len(q), chunk):
        d2 = d2_matrix(q[a:a + chunk], p)
        ok = d2 < thr
        best = np.where(ok, d2, F32(np.inf)).min(1)
        tie = ok & (d2 == best[:, None])
        cand = np.where(tie, idx[None, :], np.iinfo(np.int64).max)
        has = tie.any(1)
        r = np.argmin(cand, 1)
        out[a:a + chunk] = np.where(has, r, -1)
    return out


def correspondences(g: PointGrid, xyz, T, max_corr):
    """record index of every source point's correspondence at T (-1: none)"""
    return nearest(g, io.transform_f32(T, xyz), max_d2(max_corr))


def linearize(g: PointGrid, xyz, cov6, T, max_corr, corr=None):
    """fp64 blocks at T (the fp32-cast pose) with the correspondences of T (or `corr`) -> (dict, corr)"""
    if corr is None:
        corr = correspondences(g, xyz, T, max_corr)
    return io.linearize(g, xyz, cov6, T, max_corr, corr=corr)


def error(g: PointGrid, xyz, cov6, T_lin, T_eval, max_corr):
    """error at T_eval with the correspondences of T_lin"""
    return linearize(g, xyz, cov6, T_eval, max_corr, corr=correspondences(g, xyz, T_lin, max_corr))[0]["error"]


def align(g: PointGrid, xyz, cov6, T0, max_corr, params=None):
    """gb_vgicp_align's rule (tests/lm_oracle.py) on one grid factor, in fp64.  -> dict(T, error, num_inliers, lambda,
    iterations, trials, status)"""

    def lin(T):
        r, corr = linearize(g, xyz, cov6, T, max_corr)
        return r["H_ss"], r["b_s"], r["error"], r["num_inliers"], corr

    return lm.align_pose(lin, lambda corr, Tn: linearize(g, xyz, cov6, Tn, max_corr, corr=corr)[0]["error"], T0, params)
