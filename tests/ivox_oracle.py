"""numpy restatement of the device iVox and its GICP factor (gb_ivox_insert, gb_gicp_factor_create), written from the rules in
include/glim_b200.h and independently of the CUDA: the insert (sampling, fp64 transform and keys as tests/voxelmap_oracle.py,
sequential admission with fp32 storage, stamps, LRU eviction, ascending-key numbering, the table with drop rate 0), the
correspondence search in fp32 (np.float32 wherever the device is fp32), an fp64 GICP linearize / error, and the
Levenberg-Marquardt problem of gb_vgicp_align over them (the rule is tests/lm_oracle.py's)."""
import numpy as np

from tests import lm_oracle as lm
from tests import voxelmap_oracle as vo

F32, F64 = np.float32, np.float64
INIT_BUCKETS, MAX_SCAN = 16384, 10


def coords64(q, resolution):
    """floor(q * (1.0 / resolution)) in fp64 (resolution a double) -> (int64 coords (n,3), valid mask)"""
    inv = 1.0 / float(resolution)
    fin = np.isfinite(q).all(1)
    with np.errstate(invalid="ignore"):
        f = np.floor(np.where(fin[:, None], q, 0.0) * inv)
    ok = fin & (f >= -vo.KEY_OFFSET).all(1) & (f < vo.KEY_OFFSET).all(1)
    return np.where(ok[:, None], f, 0).astype(np.int64), ok


class IVox:
    """The map state of the rule: per voxel key, stamp and its points (fp32 position, fp32 covariance) in slot order."""

    def __init__(self, resolution, min_dist=0.1, max_points=10, mode=1, lru_horizon=100, lru_clear_cycle=10):
        self.resolution = float(resolution)
        self.min_d2 = float(min_dist) * float(min_dist)
        self.max_points, self.mode = int(max_points), int(mode)
        self.h, self.k = int(lru_horizon), int(lru_clear_cycle)
        self.counter = 0
        self.vox = {}  # packed key -> [stamp, list of fp32 xyz (3,), list of fp32 cov6 (6,)]
        self.finalize()

    def insert(self, xyz, cov6, T=None, rate=1.0, seed=0):
        T = np.eye(4) if T is None else np.asarray(T, dtype=F64)
        n = len(xyz)
        keep = vo.sample_mask(n, rate, seed)
        q, c6 = vo.transform(T, xyz, cov6)
        cc, ok = coords64(q, self.resolution)
        sel = np.nonzero(keep & ok)[0]
        keys = vo.pack(cc[sel]) if len(sel) else np.zeros(0, np.uint64)
        q32, c32 = q.astype(F32), c6.astype(F32)
        touched = set()
        for i, key in zip(sel, keys):  # original index order
            key = int(key)
            v = self.vox.setdefault(key, [self.counter, [], []])
            touched.add(key)
            if len(v[1]) >= self.max_points:
                continue
            a = q32[i].astype(F64)
            admit = True
            for p in v[1]:
                d = p.astype(F64) - a
                if (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] < self.min_d2:
                    admit = False
                    break
            if admit:
                v[1].append(q32[i])
                v[2].append(c32[i])
        for key in touched:
            self.vox[key][0] = self.counter
        self.counter += 1
        if self.h > 0 and self.counter % self.k == 0:
            self.vox = {key: v for key, v in self.vox.items() if not (v[0] + self.h < self.counter)}
        self.finalize()
        return self

    def finalize(self):
        keys = sorted(self.vox)
        self.keys = np.array(keys, dtype=np.uint64)
        self.counts = np.array([len(self.vox[k][1]) for k in keys], dtype=np.int32)
        self.stamps = np.array([self.vox[k][0] for k in keys], dtype=np.int64)
        P = int(self.counts.sum())
        self.xyz = np.array([p for k in keys for p in self.vox[k][1]], dtype=F32).reshape(P, 3)
        self.cov6 = np.array([c for k in keys for c in self.vox[k][2]], dtype=F32).reshape(P, 6)
        self.first = np.concatenate([[0], np.cumsum(self.counts)[:-1]]).astype(np.int64) if len(keys) else np.zeros(0, np.int64)
        self.vcoord = vo.unpack(self.keys) if len(keys) else np.zeros((0, 3), np.int64)
        self.index = {tuple(int(x) for x in c): v for v, c in enumerate(self.vcoord)}
        self.buckets, self.dropped = vo.build_table(self.vcoord, self.counts, INIT_BUCKETS, MAX_SCAN, 0.0, float(P))
        assert self.dropped == 0

    @property
    def num_voxels(self):
        return len(self.keys)

    @property
    def num_points(self):
        return len(self.xyz)


# ---------------------------------------------------------------------------------------------------------------------
# the correspondence rule (fp32)
# ---------------------------------------------------------------------------------------------------------------------
def fmaf(a, b, c):
    """fp32 fused multiply-add, correctly rounded: a * b is exact in fp64, the fp64 sum's error is recovered (TwoSum) and
    decides the one case where rounding the fp64 sum to fp32 is not the correctly rounded result (a sum exactly halfway
    between two floats)."""
    a, b, c = (np.asarray(x, dtype=F32) for x in (a, b, c))
    p = a.astype(F64) * b.astype(F64)
    c64 = c.astype(F64)
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c64
        bb = s - p
        err = (p - (s - bb)) + (c64 - bb)
        r = s.astype(F32)
        r64 = r.astype(F64)
        other = np.nextafter(r, np.where(s > r64, F32(np.inf), F32(-np.inf)).astype(F32))
        mid = (r64 + other.astype(F64)) * 0.5
        halfway = (s != r64) & (s == mid) & (err != 0)
        up = err > 0
        hi, lo = np.maximum(r, other), np.minimum(r, other)
        return np.where(halfway, np.where(up, hi, lo), r).astype(F32)


def pose_f32(T):
    """the sweep's fp32 pose (Isometry3f cast): R (3,3) and t (3,) as float32"""
    T = np.asarray(T, dtype=F64)
    return T[:3, :3].astype(F32), T[:3, 3].astype(F32)


def transform_f32(T, xyz):
    """q = R a + t with the kernel's fmaf order: q_r = fma(r0, x, fma(r1, y, fma(r2, z, t_r)))"""
    R, t = pose_f32(T)
    a = np.asarray(xyz, dtype=F32)
    x, y, z = a[:, 0], a[:, 1], a[:, 2]
    return np.stack([fmaf(R[r, 0], x, fmaf(R[r, 1], y, fmaf(R[r, 2], z, t[r]))) for r in range(3)], 1)


def offsets(mode):
    """the search order: centre; faces -x +x -y +y -z +z; edges (zero axis x, y, z; other signs --, -+, +-, ++); corners"""
    out = [(0, 0, 0)]
    for ax in range(3):
        for s in (-1, 1):
            o = [0, 0, 0]
            o[ax] = s
            out.append(tuple(o))
    for zero in range(3):
        rest = [a for a in range(3) if a != zero]
        for s1 in (-1, 1):
            for s2 in (-1, 1):
                o = [0, 0, 0]
                o[rest[0]], o[rest[1]] = s1, s2
                out.append(tuple(o))
    for dx in (-1, 1):
        for dy in (-1, 1):
            for dz in (-1, 1):
                out.append((dx, dy, dz))
    return out[:mode]


def fp32_coords(q, inv_res):
    """__float2int_rd(q * inv_res): NaN -> 0, saturated to int32"""
    with np.errstate(invalid="ignore", over="ignore"):
        f = np.floor((q * F32(inv_res)).astype(F32)).astype(F64)
    f = np.where(np.isnan(f), 0.0, np.clip(f, -2.0 ** 31, 2.0 ** 31 - 1))
    return f.astype(np.int64)


def correspondences(m: IVox, xyz, T, max_corr):
    """record index of every source point's correspondence (-1: none)"""
    q = transform_f32(T, xyz)
    inv_res = F32(1.0 / m.resolution)
    c = fp32_coords(q, inv_res)
    thr = F32(float(max_corr) * float(max_corr))
    out = np.full(len(q), -1, np.int64)
    offs = offsets(m.mode)
    for i in range(len(q)):
        best, best_d2 = -1, thr
        for o in offs:
            v = m.index.get((int(c[i, 0]) + o[0], int(c[i, 1]) + o[1], int(c[i, 2]) + o[2]))
            if v is None:
                continue
            f, n = int(m.first[v]), int(m.counts[v])
            d = m.xyz[f:f + n] - q[i]  # fp32
            with np.errstate(invalid="ignore", over="ignore"):
                d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
            for s in range(n):
                if d2[s] < best_d2:
                    best_d2, best = d2[s], f + s
        out[i] = best
    return out


# ---------------------------------------------------------------------------------------------------------------------
# fp64 GICP linearize / error (the math of numpy_linearize in tests/test_oracle_vgicp.py, point records for voxel records)
# ---------------------------------------------------------------------------------------------------------------------
def cov33(c6):
    c6 = np.asarray(c6, dtype=F64)
    return np.stack([c6[:, [0, 1, 2]], c6[:, [1, 3, 4]], c6[:, [2, 4, 5]]], 1)


def hat(v):
    H = np.zeros((v.shape[0], 3, 3))
    H[:, 0, 1], H[:, 0, 2] = -v[:, 2], v[:, 1]
    H[:, 1, 0], H[:, 1, 2] = v[:, 2], -v[:, 0]
    H[:, 2, 0], H[:, 2, 1] = -v[:, 1], v[:, 0]
    return H


def residuals(m: IVox, xyz, cov6, T, corr, M_pose=None):
    """fp64 at the fp32-cast pose the kernel uses, for the points with a correspondence: (a, q, r = p - q, M) with
    M = (C_p + R C_a R^T)^-1 formed at M_pose (default T)"""
    Tf = np.asarray(T, dtype=F32).astype(F64)
    Rm = np.asarray(T if M_pose is None else M_pose, dtype=F32).astype(F64)[:3, :3]
    R, t = Tf[:3, :3], Tf[:3, 3]
    k = corr >= 0
    a = np.asarray(xyz, dtype=F32)[k].astype(F64)
    CA = cov33(np.asarray(cov6, dtype=F32)[k])
    mu = m.xyz[corr[k]].astype(F64)
    CB = cov33(m.cov6[corr[k]])
    q = a @ R.T + t
    return a, q, mu - q, np.linalg.inv(CB + Rm @ CA @ Rm.T)


def linearize(m: IVox, xyz, cov6, T, max_corr, corr=None):
    """fp64 blocks at T (the fp32-cast pose the kernel uses) with the correspondences of T (or `corr`).
    -> (dict of H_tt .. num_inliers, corr)"""
    if corr is None:
        corr = correspondences(m, xyz, T, max_corr)
    R = np.asarray(T, dtype=F32).astype(F64)[:3, :3]
    a, q, r, M = residuals(m, xyz, cov6, T, corr)
    n = a.shape[0]
    Jt = np.concatenate([-hat(q), np.tile(np.eye(3), (n, 1, 1))], axis=2)
    Js = np.concatenate([R @ hat(a), np.tile(-R, (n, 1, 1))], axis=2)
    Mr = np.einsum("nij,nj->ni", M, r)
    out = {
        "H_tt": np.einsum("nki,nkl,nlj->ij", Jt, M, Jt),
        "H_ss": np.einsum("nki,nkl,nlj->ij", Js, M, Js),
        "H_ts": np.einsum("nki,nkl,nlj->ij", Jt, M, Js),
        "b_t": np.einsum("nki,nk->i", Jt, Mr),
        "b_s": np.einsum("nki,nk->i", Js, Mr),
        "error": float(np.einsum("ni,ni->", r, Mr)),
        "num_inliers": float(n),
    }
    return out, corr


def error(m: IVox, xyz, cov6, T_lin, T_eval, max_corr):
    """error at T_eval with the correspondences of T_lin"""
    corr = correspondences(m, xyz, T_lin, max_corr)
    return linearize(m, xyz, cov6, T_eval, max_corr, corr=corr)[0]["error"]


def align(m: IVox, xyz, cov6, T0, max_corr, params=None):
    """gb_vgicp_align's rule (tests/lm_oracle.py) on one GICP factor, in fp64.  -> dict(T, error, num_inliers, lambda,
    iterations, trials, status)"""

    def lin(T):
        r, corr = linearize(m, xyz, cov6, T, max_corr)
        return r["H_ss"], r["b_s"], r["error"], r["num_inliers"], corr

    return lm.align_pose(lin, lambda corr, Tn: linearize(m, xyz, cov6, Tn, max_corr, corr=corr)[0]["error"], T0, params)
