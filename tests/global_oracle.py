"""Numpy restatement of global registration (gb_cloud_estimate_fpfh, gb_fpfh_match, gb_ransac_align), written from the rules in
include/glim_b200.h and independently of the CUDA: the brute-force radius neighbourhood, the PCL / Open3D pair features and
bins, SPFH and FPFH in fp64, the sequential fp32 feature distance and its argmin, the RANSAC sample draw, Horn's estimator (here
by numpy's symmetric eigensolver) and the 4-DoF estimator, the fp32 inlier test and the selection rule."""
import math

import numpy as np

from tests.grid_oracle import d2_matrix
from tests.ivox_oracle import fp32_coords
from tests.voxelmap_oracle import rg_hash

F32, F64 = np.float32, np.float64
DIM, BINS = 33, 11
MIN_AREA2 = 1e-3
WAVE = 512
FOUND, EARLY_STOP, DEGENERATE = 0, 1, 2


def neighbours(xyz, r, chunk=512):
    """per point, the other points j with fp32 d2 < (float)(r^2), ascending index"""
    xyz = np.asarray(xyz, dtype=F32)
    thr = F32(float(r) * float(r))
    out = []
    for i0 in range(0, len(xyz), chunk):
        d2 = d2_matrix(xyz[i0:i0 + chunk], xyz)
        for k, row in enumerate(d2):
            nb = np.nonzero(row < thr)[0]
            out.append(nb[nb != i0 + k])
    return out


# the C library's atan2, as the host build calls it (numpy's vectorised arctan2 may differ from it in the last bit)
_atan2 = np.frompyfunc(math.atan2, 2, 1)


def atan2(y, x):
    return _atan2(y, x).astype(F64)


def pair_features(ps, ns, pt, nt):
    """(f1, f2, f3) of pairs (rows), fp64; zero for |d| = 0 or |v| = 0"""
    ps, ns, pt, nt = (np.atleast_2d(np.asarray(x, dtype=F64)) for x in (ps, ns, pt, nt))
    d = pt - ps
    dd = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    with np.errstate(invalid="ignore", divide="ignore"):
        ln = np.sqrt(dd)
        dot = lambda a, b: (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]
        a1, a2 = dot(ns, d) / ln, dot(nt, d) / ln
        swap = (np.abs(a1) < np.abs(a2))[:, None]
        s = np.where(swap, nt, ns)
        t = np.where(swap, ns, nt)
        d = np.where(swap, -d, d)
        f3 = np.where(swap[:, 0], -a2, a1)
        cross = lambda a, b: np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
        v = cross(d, s)
        vv = dot(v, v)
        v = v / np.sqrt(vv)[:, None]
        w = cross(s, v)
        f = np.stack([atan2(dot(w, t), dot(s, t)), dot(v, t), f3], 1)
    f[(dd == 0) | (vv == 0)] = 0.0
    return f, dd


def scaled(f):
    """the bin coordinates t in [0, 11) of each feature"""
    return np.stack([(11.0 * (f[:, 0] + np.pi)) / (2 * np.pi), (11.0 * (f[:, 1] + 1.0)) * 0.5, (11.0 * (f[:, 2] + 1.0)) * 0.5], 1)


def bins(f):
    """(n, 3) indices into the 33-bin histogram; floor clamped to [0, 10], NaN to 0"""
    t = scaled(f)
    with np.errstate(invalid="ignore"):
        b = np.where(t >= 1.0, np.where(t >= 10.0, 10, np.floor(np.where(np.isfinite(t), t, 0.0))), 0).astype(np.int64)
    return b + np.array([0, BINS, 2 * BINS])


def fpfh(xyz, normals, r, nbs=None):
    """-> (features (n, 33) fp64, spfh (n, 33), edge margin (n,): the smallest distance of any of the point's or its neighbours'
    scaled pair features to a bin edge -- a bin of a point within a few ulps of one may differ between implementations)"""
    xyz = np.asarray(xyz, dtype=F32)
    nrm = np.asarray(normals, dtype=F32)[:, :3]
    n = len(xyz)
    nbs = neighbours(xyz, r) if nbs is None else nbs
    spfh = np.zeros((n, DIM))
    own_margin = np.full(n, np.inf)
    pairs = []
    for i in range(n):
        nb = nbs[i]
        if len(nb) == 0:
            pairs.append(np.zeros(0))
            continue
        f, dd = pair_features(np.repeat(xyz[i:i + 1], len(nb), 0), np.repeat(nrm[i:i + 1], len(nb), 0), xyz[nb], nrm[nb])
        t = scaled(f)
        own_margin[i] = np.abs(t - np.round(t)).min()
        cnt = np.bincount(bins(f).reshape(-1), minlength=DIM)
        spfh[i] = cnt * (100.0 / len(nb))
        pairs.append(dd)
    feat = np.zeros((n, DIM))
    margin = own_margin.copy()
    for i in range(n):
        nb = nbs[i]
        if len(nb) == 0:
            continue
        margin[i] = min(margin[i], own_margin[nb].min())
        acc, s = np.zeros(DIM), np.zeros(3)
        for j, dd in zip(nb, pairs[i]):
            if dd == 0:
                continue
            v = spfh[j] / dd
            acc += v
            s += v.reshape(3, BINS).sum(1)
        scale = np.where(s != 0, 100.0 / np.where(s != 0, s, 1.0), 0.0)
        feat[i] = acc * np.repeat(scale, BINS) + spfh[i]
    return feat, spfh, margin


def match(target, source):
    """nearest target feature of every source feature: fp32 d2 summed sequentially over the 33 terms, ties to the smaller
    index, -1 when no distance is a number"""
    t = np.asarray(target, dtype=F32)
    s = np.asarray(source, dtype=F32)
    out = np.full(len(s), -1, np.int64)
    for i0 in range(0, len(s), 256):
        a = s[i0:i0 + 256]
        e = a[:, None, 0] - t[None, :, 0]
        d2 = e * e
        for k in range(1, DIM):
            e = a[:, None, k] - t[None, :, k]
            d2 = d2 + e * e
        d2 = np.where(np.isnan(d2), np.inf, d2)
        j = np.argmin(d2, 1)  # the first minimum
        ok = np.isfinite(d2[np.arange(len(a)), j])
        out[i0:i0 + 256] = np.where(ok, j, -1)
    return out


def sample(seed, h, ns):
    """the three source indices of hypothesis h"""
    return [int(rg_hash(seed, 3 * h + j) % np.uint64(ns)) for j in range(3)]


def area2(x):
    c = np.cross(x[1] - x[0], x[2] - x[0])
    return float(np.sqrt(c @ c))


def estimate_pose(a, b, dof):
    """T (4,4) with b ~ R a + t from three pairs, or None for an invalid sample"""
    a, b = np.asarray(a, dtype=F64), np.asarray(b, dtype=F64)
    if not (area2(a) >= MIN_AREA2 and area2(b) >= MIN_AREA2):
        return None
    ca, cb = a.mean(0), b.mean(0)
    A, B = a - ca, b - cb
    if dof == 4:
        yaw = np.arctan2((A[:, 0] * B[:, 1] - A[:, 1] * B[:, 0]).sum(), (A[:, 0] * B[:, 0] + A[:, 1] * B[:, 1]).sum())
        R = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1.0]])
    else:
        S = A.T @ B
        (sxx, sxy, sxz), (syx, syy, syz), (szx, szy, szz) = S
        N = np.array([[sxx + syy + szz, syz - szy, szx - sxz, sxy - syx],
                      [syz - szy, sxx - syy - szz, sxy + syx, szx + sxz],
                      [szx - sxz, sxy + syx, -sxx + syy - szz, syz + szy],
                      [sxy - syx, szx + sxz, syz + szy, -sxx - syy + szz]])
        w, x, y, z = np.linalg.eigh(N)[1][:, -1]
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = cb - R @ ca
    return T


def hypothesis(seed, h, src_xyz, tgt_xyz, nearest, dof):
    """(sample, T or None) of hypothesis h"""
    s = sample(seed, h, len(src_xyz))
    if len(set(s)) < 3 or min(nearest[j] for j in s) < 0:
        return s, None
    a = np.asarray(src_xyz, dtype=F32)[s].astype(F64)
    b = np.asarray(tgt_xyz, dtype=F32)[[nearest[j] for j in s]].astype(F64)
    return s, estimate_pose(a, b, dof)


def occupancy(tgt_xyz, resolution):
    """the set of cells (fp32 keys) that hold a target point"""
    inv = F32(1.0 / resolution)
    x = np.asarray(tgt_xyz, dtype=F32)
    x = x[np.isfinite(x).all(1)]
    c = fp32_coords(x, inv)
    c = c[(np.abs(c + 0.5) < 2 ** 20).all(1)]
    return {tuple(k) for k in c.tolist()}, inv


def inliers(T, src_xyz, occ):
    """the inlier count of pose T: q = ((r0 x + r1 y) + r2 z) + t in fp32, finite, in an occupied cell"""
    cells, inv = occ
    R = np.asarray(T[:3, :3], dtype=F32)
    t = np.asarray(T[:3, 3], dtype=F32)
    a = np.asarray(src_xyz, dtype=F32)
    with np.errstate(invalid="ignore", over="ignore"):
        q = np.stack([((R[r, 0] * a[:, 0] + R[r, 1] * a[:, 1]) + R[r, 2] * a[:, 2]) + t[r] for r in range(3)], 1)
    fin = np.isfinite(q).all(1)
    c = fp32_coords(q[fin], inv)
    return int(sum(tuple(k) in cells for k in c.tolist()))


def select(counts, ns, rate, max_iterations, wave=WAVE):
    """the selection rule over per-hypothesis counts (-1 invalid), scored in waves: -> (best h, status, evaluated)"""
    best, best_c, stop, evaluated = -1, 0, -1, 0
    for h0 in range(0, max_iterations, wave):
        w = min(wave, max_iterations - h0)
        evaluated = h0 + w
        for h in range(h0, h0 + w):
            c = counts[h]
            if c > best_c:
                best, best_c = h, c
            if stop < 0 and c >= 0 and c / ns >= rate:
                stop = h
        if stop >= 0:
            break
    if stop >= 0:
        return stop, EARLY_STOP, evaluated
    return best, (FOUND if best >= 0 else DEGENERATE), evaluated
