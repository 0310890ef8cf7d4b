"""Shared helpers for the test-suite: small seeded scenarios and error metrics."""
import functools
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from glim_b200 import synth  # noqa: E402

# tolerance of north_star: Hessians / gradients within 1e-4 relative (Frobenius) of the fp64 oracle
REL_TOL = 1e-4


def rel_err(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    d = np.linalg.norm(a - b)
    n = np.linalg.norm(b)
    return d / n if n > 0 else d


@functools.lru_cache(maxsize=None)
def scan_pair(sensor="hdl32", n_rays=32 * 300, step=1.0, key=0, scene="hall"):
    """Two scans `step` metres apart along the M2 arc, with PLANE covariances (k = 10).
    -> dict(points=[P0,P1] (N,4), covs=[C0,C1] (N,4,4), normals=[..], poses=[T0,T1])"""
    sc = synth.make_hall_scene() if scene == "hall" else synth.make_blocks_scene()
    traj = synth.arc_trajectory(8, step=step)
    out = {"points": [], "covs": [], "normals": [], "poses": [], "times": []}
    for i in (3, 4):
        pts, tms = synth.scan(sc, sensor, traj[i], synth.rng_for(77, key, i), n_rays=n_rays)
        nrm, cov = synth.with_covariances(pts, 10)
        out["points"].append(pts)
        out["covs"].append(cov)
        out["normals"].append(nrm)
        out["poses"].append(traj[i])
        out["times"].append(tms)
    return out


def check_linearized(got: dict, ref, tol=REL_TOL, hits=None):
    """A device record (unpacked) against a reference: a 122-double oracle record or a dict of blocks indexed [row, col].
    Inlier count exact; Hessians, gradients and error within `tol` relative of the reference (a factor without inliers: zeros).
    hits: the factor's per-hit data (Hits) or the entry-wise scales they give (EntryScale): then every entry is also held to
    its own first-order error bound (check_entrywise).  -> the largest entry-wise ratio (0.0 without hits)"""
    from oracle import oracle

    if not isinstance(ref, dict):
        ref = oracle.split122(ref)
    assert got["num_inliers"] == ref["num_inliers"]  # inlier set bit-exact
    for k in ("H_tt", "H_ss", "H_ts"):
        assert rel_err(got[k], ref[k]) < tol, (k, rel_err(got[k], ref[k]))
    # The gradient b = sum J^T M r is a sum of terms that cancel as the pose converges, so its fp32 rounding noise does
    # not shrink with |b|.  Its natural magnitude is the Cauchy-Schwarz bound sqrt(tr(H) * error) of the un-cancelled
    # sum; the tolerance is 1e-4 of max(|b|, a tenth of that bound).
    for k, hk in (("b_t", "H_tt"), ("b_s", "H_ss")):
        scale = max(np.linalg.norm(ref[k]), 0.1 * np.sqrt(np.trace(ref[hk]) * max(ref["error"], 1e-30)))
        assert np.linalg.norm(got[k] - ref[k]) <= tol * scale, (k, np.linalg.norm(got[k] - ref[k]) / scale, np.linalg.norm(got[k] - ref[k]) / np.linalg.norm(ref[k]))
    assert abs(got["error"] - ref["error"]) <= tol * abs(ref["error"]) + 1e-12
    if hits is None:
        return 0.0
    return check_entrywise(got, ref, hits if isinstance(hits, EntryScale) else record_scale(hits))


# ---------------------------------------------------------------------------------------------------------------------
# Entry-wise error bounds of a linearized record
#
# A Frobenius norm of a 6x6 block is almost all of its rotation-rotation part (it grows as |q|^2 M, the translation part as
# M), so a relative Frobenius bar hardly sees the other entries.  Here every entry e of H_tt, b_t and the error gets its own
# first-order forward-error bound, formed from the absolute values of the same per-hit factors the kernel multiplies:
#
#   |got_e - ref_e| <= ENTRY_TOL * A_e + B_e
#
#   A_e  the sum over hits of the entry's terms with every factor replaced by its magnitude (|J|^T |M| |J|, |J|^T |M| |r|,
#        |r|^T |M| |r|).  The kernel's rounding of its products and of its fp32 sums is a multiple of 2^-24 A_e;
#        ENTRY_TOL = 1e-4 ~ 1680 x 2^-24 covers the longest fp32 serial chain of the sweeps (64 hits per lane in a 2048-point
#        item, then the 5-step warp reduction) with the per-hit products on top.
#   B_e  the first-order effect of two input errors of a hit that do not grow with the chain, at their own size:
#        - the fp32 inverse M = S^-1 of the fused covariance S: |dM| <= INV_ROUNDING 2^-24 |M| |S| |M| entry-wise (dM = -M dS M
#          to first order).  This is where the condition of S enters: for a plane's covariance it is up to ~1e3 times
#          2^-24 ||M||, and it falls on the entries along the plane's normal, where M is large;
#        - the fp32 rounding of the transformed point q (the kernel's fmaf chain, 2^-24 per rounding of each partial sum)
#          where it feeds r = mu - q and hat(q).  It matters far from the origin, where 2^-24 |q| is no longer small
#          against |r|.
#
# The epilogue forms H_ss = Ad^T H_tt Ad, H_ts = -H_tt Ad and b_s = -Ad^T b_t in fp64 from the fp32-cast pose, so their
# bounds are the H_tt / b_t bounds taken through |Ad| the same way.  The reference entries are the fp64 restatement's.
# ---------------------------------------------------------------------------------------------------------------------
ENTRY_TOL = 1e-4
U32 = 2.0 ** -24
INV_ROUNDING = 16  # roundings per entry of the cofactor inverse (fused_mahalanobis), with margin
KEYS = ("H_tt", "H_ss", "H_ts", "b_t", "b_s", "error")


class Hits:
    """Per-hit data of a factor at one pose, fp64: J (n,3,6) = [-hat(q) | I], M (n,3,3), r (n,3) = mu - q, dq (n,3) a bound on
    the kernel's fp32 rounding of q, T the pose whose fp32 cast the kernel used."""

    def __init__(self, J, M, r, dq, T):
        self.J, self.M, self.r, self.dq, self.T = J, M, r, dq, np.asarray(T, dtype=np.float64)

    def __len__(self):
        return len(self.r)


class EntryScale:
    """A and B of every entry of a record (dicts of arrays keyed as the record), see above."""

    def __init__(self, A, B):
        self.A, self.B = A, B

    def __add__(self, o):
        return EntryScale({k: self.A[k] + o.A[k] for k in KEYS}, {k: self.B[k] + o.B[k] for k in KEYS})


def _cov33(c6):
    c6 = np.asarray(c6, dtype=np.float64)
    return np.stack([c6[:, [0, 1, 2]], c6[:, [1, 3, 4]], c6[:, [2, 4, 5]]], 1)


def _hat(v):
    H = np.zeros((v.shape[0], 3, 3))
    H[:, 0, 1], H[:, 0, 2] = -v[:, 2], v[:, 1]
    H[:, 1, 0], H[:, 1, 2] = v[:, 2], -v[:, 0]
    H[:, 2, 0], H[:, 2, 1] = -v[:, 1], v[:, 0]
    return H


def transform_rounding(T, xyz):
    """(the kernel's fp32 q, a per-coordinate bound on its rounding): q_r = fmaf(r0, x, fmaf(r1, y, fmaf(r2, z, t_r))) rounds
    each of its three partial sums once, by at most 2^-24 of the partial"""
    from tests import ivox_oracle as io

    R, t = (x.astype(np.float64) for x in io.pose_f32(T))
    a = np.asarray(xyz, dtype=np.float32).astype(np.float64)
    s1 = a[:, 2:3] * R[:, 2] + t
    s2 = a[:, 1:2] * R[:, 1] + s1
    q32 = io.transform_f32(T, xyz).astype(np.float64)
    return q32, U32 * (np.abs(s1) + np.abs(s2) + np.abs(q32))


def factor_hits(mu, cov_b, xyz, cov6, T, corr):
    """Per-hit data of a GICP-family factor at T from its device-layout inputs: target records (mu (m,3) fp32, cov_b (m,6) fp32
    or None for ICP, where M = I), source points / covariances (fp32) and the correspondences (record index, < 0: none).  The
    arithmetic is the restatements' (fp64 at the fp32-cast pose, M formed at T); a fused covariance with a zero or non-finite
    determinant is skipped, as the oracle and the kernel skip it."""
    Tf = np.asarray(T, dtype=np.float32).astype(np.float64)
    R, t = Tf[:3, :3], Tf[:3, 3]
    k = np.asarray(corr) >= 0
    a = np.asarray(xyz, dtype=np.float32)[k].astype(np.float64)
    q = a @ R.T + t
    r = np.asarray(mu, dtype=np.float32)[np.asarray(corr)[k]].astype(np.float64) - q
    if cov_b is None:
        M = np.tile(np.eye(3), (len(a), 1, 1))
    else:
        S = _cov33(np.asarray(cov_b, dtype=np.float32)[np.asarray(corr)[k]]) + R @ _cov33(np.asarray(cov6, dtype=np.float32)[k]) @ R.T
        det = S[:, 0, 0] * (S[:, 1, 1] * S[:, 2, 2] - S[:, 1, 2] * S[:, 2, 1]) + S[:, 0, 1] * (S[:, 1, 2] * S[:, 2, 0] - S[:, 1, 0] * S[:, 2, 2]) + S[:, 0, 2] * (S[:, 1, 0] * S[:, 2, 1] - S[:, 1, 1] * S[:, 2, 0])
        ok = (det != 0.0) & np.isfinite(det)
        a, q, r, S = a[ok], q[ok], r[ok], S[ok]
        k[np.flatnonzero(k)[~ok]] = False
        M = np.linalg.inv(S)
    _, dq = transform_rounding(T, np.asarray(xyz, dtype=np.float32)[k])
    J = np.concatenate([-_hat(q), np.tile(np.eye(3), (len(q), 1, 1))], axis=2)
    return Hits(J, M, r, dq, T)


def hit_sums(h: Hits):
    """the record the hits sum to (fp64): H_tt, b_t, error, num_inliers"""
    Mr = np.einsum("nij,nj->ni", h.M, h.r)
    return {"H_tt": np.einsum("nki,nkl,nlj->ij", h.J, h.M, h.J), "b_t": np.einsum("nki,nk->i", h.J, Mr), "error": float(np.einsum("ni,ni->", h.r, Mr)), "num_inliers": float(len(h))}


def adjoint_f32(T):
    """Ad = [[R, 0], [hat(t) R, R]] of the fp32-cast pose, as factor_epilogue forms it"""
    Tf = np.asarray(T, dtype=np.float32).astype(np.float64)
    R, t = Tf[:3, :3], Tf[:3, 3]
    Ad = np.zeros((6, 6))
    Ad[:3, :3] = Ad[3:, 3:] = R
    Ad[3:, :3] = synth.hat(t) @ R
    return Ad


def epilogue(H_tt, b_t, error, num_inliers, Ad):
    """factor_epilogue's record from the target-side sums (fp64)"""
    return {"H_tt": H_tt, "H_ss": Ad.T @ H_tt @ Ad, "H_ts": -H_tt @ Ad, "b_t": b_t, "b_s": -Ad.T @ b_t, "error": error, "num_inliers": num_inliers}


def hit_scale(h: Hits):
    """A and B of H_tt, b_t and the error (see above)"""
    if len(h) == 0:
        return {"H_tt": np.zeros((6, 6)), "b_t": np.zeros(6), "error": 0.0}, {"H_tt": np.zeros((6, 6)), "b_t": np.zeros(6), "error": 0.0}
    Ma = np.abs(h.M)
    dM = INV_ROUNDING * U32 * np.einsum("nij,njk,nkl->nil", Ma, np.abs(np.linalg.inv(h.M)), Ma)  # fp32 inverse: |M| |S| |M|
    Ja, ra = np.abs(h.J), np.abs(h.r)
    dJ = np.abs(_hat(h.dq))  # dJ = [-hat(dq) | 0]
    BH = np.einsum("nki,nkl,nlj->ij", dJ, Ma, Ja)  # rotation rows of |dJ|^T |M| |J|
    B_H = np.einsum("nki,nkl,nlj->ij", Ja, dM, Ja)
    B_H[:3, :] += BH
    B_H[:, :3] += BH.T
    A = {"H_tt": np.einsum("nki,nkl,nlj->ij", Ja, Ma, Ja), "b_t": np.einsum("nki,nkl,nl->i", Ja, Ma, ra), "error": float(np.einsum("nk,nkl,nl->", ra, Ma, ra))}
    B_b = np.einsum("nki,nkl,nl->i", Ja, dM, ra) + np.einsum("nki,nkl,nl->i", Ja, Ma, h.dq)
    B_b[:3] += np.einsum("nki,nkl,nl->i", dJ, Ma, ra)
    B = {"H_tt": B_H, "b_t": B_b, "error": float(np.einsum("nk,nkl,nl->", ra, dM, ra) + 2.0 * np.einsum("nk,nkl,nl->", ra, Ma, h.dq))}
    return A, B


def through_adjoint(part, Ad):
    """the scale of a whole record from that of its target-side sums, through |Ad| as the epilogue forms the source blocks"""
    P = np.abs(Ad)
    return {"H_tt": part["H_tt"], "H_ss": P.T @ part["H_tt"] @ P, "H_ts": part["H_tt"] @ P, "b_t": part["b_t"], "b_s": P.T @ part["b_t"], "error": part["error"]}


def record_scale(h: Hits) -> EntryScale:
    A, B = hit_scale(h)
    Ad = adjoint_f32(h.T)
    return EntryScale(through_adjoint(A, Ad), through_adjoint(B, Ad))


def check_entrywise(got: dict, ref, scale: EntryScale, tol=ENTRY_TOL, what=None):
    """|got_e - ref_e| <= tol A_e + B_e for every entry of H_tt, H_ss, H_ts, b_t, b_s and the error.  Prints and returns the
    largest ratio |got_e - ref_e| / (tol A_e + B_e)."""
    from oracle import oracle

    if not isinstance(ref, dict):
        ref = oracle.split122(ref)
    worst, where = 0.0, None
    for k in KEYS:
        d = np.abs(np.asarray(got[k], dtype=np.float64) - np.asarray(ref[k], dtype=np.float64)).ravel()
        bound = (tol * np.asarray(scale.A[k], dtype=np.float64) + np.asarray(scale.B[k], dtype=np.float64)).ravel()
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(bound > 0, d / np.where(bound > 0, bound, 1.0), np.where(d > 0, np.inf, 0.0))
        ratio = np.where(np.isnan(d), np.inf, ratio)
        i = int(np.argmax(ratio))
        entry = (k, tuple(int(x) for x in np.unravel_index(i, np.shape(got[k]))))
        if where is None or ratio[i] > worst:
            worst, where = float(ratio[i]), entry
        assert ratio[i] <= 1.0, (what, "entry-wise", entry, float(ratio[i]), float(d[i]), float(bound[i]))
    print(f"entry-wise {what if what is not None else ''}: max |got - ref| / bound = {worst:.3g} at {where}")
    return worst


def test_poses(T_gt, n=4, key=0):
    """Ground-truth delta and a handful of perturbed / adversarial deltas."""
    rng = synth.rng_for(99, key)
    poses = [T_gt]
    for _ in range(n):
        poses.append(synth.perturb(T_gt, rng, 0.01, 0.05))
    return poses


test_poses.__test__ = False


def cov_colmajor16(covs):
    n = covs.shape[0]
    return np.ascontiguousarray(np.swapaxes(covs.reshape(n, 4, 4), 1, 2)).reshape(n, 16)
