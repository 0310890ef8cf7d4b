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


def check_linearized(got: dict, ref, tol=REL_TOL):
    """A device record (unpacked) against a reference: a 122-double oracle record or a dict of blocks indexed [row, col].
    Inlier count exact; Hessians, gradients and error within `tol` relative of the reference (a factor without inliers: zeros)."""
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
