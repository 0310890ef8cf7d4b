"""Records into tests/golden/reference_tu_golden.npz what GLIM's own translation units (oracle/_ref/libglim_ref.so, built by
`make -C oracle _ref REF=<GLIM source tree>`) compute on the inputs of tests/test_oracle_vs_reference_tu.py and test_cpp_shim.py.
Run from the repository root: python tests/golden/make_reference_tu_golden.py"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from glim_b200 import synth  # noqa: E402
from oracle import oracle  # noqa: E402
from tests import test_oracle_vs_reference_tu as T  # noqa: E402
from tests.test_deskew import IMU_P, IMU_T, T_IL, V, W, scan_like  # noqa: E402
from tests.test_oracle_vs_reference_tu import _p, ref_cov, ref_deskew_cv, ref_deskew_imu, ref_preprocess  # noqa: E402
from tests.util import scan_pair  # noqa: E402

SO = os.path.join(ROOT, "oracle", "_ref", "libglim_ref.so")


def load():
    L = C.CDLL(SO)
    vp, i32 = C.c_void_p, C.c_int
    L.ref_covariance_estimate.argtypes = [i32, vp, vp, i32, i32, i32, vp, vp]
    L.ref_covariance_estimate_sample.argtypes = [i32, vp, vp, i32, i32, vp]
    L.ref_deskew_const_vel.argtypes = [vp, vp, vp, i32, vp, vp, vp]
    L.ref_deskew_imu.argtypes = [vp, i32, vp, vp, C.c_double, i32, vp, vp, vp]
    L.ref_shim_slerp.argtypes = [vp, vp, C.c_double, vp]
    return L


def record_preprocess(L, g, key, P, Tm, intensities=None, **kw):
    pts, tms, _, nb, end, seen = ref_preprocess(L, P, Tm, intensities=intensities, **kw)
    g[f"{key}/n"] = len(pts)
    g[f"{key}/end"] = end
    g[f"{key}/seen"] = np.array(seen)
    g[f"{key}/tms"] = T.digest(tms)
    g[f"{key}/tms_all_zero"] = bool(np.all(tms == 0.0))
    g[f"{key}/canonical"] = np.array([T.digest(a) for a in T.canonical(pts, tms, nb)])
    g[f"{key}/points_sorted"] = T.digest(pts[np.lexsort(pts[:, :3].T)])


def main():
    L = load()
    g = {}
    # covariance estimation (test_covariance_oracle_equals_reference_translation_unit, test_plane_regularization_...)
    sp = scan_pair()
    for c, ks in ((0, (10, 5)), (1, (None,))):
        pts = sp["points"][c]
        nb = synth.knn(pts, 10).astype(np.int32)
        rows = T.sample_rows(len(pts))
        for k in ks:
            nr, cr = ref_cov(L, pts, nb, k)
            g[f"cov{c}_k{k or 10}/normals"], g[f"cov{c}_k{k or 10}/covs"] = nr[rows], cr[rows]
        if c == 1:
            c_smp = np.zeros((len(pts), 16))
            L.ref_covariance_estimate_sample(len(pts), _p(np.ascontiguousarray(pts)), _p(nb), 10, 10, _p(c_smp))
            g["cov1_sample/covs"] = c_smp.reshape(-1, 4, 4).transpose(0, 2, 1)[rows]
    # deskewing: the scans of test_deskew_oracle_equals_reference_translation_unit (seed 3), the product's pose table (seed 4) and
    # the CloudDeskewing shim's host half in tests/test_cpp_shim.py (seed 7, 5000 points)
    for seed, n in ((3, 20000), (4, 20000), (7, 5000)):
        times, pts = scan_like(n=n, seed=seed)
        rows = T.sample_rows(n)
        for name, (v, w) in T.CONST_VEL_CASES.items():
            g[f"deskew{seed}/cv_{name}"] = ref_deskew_cv(L, T_IL, v, w, times, pts)[rows]
        for name, (dt, m) in T.IMU_CASES.items():
            g[f"deskew{seed}/imu_{name}"] = ref_deskew_imu(L, T_IL, IMU_T[:m] + dt, IMU_P[:m], 100.0, times, pts)[rows]
    # CloudPreprocessor::preprocess
    P, Tm = T.make_frame()
    lo, hi = T.CROP_LO, T.CROP_HI
    for name, (rkw, _) in T.preprocess_cases().items():
        record_preprocess(L, g, f"pre_{name}", P, Tm, **rkw)
    record_preprocess(L, g, "pre_randomgrid", P, Tm, use_random_grid_downsampling=1, downsample_resolution=1.0, downsample_target=T.RANDOM_TARGET, seed=5)
    record_preprocess(L, g, "pre_global_shutter", P, Tm, intensities=T.intensities(P), global_shutter=1)
    # every time is 0 under global shutter: order the reference's points by the ORIGINAL times, as the oracle's frame is ordered
    pts, _, it, _, _, _ = ref_preprocess(L, P, Tm, intensities=T.intensities(P), global_shutter=1)
    _, o_tms, _ = T.global_shutter_oracle(P, Tm)
    got = T.canonical(pts, o_tms, np.zeros((len(pts), 1), np.int64), it)
    g["pre_global_shutter/shutter_canonical"] = np.array([T.digest(got[0]), T.digest(got[3])])
    record_preprocess(L, g, "pre_imu_crop", P, Tm, crop_bbox_frame=2, crop_bbox_min=lo, crop_bbox_max=hi, T_imu_lidar=T.T_IMU_CROP)
    # the stand-ins' own primitives, on the inputs test_stand_in_primitives_* draw (same generators, same order)
    rng = np.random.default_rng(11)
    vals, vecs = np.zeros((400, 3)), np.zeros((400, 9))
    for trial in range(400):
        Q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        w = np.sort(rng.uniform(1e-4, 5.0, 3))
        if trial % 5 == 0:
            w[0] = w[1] * 1e-6
        A = (Q * w) @ Q.T
        A = 0.5 * (A + A.T) * rng.choice([1e-3, 1.0, 1e3])
        L.ref_shim_eigen_sym3(_p(np.ascontiguousarray(A.T.reshape(9))), _p(vals[trial]), _p(vecs[trial]))
    g["eigen/vals"], g["eigen/vecs"] = vals, vecs
    from scipy.spatial.transform import Rotation as Rot

    rng = np.random.default_rng(12)
    g["slerp/out"], g["expmap/out"] = np.zeros((200, 9)), np.zeros((200, 16))
    for trial in range(200):
        r0, r1 = Rot.from_rotvec(rng.normal(size=3) * rng.uniform(0, 2.5)), Rot.from_rotvec(rng.normal(size=3) * rng.uniform(0, 2.5))
        t = float(rng.uniform(0, 1))
        L.ref_shim_slerp(_p(np.ascontiguousarray(r0.as_matrix().T.reshape(9))), _p(np.ascontiguousarray(r1.as_matrix().T.reshape(9))), t, _p(g["slerp/out"][trial]))
    for trial in range(200):
        xi = np.concatenate([rng.normal(size=3) * rng.choice([0.0, 1e-9, 0.3, 2.0]), rng.normal(size=3) * 3.0])
        L.ref_shim_pose3_expmap(_p(xi), _p(g["expmap/out"][trial]))
    np.savez_compressed(T.GOLDEN, **g)
    print(f"wrote {T.GOLDEN}: {len(g)} arrays")


if __name__ == "__main__":
    main()
