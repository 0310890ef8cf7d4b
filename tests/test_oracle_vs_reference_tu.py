"""The oracle (and the product's host halves) against the reference's OWN translation units.

tests/golden/reference_tu_golden.npz = what GLIM's cloud_covariance_estimation.cpp, cloud_deskewing.cpp and cloud_preprocessor.cpp
compute, compiled UNMODIFIED against the stand-in headers of oracle/ref_shim/ (recipe: `make -C oracle _ref`; Eigen, GTSAM,
spdlog and gtsam_points are not installed here, the stand-ins are written in this repository).  What that pins: the control flow
and formulas of those two files -- neighbour indexing, population covariance, the PLANE regularization constants, (3,3) = 0, the
normal's flip towards the sensor, the 0.1 ms time table, the IMU cursor / clamp / held-last-pose rules, the composition order of the
transforms.  What it does not: Eigen's and GTSAM's own arithmetic (direct 3x3 eigen-solver, quaternion slerp, Pose3::Expmap), which
the stand-ins restate from the published algorithms.  The VGICP factor itself lives in gtsam_points and stays unpinned.

Recorded by tests/golden/make_reference_tu_golden.py: per-point outputs for a fixed, seeded sample of rows, exact ones as digests."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

from glim_b200 import synth
from oracle import oracle
from tests.test_deskew import IMU_P, IMU_T, T_IL, V, W, scan_like
from tests.util import scan_pair

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_tu_golden.npz")

CONST_VEL_CASES = {"vw": (V, W), "v": (V, np.zeros(3)), "w": (np.zeros(3), W), "none": (np.zeros(3), np.zeros(3))}
# (shift of the IMU times, number of IMU poses): all of them; poses that end before the scan does; a scan that starts before them
IMU_CASES = {"full": (0.0, len(IMU_T)), "short": (0.0, 6), "late": (0.05, len(IMU_T))}
CROP_LO, CROP_HI = np.array([-3.0, -2.0, -5.0]), np.array([4.0, 2.5, 5.0])
T_IMU_CROP = synth.pose(0.5, -0.2, 0.1, 0.4, 0.0, 0.0)
RANDOM_TARGET = 2000


@pytest.fixture(scope="module")
def ref():
    with np.load(GOLDEN) as g:
        return {k: g[k] for k in g.files}


def sample_rows(n, k=256):
    """the rows of an n-point output that the golden file keeps"""
    return np.sort(np.random.default_rng(20240).choice(n, min(k, n), replace=False))


def digest(a):
    """SHA-256 of an array's shape and values (as fp64 with -0.0 -> 0.0, or int64): equal digests <=> np.array_equal"""
    a = np.ascontiguousarray(a)
    a = a.astype(np.float64) + 0.0 if a.dtype.kind == "f" else a.astype(np.int64)
    return hashlib.sha256(repr(a.shape).encode() + a.tobytes()).hexdigest()


# the calls into oracle/_ref/libglim_ref.so whose results tests/golden/make_reference_tu_golden.py records
def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def ref_cov(L, pts, nb, k=None, threads=2):
    n, kc = nb.shape
    k = kc if k is None else k
    pts = np.ascontiguousarray(pts, np.float64)
    nb = np.ascontiguousarray(nb, np.int32)
    normals, covs = np.zeros((n, 4)), np.zeros((n, 16))
    L.ref_covariance_estimate(n, _p(pts), _p(nb), kc, k, threads, _p(normals), _p(covs))
    return normals, covs.reshape(n, 4, 4).transpose(0, 2, 1).copy()


def well_conditioned(pts, nb, k, rel_gap=1e-3):
    """neighbourhoods whose smallest eigenvalue is separated (SURVEY C.4): the eigenvector is then unique up to sign, and two
    solvers agree to ~1e-13 / rel_gap (the covariance itself carries ~1e-13 of cancellation error at 40 m range)"""
    P = pts[nb[:, :k], :3]
    c = np.einsum("nki,nkj->nij", P - P.mean(1, keepdims=True), P - P.mean(1, keepdims=True)) / k
    w = np.linalg.eigvalsh(c)
    return (w[:, 1] - w[:, 0]) > rel_gap * np.maximum(w[:, 2], 1e-300)


@pytest.mark.parametrize("k", [10, 5])
def test_covariance_oracle_equals_reference_translation_unit(ref, k):
    sp = scan_pair()
    pts = sp["points"][0]
    nb = synth.knn(pts, 10).astype(np.int32)
    rows = sample_rows(len(pts))
    n_ref, c_ref = ref[f"cov0_k{k}/normals"], ref[f"cov0_k{k}/covs"]
    n_orc, c_orc = oracle.covariance_estimate(pts, nb, k_neighbors=k, num_threads=2)
    n_orc, c_orc = n_orc[rows], c_orc[rows]
    assert well_conditioned(pts, nb, k).mean() > 0.9
    ok = well_conditioned(pts, nb, k)[rows]
    assert np.abs(c_ref[ok] - c_orc[ok]).max() < 1e-10
    assert np.abs(n_ref[ok] - n_orc[ok]).max() < 1e-10  # same sign: both flip towards the sensor origin
    loose = well_conditioned(pts, nb, k, 1e-6)[rows]     # nearly isotropic in the plane's normal direction: 1e-13 / gap
    assert np.abs(c_ref[loose] - c_orc[loose]).max() < 1e-6
    # invariants the reference file enforces on EVERY point, conditioned or not
    for c, nr, p in ((c_ref, n_ref, pts[rows]), (c_orc, n_orc, pts[rows])):
        assert np.all(c[:, 3, :] == 0) and np.all(c[:, :, 3] == 0) and np.all(nr[:, 3] == 0)
        assert np.all(np.einsum("ni,ni->n", p, nr) <= 1e-12)
        assert np.allclose(np.linalg.eigvalsh(c[:, :3, :3]), [1e-3, 1.0, 1.0], atol=1e-9)


def test_plane_regularization_makes_the_divisor_irrelevant(ref):
    """SURVEY C.4: the (points, neighbors, k) overload divides by k - 1 (cloud_covariance_estimation.cpp:153) -- irrelevant under
    PLANE because only the eigenvectors survive.  Checked on the reference code's own results."""
    sp = scan_pair()
    pts = sp["points"][1]
    nb = synth.knn(pts, 10).astype(np.int32)
    c_pop, c_smp = ref["cov1_k10/covs"], ref["cov1_sample/covs"]
    ok = well_conditioned(pts, nb, 10)[sample_rows(len(pts))]
    assert ok.mean() > 0.9
    assert np.abs(c_pop[ok] - c_smp[ok]).max() < 1e-9


def ref_deskew(ref, seed, times):
    """the reference's deskewed points of the scan_like(seed) scan: {case: sampled rows}, and the rows"""
    return {k.split("/", 1)[1]: v for k, v in ref.items() if k.startswith(f"deskew{seed}/")}, sample_rows(len(times))


def imu_case(name):
    dt, m = IMU_CASES[name]
    return IMU_T[:m] + dt, IMU_P[:m]


def ref_deskew_cv(L, T, v, w, times, pts):
    out = np.empty_like(pts)
    L.ref_deskew_const_vel(_p(oracle.pose_colmajor(T)), _p(np.asarray(v, np.float64)), _p(np.asarray(w, np.float64)), len(times), _p(times), _p(pts), _p(out))
    return out


def ref_deskew_imu(L, T, imu_t, imu_p, stamp, times, pts):
    out = np.empty_like(pts)
    poses = np.ascontiguousarray(np.swapaxes(np.asarray(imu_p, np.float64).reshape(-1, 4, 4), 1, 2)).reshape(-1, 16)
    imu_t = np.ascontiguousarray(imu_t, np.float64)
    L.ref_deskew_imu(_p(oracle.pose_colmajor(T)), len(imu_t), _p(imu_t), _p(poses), float(stamp), len(times), _p(times), _p(pts), _p(out))
    return out


def test_deskew_oracle_equals_reference_translation_unit(ref):
    times, pts = scan_like(seed=3)
    got, rows = ref_deskew(ref, 3, times)
    for name, (v, w) in CONST_VEL_CASES.items():
        assert np.abs(got[f"cv_{name}"] - oracle.deskew_const_vel(T_IL, v, w, times, pts)[rows]).max() < 1e-11
    # "short": IMU poses that end before the scan does: the last pose is held (cloud_deskewing.cpp:104-105);
    # "late": a scan that starts before the first IMU pose: p is clamped to 0 (:111)
    for name in IMU_CASES:
        it, ip = imu_case(name)
        assert np.abs(got[f"imu_{name}"] - oracle.deskew_imu(T_IL, it, ip, 100.0, times, pts)[rows]).max() < 1e-11


def test_product_host_pose_table_equals_reference_translation_unit(ref):
    """gb_deskew_pose_table (the product's host half, no device needed) applied in numpy == the reference's deskewed points"""
    from glim_b200 import preprocess

    times, pts = scan_like(seed=4)
    got, rows = ref_deskew(ref, 4, times)
    idx, Ts = preprocess.deskew_pose_table(T_IL, times, linear_vel=V, angular_vel=W)
    assert np.abs(np.einsum("nij,nj->ni", Ts[idx], pts)[rows] - got["cv_vw"]).max() < 1e-11
    idx, Ts = preprocess.deskew_pose_table(T_IL, times, imu_times=IMU_T, imu_poses=IMU_P, stamp=100.0)
    assert np.abs(np.einsum("nij,nj->ni", Ts[idx], pts)[rows] - got["imu_full"]).max() < 1e-11


# ------------------------------------------------------------------------------------------------------------------------
# CloudPreprocessor::preprocess: the reference's cloud_preprocessor.cpp, compiled unmodified.  Its gtsam_points leaf calls
# (voxelgrid_sampling, randomgrid_sampling, sample, filter, remove_outliers, KdTree) are [EXT] and resolve to stand-ins that forward to
# the oracle's leaves -- so what this checks is the reference file's OWN logic against the composition the GPU parity tests use as
# their oracle (`_cpu_frame` in tests/test_gpu_parity.py): which stage runs when, the finite / range gates, the sort key, global
# shutter, the crop box in either frame, where outlier removal sits, scan_end_time, the k-NN layout and its self-fill.
# ------------------------------------------------------------------------------------------------------------------------
class RefParams(C.Structure):
    _fields_ = [("distance_near_thresh", C.c_double), ("distance_far_thresh", C.c_double), ("use_random_grid_downsampling", C.c_int), ("downsample_resolution", C.c_double),
                ("downsample_target", C.c_int), ("downsample_rate", C.c_double), ("seed", C.c_ulonglong), ("global_shutter", C.c_int), ("crop_bbox_frame", C.c_int),
                ("crop_bbox_min", C.c_double * 3), ("crop_bbox_max", C.c_double * 3), ("T_imu_lidar", C.c_double * 16), ("enable_outlier_removal", C.c_int),
                ("outlier_removal_k", C.c_int), ("outlier_std_mul_factor", C.c_double), ("k_correspondences", C.c_int), ("num_threads", C.c_int)]


def ref_preprocess(L, P, T, stamp=10.0, intensities=None, **kw):
    par = RefParams(distance_near_thresh=1.0, distance_far_thresh=60.0, use_random_grid_downsampling=0, downsample_resolution=0.2, downsample_target=0, downsample_rate=0.3,
                    seed=5, global_shutter=0, crop_bbox_frame=0, enable_outlier_removal=0, outlier_removal_k=10, outlier_std_mul_factor=1.0, k_correspondences=10, num_threads=2)
    par.T_imu_lidar = (C.c_double * 16)(*oracle.pose_colmajor(np.eye(4)))
    for k, v in kw.items():
        if k in ("crop_bbox_min", "crop_bbox_max"):
            v = (C.c_double * 3)(*v)
        elif k == "T_imu_lidar":
            v = (C.c_double * 16)(*oracle.pose_colmajor(v))
        setattr(par, k, v)
    n = len(P)
    P, T = np.ascontiguousarray(P, np.float64), np.ascontiguousarray(T, np.float64)
    op, ot, oi, nb = np.zeros((n, 4)), np.zeros(n), np.zeros(n), np.zeros((n, par.k_correspondences), np.int32)
    end, seen = C.c_double(), (C.c_double * 6)()
    L.ref_preprocess.restype = C.c_int
    L.ref_preprocess.argtypes = [C.c_void_p, C.c_double, C.c_int] + [C.c_void_p] * 9
    it = np.ascontiguousarray(intensities, np.float64) if intensities is not None else None
    m = L.ref_preprocess(C.byref(par), stamp, n, _p(P), _p(T), _p(it) if it is not None else None, _p(op), _p(ot), _p(oi), _p(nb), C.byref(end), seen)
    return op[:m], ot[:m], oi[:m], nb[:m], end.value, list(seen)


def make_frame():
    sc = synth.make_hall_scene()
    P, T = synth.scan(sc, "hdl32", synth.arc_trajectory(8)[2], synth.rng_for(41), n_rays=32 * 250)
    P = P.copy()
    P[17, 1] = np.nan  # dropped by the finite gate (cloud_preprocessor.cpp:123)
    return P, T


def intensities(P):
    return np.linspace(0.0, 1.0, len(P))


def preprocess_cases():
    """{name: (reference parameters, oracle composition arguments)}"""
    return {
        "voxelgrid": (dict(), dict()),
        "cropbox lidar": (dict(crop_bbox_frame=1, crop_bbox_min=CROP_LO, crop_bbox_max=CROP_HI), dict(crop=(CROP_LO, CROP_HI))),
        "outliers": (dict(enable_outlier_removal=1, outlier_removal_k=8, outlier_std_mul_factor=1.0), dict(sor=(8, 1.0))),
    }


@pytest.fixture(scope="module")
def frame():
    return make_frame()


def canonical(pts, tms, nb, extra=None):
    """The reference orders by time with std::sort (NOT stable: the order of equal times is unspecified, SURVEY C.1) and the 32
    rings of a firing share a timestamp, so frames are compared modulo the order inside a group of equal times: rows sorted by
    (time, x, y, z), neighbour indices renumbered accordingly, every neighbour row as a sorted set."""
    perm = np.lexsort((pts[:, 2], pts[:, 1], pts[:, 0], tms))
    inv = np.empty(len(perm), np.int64)
    inv[perm] = np.arange(len(perm))
    out = [pts[perm], tms[perm], np.sort(inv[nb[perm]], axis=1)]
    if extra is not None:
        out.append(extra[perm])
    return out


def test_preprocess_composition_equals_reference_translation_unit(ref, frame):
    from tests.test_gpu_parity import _cpu_frame

    P, T = frame
    for name, (_, okw) in preprocess_cases().items():
        g = f"pre_{name}/"
        o_pts, o_tms, o_nb, _, _ = _cpu_frame(P, T, 0.2, 1.0, 60.0, 10, **okw)
        assert ref[g + "n"] == len(o_pts) > 1000, name
        assert ref[g + "tms"] == digest(o_tms), name  # the sequence of times is order-free
        assert list(ref[g + "canonical"]) == [digest(a) for a in canonical(o_pts, o_tms, o_nb)], name
        assert ref[g + "end"] == 10.0 + o_tms[-1], name
    # the code defaults of CloudPreprocessorParams (cloud_preprocessor.cpp:27-36,58) as the product's gb_preprocess_default_params
    # documents them next to the shipped config
    assert list(ref["pre_voxelgrid/seen"]) == [1.0, 100.0, 0.15, 0.3, 2.0, 8.0]
    # random grid: rate = target / N (cloud_preprocessor.cpp:105), survivors keep their order, then the same gates
    mask = oracle.randomgrid_sampling(P, 1.0, RANDOM_TARGET / len(P), seed=5)
    o_pts, o_tms, o_nb, _, _ = _cpu_frame(P, T, None, 1.0, 60.0, 10, mask=mask)
    assert ref["pre_randomgrid/n"] == len(o_pts) > 500
    assert list(ref["pre_randomgrid/canonical"]) == [digest(a) for a in canonical(o_pts, o_tms, o_nb)]


def global_shutter_oracle(P, T):
    """the oracle's voxel grid + gates of the global-shutter frame, ordered by the ORIGINAL times: (points, times, intensities)"""
    o_pts, o_tms, o_it = oracle.voxelgrid_sampling(P, 0.2, times=T, intensities=intensities(P))
    sq = (o_pts[:, :3] ** 2).sum(1)
    keep = np.nonzero((sq > 1.0) & (sq < 3600.0) & np.isfinite(o_pts).all(1))[0]
    keep = keep[np.argsort(o_tms[keep], kind="stable")]
    return o_pts[keep], o_tms[keep], o_it[keep]


def test_preprocess_global_shutter_intensities_and_imu_crop_box(ref, frame):
    P, T = frame
    # global shutter: the points are still ordered by their ORIGINAL times, then every time becomes 0 (:135-140) -> scan_end_time = stamp
    o_pts, o_tms, o_it = global_shutter_oracle(P, T)
    assert ref["pre_global_shutter/tms_all_zero"] and ref["pre_global_shutter/end"] == 10.0
    zero_nb = np.zeros((len(o_pts), 1), np.int64)
    want = canonical(o_pts, o_tms, zero_nb, o_it)
    got = ref["pre_global_shutter/shutter_canonical"]  # the reference's points / intensities, ordered by the oracle's original times
    assert got[0] == digest(want[0]) and got[1] == digest(want[3])  # intensities travel with the points
    # crop box given in the IMU frame: p_imu = T_imu_lidar * p_lidar (:152-157); points INSIDE the box are removed
    p_imu = o_pts[:, :3] @ T_IMU_CROP[:3, :3].T + T_IMU_CROP[:3, 3]
    inside = (p_imu >= CROP_LO).all(1) & (p_imu <= CROP_HI).all(1)
    assert 0 < inside.sum() < len(o_pts)
    kept = o_pts[~inside]
    assert ref["pre_imu_crop/points_sorted"] == digest(kept[np.lexsort(kept[:, :3].T)])


# ------------------------------------------------------------------------------------------------------------------------
# The stand-ins are restatements too: check the three non-trivial ones against independent implementations, so that "the reference
# file compiled against a stand-in" cannot hide a wrong stand-in.
# ------------------------------------------------------------------------------------------------------------------------
def test_stand_in_primitives_eigen_solver(ref):
    rng = np.random.default_rng(11)
    worst = 0.0
    for trial in range(400):
        Q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        w = np.sort(rng.uniform(1e-4, 5.0, 3))
        if trial % 5 == 0:
            w[0] = w[1] * 1e-6  # a flat neighbourhood: smallest eigenvalue far below the others
        A = (Q * w) @ Q.T
        A = 0.5 * (A + A.T) * rng.choice([1e-3, 1.0, 1e3])
        vals, vecs = ref["eigen/vals"][trial], ref["eigen/vecs"][trial]
        V = vecs.reshape(3, 3).T
        ew, eV = np.linalg.eigh(A)
        scale = np.abs(ew).max()
        assert np.all(np.diff(vals) >= -1e-12 * scale)  # ascending, like Eigen
        assert np.abs(vals - ew).max() < 1e-9 * scale
        assert np.abs(V.T @ V - np.eye(3)).max() < 1e-9 and np.linalg.det(V) > 0  # orthonormal, right-handed (col1 = col2 x col0)
        gap = np.min(np.diff(ew)) / scale
        if gap > 1e-3:
            err = max(min(np.abs(V[:, k] - eV[:, k]).max(), np.abs(V[:, k] + eV[:, k]).max()) for k in range(3))
            worst = max(worst, err)
    assert worst < 1e-9


def test_stand_in_primitives_slerp_and_expmap(ref):
    from scipy.spatial.transform import Rotation as Rot, Slerp

    rng = np.random.default_rng(12)
    for trial in range(200):
        r0, r1 = Rot.from_rotvec(rng.normal(size=3) * rng.uniform(0, 2.5)), Rot.from_rotvec(rng.normal(size=3) * rng.uniform(0, 2.5))
        t = float(rng.uniform(0, 1))
        out = ref["slerp/out"][trial]
        want = Slerp([0, 1], Rot.from_matrix([r0.as_matrix(), r1.as_matrix()]))([t])[0].as_matrix()
        assert np.abs(out.reshape(3, 3).T - want).max() < 1e-12
    for trial in range(200):
        xi = np.concatenate([rng.normal(size=3) * rng.choice([0.0, 1e-9, 0.3, 2.0]), rng.normal(size=3) * 3.0])
        T = ref["expmap/out"][trial]
        assert np.abs(T.reshape(4, 4).T - synth.se3_exp(xi)).max() < 1e-12  # synth.se3_exp: the closed form with the V(omega) matrix
