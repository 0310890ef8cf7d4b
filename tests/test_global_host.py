"""CPU-only checks of global registration (no GPU needed):
  * the FPFH restatement (tests/global_oracle.py) on its own properties: 11-bin blocks summing to 200, invariance under a rigid
    transform away from bin edges, hand-computed 3- and 4-point clouds, zero-distance and parallel-normal pairs;
  * the radius enumeration (grid_within of gb_grid_math.cuh, built here with g++) against the restatement and scipy's
    cKDTree.query_ball_point away from the bound;
  * the brute-force feature match against cKDTree in 33-D away from ties;
  * Horn's and the 4-DoF estimator on exact pairs, host-compiled and restated;
  * gb_global_math.cuh compiled for the host against the restatement: pair features and bins exactly, poses within 1e-12,
    sample indices and inlier counts exactly;
  * the selection rule, whatever the wave size;
  * host validation of the arguments the entry points reject before they touch a device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree

from glim_b200 import synth
from tests import global_oracle as gl
from tests import grid_oracle as go
from tests.test_grid_host import device_arrays

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def surface_cloud(n, rng):
    """points on three faces of a box and a sphere, with their exact normals: fp32 positions and normals"""
    k = n // 4
    u = rng.uniform(-2, 2, size=(k, 2))
    faces = [np.c_[u, np.full(k, -2.0)], np.c_[np.full(k, 2.0), u], np.c_[u[:, 0], np.full(k, 2.0), u[:, 1]]]
    normals = [np.tile([0, 0, 1.0], (k, 1)), np.tile([-1.0, 0, 0], (k, 1)), np.tile([0, -1.0, 0], (k, 1))]
    s = rng.normal(size=(n - 3 * k, 3))
    s /= np.linalg.norm(s, axis=1, keepdims=True)
    faces.append(s * 1.2 + [0.5, -0.3, 0.2])
    normals.append(s)
    return np.concatenate(faces).astype(F32), np.concatenate(normals).astype(F32)


@pytest.fixture(scope="module")
def gm(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("gm") / "libglobal_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so, os.path.join(ROOT, "tests", "cpp", "global_math_host.cpp")])
    L = C.CDLL(so)
    vp = C.c_void_p
    L.gm_pairs.argtypes = [C.c_int, vp, vp, vp, vp, vp, vp]
    L.gm_samples.argtypes = [C.c_uint64, C.c_int, C.c_int, C.c_int, vp]
    L.gm_pose.argtypes = [vp, vp, C.c_int, vp]
    L.gm_within.argtypes = [vp, C.c_uint, C.c_int, vp, vp, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, vp]
    L.gm_inliers.argtypes = [vp, C.c_int, vp, vp, C.c_uint, C.c_int, C.c_float]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_pose(L, a, b, dof):
    T = np.zeros(16)
    ok = L.gm_pose(_p(np.ascontiguousarray(a, dtype=np.float64)), _p(np.ascontiguousarray(b, dtype=np.float64)), dof, _p(T))
    return T.reshape(4, 4).T.copy() if ok else None


# ---------------------------------------------------------------------------------------------------------------------
# the FPFH restatement
# ---------------------------------------------------------------------------------------------------------------------
def test_blocks_sum_to_200_and_isolated_points_are_zero():
    rng = np.random.default_rng(1)
    xyz, nrm = surface_cloud(600, rng)
    xyz = np.concatenate([xyz, [[50.0, 50.0, 50.0]], [[np.nan, 0, 0]]]).astype(F32)
    nrm = np.concatenate([nrm, [[0, 0, 1]], [[0, 0, 1]]]).astype(F32)
    feat, spfh, _ = gl.fpfh(xyz, nrm, 0.6)
    nb = gl.neighbours(xyz, 0.6)
    has = np.array([len(x) > 0 for x in nb])
    assert has[:600].all() and not has[600:].any()
    sums = feat[has].reshape(-1, 3, 11).sum(2)
    assert np.allclose(sums, 200.0, rtol=0, atol=1e-9)
    assert np.allclose(spfh[has].reshape(-1, 3, 11).sum(2), 100.0, atol=1e-9)
    assert (feat[~has] == 0).all()


def test_features_are_invariant_under_a_rigid_transform():
    """Points and normals moved by a rigid transform (then rounded to fp32) give the same neighbourhoods and the same features
    (1e-4: the fp32 rounding of the moved positions) on every point whose margin to a bin edge exceeds 1e-5."""
    rng = np.random.default_rng(2)
    xyz, nrm = surface_cloud(500, rng)
    T = synth.pose(3.0, -7.0, 1.5, 2.1, 0.2, -0.1)
    x2 = (xyz.astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(F32)
    n2 = (nrm.astype(np.float64) @ T[:3, :3].T).astype(F32)
    r = 0.55
    nb1, nb2 = gl.neighbours(xyz, r), gl.neighbours(x2, r)
    d = np.linalg.norm(xyz[:, None, :].astype(np.float64) - xyz[None, :, :], axis=2)
    near_bound = (np.abs(d - r) < 1e-4).any(1)
    same = np.array([np.array_equal(a, b) for a, b in zip(nb1, nb2)])
    assert same[~near_bound].all()
    f1, _, m1 = gl.fpfh(xyz, nrm, r, nb1)
    f2, _, m2 = gl.fpfh(x2, n2, r, nb1)
    # a point is compared when neither it nor a neighbour sits near the bound, and every pair feature is off the bin edges
    affected = near_bound.copy()
    for i, nb in enumerate(nb1):
        affected[i] |= near_bound[nb].any() if len(nb) else False
    ok = ~affected & (np.minimum(m1, m2) > 1e-5)
    assert ok.sum() > 0.5 * len(xyz)
    assert np.allclose(f1[ok], f2[ok], rtol=1e-4, atol=1e-4)


def test_hand_computed_three_and_four_point_clouds():
    """Three points of a plane with a common normal: every pair feature is (0, 0, 0) (bins 5, 16, 27), SPFH = 100 there, FPFH =
    200 there.  A fourth point above with a sideways normal: the pairs' features as worked out by hand."""
    xyz = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], F32)
    nrm = np.array([[0, 0, 1]] * 3, F32)
    feat, spfh, _ = gl.fpfh(xyz, nrm, 1.5)
    want = np.zeros(33)
    want[[5, 16, 27]] = 100.0
    assert np.array_equal(spfh, np.tile(want, (3, 1)))
    assert np.allclose(feat, 2 * want, rtol=0, atol=1e-12)
    xyz4 = np.concatenate([xyz, [[0, 0, 1]]]).astype(F32)
    nrm4 = np.concatenate([nrm, [[1, 0, 0]]]).astype(F32)
    s = np.sqrt(0.5)
    f, _ = gl.pair_features(xyz4[[0, 3, 1, 3, 3]], nrm4[[0, 3, 1, 3, 3]], xyz4[[3, 0, 3, 1, 2]], nrm4[[3, 0, 3, 1, 2]])
    # (0,3), (3,0): v = d x n_s = 0 -> zero; (1,3), (3,1): f1 = -pi/2, f2 = 0, f3 = 1/sqrt 2; (3,2): swapped, f1 = 0, f2 = -1, f3 = 1/sqrt 2
    want_f = np.array([[0, 0, 0], [0, 0, 0], [-np.pi / 2, 0, s], [-np.pi / 2, 0, s], [0, -1, s]])
    assert np.allclose(f, want_f, rtol=0, atol=1e-7)
    _, spfh4, _ = gl.fpfh(xyz4, nrm4, 1.5)
    cnt = np.zeros(33)
    cnt[[5, 16, 27]] += 1           # (3, 0)
    cnt[[2, 16, 31]] += 1           # (3, 1)
    cnt[[5, 11, 31]] += 1           # (3, 2)
    assert np.allclose(spfh4[3], cnt * (100.0 / 3), rtol=0, atol=1e-12)


def test_zero_distance_and_parallel_normal_pairs():
    """A duplicated point and a pair whose normals are parallel to their offset give (0, 0, 0); the duplicate counts as a
    neighbour in the SPFH but is skipped by the distance weighting."""
    f, dd = gl.pair_features([[1, 2, 3], [0, 0, 0]], [[0, 0, 1], [1, 0, 0]], [[1, 2, 3], [2, 0, 0]], [[0, 1, 0], [1, 0, 0]])
    assert np.array_equal(f, np.zeros((2, 3))) and dd[0] == 0 and dd[1] == 4
    xyz = np.array([[0, 0, 0], [0, 0, 0], [0.3, 0, 0], [0, 0.3, 0]], F32)
    nrm = np.array([[0, 0, 1], [0, 0, 1], [0, 0, 1], [0.6, 0, 0.8]], F32)
    feat, spfh, _ = gl.fpfh(xyz, nrm, 1.0)
    assert np.allclose(spfh.reshape(4, 3, 11).sum(2), 100.0)
    assert np.allclose(feat.reshape(4, 3, 11).sum(2), 200.0)


# ---------------------------------------------------------------------------------------------------------------------
# the radius enumeration and the match
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("r", [0.4, 1.0])
def test_radius_enumeration_is_the_brute_force_set(gm, r):
    rng = np.random.default_rng(int(r * 10))
    xyz, _ = surface_cloud(1200, rng)
    xyz[::97] = np.nan
    g = go.PointGrid(xyz, np.zeros((len(xyz), 6), F32), 1.05 * r)
    thr = go.max_d2(r)
    m = go.half_width(g.inv, thr, g.key_extent)
    assert m == 1
    rec, cells, buckets = device_arrays(g)
    want = gl.neighbours(xyz, r)
    fin = np.isfinite(xyz).all(1)
    tree = cKDTree(xyz[fin].astype(np.float64))
    fin_idx = np.nonzero(fin)[0]
    d = np.linalg.norm(xyz[:, None, :].astype(np.float64) - xyz[None, fin, :], axis=2)
    out = np.empty(len(xyz), np.int32)
    for i in range(len(xyz)):
        q = xyz[i]
        k = gm.gm_within(_p(buckets), len(buckets) - 1, go.MAX_SCAN, _p(cells), _p(rec), m, g.inv, thr, float(q[0]), float(q[1]), float(q[2]), len(out), _p(out))
        got = np.sort(g.index[out[:k]])
        got = got[got != i]
        assert np.array_equal(got, want[i]), i
        if fin[i] and not (np.abs(d[i] - r) < 1e-5 * r).any():
            ball = np.sort(fin_idx[tree.query_ball_point(q.astype(np.float64), r)])
            assert np.array_equal(ball[ball != i], want[i]), i
        elif not fin[i]:
            assert len(want[i]) == 0


def test_match_is_the_exact_nearest_feature():
    rng = np.random.default_rng(5)
    t = (rng.random((700, 33)) * 20).astype(F32)
    s = (rng.random((300, 33)) * 20).astype(F32)
    s[:10] = t[[3, 9, 27, 81, 243, 5, 6, 7, 8, 100]]  # exact hits
    got = gl.match(t, s)
    dist, idx = cKDTree(t.astype(np.float64)).query(s.astype(np.float64), k=2)
    clear = (dist[:, 1] - dist[:, 0]) > 1e-4 * np.maximum(dist[:, 1], 1)
    assert clear.sum() > 250
    assert np.array_equal(got[clear], idx[clear, 0])
    # a planted tie goes to the smaller index
    t2 = np.concatenate([t, t[[50]]]).astype(F32)
    t2[[50]] = t[[50]]
    assert gl.match(t2, t[[50]])[0] == 50
    assert gl.match(t2[::-1].copy(), t[[50]])[0] == 0  # the copy, now first


# ---------------------------------------------------------------------------------------------------------------------
# the host-compiled arithmetic
# ---------------------------------------------------------------------------------------------------------------------
def random_pairs(rng, n):
    ps = rng.uniform(-5, 5, size=(n, 3))
    pt = ps + rng.normal(size=(n, 3))
    ns = rng.normal(size=(n, 3))
    nt = rng.normal(size=(n, 3))
    ns /= np.linalg.norm(ns, axis=1, keepdims=True)
    nt /= np.linalg.norm(nt, axis=1, keepdims=True)
    nt[:20] = ns[:20]                 # parallel normals
    pt[20:30] = ps[20:30]             # zero distance
    pt[30:40] = ps[30:40] + [0.0, 0.0, 1.5]  # n_s along the offset: v = 0
    ns[30:40] = [0.0, 0.0, 1.0]
    cast = lambda a: a.astype(F32).astype(np.float64)
    return cast(ps), cast(ns), cast(pt), cast(nt)


def test_host_build_pair_features_and_bins_equal_the_restatement(gm):
    rng = np.random.default_rng(11)
    n = 5000
    ps, ns, pt, nt = random_pairs(rng, n)
    f = np.empty((n, 3))
    b = np.empty((n, 3), np.int32)
    gm.gm_pairs(n, _p(ps), _p(ns), _p(pt), _p(nt), _p(f), _p(b))
    fr, _ = gl.pair_features(ps, ns, pt, nt)
    assert np.array_equal(f, fr)
    assert np.array_equal(b, gl.bins(fr))
    assert (f[20:30] == 0).all()


def test_samples_and_poses_equal_the_restatement(gm):
    s = np.empty((2000, 3), np.int32)
    gm.gm_samples(53123, 0, 2000, 30000, _p(s))
    assert all(list(s[h]) == gl.sample(53123, h, 30000) for h in range(0, 2000, 7))
    rng = np.random.default_rng(12)
    for dof in (4, 6):
        for k in range(200):
            a = rng.uniform(-20, 20, size=(3, 3))
            T = synth.pose(*rng.uniform(-30, 30, 3), rng.uniform(-np.pi, np.pi), *(rng.uniform(-0.2, 0.2, 2) if dof == 6 else (0, 0)))
            b = a @ T[:3, :3].T + T[:3, 3] + rng.normal(scale=0.05, size=(3, 3)) * (k % 2)
            Th, Tr = host_pose(gm, a, b, dof), gl.estimate_pose(a, b, dof)
            assert (Th is None) == (Tr is None)
            if Th is None:
                continue
            assert np.abs(Th - Tr).max() < 1e-12 * max(1.0, np.abs(Tr).max()), (dof, k)
            if k % 2 == 0:  # exact pairs: the known pose
                assert np.abs(Th - T).max() < 1e-12 * 40, (dof, k)
    # degenerate samples
    assert host_pose(gm, np.zeros((3, 3)), np.eye(3), 6) is None and gl.estimate_pose(np.zeros((3, 3)), np.eye(3), 6) is None
    line = np.array([[0, 0, 0], [1, 1, 1], [2, 2, 2.0]])
    assert host_pose(gm, line, np.eye(3), 4) is None and host_pose(gm, np.eye(3), line, 6) is None


def test_host_build_inlier_count_equals_the_restatement(gm):
    rng = np.random.default_rng(13)
    tgt, _ = surface_cloud(2000, rng)
    src = (tgt[rng.permutation(2000)[:800]] + rng.normal(scale=0.3, size=(800, 3))).astype(F32)
    src[::50] = np.nan
    g = go.PointGrid(tgt, np.zeros((2000, 6), F32), 0.5)
    _, _, buckets = device_arrays(g)
    occ = gl.occupancy(tgt, 0.5)
    for k in range(10):
        T = synth.pose(*rng.normal(scale=0.3, size=3), rng.normal(scale=0.2), *rng.normal(scale=0.05, size=2))
        Tc = np.ascontiguousarray(T.T.reshape(16))
        got = gm.gm_inliers(_p(Tc), len(src), _p(src), _p(buckets), len(buckets) - 1, go.MAX_SCAN, g.inv)
        assert got == gl.inliers(T, src, occ) > 0


def test_selection_does_not_depend_on_the_wave_size():
    rng = np.random.default_rng(14)
    for trial in range(50):
        H = int(rng.integers(1, 3000))
        counts = rng.integers(-1, 1000, size=H)
        counts[rng.random(H) < 0.3] = -1
        rate = float(rng.choice([0.5, 0.9, 0.99, 2.0]))
        ref = gl.select(counts, 1000, rate, H, wave=1)
        for w in (7, 64, gl.WAVE, H):
            got = gl.select(counts, 1000, rate, H, wave=w)
            assert got[:2] == ref[:2], (trial, w)
            if got[1] != gl.EARLY_STOP:
                assert got[2] == H
            else:
                assert got[0] < got[2] <= min(H, (got[0] // w + 1) * w)
    assert gl.select(np.full(10, -1), 100, 0.9, 10) == (-1, gl.DEGENERATE, 10)
    assert gl.select(np.zeros(10, int), 100, 0.9, 10) == (-1, gl.DEGENERATE, 10)


def test_invalid_arguments_are_rejected_on_the_host():
    """GB_ERR_INVALID_ARGUMENT before the call looks for a device."""
    from glim_b200 import capi, gpu

    L = capi.lib()
    dummy = C.c_void_p(1)  # never dereferenced: validation comes first
    for r in (0.0, -1.0, float("nan"), float("inf")):
        assert L.gb_cloud_estimate_fpfh(dummy, dummy, r) == 1, r
    assert L.gb_cloud_estimate_fpfh(None, None, 1.0) == 1
    assert L.gb_cloud_fpfh(None, None) == 1
    assert L.gb_fpfh_match(None, None, None, None) == 1
    res = capi.RansacResult()
    for bad in ({"max_iterations": 0}, {"early_stop_inlier_rate": 0.0}, {"early_stop_inlier_rate": float("nan")}, {"inlier_voxel_resolution": -1.0},
                {"inlier_voxel_resolution": float("inf")}, {"dof": 5}):
        p = gpu.ransac_params(**bad)
        assert L.gb_ransac_align(dummy, dummy, dummy, C.byref(p), C.byref(res), None) == 1, bad
    assert L.gb_ransac_align(dummy, dummy, dummy, None, C.byref(res), None) == 1
    p = capi.RansacParams()
    assert L.gb_ransac_default_params(C.byref(p)) == 0
    assert (p.max_iterations, p.early_stop_inlier_rate, p.inlier_voxel_resolution, p.dof, p.seed) == (5000, 0.9, 1.0, 4, 53123)
