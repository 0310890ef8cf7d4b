"""Global registration on the H100 (gb_cloud_estimate_fpfh, gb_fpfh_match, gb_ransac_align): the device features against the
numpy restatement (tests/global_oracle.py), the match bit for bit against the numpy float32 brute force, every RANSAC hypothesis
count and the selection against the restatement fed the host-compiled poses, GLIM's manual loop-closure recipe end to end, the
refusals and the launch counts."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from glim_b200 import capi, gpu, preprocess, synth
from tests import global_oracle as gl
from tests import voxelmap_oracle as vo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def pose_error(T, T_ref):
    d = synth.inv_pose(T_ref) @ T
    return float(np.linalg.norm(d[:3, 3])), float(np.degrees(np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1))))


@pytest.fixture(scope="module")
def frames():
    return vo.arc_frames(4, 32 * 150, nan_frame=1)


def cloud_of(ctx, frame, extra=None):
    """a device cloud of a frame with normals and covariances (and the host arrays it was made from)"""
    pts = frame[0]
    nrm, cov = synth.with_covariances(np.nan_to_num(pts, nan=1e4), 10)
    if extra is not None:
        pts = np.concatenate([pts, extra[0]])
        nrm = np.concatenate([nrm, extra[1]])
        cov = np.concatenate([cov, np.tile(np.eye(4) * 1e-3, (len(extra[0]), 1, 1))])
    return gpu.PointCloudGPU.clone(pts, cov, nrm, ctx=ctx), pts, nrm


@pytest.mark.parametrize("radius", [0.8, 2.0])
def test_features_match_the_restatement(ctx, frames, radius):
    """A frame with NaN points, plus an isolated point and a point of another frame: the device features equal the restatement within
    1e-5 relative on every point whose pair features (its own and its neighbours') lie more than 1e-9 from a bin edge; the NaN
    and isolated points are zero; a second call replaces the features."""
    isolated = (np.array([[500.0, 500.0, 500.0, 1.0], frames[0][0][10]]), np.array([[0, 0, 1.0, 0], [0, 0, 1.0, 0]]))
    cloud, pts, nrm = cloud_of(ctx, frames[1], isolated)
    cloud.estimate_fpfh(5.0).estimate_fpfh(radius)
    got = cloud.fpfh()
    xyz, _ = cloud.download()
    ref, _, margin = gl.fpfh(xyz, nrm.astype(F32), radius)
    ok = margin > 1e-9
    assert ok.mean() > 0.95
    assert np.allclose(got[ok], ref[ok], rtol=1e-5, atol=1e-4)
    nan = ~np.isfinite(xyz).all(1)
    assert nan.sum() > 0 and (got[nan] == 0).all() and (got[-2] == 0).all()
    has = np.abs(ref).sum(1) > 0
    assert np.allclose(got[has].reshape(-1, 3, 11).sum(2), 200.0, rtol=1e-5)


def test_match_is_bit_exact_with_a_planted_tie(ctx, frames):
    """gb_fpfh_match equals the numpy float32 brute force bit for bit.  The target holds one point twice (same position and
    normal: equal features), so the source copy of that point ties and must get the smaller index."""
    t_pts = np.concatenate([frames[2][0], frames[2][0][[100]]])
    t_nrm, t_cov = synth.with_covariances(np.nan_to_num(t_pts, nan=1e4), 10)
    t_nrm[-1] = t_nrm[100]
    tgt = gpu.PointCloudGPU.clone(t_pts, t_cov, t_nrm, ctx=ctx).estimate_fpfh(1.5)
    src, _, _ = cloud_of(ctx, frames[3])
    src.estimate_fpfh(1.5)
    ft, fs = tgt.fpfh(), src.fpfh()
    assert np.array_equal(ft[100], ft[-1])
    for a, b in ((tgt, src), (src, tgt), (tgt, tgt)):
        got = gpu.fpfh_match(a, b)
        assert np.array_equal(got, gl.match(a.fpfh(), b.fpfh()))
    assert gpu.fpfh_match(tgt, tgt)[-1] == 100


@pytest.fixture(scope="module")
def gm(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("gm") / "libglobal_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "cpp", "global_math_host.cpp")])
    L = C.CDLL(so)
    L.gm_pose.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    return L


@pytest.fixture(scope="module")
def small_problem(ctx, frames):
    """frame 2 as the target, 1500 points of frame 3 moved by a known pose as the source, features at r = 1.5"""
    tgt, t_pts, _ = cloud_of(ctx, frames[2])
    T_gt = synth.pose(4.0, -3.0, 0.2, np.radians(100), 0.02, -0.01)
    fin = np.isfinite(frames[3][0]).all(1)
    keep = np.nonzero(fin)[0][:: max(1, fin.sum() // 1500)]
    p = frames[3][0][keep].copy()
    p[:, :3] = (p[:, :3] - T_gt[:3, 3]) @ T_gt[:3, :3]
    nrm, cov = synth.with_covariances(p, 10)
    src = gpu.PointCloudGPU.clone(p, cov, nrm, ctx=ctx)
    tgt.estimate_fpfh(1.5)
    src.estimate_fpfh(1.5)
    return tgt, src, T_gt


@pytest.mark.parametrize("dof", [4, 6])
@pytest.mark.parametrize("rate", [0.3, 2.0])
def test_ransac_counts_and_selection_match_the_restatement(ctx, gm, small_problem, dof, rate):
    """Every evaluated hypothesis's count equals the restatement's with the host-compiled pose (-1 for the same invalid samples),
    and best_hypothesis, evaluated and status equal the selection rule's; without early stop (rate 2) every hypothesis is
    evaluated."""
    tgt, src, _ = small_problem
    H = 1200
    res = gpu.estimate_pose_ransac(tgt, src, hypothesis_inliers=True, max_iterations=H, early_stop_inlier_rate=rate, dof=dof, seed=77)
    counts = res["hypothesis_inliers"]
    nearest = gpu.fpfh_match(tgt, src)
    sx, _ = src.download()
    tx, _ = tgt.download()
    occ = gl.occupancy(tx, 1.0)
    ref = np.full(H, -2)
    for h in range(res["evaluated"]):
        s = gl.sample(77, h, len(sx))
        if len(set(s)) < 3 or min(nearest[j] for j in s) < 0:
            ref[h] = -1
            continue
        a = sx[s].astype(np.float64)
        b = tx[[nearest[j] for j in s]].astype(np.float64)
        T = np.zeros(16)
        if not gm.gm_pose(capi.ptr(np.ascontiguousarray(a)), capi.ptr(np.ascontiguousarray(b)), dof, capi.ptr(T)):
            ref[h] = -1
            continue
        ref[h] = gl.inliers(T.reshape(4, 4).T, sx, occ)
    diff = np.nonzero(counts != ref)[0]
    if dof == 6:
        assert len(diff) == 0, diff[:10]
    else:  # the yaw's atan2 / cos / sin may differ by ulps between device and host: a point on a cell face may move
        assert len(diff) <= 0.01 * res["evaluated"] and (np.abs(counts[diff] - ref[diff]) <= 3).all(), diff[:10]
    best, status, evaluated = gl.select(counts, len(sx), rate, H)
    assert (res["best_hypothesis"], res["status"], res["evaluated"]) == (best, status, evaluated)
    assert res["inliers"] == counts[best] and res["inlier_rate"] == counts[best] / len(sx)
    if rate > 1:
        assert evaluated == H and status == gl.FOUND
    else:
        assert status == gl.EARLY_STOP and evaluated < H
    assert (counts[evaluated:] == -2).all()


# ---------------------------------------------------------------------------------------------------------------------
# GLIM's recipe (manual_loop_close_modal.cpp:318-368 preprocessing, :370-468 global, :470-520 fine)
# ---------------------------------------------------------------------------------------------------------------------
def merged_map(ctx, frames):
    """the modal's preprocess: an iVox (resolution 5 min_distance, 50 points per cell, min distance 0.5) of the frames in the
    world frame, its points, k-NN (k = 10) and PLANE covariances -> (points (N,4), covs, normals)"""
    iv = gpu.IVoxGPU(2.5, min_dist_in_cell=0.5, max_points_in_cell=50, lru_horizon=1000000, ctx=ctx)
    for pts, cov, T in frames:
        iv.insert(gpu.PointCloudGPU.clone(pts, cov, ctx=ctx), T)
    xyz = iv.download()[2].astype(np.float64)
    p4 = np.c_[xyz, np.ones(len(xyz))]
    nb = preprocess.find_neighbors(p4, 10, ctx=ctx)
    normals, covs = preprocess.CloudCovarianceEstimation(ctx=ctx).estimate(p4, nb)
    return p4, covs, normals


@pytest.fixture(scope="module")
def maps(ctx):
    fr = vo.arc_frames(16, 32 * 400)
    return merged_map(ctx, fr[:10]), merged_map(ctx, fr[6:])


@pytest.mark.parametrize("dof", [4, 6])
def test_manual_loop_closure_recipe(ctx, maps, dof):
    """Two overlapping merged maps of the hall, the source expressed under a pose 120 degrees of yaw and 18 m away (plus a few
    degrees of roll and pitch for 6-DoF): FPFH at r = 5, RANSAC with the modal's defaults, then LM on a grid GICP factor with
    r = 1.0 (the modal's fine registration) recovers the pose."""
    (tp, tc, tn), (sp, sc, sn) = maps
    T_gt = synth.pose(15.0, -10.0, 0.5, np.radians(120), *((np.radians(3), np.radians(-2)) if dof == 6 else (0.0, 0.0)))
    Ti = synth.inv_pose(T_gt)
    sp2 = np.c_[sp[:, :3] @ Ti[:3, :3].T + Ti[:3, 3], np.ones(len(sp))]
    sc2 = np.einsum("ij,njk,lk->nil", Ti, sc, Ti)
    sn2 = np.c_[sn[:, :3] @ Ti[:3, :3].T, np.zeros(len(sn))]
    tgt = gpu.PointCloudGPU.clone(tp, tc, tn, ctx=ctx).estimate_fpfh(5.0)
    src = gpu.PointCloudGPU.clone(sp2, sc2, sn2, ctx=ctx).estimate_fpfh(5.0)
    res = gpu.estimate_pose_ransac(tgt, src, dof=dof)
    et0, er0 = pose_error(res["T_target_source"], T_gt)
    grid = gpu.PointGridGPU(tgt, 1.05, ctx=ctx)
    f = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, grid, src, 1.0, ctx=ctx)
    fine = gpu.align_vgicp([[f]], [res["T_target_source"]], params={"max_iterations": 30})[0]
    et, er = pose_error(fine["T_target_source"], T_gt)
    print(f"dof {dof}: {len(tp)} / {len(sp)} points, ransac {res['status_name']} h {res['best_hypothesis']} rate {res['inlier_rate']:.3f}"
          f" err {et0:.3f} m {er0:.3f} deg; fine {fine['status_name']} err {et:.4f} m {er:.4f} deg")
    # bars about twice the worst measured on an H100 (DESIGN.md 4.12): RANSAC 0.166 m / 0.237 deg, fine 0.0004 m / 0.0010 deg
    assert res["status"] in (gl.FOUND, gl.EARLY_STOP)
    assert et0 < 0.35 and er0 < 0.5, (et0, er0)
    assert et < 1e-3 and er < 2e-3, (et, er)


# ---------------------------------------------------------------------------------------------------------------------
# refusals and launch counts
# ---------------------------------------------------------------------------------------------------------------------
def test_refusals_come_before_any_launch(ctx, frames):
    L = capi.lib()
    pts, cov, _ = frames[0]
    bare = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)  # no normals
    withf, _, _ = cloud_of(ctx, frames[2])
    withf.estimate_fpfh(1.0)
    nofeat, _, _ = cloud_of(ctx, frames[3])
    res = capi.RansacResult()
    out = np.zeros(nofeat.n, np.int32)
    launches = ctx.kernel_launches
    assert L.gb_cloud_estimate_fpfh(ctx.h, bare.h, 1.0) == 1
    for r in (0.0, -2.0, float("nan"), float("inf")):
        assert L.gb_cloud_estimate_fpfh(ctx.h, nofeat.h, r) == 1
    with pytest.raises(capi.GlimB200Error):
        bare.fpfh()
    with pytest.raises(capi.GlimB200Error):
        nofeat.fpfh()
    for a, b in ((withf, nofeat), (nofeat, withf)):
        assert L.gb_fpfh_match(ctx.h, a.h, b.h, capi.ptr(out)) == 1
        assert L.gb_ransac_align(ctx.h, a.h, b.h, C.byref(gpu.ransac_params()), C.byref(res), None) == 1
    for bad in ({"max_iterations": 0}, {"early_stop_inlier_rate": -1.0}, {"inlier_voxel_resolution": 0.0}, {"dof": 3}):
        assert L.gb_ransac_align(ctx.h, withf.h, withf.h, C.byref(gpu.ransac_params(**bad)), C.byref(res), None) == 1
    assert ctx.kernel_launches == launches
    if L.gb_device_count() > 1:
        ctx1 = gpu.Context(1)
        other, _, _ = cloud_of(ctx1, frames[2])
        assert L.gb_cloud_estimate_fpfh(ctx.h, other.h, 1.0) == 1
        other.estimate_fpfh(1.0)
        assert L.gb_fpfh_match(ctx.h, withf.h, other.h, capi.ptr(out)) == 1
        assert L.gb_ransac_align(ctx.h, other.h, withf.h, C.byref(gpu.ransac_params()), C.byref(res), None) == 1
        assert ctx.kernel_launches == launches


def test_launch_counts(ctx, small_problem, frames):
    """FPFH: the point grid build's launches + 2; the match: 1; RANSAC: 1 + the target grid's build + 2 per wave of 512."""
    tgt, src, _ = small_problem
    for r in (1.0, 2.5):
        l0 = ctx.kernel_launches
        gpu.PointGridGPU(src, 1.05 * r, ctx=ctx)
        g = ctx.kernel_launches - l0
        l0 = ctx.kernel_launches
        src.estimate_fpfh(r)
        assert ctx.kernel_launches - l0 == g + 2, r
    tgt.estimate_fpfh(2.5)
    l0 = ctx.kernel_launches
    gpu.fpfh_match(tgt, src)
    assert ctx.kernel_launches - l0 == 1
    l0 = ctx.kernel_launches
    gpu.PointGridGPU(tgt, 1.0, ctx=ctx)
    g = ctx.kernel_launches - l0
    for H in (100, 512, 1300):
        l0 = ctx.kernel_launches
        res = gpu.estimate_pose_ransac(tgt, src, max_iterations=H, early_stop_inlier_rate=2.0)
        waves = -(-H // 512)
        assert res["evaluated"] == H and ctx.kernel_launches - l0 == 1 + g + 2 * waves, H
