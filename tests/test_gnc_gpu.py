"""GNC global registration on the H100 (gb_gnc_align): the device's reciprocal pairs exactly against the numpy restatement
(tests/gnc_oracle.py), with and without sampling, on a source with NaN points and a planted tie; the device solve and score
against the restatement on the device's own pairs; recovery of a known pose between identical content; GLIM's manual
loop-closure recipe with GNC as its global method; the refusals and the launch counts."""
import ctypes as C

import numpy as np
import pytest

from glim_b200 import capi, gpu, preprocess, synth
from tests import global_oracle as gl
from tests import gnc_oracle as gno
from tests import voxelmap_oracle as vo

pytestmark = pytest.mark.gpu

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


@pytest.fixture(scope="module")
def tie_problem(ctx, frames):
    """frame 2 as the target; frame 1 (every 7th point NaN) plus a copy of its point 100 (same position and normal) as the
    source; features at r = 1.5"""
    nrm, _ = synth.with_covariances(np.nan_to_num(frames[1][0], nan=1e4), 10)
    src, _, _ = cloud_of(ctx, frames[1], (frames[1][0][[100]], nrm[[100]]))
    tgt, _, _ = cloud_of(ctx, frames[2])
    return tgt.estimate_fpfh(1.5), src.estimate_fpfh(1.5)


@pytest.mark.parametrize("max_init_samples", [700, 10000])
def test_pairs_equal_the_restatement(ctx, tie_problem, max_init_samples):
    """The device pairs equal the restatement exactly, below and above the source size; no NaN point is in a pair; the planted
    copy ties with its original, so the reciprocal check keeps only the smaller index."""
    tgt, src = tie_problem
    res = gpu.estimate_pose_gnc(tgt, src, correspondences=True, max_init_samples=max_init_samples, seed=91)
    sx, _ = src.download()
    tx, _ = tgt.download()
    fs, ft = src.fpfh(), tgt.fpfh()
    assert np.array_equal(fs[100], fs[-1])
    ref = gno.gnc_pairs(ft, fs, tx, sx, 91, max_init_samples)
    pairs = res["pairs"]
    assert res["samples"] == min(src.n, max_init_samples) and res["correspondences"] == len(ref) >= 3
    assert np.array_equal(pairs, ref)
    assert np.isfinite(sx[pairs[:, 0]]).all() and np.isfinite(tx[pairs[:, 1]]).all()
    assert src.n - 1 not in pairs[:, 0]
    assert (~np.isfinite(sx).all(1)).sum() > 0


@pytest.fixture(scope="module")
def small_problem(ctx, frames):
    """frame 2 as the target, 1500 points of frame 3 moved by a known pose as the source, features at r = 1.5"""
    tgt, _, _ = cloud_of(ctx, frames[2])
    T_gt = synth.pose(4.0, -3.0, 0.2, np.radians(100), 0.02, -0.01)
    fin = np.isfinite(frames[3][0]).all(1)
    keep = np.nonzero(fin)[0][:: max(1, fin.sum() // 1500)]
    p = frames[3][0][keep].copy()
    p[:, :3] = (p[:, :3] - T_gt[:3, 3]) @ T_gt[:3, :3]
    nrm, cov = synth.with_covariances(p, 10)
    src = gpu.PointCloudGPU.clone(p, cov, nrm, ctx=ctx)
    return tgt.estimate_fpfh(1.5), src.estimate_fpfh(1.5), T_gt


@pytest.mark.parametrize("dof", [4, 6])
@pytest.mark.parametrize("max_init_samples", [700, 10000])
def test_solve_and_score_equal_the_restatement(ctx, small_problem, dof, max_init_samples):
    """On the device's own pairs: T and the weights equal the restatement within 1e-9, the iteration count exactly; the inlier
    count is RANSAC's test of the device's T."""
    tgt, src, _ = small_problem
    res = gpu.estimate_pose_gnc(tgt, src, correspondences=True, dof=dof, max_init_samples=max_init_samples)
    sx, _ = src.download()
    tx, _ = tgt.download()
    pairs = res["pairs"]
    T, w, it, st = gno.gnc_solve(sx[pairs[:, 0]], tx[pairs[:, 1]], dof)
    assert res["status"] == st == gno.GNC_FOUND and res["status_name"] == "FOUND"
    assert res["iterations"] == it
    assert np.abs(res["T_target_source"] - T).max() < 1e-9
    assert np.abs(res["weights"] - w).max() < 1e-9
    assert res["inliers"] == gl.inliers(res["T_target_source"], sx, gl.occupancy(tx, 1.0))
    assert res["inlier_rate"] == res["inliers"] / src.n


def test_degenerate_when_fewer_than_three_pairs(ctx, small_problem):
    """One sample can give at most one pair: DEGENERATE with T = I, 0 iterations, and the score of the identity."""
    tgt, src, _ = small_problem
    res = gpu.estimate_pose_gnc(tgt, src, correspondences=True, max_init_samples=1)
    sx, _ = src.download()
    tx, _ = tgt.download()
    assert res["status"] == gno.GNC_DEGENERATE and res["status_name"] == "DEGENERATE" and res["iterations"] == 0 and res["samples"] == 1
    assert np.array_equal(res["T_target_source"], np.eye(4)) and (res["weights"] == 0).all()
    assert res["inliers"] == gl.inliers(np.eye(4), sx, gl.occupancy(tx, 1.0))


@pytest.mark.parametrize("dof", [4, 6])
def test_identical_content_recovers_the_pose(ctx, frames, dof):
    """The source is the target's points under a known pose: GNC alone recovers it."""
    tgt, t_pts, t_nrm = cloud_of(ctx, frames[2])
    T_gt = synth.pose(6.0, 9.0, 0.3, np.radians(-140), *((np.radians(4), np.radians(-3)) if dof == 6 else (0.0, 0.0)))
    Ti = synth.inv_pose(T_gt)
    sp = np.c_[t_pts[:, :3] @ Ti[:3, :3].T + Ti[:3, 3], np.ones(len(t_pts))]
    sn = np.c_[t_nrm[:, :3] @ Ti[:3, :3].T, np.zeros(len(t_nrm))]
    _, sc = synth.with_covariances(sp, 10)
    src = gpu.PointCloudGPU.clone(sp, sc, sn, ctx=ctx).estimate_fpfh(1.5)
    tgt.estimate_fpfh(1.5)
    res = gpu.estimate_pose_gnc(tgt, src, dof=dof)
    et, er = pose_error(res["T_target_source"], T_gt)
    print(f"dof {dof}: identical content, K {res['correspondences']} of {res['samples']}, rate {res['inlier_rate']:.3f}, err {et:.5f} m {er:.5f} deg")
    assert res["status"] == gno.GNC_FOUND
    assert et < 1e-3 and er < 1e-2, (et, er)


# ---------------------------------------------------------------------------------------------------------------------
# GLIM's recipe (manual_loop_close_modal.cpp:318-368 preprocessing, :370-468 global, :470-520 fine), GNC as the global method
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
def test_manual_loop_closure_recipe_with_gnc(ctx, maps, dof):
    """Two overlapping merged maps of the hall, the source expressed under a pose 120 degrees of yaw and 18 m away (plus a few
    degrees of roll and pitch for 6-DoF): FPFH at r = 5, GNC with the modal's settings (10000 samples, the seed after the
    modal's first += 4322), then LM on a grid GICP factor with r = 1.0 (the modal's fine registration) recovers the pose."""
    (tp, tc, tn), (sp, sc, sn) = maps
    T_gt = synth.pose(15.0, -10.0, 0.5, np.radians(120), *((np.radians(3), np.radians(-2)) if dof == 6 else (0.0, 0.0)))
    Ti = synth.inv_pose(T_gt)
    sp2 = np.c_[sp[:, :3] @ Ti[:3, :3].T + Ti[:3, 3], np.ones(len(sp))]
    sc2 = np.einsum("ij,njk,lk->nil", Ti, sc, Ti)
    sn2 = np.c_[sn[:, :3] @ Ti[:3, :3].T, np.zeros(len(sn))]
    tgt = gpu.PointCloudGPU.clone(tp, tc, tn, ctx=ctx).estimate_fpfh(5.0)
    src = gpu.PointCloudGPU.clone(sp2, sc2, sn2, ctx=ctx).estimate_fpfh(5.0)
    res = gpu.estimate_pose_gnc(tgt, src, dof=dof, seed=53123 + 4322)
    et0, er0 = pose_error(res["T_target_source"], T_gt)
    grid = gpu.PointGridGPU(tgt, 1.05, ctx=ctx)
    f = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, grid, src, 1.0, ctx=ctx)
    fine = gpu.align_vgicp([[f]], [res["T_target_source"]], params={"max_iterations": 30})[0]
    et, er = pose_error(fine["T_target_source"], T_gt)
    print(f"dof {dof}: {len(tp)} / {len(sp)} points, gnc {res['status_name']} K {res['correspondences']} of {res['samples']} it {res['iterations']}"
          f" rate {res['inlier_rate']:.3f} err {et0:.3f} m {er0:.3f} deg; fine {fine['status_name']} err {et:.4f} m {er:.4f} deg")
    assert res["status"] == gno.GNC_FOUND and res["samples"] == 10000
    # bars about twice the worst measured on an H100 (DESIGN.md 4.12): GNC 0.031 m / 0.211 deg, fine 0.0004 m / 0.0010 deg
    assert et0 < 0.07 and er0 < 0.45, (et0, er0)
    assert et < 1e-3 and er < 2e-3, (et, er)


# ---------------------------------------------------------------------------------------------------------------------
# refusals and launch counts
# ---------------------------------------------------------------------------------------------------------------------
def test_refusals_come_before_any_launch(ctx, frames):
    L = capi.lib()
    withf, _, _ = cloud_of(ctx, frames[2])
    withf.estimate_fpfh(1.0)
    nofeat, _, _ = cloud_of(ctx, frames[3])
    empty = gpu.PointCloudGPU.clone(np.zeros((0, 4)), np.zeros((0, 4, 4)), np.zeros((0, 4)), ctx=ctx).estimate_fpfh(1.0)
    res = capi.GncResult()
    ok = C.byref(gpu.gnc_params())
    launches = ctx.kernel_launches
    assert L.gb_gnc_align(None, withf.h, withf.h, ok, C.byref(res), None, None) == 1
    assert L.gb_gnc_align(ctx.h, None, withf.h, ok, C.byref(res), None, None) == 1
    assert L.gb_gnc_align(ctx.h, withf.h, None, ok, C.byref(res), None, None) == 1
    assert L.gb_gnc_align(ctx.h, withf.h, withf.h, None, C.byref(res), None, None) == 1
    assert L.gb_gnc_align(ctx.h, withf.h, withf.h, ok, None, None, None) == 1
    for a, b in ((withf, nofeat), (nofeat, withf), (withf, empty), (empty, withf)):
        assert L.gb_gnc_align(ctx.h, a.h, b.h, ok, C.byref(res), None, None) == 1
    for bad in ({"max_init_samples": 0}, {"max_init_samples": (1 << 28) + 1}, {"dof": 3}, {"dof": 5}):
        assert L.gb_gnc_align(ctx.h, withf.h, withf.h, C.byref(gpu.gnc_params(**bad)), C.byref(res), None, None) == 1, bad
    assert ctx.kernel_launches == launches
    if L.gb_device_count() > 1:
        ctx1 = gpu.Context(1)
        other, _, _ = cloud_of(ctx1, frames[2])
        other.estimate_fpfh(1.0)
        assert L.gb_gnc_align(ctx.h, other.h, withf.h, ok, C.byref(res), None, None) == 1
        assert L.gb_gnc_align(ctx.h, withf.h, other.h, ok, C.byref(res), None, None) == 1
        assert ctx.kernel_launches == launches


def test_launch_counts(ctx, small_problem):
    """The target grid's build + 7; + 5 when the source has more points than max_init_samples."""
    tgt, src, _ = small_problem
    l0 = ctx.kernel_launches
    gpu.PointGridGPU(tgt, 1.0, ctx=ctx)
    g = ctx.kernel_launches - l0
    for m, extra in ((src.n, 0), (src.n + 1, 0), (src.n - 1, 5), (300, 5)):
        l0 = ctx.kernel_launches
        res = gpu.estimate_pose_gnc(tgt, src, max_init_samples=m)
        assert res["samples"] == min(m, src.n) and ctx.kernel_launches - l0 == g + 7 + extra, m
