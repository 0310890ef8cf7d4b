"""Point-to-point ICP factors on device point grids (gb_icp_grid_factor_create) on the H100: the factor through every consumer
against the fp64 restatement (tests/icp_oracle.py, correspondences from tests/grid_oracle.py), between clouds uploaded without
covariances, the modal's 200-iteration align recovering a planted pose, the refusals of mixed sets and the launch counts."""
import ctypes as C

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth
from tests import grid_oracle as go
from tests import icp_oracle as icp
from tests import voxelmap_oracle as vo
from tests import util
from tests.util import REL_TOL, check_linearized

pytestmark = pytest.mark.gpu

# the modal's fine registration of clouds without covariances (manual_loop_close_modal.cpp:479-492): 200 iterations, GTSAM's
# LM defaults, no step tests
MODAL_LM = {"max_iterations": 200, "lambda_initial": 1e-5, "lambda_factor": 10.0, "lambda_upper_bound": 1e5, "relative_error_tol": 1e-5,
            "absolute_error_tol": 1e-5, "step_translation_tol": 0.0, "step_rotation_tol": 0.0}


def pose_error(T, T_ref):
    d = synth.inv_pose(T_ref) @ T
    return float(np.linalg.norm(d[:3, 3])), float(np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1)))


@pytest.fixture(scope="module")
def frames():
    return vo.arc_frames(4, 32 * 200, nan_frame=3)


def delta(frames, a, b):
    return synth.inv_pose(frames[a][2]) @ frames[b][2]


@pytest.mark.parametrize("covs", [True, False])
@pytest.mark.parametrize("cell_size,want_m", [(1.05, 1), (0.6, 2)])
def test_factor_matches_fp64_restatement(ctx, frames, covs, cell_size, want_m):
    """Frame 2 as the target, frame 3 (with NaN points) as the source, both uploaded with or without covariances.  At m = 1 and
    2, through gb_vgicp_linearize, a factor set and a sweep at poses up to 1 m / 0.1 rad off: inlier counts exact, H / b / error
    within 1e-4 of the restatement; error() with T_lin != T_eval likewise.  A GICP factor refuses the bare source."""
    tgt = gpu.PointCloudGPU.clone(frames[2][0], frames[2][1] if covs else None, ctx=ctx)
    src = gpu.PointCloudGPU.clone(frames[3][0], frames[3][1] if covs else None, ctx=ctx)
    xt, _ = tgt.download()
    xyz, _ = src.download()
    max_corr = 1.0
    R = icp.grid(xt, cell_size)
    g = gpu.PointGridGPU(tgt, cell_size, ctx=ctx)
    T0 = delta(frames, 2, 3)
    rng = synth.rng_for(1100)
    poses = [T0, synth.perturb(T0, rng, 0.02, 0.3), synth.perturb(T0, rng, 0.05, 0.5), synth.pose(1.0, -0.5, 0.2, 0.1, 0.0, 0.0) @ T0]
    facs = [gpu.IntegratedICPFactorGPU(np.eye(4), 0, g, src, max_corr, ctx=ctx) for _ in poses]
    assert facs[0].search_half_width() == want_m == go.half_width(R.inv, go.max_d2(max_corr), R.key_extent)
    lin = [icp.linearize(R, xyz, T, max_corr) for T in poses]
    refs = [r for r, _ in lin]
    assert min(r["num_inliers"] for r in refs) > 0
    hits = [util.record_scale(util.factor_hits(R.xyz, None, xyz, None, T, corr)) for T, (_, corr) in zip(poses, lin)]
    check_linearized(facs[0].linearize({0: poses[0]}), refs[0], hits=hits[0])
    recs = gpu.NonlinearFactorSetGPU(ctx).add(facs).linearize_deltas(np.stack(poses))
    swept = gpu.Sweep(ctx, facs).linearize(np.stack(poses))
    for i in range(len(poses)):
        check_linearized(gpu.unpack_linearized(recs[i]), refs[i], hits=hits[i])
        check_linearized(gpu.unpack_linearized(swept[i]), refs[i], hits=hits[i])
    T_eval = [synth.perturb(T, rng, 0.005, 0.05) for T in poses]
    errs = gpu.NonlinearFactorSetGPU(ctx).add(facs).error_deltas(np.stack(poses), np.stack(T_eval))
    for i, (Tl, Te) in enumerate(zip(poses, T_eval)):
        ref = icp.error(R, xyz, Tl, Te, max_corr)
        assert abs(errs[i] - ref) < REL_TOL * ref, i
    assert abs(facs[0].error({0: T_eval[0]}) - icp.error(R, xyz, poses[0], T_eval[0], max_corr)) < REL_TOL * errs[0]
    if not covs:
        h = C.c_void_p()
        assert capi.lib().gb_gicp_grid_factor_create(ctx.h, g.h, src.h, max_corr, C.byref(h)) == 1 and not h.value


@pytest.fixture(scope="module")
def submap(ctx):
    """a merged submap of four frames, its copy under a planted pose, and the pose"""
    fr = vo.arc_frames(4, 32 * 300)
    clouds = [gpu.PointCloudGPU.clone(f[0], f[1], ctx=ctx) for f in fr]
    poses = [synth.inv_pose(fr[0][2]) @ f[2] for f in fr]
    pts, _, _ = gpu.merge_frames_gpu(poses, clouds, 0.1, ctx=ctx)
    T_gt = synth.pose(0.4, -0.3, 0.05, np.radians(4), np.radians(1), np.radians(-1))
    Ti = synth.inv_pose(T_gt)
    moved = np.c_[pts[:, :3] @ Ti[:3, :3].T + Ti[:3, 3], np.ones(len(pts))]
    return gpu.PointCloudGPU.clone(pts, ctx=ctx), gpu.PointCloudGPU.clone(moved, ctx=ctx), T_gt


def test_modal_align_recovers_a_planted_pose(ctx, submap):
    """The modal's ICP fine registration (r = 1.0, 200 iterations, GTSAM's LM defaults) on clouds without covariances: the same
    points under a planted pose (0.5 m, 4 degrees) are brought back onto the target from 8 starts around it (the global
    registration's result, in the modal), in one batch and alone."""
    tgt, src, T_gt = submap
    g = gpu.PointGridGPU(tgt, 1.05, ctx=ctx)
    rng = synth.rng_for(1200)
    T0 = [synth.perturb(T_gt, rng, 0.01, 0.15) for _ in range(8)]
    problems = [[gpu.IntegratedICPFactorGPU(np.eye(4), 0, g, src, 1.0, ctx=ctx)] for _ in T0]
    batch = gpu.align_vgicp(problems, T0, params=MODAL_LM)
    for i, r in enumerate(batch):
        et, er = pose_error(r["T_target_source"], T_gt)
        assert et < 1e-3 and er < 1e-4 and r["num_inliers"] > 0.95 * src.n, (i, et, er, r)
    solo = gpu.align_vgicp([problems[0]], [T0[0]], params=MODAL_LM)[0]
    assert np.abs(solo["T_target_source"] - batch[0]["T_target_source"]).max() < 1e-6


def test_mixed_sets_and_other_entry_points_are_refused_before_any_launch(ctx, frames):
    L = capi.lib()
    pts, cov, T = frames[0]
    cloud = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
    grid = gpu.PointGridGPU(cloud, 1.05, ctx=ctx)
    ivox = gpu.IVoxGPU(1.0, ctx=ctx).insert(cloud)
    vmap = gpu.IncrementalVoxelMapGPU(1.0, ctx=ctx).insert(cloud)
    fc = gpu.IntegratedICPFactorGPU(np.eye(4), 0, grid, cloud, 1.0, ctx=ctx)
    fg = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, grid, cloud, 1.0, ctx=ctx)
    fi = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, ivox, cloud, 1.0, ctx=ctx)
    fv = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, vmap, cloud, ctx=ctx)
    for f in (fc, fg, fi, fv):
        f._handle()
    sw = gpu.Sweep(ctx, [fc])
    ps = gpu.PeerSlab(ctx, 1)
    P2 = capi.pose16(np.stack([T, T]))
    h = C.c_void_p()
    launches = ctx.kernel_launches
    for other in (fg, fi, fv):
        for arr in ((C.c_void_p * 2)(fc._handle(), other._handle()), (C.c_void_p * 2)(other._handle(), fc._handle())):
            out = np.zeros(2, gpu.LIN_DTYPE)
            assert L.gb_factor_set_linearize(ctx.h, 2, C.cast(arr, C.c_void_p), capi.ptr(P2), capi.ptr(out)) == 1
            assert L.gb_factor_set_error(ctx.h, 2, C.cast(arr, C.c_void_p), capi.ptr(P2), capi.ptr(P2), capi.ptr(np.zeros(2))) == 1
            assert L.gb_sweep_create(ctx.h, 2, C.cast(arr, C.c_void_p), None, C.byref(h)) == 1 and not h.value
            off = np.array([0, 1, 2], np.uint64)
            res = (capi.AlignResult * 2)()
            assert L.gb_vgicp_align(ctx.h, 2, capi.ptr(off), C.cast(arr, C.c_void_p), capi.ptr(P2), C.byref(gpu.align_params()), C.cast(res, C.c_void_p)) == 1
    one = (C.c_void_p * 1)(fc._handle())
    assert L.gb_sweep_create(ctx.h, 1, C.cast(one, C.c_void_p), capi.ptr(np.zeros(1, np.int32)), C.byref(h)) == 1 and not h.value
    assert L.gb_sweep_attach_slab(sw.h, C.c_void_p(sw.results_device_ptr()), 1) == 1
    assert L.gb_sweep_attach_peer_slab(sw.h, ps.h) == 1
    rec = np.zeros(1, gpu.LIN_DTYPE)
    I16 = capi.pose16(np.eye(4))
    assert L.gb_ct_gicp_linearize(fc._handle(), capi.ptr(I16), capi.ptr(I16), capi.ptr(rec)) == 1
    for other in (ivox.h, vmap.h):
        assert L.gb_icp_grid_factor_create(ctx.h, other, cloud.h, 1.0, C.byref(h)) == 1 and not h.value
    for d in (0.0, -1.0, float("nan"), float("inf"), 9.0 * 1.05):
        assert L.gb_icp_grid_factor_create(ctx.h, grid.h, cloud.h, d, C.byref(h)) == 1 and not h.value
    assert ctx.kernel_launches == launches
    m = C.c_int()
    capi.check(L.gb_gicp_grid_factor_half_width(fc._handle(), C.byref(m)))
    assert m.value == 1


def test_one_launch_per_sweep_and_the_byte_count(ctx, frames):
    """A linearize is one launch (a graph), an error one launch, an align round three or four; gb_sweep_stats charges 16 B per
    source point, per stored target point and per bucket of the reference table, plus 552 B of pose and record."""
    tgt = gpu.PointCloudGPU.clone(frames[0][0], ctx=ctx)
    src = gpu.PointCloudGPU.clone(frames[1][0], ctx=ctx)
    g = gpu.PointGridGPU(tgt, 1.05, ctx=ctx)
    f = gpu.IntegratedICPFactorGPU(np.eye(4), 0, g, src, 1.0, ctx=ctx)
    T = synth.perturb(delta(frames, 0, 1), synth.rng_for(1300), 0.01, 0.1)
    f.linearize({0: T})
    for call in (lambda: f.linearize({0: T}), lambda: f.error({0: T})):
        l0 = ctx.kernel_launches
        call()
        assert ctx.kernel_launches - l0 == 1
    sw = gpu.Sweep(ctx, [f])
    sw.set_poses(np.stack([T]))
    l0 = ctx.kernel_launches
    sw.launch()
    sw.fetch()
    assert ctx.kernel_launches - l0 == 1
    nb = 16384
    while nb < g.num_cells:
        nb *= 2
    assert sw.algorithmic_bytes == 16 * (src.n + g.num_points + nb) + 552
    l0 = ctx.kernel_launches
    r = gpu.align_vgicp([[f]], [T])[0]
    n = ctx.kernel_launches - l0
    assert 3 * r["trials"] <= n <= 4 * r["trials"], (n, r)
