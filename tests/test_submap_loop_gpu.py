"""GLIM's manual loop closure on two submaps picked in the viewer (interactive_viewer.cpp:383-387 -> set_target / set_source,
manual_loop_close_modal.cpp:76-101), on the H100 from device clouds only: two overlapping merged submaps of the hall
(gb_merge_frames: covariances, no normals), each rotated by its gravity alignment as its merge pose (the transform_inplace at
:84, :96), then estimate_normals -> FPFH (r = 5) -> RANSAC or GNC at dof 4 and 6 -> LM on a GICP factor over a point grid
(20 iterations, r = 1.0).  The planted transform is recovered within 1 mm (the bar of tests/test_global_gpu.py's recipe) and
5e-3 degrees."""
import numpy as np
import pytest

from glim_b200 import capi, gpu, synth
from tests import voxelmap_oracle as vo

pytestmark = pytest.mark.gpu

FINE_LM = {"max_iterations": 20, "lambda_initial": 1e-5, "lambda_factor": 10.0, "lambda_upper_bound": 1e5, "relative_error_tol": 1e-5,
           "absolute_error_tol": 1e-5, "step_translation_tol": 0.0, "step_rotation_tol": 0.0}


def pose_error(T, T_ref):
    d = synth.inv_pose(T_ref) @ T
    return float(np.linalg.norm(d[:3, 3])), float(np.degrees(np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1))))


def gravity_aligned_submap(ctx, frames, origin, planted):
    """frames merged in the submap's origin frame (sub_mapping.cpp:481-497), turned by the rotation of the origin's world pose
    (the gravity alignment) and expressed under `planted`^-1 -> (device cloud, merge-frame-of-world transform)"""
    G = np.eye(4)
    G[:3, :3] = frames[origin][2][:3, :3]
    M = synth.inv_pose(planted) @ G @ synth.inv_pose(frames[origin][2])
    clouds = [gpu.PointCloudGPU.clone(f[0], f[1], ctx=ctx) for f in frames]
    return gpu.merge_frames_gpu([M @ f[2] for f in frames], clouds, 0.25, ctx=ctx, host_outputs=False)[2], M


@pytest.fixture(scope="module")
def hall():
    return vo.arc_frames(16, 32 * 400)


@pytest.mark.parametrize("dof", [4, 6])
def test_right_click_loop_closure_recipe(ctx, hall, dof):
    planted = synth.pose(15.0, -10.0, 0.5, np.radians(120), *((np.radians(3), np.radians(-2)) if dof == 6 else (0.0, 0.0)))
    tgt, M_t = gravity_aligned_submap(ctx, hall[:10], 0, np.eye(4))
    src, M_s = gravity_aligned_submap(ctx, hall[6:], 0, planted)
    T_gt = M_t @ synth.inv_pose(M_s)
    for c in (tgt, src):
        with pytest.raises(capi.GlimB200Error):
            c.normals()
        c.estimate_normals().estimate_fpfh(5.0)
    grid = gpu.PointGridGPU(tgt, 1.05, ctx=ctx)
    for method in ("ransac", "gnc"):
        est = gpu.estimate_pose_ransac if method == "ransac" else gpu.estimate_pose_gnc
        res = est(tgt, src, dof=dof)
        et0, er0 = pose_error(res["T_target_source"], T_gt)
        f = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, grid, src, 1.0, ctx=ctx)
        fine = gpu.align_vgicp([[f]], [res["T_target_source"]], params=FINE_LM)[0]
        et, er = pose_error(fine["T_target_source"], T_gt)
        print(f"dof {dof} {method}: {tgt.n} / {src.n} points, {res['status_name']} err {et0:.3f} m {er0:.3f} deg; "
              f"fine {fine['status_name']} it {fine['iterations']} err {et:.5f} m {er:.5f} deg")
        assert et0 < 1.0 and er0 < 3.0, (method, et0, er0)
        # The GICP optimum of two merged submaps lies 0.0014-0.0025 degrees from the planted pose whatever the global start and
        # the LM tolerances (measured on an H100 80GB HBM3 at 700 W, merge resolutions 0.1-0.5 m): voxel centroids of different
        # frame sets are not the same points.  So the rotation bar is twice the worst of those, not tests/test_global_gpu.py's
        # 2e-3 degrees, which maps built from one iVox and one covariance estimation meet.
        assert et < 1e-3 and er < 5e-3, (method, et, er)
