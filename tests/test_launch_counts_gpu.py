"""gb_ctx_kernel_launches on the H100: the exact count one call of each launching entry point adds, on small seeded inputs.

The counter's unit (include/glim_b200.h): one per kernel launch and one per cub device-wide call, one per launch of a captured
sweep graph; memsets and copies are not counted.  Each expected value below is written as a sum whose terms name the kernels
(and cub calls) of that path, so it can be read against the code.  Shared pieces:
    group    = gb_group_by_key: cub SortPairs + k_head_flags + cub InclusiveSum                   = 3
    starts   = gb_group_starts: k_voxel_starts                                                     = 1
    thin     = gb_thin: k_thin_hash + cub SortKeys + k_thin_keep                                   = 3
    table    = one table_build attempt: k_table_clear + k_table_insert + k_table_finalize          = 3
    cloud    = gb_cloud_build: k_morton_keys + cub SortPairs + k_permute_cloud                     = 3
    knn      = knn_device: k_fill_self + k_ml_keys + cub SortPairs + k_ml_gather + k_ml_cells + k_knn_pyramid = 6"""
import numpy as np
import pytest

from glim_b200 import gpu, preprocess, synth

pytestmark = pytest.mark.gpu

GROUP, STARTS, THIN, TABLE, CLOUD, KNN = 3, 1, 3, 3, 3, 6


@pytest.fixture(scope="module")
def scans():
    sc = synth.make_hall_scene()
    traj = synth.arc_trajectory(8)
    out = []
    for i in (3, 4):
        pts, times = synth.scan(sc, "hdl32", traj[i], synth.rng_for(7, i), n_rays=32 * 200)
        _, cov = synth.with_covariances(pts, 10)
        out.append((pts, times, cov))
    T = synth.perturb(synth.inv_pose(traj[3]) @ traj[4], synth.rng_for(8), 0.01, 0.05)
    return out, T


def launches(ctx, call):
    before = ctx.kernel_launches
    result = call()
    return ctx.kernel_launches - before, result


def test_cloud_upload(ctx, scans):
    pts, _, cov = scans[0][0]
    n, _ = launches(ctx, lambda: gpu.PointCloudGPU.clone(pts, cov, ctx=ctx))
    assert n == CLOUD


def test_voxelmap_build(ctx, scans):
    pts, _, cov = scans[0][0]
    cloud = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
    n, m = launches(ctx, lambda: gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(cloud))
    assert m.num_buckets == 16384 * 2 ** int(np.ceil(np.log2(max(1.0, 8 * m.num_voxels / 16384))))  # one table attempt
    assert n == 1 + GROUP + STARTS + 1 + TABLE  # k_point_keys, group, starts, k_voxel_reduce, table


def test_voxelmap_insert(ctx, scans):
    (pts0, _, cov0), (pts1, _, cov1) = scans[0]
    c0 = gpu.PointCloudGPU.clone(pts0, cov0, ctx=ctx)
    c1 = gpu.PointCloudGPU.clone(pts1, cov1, ctx=ctx)
    m = gpu.IncrementalVoxelMapGPU(0.5, ctx=ctx)
    # into the empty map, rate 1: k_merge_transform + k_grid_keys, group, starts, k_ins_merge + cub InclusiveSum + k_ins_count,
    # k_ins_emit, table
    n, _ = launches(ctx, lambda: m.insert(c0))
    assert n == 2 + GROUP + STARTS + 3 + 1 + TABLE
    # into a non-empty map, rate < 1: + k_ins_old_keys, + thin
    n, _ = launches(ctx, lambda: m.insert(c1, scans[1], sampling_rate=0.1, seed=3))
    assert n == 1 + 2 + THIN + GROUP + STARTS + 3 + 1 + TABLE


def test_overlap_covariances_and_deskew(ctx, scans):
    pts, times, cov = scans[0][0]
    T = scans[1]
    cloud = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
    m = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(cloud)
    n, _ = launches(ctx, lambda: gpu.overlap_gpu(m, cloud, T))
    assert n == 1  # k_overlap
    nb = synth.knn(pts, 10)
    n, _ = launches(ctx, lambda: preprocess.CloudCovarianceEstimation(ctx=ctx).estimate(pts, nb))
    assert n == 1  # k_covariances
    n, _ = launches(ctx, lambda: preprocess.CloudDeskewing(ctx=ctx).deskew(np.eye(4), times, pts, linear_vel=[1.0, 0.0, 0.0], angular_vel=[0.0, 0.0, 0.3]))
    assert n == 1  # k_deskew


@pytest.mark.parametrize("mode", ["brute", "pyramid"])
def test_find_neighbors(ctx, scans, monkeypatch, mode):
    monkeypatch.setenv("GB_KNN", mode)
    pts = scans[0][0][0]
    n, _ = launches(ctx, lambda: preprocess.find_neighbors(pts, 10, ctx=ctx))
    assert n == (1 if mode == "brute" else 1 + KNN)  # k_knn_bruteforce | k_set_int + knn


def test_voxelgrid_sampling(ctx, scans):
    pts, times, _ = scans[0][0]
    n, (out, _, _) = launches(ctx, lambda: preprocess.voxelgrid_sampling(pts, 0.5, times=times, ctx=ctx))
    assert len(out) > 0
    assert n == 1 + GROUP + STARTS + 1  # k_grid_keys, group, starts, k_grid_means_counted


PREPROCESS = {
    # k_set_int; downsampling; k_filter_time_keys + cub SortPairs + k_gather_frame; [outlier removal]; knn; k_covariances_planes; cloud
    "voxel_grid": (dict(downsample_resolution=0.5), 1 + (1 + GROUP + 1 + STARTS + 1) + 3 + KNN + 1 + CLOUD),  # k_grid_keys, group, k_copy_last_pos, starts, k_grid_means_counted
    "random_grid": (dict(downsample_resolution=0.5, use_random_grid_downsampling=True, downsample_rate=0.3),
                    1 + (1 + GROUP + 1 + STARTS + 1 + THIN) + 3 + KNN + 1 + CLOUD),  # ..., k_randomgrid_select, thin
    "outlier_removal": (dict(downsample_resolution=0.5, enable_outlier_removal=True),
                        1 + (1 + GROUP + 1 + STARTS + 1) + 3 + (KNN + 6) + KNN + 1 + CLOUD),  # knn + k_sor_dists + 2 cub Sum + k_sor_flags + cub InclusiveSum + k_sor_compact
}


@pytest.mark.parametrize("config", sorted(PREPROCESS))
def test_preprocess(ctx, scans, config):
    pts, times, _ = scans[0][0]
    params, expected = PREPROCESS[config]
    g = preprocess.FramePreprocessorGPU(preprocess.CloudPreprocessorParams(**params), ctx, seed=5)
    n, (fr, _, _, cloud) = launches(ctx, lambda: g.preprocess(0.0, times, pts))
    assert fr.size() > 0 and cloud is not None
    assert n == expected


def test_merge_frames(ctx, scans):
    (pts0, _, cov0), (pts1, _, cov1) = scans[0]
    frames = [gpu.PointCloudGPU.clone(pts0, cov0, ctx=ctx), gpu.PointCloudGPU.clone(pts1, cov1, ctx=ctx)]
    n, (out, _, cloud) = launches(ctx, lambda: gpu.merge_frames_gpu([np.eye(4), scans[1]], frames, 0.5, target_num_points=2000, seed=1, ctx=ctx))
    assert 0 < len(out) and cloud is not None
    # k_merge_transform + k_grid_keys, group, k_copy_last_pos, starts, k_grid_means_counted, thin + cub InclusiveSum,
    # k_merge_emit, cloud
    assert n == 2 + GROUP + 1 + STARTS + 1 + THIN + 1 + 1 + CLOUD


@pytest.mark.parametrize("path", ["graph", "plain"])
def test_factor_set_linearize(ctx, scans, monkeypatch, path):
    if path == "plain":
        monkeypatch.setenv("GB_KERNEL", "3")  # k_vgicp_sweep3: no captured graph
    (pts0, _, cov0), (pts1, _, cov1) = scans[0]
    m = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(gpu.PointCloudGPU.clone(pts0, cov0, ctx=ctx))
    f = gpu.IntegratedVGICPFactorGPU(0, 1, m, gpu.PointCloudGPU.clone(pts1, cov1, ctx=ctx), ctx=ctx)
    fs = gpu.NonlinearFactorSetGPU(ctx).add([f])
    values = {0: np.eye(4), 1: scans[1]}
    for _ in range(3):  # the first call of the graph path captures the graph; every call is one launch
        n, out = launches(ctx, lambda: fs.linearize(values))
        assert out[0]["num_inliers"] > 0
        assert n == 1  # the sweep (graph path: one graph launch)


def test_vgicp_align(ctx, scans):
    (pts0, _, cov0), (pts1, _, cov1) = scans[0]
    m = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(gpu.PointCloudGPU.clone(pts0, cov0, ctx=ctx))
    f = gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, m, gpu.PointCloudGPU.clone(pts1, cov1, ctx=ctx), ctx=ctx)
    n, (r,) = launches(ctx, lambda: gpu.align_vgicp([[f]], scans[1]))
    # three rounds, one trial each, every trial accepted (so every round starts from a fresh linearization point):
    # per round the linearize sweep + k_align_step + the error sweep + k_align_accept
    assert (r["trials"], r["iterations"], r["status_name"]) == (3, 3, "CONVERGED")
    assert n == 3 * (1 + 1 + 1 + 1)
