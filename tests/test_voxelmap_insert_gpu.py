"""gb_voxelmap_insert on the H100: the incremental device map against the numpy restatement of its rule
(tests/voxelmap_oracle.py), against gb_voxelmap_build, through every consumer, and in a device odometry loop
(gb_vgicp_align + inserts) against ground truth."""
import ctypes as C

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth
from oracle import oracle
from tests import util
from tests import voxelmap_oracle as vo
from tests.util import REL_TOL, check_linearized, cov_colmajor16, rel_err

pytestmark = pytest.mark.gpu

N_FRAMES = 22
NAN_FRAME = 9
EMPTY_INSERT = 14


def odometry_rate(k):
    if k == EMPTY_INSERT:
        return 1e-9  # keeps no point
    return 1.0 if k < 5 else 0.1


def pose_error(T, T_ref):
    d = synth.inv_pose(T_ref) @ T
    return float(np.linalg.norm(d[:3, 3])), float(np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1)))


@pytest.fixture(scope="module")
def frames():
    return vo.arc_frames(N_FRAMES, 32 * 200, nan_frame=NAN_FRAME)


def assert_same_map(m, R, k):
    buckets, vnum, vmean, vcov = m.download()
    assert m.num_voxels == R.num_voxels, k
    assert np.array_equal(buckets, R.buckets), k
    assert np.array_equal(vnum, R.n), k
    assert np.array_equal(vmean, R.means), k
    assert np.array_equal(vcov, R.covs), k


@pytest.mark.parametrize("config", ["rate1_no_lru", "odometry_lru"])
def test_insert_sequence_is_bit_exact(ctx, frames, config):
    """After every insert of a sequence at world poses, the downloaded map (table, counts, fp32 means and covariances) equals
    the restatement exactly.  One frame has NaN points; in the odometry schedule one insert keeps no point."""
    if config == "rate1_no_lru":
        res, lru, rate = 0.25, (0, 10), (lambda k: 1.0)
    else:
        res, lru, rate = 0.5, (6, 2), odometry_rate
    m = gpu.IncrementalVoxelMapGPU(res, lru_horizon=lru[0], lru_clear_cycle=lru[1], ctx=ctx)
    R = vo.IncrementalMap(res, lru_horizon=lru[0], lru_clear_cycle=lru[1])
    assert_same_map(m, R, -1)
    shrank = 0
    for k, (pts, cov, T) in enumerate(frames):
        cloud = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
        xyz, cov6 = oracle.pack_cloud(pts, cov_colmajor16(cov))
        before = R.num_voxels
        m.insert(cloud, T, sampling_rate=rate(k), seed=1000 + k)
        R.insert(xyz, cov6, T, rate(k), seed=1000 + k)
        shrank += R.num_voxels < before
        assert_same_map(m, R, k)
    if lru[0] > 0:
        assert shrank > 0


def test_single_insert_matches_build(ctx, frames):
    """At T = I and rate 1 an incremental map holds the voxels and counts of gb_voxelmap_build on the same cloud, except
    where a point's fp64 key (the incremental map, like GaussianVoxelMapCPU) differs from its fp32 key (the build): the
    voxels such points fall in are left out of the comparison and the points are counted.  At power-of-two resolutions the
    two keys agree and the maps are identical."""
    pts, cov, _ = frames[3]
    cloud = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
    xyz, _ = oracle.pack_cloud(pts, cov_colmajor16(cov))
    for res in (0.2, 0.5):
        inc = gpu.IncrementalVoxelMapGPU(res, ctx=ctx).insert(cloud)
        built = gpu.GaussianVoxelMapGPU(res, init_num_buckets=16384, ctx=ctx).insert(cloud)
        inv32 = np.float32(1.0) / np.float32(res)
        k32 = np.floor(xyz * inv32).astype(np.int64)
        k64 = np.floor(xyz.astype(np.float64) * (1.0 / float(np.float32(res)))).astype(np.int64)
        differ = (k32 != k64).any(1)
        skip = {tuple(c) for c in k32[differ]} | {tuple(c) for c in k64[differ]}

        def voxels(m):
            b, vnum, _, _ = m.download()
            occ = b[:, 3] >= 0
            return {tuple(c): int(vnum[i]) for c, i in zip(b[occ, :3], b[occ, 3]) if tuple(c) not in skip}

        a, b = voxels(inc), voxels(built)
        assert a == b, res
        print(f"resolution {res}: {int(differ.sum())} of {len(xyz)} points have fp32 and fp64 keys that differ")
        if res == 0.5:
            assert differ.sum() == 0
            assert np.array_equal(inc.download()[0], built.download()[0])


def oracle_map_of(m):
    """An oracle GpuMap with exactly the device map's records: one point per voxel at its fp32 mean with its fp32 covariance
    (the oracle's linearization reads means and covariances only).  Its table must equal the downloaded one."""
    buckets, _, vmean, vcov = m.download()
    ref = oracle.GpuMap(vmean, vcov, m.resolution, init_buckets=16384)
    assert np.array_equal(ref.buckets, buckets) and np.array_equal(ref.vmean, vmean) and np.array_equal(ref.vcov, vcov)
    return ref


def test_consumers_follow_the_map(ctx, frames):
    """A factor (its own sweep), a factor-set sweep and a user gb_sweep, all created and used before an insert, linearize after
    it as a factor created after the insert does (the sweeps' fp64 accumulation order is not fixed, so records agree to 1e-12
    relative and inlier counts exactly), and as the oracle does on the downloaded map (1e-4).  gb_overlap follows too."""
    m = gpu.IncrementalVoxelMapGPU(0.5, ctx=ctx)
    T0 = frames[0][2]
    m.insert(gpu.PointCloudGPU.clone(frames[0][0], frames[0][1], ctx=ctx), T0)
    pts, cov, T1 = frames[1]
    src = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
    xyz1, cov1 = oracle.pack_cloud(pts, cov_colmajor16(cov))
    T = synth.perturb(T1, synth.rng_for(71), 0.01, 0.05)
    f_before = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, m, src, ctx=ctx)
    fset = gpu.NonlinearFactorSetGPU(ctx).add([f_before])
    sweep = gpu.Sweep(ctx, [f_before])
    first = f_before.linearize({0: T})
    assert np.array_equal(fset.linearize_deltas(np.stack([T]))["num_inliers"], [first["num_inliers"]])
    sweep.linearize(np.stack([T]))
    ov_before = gpu.overlap_gpu(m, src, T)
    for k in (1, 2):  # the frame itself and the next one: the map grows
        m.insert(gpu.PointCloudGPU.clone(frames[k][0], frames[k][1], ctx=ctx), frames[k][2])
    f_after = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, m, src, ctx=ctx)
    want = f_after.linearize({0: T})
    assert want["num_inliers"] > first["num_inliers"]  # the source's own frame is in the map now
    got = {
        "factor": f_before.linearize({0: T}),
        "factor_set": gpu.unpack_linearized(fset.linearize_deltas(np.stack([T]))[0]),
        "sweep": gpu.unpack_linearized(sweep.linearize(np.stack([T]))[0]),
    }
    rm = oracle_map_of(m)
    rec, corr = oracle.linearize_gpumap(rm, xyz1, cov1, T)
    ref = oracle.split122(rec)
    scale = util.record_scale(util.factor_hits(rm.vmean, rm.vcov, xyz1, cov1, T, corr))
    for name, g in got.items():
        check_linearized(g, ref, hits=scale)
        assert g["num_inliers"] == want["num_inliers"] == ref["num_inliers"], name
        for key in ("H_ss", "b_s"):
            assert np.abs(g[key] - want[key]).max() <= 1e-12 * np.abs(want[key]).max(), (name, key)
            assert rel_err(g[key], ref[key]) < REL_TOL, (name, key)
        assert abs(g["error"] - want["error"]) <= 1e-12 * want["error"], name
        assert abs(g["error"] - ref["error"]) < REL_TOL * ref["error"], name
    # the factor-set error sweep (same cached sweep, error mode)
    e = fset.error_deltas(np.stack([T]), np.stack([T]))[0]
    assert abs(e - want["error"]) <= 1e-12 * want["error"]
    ov = gpu.overlap_gpu(m, src, T)
    assert ov == oracle.overlap_gpumap([oracle_map_of(m)], xyz1, [T]) and ov > ov_before


def test_device_odometry_loop(ctx):
    """GLIM's scan-to-map odometry on the device: each frame is registered to two incremental maps (0.2 / 0.4 m) with
    gb_vgicp_align (max_iterations 5) from the last estimate times a perturbed ground-truth increment, then inserted into
    both at the estimate (rate 0.1 from frame 5, LRU horizon 100 / cycle 10).  Every frame's pose error stays below the bar."""
    n_frames = 42
    frames = vo.arc_frames(n_frames, 32 * 600)
    world0 = synth.inv_pose(frames[0][2])
    gt = [world0 @ f[2] for f in frames]
    maps = [gpu.IncrementalVoxelMapGPU(r, lru_horizon=100, lru_clear_cycle=10, ctx=ctx) for r in (0.2, 0.4)]
    est = [np.eye(4)]
    cloud = gpu.PointCloudGPU.clone(frames[0][0], frames[0][1], ctx=ctx)
    for mp in maps:
        mp.insert(cloud, est[0], sampling_rate=1.0, seed=0)
    rng = synth.rng_for(88)
    errs = []
    for k in range(1, n_frames):
        cloud = gpu.PointCloudGPU.clone(frames[k][0], frames[k][1], ctx=ctx)
        inc = synth.perturb(synth.inv_pose(gt[k - 1]) @ gt[k], rng, 0.01, 0.1)
        facs = [gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, mp, cloud, ctx=ctx) for mp in maps]
        r = gpu.align_vgicp([facs], [est[-1] @ inc], params={"max_iterations": 5})[0]
        est.append(r["T_target_source"])
        for mp in maps:
            mp.insert(cloud, est[-1], sampling_rate=1.0 if k < 5 else 0.1, seed=k)
        errs.append(pose_error(est[-1], gt[k]))
    et = max(e[0] for e in errs)
    er = max(e[1] for e in errs)
    print(f"device odometry, {n_frames} frames: max translation error {et:.4f} m, max rotation error {np.degrees(er):.4f} deg; "
          f"maps {maps[0].num_voxels} / {maps[1].num_voxels} voxels")
    # bar: about twice the first H100 run's worst frame (0.022 m, 0.043 deg)
    assert et < 0.05 and er < np.radians(0.1), (et, er)


def test_invalid_inputs_are_rejected_before_any_launch(ctx, frames):
    L = capi.lib()
    pts, cov, T = frames[0]
    cloud = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
    m = gpu.IncrementalVoxelMapGPU(0.5, ctx=ctx)
    built = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(cloud)
    good = capi.pose16(T)
    bad = good.copy()
    bad[13] = np.nan
    launches = ctx.kernel_launches
    assert L.gb_voxelmap_insert(ctx.h, built.h, cloud.h, capi.ptr(good), 1.0, 0) == 1  # a built map keeps no sums
    assert L.gb_voxelmap_insert(ctx.h, m.h, cloud.h, capi.ptr(bad), 1.0, 0) == 1
    bad[13] = np.inf
    assert L.gb_voxelmap_insert(ctx.h, m.h, cloud.h, capi.ptr(bad), 1.0, 0) == 1
    for rate in (0.0, -0.5, 1.0000001, float("nan")):
        assert L.gb_voxelmap_insert(ctx.h, m.h, cloud.h, capi.ptr(good), rate, 0) == 1, rate
    assert L.gb_voxelmap_insert(ctx.h, m.h, None, capi.ptr(good), 1.0, 0) == 1
    h = C.c_void_p()
    assert L.gb_voxelmap_create_incremental(ctx.h, 0.5, 16384, 10, 1e-3, 100, 0, C.byref(h)) == 1 and not h.value
    assert L.gb_voxelmap_create_incremental(ctx.h, 0.5, 1000, 10, 1e-3, 100, 10, C.byref(h)) == 1 and not h.value
    assert L.gb_voxelmap_create_incremental(ctx.h, -0.5, 16384, 10, 1e-3, 100, 10, C.byref(h)) == 1 and not h.value
    assert ctx.kernel_launches == launches
    assert m.num_voxels == 0
    if L.gb_device_count() > 1:  # a cloud on another device than the map
        ctx1 = gpu.Context(1)
        other = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx1)
        assert L.gb_voxelmap_insert(ctx.h, m.h, other.h, capi.ptr(good), 1.0, 0) == 1
        assert ctx.kernel_launches == launches
    m.insert(cloud, T)  # the map is still usable
    assert m.num_voxels > 0
