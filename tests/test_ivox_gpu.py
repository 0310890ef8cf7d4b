"""The device iVox and its GICP factor on the H100 (gb_ivox_insert, gb_gicp_factor_create): the map against the numpy
restatement of its rule bit for bit, the factor through every consumer against the fp64 restatement (tests/ivox_oracle.py),
gb_vgicp_align on GICP problems, and GLIM's shipped GICP odometry configuration end to end against ground truth."""
import ctypes as C

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth, workloads
from oracle import oracle
from tests import ivox_oracle as io
from tests import voxelmap_oracle as vo
from tests import util
from tests.util import REL_TOL, check_linearized, cov_colmajor16

pytestmark = pytest.mark.gpu

N_FRAMES = 22
NAN_FRAME = 9
EMPTY_INSERT = 14
MAX_CORR = 2.0


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


def packed(frame):
    return oracle.pack_cloud(frame[0], cov_colmajor16(frame[1]))


def assert_same_ivox(m, R, k):
    coords, counts, xyz, cov6 = m.download()
    assert (m.num_voxels, m.num_points) == (R.num_voxels, R.num_points), k
    assert np.array_equal(coords, R.vcoord), k
    assert np.array_equal(counts, R.counts), k
    assert np.array_equal(xyz, R.xyz), k
    assert np.array_equal(cov6, R.cov6), k


CONFIGS = {
    # GLIM's shipped iVox: 1.0 m, min_dist 0.1, 10 points, mode 1, LRU 100 / 10
    "mode1": dict(res=1.0, min_dist=0.1, cap=10, mode=1, lru=(100, 10)),
    # small cells, a low cap and fast eviction
    "mode7": dict(res=0.5, min_dist=0.05, cap=4, mode=7, lru=(6, 2)),
}


def make_pair(ctx, cfg):
    m = gpu.IVoxGPU(cfg["res"], cfg["min_dist"], cfg["cap"], cfg["mode"], cfg["lru"][0], cfg["lru"][1], ctx=ctx)
    R = io.IVox(cfg["res"], cfg["min_dist"], cfg["cap"], cfg["mode"], cfg["lru"][0], cfg["lru"][1])
    return m, R


@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_insert_sequence_is_bit_exact(ctx, frames, config):
    """After every insert of a sequence at world poses (odometry sampling, a frame with NaN points, an insert that keeps no
    point) the downloaded iVox equals the restatement exactly: voxels, counts, fp32 points and covariances."""
    cfg = CONFIGS[config]
    m, R = make_pair(ctx, cfg)
    shrank = 0
    for k, frame in enumerate(frames):
        cloud = gpu.PointCloudGPU.clone(frame[0], frame[1], ctx=ctx)
        xyz, cov6 = packed(frame)
        before = R.num_voxels
        m.insert(cloud, frame[2], sampling_rate=odometry_rate(k), seed=900 + k)
        R.insert(xyz, cov6, frame[2], odometry_rate(k), seed=900 + k)
        shrank += R.num_voxels < before
        assert_same_ivox(m, R, k)
    assert (R.counts == cfg["cap"]).any()
    if cfg["lru"][0] < N_FRAMES:
        assert shrank > 0


@pytest.fixture(scope="module")
def target(ctx, frames):
    """an iVox (mode 7) of frames 0-2 on the device and restated, and frame 3 as the source"""
    cfg = dict(CONFIGS["mode1"], mode=7)
    m, R = make_pair(ctx, cfg)
    for k in (0, 1, 2):
        cloud = gpu.PointCloudGPU.clone(frames[k][0], frames[k][1], ctx=ctx)
        xyz, cov6 = packed(frames[k])
        m.insert(cloud, frames[k][2])
        R.insert(xyz, cov6, frames[k][2])
    src = gpu.PointCloudGPU.clone(frames[3][0], frames[3][1], ctx=ctx)
    return m, R, src, packed(frames[3]), frames[3][2]


def test_factor_matches_fp64_restatement(ctx, target):
    """Through the factor set at several poses: inlier counts exact, H / b / error within 1e-4 of the fp64 restatement;
    error() with T_lin != T_eval likewise."""
    m, R, src, (xyz, cov6), T3 = target
    rng = synth.rng_for(910)
    poses = [T3] + [synth.perturb(T3, rng, 0.02, 0.3) for _ in range(3)]
    facs = [gpu.IntegratedGICPFactorGPU(np.eye(4), 0, m, src, MAX_CORR, ctx=ctx) for _ in poses]
    fset = gpu.NonlinearFactorSetGPU(ctx).add(facs)
    recs = fset.linearize_deltas(np.stack(poses))
    for i, T in enumerate(poses):
        ref, corr = io.linearize(R, xyz, cov6, T, MAX_CORR)
        assert ref["num_inliers"] > 0, i
        check_linearized(gpu.unpack_linearized(recs[i]), ref, hits=util.factor_hits(R.xyz, R.cov6, xyz, cov6, T, corr))
    T_eval = [synth.perturb(T, rng, 0.005, 0.05) for T in poses]
    errs = fset.error_deltas(np.stack(poses), np.stack(T_eval))
    for i, (Tl, Te) in enumerate(zip(poses, T_eval)):
        ref = io.error(R, xyz, cov6, Tl, Te, MAX_CORR)
        assert abs(errs[i] - ref) < REL_TOL * ref, i
    # the factor's own error(): correspondences of its last linearization point, evaluated at the new values
    facs[0].linearize({0: poses[0]})
    assert abs(facs[0].error({0: T_eval[0]}) - io.error(R, xyz, cov6, poses[0], T_eval[0], MAX_CORR)) < REL_TOL * errs[0]


def test_factor_3km_from_the_origin(ctx, frames):
    """GLIM's odometry keeps its iVox in the world frame: frames 0-2 inserted and frame 3 registered ~3 km from the origin,
    where the fp32 transform rounds q by ~1e-4 m and the adjoint carries the 3 km translation into H_ss, H_ts and b_s.  Inlier
    counts exact and every entry within its own bound (the relative Frobenius bar is not asked of this case: H_ss = Ad^T H_tt
    Ad cancels ~|t|^2 of H_tt's fp32 rounding there)."""
    far = synth.pose(2400.0, -1800.0, 35.0, 0.7)
    cfg = CONFIGS["mode1"]
    m, R = make_pair(ctx, cfg)
    for k in (0, 1, 2):
        m.insert(gpu.PointCloudGPU.clone(frames[k][0], frames[k][1], ctx=ctx), far @ frames[k][2])
        R.insert(*packed(frames[k]), far @ frames[k][2])
    assert_same_ivox(m, R, "3 km")
    src = gpu.PointCloudGPU.clone(frames[3][0], frames[3][1], ctx=ctx)
    xyz, cov6 = packed(frames[3])
    rng = synth.rng_for(916)
    poses = [far @ frames[3][2]] + [synth.perturb(far @ frames[3][2], rng, 0.01, 0.1) for _ in range(2)]
    assert min(np.linalg.norm(T[:3, 3]) for T in poses) > 2900.0
    recs = gpu.NonlinearFactorSetGPU(ctx).add([gpu.IntegratedGICPFactorGPU(np.eye(4), 0, m, src, MAX_CORR, ctx=ctx) for _ in poses]).linearize_deltas(np.stack(poses))
    for i, T in enumerate(poses):
        ref, corr = io.linearize(R, xyz, cov6, T, MAX_CORR)
        got = gpu.unpack_linearized(recs[i])
        assert got["num_inliers"] == ref["num_inliers"] > 1000, i
        print("3 km, relative Frobenius error:", {k: f"{util.rel_err(got[k], ref[k]):.2e}" for k in ("H_tt", "H_ss", "H_ts", "b_t", "b_s")})
        util.check_entrywise(got, ref, util.record_scale(util.factor_hits(R.xyz, R.cov6, xyz, cov6, T, corr)), what=("3 km", i))


def test_consumers_follow_the_ivox(ctx, frames):
    """A factor (its own sweep), a factor-set sweep and a user sweep created and used before an insert linearize after it as
    a factor created after the insert does, and as the restatement does on the new map."""
    cfg = CONFIGS["mode1"]
    m, R = make_pair(ctx, cfg)
    m.insert(gpu.PointCloudGPU.clone(frames[0][0], frames[0][1], ctx=ctx), frames[0][2])
    R.insert(*packed(frames[0]), frames[0][2])
    src = gpu.PointCloudGPU.clone(frames[1][0], frames[1][1], ctx=ctx)
    xyz1, cov1 = packed(frames[1])
    T = synth.perturb(frames[1][2], synth.rng_for(911), 0.01, 0.05)
    f_before = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, m, src, MAX_CORR, ctx=ctx)
    fset = gpu.NonlinearFactorSetGPU(ctx).add([f_before])
    sweep = gpu.Sweep(ctx, [f_before])
    first = f_before.linearize({0: T})
    fset.linearize_deltas(np.stack([T]))
    sweep.linearize(np.stack([T]))
    for k in (1, 2):
        m.insert(gpu.PointCloudGPU.clone(frames[k][0], frames[k][1], ctx=ctx), frames[k][2])
        R.insert(*packed(frames[k]), frames[k][2])
    want = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, m, src, MAX_CORR, ctx=ctx).linearize({0: T})
    assert want["num_inliers"] > first["num_inliers"]
    ref, corr = io.linearize(R, xyz1, cov1, T, MAX_CORR)
    assert ref["num_inliers"] > 0
    scale = util.record_scale(util.factor_hits(R.xyz, R.cov6, xyz1, cov1, T, corr))
    got = {
        "factor": f_before.linearize({0: T}),
        "factor_set": gpu.unpack_linearized(fset.linearize_deltas(np.stack([T]))[0]),
        "sweep": gpu.unpack_linearized(sweep.linearize(np.stack([T]))[0]),
    }
    for name, g in got.items():
        assert g["num_inliers"] == want["num_inliers"], name
        for key in ("H_ss", "b_s"):
            assert np.abs(g[key] - want[key]).max() <= 1e-12 * np.abs(want[key]).max(), (name, key)
        check_linearized(g, ref, hits=scale)


def test_align_matches_restated_lm(ctx, target):
    """gb_vgicp_align on GICP problems agrees with the restated LM within 2e-3 m / rad, and a batch equals the same problems
    run one at a time."""
    m, R, src, (xyz, cov6), T3 = target
    rng = synth.rng_for(912)
    T0 = [synth.perturb(T3, rng, 0.02, 0.25) for _ in range(4)]
    problems = [[gpu.IntegratedGICPFactorGPU(np.eye(4), 0, m, src, MAX_CORR, ctx=ctx)] for _ in T0]
    launches = ctx.kernel_launches
    batch = gpu.align_vgicp(problems, T0)
    launches = ctx.kernel_launches - launches
    assert launches <= 4 * (max(r["trials"] for r in batch) + 1)
    for i, (r, T) in enumerate(zip(batch, T0)):
        ref = io.align(R, xyz, cov6, T, MAX_CORR)
        et, er = pose_error(r["T_target_source"], ref["T"])
        assert et < 2e-3 and er < 2e-3, (i, et, er, r, ref)
        solo = gpu.align_vgicp([problems[i]], [T])[0]
        et, er = pose_error(r["T_target_source"], solo["T_target_source"])
        if (r["iterations"], r["trials"], r["status"]) == (solo["iterations"], solo["trials"], solo["status"]):
            assert et < 1e-6 and er < 1e-6, (i, et, er)
        else:  # a tie at the fp32 noise floor decided differently: within one step tolerance
            assert et < 1e-3 and er < 1e-4, (i, et, er)
        gt, gr = pose_error(r["T_target_source"], T3)
        assert gt < 0.05 and gr < 2e-3, (i, gt, gr)


def test_shipped_gicp_odometry_end_to_end(ctx):
    """GLIM's CPU odometry as shipped (registration_type GICP) on the device: 42 hdl32 frames (19 200 rays) on the arc with
    covariances estimated on the device (k = 10), each frame GICP-aligned into a 1.0 m iVox (min_dist 0.1, mode 1,
    max_correspondence_distance 2.0, max_iterations 8) from the last estimate times a perturbed ground-truth increment, then
    inserted at the estimate (rate 0.1 from frame 5, LRU 100 / 10).
    Bar: about twice the first H100 run's worst frame (0.049 m, 0.13 deg).  That run does not reach the VGICP loop's bar
    (0.05 m, 0.1 deg): one 1.0 m iVox searched in the centre voxel only constrains the rotation less than two fine voxel maps."""
    n_frames = 42
    sc = synth.make_hall_scene()
    traj = synth.arc_trajectory(n_frames)
    world0 = synth.inv_pose(traj[0])
    gt = [world0 @ T for T in traj]
    ivox = gpu.IVoxGPU(1.0, 0.1, 10, 1, 100, 10, ctx=ctx)
    est = [np.eye(4)]
    rng = synth.rng_for(913)
    errs = []
    for k in range(n_frames):
        pts, cov = workloads.make_scan(sc, "hdl32", traj[k], synth.rng_for(914, k), n_rays=32 * 600, ctx=ctx, use_gpu=True)
        cloud = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
        if k > 0:
            inc = synth.perturb(synth.inv_pose(gt[k - 1]) @ gt[k], rng, 0.01, 0.1)
            fac = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, ivox, cloud, 2.0 * ivox.resolution, ctx=ctx)
            r = gpu.align_vgicp([[fac]], [est[-1] @ inc], params={"max_iterations": 8})[0]
            est.append(r["T_target_source"])
            errs.append(pose_error(est[-1], gt[k]))
        ivox.insert(cloud, est[-1], sampling_rate=1.0 if k < 5 else 0.1, seed=k)
    et = max(e[0] for e in errs)
    er = max(e[1] for e in errs)
    print(f"device GICP odometry, {n_frames} frames: max translation error {et:.4f} m, max rotation error {np.degrees(er):.4f} deg; "
          f"iVox {ivox.num_voxels} voxels / {ivox.num_points} points")
    assert et < 0.1 and er < np.radians(0.25), (et, er)


def test_invalid_and_mixed_inputs_are_rejected_before_any_launch(ctx, frames):
    L = capi.lib()
    pts, cov, T = frames[0]
    cloud = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
    m = gpu.IVoxGPU(1.0, ctx=ctx)
    m.insert(cloud, T)
    vmap = gpu.IncrementalVoxelMapGPU(1.0, ctx=ctx).insert(cloud, T)
    built = gpu.GaussianVoxelMapGPU(1.0, ctx=ctx).insert(cloud)
    g = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, m, cloud, MAX_CORR, ctx=ctx)
    v = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, vmap, cloud, ctx=ctx)
    good = capi.pose16(T)
    launches = ctx.kernel_launches
    h = C.c_void_p()
    # mixed kinds: factor set, sweep, align
    arr = (C.c_void_p * 2)(g._handle(), v._handle())
    launches = ctx.kernel_launches
    P2 = capi.pose16(np.stack([T, T]))
    out = np.zeros(2, gpu.LIN_DTYPE)
    assert L.gb_factor_set_linearize(ctx.h, 2, C.cast(arr, C.c_void_p), capi.ptr(P2), capi.ptr(out)) == 1
    assert L.gb_sweep_create(ctx.h, 2, C.cast(arr, C.c_void_p), None, C.byref(h)) == 1 and not h.value
    off = np.array([0, 2], np.uint64)
    res = (capi.AlignResult * 1)()
    assert L.gb_vgicp_align(ctx.h, 1, capi.ptr(off), C.cast(arr, C.c_void_p), capi.ptr(good), C.byref(gpu.align_params()), C.cast(res, C.c_void_p)) == 1
    # pair index and slabs on GICP sweeps
    one = (C.c_void_p * 1)(g._handle())
    pi = np.zeros(1, np.int32)
    assert L.gb_sweep_create(ctx.h, 1, C.cast(one, C.c_void_p), capi.ptr(pi), C.byref(h)) == 1 and not h.value
    sw = gpu.Sweep(ctx, [g])
    assert L.gb_sweep_attach_slab(sw.h, C.c_void_p(sw.results_device_ptr()), 1) == 1
    ps = gpu.PeerSlab(ctx, 1)
    assert L.gb_sweep_attach_peer_slab(sw.h, ps.h) == 1
    # insert / factor arguments
    bad = good.copy()
    bad[13] = np.nan
    assert L.gb_ivox_insert(ctx.h, m.h, cloud.h, capi.ptr(bad), 1.0, 0) == 1
    for rate in (0.0, 1.5, float("nan")):
        assert L.gb_ivox_insert(ctx.h, m.h, cloud.h, capi.ptr(good), rate, 0) == 1
    for d in (0.0, -1.0, float("inf"), float("nan")):
        assert L.gb_gicp_factor_create(ctx.h, m.h, cloud.h, d, C.byref(h)) == 1 and not h.value
    for args in ((0.0, 0.1, 10, 1), (1.0, -0.1, 10, 1), (1.0, 0.1, 0, 1), (1.0, 0.1, 65, 1), (1.0, 0.1, 10, 5)):
        assert L.gb_ivox_create(ctx.h, *args, 100, 10, C.byref(h)) == 1 and not h.value
    assert L.gb_ivox_create(ctx.h, 1.0, 0.1, 10, 1, 100, 0, C.byref(h)) == 1 and not h.value
    # a map of another kind: each entry point takes only the kinds it serves
    for other in (vmap.h, built.h):
        assert L.gb_ivox_insert(ctx.h, other, cloud.h, capi.ptr(good), 1.0, 0) == 1
        assert L.gb_ivox_info(other, None, None, None) == 1
        assert L.gb_ivox_download(other, None, None, None, None) == 1
        assert L.gb_gicp_factor_create(ctx.h, other, cloud.h, MAX_CORR, C.byref(h)) == 1 and not h.value
    assert L.gb_voxelmap_insert(ctx.h, m.h, cloud.h, capi.ptr(good), 1.0, 0) == 1
    assert L.gb_vgicp_factor_create(ctx.h, m.h, cloud.h, 0, C.byref(h)) == 1 and not h.value
    assert L.gb_voxelmap_download(m.h, None, None, None, None) == 1
    assert ctx.kernel_launches == launches
    if L.gb_device_count() > 1:
        ctx1 = gpu.Context(1)
        other = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx1)
        assert L.gb_ivox_insert(ctx.h, m.h, other.h, capi.ptr(good), 1.0, 0) == 1
        assert L.gb_gicp_factor_create(ctx.h, m.h, other.h, MAX_CORR, C.byref(h)) == 1
        assert ctx.kernel_launches == launches
    # still usable; the sweep runs
    sw.linearize(np.stack([T]))
    m.insert(cloud, T)


def test_launches_per_insert_and_align_round(ctx, frames):
    """A GICP insert into a non-empty iVox is 18 launches at rate < 1 (15 at rate 1): stored keys, transform, keys, sampling
    (3), grouping (4), merge, two scans, count, emit, table (3); into an empty one the stored keys are skipped.  With drop
    rate 0 the table is rebuilt at twice the size whenever a voxel is left out: three more launches per extra attempt.  An
    align round is three or four launches."""
    m = gpu.IVoxGPU(1.0, ctx=ctx)

    def insert(k, rate):
        cloud = gpu.PointCloudGPU.clone(frames[k][0], frames[k][1], ctx=ctx)
        l0 = ctx.kernel_launches
        m.insert(cloud, frames[k][2], sampling_rate=rate, seed=k)
        return ctx.kernel_launches - l0

    for k, rate, base in ((0, 1.0, 14), (1, 1.0, 15), (2, 0.1, 18), (3, 0.1, 18)):
        n = insert(k, rate)
        assert n >= base and (n - base) % 3 == 0 and n - base <= 6, (k, n, base)
    src = gpu.PointCloudGPU.clone(frames[4][0], frames[4][1], ctx=ctx)
    fac = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, m, src, MAX_CORR, ctx=ctx)
    fac._handle()
    l0 = ctx.kernel_launches
    r = gpu.align_vgicp([[fac]], [synth.perturb(frames[4][2], synth.rng_for(915), 0.01, 0.1)])[0]
    n = ctx.kernel_launches - l0
    assert n <= 4 * r["trials"] and n >= 3 * r["trials"], (n, r)
