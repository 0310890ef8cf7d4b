"""The device point grid and its GICP factor on the H100 (gb_point_grid_build, gb_gicp_grid_factor_create): the grid against the
numpy restatement of its rule bit for bit, the factor through every consumer against the fp64 restatement (tests/grid_oracle.py),
gb_vgicp_align on grid problems, GLIM's three GICP between-frame recipes on synthetic scenes with ground truth, the kind
refusals, and the launch counts."""
import ctypes as C

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth
from oracle import oracle
from tests import grid_oracle as go
from tests import voxelmap_oracle as vo
from tests import util
from tests.util import REL_TOL, check_linearized, cov_colmajor16, rel_err

pytestmark = pytest.mark.gpu

N_FRAMES = 12
NAN_FRAME = 5
# the recipes' cell size per max correspondence distance: r / cell_size just below 1, so that the search is the 27 cells of
# m = 1 (scripts/bench_align.py, DESIGN.md 4.11)
RECIPE_CELL = 1.05


def pose_error(T, T_ref):
    d = synth.inv_pose(T_ref) @ T
    return float(np.linalg.norm(d[:3, 3])), float(np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1)))


@pytest.fixture(scope="module")
def frames():
    return vo.arc_frames(N_FRAMES, 32 * 200, nan_frame=NAN_FRAME)


def packed(frame):
    return oracle.pack_cloud(frame[0], cov_colmajor16(frame[1]))


def delta(frames, a, b):
    return synth.inv_pose(frames[a][2]) @ frames[b][2]


def submap(ctx, frames, first, count=4, resolution=0.1):
    """frames first .. first + count - 1 merged in the frame of `first` (sub_mapping.cpp:481-497) -> PointCloudGPU"""
    clouds = [gpu.PointCloudGPU.clone(frames[k][0], frames[k][1], ctx=ctx) for k in range(first, first + count)]
    poses = [delta(frames, first, k) for k in range(first, first + count)]
    return gpu.merge_frames_gpu(poses, clouds, resolution, ctx=ctx, host_outputs=False)[2]


def restated(cloud, cell_size):
    xyz, cov6 = cloud.download()
    return go.PointGrid(xyz, cov6, cell_size), xyz, cov6


def assert_same_grid(g, R):
    coords, counts, idx, xyz, cov6 = g.download()
    assert (g.num_cells, g.num_points) == (R.num_cells, R.num_points)
    assert np.array_equal(coords, R.vcoord)
    assert np.array_equal(counts, R.counts)
    assert np.array_equal(idx, R.index)
    assert np.array_equal(xyz, R.xyz, equal_nan=True)
    assert np.array_equal(cov6, R.cov6)


@pytest.mark.parametrize("which", ["frame_with_nan", "submap"])
@pytest.mark.parametrize("cell_size", [0.5, 2.05])
def test_grid_is_bit_exact(ctx, frames, which, cell_size):
    """The downloaded grid equals the restatement: cell coordinates and counts in key order, original indices, fp32 points and
    covariances in record order (the NaN points last).  The cloud may go first."""
    if which == "submap":
        cloud = submap(ctx, frames, 0)
    else:
        cloud = gpu.PointCloudGPU.clone(frames[NAN_FRAME][0], frames[NAN_FRAME][1], ctx=ctx)
    R, xyz, _ = restated(cloud, cell_size)
    g = gpu.PointGridGPU(cloud, cell_size, ctx=ctx)
    del cloud
    assert_same_grid(g, R)
    if which != "submap":
        assert R.num_keyed < R.num_points
    empty = gpu.PointGridGPU(gpu.PointCloudGPU.clone(np.zeros((0, 4)), np.zeros((0, 4, 4)), ctx=ctx), 1.0, ctx=ctx)
    assert (empty.num_cells, empty.num_points) == (0, 0)


@pytest.fixture(scope="module")
def pair(ctx, frames):
    """frame 2 as the target, frame 3 as the source"""
    tgt = gpu.PointCloudGPU.clone(frames[2][0], frames[2][1], ctx=ctx)
    src = gpu.PointCloudGPU.clone(frames[3][0], frames[3][1], ctx=ctx)
    return tgt, src, packed(frames[2]), packed(frames[3]), delta(frames, 2, 3)


@pytest.mark.parametrize("cell_size,want_m", [(1.05, 1), (0.6, 2)])
def test_factor_matches_fp64_restatement(ctx, pair, cell_size, want_m):
    """At m = 1 and m = 2, through gb_vgicp_linearize, a factor set and a sweep at several poses: inlier counts exact, H / b /
    error within 1e-4 of the fp64 restatement; error() with T_lin != T_eval likewise."""
    tgt, src, (xt, ct), (xyz, cov6), T0 = pair
    max_corr = 1.0
    R = go.PointGrid(xt, ct, cell_size)
    g = gpu.PointGridGPU(tgt, cell_size, ctx=ctx)
    rng = synth.rng_for(920)
    poses = [T0] + [synth.perturb(T0, rng, 0.02, 0.3) for _ in range(3)]
    facs = [gpu.IntegratedGICPFactorGPU(np.eye(4), 0, g, src, max_corr, ctx=ctx) for _ in poses]
    assert facs[0].search_half_width() == want_m == go.half_width(R.inv, go.max_d2(max_corr), R.key_extent)
    lin = [go.linearize(R, xyz, cov6, T, max_corr) for T in poses]
    refs = [r for r, _ in lin]
    assert min(r["num_inliers"] for r in refs) > 0
    hits = [util.record_scale(util.factor_hits(R.xyz, R.cov6, xyz, cov6, T, corr)) for T, (_, corr) in zip(poses, lin)]
    check_linearized(facs[0].linearize({0: poses[0]}), refs[0], hits=hits[0])
    recs = gpu.NonlinearFactorSetGPU(ctx).add(facs).linearize_deltas(np.stack(poses))
    swept = gpu.Sweep(ctx, facs).linearize(np.stack(poses))
    for i in range(len(poses)):
        check_linearized(gpu.unpack_linearized(recs[i]), refs[i], hits=hits[i])
        check_linearized(gpu.unpack_linearized(swept[i]), refs[i], hits=hits[i])
    T_eval = [synth.perturb(T, rng, 0.005, 0.05) for T in poses]
    errs = gpu.NonlinearFactorSetGPU(ctx).add(facs).error_deltas(np.stack(poses), np.stack(T_eval))
    for i, (Tl, Te) in enumerate(zip(poses, T_eval)):
        ref = go.error(R, xyz, cov6, Tl, Te, max_corr)
        assert abs(errs[i] - ref) < REL_TOL * ref, i
    assert abs(facs[0].error({0: T_eval[0]}) - go.error(R, xyz, cov6, poses[0], T_eval[0], max_corr)) < REL_TOL * errs[0]


def test_ties_go_to_the_smaller_original_index(ctx):
    """Every source point has two target points at the same fp32 distance on either side along x, in different cells, the one in
    the lower cell with the LARGER original index, and the two with different covariances: only the pick of the smaller index
    gives the restatement's H.  At m = 1 (cell 0.5) and m = 2 (cell 0.3)."""
    rng = np.random.default_rng(930)
    n = 600
    q = np.round(rng.uniform(-100, 100, size=(n, 3)) * 64) / 64  # dyadic: q +- d is exact; sparse: no other point is near
    d = 0.375
    lo, hi = q - [d, 0, 0], q + [d, 0, 0]
    tgt = np.concatenate([hi, lo])  # hi first: the smaller original indices sit in the upper cells
    covs_t = np.zeros((2 * n, 4, 4))
    covs_t[:n, :3, :3] = np.diag([0.01, 0.02, 0.03])
    covs_t[n:, :3, :3] = np.array([[0.05, 0.01, 0.0], [0.01, 0.02, 0.0], [0.0, 0.0, 0.002]])
    src_cov = np.zeros((n, 4, 4))
    src_cov[:, :3, :3] = np.diag([0.02, 0.01, 0.02])
    tp = np.concatenate([tgt, np.ones((2 * n, 1))], 1)
    sp = np.concatenate([q, np.ones((n, 1))], 1)
    tc = gpu.PointCloudGPU.clone(tp, covs_t, ctx=ctx)
    sc = gpu.PointCloudGPU.clone(sp, src_cov, ctx=ctx)
    xt, ct = tc.download()
    xs, cs = sc.download()
    for cell in (0.5, 0.3):
        R = go.PointGrid(xt, ct, cell)
        g = gpu.PointGridGPU(tc, cell, ctx=ctx)
        f = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, g, sc, 0.5, ctx=ctx)
        ref, corr = go.linearize(R, xs, cs, np.eye(4), 0.5)
        assert (R.index[corr] < n).all()  # the restatement picks the upper point every time
        assert ref["num_inliers"] > 0
        check_linearized(f.linearize({0: np.eye(4)}), ref, hits=util.factor_hits(R.xyz, R.cov6, xs, cs, np.eye(4), corr))


@pytest.fixture(scope="module")
def loop_target(ctx, frames):
    """a submap of frames 4-7 as the target grid (cell 1.05, r = 1.0) and frame 8 as the source"""
    cloud = submap(ctx, frames, 4)
    R, _, _ = restated(cloud, 1.05)
    g = gpu.PointGridGPU(cloud, 1.05, ctx=ctx)
    src = gpu.PointCloudGPU.clone(frames[8][0], frames[8][1], ctx=ctx)
    return g, R, src, packed(frames[8]), delta(frames, 4, 8)


def test_align_matches_restated_lm(ctx, loop_target):
    """gb_vgicp_align on grid problems agrees with the restated LM within 2e-3 m / rad, and each of a 64-candidate batch
    ends with its solo call's status and pose (within the same tolerance)."""
    g, R, src, (xyz, cov6), T_gt = loop_target
    rng = synth.rng_for(940)
    T0 = [synth.perturb(T_gt, rng, 0.02, 0.25) for _ in range(64)]
    problems = [[gpu.IntegratedGICPFactorGPU(np.eye(4), 0, g, src, 1.0, ctx=ctx)] for _ in T0]
    batch = gpu.align_vgicp(problems, T0)
    for i in range(2):
        ref = go.align(R, xyz, cov6, T0[i], 1.0)
        et, er = pose_error(batch[i]["T_target_source"], ref["T"])
        assert batch[i]["status"] == ref["status"] and et < 2e-3 and er < 2e-3, (i, et, er, batch[i], ref)
    for i, (r, T) in enumerate(zip(batch, T0)):
        solo = gpu.align_vgicp([problems[i]], [T])[0]
        et, er = pose_error(r["T_target_source"], solo["T_target_source"])
        assert r["status"] == solo["status"] and et < 2e-3 and er < 2e-3, (i, et, er)
        gt, gr = pose_error(r["T_target_source"], T_gt)
        assert gt < 0.05 and gr < 2e-3, (i, gt, gr)


# ---------------------------------------------------------------------------------------------------------------------
# GLIM's three recipes
# ---------------------------------------------------------------------------------------------------------------------
def test_sub_mapping_between_factor(ctx, pair):
    """create_between_factors with between_registration_type GICP (sub_mapping.cpp:189-211): one linearize of the binary factor
    (X(last), X(current)) at the odometry delta; the X(current) block G22 of gb_hessian_blocks matches the restatement's H_ss."""
    tgt, src, (xt, ct), (xyz, cov6), T_delta = pair
    r = 1.0  # [EXT] the factor's default max correspondence distance is not vendored
    g = gpu.PointGridGPU(tgt, RECIPE_CELL * r, ctx=ctx)
    f = gpu.IntegratedGICPFactorGPU(0, 1, g, src, r, ctx=ctx)
    T_odom = synth.perturb(T_delta, synth.rng_for(950), 0.005, 0.02)
    values = {0: synth.pose(1.0, 2.0, 0.0, 0.3), 1: None}
    values[1] = values[0] @ T_odom
    rec = gpu.NonlinearFactorSetGPU(ctx).add([f]).linearize_deltas(np.stack([f.delta(values)]))
    G22, g2, e = np.zeros(36), np.zeros(6), C.c_double()
    capi.check(capi.lib().gb_hessian_blocks(capi.ptr(rec), 1.0, None, None, None, capi.ptr(G22), capi.ptr(g2), C.byref(e)))
    ref = go.linearize(go.PointGrid(xt, ct, RECIPE_CELL * r), xyz, cov6, f.delta(values), r)[0]
    assert rel_err(G22.reshape(6, 6).T, ref["H_ss"]) < REL_TOL
    assert np.linalg.norm(g2 + ref["b_s"]) < REL_TOL * max(np.linalg.norm(ref["b_s"]), 0.1 * np.sqrt(np.trace(ref["H_ss"]) * ref["error"]))
    assert np.linalg.eigvalsh(G22.reshape(6, 6)).min() > 0


def test_global_mapping_between_registration(ctx, frames):
    """create_between_factors of global mapping (global_mapping.cpp:379-428): LM between consecutive submaps (max distance
    0.5, lambdaInitial 1e-12, 10 iterations) from a perturbed delta, then H + 1e6 I at the result.  GLIM's X(0) prior of
    precision 1e6 is taken as a fixed target pose (the unary problem of gb_vgicp_align)."""
    A = submap(ctx, frames, 0)
    B = submap(ctx, frames, 4)
    T_gt = delta(frames, 0, 4)
    r = 0.5
    g = gpu.PointGridGPU(A, RECIPE_CELL * r, ctx=ctx)
    f = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, g, B, r, ctx=ctx)
    for k in range(3):
        T0 = synth.perturb(T_gt, synth.rng_for(960, k), 0.01, 0.1)
        res = gpu.align_vgicp([[f]], [T0], params={"lambda_initial": 1e-12, "max_iterations": 10})[0]
        et, er = pose_error(res["T_target_source"], T_gt)
        e0, _ = pose_error(T0, T_gt)
        assert et < 0.02 and er < np.radians(0.1) and et < e0, (k, et, er, res)
        H = f.linearize({0: res["T_target_source"]})["H_ss"] + 1e6 * np.eye(6)
        assert np.linalg.eigvalsh(H).min() > 1e6 - 1


def test_pose_graph_loop_candidates(ctx, frames):
    """Loop candidates of the pose-graph back-end with registration_type GICP (global_mapping_pose_graph.cpp:391-405): target =
    the whole submap, source = 10 % of the candidate submap, r = 2.0, 10 iterations, all candidates in one gb_vgicp_align; a
    candidate is kept iff num_inliers / n_source >= 0.5.  The true loops are kept, the non-overlapping candidates rejected."""
    r = 2.0
    targets = [gpu.PointGridGPU(submap(ctx, frames, k), RECIPE_CELL * r, ctx=ctx) for k in (0, 4)]
    rng = np.random.default_rng(970)
    problems, T0, truth = [], [], []
    for t, k_t in enumerate((0, 4)):
        for k_s in (2, 6, 8):
            pts = np.concatenate([frames[j][0] for j in (k_s,)])
            covs = np.concatenate([frames[j][1] for j in (k_s,)])
            fin = np.isfinite(pts).all(1)
            keep = np.nonzero(fin)[0][rng.random(fin.sum()) < 0.1]
            src = gpu.PointCloudGPU.clone(pts[keep], covs[keep], ctx=ctx)
            T_true = delta(frames, k_t, k_s)
            overlapping = k_s - k_t in (2, 4) and k_s >= k_t
            if not overlapping:  # a candidate whose source lies nowhere near the target: 60 m above it
                lift = np.eye(4)
                lift[2, 3] = 60.0
                T_true = lift @ T_true
            problems.append([gpu.IntegratedGICPFactorGPU(np.eye(4), 0, targets[t], src, r, ctx=ctx)])
            T0.append(synth.perturb(T_true, rng, 0.01, 0.2))
            truth.append((overlapping, T_true, len(keep)))
    res = gpu.align_vgicp(problems, T0, params={"max_iterations": 10})
    for (overlapping, T_true, n), rr in zip(truth, res):
        kept = rr["num_inliers"] / n >= 0.5
        assert kept == overlapping, (rr, n)
        if overlapping:
            et, er = pose_error(rr["T_target_source"], T_true)
            assert et < 0.05 and er < np.radians(0.25), (et, er)
    assert sum(t[0] for t in truth) >= 3 and sum(not t[0] for t in truth) >= 2


# ---------------------------------------------------------------------------------------------------------------------
# refusals and launch counts
# ---------------------------------------------------------------------------------------------------------------------
def test_invalid_and_mixed_inputs_are_rejected_before_any_launch(ctx, frames):
    L = capi.lib()
    pts, cov, T = frames[0]
    cloud = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
    bare = gpu.PointCloudGPU.clone(pts, ctx=ctx)  # no covariances
    grid = gpu.PointGridGPU(cloud, 1.05, ctx=ctx)
    ivox = gpu.IVoxGPU(1.0, ctx=ctx).insert(cloud)
    vmap = gpu.IncrementalVoxelMapGPU(1.0, ctx=ctx).insert(cloud)
    built = gpu.GaussianVoxelMapGPU(1.0, ctx=ctx).insert(cloud)
    fg = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, grid, cloud, 1.0, ctx=ctx)
    fi = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, ivox, cloud, 1.0, ctx=ctx)
    fv = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, vmap, cloud, ctx=ctx)
    for f in (fg, fi, fv):
        f._handle()
    sw = gpu.Sweep(ctx, [fg])
    ps = gpu.PeerSlab(ctx, 1)
    good = capi.pose16(T)
    P2 = capi.pose16(np.stack([T, T]))
    h = C.c_void_p()
    launches = ctx.kernel_launches
    # mixed target classes: factor set, sweep, align
    for other in (fi, fv):
        arr = (C.c_void_p * 2)(fg._handle(), other._handle())
        out = np.zeros(2, gpu.LIN_DTYPE)
        assert L.gb_factor_set_linearize(ctx.h, 2, C.cast(arr, C.c_void_p), capi.ptr(P2), capi.ptr(out)) == 1
        assert L.gb_factor_set_error(ctx.h, 2, C.cast(arr, C.c_void_p), capi.ptr(P2), capi.ptr(P2), capi.ptr(np.zeros(2))) == 1
        assert L.gb_sweep_create(ctx.h, 2, C.cast(arr, C.c_void_p), None, C.byref(h)) == 1 and not h.value
        off = np.array([0, 1, 2], np.uint64)
        res = (capi.AlignResult * 2)()
        assert L.gb_vgicp_align(ctx.h, 2, capi.ptr(off), C.cast(arr, C.c_void_p), capi.ptr(P2), C.byref(gpu.align_params()), C.cast(res, C.c_void_p)) == 1
    # pair index, slab and peer slab on grid sweeps
    one = (C.c_void_p * 1)(fg._handle())
    assert L.gb_sweep_create(ctx.h, 1, C.cast(one, C.c_void_p), capi.ptr(np.zeros(1, np.int32)), C.byref(h)) == 1 and not h.value
    assert L.gb_sweep_attach_slab(sw.h, C.c_void_p(sw.results_device_ptr()), 1) == 1
    assert L.gb_sweep_attach_peer_slab(sw.h, ps.h) == 1
    # a grid where another kind is expected
    assert L.gb_vgicp_factor_create(ctx.h, grid.h, cloud.h, 0, C.byref(h)) == 1 and not h.value
    assert L.gb_gicp_factor_create(ctx.h, grid.h, cloud.h, 1.0, C.byref(h)) == 1 and not h.value
    assert L.gb_ct_gicp_factor_create(ctx.h, grid.h, cloud.h, 1.0, C.byref(h)) == 1 and not h.value
    assert L.gb_voxelmap_insert(ctx.h, grid.h, cloud.h, capi.ptr(good), 1.0, 0) == 1
    assert L.gb_voxelmap_download(grid.h, None, None, None, None) == 1
    assert L.gb_ivox_insert(ctx.h, grid.h, cloud.h, capi.ptr(good), 1.0, 0) == 1
    assert L.gb_ivox_info(grid.h, None, None, None) == 1
    assert L.gb_ivox_download(grid.h, None, None, None, None) == 1
    targets = (C.c_void_p * 2)(built.h, grid.h)
    ov = C.c_double()
    assert L.gb_overlap(ctx.h, 2, C.cast(targets, C.c_void_p), cloud.h, capi.ptr(P2), C.byref(ov)) == 1
    # another kind where a grid is expected
    for other in (ivox.h, vmap.h, built.h):
        assert L.gb_gicp_grid_factor_create(ctx.h, other, cloud.h, 1.0, C.byref(h)) == 1 and not h.value
        assert L.gb_point_grid_info(other, None, None, None) == 1
        assert L.gb_point_grid_download(other, None, None, None, None, None) == 1
    # invalid arguments
    for cs in (0.0, -1.0, float("nan"), float("inf")):
        assert L.gb_point_grid_build(ctx.h, cloud.h, cs, C.byref(h)) == 1 and not h.value
    for d in (0.0, -1.0, float("nan"), float("inf"), 9.0 * 1.05):
        assert L.gb_gicp_grid_factor_create(ctx.h, grid.h, cloud.h, d, C.byref(h)) == 1 and not h.value
    assert L.gb_gicp_grid_factor_create(ctx.h, grid.h, bare.h, 1.0, C.byref(h)) == 1 and not h.value
    assert ctx.kernel_launches == launches
    if L.gb_device_count() > 1:
        ctx1 = gpu.Context(1)
        other = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx1)
        assert L.gb_point_grid_build(ctx.h, other.h, 1.0, C.byref(h)) == 1 and not h.value
        assert L.gb_gicp_grid_factor_create(ctx.h, grid.h, other.h, 1.0, C.byref(h)) == 1 and not h.value
        assert ctx.kernel_launches == launches
    # valid calls still run: a grid factor on a bare target grid (the target's covariances may be zero), the grid sweep
    assert gpu.PointGridGPU(bare, 1.05, ctx=ctx).num_points == len(pts)
    sw.linearize(np.stack([T]))
    assert gpu.overlap_gpu(built, cloud, T) > 0


def test_launches_per_build_and_align_round(ctx, frames):
    """A build is 9 launches (k_point_keys, grouping (3: sort, flags, scan), starts, k_grid_emit, table (3)), three more per
    extra table attempt; an empty cloud's is the table's two (clear, finalize).  A grid factor's linearize is one launch (a
    graph), and an align round three or four."""
    cloud = gpu.PointCloudGPU.clone(frames[0][0], frames[0][1], ctx=ctx)
    for cell in (0.3, 1.05, 2.05):
        l0 = ctx.kernel_launches
        g = gpu.PointGridGPU(cloud, cell, ctx=ctx)
        n = ctx.kernel_launches - l0
        assert n >= 9 and (n - 9) % 3 == 0 and n - 9 <= 6, (cell, n)
    empty = gpu.PointCloudGPU.clone(np.zeros((0, 4)), np.zeros((0, 4, 4)), ctx=ctx)
    l0 = ctx.kernel_launches
    gpu.PointGridGPU(empty, 1.0, ctx=ctx)
    assert ctx.kernel_launches - l0 == 2
    src = gpu.PointCloudGPU.clone(frames[1][0], frames[1][1], ctx=ctx)
    f = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, g, src, 2.0, ctx=ctx)
    T = synth.perturb(delta(frames, 0, 1), synth.rng_for(980), 0.01, 0.1)
    f.linearize({0: T})
    l0 = ctx.kernel_launches
    f.linearize({0: T})
    assert ctx.kernel_launches - l0 == 1
    l0 = ctx.kernel_launches
    r = gpu.align_vgicp([[f]], [T])[0]
    n = ctx.kernel_launches - l0
    assert 3 * r["trials"] <= n <= 4 * r["trials"], (n, r)
