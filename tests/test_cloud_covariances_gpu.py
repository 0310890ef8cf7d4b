"""gb_cloud_estimate_covariances on the H100: a device cloud's covariances and normals from its own k nearest neighbours, written
back into the cloud.  Checked bit for bit against the host composition gb_find_neighbors -> gb_covariances -> gb_cloud_upload
on the downloaded positions; independently against the C oracle's brute-force k-NN and covariance estimation (and scipy's
cKDTree off ties); for its side effects (covariance flag, normals block, FPFH features); in GLIM's three call sites (the
manual loop closure's merged map, the map editor's min-cut participants, SubMap::load); and for its refusals and launch counts."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial import cKDTree

from glim_b200 import capi, gpu, preprocess, synth
from oracle import oracle
from tests import global_oracle as gl
from tests import mincut_oracle as mo
from tests import voxelmap_oracle as vo
from tests.test_global_gpu import pose_error
from tests.test_mincut_gpu import DEFAULTS, plane, pole

pytestmark = pytest.mark.gpu
F32, F64, U32 = np.float32, np.float64, np.uint32
COV, NRM = capi.GB_CLOUD_COVARIANCES, capi.GB_CLOUD_NORMALS
UPPER = ([0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2])


def h4(xyz):
    """fp32 (or fp64) positions -> (N, 4) fp64 with w = 1: the widening of the rule"""
    xyz = np.asarray(xyz, F64)
    return np.c_[xyz, np.ones(len(xyz))]


def cov44(cov6):
    """(N, 6) upper triangles -> (N, 4, 4) fp64 [i, row, col]"""
    c = np.zeros((len(cov6), 4, 4))
    for e, (r, q) in enumerate(zip(*UPPER)):
        c[:, r, q] = c[:, q, r] = np.asarray(cov6, F64)[:, e]
    return c


def has_normals(cloud):
    p = C.c_void_p()
    capi.check(capi.lib().gb_cloud_device_ptrs(cloud.h, None, None, None, C.byref(p)))
    return bool(p.value)


def has_covariances(ctx, grid, cloud):
    """whether a GICP factor on a point grid, which needs a source with covariances, takes the cloud (the factor is destroyed
    again)"""
    L = capi.lib()
    h = C.c_void_p()
    st = L.gb_gicp_grid_factor_create(ctx.h, grid.h, cloud.h, 1.0, C.byref(h))
    if st == 0:
        L.gb_vgicp_factor_destroy(h)
    return st == 0


def state(cloud):
    """(xyz, cov6, normals or None) in the caller's order, as stored"""
    xyz, cov6 = cloud.download()
    return xyz, cov6, (cloud.normals() if has_normals(cloud) else None)


def assert_same_bits(a, b, what):
    """bit-identical fp32 arrays; a NaN must be a NaN in both"""
    a, b = np.ascontiguousarray(a, F32), np.ascontiguousarray(b, F32)
    assert a.shape == b.shape, what
    na, nb = np.isnan(a), np.isnan(b)
    assert np.array_equal(na, nb), what
    assert np.array_equal(a.view(U32)[~na], b.view(U32)[~nb]), what


def assert_same_state(got, want, what):
    for name, g, w in zip(("positions", "covariances", "normals"), got, want):
        assert (g is None) == (w is None), (what, name)
        if g is not None:
            assert_same_bits(g, w, (what, name))


def composition(ctx, before, had_covs, k, outputs):
    """gb_cloud_upload(widened positions, gb_covariances(gb_find_neighbors(...))) with the planes the call keeps -> (cloud, rows)"""
    xyz, cov6, nrm = before
    p4 = h4(xyz)
    nb = preprocess.find_neighbors(p4, k, ctx=ctx)
    n4, covs = preprocess.CloudCovarianceEstimation(ctx=ctx).estimate(p4, nb)
    c = covs if outputs & COV else (cov44(cov6) if had_covs else None)
    nr = n4 if outputs & NRM else (np.c_[nrm.astype(F64), np.zeros(len(nrm))] if nrm is not None else None)
    return gpu.PointCloudGPU.clone(p4, c, nr, ctx=ctx), nb.reshape(len(xyz), k)


@pytest.fixture(scope="module")
def clouds():
    """a synthetic hall scan; random points; the hall with duplicated points, NaN points and one point outside the k-NN's
    21-bit range -> {name: (points (N, 4), normals (N, 4), covs (N, 4, 4))}"""
    rng = np.random.default_rng(11)
    hall = vo.arc_frames(1, 32 * 150)[0][0]
    rand = h4(rng.uniform(-20.0, 20.0, size=(3000, 3)))
    dup = vo.arc_frames(2, 32 * 60)[1][0]
    dup = np.concatenate([dup, dup[rng.integers(0, len(dup), 400)], dup[:5], dup[:5]])
    dup[::9, :3] = np.nan
    dup = np.concatenate([dup, [[3.0e5, 1.0, 2.0, 1.0]]])
    out = {}
    for name, p in (("hall", hall), ("random", rand), ("dup_nan", dup)):
        nrm, cov = synth.with_covariances(np.nan_to_num(p, nan=1e4), 10)
        out[name] = (np.ascontiguousarray(p), nrm, cov)
    return out


def upload(ctx, c, with_covs, with_normals):
    p, nrm, cov = c
    return gpu.PointCloudGPU.clone(p, cov if with_covs else None, nrm if with_normals else None, ctx=ctx)


@pytest.mark.parametrize("name", ["hall", "random", "dup_nan"])
def test_composition_bit_for_bit(ctx, clouds, name):
    """Every outputs value, k in {1, 10, 20, 32}, the cloud uploaded with and without covariances and normals: positions,
    covariances and normals equal the host composition's upload bit for bit, and the planes not asked for keep their values."""
    for with_covs in (False, True):
        for with_normals in (False, True):
            for k in (1, 10, 20, 32):
                for outputs in (COV, NRM, COV | NRM):
                    what = (name, with_covs, with_normals, k, outputs)
                    cloud = upload(ctx, clouds[name], with_covs, with_normals)
                    before = state(cloud)
                    if outputs & COV:
                        assert cloud.estimate_covariances(k, normals=bool(outputs & NRM)) is cloud
                    else:
                        assert cloud.estimate_normals(k) is cloud
                    ref, _ = composition(ctx, before, with_covs, k, outputs)
                    got = state(cloud)
                    assert_same_state(got, state(ref), what)
                    assert_same_bits(got[0], before[0], what)
                    if not outputs & COV:
                        assert_same_bits(got[1], before[1], what)
                    if not outputs & NRM:
                        assert (got[2] is None) == (before[2] is None), what
                        if got[2] is not None:
                            assert_same_bits(got[2], before[2], what)


@pytest.mark.parametrize("name", ["hall", "random", "dup_nan"])
@pytest.mark.parametrize("k", [10, 20])
def test_against_the_oracle(ctx, clouds, name, k):
    """The rows equal the oracle's brute-force k-NN (for every finite, in-range query; the others are their own index k times)
    and, off exact ties, scipy's cKDTree; covariances and normals are within fp32 tolerance of the oracle's estimation on the
    downloaded positions."""
    cloud = upload(ctx, clouds[name], False, False).estimate_covariances(k, normals=True)
    xyz, cov6, nrm = state(cloud)
    p4 = h4(xyz)
    rows = preprocess.find_neighbors(p4, k, ctx=ctx).reshape(-1, k)
    ok = np.isfinite(xyz).all(1) & (np.abs(p4[:, :3]) < 2.0e5).all(1)
    keep = np.nonzero(ok)[0]  # the brute force over the finite, in-range points: the others are nobody's neighbour
    bf, _ = oracle.knn_bruteforce(p4[ok], k)
    assert np.array_equal(rows[ok], keep[bf])
    assert (rows[~ok] == np.arange(len(xyz))[~ok, None]).all()
    d, idx = cKDTree(p4[ok, :3]).query(p4[ok, :3], k + 1)
    distinct = (np.diff(d, axis=1) > 1e-9 * (1.0 + d[:, 1:])).all(1)
    assert distinct.sum() >= 50  # a scan's regular geometry and the planted duplicates tie many rows
    assert np.array_equal(np.nonzero(ok)[0][idx[distinct, :k]], rows[ok][distinct])
    on, oc = oracle.covariance_estimate(p4, rows)
    fin = ok & np.isfinite(cov6).all(1)
    assert fin.sum() == ok.sum()
    close_c = np.isclose(cov6[fin], oc[fin][:, UPPER[0], UPPER[1]], rtol=1e-5, atol=1e-6).all(1)
    close_n = np.isclose(nrm[fin], on[fin, :3], rtol=1e-5, atol=1e-6).all(1)
    # the eigen solver may amplify the last fp64 bits of atan2 / cos / sin on a degenerate neighbourhood
    assert close_c.mean() > 0.999 and close_n.mean() > 0.999, (close_c.mean(), close_n.mean())


def test_side_effects(ctx, clouds):
    """Covariances alone keep normals and FPFH features; normals discard the features.  A cloud without covariances is refused as
    a GICP source (gb_gicp_grid_factor_create) until covariances are estimated, normals alone not sufficing; then it is
    accepted, and as a VGICP source it linearizes exactly like an upload of the same values."""
    c = upload(ctx, clouds["hall"], True, True).estimate_fpfh(1.0)
    f0 = c.fpfh()
    c.estimate_covariances(10)
    assert np.array_equal(c.fpfh(), f0)
    c.estimate_normals(k=10)
    with pytest.raises(capi.GlimB200Error):
        c.fpfh()
    c.estimate_fpfh(1.0).estimate_covariances(10, normals=True)
    with pytest.raises(capi.GlimB200Error):
        c.fpfh()

    hall = upload(ctx, clouds["hall"], True, False)
    target = gpu.GaussianVoxelMapGPU(1.0, ctx=ctx).insert(hall)
    grid = gpu.PointGridGPU(hall, 1.05, ctx=ctx)
    bare = upload(ctx, clouds["hall"], False, False)
    assert not has_covariances(ctx, grid, bare)
    bare.estimate_normals(k=10)  # normals alone do not make covariances
    assert not has_covariances(ctx, grid, bare)
    bare.estimate_covariances(10)
    assert has_covariances(ctx, grid, bare)
    xyz, cov6, _ = state(bare)
    twin = gpu.PointCloudGPU.clone(h4(xyz), cov44(cov6), ctx=ctx)
    T = synth.pose(0.05, -0.03, 0.02, 0.01, 0.005, -0.004)
    a = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, target, bare, ctx=ctx).linearize({0: T})
    b = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, target, twin, ctx=ctx).linearize({0: T})
    assert a["num_inliers"] > 1000
    for key in a:
        assert np.array_equal(a[key], b[key]), key


def test_manual_loop_closure_on_the_device(ctx):
    """ManualLoopCloseModal::preprocess_maps without the host: iVox -> voxel_data() -> estimate_covariances(10, normals=True)
    gives the planes of test_global_gpu's merged_map (download, k-NN, covariances, upload) bit for bit; FPFH + RANSAC + fine
    GICP on the device-made maps then recover the pose within test_manual_loop_closure_recipe's bars."""
    fr = vo.arc_frames(16, 32 * 400)
    ivs = []
    for part in (fr[:10], fr[6:]):
        iv = gpu.IVoxGPU(2.5, min_dist_in_cell=0.5, max_points_in_cell=50, lru_horizon=1000000, ctx=ctx)
        for pts, cov, T in part:
            iv.insert(gpu.PointCloudGPU.clone(pts, cov, ctx=ctx), T)
        ivs.append(iv)
        host = h4(iv.download()[2])
        nb = preprocess.find_neighbors(host, 10, ctx=ctx)
        n4, covs = preprocess.CloudCovarianceEstimation(ctx=ctx).estimate(host, nb)
        dev = iv.voxel_data().estimate_covariances(10, normals=True)
        assert_same_state(state(dev), state(gpu.PointCloudGPU.clone(host, covs, n4, ctx=ctx)), "merged map")
    for dof in (4, 6):
        T_gt = synth.pose(15.0, -10.0, 0.5, np.radians(120), *((np.radians(3), np.radians(-2)) if dof == 6 else (0.0, 0.0)))
        tgt = ivs[0].voxel_data().estimate_covariances(10, normals=True).estimate_fpfh(5.0)
        src = ivs[1].voxel_data(synth.inv_pose(T_gt)).estimate_covariances(10, normals=True).estimate_fpfh(5.0)
        res = gpu.estimate_pose_ransac(tgt, src, dof=dof)
        et0, er0 = pose_error(res["T_target_source"], T_gt)
        grid = gpu.PointGridGPU(tgt, 1.05, ctx=ctx)
        f = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, grid, src, 1.0, ctx=ctx)
        fine = gpu.align_vgicp([[f]], [res["T_target_source"]], params={"max_iterations": 30})[0]
        et, er = pose_error(fine["T_target_source"], T_gt)
        print(f"dof {dof}: ransac {res['status_name']} err {et0:.3f} m {er0:.3f} deg; fine {fine['status_name']} err {et:.5f} m {er:.5f} deg")
        assert res["status"] in (gl.FOUND, gl.EARLY_STOP)
        assert et0 < 0.35 and er0 < 0.5, (dof, et0, er0)
        assert et < 1e-3 and er < 2e-3, (dof, et, er)


def test_editor_min_cut_on_knn_normals(ctx):
    """PointsSelector::select_points_segmentation: a concat_frames window, the participants within background_mask_radius + 1
    of the picked point (select_radius INSIDE, remove_points of the rest), estimate_normals(k=20), min_cut.  The selection
    equals the min-cut oracle's on the same positions and normals."""
    rng = np.random.default_rng(7)
    poses, frames = [], []
    for k in range(6):
        T = np.eye(4)
        yaw = rng.uniform(-np.pi, np.pi)
        T[:2, :2] = [[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]]
        T[:3, 3] = [6.0 * (k % 3), 6.0 * (k // 3), 0.0]
        parts = [plane(rng, (T[0, 3] - 4, T[1, 3] - 4), (T[0, 3] + 4, T[1, 3] + 4), 0.12, 2, 0.0)]
        if k == 1:
            parts.append(pole(rng, (6.0, 0.0)))
        Pw = np.concatenate([q for q, _ in parts])
        local = h4(((Pw - T[:3, 3]) @ T[:3, :3]).astype(F32))
        _, covs = synth.with_covariances(local, 10)
        poses.append(T)
        frames.append(gpu.PointCloudGPU.clone(local, covs, ctx=ctx))
    picked = np.array([6.15, 0.0, 1.0])
    c = np.floor(picked / 2.0).astype(int)
    cloud, _ = gpu.concat_frames(poses, frames, window=(2.0, tuple(c - 5), tuple(c + 5)), ctx=ctx)
    inside = gpu.select_radius(cloud, picked, "inside", radius=DEFAULTS["background_mask_radius"] + 1.0)["selected"]
    rest = np.setdiff1d(np.arange(cloud.n), inside).astype(np.uint64)
    part = gpu.remove_points([cloud], rest, ctx=ctx)["frames"][0]
    assert part.n == len(inside) > 1000
    part.estimate_normals(k=20)
    got = gpu.min_cut(part, picked, ctx=ctx)
    xyz, _ = part.download()
    ref = mo.min_cut(xyz, part.normals(), picked, **DEFAULTS)
    assert got["status"] == capi.MINCUT_FOUND and got["num_selected"] > 300
    assert np.array_equal(got["selected"], ref["selected"])


def test_submap_load_recipe(ctx):
    """SubMap::load of a submap whose covariances are missing: a gb_merge_frames submap uploaded without covariances ->
    estimate_covariances(10) -> voxel map + VGICP factor linearizes exactly like the submap uploaded with those covariances."""
    fr = vo.arc_frames(4, 32 * 200)
    frames = [gpu.PointCloudGPU.clone(p, c, ctx=ctx) for p, c, _ in fr]
    T0 = synth.inv_pose(fr[0][2])
    pts, _, _ = gpu.merge_frames_gpu([T0 @ T for _, _, T in fr], frames, 0.25, ctx=ctx)
    sub = gpu.PointCloudGPU.clone(pts, ctx=ctx).estimate_covariances(10)
    xyz, cov6, _ = state(sub)
    p4 = h4(xyz)
    _, covs = preprocess.CloudCovarianceEstimation(ctx=ctx).estimate(p4, preprocess.find_neighbors(p4, 10, ctx=ctx))
    ref = gpu.PointCloudGPU.clone(p4, covs, ctx=ctx)
    assert_same_state(state(sub), state(ref), "submap")
    src = frames[3]
    T = T0 @ fr[3][2] @ synth.pose(0.03, -0.02, 0.01, 0.004, -0.002, 0.003)
    for res in (0.5, 1.0):
        ma, mb = gpu.GaussianVoxelMapGPU(res, ctx=ctx).insert(sub), gpu.GaussianVoxelMapGPU(res, ctx=ctx).insert(ref)
        for x, y in zip(ma.download(), mb.download()):
            assert np.array_equal(x, y)
        a = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, ma, src, ctx=ctx).linearize({0: T})
        b = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, mb, src, ctx=ctx).linearize({0: T})
        c = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, gpu.GaussianVoxelMapGPU(res, ctx=ctx).insert(src), sub, ctx=ctx).linearize({0: np.linalg.inv(T)})
        d = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, gpu.GaussianVoxelMapGPU(res, ctx=ctx).insert(src), ref, ctx=ctx).linearize({0: np.linalg.inv(T)})
        assert a["num_inliers"] > 1000 and c["num_inliers"] > 1000
        for key in a:
            assert np.array_equal(a[key], b[key]) and np.array_equal(c[key], d[key]), key


def test_refusals_and_launch_counts(ctx, clouds):
    """Each refusal leaves the launch counter and the cloud unchanged; an empty cloud makes no launch; any other makes 8."""
    L = capi.lib()
    cloud = upload(ctx, clouds["hall"], False, True).estimate_fpfh(1.0)
    before, f0 = state(cloud), cloud.fpfh()
    launches = ctx.kernel_launches
    assert L.gb_cloud_estimate_covariances(None, cloud.h, 10, COV) == 1
    assert L.gb_cloud_estimate_covariances(ctx.h, None, 10, COV) == 1
    for k in (0, -1, 11, 13, 14, 17, 33, 64):
        assert L.gb_cloud_estimate_covariances(ctx.h, cloud.h, k, NRM) == 1, k
    for outputs in (0, 4, 7, -1, -3):
        assert L.gb_cloud_estimate_covariances(ctx.h, cloud.h, 10, outputs) == 1, outputs
    if L.gb_device_count() > 1:
        other = gpu.Context(1)
        assert L.gb_cloud_estimate_covariances(other.h, cloud.h, 10, COV) == 1
    assert ctx.kernel_launches == launches
    assert_same_state(state(cloud), before, "refused")
    assert np.array_equal(cloud.fpfh(), f0)
    assert not has_covariances(ctx, gpu.PointGridGPU(cloud, 1.05, ctx=ctx), cloud)  # still a cloud without covariances

    empty = gpu.PointCloudGPU.clone(np.zeros((0, 4)), ctx=ctx)
    for outputs in (COV, NRM, COV | NRM):
        l0 = ctx.kernel_launches
        capi.check(L.gb_cloud_estimate_covariances(ctx.h, empty.h, 10, outputs))
        assert ctx.kernel_launches == l0
    rng = np.random.default_rng(3)
    for n in (1, 1000, 100_000):
        c = gpu.PointCloudGPU.clone(h4(rng.uniform(-30, 30, size=(n, 3))), ctx=ctx)
        for k, outputs in ((1, COV), (10, COV | NRM), (32, NRM)):
            l0 = ctx.kernel_launches
            capi.check(L.gb_cloud_estimate_covariances(ctx.h, c.h, k, outputs))
            assert ctx.kernel_launches - l0 == 8, (n, k, outputs)


def test_refuses_n_times_k_at_2_pow_30(ctx):
    """N * k >= 2^30 is refused before any launch (N = 2^25 + 1 at k = 32 and 2^25 at k = 32); k = 1 on the same cloud runs."""
    L = capi.lib()
    n = (1 << 25) + 1
    pts = np.zeros((n, 4))
    pts[:, 0] = np.arange(n) * 1e-3
    pts[:, 3] = 1.0
    big = gpu.PointCloudGPU.clone(pts, ctx=ctx)
    edge = gpu.PointCloudGPU.clone(pts[:-1], ctx=ctx)
    del pts
    l0 = ctx.kernel_launches
    assert L.gb_cloud_estimate_covariances(ctx.h, big.h, 32, COV) == 1
    assert L.gb_cloud_estimate_covariances(ctx.h, edge.h, 32, COV) == 1
    assert ctx.kernel_launches == l0
    capi.check(L.gb_cloud_estimate_covariances(ctx.h, big.h, 1, COV))
    assert ctx.kernel_launches - l0 == 8
