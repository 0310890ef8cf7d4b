"""GPU parity tests proper: the CUDA path, called through the C-ABI (libglim_b200.so), against the CPU oracle
on the same seeded inputs.  Bar (north_star): voxel coordinates / indices / inlier sets bit-exact, Hessians /
gradients / errors within 1e-4 relative (Frobenius) of the fp64 oracle.
"""
import numpy as np
import pytest

from oracle import oracle
from glim_b200 import gpu, synth
from tests import util
from tests.util import check_linearized

pytestmark = pytest.mark.gpu

REL_TOL = util.REL_TOL  # 1e-4, north_star


@pytest.fixture(scope="module")
def pair():
    return util.scan_pair()


@pytest.fixture(scope="module")
def dev(ctx, pair):
    """Clouds on the GPU + oracle twins of the device-layout data."""
    d = {"cloud": [], "xyz": [], "cov6": []}
    for P, Cv, N in zip(pair["points"], pair["covs"], pair["normals"]):
        d["cloud"].append(gpu.PointCloudGPU.clone(P, Cv, N, ctx=ctx))
        xyz, cov6 = oracle.pack_cloud(P, util.cov_colmajor16(Cv))
        d["xyz"].append(xyz)
        d["cov6"].append(cov6)
    d["T_gt"] = synth.inv_pose(pair["poses"][0]) @ pair["poses"][1]
    return d


def test_cloud_upload_is_bit_exact(dev):
    for c, xyz, cov6 in zip(dev["cloud"], dev["xyz"], dev["cov6"]):
        gx, gc = c.download()
        assert np.array_equal(gx, xyz) and np.array_equal(gc, cov6)


@pytest.mark.parametrize("res", [0.1, 0.25, 0.5, 1.0])
def test_voxelmap_build_is_bit_exact(ctx, dev, res):
    m = gpu.GaussianVoxelMapGPU(res, ctx=ctx).insert(dev["cloud"][0])
    ref = oracle.GpuMap(dev["xyz"][0], dev["cov6"][0], res)
    assert (m.num_voxels, m.num_buckets) == (ref.num_voxels, ref.num_buckets)
    buckets, vnum, vmean, vcov = m.download()
    assert np.array_equal(buckets, ref.buckets)  # coordinates, voxel numbering and bucket placement
    assert np.array_equal(vnum, ref.vnum)
    assert np.array_equal(vmean, ref.vmean) and np.array_equal(vcov, ref.vcov)  # fp32 sums in the same order


def test_voxelmap_growth_loop_matches_oracle(ctx):
    rng = synth.rng_for(12)
    pts = rng.uniform(-200, 200, size=(60000, 3))
    P = np.concatenate([pts, np.ones((len(pts), 1))], axis=1)
    C = np.tile(np.diag([1.0, 1.0, 1.0, 0.0]), (len(P), 1, 1))
    cloud = gpu.PointCloudGPU.clone(P, C, ctx=ctx)
    xyz, cov6 = oracle.pack_cloud(P, util.cov_colmajor16(C))
    for init in (1024, 16384):
        m = gpu.GaussianVoxelMapGPU(0.5, init_num_buckets=init, ctx=ctx).insert(cloud)
        ref = oracle.GpuMap(xyz, cov6, 0.5, init_buckets=init)
        assert (m.num_voxels, m.num_buckets) == (ref.num_voxels, ref.num_buckets)
        assert np.array_equal(m.download()[0], ref.buckets)


@pytest.mark.parametrize("res", [0.25, 0.5, 0.1])
def test_linearize_matches_oracle(ctx, dev, res):
    m = gpu.GaussianVoxelMapGPU(res, ctx=ctx).insert(dev["cloud"][0])
    ref_map = oracle.GpuMap(dev["xyz"][0], dev["cov6"][0], res)
    # binary factor: keys 0 (target) and 1 (source)
    fac = gpu.IntegratedVGICPFactorGPU(0, 1, m, dev["cloud"][1], ctx=ctx)
    for T in util.test_poses(dev["T_gt"], 4, key=int(res * 100)):
        got = fac.linearize({0: np.eye(4), 1: T})
        ref, corr = oracle.linearize_gpumap(ref_map, dev["xyz"][1], dev["cov6"][1], T)
        assert ref[121] > 300  # enough inliers for the comparison to mean something (sparse 5 k-point test scans)
        check_linearized(got, ref, hits=util.factor_hits(ref_map.vmean, ref_map.vcov, dev["xyz"][1], dev["cov6"][1], T, corr))


def test_linearize_adversarial_poses(ctx, dev):
    """identity, 180 deg yaw, large translations (hash wrap, negative coordinates), no overlap at all."""
    m = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(dev["cloud"][0])
    ref_map = oracle.GpuMap(dev["xyz"][0], dev["cov6"][0], 0.5)
    fac = gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, m, dev["cloud"][1], ctx=ctx)  # unary form
    poses = [np.eye(4), synth.pose(0, 0, 0, np.pi), synth.pose(3.0, -2.0, 0.1, 0.3, 0.02, -0.01), synth.pose(-7.5, 4.25, 0.0, -2.0)]
    for T in poses:
        got = fac.linearize({1: T})
        ref, corr = oracle.linearize_gpumap(ref_map, dev["xyz"][1], dev["cov6"][1], T)
        check_linearized(got, ref, hits=util.factor_hits(ref_map.vmean, ref_map.vcov, dev["xyz"][1], dev["cov6"][1], T, corr))
    far = synth.pose(5000.0, -3000.0, 100.0, 1.0)
    got = fac.linearize({1: far})
    assert got["num_inliers"] == 0 and got["error"] == 0 and not got["H_ss"].any()


def test_unary_and_binary_forms_agree(ctx, dev):
    m = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(dev["cloud"][0])
    Tt = synth.pose(10.0, -4.0, 0.5, 0.7, 0.01, 0.02)
    Ts = Tt @ dev["T_gt"]
    a = gpu.IntegratedVGICPFactorGPU(0, 1, m, dev["cloud"][1], ctx=ctx).linearize({0: Tt, 1: Ts})
    b = gpu.IntegratedVGICPFactorGPU(Tt, 1, m, dev["cloud"][1], ctx=ctx).linearize({1: Ts})
    for k in ("H_ss", "b_s", "H_tt"):
        assert util.rel_err(a[k], b[k]) < 1e-6


def test_binary_factor_between_poses_3km_out(ctx, dev):
    """A binary factor whose two world poses are ~3 km from the origin: the device sees only their delta, which is local, so
    every entry of the record stays within its own bound of the oracle at that delta."""
    res = 0.5
    m = gpu.GaussianVoxelMapGPU(res, ctx=ctx).insert(dev["cloud"][0])
    ref_map = oracle.GpuMap(dev["xyz"][0], dev["cov6"][0], res)
    fac = gpu.IntegratedVGICPFactorGPU(0, 1, m, dev["cloud"][1], ctx=ctx)
    Tt = synth.pose(2400.0, -1800.0, 35.0, 0.7, 0.01, -0.02)
    for T in util.test_poses(dev["T_gt"], 2, key=3000):
        values = {0: Tt, 1: Tt @ T}
        d = fac.delta(values)
        got = fac.linearize(values)
        ref, corr = oracle.linearize_gpumap(ref_map, dev["xyz"][1], dev["cov6"][1], d)
        assert ref[121] > 300
        check_linearized(got, ref, hits=util.factor_hits(ref_map.vmean, ref_map.vcov, dev["xyz"][1], dev["cov6"][1], d, corr))


def test_error_matches_oracle(ctx, dev):
    m = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(dev["cloud"][0])
    ref_map = oracle.GpuMap(dev["xyz"][0], dev["cov6"][0], 0.5)
    fac = gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, m, dev["cloud"][1], ctx=ctx)
    T_lin = dev["T_gt"]
    lin = fac.linearize({1: T_lin})
    assert abs(fac.error({1: T_lin}) - lin["error"]) <= 1e-5 * lin["error"]
    for T_eval in util.test_poses(dev["T_gt"], 3, key=5)[1:]:
        e = fac.error({1: T_eval})
        ref = oracle.error_gpumap(ref_map, dev["xyz"][1], dev["cov6"][1], T_lin, T_eval)
        assert abs(e - ref) <= REL_TOL * ref


def test_overlap_matches_oracle(ctx, dev):
    maps = [gpu.GaussianVoxelMapGPU(r, ctx=ctx).insert(dev["cloud"][0]) for r in (0.5, 1.0)]
    refs = [oracle.GpuMap(dev["xyz"][0], dev["cov6"][0], r) for r in (0.5, 1.0)]
    T = dev["T_gt"]
    far = synth.pose(900.0, 0, 0, 0)
    assert gpu.overlap_gpu(maps[0], dev["cloud"][1], T) == oracle.overlap_gpumap([refs[0]], dev["xyz"][1], [T])
    assert gpu.overlap_gpu(maps, dev["cloud"][1], [far, T]) == oracle.overlap_gpumap(refs, dev["xyz"][1], [far, T])
    assert gpu.overlap_gpu(maps[0], dev["cloud"][1], far) == 0.0
    T2 = synth.pose(6.0, 1.0, 0.0, 0.5)
    assert gpu.overlap_gpu(maps, dev["cloud"][1], [T2, T]) == oracle.overlap_gpumap(refs, dev["xyz"][1], [T2, T])


def test_factor_set_batch_equals_individual_and_is_repeatable(ctx, dev):
    """NonlinearFactorSetGPU: one launch over several factors (two levels x two directions, ragged sizes, one empty
    source) == per-factor calls; a second identical sweep gives identical bits (accumulators are self-cleaning)."""
    maps0 = [gpu.GaussianVoxelMapGPU(r, ctx=ctx).insert(dev["cloud"][0]) for r in (0.25, 0.5)]
    maps1 = [gpu.GaussianVoxelMapGPU(r, ctx=ctx).insert(dev["cloud"][1]) for r in (0.25, 0.5)]
    empty = gpu.PointCloudGPU.clone(np.zeros((0, 4)), np.zeros((0, 4, 4)), ctx=ctx)
    few = gpu.PointCloudGPU.clone(util.scan_pair()["points"][1][:777], util.scan_pair()["covs"][1][:777], ctx=ctx)
    T = dev["T_gt"]
    Ti = synth.inv_pose(T)
    facs, deltas = [], []
    for m in maps0:
        facs.append(gpu.IntegratedVGICPFactorGPU(0, 1, m, dev["cloud"][1], ctx=ctx)); deltas.append(T)
    for m in maps1:
        facs.append(gpu.IntegratedVGICPFactorGPU(1, 0, m, dev["cloud"][0], ctx=ctx)); deltas.append(Ti)
    facs.append(gpu.IntegratedVGICPFactorGPU(0, 1, maps0[1], empty, ctx=ctx)); deltas.append(T)
    facs.append(gpu.IntegratedVGICPFactorGPU(0, 1, maps0[1], few, ctx=ctx)); deltas.append(T)
    fs = gpu.NonlinearFactorSetGPU(ctx).add(facs)
    deltas = np.stack(deltas)
    a = fs.linearize_deltas(deltas)
    b = fs.linearize_deltas(deltas)
    assert a.tobytes() == b.tobytes()
    assert a[4]["num_inliers"] == 0 and not np.asarray(a[4]["H_ss"]).any()
    for i, f in enumerate(facs):
        single = np.zeros(1, gpu.LIN_DTYPE)
        from glim_b200.capi import check, lib, pose16, ptr
        check(lib().gb_vgicp_linearize(f._handle(), ptr(pose16(deltas[i])), ptr(single)))
        for k in ("H_tt", "H_ss", "H_ts", "b_t", "b_s"):
            assert util.rel_err(np.asarray(a[i][k]), np.asarray(single[0][k])) < 1e-6 or not np.asarray(single[0][k]).any()
        assert a[i]["num_inliers"] == single[0]["num_inliers"]
    # against the oracle
    ref_map = oracle.GpuMap(dev["xyz"][0], dev["cov6"][0], 0.25)
    ref, corr = oracle.linearize_gpumap(ref_map, dev["xyz"][1], dev["cov6"][1], T)
    check_linearized(gpu.unpack_linearized(a[0]), ref, hits=util.factor_hits(ref_map.vmean, ref_map.vcov, dev["xyz"][1], dev["cov6"][1], T, corr))
    # error sweep
    e = fs.error_deltas(deltas, deltas)
    assert np.allclose(e, a["error"], rtol=1e-5)


def test_pair_slab_accumulates_levels(ctx, dev):
    import torch

    maps0 = [gpu.GaussianVoxelMapGPU(r, ctx=ctx).insert(dev["cloud"][0]) for r in (0.25, 0.5)]
    facs = [gpu.IntegratedVGICPFactorGPU(0, 1, m, dev["cloud"][1], ctx=ctx) for m in maps0]
    sw = gpu.Sweep(ctx, facs, pair_index=[1, 1])
    slab = torch.zeros((3, gpu.capi.GB_SLAB_STRIDE), dtype=torch.float32, device="cuda:0")
    torch.cuda.synchronize()
    sw.attach_slab(slab.data_ptr(), 3)
    sw.set_poses(np.stack([dev["T_gt"]] * 2))
    sw.launch()
    rec = sw.fetch()
    ctx.synchronize()
    s = slab.cpu().numpy().astype(np.float64)
    assert not s[0].any() and not s[2].any()
    tot = {k: np.asarray(rec[0][k]) + np.asarray(rec[1][k]) for k in ("H_tt", "H_ss", "H_ts", "b_t", "b_s")}
    iu = np.triu_indices(6)
    Htt = tot["H_tt"].reshape(6, 6).T
    Hss = tot["H_ss"].reshape(6, 6).T
    # fp32 slab: each entry is float(level0) + float(level1): ~1e-7 of the block's largest entry
    assert np.allclose(s[1][0:21], Htt[iu], rtol=1e-6, atol=1e-6 * np.abs(Htt).max())
    assert np.allclose(s[1][21:57], tot["H_ts"], rtol=1e-6, atol=1e-6 * np.abs(tot["H_ts"]).max())
    assert np.allclose(s[1][57:78], Hss[iu], rtol=1e-6, atol=1e-6 * np.abs(Hss).max())
    assert np.allclose(s[1][78:84], tot["b_t"], rtol=1e-5, atol=1e-6 * np.abs(tot["b_t"]).max())
    assert np.allclose(s[1][84:90], tot["b_s"], rtol=1e-5, atol=1e-6 * np.abs(tot["b_s"]).max())
    assert s[1][90] == pytest.approx(rec[0]["error"] + rec[1]["error"], rel=1e-6)
    assert s[1][91] == rec[0]["num_inliers"] + rec[1]["num_inliers"]


def test_peer_slab_world1_is_deterministic_sum_of_levels(ctx, dev):
    """Fused exchange with world == 1: the epilogue of a pair's last factor sums the pair's records in fp64 and stores the
    fp32 row (no float atomics): rows equal the sum of the levels, untouched pairs stay zero, repeated steps are bit-identical
    (ping-pong buffers), and the values agree with the atomic-slab path."""
    from glim_b200 import multi_gpu

    maps0 = [gpu.GaussianVoxelMapGPU(r, ctx=ctx).insert(dev["cloud"][0]) for r in (0.25, 0.5)]
    maps1 = [gpu.GaussianVoxelMapGPU(r, ctx=ctx).insert(dev["cloud"][1]) for r in (0.25, 0.5)]
    T = dev["T_gt"]
    facs = [gpu.IntegratedVGICPFactorGPU(0, 1, m, dev["cloud"][1], ctx=ctx) for m in maps0] + [gpu.IntegratedVGICPFactorGPU(1, 0, m, dev["cloud"][0], ctx=ctx) for m in maps1]
    sw = gpu.Sweep(ctx, facs, pair_index=[3, 3, 0, 0])
    ps = gpu.PeerSlab(ctx, 5)
    sw.attach_peer_slab(ps)
    sw.set_poses(np.stack([T, T, synth.inv_pose(T), synth.inv_pose(T)]))
    rows = []
    for _ in range(3):
        sw.launch()
        ps.signal_wait()
        rows.append(ps.fetch())
    rec = sw.fetch()
    assert rows[0].tobytes() == rows[1].tobytes() == rows[2].tobytes()
    assert not rows[0][[1, 2, 4]].any()
    for pair, (a, b) in ((3, (0, 1)), (0, (2, 3))):
        got = multi_gpu.unpack_slab_row(rows[0][pair])
        for k in ("H_tt", "H_ss", "H_ts", "b_t", "b_s"):
            want = gpu.unpack_linearized(rec[a])[k] + gpu.unpack_linearized(rec[b])[k]
            assert np.allclose(got[k], want, rtol=2e-7, atol=2e-7 * np.abs(want).max())
        assert got["num_inliers"] == rec[a]["num_inliers"] + rec[b]["num_inliers"]


# ---------------------------------------------------------------------------------------------- preprocess kernels
def test_covariances_match_oracle(ctx, pair):
    from glim_b200 import preprocess

    P = pair["points"][0]
    nb = synth.knn(P, 10)
    normals, covs = preprocess.CloudCovarianceEstimation(ctx=ctx).estimate(P, nb)
    n_ref, c_ref = oracle.covariance_estimate(P, nb)
    assert np.allclose(covs, c_ref, atol=1e-9)
    # normals with their sign (p . n > 0 flips, :99-101): the kernel makes the oracle's uncontracted decision
    assert np.allclose(normals, n_ref, atol=1e-9)
    n5, c5 = preprocess.CloudCovarianceEstimation(ctx=ctx).estimate(P, nb, k_neighbors=5)
    n5r, c5r = oracle.covariance_estimate(P, nb, k_neighbors=5)
    assert np.allclose(c5, c5r, atol=1e-9) and np.allclose(n5, n5r, atol=1e-9)
    e_n, e_c = preprocess.CloudCovarianceEstimation(ctx=ctx).estimate(np.zeros((0, 4)), np.zeros((0,), np.int32))
    assert e_n.shape == (0, 4) and e_c.shape == (0, 4, 4)


def test_find_neighbors_matches_oracle(ctx):
    from glim_b200 import preprocess

    P = util.scan_pair(n_rays=32 * 100)["points"][0]
    for k in (10, 5, 20):
        nb = preprocess.find_neighbors(P, k, ctx=ctx).reshape(len(P), k)
        ref, _ = oracle.knn_bruteforce(P, k)
        assert np.array_equal(nb, ref)  # identical distances (no FMA contraction) and tie rule -> identical indices
    nb = preprocess.find_neighbors(P[:4], 10, ctx=ctx).reshape(4, 10)
    assert (nb[:, 4:] == np.arange(4)[:, None]).all()


def test_default_knn_is_exact_on_a_full_scan(ctx):
    """The default k-NN path on a full 60 k-point scan (the grid pyramid) returns exactly the oracle's indices: same
    distances, same tie rule."""
    from glim_b200 import preprocess

    sc = synth.make_hall_scene()
    big, _ = synth.scan(sc, "hdl32", synth.arc_trajectory(8)[2], synth.rng_for(32))
    assert len(big) == 60000
    nb = preprocess.find_neighbors(big, 10, ctx=ctx).reshape(-1, 10)
    ref, _ = oracle.knn_bruteforce(big, 10)
    assert np.array_equal(nb, ref)


def test_voxelgrid_sampling_matches_oracle(ctx, pair):
    from glim_b200 import preprocess

    P, T = pair["points"][0], pair["times"][0]
    for res in (0.25, 0.1, 1.0):
        out, ot, _ = preprocess.voxelgrid_sampling(P, res, times=T, ctx=ctx)
        ref, rt, _ = oracle.voxelgrid_sampling(P, res, times=T)
        assert np.array_equal(out, ref) and np.array_equal(ot, rt)  # same sums in the same order: bit-exact


def test_preprocess_pipeline(ctx, pair):
    """CloudPreprocessor::preprocess order (cloud_preprocessor.cpp:92-188): downsample -> range gate -> time sort -> k-NN."""
    from glim_b200 import preprocess

    P, T = pair["points"][0], pair["times"][0]
    fr = preprocess.CloudPreprocessor(preprocess.CloudPreprocessorParams(downsample_resolution=0.3, distance_near_thresh=2.0, distance_far_thresh=30.0, k_correspondences=10), ctx=ctx).preprocess(100.0, T, P)
    d = np.linalg.norm(fr.points[:, :3], axis=1)
    assert (d > 2.0).all() and (d < 30.0).all() and (np.diff(fr.times) >= 0).all()
    assert fr.scan_end_time == 100.0 + fr.times[-1] and fr.neighbors.shape == (fr.size() * 10,)
    ref_pts, ref_t, _ = oracle.voxelgrid_sampling(P, 0.3, times=T)
    sq = (ref_pts[:, :3] ** 2).sum(1)
    keep = (sq > 4.0) & (sq < 900.0)
    assert fr.size() == keep.sum()
    ref_nb, _ = oracle.knn_bruteforce(fr.points, 10)
    assert np.array_equal(fr.neighbors.reshape(-1, 10), ref_nb)


# ---------------------------------------------------------------------------------------------- full-size properties
@pytest.mark.parametrize("sensor,n_rays,res", [("generic64", None, 0.5), ("os1_64", None, 0.25)])
def test_full_size_properties(ctx, sensor, n_rays, res):
    """BASELINE sizes (100 k / 130 k points) through size-independent properties: additivity over a split of the source
    cloud, adjoint identities (A.4) on the returned blocks, symmetry / PSD, inliers == overlap * N, and the
    oracle itself on the full input."""
    sc = synth.make_hall_scene()
    traj = synth.arc_trajectory(8)
    clouds = []
    for i in (3, 4):
        pts, _ = synth.scan(sc, sensor, traj[i], synth.rng_for(55, i), n_rays=n_rays)
        _, cov = synth.with_covariances(pts, 10)
        clouds.append((pts, cov))
    assert len(clouds[1][0]) > 90_000
    tgt = gpu.PointCloudGPU.clone(*clouds[0], ctx=ctx)
    m = gpu.GaussianVoxelMapGPU(res, ctx=ctx).insert(tgt)
    P, Cv = clouds[1]
    T = synth.perturb(synth.inv_pose(traj[3]) @ traj[4], synth.rng_for(56), 0.01, 0.05)
    whole = gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, m, gpu.PointCloudGPU.clone(P, Cv, ctx=ctx), ctx=ctx).linearize({1: T})
    h = len(P) // 3
    parts = [gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, m, gpu.PointCloudGPU.clone(P[a:b], Cv[a:b], ctx=ctx), ctx=ctx).linearize({1: T}) for a, b in ((0, h), (h, len(P)))]
    for k in ("H_tt", "H_ss", "H_ts", "b_t", "b_s"):
        assert util.rel_err(parts[0][k] + parts[1][k], whole[k]) < 2e-5 or np.linalg.norm(parts[0][k] + parts[1][k] - whole[k]) < 2e-5 * np.sqrt(np.trace(whole["H_ss"]) * whole["error"])
    assert parts[0]["num_inliers"] + parts[1]["num_inliers"] == whole["num_inliers"]
    Tf = T.astype(np.float32).astype(np.float64)
    Ad = np.zeros((6, 6))
    Ad[:3, :3] = Tf[:3, :3]; Ad[3:, 3:] = Tf[:3, :3]; Ad[3:, :3] = synth.hat(Tf[:3, 3]) @ Tf[:3, :3]
    assert util.rel_err(Ad.T @ whole["H_tt"] @ Ad, whole["H_ss"]) < 1e-9
    assert util.rel_err(-whole["H_tt"] @ Ad, whole["H_ts"]) < 1e-9
    assert np.linalg.eigvalsh(whole["H_ss"]).min() > 0
    src = gpu.PointCloudGPU.clone(P, Cv, ctx=ctx)
    assert gpu.overlap_gpu(m, src, T) * len(P) == pytest.approx(whole["num_inliers"], abs=0.5)
    # and the oracle on the full-size input (a few seconds)
    xyz0, cov0 = oracle.pack_cloud(clouds[0][0], util.cov_colmajor16(clouds[0][1]))
    xyz1, cov1 = oracle.pack_cloud(P, util.cov_colmajor16(Cv))
    ref_map = oracle.GpuMap(xyz0, cov0, res)
    ref, corr = oracle.linearize_gpumap(ref_map, xyz1, cov1, T)
    check_linearized(whole, ref, hits=util.factor_hits(ref_map.vmean, ref_map.vcov, xyz1, cov1, T, corr))


# ---------------------------------------------------------------------------------------------- round-2 parity holes
def test_nan_points_and_singular_covariances_match_oracle(ctx, dev, pair):
    """Degenerate inputs (ADVICE r1): a NaN source point must be a MISS (it used to probe voxel (0,0,0)), and a point whose
    fused covariance is singular (zero source and zero voxel covariance) is skipped and NOT counted, as in the oracle."""
    P0, C0 = pair["points"][0], pair["covs"][0]
    P1, C1 = pair["points"][1].copy(), pair["covs"][1].copy()
    # a target whose voxel at the origin is occupied, so that a NaN -> (0,0,0) probe would hit something
    P0 = np.concatenate([P0, [[0.1, 0.1, 0.1, 1.0], [0.2, 0.1, 0.3, 1.0]]])
    C0 = np.concatenate([C0, np.tile(np.diag([1.0, 1.0, 1.0, 0.0]), (2, 1, 1))])
    P1[5, 0] = np.nan
    P1[77, :3] = np.nan
    P1[301, 2] = np.inf
    T = dev["T_gt"]
    tgt = gpu.PointCloudGPU.clone(P0, C0, ctx=ctx)
    src = gpu.PointCloudGPU.clone(P1, C1, ctx=ctx)
    m = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(tgt)
    xyz0, cov0 = oracle.pack_cloud(P0, util.cov_colmajor16(C0))
    xyz1, cov1 = oracle.pack_cloud(P1, util.cov_colmajor16(C1))
    ref_map = oracle.GpuMap(xyz0, cov0, 0.5)
    assert np.array_equal(m.download()[0], ref_map.buckets)
    got = gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, m, src, ctx=ctx).linearize({1: T})
    ref, corr = oracle.linearize_gpumap(ref_map, xyz1, cov1, T)
    assert corr[5] < 0 and corr[77] < 0 and corr[301] < 0
    assert np.isfinite(got["H_ss"]).all() and np.isfinite(got["b_s"]).all()
    check_linearized(got, ref, hits=util.factor_hits(ref_map.vmean, ref_map.vcov, xyz1, cov1, T, corr))
    assert gpu.overlap_gpu(m, src, T) == oracle.overlap_gpumap([ref_map], xyz1, [T])
    # singular fused covariance: zero covariances on both sides for half of the source points
    Z0 = np.zeros_like(pair["covs"][0])
    Z1 = pair["covs"][1].copy()
    Z1[: len(Z1) // 2] = 0.0
    tgt0 = gpu.PointCloudGPU.clone(pair["points"][0], Z0, ctx=ctx)
    src0 = gpu.PointCloudGPU.clone(pair["points"][1], Z1, ctx=ctx)
    m0 = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(tgt0)
    x0, c0 = oracle.pack_cloud(pair["points"][0], util.cov_colmajor16(Z0))
    x1, c1 = oracle.pack_cloud(pair["points"][1], util.cov_colmajor16(Z1))
    r0 = oracle.GpuMap(x0, c0, 0.5)
    got0 = gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, m0, src0, ctx=ctx).linearize({1: T})
    ref0, corr0 = oracle.linearize_gpumap(r0, x1, c1, T)
    assert (corr0[: len(Z1) // 2] >= 0).sum() > 100  # there ARE correspondences among the singular points ...
    assert ref0[121] < (corr0 >= 0).sum()  # ... and the oracle does not count them
    hits0 = util.factor_hits(r0.vmean, r0.vcov, x1, c1, T, corr0)
    assert len(hits0) == ref0[121]  # the per-hit data skip the singular ones too
    check_linearized(got0, ref0, hits=hits0)


def test_kernel_generations_agree(ctx, dev, monkeypatch):
    """k_vgicp_sweep3 (large sweeps, contiguous items) and k_vgicp_sweep5 (small sweeps, strided items) on the same factor
    set: identical inlier counts, blocks equal to fp32 summation-order noise."""
    maps0 = [gpu.GaussianVoxelMapGPU(r, ctx=ctx).insert(dev["cloud"][0]) for r in (0.25, 0.5)]
    T = dev["T_gt"]
    outs = {}
    for name, kernel in (("v3", "3"), ("v5", "5")):
        monkeypatch.setenv("GB_KERNEL", kernel)
        facs = [gpu.IntegratedVGICPFactorGPU(0, 1, m, dev["cloud"][1], ctx=ctx) for m in maps0]
        fs = gpu.NonlinearFactorSetGPU(ctx).add(facs)
        outs[name] = fs.linearize_deltas(np.stack([T, T]))
        e = fs.error_deltas(np.stack([T, T]), np.stack([T, T]))
        assert np.allclose(e, outs[name]["error"], rtol=1e-5)
    for i in range(2):
        assert outs["v5"][i]["num_inliers"] == outs["v3"][i]["num_inliers"]
        for k in ("H_tt", "H_ss", "H_ts"):
            assert util.rel_err(outs["v5"][i][k], outs["v3"][i][k]) < 1e-5, k


def test_large_sweep_matches_oracle(ctx):
    """A factor set that is large by the library's own size rule, with no kernel or item-size override: 240 factors sharing
    one 131 k-point source cloud and one map (31 M point-factors).  It runs sweep3 with 2048-point items (four 512-point
    rounds each) drawn from the queue, and a tapered tail.  Every record must match the oracle of that one pair."""
    sc = synth.make_hall_scene()
    traj = synth.arc_trajectory(8)
    clouds = []
    for i in (3, 4):
        pts, _ = synth.scan(sc, "os1_64", traj[i], synth.rng_for(55, i))
        _, cov = synth.with_covariances(pts, 10)
        clouds.append((pts, cov))
    m = gpu.GaussianVoxelMapGPU(0.25, ctx=ctx).insert(gpu.PointCloudGPU.clone(*clouds[0], ctx=ctx))
    src = gpu.PointCloudGPU.clone(*clouds[1], ctx=ctx)
    T = synth.perturb(synth.inv_pose(traj[3]) @ traj[4], synth.rng_for(56), 0.01, 0.05)
    F = 240
    sw = gpu.Sweep(ctx, [gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, m, src, ctx=ctx) for _ in range(F)])
    assert sw.point_factors >= 2048 * 6 * sw.grid * 8  # ~6 items per warp would exceed 2048 points: items of 2048
    assert sw.num_tiles > sw.grid * 8  # the queue path
    sw.set_poses(np.stack([T] * F))
    sw.launch()
    rec = sw.fetch()
    xyz0, cov0 = oracle.pack_cloud(clouds[0][0], util.cov_colmajor16(clouds[0][1]))
    xyz1, cov1 = oracle.pack_cloud(clouds[1][0], util.cov_colmajor16(clouds[1][1]))
    ref_map = oracle.GpuMap(xyz0, cov0, 0.25)
    ref, corr = oracle.linearize_gpumap(ref_map, xyz1, cov1, T)
    scale = util.record_scale(util.factor_hits(ref_map.vmean, ref_map.vcov, xyz1, cov1, T, corr))
    for r in rec:
        check_linearized(gpu.unpack_linearized(r), ref, hits=scale)


def _oracle_check_factors(ctx, w, fset, picks, tol=REL_TOL):
    """Compare the BATCHED sweep's records for the picked factors of a workload factor set with the oracle."""
    gf = w.gpu_factors(fset)
    sw = gpu.Sweep(ctx, gf, pair_index=[f.pair for f in fset.factors])
    sw.set_poses(fset.deltas)
    sw.launch()
    rec = sw.fetch()
    maps = {}
    packed = {}
    worst = 0.0
    for k in picks:
        f = fset.factors[k]
        for c in (f.target, f.source):
            if c not in packed:
                packed[c] = oracle.pack_cloud(w.host_clouds[c][0], util.cov_colmajor16(w.host_clouds[c][1]))
        if (f.target, f.level) not in maps:
            maps[(f.target, f.level)] = oracle.GpuMap(*packed[f.target], w.resolutions[f.level])
        m = maps[(f.target, f.level)]
        ref, corr = oracle.linearize_gpumap(m, *packed[f.source], fset.deltas[k], normals=w.host_normals[f.source] if w.surface_validation else None)
        got = gpu.unpack_linearized(rec[k])
        check_linearized(got, ref, tol, hits=util.factor_hits(m.vmean, m.vcov, *packed[f.source], fset.deltas[k], corr))
        worst = max(worst, util.rel_err(got["H_ss"], oracle.split122(ref)["H_ss"]))
    return sw, rec, worst


@pytest.mark.parametrize("kernel", ["auto", "3"])
def test_global_mapping_factors_match_oracle(ctx, monkeypatch, kernel):
    """M4 data distribution at full submap size (50 k points, 0.5 / 1.0 m voxels, ~35 % inliers) on a short loop.  kernel=3:
    the batched sweep runs sweep3 through the dynamic item queue (items > warps) and replicated accumulators; kernel=auto
    (sweep5, what a sweep of this size gets by default): one wave of strided items, re-sized after the first fetch.  Picked
    factors vs the oracle."""
    from glim_b200 import workloads

    monkeypatch.setenv("GB_KERNEL", kernel)
    w = workloads.global_mapping(ctx, n_submaps=12, laps=1, side=60.0, use_gpu=True)
    fset = w.sets[0]
    assert len(fset.factors) >= 10 and min(len(c[0]) for c in w.host_clouds) == 50000
    rng = np.random.default_rng(5)
    picks = sorted(rng.choice(len(fset.factors), 6, replace=False).tolist())
    sw, rec, worst = _oracle_check_factors(ctx, w, fset, picks)
    if kernel == "3":
        assert sw.num_tiles > sw.grid * 8  # the queue path
    else:
        assert sw.num_tiles <= sw.grid * 8  # one wave
        # the fetch above re-sized the item table from the measured inlier fractions: same results from the new table
        sw.launch()
        rec2 = sw.fetch()
        assert np.array_equal(rec2["num_inliers"], rec["num_inliers"])
        for k in ("H_tt", "H_ss"):
            assert util.rel_err(np.asarray(rec2[k]), np.asarray(rec[k])) < 1e-5
    inl = rec["num_inliers"] / 50000.0
    assert 0.05 < np.median(inl) < 0.9


def test_livox_dense_factor_matches_oracle(ctx):
    """M5 shape: 500 k-point MID-360-like clouds, 0.1 / 0.2 m voxels (tables of ~10^6 buckets): both levels of one pair."""
    from glim_b200 import workloads

    w = workloads.livox_stress(ctx, n_rays=500_000, use_gpu=True, n_targets=2)
    fset = w.sets[0]
    assert len(w.host_clouds[0][0]) > 400_000
    picks = [k for k, f in enumerate(fset.factors) if f.target == 0]
    assert len(picks) == 2
    _oracle_check_factors(ctx, w, fset, picks)


# ---------------------------------------------------------------------------------------------- gb_preprocess (device-resident frame pipeline)
def _cpu_frame(P, T, res, near, far, k, mask=None, crop=None, sor=None):
    """oracle composition of CloudPreprocessor::preprocess_impl + CloudCovarianceEstimation::estimate"""
    if mask is None:
        pts, tms, _ = oracle.voxelgrid_sampling(P, res, times=T)
    else:
        pts, tms = P[mask], T[mask]
    sq = (pts[:, :3] ** 2).sum(1)
    keep = (sq > near * near) & (sq < far * far) & np.isfinite(pts).all(axis=1)
    if crop is not None:
        lo, hi = crop
        keep &= ~((pts[:, :3] >= lo).all(1) & (pts[:, :3] <= hi).all(1))
    idx = np.nonzero(keep)[0]
    idx = idx[np.argsort(tms[idx], kind="stable")]
    pts, tms = np.ascontiguousarray(pts[idx]), tms[idx]
    if sor is not None:  # gtsam_points::remove_outliers [EXT]: mean neighbour distance vs mean + std_mul * stddev over the frame
        ko, mul = sor
        nbo, _ = oracle.knn_bruteforce(pts, ko)
        d = np.zeros(len(pts))
        for j in range(ko):
            e = pts[:, :3] - pts[nbo[:, j], :3]
            d = d + np.sqrt((e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2])
        d = d / ko
        mean = d.sum() / len(d)
        var = (d * d).sum() / len(d) - mean * mean
        keep = d < mean + mul * np.sqrt(max(var, 0.0))
        pts, tms = np.ascontiguousarray(pts[keep]), tms[keep]
    nb, _ = oracle.knn_bruteforce(pts, k)
    normals, covs = oracle.covariance_estimate(pts, nb)
    return pts, tms, nb, normals, covs


@pytest.mark.parametrize("mode", ["voxelgrid", "randomgrid", "cropbox", "outliers"])
def test_gb_preprocess_matches_oracle_pipeline(ctx, mode):
    """One device-resident call = the reference's whole per-frame preprocess + covariance estimation + PointCloudGPU::clone:
    frame points / times bit-exact, neighbour indices exact, covariances 1e-9, and the device cloud equals the fp32 cast of
    the host products."""
    from glim_b200 import preprocess

    sc = synth.make_hall_scene()
    P, T = synth.scan(sc, "hdl32", synth.arc_trajectory(8)[2], synth.rng_for(41), n_rays=32 * 700)
    P = P.copy()
    P[17, 1] = np.nan  # a non-finite raw point is dropped by the gate (cloud_preprocessor.cpp:123)
    k = 10
    if mode == "randomgrid":
        par = preprocess.CloudPreprocessorParams(distance_near_thresh=1.0, distance_far_thresh=60.0, use_random_grid_downsampling=True, downsample_resolution=1.0, downsample_target=6000, k_correspondences=k)
        mask = oracle.randomgrid_sampling(P, 1.0, 6000 / len(P), seed=5)
        assert 5000 < mask.sum() <= int(len(P) * (6000 / len(P)) * 1.2)
        ref = _cpu_frame(P, T, None, 1.0, 60.0, k, mask=mask)
    elif mode == "outliers":
        par = preprocess.CloudPreprocessorParams(distance_near_thresh=1.0, distance_far_thresh=60.0, downsample_resolution=0.2, k_correspondences=k, enable_outlier_removal=True, outlier_removal_k=8, outlier_std_mul_factor=1.0)
        ref = _cpu_frame(P, T, 0.2, 1.0, 60.0, k, sor=(8, 1.0))
        assert len(ref[0]) < 0.97 * len(_cpu_frame(P, T, 0.2, 1.0, 60.0, k)[0])  # the filter removes a real share of the (far, sparse) points
    elif mode == "cropbox":
        par = preprocess.CloudPreprocessorParams(distance_near_thresh=1.0, distance_far_thresh=60.0, downsample_resolution=0.2, k_correspondences=k, enable_cropbox_filter=True, crop_bbox_min=(-3.0, -2.0, -5.0), crop_bbox_max=(4.0, 2.5, 5.0))
        ref = _cpu_frame(P, T, 0.2, 1.0, 60.0, k, crop=(np.array([-3.0, -2.0, -5.0]), np.array([4.0, 2.5, 5.0])))
    else:
        par = preprocess.CloudPreprocessorParams(distance_near_thresh=1.0, distance_far_thresh=60.0, downsample_resolution=0.2, k_correspondences=k)
        ref = _cpu_frame(P, T, 0.2, 1.0, 60.0, k)
    fr, normals, covs, cloud = preprocess.FramePreprocessorGPU(par, ctx, seed=5).preprocess(10.0, T, P)
    pts, tms, nb, n_ref, c_ref = ref
    assert fr.size() == len(pts) > 3000
    assert np.array_equal(fr.points, pts) and np.array_equal(fr.times, tms) and fr.scan_end_time == 10.0 + tms[-1]
    assert np.array_equal(fr.neighbors.reshape(-1, k), nb)
    assert np.allclose(covs, c_ref, atol=1e-9)
    assert np.allclose(normals, n_ref, atol=1e-9)  # sign included
    gx, gc = cloud.download()
    xyz, cov6 = oracle.pack_cloud(fr.points, util.cov_colmajor16(covs))
    assert np.array_equal(gx, xyz) and np.array_equal(gc, cov6)  # the planes were written from the same fp64 values
    # and the frame is usable as a VGICP source right away
    m = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(cloud)
    got = gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, m, cloud, ctx=ctx).linearize({1: np.eye(4)})
    assert fr.size() * 0.995 <= got["num_inliers"] <= fr.size()  # (the table may drop <= target_points_drop_rate of the points)
    # the PreprocessedFrame-only entry (CloudPreprocessor mirror) agrees
    fr2 = preprocess.CloudPreprocessor(par, ctx=ctx, seed=5).preprocess(10.0, T, P)
    assert np.array_equal(fr2.points, fr.points) and np.array_equal(fr2.neighbors, fr.neighbors)


def test_pyramid_knn_is_exact_on_hard_clouds(ctx):
    """The grid-pyramid k-NN on duplicated points, far outliers (coarsest-level / full-scan fallback), tiny clouds; a point
    whose 0.25 m cell is outside the 21-bit key range gets a row of itself and is no point's neighbour, whatever the size."""
    from glim_b200 import preprocess

    P = util.scan_pair(n_rays=32 * 100)["points"][0]
    rng = synth.rng_for(31)
    dup = np.concatenate([P[:500], P[:500], P[100:200] + [1e-9, 0, 0, 0], [[500.0, -300.0, 20.0, 1.0], [-800.0, 10.0, 5.0, 1.0]], rng.normal(0, 0.01, (64, 4)) * [1, 1, 1, 0] + [3, 3, 3, 1]])
    for cloud in (P, dup, P[:7]):
        for k in (10, 5):
            nb = preprocess.find_neighbors(cloud, k, ctx=ctx).reshape(len(cloud), k)
            ref, _ = oracle.knn_bruteforce(cloud, k)
            assert np.array_equal(nb, ref)
    far = np.concatenate([P[:300], [[3e5, 0.0, 0.0, 1.0]]])
    nb = preprocess.find_neighbors(far, 10, ctx=ctx).reshape(len(far), 10)
    assert np.array_equal(nb[:300], oracle.knn_bruteforce(P[:300], 10)[0]) and (nb[300] == 300).all()


def test_merge_frames_gpu_matches_oracle(ctx):
    """SURVEY 8(f) row 3 -- gtsam_points::merge_frames as SubMapping::create_submap calls it (sub_mapping.cpp:481-497): five
    keyframe clouds transformed into the submap origin frame, voxel-grid averaged (points and covariances), thinned to a target
    size.  fp64 sums in the same order as the oracle: bit-exact; the device cloud is the fp32 cast of the host product."""
    sc = synth.make_hall_scene()
    traj = synth.arc_trajectory(8, step=1.5)
    clouds, packed, poses = [], [], []
    origin = traj[2]
    for i in range(5):
        pts, _ = synth.scan(sc, "hdl32", traj[i], synth.rng_for(61, i), n_rays=32 * 250)
        _, cov = synth.with_covariances(pts, 10)
        clouds.append(gpu.PointCloudGPU.clone(pts, cov, ctx=ctx))
        packed.append(oracle.pack_cloud(pts, util.cov_colmajor16(cov)))
        poses.append(synth.inv_pose(origin) @ traj[i])
    for target in (0, 3000):
        pts, covs, merged = gpu.merge_frames_gpu(poses, clouds, 0.25, target, seed=9, ctx=ctx)
        rp, rc = oracle.merge_frames(poses, packed, 0.25, target, seed=9)
        assert len(pts) == len(rp) and (target == 0 or len(pts) == target)
        assert np.array_equal(pts, rp) and np.array_equal(covs, rc)
        gx, gc = merged.download()
        xyz, cov6 = oracle.pack_cloud(pts, util.cov_colmajor16(covs))
        assert np.array_equal(gx, xyz) and np.array_equal(gc, cov6)
        # covariances stay symmetric PSD with zero last row / column (the invariants SubMap::load checks, sub_map.cpp:151-166)
        assert np.allclose(covs, covs.transpose(0, 2, 1)) and not covs[:, 3, :].any() and not covs[:, :, 3].any()
        assert np.linalg.eigvalsh(covs[:, :3, :3]).min() > 0
    # the merged submap is a valid VGICP target / source
    m = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(merged)
    got = gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, m, merged, ctx=ctx).linearize({1: np.eye(4)})
    assert merged.size() * 0.995 <= got["num_inliers"] <= merged.size()  # (the table may drop <= target_points_drop_rate of the points)


def test_surface_validation_matches_oracle(ctx, dev, pair):
    """set_enable_surface_validation(true) (odometry_estimation_gpu.cpp:145, :162): the orientation-consistency gate
    3 n^T C_B n <= tr(C_B) (DESIGN ledger; the reference rule is unpinned) -- kernel and oracle take the same decisions (fp32,
    canonical operation order), the gate rejects a real fraction of the correspondences, and it needs the source normals."""
    res = 0.5
    m = gpu.GaussianVoxelMapGPU(res, ctx=ctx).insert(dev["cloud"][0])
    ref_map = oracle.GpuMap(dev["xyz"][0], dev["cov6"][0], res)
    nrm = pair["normals"][1]
    fac = gpu.IntegratedVGICPFactorGPU(0, 1, m, dev["cloud"][1], ctx=ctx)
    fac.set_enable_surface_validation(True)
    off = gpu.IntegratedVGICPFactorGPU(0, 1, m, dev["cloud"][1], ctx=ctx)
    for T in util.test_poses(dev["T_gt"], 3, key=77):
        got = fac.linearize({0: np.eye(4), 1: T})
        ref, corr = oracle.linearize_gpumap(ref_map, dev["xyz"][1], dev["cov6"][1], T, normals=nrm.astype(np.float32))
        check_linearized(got, ref, hits=util.factor_hits(ref_map.vmean, ref_map.vcov, dev["xyz"][1], dev["cov6"][1], T, corr))
        base = off.linearize({0: np.eye(4), 1: T})
        rejected = int((corr == -2).sum())
        assert rejected > 0 and got["num_inliers"] == base["num_inliers"] - rejected
        e = fac.error({0: np.eye(4), 1: T})
        assert abs(e - got["error"]) <= 1e-5 * got["error"]
    # a pose that turns the source by 60 degrees about x: normals no longer agree with the voxels they fall into
    Tbad = dev["T_gt"] @ synth.pose(0, 0, 0, 0.0, 0.0, np.pi / 3)
    got = fac.linearize({0: np.eye(4), 1: Tbad})
    ref, corr = oracle.linearize_gpumap(ref_map, dev["xyz"][1], dev["cov6"][1], Tbad, normals=nrm.astype(np.float32))
    assert got["num_inliers"] == ref[121] and (corr == -2).sum() > 0.05 * (corr != -1).sum() > 0
    # batched, mixed with a factor that has the gate off
    out = gpu.NonlinearFactorSetGPU(ctx).add([fac, off]).linearize({0: np.eye(4), 1: dev["T_gt"]})
    assert out[0]["num_inliers"] < out[1]["num_inliers"]
    # a frame without normals cannot use the gate: loud error, not a silent no-op
    bare = gpu.PointCloudGPU.clone(pair["points"][1], pair["covs"][1], ctx=ctx)
    f2 = gpu.IntegratedVGICPFactorGPU(0, 1, m, bare, ctx=ctx)
    f2.set_enable_surface_validation(True)
    with pytest.raises(Exception):
        f2.linearize({0: np.eye(4), 1: dev["T_gt"]})
