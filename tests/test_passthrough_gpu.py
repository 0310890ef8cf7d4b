"""GLIM's passthrough sub-mapping on the device: gb_ivox_extract (IVoxGPU.voxel_data) against the numpy restatement
(tests/passthrough_oracle.py) bit for bit, for the identity and a general pose, no target, a target at or above the map's size,
target 1 (m = 0 included) and the 65 692-point map thinned to 50 000 (49 999 kept); the extracted cloud against an upload of the
restated arrays, through download, normals, a voxel map and a VGICP linearization; the map left unchanged; launch counts
independent of the map's size and no launch on a refusal; the fp32 world-frame error bound 3 km from the origin; and the module
end to end on preprocessed synthetic scans, against the restatement, with its last submap registered against its first as the
pose graph's loop candidates are."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial import cKDTree

from glim_b200 import capi, gpu, preprocess, synth
from glim_b200 import sub_mapping_passthrough as spt
from tests import passthrough_oracle as po

pytestmark = pytest.mark.gpu
F32, F64 = np.float32, np.float64
INT_MAX = 2**31 - 1


@pytest.fixture(scope="module")
def ctx():
    return gpu.Context(0)


def homog(xyz):
    xyz = np.asarray(xyz, F64)
    return np.concatenate([xyz, np.ones((len(xyz), 1))], axis=1)


def cloud(ctx, xyz, rng):
    """a device cloud of the points with random covariances"""
    L = rng.normal(scale=0.05, size=(len(xyz), 3, 3))
    cov = np.zeros((len(xyz), 4, 4))
    cov[:, :3, :3] = L @ np.swapaxes(L, 1, 2) + 1e-4 * np.eye(3)
    return gpu.PointCloudGPU.clone(homog(xyz), cov, ctx=ctx)


def general_pose(rng, spread=30.0):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    T = np.eye(4)
    T[:3, :3] = q * np.sign(np.linalg.det(q))
    T[:3, 3] = rng.uniform(-spread, spread, 3)
    return T


def new_ivox(ctx):
    return gpu.IVoxGPU(0.5, 0.2, 64, 1, 0, INT_MAX, ctx=ctx)  # the module's map


def random_map(ctx, rng, inserts=3, n=20000, extent=20.0):
    m = new_ivox(ctx)
    for _ in range(inserts):
        m.insert(cloud(ctx, rng.uniform(-extent, extent, (n, 3)), rng), general_pose(rng))
    return m


def lattice_map(ctx, rng, P, spacing):
    """exactly P points: a lattice whose points are all admitted (spacing >= 0.2 m, at most 8 to a 0.5 m cell)"""
    side = int(np.ceil(P ** (1 / 3)))
    g = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3)[:P]
    m = new_ivox(ctx).insert(cloud(ctx, 0.1 + spacing * g, rng))
    assert m.num_points == P
    return m


def same_cloud(a, b):
    xa, ca = a.download()
    xb, cb = b.download()
    assert a.n == b.n
    assert xa.tobytes() == xb.tobytes() and ca.tobytes() == cb.tobytes()


def check_extract(ivox, T, target, seed):
    """the device extraction against the restatement over the map's own download -> (cloud, q, c6)"""
    _, _, xyz, cov6 = ivox.download()
    q, c6 = po.extract(xyz, cov6, T, target, seed)
    out = ivox.voxel_data(T, target, seed)
    assert out.n == len(q) == po.thin_count(len(xyz), target)
    gx, gc = out.download()
    assert gx.tobytes() == q.astype(F32).tobytes() and gc.tobytes() == c6.astype(F32).tobytes()
    return out, q, c6


def snapshot(ivox):
    return [a.tobytes() for a in ivox.download()] + [ivox.info()]


def test_extraction_matches_the_restatement(ctx):
    rng = np.random.default_rng(1)
    m = random_map(ctx, rng)
    P = m.num_points
    assert P > 20000 and m.download()[1].max() > 1  # some cells hold several points
    before = snapshot(m)
    T = general_pose(rng)
    for Tc, target in ((None, 0), (T, 0), (T, -7), (T, P), (T, P + 11), (T, 1), (T, P // 3), (T, 20000)):
        check_extract(m, Tc, target, 77 + target)
    # a target beyond the C call's int keeps every point, as a 64-bit target would (not a wrapped count)
    for big in (2**31, 2**32 + 5):
        whole = m.voxel_data(T, big, 1)
        assert whole.n == P and whole.download()[0].tobytes() == m.voxel_data(T, 0, 1).download()[0].tobytes()
    # thinned sets depend on the seed, and the same seed gives the same set
    a, _, _ = check_extract(m, T, P // 2, 5)
    b, _, _ = check_extract(m, T, P // 2, 6)
    assert a.download()[0].tobytes() != b.download()[0].tobytes()
    assert snapshot(m) == before  # the map is only read


def test_count_rule_and_empty_results(ctx):
    rng = np.random.default_rng(2)
    m = lattice_map(ctx, rng, 65692, 0.25)
    out, _, _ = check_extract(m, general_pose(rng), 50000, 12345)
    assert out.n == 49999  # random_sampling's count at the module's rate, one short of the target
    small = lattice_map(ctx, rng, 49, 1.0)
    out, _, _ = check_extract(small, None, 1, 3)
    assert out.n == 0  # 49 * (1.0 / 49) < 1: nothing stays, and the result is a valid empty cloud
    assert out.download()[0].shape == (0, 3)
    out, _, _ = check_extract(lattice_map(ctx, rng, 50, 1.0), None, 1, 3)
    assert out.n == 1
    empty = new_ivox(ctx)
    for target in (0, 5):
        assert empty.voxel_data(None, target, 1).n == 0


def test_cloud_is_bit_identical_to_an_upload(ctx):
    rng = np.random.default_rng(3)
    m = random_map(ctx, rng, inserts=2, n=15000)
    for target_num_points in (0, m.num_points // 2):
        T = general_pose(rng)
        out, q, c6 = check_extract(m, T, target_num_points, 99)
        ref = gpu.PointCloudGPU.clone(homog(q), po.cov4x4(c6), ctx=ctx)
        same_cloud(out, ref)
        assert out.estimate_normals().normals().tobytes() == ref.estimate_normals().normals().tobytes()
        for x, y in zip(gpu.GaussianVoxelMapGPU(1.0, ctx=ctx).insert(out).download(), gpu.GaussianVoxelMapGPU(1.0, ctx=ctx).insert(ref).download()):
            assert x.tobytes() == y.tobytes()
        target = gpu.GaussianVoxelMapGPU(1.0, ctx=ctx).insert(ref)
        D = np.eye(4)
        D[:3, 3] = [0.05, -0.02, 0.01]
        la = gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, target, out, ctx=ctx).linearize({1: D})
        lb = gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, target, ref, ctx=ctx).linearize({1: D})
        assert la["num_inliers"] > 0
        for key in la:
            assert np.asarray(la[key]).tobytes() == np.asarray(lb[key]).tobytes(), key


def launches(ctx, fn):
    before = ctx.kernel_launches
    out = fn()
    return ctx.kernel_launches - before, out


def test_launch_counts_and_refusals(ctx):
    rng = np.random.default_rng(4)
    small = random_map(ctx, rng, inserts=1, n=1000)
    large = random_map(ctx, rng, inserts=3, n=100000, extent=100.0)
    assert small.num_points <= 1000 and large.num_points >= 290000
    T = general_pose(rng)
    for m in (small, large):
        n, out = launches(ctx, lambda: m.voxel_data(T))
        assert n == 1 + 3 and out.n == m.num_points  # k_ivox_extract, gb_cloud_build
        n, out = launches(ctx, lambda: m.voxel_data(T, m.num_points // 2, 7))
        assert n == 3 + 1 + 1 + 3 and out.n == po.thin_count(m.num_points, m.num_points // 2)  # gb_thin, the scan of its flags, k_ivox_extract, gb_cloud_build
    # the one exception to the fixed counts: an empty result makes no launch
    empty = new_ivox(ctx)
    assert launches(ctx, lambda: empty.voxel_data(T, 5, 1))[0] == 0
    small49 = lattice_map(ctx, rng, 49, 1.0)
    n, out = launches(ctx, lambda: small49.voxel_data(T, 1, 1))
    assert n == 0 and out.n == 0  # m = (size_t)(49 * (1.0 / 49)) = 0
    L = capi.lib()
    vmap = gpu.IncrementalVoxelMapGPU(0.5, ctx=ctx)
    built = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(cloud(ctx, rng.uniform(-5, 5, (500, 3)), rng))
    grid = gpu.PointGridGPU(cloud(ctx, rng.uniform(-5, 5, (500, 3)), rng), 1.0, ctx=ctx)
    good = capi.pose16(T)
    bad_nan, bad_inf = good.copy(), good.copy()
    bad_nan[5], bad_inf[12] = np.nan, np.inf
    h = C.c_void_p()
    before = ctx.kernel_launches
    refused = [(None, small.h, good), (ctx.h, None, good), (ctx.h, vmap.h, good), (ctx.h, built.h, good), (ctx.h, grid.h, good), (ctx.h, small.h, bad_nan),
               (ctx.h, small.h, bad_inf)]
    for c, mh, Tc in refused:
        assert L.gb_ivox_extract(c, mh, capi.ptr(Tc), 10, 1, C.byref(h)) == 1 and not h.value
    assert L.gb_ivox_extract(ctx.h, small.h, capi.ptr(good), 10, 1, None) == 1
    if L.gb_device_count() > 1:
        other = gpu.Context(1)
        assert L.gb_ivox_extract(other.h, small.h, capi.ptr(good), 10, 1, C.byref(h)) == 1 and not h.value
    assert ctx.kernel_launches == before


def test_far_from_the_origin_within_the_world_frame_bound(ctx):
    """frames 3 km from the world origin: the map stores fp32 world points, so an extracted point is within
    sqrt(3) 2^-24 (max|q_world| + max|q_out|) of the fp64 world restatement (DESIGN.md section 7)"""
    rng = np.random.default_rng(5)
    T_ws = synth.pose(3000.0, -1200.0, 40.0, 0.3) @ general_pose(rng, spread=10.0)
    m = new_ivox(ctx)
    world = []
    g = np.stack(np.meshgrid(*[np.arange(14)] * 3, indexing="ij"), -1).reshape(-1, 3)
    for k in range(3):  # three inserts of blocks 12 m apart in the sensor frame, each point at least 0.6 m from the others
        a = (0.7 * g + rng.uniform(-0.05, 0.05, g.shape) - 4.5 + [12.0 * k, 0.0, 0.0]).astype(F32).astype(F64)
        m.insert(cloud(ctx, a, rng), T_ws)
        world.append(a @ T_ws[:3, :3].T + T_ws[:3, 3])
    world = np.concatenate(world)
    assert m.num_points == len(world)  # every point admitted: a one-to-one match
    T_out = synth.inv_pose(T_ws @ general_pose(rng, spread=5.0))  # a submap origin near the points
    q_out = world @ T_out[:3, :3].T + T_out[:3, 3]
    got = m.voxel_data(T_out).download()[0].astype(F64)
    dist, idx = cKDTree(q_out).query(got)
    assert len(np.unique(idx)) == len(world)
    bound = np.sqrt(3.0) * 2.0**-24 * (np.abs(world).max() + np.abs(q_out).max())
    assert np.abs(world).max() > 2900.0 and dist.max() <= bound, (dist.max(), bound)
    assert dist.max() > 1e-6  # the fp32 world frame does cost something this far out


def pose_error(T, T_ref):
    d = synth.inv_pose(T_ref) @ T
    return float(np.linalg.norm(d[:3, 3])), float(np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1)))


def test_module_end_to_end(ctx):
    """Preprocessed scans along a path that goes out and comes back to its start, through the module mirror on the device and
    through the restatement: the same keyframes, cuts and poses, and bit-identical submap clouds; no iVox cell reaches 64
    points.  The last submap is then registered against the first as the pose graph registers a loop candidate."""
    sc = synth.make_hall_scene()
    out_path = synth.arc_trajectory(24, step=0.5)
    traj = out_path + out_path[::-1][1:] + [out_path[0]]  # back to the start, where the last pose repeats (not a keyframe)
    pre = preprocess.FramePreprocessorGPU(preprocess.CloudPreprocessorParams(downsample_resolution=0.25, k_correspondences=10), ctx)
    frames, clouds = [], []
    for i, T in enumerate(traj):
        pts, times = synth.scan(sc, "hdl32", T, synth.rng_for(60, i), n_rays=32 * 400)
        c = pre.preprocess(0.1 * i, times, pts, host_outputs=False)[3]
        xyz, cov6 = c.download()
        frames.append((1000 + i, xyz, cov6, T))
        clouds.append(c)
    params = spt.SubMappingPassthroughParams(max_num_keyframes=10, submap_target_num_points=20000)
    ref = po.run(params, frames)
    mod = spt.SubMappingPassthroughGPU(params, ctx=ctx)
    mine = []
    for idx, ((fid, _, _, T), c) in enumerate(zip(frames, clouds)):
        mod.insert_frame(fid, c, T)
        mine += [(s, idx) for s in mod.get_submaps()]
    mine += [(s, len(frames)) for s in mod.submit_end_of_sequence()]
    assert len(ref) >= 4 and [a for _, a in mine] == [r["after"] for r in ref]
    for (s, _), r in zip(mine, ref):
        assert s.id == r["id"] and s.odom_frame_ids == r["odom_frame_ids"] and s.keyframe_ids == r["keyframe_ids"]
        for k in ("T_world_origin", "T_origin_endpoint_L", "T_origin_endpoint_R"):
            assert np.array_equal(getattr(s, k), r[k]), k
        gx, gc = s.frame.download()
        assert s.frame.n == len(r["q"]) and gx.tobytes() == r["q"].astype(F32).tobytes() and gc.tobytes() == r["c6"].astype(F32).tobytes()
        assert r["max_cell"] < 64  # the capacity clamp (100 -> 64) changed nothing
    assert any(len(r["q"]) < r["P"] for r in ref)  # some submap was thinned
    assert 1000 + len(traj) - 1 not in [k for r in ref for k in r["keyframe_ids"]]

    # the pose graph's loop candidate (global_mapping_pose_graph.cpp:391-405): target the whole first submap in a point grid,
    # source 10 % of the last, r = 2.0, 10 iterations, kept iff num_inliers / n_source >= 0.5
    first, last = mine[0][0], mine[-1][0]
    r = 2.0
    grid = gpu.PointGridGPU(first.frame, 1.05 * r, ctx=ctx)
    rng = np.random.default_rng(61)
    xyz, cov6 = last.frame.download()
    keep = rng.random(len(xyz)) < 0.1
    src = gpu.PointCloudGPU.clone(homog(xyz[keep]), po.cov4x4(cov6[keep].astype(F64)), ctx=ctx)
    T_true = synth.inv_pose(first.T_world_origin) @ last.T_world_origin
    res = gpu.align_vgicp([[gpu.IntegratedGICPFactorGPU(np.eye(4), 0, grid, src, r, ctx=ctx)]], [synth.perturb(T_true, rng, 0.01, 0.2)],
                          params={"max_iterations": 10})[0]
    assert res["num_inliers"] / src.n >= 0.5, res
    et, er = pose_error(res["T_target_source"], T_true)
    assert et < 0.05 and er < np.radians(0.25), (et, er)
