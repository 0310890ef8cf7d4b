"""The map editor's segmentation on the device (gb_concat_frames, gb_region_growing) against the numpy restatement
(tests/segment_oracle.py): labels, selection, seed and counts bit for bit on scenes that separate by angle, by side, by
distance and by key range, with normals uploaded and with normals from gb_cloud_estimate_normals; the concatenation bit for
bit with and without a window; the editor's recipe end to end; refusals and launch counts."""
import math

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth
from tests import segment_oracle as so

pytestmark = pytest.mark.gpu
F32, F64 = np.float32, np.float64


@pytest.fixture(scope="module")
def ctx():
    return gpu.Context(0)


def homog(xyz):
    xyz = np.asarray(xyz, F64)
    return np.concatenate([xyz, np.ones((len(xyz), 1))], axis=1)


def upload(ctx, xyz, nrm=None, covs=None):
    n4 = None if nrm is None else np.concatenate([np.asarray(nrm, F64), np.zeros((len(nrm), 1))], axis=1)
    return gpu.PointCloudGPU.clone(homog(xyz), covs, n4, ctx=ctx)


def check_region(ctx, cloud, xyz, nrm, seed_point, dt, ang, dil):
    got = gpu.region_growing(cloud, seed_point, ctx=ctx, labels=True, distance_threshold=dt, angle_threshold=ang, dilation_radius=dil)
    ref = so.region_growing(xyz, nrm, seed_point, dt, ang, dil)
    assert np.array_equal(got["labels"], ref["labels"])
    assert np.array_equal(got["selected"], ref["selected"])
    for k in ("seed", "status", "num_region", "num_selected", "num_components"):
        assert got[k] == ref[k], k
    return got, ref


def plane(rng, lo, hi, step, axis, at, noise=0.0):
    """grid points of the plane `axis` = at over [lo, hi) in the two other axes"""
    u = np.arange(lo[0], hi[0], step)
    v = np.arange(lo[1], hi[1], step)
    U, V = np.meshgrid(u, v, indexing="ij")
    P = np.zeros((U.size, 3))
    others = [a for a in range(3) if a != axis]
    P[:, others[0]], P[:, others[1]], P[:, axis] = U.ravel(), V.ravel(), at
    P += rng.normal(scale=noise, size=P.shape) if noise else 0
    N = np.zeros_like(P)
    N[:, axis] = 1.0
    return P, N


def room(rng):
    """a floor, two walls and a box standing on the floor; a few NaN points"""
    parts = [plane(rng, (0, 0), (6, 6), 0.1, 2, 0.0, 0.005), plane(rng, (0, 0), (6, 3), 0.1, 0, 0.0, 0.005),
             plane(rng, (0, 0), (6, 3), 0.1, 1, 0.0, 0.005), plane(rng, (3, 3), (4, 4), 0.1, 2, 1.0, 0.002),
             plane(rng, (3, 0), (4, 1), 0.1, 0, 3.0), plane(rng, (3, 0), (4, 1), 0.1, 1, 3.0)]
    P = np.concatenate([p for p, _ in parts]).astype(F32)
    N = np.concatenate([n for _, n in parts]).astype(F32)
    perm = rng.permutation(len(P))
    P, N = P[perm], N[perm]
    P[rng.choice(len(P), 7, replace=False)] = np.nan
    return P, N


def test_room_uploaded_normals(ctx):
    rng = np.random.default_rng(1)
    P, N = room(rng)
    cloud = upload(ctx, P, N)
    for ang, dil in ((math.radians(20), 0.35), (math.radians(20), 0.0), (math.pi, 0.5), (0.0, 0.0)):
        got, ref = check_region(ctx, cloud, P, N, [2.0, 2.0, 0.0], 0.15, ang, dil)
    got, _ = check_region(ctx, cloud, P, N, [2.0, 2.0, 0.0], 0.15, math.radians(20), 0.35)
    assert got["num_selected"] > got["num_region"] > 3000  # the floor, and the dilation reaches past its edge onto the walls
    again = gpu.region_growing(cloud, [2.0, 2.0, 0.0], ctx=ctx, labels=True, distance_threshold=0.15, angle_threshold=math.radians(20), dilation_radius=0.35)
    assert np.array_equal(again["labels"], got["labels"]) and np.array_equal(again["selected"], got["selected"])


def test_room_estimated_normals(ctx):
    rng = np.random.default_rng(2)
    P, _ = room(rng)
    P = P[np.isfinite(P).all(axis=1)]
    _, covs = synth.with_covariances(homog(P), 10)
    cloud = gpu.PointCloudGPU.clone(homog(P), covs, ctx=ctx).estimate_normals()
    N = cloud.normals()
    for ang, dil in ((math.radians(15), 0.3), (math.radians(60), 0.0)):
        check_region(ctx, cloud, P, N, [1.0, 1.0, 0.0], 0.15, ang, dil)


def test_parallel_planes_with_opposite_normals(ctx):
    rng = np.random.default_rng(3)
    a, na = plane(rng, (0, 0), (5, 5), 0.1, 2, 0.0)
    b, nb = plane(rng, (0, 0), (5, 5), 0.1, 2, 0.05)
    P = np.concatenate([a, b]).astype(F32)
    N = np.concatenate([na, -nb]).astype(F32)
    cloud = upload(ctx, P, N)
    got, _ = check_region(ctx, cloud, P, N, [1.0, 1.0, 0.0], 0.2, math.radians(30), 0.0)
    assert got["num_region"] == len(a) and got["num_components"] == 2
    got, _ = check_region(ctx, cloud, P, N, [1.0, 1.0, 0.0], 0.2, math.pi, 0.0)
    assert got["num_components"] == 1


def test_long_chain(ctx):
    """diameter about N: a union-find that misses a hook, or a level-by-level growth cut short, shows here"""
    rng = np.random.default_rng(4)
    n = 100_000
    P = np.zeros((n, 3))
    P[:, 0] = 0.4 * np.arange(n)
    P[:, 1] = 1000.0
    perm = rng.permutation(n)
    P, N = P[perm].astype(F32), np.tile(np.array([0, 0, 1], F32), (n, 1))
    cloud = upload(ctx, P, N)
    got, _ = check_region(ctx, cloud, P, N, [0.4 * (n - 1), 1000.0, 0.0], 0.5, 0.1, 0.0)
    assert got["num_region"] == n and got["num_components"] == 1
    P2 = P.copy()
    P2[perm == n // 2] = np.nan  # cut in the middle
    cloud2 = upload(ctx, P2, N)
    got, _ = check_region(ctx, cloud2, P2, N, [0.0, 1000.0, 0.0], 0.5, 0.1, 0.0)
    assert got["num_region"] == n // 2 and got["num_components"] == 2


def test_dense_plane_one_component(ctx):
    rng = np.random.default_rng(5)
    side = 1415  # about 2 M points
    P, N = plane(rng, (0, 0), (side * 0.05, side * 0.05), 0.05, 2, 0.0)
    P = P[: side * side].astype(F32)
    N = N[: side * side].astype(F32)
    P[:, 2] += rng.normal(scale=0.002, size=len(P)).astype(F32)
    cloud = upload(ctx, P, N)
    got, _ = check_region(ctx, cloud, P, N, [30.0, 30.0, 0.0], 0.12, math.radians(5), 0.0)
    assert got["num_components"] == 1 and got["num_region"] == len(P)


def test_many_small_clusters(ctx):
    rng = np.random.default_rng(6)
    centres = rng.uniform(-100, 100, (2000, 3))
    P = (np.repeat(centres, 20, axis=0) + rng.normal(scale=0.1, size=(40000, 3))).astype(F32)
    N = rng.normal(size=P.shape)
    N = (N / np.linalg.norm(N, axis=1, keepdims=True)).astype(F32)
    N[::97] = 0
    N[::101] = np.nan
    P[::53] = np.nan
    cloud = upload(ctx, P, N)
    for ang, dil in ((math.pi, 0.0), (math.radians(70), 0.25), (math.radians(120), 1.0)):
        got, _ = check_region(ctx, cloud, P, N, centres[17], 0.2, ang, dil)
        assert got["num_components"] > 2000


def test_key_range_and_no_seed(ctx):
    rng = np.random.default_rng(7)
    P, N = plane(rng, (0, 0), (2, 2), 0.1, 2, 0.0)
    far = np.array([[1.2e6, 0, 0], [1.2e6 + 0.05, 0, 0], [-3e38, 0, 0]])  # keys outside the 21-bit range at cell 0.105 m
    P = np.concatenate([P, far]).astype(F32)
    N = np.concatenate([N, np.tile([0, 0, 1], (3, 1))]).astype(F32)
    cloud = upload(ctx, P, N)
    got, _ = check_region(ctx, cloud, P, N, [1.2e6, 0, 0], 0.1, math.pi, 0.0)
    assert got["num_region"] == 1  # the far pair is close but takes part in no search
    bad = upload(ctx, np.full((5, 3), np.nan, F32), np.zeros((5, 3), F32))
    got, _ = check_region(ctx, bad, np.full((5, 3), np.nan, F32), np.zeros((5, 3), F32), [0, 0, 0], 0.5, 0.5, 1.0)
    assert got["status"] == capi.REGION_NO_SEED and got["seed"] == -1 and got["num_selected"] == 0
    assert (got["labels"] == -1).all()


def rotation(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def frames_and_poses(rng, K, n, covs=True, normals=True):
    poses, host = [], []
    for k in range(K):
        T = np.eye(4)
        T[:3, :3] = rotation(rng)
        T[:3, 3] = rng.uniform(-30, 30, 3)
        xyz = rng.uniform(-10, 10, (n + k, 3)).astype(F32)
        xyz[3] = np.nan
        A = rng.normal(size=(n + k, 3, 3))
        C = (A @ A.transpose(0, 2, 1) * 0.01) if covs else None
        nrm = rng.normal(size=(n + k, 3)).astype(F32) if normals else None
        poses.append(T)
        host.append((xyz, C, nrm))
    return poses, host


def as_oracle_frame(xyz, C, nrm):
    cov6 = None if C is None else C[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].astype(F32)
    return xyz, cov6, nrm


def upload_frame(ctx, xyz, C, nrm):
    c4 = None
    if C is not None:
        c4 = np.zeros((len(xyz), 4, 4))
        c4[:, :3, :3] = C
    return upload(ctx, xyz, nrm, c4)


WINDOW = (2.0, (-10, -9, -10), (10, 8, 9))


@pytest.mark.parametrize("window, K, n, empty_every", [pytest.param(None, 4, 3000, 0, id="None"), pytest.param(WINDOW, 4, 3000, 0, id="window1"),
                                                      pytest.param(None, 64, 300, 3, id="empty-frames"), pytest.param(WINDOW, 64, 300, 3, id="empty-frames-window")])
def test_concat_bit_exact(ctx, window, K, n, empty_every):
    rng = np.random.default_rng(8)
    poses, host = frames_and_poses(rng, K, n)
    if empty_every:  # frames with no points among the others, the first and the last included
        host = [tuple(a[:0] for a in h) if k % empty_every == 0 else h for k, h in enumerate(host)]
    frames = [upload_frame(ctx, *h) for h in host]
    cloud, ids = gpu.concat_frames(poses, frames, window=window, ctx=ctx)
    ref = so.concat_frames(poses, [as_oracle_frame(*h) for h in host], window)
    xyz, cov6 = cloud.download()
    assert cloud.size() == len(ref["xyz"]) > 0
    assert np.array_equal(xyz, ref["xyz"], equal_nan=True)
    assert np.array_equal(cov6, ref["cov6"], equal_nan=True)
    assert np.array_equal(cloud.normals(), ref["normals"], equal_nan=True)
    assert np.array_equal(ids, ref["ids"])
    if window is not None:
        assert cloud.size() < sum(f.n for f in frames)


def test_concat_carries_only_common_planes(ctx):
    rng = np.random.default_rng(9)
    poses, host = frames_and_poses(rng, 2, 500)
    _, host_nc = frames_and_poses(rng, 1, 500, covs=False)
    _, host_nn = frames_and_poses(rng, 1, 500, normals=False)
    base = [upload_frame(ctx, *h) for h in host]
    no_covs = upload_frame(ctx, *host_nc[0])
    no_nrm = upload_frame(ctx, *host_nn[0])
    cloud, _ = gpu.concat_frames(poses + [np.eye(4)], base + [no_nrm], ctx=ctx)
    with pytest.raises(capi.GlimB200Error):
        cloud.normals()
    cloud.estimate_normals()  # it carries covariances
    cloud, _ = gpu.concat_frames(poses + [np.eye(4)], base + [no_covs], ctx=ctx)
    ref = so.concat_frames(poses + [np.eye(4)], [as_oracle_frame(*h) for h in host + host_nc])
    assert np.array_equal(cloud.normals(), ref["normals"], equal_nan=True)
    assert not cloud.download()[1].any()  # zero covariances
    with pytest.raises(capi.GlimB200Error):
        cloud.estimate_normals()
    empty, ids = gpu.concat_frames([], [], ctx=ctx)
    assert empty.size() == 0 and len(ids) == 0
    none, ids = gpu.concat_frames(poses, base, window=(1.0, (10**6,) * 3, (10**6,) * 3), ctx=ctx)
    assert none.size() == 0 and len(ids) == 0


def test_merge_frames_unchanged_by_the_shared_transform(ctx):
    """gb_merge_frames without downsampling effect (a tiny voxel) keeps the transformed points: they match the oracle's
    transform of the same frames, through the same kernel gb_concat_frames uses.  A frame at a NaN pose is accepted and
    changes nothing: its points get no voxel key, and the other frames keep their order."""
    rng = np.random.default_rng(10)
    poses, host = frames_and_poses(rng, 3, 400)
    host = [(x[np.isfinite(x).all(axis=1)], C[np.isfinite(x).all(axis=1)], n) for x, C, n in host]
    frames = [upload_frame(ctx, x, C, None) for x, C, _ in host]
    pts, covs, _ = gpu.merge_frames_gpu(poses, frames, 1e-4, ctx=ctx)
    q = np.concatenate([so.transform_points(T, x) for T, (x, _, _) in zip(poses, host)])
    rows = lambda a: a[np.lexsort(a.T[::-1])]
    assert len(pts) == len(q)
    assert np.array_equal(rows(pts[:, :3]), rows(q))
    cat, _ = gpu.concat_frames(poses, frames, ctx=ctx)
    assert np.array_equal(cat.download()[0], q.astype(F32))
    nan_pose = np.full((4, 4), np.nan)
    pts_nan, covs_nan, _ = gpu.merge_frames_gpu(poses[:1] + [nan_pose] + poses[1:], frames[:1] + [frames[1]] + frames[1:], 1e-4, ctx=ctx)
    assert np.array_equal(pts_nan, pts) and np.array_equal(covs_nan, covs)


def test_editor_recipe_end_to_end(ctx):
    """submaps with local-frame normals -> concat_frames with a 2 m x +-5-cell window around a picked point -> region
    growing -> ids[selected], against the oracle on host-transformed fp64 copies under the same rules"""
    rng = np.random.default_rng(11)
    poses, host, frames = [], [], []
    for k in range(12):
        T = np.eye(4)
        yaw = rng.uniform(-np.pi, np.pi)
        T[:2, :2] = [[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]]
        T[:3, 3] = [8.0 * (k % 4), 8.0 * (k // 4), 0.0]
        world, wn = plane(rng, (T[0, 3] - 5, T[1, 3] - 5), (T[0, 3] + 5, T[1, 3] + 5), 0.15, 2, 0.0, 0.005)
        wall, wwn = plane(rng, (T[1, 3] - 5, 0), (T[1, 3] + 5, 3), 0.15, 0, T[0, 3] + 4.0, 0.005)
        Pw = np.concatenate([world, wall])
        Nw = np.concatenate([wn, wwn])
        R, t = T[:3, :3], T[:3, 3]
        local = ((Pw - t) @ R).astype(F32)  # R^T (p - t)
        ln = (Nw @ R).astype(F32)
        poses.append(T)
        host.append((local, None, ln))
        frames.append(upload(ctx, local, ln))
    picked = np.array([9.0, 7.0, 0.0])
    cell, w = 2.0, 5
    centre = np.floor(picked / cell).astype(int)
    window = (cell, tuple(centre - w), tuple(centre + w))
    cloud, ids = gpu.concat_frames(poses, frames, window=window, ctx=ctx)
    got = gpu.region_growing(cloud, picked, ctx=ctx, distance_threshold=0.3, angle_threshold=math.radians(10), dilation_radius=0.5)
    ref_cat = so.concat_frames(poses, host, window)
    ref = so.region_growing(ref_cat["xyz"], ref_cat["normals"], picked, 0.3, math.radians(10), 0.5)
    assert np.array_equal(ids, ref_cat["ids"])
    assert np.array_equal(ids[got["selected"]], ref_cat["ids"][ref["selected"]])
    assert got["num_region"] == ref["num_region"] > 1000 and got["num_selected"] > got["num_region"]


def launches(ctx, fn):
    before = ctx.kernel_launches
    fn()
    return ctx.kernel_launches - before


def test_refusals_make_no_launch(ctx):
    rng = np.random.default_rng(12)
    P, N = plane(rng, (0, 0), (2, 2), 0.1, 2, 0.0)
    cloud = upload(ctx, P.astype(F32), N.astype(F32))
    bare = upload(ctx, P.astype(F32))
    bad = [dict(cloud=bare), dict(seed=[np.nan, 0, 0]), dict(distance_threshold=0.0), dict(distance_threshold=np.inf),
           dict(angle_threshold=-0.1), dict(angle_threshold=3.2), dict(angle_threshold=np.nan), dict(dilation_radius=-1.0),
           dict(dilation_radius=np.inf)]
    for b in bad:
        c = b.pop("cloud", cloud)
        s = b.pop("seed", [0, 0, 0])

        def call():
            with pytest.raises(capi.GlimB200Error):
                gpu.region_growing(c, s, ctx=ctx, **b)
        assert launches(ctx, call) == 0, b
    T = np.eye(4)
    for poses, window in (([np.full((4, 4), np.nan)], None), ([T], (0.0, (0, 0, 0), (1, 1, 1))), ([T], (np.nan, (0, 0, 0), (1, 1, 1))),
                          ([T], (1.0, (0, 2, 0), (1, 1, 1)))):
        def call():
            with pytest.raises(capi.GlimB200Error):
                gpu.concat_frames(poses, [cloud], window=window, ctx=ctx)
        assert launches(ctx, call) == 0


@pytest.mark.parametrize("n", [1000, 100_000])
def test_launch_counts_are_constant(ctx, n):
    P = np.zeros((n, 3), F32)
    P[:, 0] = 0.4 * np.arange(n)
    N = np.tile(np.array([0, 0, 1], F32), (n, 1))
    for shape in ("chain", "ball"):
        if shape == "ball":
            P = np.random.default_rng(n).normal(size=(n, 3)).astype(F32)
        cloud = upload(ctx, P, N)
        g1 = launches(ctx, lambda: gpu.PointGridGPU(cloud, 1.05 * 0.5, ctx=ctx))
        g2 = launches(ctx, lambda: gpu.PointGridGPU(cloud, 1.05 * 0.7, ctx=ctx))
        assert launches(ctx, lambda: gpu.region_growing(cloud, P[0], ctx=ctx, distance_threshold=0.5, angle_threshold=0.1)) == g1 + 4
        assert launches(ctx, lambda: gpu.region_growing(cloud, P[0], ctx=ctx, distance_threshold=0.5, angle_threshold=0.1, dilation_radius=0.7)) == g1 + g2 + 5
        assert launches(ctx, lambda: gpu.concat_frames([np.eye(4)], [cloud], ctx=ctx)) == 7
        assert launches(ctx, lambda: gpu.concat_frames([np.eye(4)], [cloud], window=(1.0, (10**6,) * 3, (10**6,) * 3), ctx=ctx)) == 4
    empty = upload(ctx, np.zeros((0, 3), F32), np.zeros((0, 3), F32))
    assert launches(ctx, lambda: gpu.region_growing(empty, [0, 0, 0], ctx=ctx, dilation_radius=1.0)) == 0
    assert launches(ctx, lambda: gpu.concat_frames([np.eye(4)], [empty], ctx=ctx)) == 0
