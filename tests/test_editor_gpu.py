"""The map editor's selection tools and point removal on the device (gb_select_gizmo, gb_select_radius, gb_remove_points)
against the numpy restatement (tests/editor_oracle.py): gizmo ids exactly on rotated, scaled and sheared boxes and spheres;
the radius tools' selections exactly (OUTLIERS up to points within 1e-12 relative of the threshold, reported); removed clouds
bit for bit against a re-upload of their survivors, through download, normals, a VGICP linearization and a voxel map; the
editor's recipe end to end; refusals and launch counts."""
import numpy as np
import pytest

from glim_b200 import capi, gpu
from tests import editor_oracle as eo
from tests import segment_oracle as so

pytestmark = pytest.mark.gpu
F32, F64 = np.float32, np.float64


@pytest.fixture(scope="module")
def ctx():
    return gpu.Context(0)


def homog(xyz):
    xyz = np.asarray(xyz, F64)
    return np.concatenate([xyz, np.ones((len(xyz), 1))], axis=1)


def covs44(cov6):
    c = np.asarray(cov6, F64)
    C = np.zeros((len(c), 4, 4))
    for (r, s), e in zip(((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)), range(6)):
        C[:, r, s] = C[:, s, r] = c[:, e]
    return C


def upload(ctx, xyz, covs=True, nrm=None):
    n4 = None if nrm is None else np.concatenate([np.asarray(nrm, F64), np.zeros((len(nrm), 1))], axis=1)
    cov = None
    if covs:
        rng = np.random.default_rng(len(xyz))
        L = rng.normal(scale=0.05, size=(len(xyz), 3, 3))
        cov = np.zeros((len(xyz), 4, 4))
        cov[:, :3, :3] = L @ np.swapaxes(L, 1, 2) + 1e-4 * np.eye(3)
    return gpu.PointCloudGPU.clone(homog(xyz), cov, n4, ctx=ctx)


def pose(rng, spread=40.0):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    T = np.eye(4)
    T[:3, :3] = q * np.sign(np.linalg.det(q))
    T[:3, 3] = rng.uniform(-spread, spread, 3)
    return T


def submaps(ctx, rng, K=14, n=3000):
    """K submaps around the origin of the world; frame 3 is empty, frame 5 has no covariances, a few NaN points"""
    frames, poses, xyz = [], [], []
    for k in range(K):
        m = 0 if k == 3 else n + int(rng.integers(0, 500))
        a = rng.uniform(-8, 8, (m, 3)).astype(F32)
        if m:
            a[:3] = np.nan
        T = pose(rng, 6.0)
        frames.append(upload(ctx, a, covs=k != 5))
        poses.append(T)
        xyz.append(a)
    return frames, poses, xyz


def gizmo(rng, scale, shear=0.0):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    S = np.diag(scale).astype(F64)
    S[0, 1] = shear
    model = np.eye(4)
    model[:3, :3] = q @ S
    model[:3, 3] = rng.uniform(-3, 3, 3)
    A = np.linalg.inv(model)
    A[3] = [0, 0, 0, 1]
    return A


def test_gizmo_ids_match_oracle(ctx):
    rng = np.random.default_rng(1)
    frames, poses, xyz = submaps(ctx, rng)
    cases = [gizmo(rng, [6, 4, 5]), gizmo(rng, [9, 2.5, 7], 1.5), gizmo(rng, [3, 3, 3])]
    far = np.eye(4)
    far[:3, 3] = -1e4  # a gizmo that holds no point
    whole = np.linalg.inv(poses[0])  # a unit gizmo scaled to hold submap 0 whole
    whole = np.diag([1 / 100, 1 / 100, 1 / 100, 1.0]) @ whole
    whole[3] = [0, 0, 0, 1]
    for A in cases + [far, whole]:
        for shape in ("box", "sphere"):
            got = gpu.select_gizmo(poses, frames, A, shape, ctx=ctx)
            ref = eo.select_gizmo(poses, xyz, A, shape)
            assert np.array_equal(got, ref), shape
    assert len(gpu.select_gizmo(poses, frames, far, "box", ctx=ctx)) == 0
    got = gpu.select_gizmo(poses, frames, whole, "box", ctx=ctx)
    assert np.sum((got >> np.uint64(32)) == 0) == len(xyz[0]) - 3  # every finite point of submap 0


def scene(rng):
    """a floor, a wall, sprinkled noise and duplicate points"""
    floor = np.stack([rng.uniform(-6, 6, 6000), rng.uniform(-6, 6, 6000), rng.normal(scale=0.01, size=6000)], 1)
    wall = np.stack([rng.uniform(-6, 6, 3000), np.full(3000, 2.0) + rng.normal(scale=0.01, size=3000), rng.uniform(0, 3, 3000)], 1)
    noise = rng.uniform([-6, -6, -1], [6, 6, 4], (300, 3))
    dup = np.repeat(floor[:20], 3, axis=0)
    xyz = np.concatenate([floor, wall, noise, dup]).astype(F32)
    xyz[rng.permutation(len(xyz))[:5]] = np.nan
    return xyz


def check_outliers(got, ref):
    """the selections agree except at points whose d_i lies within 1e-12 relative of the threshold; -> the exempted count"""
    assert got["status"] == ref["status"] and got["num_participants"] == ref["num_participants"]
    if ref["status"] != 0:
        assert got["num_selected"] == 0
        return 0
    assert abs(got["threshold"] - ref["threshold"]) <= 1e-12 * abs(ref["threshold"])
    near = ref["nodes"][np.abs(ref["d"] - ref["threshold"]) <= 1e-12 * abs(ref["threshold"])]
    a, b = set(got["selected"].tolist()), set(ref["selected"].tolist())
    assert (a ^ b) <= set(near.tolist())
    return len(near)


def test_radius_tools_match_oracle(ctx):
    rng = np.random.default_rng(2)
    xyz = scene(rng)
    cloud = upload(ctx, xyz)
    exempt = 0
    for center, radius in (((0.5, 1.5, 0.2), 2.0), ((-3.0, 2.0, 1.0), 1.5), ((2.0, -2.0, 0.0), 4.0)):
        got = gpu.select_radius(cloud, center, "inside", ctx=ctx, radius=radius)
        ref = eo.select_radius(xyz, center, "inside", radius=radius)
        assert got["status"] == 0 and np.array_equal(got["selected"], ref["selected"])
        for k in (10, 4, 16):
            got = gpu.select_radius(cloud, center, "outliers", ctx=ctx, radius=radius, k=k)
            ref = eo.select_radius(xyz, center, "outliers", radius=radius, k=k)
            exempt += check_outliers(got, ref)
            again = gpu.select_radius(cloud, center, "outliers", ctx=ctx, radius=radius, k=k)
            assert np.array_equal(again["selected"], got["selected"]) and again["threshold"] == got["threshold"]  # bit-identical
    print(f"outlier points exempted within 1e-12 of the threshold: {exempt}")
    assert exempt == 0
    few = gpu.select_radius(cloud, (100.0, 100.0, 0.0), "outliers", ctx=ctx, radius=2.0)
    assert few["status_name"] == "NOT_ENOUGH_POINTS" and few["num_selected"] == 0
    empty = upload(ctx, np.zeros((0, 3), F32), covs=False)
    assert gpu.select_radius(empty, (0, 0, 0), "outliers", ctx=ctx)["status"] == capi.RADIUS_NOT_ENOUGH_POINTS
    assert gpu.select_radius(empty, (0, 0, 0), "inside", ctx=ctx)["num_selected"] == 0


def reupload(ctx, frame, keep):
    xyz, cov6 = frame.download()
    covs = covs44(cov6[keep]) if frame_has_covs(frame) else None
    nrm = None
    try:
        nrm = frame.normals()[keep]
    except capi.GlimB200Error:
        pass
    n4 = None if nrm is None else np.concatenate([nrm.astype(F64), np.zeros((len(nrm), 1))], axis=1)
    return gpu.PointCloudGPU.clone(homog(xyz[keep]), covs, n4, ctx=ctx)


_COVS = {}


def frame_has_covs(frame):
    return _COVS.get(id(frame), True)


def same_cloud(a, b):
    xa, ca = a.download()
    xb, cb = b.download()
    assert a.n == b.n
    assert xa.tobytes() == xb.tobytes() and ca.tobytes() == cb.tobytes()


def test_removal_bit_identical_to_reupload(ctx):
    rng = np.random.default_rng(3)
    K = 12
    frames = []
    for k in range(K):
        n = 2000 + 100 * k
        a = rng.uniform(-10, 10, (n, 3)).astype(F32)
        a[5] = a[6]  # a duplicate point: equal Morton keys, ordered by index
        f = upload(ctx, a, covs=k != 2, nrm=rng.normal(size=(n, 3)) if k == 4 else None)
        _COVS[id(f)] = k != 2
        if k in (1, 7):
            f.estimate_normals()
        if k == 7:
            f.add_times(np.linspace(0.0, 0.1, n)).estimate_fpfh(2.5)
        frames.append(f)
    sizes = [f.n for f in frames]
    for trial in range(3):
        ids = []
        for k in rng.choice(K, 5, replace=False):
            i = rng.choice(sizes[k], int(rng.integers(1, sizes[k] // 3)), replace=False)
            ids.append((np.uint64(k) << np.uint64(32)) | i.astype(np.uint64))
        ids.append(np.array([(np.uint64(9) << np.uint64(32)) | np.uint64(j) for j in range(sizes[9])], np.uint64))  # a whole frame
        ids = np.concatenate(ids)
        ids = np.concatenate([ids, ids[: len(ids) // 4],  # duplicates
                              np.array([(np.uint64(K) << np.uint64(32)), (np.uint64(0) << np.uint64(32)) | np.uint64(sizes[0]),
                                        np.uint64(0xFFFFFFFFFFFFFFFF)], np.uint64)])  # out of range, index == size
        rng.shuffle(ids)
        res = gpu.remove_points(frames, ids, ctx=ctx)
        keep, removed, ignored = eo.remove_points(sizes, ids)
        assert res["num_removed"] == removed and res["num_ignored"] == ignored == 3
        assert res["num_changed"] == sum(kp is not None for kp in keep)
        for k in range(K):
            new = res["frames"][k]
            if keep[k] is None:
                assert new is frames[k]
                continue
            assert new is not frames[k] and new.n == len(keep[k])
            if new.n == 0:
                assert k == 9
                continue
            ref = reupload(ctx, frames[k], keep[k])
            same_cloud(new, ref)
            if k in (1, 4, 7):
                assert new.normals().tobytes() == ref.normals().tobytes()
            if k == 7:
                assert new.time_table()[1].size == 0
                with pytest.raises(capi.GlimB200Error):
                    new.fpfh()
            if k == 2:
                continue  # no covariances: no voxel map statistics to compare beyond the planes
            ma, mb = gpu.GaussianVoxelMapGPU(1.0, ctx=ctx).insert(new), gpu.GaussianVoxelMapGPU(1.0, ctx=ctx).insert(ref)
            for x, y in zip(ma.download(), mb.download()):
                assert x.tobytes() == y.tobytes()
            target = gpu.GaussianVoxelMapGPU(1.0, ctx=ctx).insert(frames[(k + 1) % K])
            T = np.eye(4)
            T[:3, 3] = [0.05, -0.02, 0.01]
            la = gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, target, new, ctx=ctx).linearize({1: T})
            lb = gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, target, ref, ctx=ctx).linearize({1: T})
            for key in la:
                assert np.asarray(la[key]).tobytes() == np.asarray(lb[key]).tobytes(), key
        # the inputs are untouched
        assert [f.n for f in frames] == sizes
    nothing = gpu.remove_points(frames, np.array([np.uint64(K) << np.uint64(32)], np.uint64), ctx=ctx)
    assert all(a is b for a, b in zip(nothing["frames"], frames)) and nothing["num_ignored"] == 1


def test_editor_recipe_end_to_end(ctx):
    rng = np.random.default_rng(4)
    frames, poses, xyz = [], [], []
    for k in range(6):
        a = scene(np.random.default_rng(10 + k))[:5000]
        frames.append(upload(ctx, a))
        poses.append(pose(rng, 3.0))
        xyz.append(a)
    for f in frames:
        f.estimate_normals()
    window, ids = gpu.concat_frames(poses, frames, ctx=ctx)
    center = so.transform_points(poses[0], xyz[0][10:11])[0]
    cut = gpu.min_cut(window, center, ctx=ctx)
    outl = gpu.select_radius(window, center, "outliers", ctx=ctx, radius=3.0)
    sel = np.concatenate([ids[cut["selected"]], ids[outl["selected"]], gpu.select_gizmo(poses, frames, gizmo(rng, [2, 2, 2]), "sphere", ctx=ctx)])
    assert len(sel) > 0
    res = gpu.remove_points(frames, sel, ctx=ctx)
    keep, removed, _ = eo.remove_points([f.n for f in frames], sel)
    assert res["num_removed"] == removed
    after, ids2 = gpu.concat_frames(poses, res["frames"], ctx=ctx)
    surv_xyz = [x if kp is None else x[kp] for x, kp in zip(xyz, keep)]
    ref_cloud = so.concat_frames(poses, [(x, None, None) for x in surv_xyz])
    ax, _ = after.download()
    assert after.n == sum(len(x) for x in surv_xyz)
    assert np.array_equal(ax, np.asarray(ref_cloud["xyz"], F32), equal_nan=True)
    # map the new ids back to the old numbering: no removed id reappears
    old = []
    for k in range(len(frames)):
        mine = ids2[(ids2 >> np.uint64(32)) == k] & np.uint64(0xFFFFFFFF)
        base = np.arange(frames[k].n) if keep[k] is None else keep[k]
        old.append((np.uint64(k) << np.uint64(32)) | base[mine.astype(np.int64)].astype(np.uint64))
    assert not set(np.concatenate(old).tolist()) & set(sel.tolist())


def launches(ctx, fn):
    before = ctx.kernel_launches
    fn()
    return ctx.kernel_launches - before


def test_refusals_and_launch_counts(ctx):
    rng = np.random.default_rng(5)
    f1 = [upload(ctx, rng.uniform(-5, 5, (1000, 3)).astype(F32))]
    f100 = [upload(ctx, rng.uniform(-5, 5, (1000, 3)).astype(F32)) for _ in range(100)]
    big = [upload(ctx, rng.uniform(-5, 5, (100000, 3)).astype(F32))]
    A = gizmo(rng, [4, 4, 4])
    for fr in (f1, f100, big):
        P = [np.eye(4)] * len(fr)
        assert launches(ctx, lambda: gpu.select_gizmo(P, fr, A, "box", ctx=ctx)) == 4
        ids = np.array([(np.uint64(len(fr) - 1) << np.uint64(32)) | np.uint64(3), np.uint64(7)], np.uint64)
        assert launches(ctx, lambda: gpu.remove_points(fr, ids, ctx=ctx)) == 5
        assert launches(ctx, lambda: gpu.select_radius(fr[0], (0, 0, 0), "inside", ctx=ctx)) == 2
        assert launches(ctx, lambda: gpu.select_radius(fr[0], (0, 0, 0), "outliers", ctx=ctx, radius=3.0)) == 14
        assert launches(ctx, lambda: gpu.select_radius(fr[0], (100, 0, 0), "outliers", ctx=ctx)) == 3
    assert launches(ctx, lambda: gpu.remove_points(f1, np.zeros(0, np.uint64), ctx=ctx)) == 0
    bad_bottom = np.eye(4)
    bad_bottom[3, 0] = 1e-9
    nan = np.eye(4)
    nan[0, 1] = np.nan
    for T, shape in ((bad_bottom, "box"), (nan, "sphere")):
        assert launches(ctx, lambda: pytest.raises(capi.GlimB200Error, gpu.select_gizmo, [np.eye(4)], f1, T, shape, ctx=ctx)) == 0
    for params in ({"radius": 0.0}, {"radius": np.inf}, {"k": 11, "mode": 1}, {"radius_offset": -1.0, "mode": 1}, {"mode": 5}):
        mode = params.pop("mode", 0)
        p = gpu.select_radius_params(mode=mode, **params)
        r = capi.SelectRadiusResult()
        q = np.zeros(3)
        before = ctx.kernel_launches
        assert capi.lib().gb_select_radius(ctx.h, f1[0].h, capi.ptr(q), capi.C.byref(p), capi.C.byref(r), None) == 1
        assert ctx.kernel_launches == before
