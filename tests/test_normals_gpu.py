"""gb_cloud_estimate_normals on the H100: the normals of a cloud with covariances against numpy.linalg.eigh plus the sign rule
(tests/normals_oracle.py) and bit for bit against the host build of the same function (tests/cpp/icp_normals_host.cpp); zero
normals for non-finite points; uploaded normals overwritten; FPFH features discarded; the refusals and the launch counts."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth
from tests import normals_oracle as no
from tests import voxelmap_oracle as vo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


@pytest.fixture(scope="module")
def hl(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("nrm") / "libicp_normals_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "cpp", "icp_normals_host.cpp")])
    L = C.CDLL(so)
    L.normals.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


@pytest.fixture(scope="module")
def frames():
    return vo.arc_frames(6, 32 * 200, nan_frame=1)


def merged(ctx, frames):
    """a merged submap of frames 2-5 (gb_merge_frames): covariances, no normals"""
    clouds = [gpu.PointCloudGPU.clone(f[0], f[1], ctx=ctx) for f in frames[2:6]]
    poses = [synth.inv_pose(frames[2][2]) @ f[2] for f in frames[2:6]]
    return gpu.merge_frames_gpu(poses, clouds, 0.1, ctx=ctx, host_outputs=False)[2]


def with_adversarial(frame):
    """a frame with NaN points (every 7th), plus points with an infinite covariance entry, a zero covariance and a repeated
    smallest eigenvalue"""
    pts, cov = frame[0].copy(), frame[1].copy()
    cov[3, 1, 1] = np.inf
    cov[5, :3, :3] = 0.0
    cov[8, :3, :3] = np.diag([0.01, 0.01, 0.5])
    return pts, cov


def host_normals(hl, xyz, cov6):
    out = np.empty((len(xyz), 3), F32)
    hl.normals(len(xyz), capi.ptr(np.ascontiguousarray(xyz, dtype=F32)), capi.ptr(np.ascontiguousarray(cov6, dtype=F32)), capi.ptr(out))
    return out


@pytest.mark.parametrize("which", ["frame", "submap"])
def test_normals_match_the_restatement_and_the_host_build(ctx, hl, frames, which):
    """Within 1e-9 (1 - |cos|) of eigh wherever the relative eigen-gap exceeds 1e-3; the sign rule exact wherever |p . n| >
    1e-6 |p|; bit-identical to the host build on the same fp32 inputs; zero for the non-finite points."""
    if which == "submap":
        cloud = merged(ctx, frames)
    else:
        cloud = gpu.PointCloudGPU.clone(*with_adversarial(frames[1]), ctx=ctx)
    got = cloud.estimate_normals().normals()
    xyz, cov6 = cloud.download()
    assert np.array_equal(got, host_normals(hl, xyz, cov6))
    ref, gap = no.normals(xyz, cov6)
    g = got.astype(np.float64)
    bad = ~(np.isfinite(xyz).all(1) & np.isfinite(cov6).all(1))
    ok = gap > 1e-3
    assert ok[~bad].mean() > 0.9
    cos = np.abs((g * ref).sum(1)) / np.maximum(np.linalg.norm(g, axis=1), 1e-30)
    assert (1.0 - cos[ok]).max() < 1e-9
    pn = (xyz.astype(np.float64) * g).sum(1)
    big = np.abs(pn) > 1e-6 * np.linalg.norm(xyz, axis=1)
    assert (pn[big] <= 0).all()
    assert (got[bad] == 0).all() and (np.linalg.norm(g[~bad], axis=1) > 0.999).all()
    if which == "frame":
        assert bad.sum() > 100 and bad[3]
        assert np.array_equal(np.abs(got[5]), [1, 0, 0]) and abs(got[8][2]) < 1e-6


def test_uploaded_normals_are_overwritten_and_features_discarded(ctx, frames):
    """A cloud uploaded with (wrong) normals gets the same normals as one uploaded without; its FPFH features are discarded, so
    gb_cloud_fpfh and the matcher refuse it until they are estimated again, and then equal the bare cloud's."""
    pts, cov, _ = frames[3]
    wrong = np.tile([0.0, 0.0, 1.0, 0.0], (len(pts), 1))
    a = gpu.PointCloudGPU.clone(pts, cov, wrong, ctx=ctx).estimate_fpfh(1.5)
    b = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
    assert np.array_equal(a.normals(), wrong[:, :3].astype(F32))
    a.estimate_normals()
    b.estimate_normals()
    assert np.array_equal(a.normals(), b.normals())
    with pytest.raises(capi.GlimB200Error):
        a.fpfh()
    b.estimate_fpfh(1.5)
    with pytest.raises(capi.GlimB200Error):
        gpu.fpfh_match(a, b)
    assert np.array_equal(a.estimate_fpfh(1.5).fpfh(), b.fpfh())
    nrm = C.c_void_p()
    capi.check(capi.lib().gb_cloud_device_ptrs(b.h, None, None, None, C.byref(nrm)))
    assert nrm.value


def test_refusals_and_launch_counts(ctx, frames):
    """A cloud without covariances is refused before any launch; an empty cloud makes no launch, any other exactly one."""
    L = capi.lib()
    pts, cov, _ = frames[0]
    bare = gpu.PointCloudGPU.clone(pts, ctx=ctx)
    l0 = ctx.kernel_launches
    assert L.gb_cloud_estimate_normals(ctx.h, bare.h) == 1
    assert L.gb_cloud_normals(bare.h, capi.ptr(np.zeros((len(pts), 3), F32))) == 1
    assert ctx.kernel_launches == l0
    empty = gpu.PointCloudGPU.clone(np.zeros((0, 4)), np.zeros((0, 4, 4)), ctx=ctx)
    empty.estimate_normals()
    assert ctx.kernel_launches == l0 and empty.normals().shape == (0, 3)
    cloud = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
    for _ in range(2):
        l0 = ctx.kernel_launches
        cloud.estimate_normals()
        assert ctx.kernel_launches - l0 == 1
    if L.gb_device_count() > 1:
        ctx1 = gpu.Context(1)
        other = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx1)
        l0 = ctx.kernel_launches
        assert L.gb_cloud_estimate_normals(ctx.h, other.h) == 1 and ctx.kernel_launches == l0
