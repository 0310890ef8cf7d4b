"""CPU-only parity of the sweep kernels' per-point arithmetic.

glim_b200/csrc/gb_vgicp_math.cuh holds the text both k_vgicp_sweep3 / 5 compile for the device (transform, voxel coordinate,
hash, fused Mahalanobis matrix, the 29 accumulators of a hit, the surface-validation gate, the slab <-> record map).  Here the
SAME text is compiled for the host with g++ (tests/cpp/kernel_math_host.cpp drives it with a scalar emulation of sweep3's item
structure) and checked against the fp64 oracle -- so a change to the kernel arithmetic is caught on the CPU-only box, before the
GPU parity tests (`-m gpu`) run.  This is a test of the TEXT, not of the device build: nvcc contracts a*b+c into FMAs where g++
(with -ffp-contract=off) does not, so Hessians agree to fp32 rounding, while everything the kernel writes with explicit fmaf --
the lookup transform and the surface-validation gate -- is bit-identical by construction (inlier sets and gate decisions exact).
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle
from tests import util
from tests.util import REL_TOL, cov_colmajor16, rel_err, scan_pair, test_poses
from glim_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def km(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("km") / "libkernel_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so, os.path.join(ROOT, "tests", "cpp", "kernel_math_host.cpp")])
    L = C.CDLL(so)
    vp = C.c_void_p
    L.km_sweep.argtypes = [C.c_int, vp, vp, vp, vp, vp, C.c_uint, C.c_int, vp, C.c_float, vp, vp, C.c_int, vp, vp]
    L.km_coord.argtypes = [C.c_float, C.c_float]
    L.km_hash.restype = C.c_uint
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def planes(xyz, cov6):
    """device layout of a cloud (DESIGN.md 3): p0 = {x y z c00}, p1 = {c01 c02 c11 c12}, p2 = c22; cov6 = (c00 c01 c02 c11 c12 c22)"""
    p0 = np.ascontiguousarray(np.concatenate([xyz, cov6[:, 0:1]], axis=1), dtype=np.float32)
    p1 = np.ascontiguousarray(cov6[:, 1:5], dtype=np.float32)
    p2 = np.ascontiguousarray(cov6[:, 5], dtype=np.float32)
    return p0, p1, p2


def voxel_records(m):
    v = np.zeros((m.num_voxels, 12), np.float32)
    v[:, 0:3] = m.vmean
    v[:, 3] = m.vcov[:, 0]
    v[:, 4:8] = m.vcov[:, 1:5]
    v[:, 8] = m.vcov[:, 5]
    v[:, 9] = m.vnum
    return v


def sweep(km, m, xyz, cov6, T_lin, T_eval=None, normals=None, chunk=2048):
    p0, p1, p2 = planes(xyz, cov6)
    nr = None
    if normals is not None:
        nr = np.zeros((len(xyz), 4), np.float32)
        nr[:, :3] = np.asarray(normals)[:, :3]
    acc = np.zeros(29)
    corr = np.empty(len(xyz), np.int32)
    vox = voxel_records(m)
    buckets = np.ascontiguousarray(m.buckets, dtype=np.int32)
    assert m.num_buckets & (m.num_buckets - 1) == 0
    Tl = oracle.pose_colmajor(T_lin)
    Te = oracle.pose_colmajor(T_eval) if T_eval is not None else None
    km.km_sweep(len(xyz), _p(p0), _p(p1), _p(p2), _p(nr), _p(buckets), m.num_buckets - 1, 10, _p(vox), np.float32(1.0) / np.float32(m.resolution), _p(Tl), _p(Te), chunk, _p(acc), _p(corr))
    return acc, corr


def unpack29(acc):
    H = np.zeros((6, 6))
    k = 0
    for i in range(6):
        for j in range(i, 6):
            H[i, j] = H[j, i] = acc[k]
            k += 1
    return H, acc[21:27].copy(), acc[27], acc[28]


def adjoint(T):
    """GTSAM Pose3::AdjointMap of T, tangent order [rot; trans] (SURVEY A.4)"""
    R, t = T[:3, :3], T[:3, 3]
    Ad = np.zeros((6, 6))
    Ad[:3, :3] = R
    Ad[3:, 3:] = R
    Ad[3:, :3] = synth.hat(t) @ R
    return Ad


@pytest.fixture(scope="module")
def data():
    sp = scan_pair()
    packed = [oracle.pack_cloud(sp["points"][k], cov_colmajor16(sp["covs"][k])) for k in (0, 1)]
    T_gt = synth.inv_pose(sp["poses"][0]) @ sp["poses"][1]
    return sp, packed, T_gt


@pytest.mark.parametrize("res", [0.25, 0.5, 1.0])
def test_host_build_of_the_kernel_arithmetic_matches_oracle(km, data, res):
    sp, packed, T_gt = data
    m = oracle.GpuMap(*packed[0], res)
    xyz, cov6 = packed[1]
    for T in test_poses(T_gt, 3):
        acc, corr = sweep(km, m, xyz, cov6, T)
        ref_raw, ref_corr = oracle.linearize_gpumap(m, xyz, cov6, T)
        ref = oracle.split122(ref_raw)
        assert np.array_equal(corr, ref_corr), "inlier set differs from the oracle"
        H, b, e, n = unpack29(acc)
        assert n == ref["num_inliers"] > 0
        assert rel_err(H, ref["H_tt"]) < REL_TOL
        assert abs(e - ref["error"]) < REL_TOL * ref["error"]
        scale = max(np.linalg.norm(ref["b_t"]), 0.1 * np.sqrt(np.trace(ref["H_tt"]) * ref["error"]))
        assert np.linalg.norm(b - ref["b_t"]) < REL_TOL * scale
        # the epilogue's identities (SURVEY A.4) applied to the host-built H_tt / b_t reproduce the oracle's source blocks,
        # which the oracle forms from J_s directly
        Tf = np.asarray(T, dtype=np.float32).astype(np.float64)  # the kernel's Isometry3f cast
        Ad = adjoint(Tf)
        assert rel_err(Ad.T @ H @ Ad, ref["H_ss"]) < REL_TOL
        assert rel_err(-H @ Ad, ref["H_ts"]) < REL_TOL
        scale_s = max(np.linalg.norm(ref["b_s"]), 0.1 * np.sqrt(np.trace(ref["H_ss"]) * ref["error"]))
        assert np.linalg.norm(-Ad.T @ b - ref["b_s"]) < REL_TOL * scale_s
        # every entry of the record the epilogue forms from the host-built sums within its own error bound
        hits = util.factor_hits(m.vmean, m.vcov, xyz, cov6, T, corr)
        util.check_entrywise(util.epilogue(H, b, e, n, Ad), ref, util.record_scale(hits), what=("host build", res))


def test_item_size_does_not_change_the_result_beyond_rounding(km, data):
    sp, packed, T_gt = data
    m = oracle.GpuMap(*packed[0], 0.5)
    xyz, cov6 = packed[1]
    a, ca = sweep(km, m, xyz, cov6, T_gt, chunk=2048)
    b, cb = sweep(km, m, xyz, cov6, T_gt, chunk=128)  # tapered items at the tail of a sweep
    assert np.array_equal(ca, cb) and a[28] == b[28]
    assert np.allclose(a, b, rtol=2e-5, atol=1e-6 * np.abs(a).max())


def test_error_mode_uses_inliers_of_the_linearization_pose(km, data):
    sp, packed, T_gt = data
    m = oracle.GpuMap(*packed[0], 0.5)
    xyz, cov6 = packed[1]
    T_lin = T_gt
    T_eval = synth.perturb(T_gt, synth.rng_for(5), 0.01, 0.05)
    acc, corr = sweep(km, m, xyz, cov6, T_lin, T_eval=T_eval)
    ref = oracle.error_gpumap(m, xyz, cov6, T_lin, T_eval)
    assert abs(acc[27] - ref) < REL_TOL * ref
    assert np.array_equal(corr, m.correspondences(xyz, T_lin))
    assert np.all(acc[:27] == 0.0)  # error mode accumulates error and count only


def test_surface_validation_gate_is_bit_identical_with_oracle(km, data):
    sp, packed, T_gt = data
    m = oracle.GpuMap(*packed[0], 0.5)
    xyz, cov6 = packed[1]
    nrm = sp["normals"][1]
    rejected = 0
    for T in (T_gt, synth.perturb(T_gt, synth.rng_for(6), 0.5, 0.3)):  # a good pose and a ~30 degree misalignment
        acc, corr = sweep(km, m, xyz, cov6, T, normals=nrm)
        ref_raw, ref_corr = oracle.linearize_gpumap(m, xyz, cov6, T, normals=nrm)
        assert np.array_equal(corr, ref_corr), "gate decisions differ from the oracle"
        ref = oracle.split122(ref_raw)
        H, b, e, n = unpack29(acc)
        assert n == ref["num_inliers"]
        assert rel_err(H, ref["H_tt"]) < REL_TOL
        rejected += int((corr == -2).sum())
    assert rejected > 0


def test_nan_point_and_singular_covariance_contribute_nothing(km, data):
    sp, packed, T_gt = data
    m = oracle.GpuMap(*packed[0], 0.5)
    xyz, cov6 = (a.copy() for a in packed[1])
    xyz[5] = np.nan
    xyz[6, 1] = np.inf
    hit = int(np.flatnonzero(m.correspondences(xyz, T_gt) >= 0)[10])
    cov6[hit] = 0.0  # with a zero source covariance the fused covariance is the voxel's: still regular -> counted
    acc, corr = sweep(km, m, xyz, cov6, T_gt)
    ref_raw, _ = oracle.linearize_gpumap(m, xyz, cov6, T_gt)
    ref = oracle.split122(ref_raw)
    H, b, e, n = unpack29(acc)
    assert np.isfinite(acc).all()
    assert n == ref["num_inliers"]
    assert rel_err(H, ref["H_tt"]) < REL_TOL


def test_coord_hash_and_slab_map(km):
    L = oracle.lib()
    rng = np.random.default_rng(3)
    for res in (0.1, 0.25, 0.5, 1.0):
        inv = np.float32(1.0) / np.float32(res)
        for p in np.concatenate([rng.uniform(-200, 200, 200), np.arange(-3, 3, 0.25), [-0.0, 1e-7, -1e-7]]).astype(np.float32):
            c = np.zeros(3, np.int32)
            pp = np.array([p, p, p], np.float32)
            L.go_voxel_coord_f32(pp.ctypes.data_as(C.c_void_p), C.c_float(inv), c.ctypes.data_as(C.c_void_p))
            assert km.km_coord(C.c_float(p), C.c_float(inv)) == c[0]
    for x, y, z in rng.integers(-(1 << 20), 1 << 20, (200, 3)):
        assert km.km_hash(int(x), int(y), int(z)) == (L.go_voxel_hash(int(x), int(y), int(z)) & 0xFFFFFFFF)
    # slab row element -> record index: a bijection onto the record entries a row carries, consistent with multi_gpu.pack_slab_row
    from glim_b200 import multi_gpu

    rec = np.arange(122, dtype=np.float64) + 1.0
    # symmetric H blocks so that upper-triangle packing is well defined
    d = oracle.split122(rec)
    for k in ("H_tt", "H_ss"):
        d[k] = np.triu(d[k]) + np.triu(d[k], 1).T
    row = multi_gpu.pack_slab_row(d)
    flat = np.zeros(122)
    flat[0:36] = d["H_tt"].T.reshape(36)
    flat[36:72] = d["H_ss"].T.reshape(36)
    flat[72:108] = d["H_ts"].T.reshape(36)
    flat[108:114], flat[114:120], flat[120], flat[121] = d["b_t"], d["b_s"], d["error"], d["num_inliers"]
    idx = [km.km_slab_to_record(e) for e in range(92)]
    assert len(set(idx)) == 92
    assert np.array_equal(np.asarray(row[:92], dtype=np.float64), flat[idx])


def test_adversarial_and_generated_poses(km, data):
    """SURVEY section 4 'kernel parity' tier on the CPU-only box: identity, 180 degree yaw, large translations (negative
    coordinates, hash wrap), no overlap at all -- then hypothesis-generated poses.  Inlier sets must be exact for every pose
    (the lookup is integer work on explicitly fused fp32 arithmetic), Hessians within the 1e-4 bar wherever there are inliers."""
    from hypothesis import HealthCheck, given, settings, strategies as st

    sp, packed, T_gt = data
    m = oracle.GpuMap(*packed[0], 0.5)
    xyz, cov6 = packed[1]

    def check(T):
        acc, corr = sweep(km, m, xyz, cov6, T)
        ref_raw, ref_corr = oracle.linearize_gpumap(m, xyz, cov6, T)
        ref = oracle.split122(ref_raw)
        assert np.array_equal(corr, ref_corr)
        H, b, e, n = unpack29(acc)
        assert n == ref["num_inliers"]
        if n >= 50:  # a handful of inliers is a cancelling sum of a few terms: the bar is stated for a registration-sized set
            assert rel_err(H, ref["H_tt"]) < REL_TOL
            assert abs(e - ref["error"]) < REL_TOL * max(ref["error"], 1e-12)
        return n

    assert check(np.eye(4)) > 0
    for T in (synth.pose(0, 0, 0, np.pi), synth.pose(3.0, -2.0, 0.1, 0.3, 0.02, -0.01), synth.pose(-7.5, 4.25, 0.0, -2.0)):
        check(T)
    assert check(synth.pose(5000.0, -3000.0, 100.0, 1.0)) == 0
    assert check(synth.pose(-40000.0, 65000.0, -300.0, -0.7)) == 0  # |voxel coordinate| ~ 1.3e5: the u32 hash wraps

    @settings(max_examples=25, deadline=None, derandomize=True, suppress_health_check=list(HealthCheck))
    @given(st.floats(-np.pi, np.pi), st.floats(-0.3, 0.3), st.floats(-0.3, 0.3), st.floats(-8, 8), st.floats(-8, 8), st.floats(-1, 1))
    def generated(yaw, pitch, roll, x, y, z):
        check(T_gt @ synth.pose(x, y, z, yaw, pitch, roll))

    generated()
