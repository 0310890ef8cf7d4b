"""CPU-only checks of the ICP factor's per-hit arithmetic and of the per-point normal (no GPU needed):
  * accumulate_icp_hit (glim_b200/csrc/gb_vgicp_math.cuh) compiled for the host (tests/cpp/icp_normals_host.cpp) against the fp64
    restatement (tests/icp_oracle.py) on seeded hits, hits far from the origin and exact hits; the error mode sums only the error
    and the count;
  * covariance_normal (glim_b200/csrc/gb_cov_math.cuh) compiled for the host against numpy.linalg.eigh plus the sign rule
    (tests/normals_oracle.py) on seeded covariances, and on non-finite, zero and repeated-eigenvalue inputs;
  * the arguments gb_cloud_estimate_normals, gb_cloud_normals and gb_icp_grid_factor_create reject before they touch a device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import icp_oracle as icp
from tests import normals_oracle as no

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


@pytest.fixture(scope="module")
def hl(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("icpn") / "libicp_normals_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so,
                           os.path.join(ROOT, "tests", "cpp", "icp_normals_host.cpp")])
    L = C.CDLL(so)
    vp = C.c_void_p
    L.icp_hit.argtypes = [C.c_int, vp, vp, vp, vp]
    L.normals.argtypes = [C.c_int, vp, vp, vp]
    return L


def p(a):
    return a.ctypes.data_as(C.c_void_p)


def rotation(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def host_hit(hl, mode, T, a, v):
    Tf = np.asarray(T, dtype=F32)
    pose12 = np.ascontiguousarray(np.concatenate([Tf[:3, :3].reshape(-1), Tf[:3, 3]]), dtype=F32)
    acc = np.zeros(32, F32)
    hl.icp_hit(mode, p(pose12), p(np.ascontiguousarray(a, dtype=F32)), p(np.ascontiguousarray(v, dtype=F32)), p(acc))
    return acc


def hits(rng, n, offset):
    for _ in range(n):
        T = np.eye(4)
        T[:3, :3] = rotation(rng)
        T[:3, 3] = rng.uniform(-20, 20, 3) + offset
        a = rng.uniform(-50, 50, 3)
        v = (T[:3, :3] @ a + T[:3, 3]) + rng.normal(scale=0.3, size=3)
        yield T, a.astype(F32), v.astype(F32)


@pytest.mark.parametrize("offset", [0.0, 1000.0])
def test_icp_hit_matches_fp64_restatement(hl, offset):
    """Every accumulator of one hit within 2e-6 of the restatement, relative to the hit's scale (1 + |q| + |r|)^2; with the
    target point on the transformed source point the error is zero and b_t vanishes."""
    rng = np.random.default_rng(4100 + int(offset))
    for T, a, v in hits(rng, 400, offset):
        got = host_hit(hl, 0, T, a, v)
        ref = icp.hit(T, a, v)
        Tf = np.asarray(T, dtype=F32).astype(np.float64)
        q = Tf[:3, :3] @ a.astype(np.float64) + Tf[:3, 3]
        scale = (1.0 + np.linalg.norm(q) + np.linalg.norm(v - q)) ** 2
        assert np.abs(got[:29] - ref).max() < 2e-6 * scale, (got[:29] - ref)
        assert (got[29:] == 0).all()
    T = np.eye(4)
    T[:3, 3] = [1.0, 2.0, 3.0]
    a = np.array([0.5, -0.25, 2.0], F32)
    got = host_hit(hl, 0, T, a, a + np.array([1.0, 2.0, 3.0], F32))
    assert got[27] == 0 and (got[21:27] == 0).all() and got[28] == 1


def test_icp_error_mode_sums_error_and_count_only(hl):
    rng = np.random.default_rng(4200)
    for T, a, v in hits(rng, 100, 0.0):
        got = host_hit(hl, 1, T, a, v)
        ref = icp.hit(T, a, v)
        scale = (1.0 + np.linalg.norm(a) + np.linalg.norm(T[:3, 3]) + np.sqrt(ref[27])) ** 2
        assert abs(got[27] - ref[27]) < 2e-6 * scale and got[28] == 1
        assert (np.delete(got, [27, 28]) == 0).all()


def host_normals(hl, xyz, cov6):
    xyz, cov6 = np.ascontiguousarray(xyz, dtype=F32), np.ascontiguousarray(cov6, dtype=F32)
    out = np.empty((len(xyz), 3), F32)
    hl.normals(len(xyz), p(xyz), p(cov6), p(out))
    return out


def random_covs(rng, n, spread):
    """covariances R diag(l) R^T with eigenvalues drawn log-uniformly over `spread` decades -> (n,6) fp32"""
    out = np.empty((n, 6))
    for i in range(n):
        R = rotation(rng)
        C6 = R @ np.diag(10.0 ** rng.uniform(-spread, 0, 3)) @ R.T
        out[i] = C6[[0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    return out.astype(F32)


def test_normals_match_eigh_and_the_sign_rule(hl):
    """1 - |cos| < 1e-9 against eigh wherever the relative eigen-gap exceeds 1e-3; p . n <= 0 wherever |p . n| > 1e-6 |p|."""
    rng = np.random.default_rng(4300)
    n = 4000
    xyz = rng.uniform(-80, 80, (n, 3)).astype(F32)
    xyz[:100] += F32(5000.0)  # far from the origin
    cov6 = random_covs(rng, n, 4)
    got = host_normals(hl, xyz, cov6).astype(np.float64)
    ref, gap = no.normals(xyz, cov6)
    ok = gap > 1e-3
    assert ok.mean() > 0.9
    cos = np.abs((got * ref).sum(1)) / np.maximum(np.linalg.norm(got, axis=1), 1e-30)  # the fp32 rounding of the length
    assert (1.0 - cos[ok]).max() < 1e-9
    assert np.abs(np.linalg.norm(got, axis=1) - 1).max() < 1e-6
    pn = (xyz.astype(np.float64) * got).sum(1)
    big = np.abs(pn) > 1e-6 * np.linalg.norm(xyz, axis=1)
    assert big.mean() > 0.99 and (pn[big] <= 0).all()
    assert np.array_equal(np.sign(pn[ok & big]), np.sign((xyz.astype(np.float64) * ref).sum(1)[ok & big]))


def test_normals_of_adversarial_inputs(hl):
    """Non-finite position or covariance: zero.  Zero covariance: the solver's axis (1, 0, 0), sign-ruled.  A repeated smallest
    eigenvalue: a unit vector of that eigenspace, sign-ruled."""
    nan, inf = F32(np.nan), F32(np.inf)
    xyz = np.array([[nan, 1, 2], [1, inf, 2], [1, 2, 3], [1, 2, 3], [3, 1, 2], [-3, 1, 2], [2, -1, 5], [0, 0, 0]], F32)
    cov6 = np.array([[1, 0, 0, 1, 0, 1], [1, 0, 0, 1, 0, 1], [nan, 0, 0, 1, 0, 1], [1, 0, 0, inf, 0, 1],
                     [0, 0, 0, 0, 0, 0], [0, 0, 0, 0, 0, 0], [1, 0, 0, 1, 0, 2], [1, 0, 0, 1, 0, 2]], F32)
    got = host_normals(hl, xyz, cov6)
    assert (got[:4] == 0).all()
    assert np.array_equal(got[4], [-1, 0, 0]) and np.array_equal(got[5], [1, 0, 0])
    for i in (6, 7):
        assert got[i][2] == 0 and abs(np.linalg.norm(got[i]) - 1) < 1e-6
    assert (xyz[6] * got[6]).sum() <= 0


def test_invalid_arguments_are_rejected_on_the_host():
    """GB_ERR_INVALID_ARGUMENT before the call looks for a device."""
    from glim_b200 import capi

    L = capi.lib()
    dummy = C.c_void_p(1)  # never dereferenced: validation comes first
    out = np.zeros(3, F32)
    h = C.c_void_p()
    assert L.gb_cloud_estimate_normals(None, dummy) == 1 and L.gb_cloud_estimate_normals(dummy, None) == 1
    assert L.gb_cloud_normals(None, capi.ptr(out)) == 1 and L.gb_cloud_normals(dummy, None) == 1
    assert L.gb_icp_grid_factor_create(None, dummy, dummy, 1.0, C.byref(h)) == 1
    assert L.gb_icp_grid_factor_create(dummy, dummy, dummy, 1.0, None) == 1
    for r in (0.0, -1.0, float("nan"), float("inf")):
        assert L.gb_icp_grid_factor_create(dummy, dummy, dummy, r, C.byref(h)) == 1 and not h.value
