"""CPU-only checks of GNC global registration (no GPU needed):
  * the schedule of gb_global_math.cuh compiled for the host (tests/cpp/gnc_math_host.cpp, the functions k_gnc_solve calls)
    against the numpy restatement (tests/gnc_oracle.py): same iteration count, pose and weights within 1e-10;
  * with unit weights the moment form equals RANSAC's three-point estimator;
  * the rule recovers a pose from planted correspondences mixed with uniform outliers;
  * fewer than three pairs are DEGENERATE;
  * sample picks and host validation of the arguments gb_gnc_align rejects before it touches a device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from glim_b200 import synth
from tests import gnc_oracle as gno

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


@pytest.fixture(scope="module")
def gn(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("gn") / "libgnc_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so, os.path.join(ROOT, "tests", "cpp", "gnc_math_host.cpp")])
    L = C.CDLL(so)
    vp = C.c_void_p
    L.gnc_solve.argtypes = [C.c_int, vp, vp, C.c_int, vp, vp, vp]
    L.gnc_pose_weighted.argtypes = [C.c_int, vp, vp, vp, C.c_int, vp]
    L.ransac_pose3.argtypes = [vp, vp, C.c_int, vp]
    return L


def p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_solve(gn, a, b, dof):
    a = np.ascontiguousarray(np.asarray(a, dtype=F32), dtype=np.float64)
    b = np.ascontiguousarray(np.asarray(b, dtype=F32), dtype=np.float64)
    T, w, it = np.zeros(16), np.zeros(len(a)), C.c_int()
    st = gn.gnc_solve(len(a), p(a), p(b), dof, p(T), p(w), C.byref(it))
    return T.reshape(4, 4).T, w, it.value, st


def planted(K, outlier_rate, dof, rng, noise=0.02, box=50.0):
    """K pairs: exact pairs under a known pose with `noise` m Gaussian noise, a fraction replaced by uniform outliers in a box
    -> (a, b fp32, T_gt, inlier mask)"""
    T = synth.pose(12.0, -7.0, 1.5, np.radians(75), *((np.radians(8), np.radians(-5)) if dof == 6 else (0.0, 0.0)))
    a = rng.uniform(-box / 2, box / 2, size=(K, 3))
    b = a @ T[:3, :3].T + T[:3, 3] + rng.normal(scale=noise, size=(K, 3))
    out = rng.random(K) < outlier_rate
    b[out] = rng.uniform(-box / 2, box / 2, size=(out.sum(), 3)) + T[:3, 3]
    return a.astype(F32), b.astype(F32), T, ~out


def pose_error(T, T_ref):
    d = synth.inv_pose(T_ref) @ T
    return float(np.linalg.norm(d[:3, 3])), float(np.degrees(np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1))))


@pytest.mark.parametrize("dof", [4, 6])
@pytest.mark.parametrize("K", [3, 50, 5000])
def test_host_schedule_matches_the_restatement(gn, dof, K):
    rng = np.random.default_rng(K * 10 + dof)
    a, b, _, _ = planted(K, 0.4 if K > 3 else 0.0, dof, rng, noise=0.05)
    T, w, it, st = host_solve(gn, a, b, dof)
    T_ref, w_ref, it_ref, st_ref = gno.gnc_solve(a, b, dof)
    assert (st, it) == (st_ref, it_ref) == (gno.GNC_FOUND, it_ref)
    assert 1 <= it <= 22
    assert np.abs(T - T_ref).max() < 1e-10
    assert np.abs(w - w_ref).max() < 1e-10


@pytest.mark.parametrize("dof", [4, 6])
def test_unit_weights_equal_the_three_point_estimator(gn, dof):
    rng = np.random.default_rng(5 + dof)
    n = 0
    for _ in range(200):
        a = rng.uniform(-20, 20, size=(3, 3)) + [400.0, -250.0, 10.0]
        b = rng.uniform(-20, 20, size=(3, 3)) + [-100.0, 50.0, 3.0]
        a, b = np.asarray(a, F32).astype(np.float64), np.asarray(b, F32).astype(np.float64)
        T3, Tw = np.zeros(16), np.zeros(16)
        if not gn.ransac_pose3(p(a), p(b), dof, p(T3)):
            continue
        gn.gnc_pose_weighted(3, p(a), p(b), p(np.ones(3)), dof, p(Tw))
        assert np.abs(T3 - Tw).max() < 1e-12
        n += 1
    assert n > 190


@pytest.mark.parametrize("dof", [4, 6])
@pytest.mark.parametrize("outlier_rate", [0.5, 0.7])
def test_recovers_planted_correspondences(gn, dof, outlier_rate):
    rng = np.random.default_rng(int(outlier_rate * 10) + dof)
    a, b, T_gt, inl = planted(2000, outlier_rate, dof, rng)
    T, w, it, st = host_solve(gn, a, b, dof)
    et, er = pose_error(T, T_gt)
    assert st == gno.GNC_FOUND and et < 1e-2 and er < 0.1, (et, er, it)
    assert w[inl].mean() > 0.9 and w[~inl].mean() < 0.05


def test_fewer_than_three_pairs_are_degenerate(gn):
    for K in (0, 1, 2):
        a = np.arange(3 * K, dtype=F32).reshape(K, 3)
        T, w, it, st = host_solve(gn, a, a + 1, 6)
        assert (st, it) == (gno.GNC_DEGENERATE, 0) and np.array_equal(T, np.eye(4)) and (w == 0).all()
        assert gno.gnc_solve(a, a + 1, 6)[2:] == (0, gno.GNC_DEGENERATE)


def test_sample_pick():
    assert np.array_equal(gno.gnc_samples(1, 50, 50), np.arange(50))
    s = gno.gnc_samples(53123, 1000, 100)
    assert len(s) == 100 and (np.diff(s) > 0).all()
    h = gno.rg_hash(53123, np.arange(1000))
    assert h[s].max() < np.delete(h, s).min()


def test_invalid_arguments_are_rejected_on_the_host():
    """GB_ERR_INVALID_ARGUMENT before the call looks for a device."""
    from glim_b200 import capi, gpu

    L = capi.lib()
    dummy = C.c_void_p(1)  # never dereferenced: validation comes first
    res = capi.GncResult()
    for bad in ({"max_init_samples": 0}, {"max_init_samples": (1 << 28) + 1}, {"dof": 5}, {"dof": 3}):
        prm = gpu.gnc_params(**bad)
        assert L.gb_gnc_align(dummy, dummy, dummy, C.byref(prm), C.byref(res), None, None) == 1, bad
    assert L.gb_gnc_align(dummy, dummy, dummy, None, C.byref(res), None, None) == 1
    assert L.gb_gnc_align(dummy, dummy, dummy, C.byref(gpu.gnc_params()), None, None, None) == 1
    assert L.gb_gnc_align(None, None, None, C.byref(gpu.gnc_params()), C.byref(res), None, None) == 1
    prm = capi.GncParams()
    assert L.gb_gnc_default_params(C.byref(prm)) == 0
    assert (prm.max_init_samples, prm.dof, prm.seed) == (10000, 4, 53123)
