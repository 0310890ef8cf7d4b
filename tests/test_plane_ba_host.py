"""CPU-only checks of the plane bundle adjustment (no GPU needed):
  * the per-point restatement of PlaneEVMFactor (tests/plane_ba_oracle.py) against central finite differences: the point
    gradient and Hessian of lambda_0, the pose gradient and the exact pose Hessian along X_k Exp(xi_k), and its gauge freedom;
  * the moment form of glim_b200/csrc/gb_plane_math.cuh, compiled for the host (tests/cpp/plane_math_host.cpp), against that
    restatement: K = 1 to 8 keys of unequal sizes, thin planes and poses 10 km from the origin;
  * the patch statistics of the host build against the oracle's;
  * the modal's auto-radius loop on each of its exits;
  * the arguments the patch calls reject before they touch a device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from glim_b200 import synth
from tests import plane_ba_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def hl(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("plane") / "libplane_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", out,
                           os.path.join(ROOT, "tests", "cpp", "plane_math_host.cpp")])
    L = C.CDLL(out)
    vp = C.c_void_p
    L.patch_stats.argtypes = [C.c_double, vp, vp, vp]
    L.plane_evm.argtypes = [C.c_int, vp, vp, vp, vp, vp, vp]
    L.plane_evm.restype = C.c_int
    return L


def p(a):
    return a.ctypes.data_as(C.c_void_p)


def lam0(pts):
    d = pts - pts.mean(0)
    return np.linalg.eigh(d.T @ d / len(pts))


def point_grad(pts):
    lam, U = lam0(pts)
    d = pts - pts.mean(0)
    return (2.0 / len(pts)) * (d @ U[:, 0])[:, None] * U[:, 0][None, :]


def point_hess(pts):
    """the issue's per-point Hessian of lambda_0: (3N, 3N)"""
    N = len(pts)
    lam, U = lam0(pts)
    d = pts - pts.mean(0)
    u0 = U[:, 0]
    H = np.kron((2.0 / N) * (np.eye(N) - 1.0 / N), np.outer(u0, u0))
    for m in (1, 2):
        w = (d @ u0)[:, None] * U[:, m][None, :] + (d @ U[:, m])[:, None] * u0[None, :]
        H += (2.0 / N**2) * np.outer(w.reshape(-1), w.reshape(-1)) / (lam[0] - lam[m])
    return H


def cloud(rng, n, thick, R=None):
    """a planar patch of n points, extent ~1 m, `thick` across, rotated by R (random if None)"""
    pts = np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-0.7, 0.7, n), rng.normal(0, thick, n)])
    return pts @ (synth.so3_exp(rng.normal(0, 1, 3)) if R is None else R).T


def rel(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


@pytest.mark.parametrize("seed", range(12))
def test_point_derivatives_match_finite_differences(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(4, 51))
    pts = cloud(rng, n, [0.3, 0.05, 1e-3][seed % 3])
    g = point_grad(pts).reshape(-1)
    H = point_hess(pts)
    h = 1e-5
    fd_g, fd_H = np.zeros_like(g), np.zeros_like(H)
    for i in range(3 * n):
        e = np.zeros(3 * n)
        e[i] = h
        plus, minus = pts + e.reshape(n, 3), pts - e.reshape(n, 3)
        fd_g[i] = (lam0(plus)[0][0] - lam0(minus)[0][0]) / (2 * h)
        fd_H[:, i] = (point_grad(plus).reshape(-1) - point_grad(minus).reshape(-1)) / (2 * h)
    assert rel(g, fd_g) < 1e-6
    assert rel(H, fd_H) < 1e-6


def scene(rng, K, n_range=(5, 40), thick=0.05, far=0.0):
    """K keys of local points (unequal sizes) seeing one plane patch, their poses, and the offset o"""
    base = np.array([far, -0.5 * far, 0.25 * far])
    R = synth.so3_exp(rng.normal(0, 1, 3))
    X, key_pts = [], []
    for k in range(K):
        n = int(rng.integers(*n_range))
        w = cloud(rng, n, thick, R) + base
        T = np.eye(4)
        T[:3, :3] = synth.so3_exp(rng.normal(0, 0.5, 3))
        T[:3, 3] = base + rng.normal(0, 3, 3)
        key_pts.append((w - T[:3, 3]) @ T[:3, :3])  # local = R^T (w - t)
        X.append(T)
    o = base + rng.normal(0, 0.1, 3)
    return key_pts, X, o


@pytest.mark.parametrize("seed", range(6))
def test_pose_derivatives_match_finite_differences(seed):
    rng = np.random.default_rng(100 + seed)
    K = 2 + seed % 3  # one key alone is a gauge freedom: its b and H vanish
    key_pts, X, o = scene(rng, K, thick=0.1)
    e, b, H, deg = po.linearize(key_pts, X, o)
    assert not deg
    assert abs(e - po.error(key_pts, X, o)) <= 1e-14 * abs(e) + 1e-18
    h = 1e-4
    n6 = 6 * K
    E = lambda xi: po.error(key_pts, po.perturbed(X, xi), o)
    hb = 1e-5
    fd_b = np.array([(E(hb * np.eye(n6)[i]) - E(-hb * np.eye(n6)[i])) / (4 * hb) for i in range(n6)])
    fd_H = np.zeros((n6, n6))
    for i in range(n6):
        for j in range(i, n6):
            ei, ej = h * np.eye(n6)[i], h * np.eye(n6)[j]
            fd_H[i, j] = fd_H[j, i] = (E(ei + ej) - E(ei - ej) - E(-ei + ej) + E(-ei - ej)) / (8 * h * h)
    assert rel(b, fd_b) < 1e-6
    assert np.max(np.abs(H - fd_H)) < 1e-6 * np.max(np.abs(H))


@pytest.mark.parametrize("seed", range(4))
def test_global_motion_is_a_gauge_freedom(seed):
    rng = np.random.default_rng(200 + seed)
    K = 2 + seed
    key_pts, X, o = scene(rng, K)
    e, b, H, _ = po.linearize(key_pts, X, o)
    for _ in range(6):
        zeta = rng.normal(0, 1, 6)
        v = np.concatenate([po.adjoint(synth.inv_pose(T)) @ zeta for T in X])
        scale = np.linalg.norm(v)
        assert abs(b @ v) < 1e-9 * np.max(np.abs(b)) * scale
        assert abs(v @ H @ v) < 1e-9 * np.max(np.abs(H)) * scale * scale


def host_evm(hl, key_pts, X, o):
    K = len(key_pts)
    mom = np.zeros((K, 10))
    for k, a in enumerate(key_pts):
        n, m, S = po.moments(a)
        mom[k, 0], mom[k, 1:4] = n, m
        mom[k, 4:] = [S[0, 0], S[0, 1], S[0, 2], S[1, 1], S[1, 2], S[2, 2]]
    Xc = np.ascontiguousarray(np.stack([np.asarray(T).T.reshape(16) for T in X]))
    H = np.zeros(36 * K * K)
    b = np.zeros(6 * K)
    e = C.c_double()
    deg = hl.plane_evm(K, p(mom), p(Xc), p(np.asarray(o, np.float64)), p(H), p(b), C.byref(e))
    return e.value, b, H.reshape(6 * K, 6 * K).T, bool(deg)


@pytest.mark.parametrize("case", [(K, thick, far) for K in (1, 2, 3, 5, 8) for thick, far in ((0.05, 0.0), (1e-3, 0.0), (0.05, 1e4), (1e-3, 1e4))])
def test_moment_form_matches_the_per_point_oracle(hl, case):
    K, thick, far = case
    rng = np.random.default_rng(hash(case) % 2**32)
    key_pts, X, o = scene(rng, K, n_range=(3, 300), thick=thick, far=far)
    e, b, H, deg = host_evm(hl, key_pts, X, o)
    re, rb, rH, rdeg = po.linearize(key_pts, X, o)
    lam = np.linalg.eigvalsh(np.cov(np.concatenate(po.points_world(key_pts, X, o)).T, bias=True))
    if thick == 1e-3:
        assert lam[0] / lam[2] < 1e-5
    assert not deg and not rdeg
    assert abs(e - re) <= 1e-10 * lam[2]
    scale = max(np.max(np.abs(rH)), lam[2])  # one key alone is a gauge freedom: its H is rounding noise about 0
    assert np.max(np.abs(H - rH)) <= 1e-10 * scale
    assert np.max(np.abs(b - rb)) <= 1e-10 * scale


def test_degenerate_factor_has_zero_hessian(hl):
    # points on a circle in a plane: lambda_0 = 0 < lambda_1 = lambda_2 (not degenerate); a line: lambda_0 = lambda_1 = 0
    t = np.linspace(0, 2 * np.pi, 12, endpoint=False)
    circle = np.column_stack([np.cos(t), np.sin(t), np.zeros_like(t)])
    line = np.column_stack([t, np.zeros_like(t), np.zeros_like(t)])
    e, b, H, deg = host_evm(hl, [circle], [np.eye(4)], np.zeros(3))
    assert not deg and np.all(np.isfinite(H))
    e, b, H, deg = host_evm(hl, [line], [np.eye(4)], np.zeros(3))
    assert deg and not H.any() and not b.any()


@pytest.mark.parametrize("seed", range(8))
def test_patch_statistics_match_the_oracle(hl, seed):
    rng = np.random.default_rng(300 + seed)
    q = cloud(rng, int(rng.integers(3, 2000)), [0.2, 1e-3][seed % 2]) * rng.uniform(0.2, 3)
    n, ev = po.stats(q)
    s = q.sum(0)
    S = q.T @ q
    got = np.zeros(3)
    hl.patch_stats(float(n), p(s), p(np.array([S[0, 0], S[0, 1], S[0, 2], S[1, 1], S[1, 2], S[2, 2]])), p(got))
    assert np.array_equal(got, ev)
    hl.patch_stats(0.0, p(s), p(s), p(got))
    assert np.all(np.isnan(got))


def scripted(seq):
    """stats_at returning (n, ev) by ratio from a table keyed by the rounded radius"""
    def at(r):
        n, ratio = seq(r)
        return n, np.array([ratio, 0.5, 1.0])
    return at


def test_auto_radius_loop_exits():
    p = po.params()
    # planar everywhere: grows until above max_radius (1.1^k > 5 never within 10 trials from 1.0: all 10 trials run)
    r, n, ev, trials = po.auto_radius_loop(scripted(lambda r: (100, 0.001)), p)
    assert len(trials) == 10 and r == trials[-1][0] and r > 1.0
    # planar, starting near max_radius: the next growth leaves [min_radius, max_radius]
    r, n, ev, trials = po.auto_radius_loop(scripted(lambda r: (100, 0.001)), po.params(radius=4.8))
    assert trials == [] and r == 4.8
    # never planar: shrinks until below min_radius
    r, n, ev, trials = po.auto_radius_loop(scripted(lambda r: (100, 0.5)), p)
    assert len(trials) == 10 and r == trials[-1][0] and r > p["min_radius"]
    r, n, ev, trials = po.auto_radius_loop(scripted(lambda r: (100, 0.5)), po.params(radius=0.11))
    assert trials == [] and r == 0.11
    # fewer than 10 points at the first trial: stop, keep the start
    r, n, ev, trials = po.auto_radius_loop(scripted(lambda r: (100 if r == 1.0 else 9, 0.5)), p)
    assert trials == [(0.8, 9)] and r == 1.0 and n == 100
    # grown past the start and no longer planar: stop, keep the last planar radius
    r, n, ev, trials = po.auto_radius_loop(scripted(lambda r: (100, 0.001 if r < 1.25 else 0.5)), p)
    assert [t for t, _ in trials] == [1.1, 1.1 * 1.1, 1.1 * 1.1 * 1.1] and r == 1.1 * 1.1
    # a NaN ratio (no points) grows; the trial then has fewer than 10 points
    r, n, ev, trials = po.auto_radius_loop(lambda r: (0, np.full(3, np.nan)), p)
    assert trials == [(1.1, 0)] and r == 1.0 and n == 0


def test_rejected_arguments_need_no_device():
    from glim_b200 import capi

    L = capi.lib()
    prm = capi.PlanePatchParams()
    assert L.gb_plane_patch_default_params(C.byref(prm)) == 0
    assert (prm.radius, prm.max_frame_distance, prm.min_radius, prm.max_radius, prm.plane_eps) == (1.0, 25.0, 0.1, 5.0, 0.01)
    r = capi.PlanePatchResult()
    assert L.gb_plane_patch(None, 0, None, None, C.byref(prm), C.byref(r), None) == 1
    assert L.gb_plane_auto_radius(None, 0, None, None, C.byref(prm), C.byref(r)) == 1
    h = C.c_void_p()
    assert L.gb_plane_evm_factor_create(None, 0, None, None, C.byref(prm), C.byref(h)) == 1 and not h.value
    assert L.gb_plane_evm_factor_info(None, None, None, None, None) == 1
    e = np.zeros(1)
    assert L.gb_plane_evm_error(None, 0, None, None, p(e)) == 1
