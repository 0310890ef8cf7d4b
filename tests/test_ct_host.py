"""CPU-only checks of the continuous-time GICP factor's arithmetic and of its restatement.

glim_b200/csrc/gb_ct_math.cuh holds the text the CT kernels compile for the device (time table, SE(3) Exp / Log / J_r / Ad, the
chain-rule blocks D0 / D1, the prior and between terms, the 12x12 Cholesky solve and the trial / accept step).  Here the SAME
text is compiled for the host with g++ (tests/cpp/ct_math_host.cpp) and checked against tests/ct_oracle.py; the oracle itself
is checked by finite differences, symmetry and the identities of the rule."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from glim_b200 import capi, synth
from oracle import oracle
from tests import ct_oracle as co
from tests import lm_oracle as lm
from tests import ivox_oracle as io
from tests import voxelmap_oracle as vo
from tests.util import cov_colmajor16

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIN_CB = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double))
ERR_CB = C.CFUNCTYPE(C.c_double, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double))


@pytest.fixture(scope="module")
def cm(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cm") / "libct_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so, os.path.join(ROOT, "tests", "cpp", "ct_math_host.cpp")])
    L = C.CDLL(so)
    vp, f64, i32 = C.c_void_p, C.c_double, C.c_int
    L.cm_time_table.argtypes = [vp, i32, vp, vp]
    L.cm_time_table.restype = i32
    L.cm_exp.argtypes = [vp, vp]
    L.cm_log.argtypes = [vp, vp]
    L.cm_jr.argtypes = [vp, i32, vp]
    L.cm_adjoint.argtypes = [vp, vp]
    L.cm_entry_pose.argtypes = [vp, vp, f64, vp]
    L.cm_entry_blocks.argtypes = [vp, vp, f64, vp, vp]
    L.cm_small_terms.argtypes = [vp, vp, vp, f64, f64, vp, vp]
    L.cm_small_terms.restype = f64
    L.cm_solve12.argtypes = [vp, vp, f64, vp]
    L.cm_solve12.restype = i32
    L.cm_align.argtypes = [vp, f64, f64, vp, vp, vp, LIN_CB, ERR_CB, vp, vp, vp]
    L.cm_align.restype = i32
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def cm16(T):
    """4x4 -> column-major 16"""
    return np.ascontiguousarray(np.asarray(T, dtype=np.float64).T).reshape(16)


def from16(a):
    return np.asarray(a).reshape(4, 4).T.copy()


def tangents():
    rng = synth.rng_for(4400)
    out = [np.zeros(6), np.array([1e-7, -2e-7, 3e-8, 0.1, -0.2, 0.05]), np.array([0.004, -0.003, 0.002, 1.0, 0.2, -0.1])]
    for s in (0.02, 0.3, 1.5):
        for _ in range(3):
            out.append(np.concatenate([rng.normal(0, s, 3), rng.normal(0, 2.0, 3)]))
    return out


def random_pose(rng, rot=0.4, trans=3.0):
    return co.se3_exp(np.concatenate([rng.normal(0, rot, 3), rng.normal(0, trans, 3)]))


# ---------------------------------------------------------------------------------------------------------------------
# the time table
# ---------------------------------------------------------------------------------------------------------------------
TIME_CASES = {
    "scan": np.sort(synth.rng_for(4401).uniform(0.0, 0.1, 5000)),
    "all_equal": np.full(300, 0.0425),
    "single": np.array([0.017]),
    "gaps": np.concatenate([np.linspace(0.0, 0.0004, 20), np.linspace(0.02, 0.021, 30), np.linspace(0.05, 0.0999, 400)]),
    "exact_eps": np.array([0.0, 0.001, 0.002, 0.0025, 0.0035, 0.0045, 0.0045, 0.006]),  # a gap of exactly time_eps opens no entry
}


@pytest.mark.parametrize("case", sorted(TIME_CASES))
def test_time_table_is_exact(cm, case):
    t = np.ascontiguousarray(TIME_CASES[case])
    n = len(t)
    starts, tau = np.zeros(n + 1, np.int32), np.zeros(n)
    B = cm.cm_time_table(_p(t), n, _p(starts), _p(tau))
    s_ref, tau_ref = co.time_table(t)
    assert B == len(tau_ref)
    assert np.array_equal(starts[:B + 1], s_ref)
    assert np.array_equal(tau[:B], tau_ref)
    if case == "all_equal" or case == "single":
        assert B == 1 and tau[0] == 0.0
    if case == "exact_eps":
        assert np.array_equal(s_ref, [0, 2, 4, 7, 8])  # 0.001 - 0 is not more than time_eps; 0.006 - 0.0045 is


# ---------------------------------------------------------------------------------------------------------------------
# SE(3)
# ---------------------------------------------------------------------------------------------------------------------
def test_se3_exp_log_jacobians_adjoint_match_the_oracle(cm):
    for xi in tangents():
        xi = np.ascontiguousarray(xi)
        T = np.zeros(16)
        cm.cm_exp(_p(xi), _p(T))
        assert np.abs(from16(T) - co.se3_exp(xi)).max() < 1e-12
        back = np.zeros(6)
        cm.cm_log(_p(T), _p(back))
        assert np.abs(back - co.se3_log(from16(T))).max() < 1e-12
        assert np.abs(back - xi).max() < 1e-10
        for inverse, ref in ((0, co.jr(xi)), (1, co.jr_inv(xi))):
            J = np.zeros(36)
            cm.cm_jr(_p(xi), inverse, _p(J))
            assert np.abs(J.reshape(6, 6) - ref).max() < 1e-12, (xi, inverse)
        A = np.zeros(36)
        cm.cm_adjoint(_p(T), _p(A))
        assert np.abs(A.reshape(6, 6) - co.adjoint(from16(T))).max() < 1e-12
    # near pi
    T = cm16(co.se3_exp(np.array([0.0, 3.1, 0.2, 1.0, 2.0, 3.0])))
    back = np.zeros(6)
    cm.cm_log(_p(T), _p(back))
    assert np.abs(back - co.se3_log(from16(T))).max() < 1e-9


def test_right_jacobian_is_the_derivative_of_exp():
    """the oracle's J_r: Exp(xi + d) = Exp(xi) Exp(J_r(xi) d) to first order"""
    for xi in tangents()[1:]:
        J = np.zeros((6, 6))
        h = 1e-6
        for k in range(6):
            d = np.zeros(6)
            d[k] = h
            J[:, k] = (co.se3_log(co.inv(co.se3_exp(xi)) @ co.se3_exp(xi + d)) - co.se3_log(co.inv(co.se3_exp(xi)) @ co.se3_exp(xi - d))) / (2 * h)
        assert np.abs(J - co.jr(xi)).max() < 1e-8


def fd_entry_blocks(X, Y, tau, h=1e-5):
    T = co.entry_pose(X, Y, tau)
    D0, D1 = np.zeros((6, 6)), np.zeros((6, 6))
    for k in range(6):
        d = np.zeros(6)
        d[k] = h
        for D, f in ((D0, lambda s: co.entry_pose(X @ co.se3_exp(s), Y, tau)), (D1, lambda s: co.entry_pose(X, Y @ co.se3_exp(s), tau))):
            D[:, k] = (co.se3_log(co.inv(T) @ f(d)) - co.se3_log(co.inv(T) @ f(-d))) / (2 * h)
    return D0, D1


def test_entry_blocks_match_finite_differences(cm):
    rng = synth.rng_for(4402)
    for k in range(6):
        X = random_pose(rng)
        Y = X @ co.se3_exp(np.concatenate([rng.normal(0, 0.05 * (k + 1), 3), rng.normal(0, 0.5 * (k + 1), 3)]))
        for tau in (0.0, 0.3, 0.77, 1.0):
            D0, D1 = np.zeros(36), np.zeros(36)
            cm.cm_entry_blocks(_p(cm16(X)), _p(cm16(Y)), tau, _p(D0), _p(D1))
            D0, D1 = D0.reshape(6, 6), D1.reshape(6, 6)
            R0, R1 = co.entry_blocks(X, Y, tau)
            assert np.abs(D0 - R0).max() < 1e-12 and np.abs(D1 - R1).max() < 1e-12
            F0, F1 = fd_entry_blocks(X, Y, tau)
            assert np.abs(D0 - F0).max() < 1e-9 and np.abs(D1 - F1).max() < 1e-9, (k, tau)
            T = np.zeros(16)
            cm.cm_entry_pose(_p(cm16(X)), _p(cm16(Y)), tau, _p(T))
            assert np.abs(from16(T) - co.entry_pose(X, Y, tau)).max() < 1e-12
            if tau == 0.0:
                assert np.array_equal(D0, np.eye(6)) and np.array_equal(D1, np.zeros((6, 6)))
                assert np.array_equal(from16(T), X)
            if tau == 1.0:
                assert np.abs(D0).max() < 1e-12 and np.abs(D1 - np.eye(6)).max() < 1e-12
                assert np.abs(from16(T) - Y).max() < 1e-12


def test_small_terms_match_oracle_and_finite_differences(cm):
    rng = synth.rng_for(4403)
    wl, wc = 1e-3, 1e3
    for _ in range(4):
        Xp = random_pose(rng)
        X = Xp @ co.se3_exp(rng.normal(0, 0.05, 6))
        Y = X @ co.se3_exp(rng.normal(0, 0.05, 6))
        H, b = np.zeros(144), np.zeros(12)
        e = cm.cm_small_terms(_p(cm16(X)), _p(cm16(Y)), _p(cm16(Xp)), wl, wc, _p(H), _p(b))
        e_ref, H_ref, b_ref = co.small_terms(X, Y, Xp, wl, wc)
        assert abs(e - e_ref) < 1e-12 * max(1.0, e_ref)
        assert np.abs(H.reshape(12, 12) - H_ref).max() < 1e-9 * max(1.0, np.abs(H_ref).max())
        assert np.abs(b - b_ref).max() < 1e-9 * max(1.0, np.abs(b_ref).max())
        # the gradient of e is 2 b
        h = 1e-6
        g = np.zeros(12)
        for k in range(12):
            d = np.zeros(12)
            d[k] = h
            ep = co.small_terms(X @ co.se3_exp(d[:6]), Y @ co.se3_exp(d[6:]), Xp, wl, wc)[0]
            em = co.small_terms(X @ co.se3_exp(-d[:6]), Y @ co.se3_exp(-d[6:]), Xp, wl, wc)[0]
            g[k] = (ep - em) / (2 * h)
        assert np.abs(g - 2 * b_ref).max() < 1e-6 * max(1.0, np.abs(b_ref).max())


def test_cholesky_12_matches_numpy(cm):
    rng = synth.rng_for(4404)
    for lam in (0.0, 1e-10, 1e-3, 10.0):
        A = rng.normal(size=(12, 12))
        H = A @ A.T + 1e-3 * np.eye(12)
        b = rng.normal(size=12)
        d = np.zeros(12)
        assert cm.cm_solve12(_p(np.ascontiguousarray(H)), _p(b), lam, _p(d)) == 1
        ref = np.linalg.solve(H + lam * np.eye(12), -b)
        assert np.abs(d - ref).max() < 1e-9 * np.abs(ref).max()
    H = -np.eye(12)
    assert cm.cm_solve12(_p(H), _p(np.zeros(12)), 0.0, _p(np.zeros(12))) == 0


def test_default_params_are_the_shipped_ct_values():
    p = capi.CtParams()
    assert capi.lib().gb_ct_default_params(C.byref(p)) == 0  # host only: no device needed
    for k, v in lm.CT_DEFAULTS.items():
        assert getattr(p.lm, k) == v, k
    assert (p.location_consistency_inf_scale, p.constant_velocity_inf_scale) == (co.W_PRIOR, co.W_BETWEEN)
    assert capi.lib().gb_ct_default_params(None) == 1


# ---------------------------------------------------------------------------------------------------------------------
# the factor's restatement on a small problem
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def problem():
    """an iVox of two arc frames, and a third frame with times, covariances and a motion (X at its start, Y at its end)"""
    frames = vo.arc_frames(4, 32 * 40)
    m = io.IVox(1.0, 0.1, 10, 7)
    for k in (0, 1):
        xyz, cov6 = oracle.pack_cloud(frames[k][0], cov_colmajor16(frames[k][1]))
        m.insert(xyz, cov6, frames[k][2])
    xyz, cov6 = oracle.pack_cloud(frames[2][0], cov_colmajor16(frames[2][1]))
    n = len(xyz)
    times = np.sort(synth.rng_for(4405).uniform(0.0, 0.1, n))
    starts, tau = co.time_table(np.repeat(np.round(times, 2), 1))  # ~10 entries
    X = frames[2][2] @ co.se3_exp(np.array([0.003, -0.002, 0.004, 0.05, -0.03, 0.02]))
    Y = X @ co.se3_exp(np.array([0.0, 0.0, 0.05, 0.8, 0.05, 0.0]))
    return m, xyz, cov6, starts, tau, X, Y, frames[2][2]


def test_oracle_gradient_is_half_the_derivative_of_the_error(problem):
    """finite differences of E with correspondences and M frozen at the linearization poses, in fp64 without the fp32 cast"""
    m, xyz, cov6, starts, tau, X, Y, _ = problem
    r, corr = co.linearize(m, xyz, cov6, starts, tau, X, Y, 2.0, cast=False)
    assert r["num_inliers"] > 100
    h = 1e-6
    g = np.zeros(12)
    for k in range(12):
        d = np.zeros(12)
        d[k] = h
        ep = co.error(m, xyz, cov6, starts, tau, X, Y, X @ co.se3_exp(d[:6]), Y @ co.se3_exp(d[6:]), 2.0, cast=False, freeze_M=True)
        em = co.error(m, xyz, cov6, starts, tau, X, Y, X @ co.se3_exp(-d[:6]), Y @ co.se3_exp(-d[6:]), 2.0, cast=False, freeze_M=True)
        g[k] = (ep - em) / (2 * h)
    assert np.linalg.norm(g - 2 * r["b"]) < 1e-5 * np.linalg.norm(r["b"])
    H = r["H"]
    assert np.abs(H - H.T).max() < 1e-9 * np.abs(H).max()
    assert np.linalg.eigvalsh(H).min() > -1e-9 * np.abs(H).max()


def test_oracle_with_one_entry_is_the_gicp_factor_at_X(problem):
    """all times equal: H_XX, b_X, error and inliers are ivox_oracle.linearize's at X; the Y blocks are zero"""
    m, xyz, cov6, _, _, X, Y, _ = problem
    starts, tau = co.time_table(np.zeros(len(xyz)))
    r, _ = co.linearize(m, xyz, cov6, starts, tau, X, Y, 2.0)
    g, _ = io.linearize(m, xyz, cov6, X, 2.0)
    assert r["num_inliers"] == g["num_inliers"]
    assert np.abs(r["H_tt"] - g["H_ss"]).max() < 1e-9 * np.abs(g["H_ss"]).max()
    assert np.abs(r["b_t"] - g["b_s"]).max() < 1e-9 * np.abs(g["b_s"]).max()
    assert abs(r["error"] - g["error"]) < 1e-12 * g["error"]
    assert not r["H_ss"].any() and not r["H_ts"].any() and not r["b_s"].any()


def test_host_round_structure_matches_the_oracle_lm(cm, problem):
    """gb_ct_gicp_align's round structure (gb_ct_math.cuh compiled for the host) on the oracle's factor equals the oracle's
    LM: same poses, iterations, trials and status"""
    m, xyz, cov6, starts, tau, X, Y, T_gt = problem
    Xp = X @ co.se3_exp(np.array([0.001, 0.0, -0.002, 0.1, 0.0, 0.05]))
    X0 = X @ co.se3_exp(np.array([0.0, 0.0, 0.01, 0.2, -0.1, 0.0]))
    Y0 = Y @ co.se3_exp(np.array([0.0, 0.01, 0.0, -0.1, 0.1, 0.05]))
    cache = {}

    def lin(Xc, Yc, sys):
        Xm, Ym = from16(np.ctypeslib.as_array(Xc, (16,))), from16(np.ctypeslib.as_array(Yc, (16,)))
        r, corr = co.linearize(m, xyz, cov6, starts, tau, Xm, Ym, 2.0)
        cache["corr"] = corr
        out = np.ctypeslib.as_array(sys, (158,))
        out[:144] = r["H"].reshape(144)
        out[144:156] = r["b"]
        out[156], out[157] = r["error"], r["num_inliers"]

    def err(Xl, Yl, Xe, Ye):
        Xm, Ym = from16(np.ctypeslib.as_array(Xe, (16,))), from16(np.ctypeslib.as_array(Ye, (16,)))
        return co.linearize(m, xyz, cov6, starts, tau, Xm, Ym, 2.0, corr=cache["corr"])[0]["error"]

    P = capi.CtParams()
    capi.lib().gb_ct_default_params(C.byref(P))
    Xo, Yo, st = np.zeros(16), np.zeros(16), np.zeros(5)
    lin_cb, err_cb = LIN_CB(lin), ERR_CB(err)
    status = cm.cm_align(C.byref(P.lm), co.W_PRIOR, co.W_BETWEEN, _p(cm16(X0)), _p(cm16(Y0)), _p(cm16(Xp)), lin_cb, err_cb, _p(Xo), _p(Yo), _p(st))
    ref = co.align(m, xyz, cov6, starts, tau, X0, Y0, Xp, 2.0)
    assert status == ref["status"]
    assert (int(st[3]), int(st[4])) == (ref["iterations"], ref["trials"])
    assert np.abs(from16(Xo) - ref["X"]).max() < 1e-9
    assert np.abs(from16(Yo) - ref["Y"]).max() < 1e-9
    assert abs(st[0] - ref["error"]) < 1e-9 * ref["error"]
