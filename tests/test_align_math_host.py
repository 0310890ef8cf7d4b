"""CPU-only checks of gb_vgicp_align's arithmetic and rule.

glim_b200/csrc/gb_align_math.cuh holds the text k_align_step / k_align_accept compile for the device (record sum, 6x6 Cholesky
solve, Exp, compose, step norms, the accept / terminate rule).  Here the SAME text is compiled for the host with g++
(tests/cpp/align_math_host.cpp) and checked against numpy, synth.se3_exp and the rule's independent restatement
in tests/lm_oracle.py (on the CPU oracle, through tests/align_oracle.py) -- so a change to the rule or its arithmetic is caught on the CPU-only box before the GPU tests run.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from glim_b200 import capi, synth
from oracle import oracle
from tests import align_oracle
from tests import lm_oracle as lm
from tests.util import cov_colmajor16, scan_pair

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIN_CB = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.POINTER(C.c_double))
ERR_CB = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double))
ACTIVE = -1


@pytest.fixture(scope="module")
def am(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("am") / "libalign_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so, os.path.join(ROOT, "tests", "cpp", "align_math_host.cpp")])
    L = C.CDLL(so)
    vp, f64, i32 = C.c_void_p, C.c_double, C.c_int
    L.am_solve.argtypes = [vp, vp, f64, vp]
    L.am_exp.argtypes = [vp, vp]
    L.am_compose.argtypes = [vp, vp, vp]
    L.am_step_norms.argtypes = [vp, vp, vp]
    L.am_conclude.argtypes = [vp, i32, f64, f64, f64, f64, i32, f64, vp, vp, vp]
    L.am_align.argtypes = [vp, i32, vp, LIN_CB, ERR_CB, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def params(**kw):
    p = capi.AlignParams()
    for k, v in dict(lm.ALIGN_DEFAULTS, **kw).items():
        setattr(p, k, v)
    return p


def test_default_params_are_the_odometry_cpu_values():
    p = capi.AlignParams()
    assert capi.lib().gb_align_default_params(C.byref(p)) == 0  # host only: no device needed
    for k, v in lm.ALIGN_DEFAULTS.items():
        assert getattr(p, k) == v, k
    assert capi.lib().gb_align_default_params(None) == 1


def test_cholesky_solve_matches_numpy(am):
    rng = np.random.default_rng(7)
    for it in range(200):
        A = rng.normal(size=(6, 6)) * rng.uniform(0.1, 1e3, size=6)  # badly scaled columns, like rotation vs translation
        H = A @ A.T
        b = rng.normal(size=6) * 10.0 ** rng.uniform(-3, 3)
        lam = 10.0 ** rng.uniform(-8, 2)
        d = np.zeros(6)
        assert am.am_solve(_p(np.ascontiguousarray(H).ravel()), _p(b), lam, _p(d)) == 1
        ref = np.linalg.solve(H + lam * np.eye(6), -b)
        assert np.linalg.norm(d - ref) <= 1e-14 * np.linalg.cond(H + lam * np.eye(6)) * np.linalg.norm(ref)
    # not positive definite (lambda = 0 on a rank-deficient H, or an indefinite H), or NaN: the trial is rejected
    v = rng.normal(size=(6, 1))
    for H, lam in ((v @ v.T, 0.0), (-np.eye(6), 1e-5), (np.full((6, 6), np.nan), 1.0)):
        assert am.am_solve(_p(np.ascontiguousarray(H).ravel()), _p(np.ones(6)), lam, _p(np.zeros(6))) == 0


def test_exp_compose_and_step_norms_match_synth(am):
    rng = np.random.default_rng(8)
    xis = [rng.normal(size=6) * s for s in (1.0, 0.1, 1e-3, 1e-6)] + [np.array([0, 0, 0, 0.1, -0.2, 0.3]), np.array([1e-11, -2e-11, 0, 1e-3, 0, 0]), np.zeros(6)]
    for xi in xis:
        E = np.zeros(16)
        am.am_exp(_p(np.ascontiguousarray(xi)), _p(E))
        ref = synth.se3_exp(xi)
        assert np.abs(E.reshape(4, 4).T - ref).max() < 1e-14
        dt, dr = C.c_double(), C.c_double()
        am.am_step_norms(_p(np.ascontiguousarray(xi)), C.byref(dt), C.byref(dr))
        assert abs(dt.value - np.linalg.norm(ref[:3, 3])) < 1e-14 and abs(dr.value - np.linalg.norm(xi[:3])) < 1e-15
    A, B = synth.perturb(np.eye(4), rng, 1.0, 5.0), synth.perturb(np.eye(4), rng, 1.0, 5.0)
    Cm = np.zeros(16)
    am.am_compose(_p(oracle.pose_colmajor(A)), _p(oracle.pose_colmajor(B)), _p(Cm))
    assert np.abs(Cm.reshape(4, 4).T - A @ B).max() < 1e-13


# (name, params, solved, e, e_new, dt, dr, iterations, lambda) -> (status, need_lin, lambda after, e after)
TOL_R = 1e-3 * np.pi / 180.0
DECISIONS = [
    ("accept, keep going", {}, 1, 100.0, 50.0, 0.1, 0.01, 1, 1e-5, ACTIVE, 1, 1e-6, 50.0),
    ("accept, small step converges", {}, 1, 100.0, 50.0, 5e-4, 0.5 * TOL_R, 1, 1e-5, lm.ALIGN_CONVERGED, 1, 1e-6, 50.0),
    ("accept, small translation but large rotation", {}, 1, 100.0, 50.0, 5e-4, 2 * TOL_R, 1, 1e-5, ACTIVE, 1, 1e-6, 50.0),
    ("accept, step under 1e-10 does not count", {}, 1, 100.0, 50.0, 1e-11, 1e-11, 1, 1e-5, ACTIVE, 1, 1e-6, 50.0),
    ("accept, only the translation under 1e-10 still counts", {}, 1, 100.0, 50.0, 1e-11, 0.5 * TOL_R, 1, 1e-5, lm.ALIGN_CONVERGED, 1, 1e-6, 50.0),
    ("accept, step test off", dict(step_translation_tol=0.0, step_rotation_tol=0.0), 1, 100.0, 50.0, 5e-4, 0.5 * TOL_R, 1, 1e-5, ACTIVE, 1, 1e-6, 50.0),
    ("accept, absolute decrease", {}, 1, 100.0, 99.95, 0.1, 0.01, 1, 1e-5, lm.ALIGN_CONVERGED, 1, 1e-6, 99.95),
    ("accept, absolute decrease at the bound", dict(absolute_error_tol=0.5), 1, 100.0, 99.5, 0.1, 0.01, 1, 1e-5, lm.ALIGN_CONVERGED, 1, 1e-6, 99.5),
    ("accept, relative decrease", dict(absolute_error_tol=0.0), 1, 1e9, 1e9 - 1e3, 0.1, 0.01, 1, 1e-5, lm.ALIGN_CONVERGED, 1, 1e-6, 1e9 - 1e3),
    ("accept, last iteration", dict(max_iterations=3), 1, 100.0, 50.0, 0.1, 0.01, 3, 1e-5, lm.ALIGN_MAX_ITERATIONS, 1, 1e-6, 50.0),
    ("accept, convergence wins over the last iteration", dict(max_iterations=3), 1, 100.0, 99.99, 0.1, 0.01, 3, 1e-5, lm.ALIGN_CONVERGED, 1, 1e-6, 99.99),
    ("reject, equal error", {}, 1, 100.0, 100.0, 0.1, 0.01, 1, 1e-5, ACTIVE, 0, 1e-4, 100.0),
    ("reject, larger error", {}, 1, 100.0, 200.0, 0.1, 0.01, 5, 1e-5, ACTIVE, 0, 1e-4, 100.0),
    ("reject, failed factorization", {}, 0, 100.0, 0.0, 0.0, 0.0, 1, 1e-5, ACTIVE, 0, 1e-4, 100.0),
    ("reject at the lambda bound", {}, 1, 100.0, 200.0, 0.1, 0.01, 1, 1e4, ACTIVE, 0, 1e5, 100.0),
    ("reject over the lambda bound", {}, 1, 100.0, 200.0, 0.1, 0.01, 1, 1e5, lm.ALIGN_LAMBDA_EXCEEDED, 0, 1e6, 100.0),
]


@pytest.mark.parametrize("case", DECISIONS, ids=[c[0] for c in DECISIONS])
def test_decision_table(am, case):
    _, kw, solved, e, e_new, dt, dr, iters, lam, status, need_lin, lam_after, e_after = case
    p = params(**kw)
    lo, nl, eo = C.c_double(), C.c_int(), C.c_double()
    got = am.am_conclude(C.byref(p), solved, e, e_new, dt, dr, iters, lam, C.byref(lo), C.byref(nl), C.byref(eo))
    assert (got, nl.value, eo.value) == (status, need_lin, e_after)
    assert abs(lo.value - lam_after) <= 1e-12 * lam_after


@pytest.fixture(scope="module")
def problem():
    pair = scan_pair(n_rays=32 * 200)
    xyz0, cov0 = oracle.pack_cloud(pair["points"][0], cov_colmajor16(pair["covs"][0]))
    xyz1, cov1 = oracle.pack_cloud(pair["points"][1], cov_colmajor16(pair["covs"][1]))
    maps = [oracle.GpuMap(xyz0, cov0, r) for r in (0.5, 1.0)]
    T_gt = synth.inv_pose(pair["poses"][0]) @ pair["poses"][1]
    return pair, xyz1, cov1, maps, T_gt


def pose_error(T, T_gt):
    d = synth.inv_pose(T_gt) @ T
    return float(np.linalg.norm(d[:3, 3])), float(np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1)))


def host_align(am, maps, xyz, cov6, T0, normals=None, **kw):
    """the host-compiled state machine, every linearization and error from the oracle"""
    F = len(maps)

    def lin(T, out):
        Tm = np.ctypeslib.as_array(T, shape=(16,)).reshape(4, 4).T
        o = np.ctypeslib.as_array(out, shape=(F * 122,))
        for f, m in enumerate(maps):
            o[f * 122:(f + 1) * 122] = oracle.linearize_gpumap(m, xyz, cov6, Tm, normals=normals)[0]

    def err(Tl, Te, out):
        Tl = np.ctypeslib.as_array(Tl, shape=(16,)).reshape(4, 4).T
        Te = np.ctypeslib.as_array(Te, shape=(16,)).reshape(4, 4).T
        o = np.ctypeslib.as_array(out, shape=(F * 122,))
        for f, m in enumerate(maps):
            keep = oracle.linearize_gpumap(m, xyz, cov6, Tl, with_derivs=False, normals=normals)[1] != -2
            o[f * 122 + 120] = oracle.error_gpumap(m, xyz[keep], cov6[keep], Tl, Te)

    p = params(**kw)
    r = capi.AlignResult()
    lin_cb, err_cb = LIN_CB(lin), ERR_CB(err)
    am.am_align(C.byref(p), F, _p(oracle.pose_colmajor(T0)), lin_cb, err_cb, C.byref(r))
    return dict(T=np.array(r.T_target_source[:]).reshape(4, 4).T, error=r.error, num_inliers=r.num_inliers, iterations=r.iterations, trials=r.trials, status=r.status)


def test_oracle_registers_the_scan_pair(problem):
    """Both voxel levels, starts perturbed by 0.25 m / 0.02 rad.  Every run reaches the ground-truth bar within 8
    linearizations.  It then stops either CONVERGED or, after its last accepted step, LAMBDA_EXCEEDED: the VGICP linearization
    ignores how the fused covariance R C R^T turns with the pose, so at the point where b = 0 no damped step lowers the
    error any more (GTSAM's LM gives up the same way)."""
    _, xyz1, cov1, maps, T_gt = problem
    statuses = []
    for seed in range(40, 46):
        T0 = synth.perturb(T_gt, synth.rng_for(seed), 0.02, 0.25)
        r = align_oracle.align_gpumap(maps, xyz1, cov1, T0)
        et, er = pose_error(r["T"], T_gt)
        assert r["iterations"] <= 8 and et < 0.03 and er < 2e-3, (seed, et, er, r)
        assert r["status"] in (lm.ALIGN_CONVERGED, lm.ALIGN_LAMBDA_EXCEEDED), r
        statuses.append(r["status"])
    assert statuses.count(lm.ALIGN_CONVERGED) >= 3, statuses


@pytest.mark.parametrize("case", ["default", "one_iteration", "one_level", "surface_validation", "no_step_test", "degenerate", "lambda_bound"])
def test_host_state_machine_takes_the_oracles_decisions(am, problem, case):
    pair, xyz1, cov1, maps, T_gt = problem
    T0 = synth.perturb(T_gt, synth.rng_for(43), 0.02, 0.25)
    kw, normals, ms = {}, None, maps
    if case == "one_iteration":
        kw = dict(max_iterations=1)
    elif case == "one_level":
        ms = maps[:1]
    elif case == "surface_validation":
        normals = pair["normals"][1]
    elif case == "no_step_test":
        kw = dict(max_iterations=10, step_translation_tol=0.0, step_rotation_tol=0.0, absolute_error_tol=0.0)
    elif case == "degenerate":
        T0 = T_gt.copy()
        T0[:3, 3] += 1000.0
    elif case == "lambda_bound":
        kw = dict(lambda_initial=1e3, lambda_upper_bound=1e4)  # large damping: the first trials are too short to decrease e
    ref = align_oracle.align_gpumap(ms, xyz1, cov1, T0, params=kw, normals=normals)
    got = host_align(am, ms, xyz1, cov1, T0, normals=normals, **kw)
    assert (got["iterations"], got["trials"], got["status"]) == (ref["iterations"], ref["trials"], ref["status"]), (got, ref)
    assert np.abs(got["T"] - ref["T"]).max() < 1e-9
    assert got["num_inliers"] == ref["num_inliers"]
    assert abs(got["error"] - ref["error"]) <= 1e-9 * max(ref["error"], 1.0)
    if case == "degenerate":
        assert ref["status"] == lm.ALIGN_DEGENERATE and np.array_equal(got["T"], T0) and got["trials"] == 0
    if case == "one_iteration":
        assert ref["iterations"] == 1
