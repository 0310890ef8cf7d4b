"""CPU-only checks of gb_imu_preintegrate's and gb_nav_graph_optimize's arithmetic.

glim_b200/csrc/gb_imu_math.cuh (one preintegration step, the window, the IMU and vector terms) and the navigation part of
gb_pose_graph_math.cuh hold the text the device compiles.  Here the SAME text is compiled for the host with g++
(tests/cpp/imu_math_host.cpp), one thread and no barrier, and checked against central differences, numpy's restatement in
tests/imu_oracle.py and the rule's restatement in tests/nav_graph_oracle.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth
from tests import graph_oracle as go
from tests import imu_oracle as io
from tests import lm_oracle as lm
from tests import nav_graph_oracle as ngo
from tests import pose_graph_oracle as pgo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def im(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("im") / "libimu_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so,
                           os.path.join(ROOT, "tests", "cpp", "imu_math_host.cpp")])
    L = C.CDLL(so)
    vp, f64, i32 = C.c_void_p, C.c_double, C.c_int
    L.imh_step.argtypes = [vp, vp, vp, f64, vp, vp, vp, vp]
    L.imh_preintegrate.argtypes = [vp, i32, f64, f64, vp, vp, vp]
    L.imh_imu_residual.argtypes = [vp] * 8
    L.imh_vector_residual.argtypes = [vp] * 5
    L.imh_vector_residual.restype = i32
    L.imh_nav_assemble.argtypes = [i32, i32, i32, i32, vp, i32, vp, vp, vp, i32, vp, i32, vp, vp, vp, f64, vp, vp, vp, vp, vp, vp]
    L.imh_nav_optimize.argtypes = [vp, i32, i32, i32, i32, vp, i32, vp, vp, vp, i32, vp, i32, vp, vp, vp, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def imu_params(**kw):
    p = capi.ImuParams()
    P = dict(io.DEFAULT_PARAMS, **kw)
    p.acc_noise, p.gyro_noise, p.int_noise = P["acc_noise"], P["gyro_noise"], P["int_noise"]
    p.gravity[:] = list(P["gravity"])
    return p


def host_preintegrate(im, samples, start, end, bias, **kw):
    smp = np.ascontiguousarray(np.reshape(samples, (-1, 7)), dtype=np.float64)
    out = np.zeros(1, capi.PREINTEGRATED_DTYPE)
    im.imh_preintegrate(_p(smp), len(smp), float(start), float(end), _p(np.asarray(bias, dtype=np.float64)), C.byref(imu_params(**kw)), _p(out))
    return out[0]


def rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(b).max(), 1e-300)


def assert_record_close(got, ref, tol=1e-12):
    assert int(got["num_integrated"]) == ref["num_integrated"]
    assert abs(got["delta_t"] - ref["delta_t"]) <= 1e-15 * max(1.0, ref["delta_t"])
    for k in ("preintegrated", "H_bias_acc", "H_bias_omega", "covariance"):
        if np.abs(ref[k]).max() == 0.0:
            assert np.abs(got[k]).max() == 0.0, k
        else:
            assert rel(got[k], ref[k]) <= tol, (k, rel(got[k], ref[k]))
    assert np.array_equal(got["covariance"], np.asarray(got["covariance"]).T)  # exactly symmetric


def noisy_samples(rng, t0, t1, rate):
    ts = np.sort(rng.uniform(t0, t1, size=int((t1 - t0) * rate)))
    return np.column_stack([ts, rng.normal(size=(len(ts), 3)) * 2.0 + [0, 0, 9.81], rng.normal(size=(len(ts), 3)) * 0.5])


def test_window_matches_the_deque_restatement(im):
    """duplicate stamps, samples before start, an end past the last sample, an empty array and consecutive intervals: the
    host build, numpy's window and GLIM's deque-and-erase loop agree"""
    rng = np.random.default_rng(7)
    s = noisy_samples(rng, 0.0, 2.0, 200)
    s[10, 0] = s[9, 0]  # duplicate stamps
    s[11, 0] = s[9, 0]
    bias = np.array([0.05, -0.02, 0.1, 0.003, -0.002, 0.001])
    edges = [0.013, 0.31, 0.31, 0.7, 1.3, 1.97]  # consecutive, one of zero length; samples continue past the last end
    intervals = list(zip(edges[:-1], edges[1:]))
    deque = io.integrate_imu_deque(s, intervals, [bias] * len(intervals))
    for (a, b), ref in zip(intervals, deque):
        mine = io.preintegrate(s, a, b, bias)
        assert_record_close(host_preintegrate(im, s, a, b, bias), mine)
        for k in ("preintegrated", "covariance"):
            assert np.array_equal(mine[k], ref[k])
        assert mine["num_integrated"] == ref["num_integrated"] and mine["delta_t"] == ref["delta_t"]
    assert sum(r["num_integrated"] for r in deque) > 300
    # one interval ending past the last sample: the last sample runs the final step
    ref = io.integrate_imu_deque(s, [(1.5, 2.4)], [bias])[0]
    got = host_preintegrate(im, s, 1.5, 2.4, bias)
    assert_record_close(got, ref)
    assert abs(got["delta_t"] - 0.9) < 1e-12
    # samples only before start: one final step of end - start with the last sample
    got = host_preintegrate(im, s[:5], 1.0, 1.1, bias)
    assert got["num_integrated"] == 0 and abs(got["delta_t"] - 0.1) < 1e-15
    assert_record_close(got, io.integrate_imu_deque(s[:5], [(1.0, 1.1)], [bias])[0])
    # an empty array integrates nothing
    got = host_preintegrate(im, np.zeros((0, 7)), 0.0, 1.0, bias)
    assert got["delta_t"] == 0.0 and got["num_integrated"] == 0 and not np.any(got["covariance"])
    assert np.array_equal(got["bias_hat"], bias) and np.array_equal(got["gravity"], io.DEFAULT_PARAMS["gravity"])


@pytest.mark.parametrize("theta", [0.0, 1e-3, 0.05, 0.5, 2.5])
def test_step_jacobians_against_central_differences(im, theta):
    rng = np.random.default_rng(int(theta * 1000) + 1)
    ax = rng.normal(size=3)
    x = np.concatenate([theta * ax / np.linalg.norm(ax), rng.normal(size=6)])
    a, w, dt = rng.normal(size=3) * 3.0, rng.normal(size=3), 0.004

    def host(x, a, w):
        xn, A, B, Cm = np.zeros(9), np.zeros((9, 9)), np.zeros((9, 3)), np.zeros((9, 3))
        im.imh_step(_p(np.asarray(x, float)), _p(np.asarray(a, float)), _p(np.asarray(w, float)), dt, _p(xn), _p(A), _p(B), _p(Cm))
        return xn, A, B, Cm

    xn, A, B, Cm = host(x, a, w)
    ref = io.step(x, a, w, dt)
    for got, r in zip((xn, A, B, Cm), ref):
        assert np.abs(got - r).max() <= 1e-12 * max(1.0, np.abs(r).max())
    h = 1e-6
    An = np.stack([(host(x + h * u, a, w)[0] - host(x - h * u, a, w)[0]) / (2 * h) for u in np.eye(9)], axis=1)
    Bn = np.stack([(host(x, a + h * u, w)[0] - host(x, a - h * u, w)[0]) / (2 * h) for u in np.eye(3)], axis=1)
    Cn = np.stack([(host(x, a, w + h * u)[0] - host(x, a, w - h * u)[0]) / (2 * h) for u in np.eye(3)], axis=1)
    assert np.abs(An - A).max() <= 1e-8
    assert np.abs(Bn - B).max() <= 1e-8 and np.abs(Cn - Cm).max() <= 1e-8


def test_bias_jacobians_against_reintegration(im):
    """H_bias_acc / H_bias_omega against central differences of the whole window in the bias estimate"""
    T0 = 1.0
    bias = np.array([0.1, -0.05, 0.2, 0.01, -0.02, 0.015])
    s = io.samples(T0, T0 + 1.0, 200, bias)
    rec = host_preintegrate(im, s, T0, T0 + 0.9, bias)
    h = 1e-6
    Hn = np.stack([(host_preintegrate(im, s, T0, T0 + 0.9, bias + h * u)["preintegrated"] - host_preintegrate(im, s, T0, T0 + 0.9, bias - h * u)["preintegrated"]) / (2 * h)
                   for u in np.eye(6)], axis=1)
    assert np.abs(Hn[:, :3] - rec["H_bias_acc"]).max() <= 1e-6 * np.abs(rec["H_bias_acc"]).max()
    assert np.abs(Hn[:, 3:] - rec["H_bias_omega"]).max() <= 1e-6 * np.abs(rec["H_bias_omega"]).max()


def nav_state(rng):
    Ti, Tj = synth.perturb(np.eye(4), rng, 0.8, 3.0), synth.perturb(np.eye(4), rng, 0.8, 3.0)
    return Ti, rng.normal(size=3), Tj, rng.normal(size=3), rng.normal(size=6) * 0.1


def host_imu_residual(im, Ti, vi, Tj, vj, b, rec):
    r, J = np.zeros(9), np.zeros((9, 30))
    im.imh_imu_residual(_p(capi.pose16(Ti)), _p(np.asarray(vi, float)), _p(capi.pose16(Tj)), _p(np.asarray(vj, float)), _p(np.asarray(b, float)), _p(rec), _p(r), _p(J))
    return r, J


def a_record(im, seed=3):
    bias = np.array([0.02, 0.01, -0.03, 0.002, 0.001, -0.004])
    s = io.samples(0.0, 1.5, 400, bias * 2.0)
    return host_preintegrate(im, s, 0.1, 1.2, bias)


def test_imu_term_against_numpy_and_differences(im):
    rng = np.random.default_rng(11)
    rec = np.zeros(1, capi.PREINTEGRATED_DTYPE)
    rec[0] = a_record(im)
    recd = io.record_of(rec[0])
    for it in range(6):
        Ti, vi, Tj, vj, b = nav_state(rng)
        r, J = host_imu_residual(im, Ti, vi, Tj, vj, b, rec)
        rr, Jr = io.imu_residual(Ti, vi, Tj, vj, b, recd)
        assert rel(r, rr) <= 1e-12 and rel(J, Jr) <= 1e-12, it
        assert not J[:, 9:12].any() and not J[:, 21:24].any()  # the dead velocity dofs

        def res(d):
            return host_imu_residual(im, Ti @ synth.se3_exp(d[0:6]), vi + d[6:9], Tj @ synth.se3_exp(d[12:18]), vj + d[18:21], b + d[24:30], rec)[0]

        h = 1e-6
        Jn = np.stack([(res(h * u) - res(-h * u)) / (2 * h) for u in np.eye(30)], axis=1)
        assert np.abs(Jn - J).max() <= 1e-6 * max(1.0, np.abs(J).max()), it


@pytest.mark.parametrize("kind", range(5))
def test_vector_terms_against_numpy_and_differences(im, kind):
    rng = np.random.default_rng(20 + kind)
    z = rng.normal(size=6)
    term = gpu.vector_term_array([(list(capi.VECTOR_KINDS)[kind], 0, None if kind in (0, 1) else 1, z[:6 if kind in (1, 3) else 3], 3.0)],
                                 {0: 0}, {0: 0, 1: 1}, {0: 0, 1: 1})
    d = 6 if kind in (1, 3) else 3
    xa = synth.perturb(np.eye(4), rng, 0.5, 2.0) if kind == 4 else rng.normal(size=d)
    xb = rng.normal(size=3 if kind == 4 else d)

    def host(xa, xb):
        ca = np.zeros(16)
        ca[:16 if kind == 4 else d] = capi.pose16(xa) if kind == 4 else xa
        cb = np.zeros(16)
        cb[:len(xb)] = xb
        r, J = np.zeros(6), np.zeros((6, 12))
        m = im.imh_vector_residual(_p(term), _p(ca), _p(cb), _p(r), _p(J))
        return r[:m], J[:m]

    r, J = host(xa, xb)
    rr, Jr = io.vector_residual(kind, xa, xb, z)
    assert np.abs(r - rr).max() <= 1e-14 * max(1.0, np.abs(rr).max()) and np.abs(J - Jr).max() <= 1e-14 * max(1.0, np.abs(Jr).max())
    h = 1e-6

    def moved(u, s):
        ua, ub = u[:6], u[6:]
        a2 = xa @ synth.se3_exp(s * ua) if kind == 4 else xa + s * ua[:d]
        return host(a2, xb + s * ub[:len(xb)])[0]

    Jn = np.stack([(moved(u, h) - moved(u, -h)) / (2 * h) for u in np.eye(12)], axis=1)
    assert np.abs(Jn - J).max() <= 1e-7


def test_analytic_trajectory_prediction_and_residual(im):
    """exact 400 Hz samples of the analytic trajectory with known biases: the preintegrated prediction reaches the true end
    state to discretization error, and the residual at the true states is near zero"""
    bias = np.array([0.08, -0.05, 0.12, 0.01, -0.006, 0.004])
    t0, t1 = 2.0, 3.0
    s = io.samples(t0 - 0.1, t1 + 0.1, 400, bias)
    rec = np.zeros(1, capi.PREINTEGRATED_DTYPE)
    rec[0] = host_preintegrate(im, s, t0, t1, bias)
    assert rec[0]["num_integrated"] == 400 and abs(rec[0]["delta_t"] - 1.0) < 1e-9
    Ti, vi, _, _ = io.truth(t0)
    Tj, vj, _, _ = io.truth(t1)
    r, _ = host_imu_residual(im, Ti, vi, Tj, vj, bias, rec)
    assert np.linalg.norm(r[:3]) < 5e-3 and np.linalg.norm(r[3:6]) < 5e-3 and np.linalg.norm(r[6:]) < 1e-2, r
    # a wrong bias estimate corrected to first order through H_bias: the residual stays near zero
    rec2 = np.zeros(1, capi.PREINTEGRATED_DTYPE)
    rec2[0] = host_preintegrate(im, s, t0, t1, bias + np.array([0.01, -0.01, 0.01, 0.001, 0.001, -0.001]))
    r2, _ = host_imu_residual(im, Ti, vi, Tj, vj, bias, rec2)
    assert np.linalg.norm(r2 - r) < 2e-3
    # and a wrong end state is seen
    r3, _ = host_imu_residual(im, Ti, vi, Tj @ synth.pose(0.2, 0, 0, 0), vj, bias, rec)
    assert np.linalg.norm(r3[3:6]) > 0.15


def nav_problem(im, n=5, seed=1, drift=True):
    """a chain of n navigation states on the analytic trajectory: poses, velocities, biases; IMU terms between neighbours, a
    velocity between in place of one of them, rotate-velocity terms, bias priors and betweens, a pose prior; drifted starts"""
    rng = np.random.default_rng(seed)
    bias = np.array([0.03, -0.02, 0.05, 0.004, -0.003, 0.002])
    times = np.linspace(1.0, 1.0 + 0.5 * (n - 1), n)
    s = io.samples(times[0] - 0.05, times[-1] + 0.05, 300, bias)
    truth = [io.truth(t) for t in times]
    T = np.stack([x[0] for x in truth])
    V = np.stack([x[1] for x in truth])
    B = np.stack([bias] * n)
    imu, vec = [], []
    for k in range(n - 1):
        if k == 1:
            vec.append((io.VELOCITY_BETWEEN, k, k + 1, V[k + 1] - V[k], 1.0))
            continue
        r = np.zeros(1, capi.PREINTEGRATED_DTYPE)
        r[0] = host_preintegrate(im, s, times[k], times[k + 1], bias * 0.5)
        imu.append((k, k, k + 1, k + 1, k, r[0]))
        vec.append((io.BIAS_BETWEEN, k, k + 1, np.zeros(6), 1e6))
    vec.append((io.BIAS_PRIOR, 0, None, np.zeros(6), 1e3))
    vec.append((io.VELOCITY_PRIOR, 0, None, V[0], 1e3))
    for k in range(n):
        vec.append((io.ROTATE_VELOCITY, k, k, T[k][:3, :3].T @ V[k], 1.0))
    priors = [(0, T[0], 1e6)]
    betweens = [(k, k + 1, synth.inv_pose(T[k]) @ T[k + 1], 1e2, None) for k in range(n - 1)]
    X0 = (np.stack([T[0]] + [synth.perturb(T[k], rng, 0.01, 0.05) for k in range(1, n)]) if drift else T, V + (rng.normal(size=V.shape) * 0.05 if drift else 0),
          np.zeros((n, 6)))
    return ngo.Graph(n, n, n, priors, [(i, j, Z, w * np.eye(6), 0.0) for i, j, Z, w, _ in betweens], imu, vec), X0, (T, V, B), betweens


def host_arrays(g, X):
    T, V, B = X
    Xs = np.zeros((g.K, 16))
    Xs[:g.KX] = capi.pose16(T)
    Xs[g.KX:g.KX + g.KV, :3] = V
    Xs[g.KX + g.KV:, :6] = B
    it = np.zeros(len(g.imu), capi.IMU_TERM_DTYPE)
    for m, (xi, vi, xj, vj, bi, rec) in enumerate(g.imu):
        it[m]["pose_i"], it[m]["vel_i"], it[m]["pose_j"], it[m]["vel_j"], it[m]["bias_i"] = xi, vi, xj, vj, bi
        it[m]["pim"] = rec
    vt = np.zeros(len(g.vec), capi.VECTOR_TERM_DTYPE)
    for m, (kind, a, b, z, w) in enumerate(g.vec):
        vt[m]["kind"], vt[m]["key_a"], vt[m]["key_b"], vt[m]["precision"] = kind, a, -1 if b is None else b, w
        vt[m]["z"][:len(z)] = z
    sl = np.full((len(g.imu) + len(g.vec), 5), -1, np.int32)
    for m, s in enumerate(g.slots()):
        sl[m, :len(s)] = s
    bt = gpu.between_terms([(i, j, Z, L, k or None) for i, j, Z, L, k in g.betweens])
    pk = np.ascontiguousarray([k for k, _, _ in g.priors], dtype=np.int32)
    pz = np.ascontiguousarray([capi.pose16(Z) for _, Z, _ in g.priors]).reshape(-1, 16)
    pw = np.ascontiguousarray([w for _, _, w in g.priors], dtype=np.float64)
    return Xs, it, vt, sl, bt, pk, pz, pw


def oracle_graph(g):
    """the oracle's view of the graph: records as dicts"""
    return ngo.Graph(g.KX, g.KV, g.KB, g.priors, g.betweens, [t[:5] + (io.record_of(t[5]),) for t in g.imu], g.vec)


def test_assembly_matches_the_restatement_entry_for_entry(im):
    """every term kind: every entry of H and b the restatement's sum in the stated order over the host's own records, bit for
    bit; the records the restatement's terms; the pinned velocity dofs a unit diagonal with zero right-hand side"""
    g, X0, _, _ = nav_problem(im, 5)
    Xs, it, vt, sl, bt, pk, pz, pw = host_arrays(g, X0)
    n = 6 * g.K
    N = (n + 63) // 64 * 64
    H, b, nrec, A, x, e = np.zeros((n, n)), np.zeros(n), np.zeros((len(sl), 931)), np.zeros((N, N)), np.zeros(N), C.c_double()
    lam = 1e-3
    im.imh_nav_assemble(g.KX, g.KV, g.KB, len(bt), _p(bt), len(pk), _p(pk), _p(pz), _p(pw), len(it), _p(it), len(vt), _p(vt), _p(sl), _p(Xs), lam, _p(H), _p(b),
                        _p(nrec), _p(A), _p(x), C.byref(e))
    og = oracle_graph(g)
    brecs = [pgo.between_record(X0[0][i], X0[0][j], Z, L, k) for i, j, Z, L, k in g.betweens]
    qblocks = [go.prior_term(X0[0][k], Z, w)[1:] + (go.prior_term(X0[0][k], Z, w)[0],) for k, Z, w in g.priors]
    ref_terms = og.terms(X0)
    host_terms = []
    for (s, Hr, br, er), rec in zip(ref_terms, nrec):
        m = 6 * len(s)
        Hh, bh = rec[:900].reshape(30, 30)[:m, :m], rec[900:900 + m]
        assert np.abs(Hh - Hr).max() <= 1e-9 * np.abs(Hr).max() and np.abs(bh - br).max() <= 1e-9 * max(np.abs(br).max(), 1e-9)
        assert abs(rec[930] - er) <= 1e-9 * max(er, 1e-12)
        host_terms.append((s, Hh, bh, rec[930]))
    Hr, br, er = ngo.assemble(g.K, [], [], [(i, j) for i, j, _, _, _ in g.betweens], brecs, host_terms, list(pk), qblocks)
    assert np.abs(np.tril(H) - np.tril(Hr)).max() <= 1e-9 * np.abs(Hr).max()
    dead = ngo.pinned(g)
    live = [i for i in range(n) if i not in dead]
    assert not H[dead].any() and not H[:, dead].any() and not b[dead].any()
    assert np.all(np.diag(A)[dead] == 1.0) and not x[dead].any() and np.all(np.diag(A)[n:] == 1.0)
    assert np.array_equal(np.diag(A)[live], np.diag(H)[live] + lam)
    assert abs(e.value - er) <= 1e-9 * er
    # bit for bit: the host's sums are the restatement's sums in the same order, given the same records
    nav_only = ngo.Graph(g.KX, g.KV, g.KB, [], [], og.imu, og.vec)
    Xs2, it2, vt2, sl2, bt2, pk2, pz2, pw2 = host_arrays(ngo.Graph(g.KX, g.KV, g.KB, [], [], g.imu, g.vec), X0)
    H2, b2, nrec2 = np.zeros((n, n)), np.zeros(n), np.zeros((len(sl2), 931))
    im.imh_nav_assemble(g.KX, g.KV, g.KB, 0, None, 0, None, None, None, len(it2), _p(it2), len(vt2), _p(vt2), _p(sl2), _p(Xs2), lam, _p(H2), _p(b2), _p(nrec2),
                        _p(np.zeros((N, N))), _p(np.zeros(N)), C.byref(C.c_double()))
    terms2 = [(s, r[:900].reshape(30, 30)[:6 * len(s), :6 * len(s)], r[900:900 + 6 * len(s)], r[930]) for s, r in zip(nav_only.slots(), nrec2)]
    Hr2, br2, _ = ngo.assemble(g.K, [], [], [], [], terms2, [], [])
    assert np.array_equal(np.tril(H2), np.tril(Hr2)) and np.array_equal(b2, br2)


@pytest.mark.parametrize("case", ["chain", "no_drift", "nav_only"])
def test_host_state_machine_takes_the_restatements_decisions(im, case):
    g, X0, truth, _ = nav_problem(im, 5, seed=3, drift=case != "no_drift")
    if case == "nav_only":  # no between terms: the IMU, vector terms and the prior alone
        g = ngo.Graph(g.KX, g.KV, g.KB, g.priors, [], g.imu, g.vec)
    Xs, it, vt, sl, bt, pk, pz, pw = host_arrays(g, X0)
    prm = capi.AlignParams()
    for k, v in dict(lm.ALIGN_DEFAULTS, max_iterations=20).items():
        setattr(prm, k, v)
    r = capi.GraphResult()
    im.imh_nav_optimize(C.byref(prm), g.KX, g.KV, g.KB, len(bt), _p(bt), len(pk), _p(pk), _p(pz), _p(pw), len(it), _p(it), len(vt), _p(vt), _p(sl), _p(Xs), C.byref(r))
    ref = ngo.optimize(oracle_graph(g), X0, dict(max_iterations=20))
    assert (r.iterations, r.trials, r.status) == (ref["iterations"], ref["trials"], ref["status"])
    T = Xs[:g.KX].reshape(-1, 4, 4).transpose(0, 2, 1)
    # the host whitens by the covariance's Cholesky factor, the restatement multiplies by its inverse
    assert np.abs(T - ref["x"][0]).max() < 1e-6
    assert np.abs(Xs[g.KX:g.KX + g.KV, :3] - ref["x"][1]).max() < 1e-6
    assert np.abs(Xs[g.KX + g.KV:, :6] - ref["x"][2]).max() < 1e-6
    assert not Xs[g.KX:g.KX + g.KV, 3:].any()  # the pinned dofs never move
    assert abs(r.error - ref["error"]) <= 1e-9 * max(ref["error"], 1.0)
    if case != "no_drift":
        assert ref["iterations"] >= 2
    if case == "chain":
        assert np.abs(T[:, :3, 3] - truth[0][:, :3, 3]).max() < 0.05


def test_binding_layouts():
    """the record, term and parameter layouts the header states"""
    dt = capi.PREINTEGRATED_DTYPE
    assert dt.itemsize == 1240 and [dt.fields[k][1] for k in ("delta_t", "preintegrated", "H_bias_acc", "H_bias_omega", "covariance", "bias_hat", "gravity", "num_integrated")] == \
        [0, 8, 80, 296, 512, 1160, 1208, 1232]
    assert capi.IMU_TERM_DTYPE.itemsize == 1264 and capi.IMU_TERM_DTYPE.fields["pim"][1] == 24
    assert capi.VECTOR_TERM_DTYPE.itemsize == 72 and capi.VECTOR_TERM_DTYPE.fields["z"][1] == 16
    p = capi.ImuParams()
    assert capi.lib().gb_imu_default_params(C.byref(p)) == 0
    assert (p.acc_noise, p.gyro_noise, p.int_noise, list(p.gravity)) == (0.05, 0.02, 0.001, [0.0, 0.0, -9.81])
