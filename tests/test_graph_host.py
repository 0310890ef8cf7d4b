"""CPU-only checks of gb_graph_optimize's arithmetic and rule.

glim_b200/csrc/gb_graph_math.cuh holds the text k_graph_step / k_graph_accept compile for the device (assembly of the 6K x 6K
system from the records, the priors, the packed Cholesky solve, the retraction of every key, the round's two halves).  Here the
SAME text is compiled for the host with g++ (tests/cpp/graph_math_host.cpp), one thread and no barrier, and checked against
numpy and the rule's restatement in tests/graph_oracle.py on the CPU oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from glim_b200 import capi, synth
from oracle import oracle
from tests import graph_oracle as go
from tests import lm_oracle as lm
from tests import voxelmap_oracle as vo
from tests.util import cov_colmajor16

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIN_CB = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.POINTER(C.c_double))
ERR_CB = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double))


@pytest.fixture(scope="module")
def gm(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("gm") / "libgraph_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so, os.path.join(ROOT, "tests", "cpp", "graph_math_host.cpp")])
    L = C.CDLL(so)
    vp, f64, i32 = C.c_void_p, C.c_double, C.c_int
    L.gm_solve.argtypes = [i32, vp, vp, f64, vp]
    L.gm_assemble.argtypes = [i32, i32, vp, vp, vp, vp]
    L.gm_prior.argtypes = [vp, vp, f64, vp, vp]
    L.gm_prior.restype = f64
    L.gm_optimize.argtypes = [vp, i32, i32, vp, i32, vp, vp, vp, vp, LIN_CB, ERR_CB, vp, vp, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def params(**kw):
    p = capi.AlignParams()
    for k, v in dict(lm.ALIGN_DEFAULTS, **kw).items():
        setattr(p, k, v)
    return p


@pytest.mark.parametrize("n", [12, 18, 60, 96, 192])
def test_packed_cholesky_solve_matches_numpy(gm, n):
    rng = np.random.default_rng(n)
    for _ in range(5):
        A = rng.normal(size=(n, n)) * rng.uniform(0.1, 1e2, size=n)
        H = A @ A.T
        b = rng.normal(size=n) * 10.0 ** rng.uniform(-3, 3)
        lam = 10.0 ** rng.uniform(-8, 2)
        d = np.zeros(n)
        assert gm.gm_solve(n, _p(np.ascontiguousarray(H)), _p(b), lam, _p(d)) == 1
        M = H + lam * np.eye(n)
        ref = np.linalg.solve(M, -b)
        assert np.linalg.norm(d - ref) <= 1e-13 * np.linalg.cond(M) * np.linalg.norm(ref)
    # only the lower triangle is read
    d2 = np.zeros(n)
    assert gm.gm_solve(n, _p(np.ascontiguousarray(np.tril(H))), _p(b), lam, _p(d2)) == 1 and np.array_equal(d, d2)
    v = rng.normal(size=(n, 1))
    for H, lam in ((v @ v.T, 0.0), (-np.eye(n), 1e-5), (np.full((n, n), np.nan), 1.0)):
        assert gm.gm_solve(n, _p(np.ascontiguousarray(H)), _p(np.ones(n)), lam, _p(np.zeros(n))) == 0


def random_record(rng):
    A = rng.normal(size=(12, 12))
    S = A @ A.T
    raw = np.zeros(122)
    raw[0:36] = S[:6, :6].T.ravel()
    raw[36:72] = S[6:, 6:].T.ravel()
    raw[72:108] = S[:6, 6:].T.ravel()
    raw[108:120] = rng.normal(size=12)
    raw[120] = rng.uniform(1, 100)
    raw[121] = float(rng.integers(0, 1000))
    return raw


@pytest.mark.parametrize("seed", range(6))
def test_assembly_matches_the_restatement_entry_for_entry(gm, seed):
    """random topologies, the last key touched by no factor, one pair carrying two factors (and both orders of a pair)"""
    rng = np.random.default_rng(100 + seed)
    K = int(rng.integers(3, 33))
    keys = [(0, 1), (0, 1), (1, 0)]
    for _ in range(int(rng.integers(1, 40))):
        t, s = rng.choice(K - 1, 2, replace=False)
        keys.append((int(t), int(s)))
    raws = np.stack([random_record(rng) for _ in keys])
    n = 6 * K
    H, b = np.zeros((n, n)), np.zeros(n)
    gm.gm_assemble(K, len(keys), _p(np.ascontiguousarray(keys, dtype=np.int32)), _p(raws), _p(H), _p(b))
    Hr, br, _, _ = go.assemble(K, keys, [oracle.split122(r) for r in raws])
    assert np.array_equal(np.tril(H), np.tril(Hr))  # the same sums in the same order
    assert np.array_equal(b, br)
    assert not H[-6:].any() and not b[-6:].any()


def test_prior_term_against_central_differences(gm):
    rng = np.random.default_rng(7)
    for it in range(20):
        Z = synth.perturb(np.eye(4), rng, 1.0, 5.0)
        T = synth.perturb(Z, rng, 0.3 if it % 2 else 1e-3, 0.5)
        w = 10.0 ** rng.uniform(-3, 8)
        H, b = np.zeros(36), np.zeros(6)
        e = gm.gm_prior(_p(oracle.pose_colmajor(T)), _p(oracle.pose_colmajor(Z)), w, _p(H), _p(b))
        H = H.reshape(6, 6)
        ep, Hp, bp = go.prior_term(T, Z, w)
        assert abs(e - ep) <= 1e-12 * max(ep, 1e-300)

        def res(xi):
            return go.se3_log(synth.inv_pose(Z) @ T @ synth.se3_exp(xi))

        h = 1e-6
        J = np.stack([(res(h * u) - res(-h * u)) / (2 * h) for u in np.eye(6)], axis=1)
        r = res(np.zeros(6))
        grad = np.array([(w * res(h * u) @ res(h * u) - w * res(-h * u) @ res(-h * u)) / (2 * h) for u in np.eye(6)])
        assert np.abs(b - 0.5 * grad).max() <= 1e-6 * max(np.abs(grad).max(), w * 1e-9)
        assert np.abs(b - w * J.T @ r).max() <= 1e-6 * w * max(np.abs(r).max(), 1e-9)
        assert np.abs(H - w * J.T @ J).max() <= 1e-6 * w * np.abs(J.T @ J).max()
        assert np.abs(H - Hp).max() <= 1e-9 * np.abs(Hp).max() and np.abs(b - bp).max() <= 1e-9 * max(np.abs(bp).max(), 1e-300)


def test_largest_step_over_keys(gm):
    """one trial on a fixed quadratic system: the step tests read the largest translation and rotation steps of any key"""
    rng = np.random.default_rng(9)
    K = 4
    keys = [(0, 1), (1, 2), (2, 3), (0, 3)]
    raws = np.stack([random_record(rng) for _ in keys])
    raws[:, 121] = 10.0
    Ts = np.stack([oracle.pose_colmajor(synth.perturb(np.eye(4), rng, 0.5, 5.0)) for _ in range(K)])

    def lin(rows, out):
        np.ctypeslib.as_array(out, shape=(len(keys) * 122,))[:] = raws.ravel()

    def err(rl, re, out):
        o = np.ctypeslib.as_array(out, shape=(len(keys) * 122,))
        o[120::122] = 0.0

    r, dt, dr = capi.GraphResult(), C.c_double(), C.c_double()
    lcb, ecb = LIN_CB(lin), ERR_CB(err)
    kz = np.ascontiguousarray(keys, dtype=np.int32)
    gm.gm_optimize(C.byref(params(max_iterations=1)), K, len(keys), _p(kz), 0, None, None, None, _p(Ts), lcb, ecb, C.byref(r), C.byref(dt), C.byref(dr))
    H, b, _, _ = go.assemble(K, keys, [oracle.split122(x) for x in raws])
    d = np.linalg.solve(H + 1e-5 * np.eye(6 * K), -b)
    steps = [synth.se3_exp(d[6 * k:6 * k + 6]) for k in range(K)]
    assert (r.iterations, r.trials, r.status) == (1, 1, lm.ALIGN_MAX_ITERATIONS)
    assert abs(dt.value - max(np.linalg.norm(E[:3, 3]) for E in steps)) <= 1e-9 * dt.value
    assert abs(dr.value - max(np.linalg.norm(d[6 * k:6 * k + 3]) for k in range(K))) <= 1e-9 * dr.value


@pytest.fixture(scope="module")
def keyframes():
    """three hdl32 keyframes 1 m apart, maps of the first two at 0.5 / 1.0 m"""
    fr = vo.arc_frames(3, 32 * 150)
    packed = [oracle.pack_cloud(p, cov_colmajor16(c)) for p, c, _ in fr]
    maps = {(k, r): oracle.GpuMap(*packed[k], r) for k in (0, 1) for r in (0.5, 1.0)}
    return fr, packed, maps


def host_optimize(gm, fac, keys, T0, priors, **kw):
    """the host-compiled state machine, every linearization and error from the oracle; fac[f] = (map, source xyz, cov6)"""
    F, K = len(fac), len(T0)

    def lin(rows, out):
        R = np.ctypeslib.as_array(rows, shape=(F * 16,)).reshape(F, 4, 4).transpose(0, 2, 1)
        o = np.ctypeslib.as_array(out, shape=(F * 122,))
        for f, (m, xyz, cov6) in enumerate(fac):
            o[f * 122:(f + 1) * 122] = oracle.linearize_gpumap(m, xyz, cov6, R[f])[0]

    def err(rl, re, out):
        Rl = np.ctypeslib.as_array(rl, shape=(F * 16,)).reshape(F, 4, 4).transpose(0, 2, 1)
        Re = np.ctypeslib.as_array(re, shape=(F * 16,)).reshape(F, 4, 4).transpose(0, 2, 1)
        o = np.ctypeslib.as_array(out, shape=(F * 122,))
        for f, (m, xyz, cov6) in enumerate(fac):
            o[f * 122 + 120] = oracle.error_gpumap(m, xyz, cov6, Rl[f], Re[f])

    T = np.ascontiguousarray(np.stack([oracle.pose_colmajor(x) for x in T0]))
    pk = np.ascontiguousarray([k for k, _, _ in priors], dtype=np.int32)
    pz = np.ascontiguousarray([oracle.pose_colmajor(Z) for _, Z, _ in priors]).reshape(-1, 16)
    pw = np.ascontiguousarray([w for _, _, w in priors], dtype=np.float64)
    r, dt, dr = capi.GraphResult(), C.c_double(), C.c_double()
    lcb, ecb = LIN_CB(lin), ERR_CB(err)
    gm.gm_optimize(C.byref(params(**kw)), K, F, _p(np.ascontiguousarray(keys, dtype=np.int32)), len(priors), _p(pk), _p(pz), _p(pw), _p(T), lcb, ecb,
                   C.byref(r), C.byref(dt), C.byref(dr))
    return dict(T=T.reshape(K, 4, 4).transpose(0, 2, 1), error=r.error, num_inliers=r.num_inliers, iterations=r.iterations, trials=r.trials, status=r.status)


@pytest.mark.parametrize("case", ["default", "one_iteration", "no_step_test", "degenerate", "untouched_key"])
def test_host_state_machine_takes_the_restatements_decisions(gm, keyframes, case):
    fr, packed, maps = keyframes
    # (target, source, level): two factors on the pair (0, 1), one each on (0, 2) and (1, 2)
    spec = [(0, 1, 0.5), (0, 1, 1.0), (0, 2, 0.5), (1, 2, 0.5)]
    fac = [(maps[(t, r)],) + packed[s] for t, s, r in spec]
    keys = [(t, s) for t, s, _ in spec]
    rng = synth.rng_for(1300)
    T0 = [fr[0][2]] + [synth.perturb(fr[k][2], rng, 0.01, 0.1) for k in (1, 2)]
    priors = [(0, fr[0][2], 1e6)]
    kw = {}
    if case == "one_iteration":
        kw = dict(max_iterations=1)
    elif case == "no_step_test":
        kw = dict(max_iterations=10, step_translation_tol=0.0, step_rotation_tol=0.0, absolute_error_tol=0.0)
    elif case == "degenerate":
        T0[1] = T0[1].copy()
        T0[1][:3, 3] += 1000.0
        T0[2] = T0[2].copy()
        T0[2][:3, 3] += (0.0, 1000.0, 0.0)  # every factor's relative pose is 1 km off
    elif case == "untouched_key":
        T0 = T0 + [synth.pose(3.0, 1.0, 0.0, 0.2)]
    ref = go.optimize(lambda f, d: (oracle.split122(oracle.linearize_gpumap(fac[f][0], *fac[f][1:], d)[0]), d),
                      lambda f, dl, d: oracle.error_gpumap(fac[f][0], *fac[f][1:], dl, d), keys, T0, priors, kw)
    got = host_optimize(gm, fac, keys, T0, priors, **kw)
    assert (got["iterations"], got["trials"], got["status"]) == (ref["iterations"], ref["trials"], ref["status"]), (got, ref)
    assert np.abs(got["T"] - ref["T"]).max() < 1e-8
    assert got["num_inliers"] == ref["num_inliers"]
    assert abs(got["error"] - ref["error"]) <= 1e-9 * max(ref["error"], 1.0)
    if case == "degenerate":
        assert ref["status"] == lm.ALIGN_DEGENERATE and np.array_equal(got["T"], np.stack(T0)) and got["trials"] == 0
    if case == "untouched_key":
        assert np.array_equal(got["T"][3], T0[3])
    if case == "default":
        assert ref["iterations"] >= 2
