"""CPU-only checks of gb_pose_graph_optimize's arithmetic, rule and binding.

glim_b200/csrc/gb_pose_graph_math.cuh holds the text k_pose_graph_step / k_pose_graph_accept compile for the device (the between
term, the assembly, the damped padded copy, the tile schedule of the Cholesky and the substitution, the round's two halves).
Here the SAME text is compiled for the host with g++ (tests/cpp/pose_graph_math_host.cpp), one thread, no barrier and scalar
tile products, and checked against numpy and the rule's restatement in tests/pose_graph_oracle.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth
from oracle import oracle
from tests import graph_oracle as go
from tests import lm_oracle as lm
from tests import pose_graph_oracle as pgo
from tests import voxelmap_oracle as vo
from tests.util import cov_colmajor16

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIN_CB = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.POINTER(C.c_double))
ERR_CB = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double))


@pytest.fixture(scope="module")
def pm(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pm") / "libpose_graph_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so,
                           os.path.join(ROOT, "tests", "cpp", "pose_graph_math_host.cpp")])
    L = C.CDLL(so)
    vp, f64, i32 = C.c_void_p, C.c_double, C.c_int
    L.pgm_between.argtypes = [vp, vp, vp, vp]
    L.pgm_between.restype = f64
    L.pgm_solve.argtypes = [i32, vp, vp, f64, vp]
    L.pgm_assemble.argtypes = [i32, i32, vp, vp, i32, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp]
    L.pgm_optimize.argtypes = [vp, i32, i32, vp, i32, vp, i32, vp, vp, vp, vp, LIN_CB, ERR_CB, vp, vp, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def params(**kw):
    p = capi.AlignParams()
    for k, v in dict(lm.ALIGN_DEFAULTS, **kw).items():
        setattr(p, k, v)
    return p


def spd(rng, scale=1.0):
    A = rng.normal(size=(6, 6))
    L = A @ A.T + 0.5 * np.eye(6)
    L = 0.5 * (L + L.T)
    return scale * L


def big_rotation(rng, max_deg=170.0):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    th = np.radians(rng.uniform(0.0, max_deg))
    return synth.se3_exp(np.concatenate([th * axis, rng.normal(size=3) * 5.0]))


def record(Ti, Tj, Z, L, k, pm):
    bt = gpu.between_terms([(0, 1, Z, L, k)])
    rec = np.zeros(122)
    e = pm.pgm_between(_p(oracle.pose_colmajor(Ti)), _p(oracle.pose_colmajor(Tj)), _p(bt), _p(rec))
    return e, oracle.split122(rec)


@pytest.mark.parametrize("huber", ["none", "inside", "outside"])
def test_between_term_against_gtsam_jacobians_and_differences(pm, huber):
    rng = np.random.default_rng({"none": 1, "inside": 2, "outside": 3}[huber])
    for it in range(20):
        Ti, Tj = big_rotation(rng), big_rotation(rng)
        Z = synth.perturb(synth.inv_pose(Ti) @ Tj, rng, 0.3 if it % 2 else 1e-3, 0.5)
        L = spd(rng, 10.0 ** rng.uniform(-2, 4))
        m = np.sqrt(pgo.between_term(Ti, Tj, Z, L, 0.0)[4] @ L @ pgo.between_term(Ti, Tj, Z, L, 0.0)[4])
        k = {"none": None, "inside": 2.0 * m + 1e-6, "outside": 0.3 * m}[huber]
        e, rec = record(Ti, Tj, Z, L, k, pm)
        ref = pgo.between_record(Ti, Tj, Z, L, k or 0.0)
        assert abs(e - ref["error"]) <= 1e-9 * ref["error"] + 1e-300
        for key in ("H_tt", "H_ss", "H_ts", "b_t", "b_s"):
            scale = max(np.abs(ref[key]).max(), 1e-300)
            assert np.abs(rec[key] - ref[key]).max() <= 1e-8 * scale, (it, key)
        # GTSAM's closed form against central differences of r(T_i Exp(xi_i), T_j Exp(xi_j))
        _, w, Ji, Jj, r = pgo.between_term(Ti, Tj, Z, L, k or 0.0)

        def res(xi, j):
            a = Ti @ synth.se3_exp(xi) if j == 0 else Ti
            b = Tj @ synth.se3_exp(xi) if j == 1 else Tj
            return go.se3_log(synth.inv_pose(Z) @ synth.inv_pose(a) @ b)

        h = 1e-6
        for j, J in ((0, Ji), (1, Jj)):
            Jn = np.stack([(res(h * u, j) - res(-h * u, j)) / (2 * h) for u in np.eye(6)], axis=1)
            assert np.abs(Jn - J).max() <= 1e-5 * max(1.0, np.abs(J).max()), (it, j)
        # the error's gradient is 2 w J^T L r where the weight is flat (b = half the gradient of the error)
        if huber != "outside":
            grad = np.array([(pgo.between_term(Ti @ synth.se3_exp(h * u), Tj, Z, L, k or 0.0)[0] - pgo.between_term(Ti @ synth.se3_exp(-h * u), Tj, Z, L, k or 0.0)[0]) / (2 * h) for u in np.eye(6)])
            assert np.abs(rec["b_t"] - 0.5 * grad).max() <= 1e-5 * max(np.abs(grad).max(), 1e-6)
        if huber == "outside":
            assert w < 1.0 and abs(e - (2 * k * m - k * k)) <= 1e-9 * e
        else:
            assert w == 1.0 and abs(e - r @ L @ r) <= 1e-9 * e + 1e-300


@pytest.mark.parametrize("n", [198, 384, 1536, 2000])
def test_tiled_cholesky_solve_matches_numpy(pm, n):
    rng = np.random.default_rng(n)
    A = rng.normal(size=(n, n)) / np.sqrt(n)
    H = A @ A.T + np.diag(rng.uniform(0.5, 2.0, size=n))
    b = rng.normal(size=n)
    lam = 1e-3
    d = np.zeros(n)
    assert pm.pgm_solve(n, _p(np.ascontiguousarray(H)), _p(b), lam, _p(d)) == 1
    M = H + lam * np.eye(n)
    np.linalg.cholesky(M)
    ref = np.linalg.solve(M, -b)
    assert np.linalg.norm(d - ref) <= 1e-12 * np.linalg.cond(M) * np.linalg.norm(ref)
    d2 = np.zeros(n)  # only the lower triangle is read
    assert pm.pgm_solve(n, _p(np.ascontiguousarray(np.tril(H))), _p(b), lam, _p(d2)) == 1 and np.array_equal(d, d2)
    bad = H.copy()
    bad[n - 3, n - 3] = -10.0  # a pivot of the last tile column fails
    assert pm.pgm_solve(n, _p(np.ascontiguousarray(bad)), _p(b), lam, _p(np.zeros(n))) == 0
    nan = H.copy()
    nan[n // 2, n // 2] = np.nan
    assert pm.pgm_solve(n, _p(np.ascontiguousarray(nan)), _p(b), lam, _p(np.zeros(n))) == 0


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
def test_assembly_matches_the_restatement_entry_for_entry(pm, seed):
    """random topologies with factors, between terms and priors (several on one pair and one key, both orders of a pair,
    the last key touched by nothing): every entry of H and b the restatement's sum in the stated order, bit for bit"""
    rng = np.random.default_rng(300 + seed)
    K = int(rng.integers(3, 41))
    fkeys = [(0, 1), (1, 0)] + [tuple(int(x) for x in rng.choice(K - 1, 2, replace=False)) for _ in range(int(rng.integers(0, 40)))]
    if seed == 5:
        fkeys = []
    bkeys = [(1, 0), (0, 1)] + [tuple(int(x) for x in rng.choice(K - 1, 2, replace=False)) for _ in range(int(rng.integers(1, 30)))]
    T = [big_rotation(rng, 60.0) for _ in range(K)]
    bts = [(i, j, synth.perturb(synth.inv_pose(T[i]) @ T[j], rng, 0.2, 0.5), spd(rng), (None, 0.5)[m % 2]) for m, (i, j) in enumerate(bkeys)]
    qkeys = [0, 0] + [int(x) for x in rng.integers(0, K - 1, size=int(rng.integers(0, 6)))]
    qz = [synth.perturb(T[k], rng, 0.1, 0.2) for k in qkeys]
    qw = list(10.0 ** rng.uniform(0, 8, size=len(qkeys)))
    raws = np.stack([random_record(rng) for _ in fkeys]) if fkeys else np.zeros((0, 122))
    n, B, Q = 6 * K, len(bts), len(qkeys)
    H, b, brec, prec = np.zeros((n, n)), np.zeros(n), np.zeros((B, 122)), np.zeros((Q, 43))
    Tc = np.ascontiguousarray(np.stack([oracle.pose_colmajor(x) for x in T]))
    pm.pgm_assemble(K, len(fkeys), _p(np.ascontiguousarray(fkeys, dtype=np.int32).reshape(-1, 2)), _p(raws), B, _p(gpu.between_terms(bts)), Q,
                    _p(np.ascontiguousarray(qkeys, dtype=np.int32)), _p(np.ascontiguousarray([oracle.pose_colmajor(z) for z in qz])), _p(np.asarray(qw)),
                    _p(Tc), _p(H), _p(b), _p(brec), _p(prec))
    Hr, br, _, _ = pgo.assemble(K, fkeys, [oracle.split122(r) for r in raws], bkeys, [oracle.split122(r) for r in brec], qkeys,
                                [(p[:36].reshape(6, 6), p[36:42], p[42]) for p in prec])
    assert np.array_equal(np.tril(H), np.tril(Hr))  # the same sums in the same order
    assert np.array_equal(b, br)
    assert not H[-6:].any() and not b[-6:].any()
    for m, (i, j, Z, L, k) in enumerate(bts):  # and the terms themselves are the restatement's
        ref = pgo.between_record(T[i], T[j], Z, L, k or 0.0)
        assert np.abs(oracle.split122(brec[m])["H_ts"] - ref["H_ts"]).max() <= 1e-8 * np.abs(ref["H_ts"]).max()


def host_optimize(pm, fac, fkeys, T0, priors, betweens, **kw):
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
    bt = gpu.between_terms(betweens)
    r, dt, dr = capi.GraphResult(), C.c_double(), C.c_double()
    lcb, ecb = LIN_CB(lin), ERR_CB(err)
    pm.pgm_optimize(C.byref(params(**kw)), K, F, _p(np.ascontiguousarray(fkeys, dtype=np.int32).reshape(-1, 2)), len(bt), _p(bt), len(priors), _p(pk), _p(pz), _p(pw),
                    _p(T), lcb, ecb, C.byref(r), C.byref(dt), C.byref(dr))
    return dict(T=T.reshape(K, 4, 4).transpose(0, 2, 1), error=r.error, num_inliers=r.num_inliers, iterations=r.iterations, trials=r.trials, status=r.status)


def pose_graph_problem(K, seed, wrong=(), sigma=0.5, huber=0.1):
    """an odometry chain on a loop with loop closures (two of them wrong), drifted starts"""
    rng = np.random.default_rng(seed)
    gt = synth.loop_trajectory(K, 1, side=20.0)[:K]
    odo = 1.0 / sigma**2
    bts = [(k, k + 1, synth.perturb(synth.inv_pose(gt[k]) @ gt[k + 1], rng, 0.002, 0.01), odo, None) for k in range(K - 1)]
    for m, (i, j) in enumerate([(0, K - 1), (1, K - 2), (2, K // 2), (3, K // 2 + 1)]):
        Z = synth.inv_pose(gt[i]) @ gt[j]
        if m in wrong:
            Z = Z @ synth.pose(3.0, -2.0, 0.5, 0.4)
        bts.append((i, j, Z, np.eye(6) * 4.0, huber))
    drift = np.array([0.0, 0.0, 0.003, 0.02, 0.01, 0.0])
    T0 = [gt[0]] + [gt[k] @ synth.se3_exp(k * drift) for k in range(1, K)]
    return gt, T0, bts


@pytest.fixture(scope="module")
def keyframes():
    fr = vo.arc_frames(3, 32 * 150)
    packed = [oracle.pack_cloud(p, cov_colmajor16(c)) for p, c, _ in fr]
    maps = {(k, r): oracle.GpuMap(*packed[k], r) for k in (0, 1) for r in (0.5, 1.0)}
    return fr, packed, maps


@pytest.mark.parametrize("case", ["pose_graph", "huber_loops", "factors_and_betweens", "degenerate", "untouched_key"])
def test_host_state_machine_takes_the_restatements_decisions(pm, keyframes, case):
    kw = {}
    if case in ("pose_graph", "huber_loops"):
        gt, T0, bts = pose_graph_problem(12, 40, wrong=(2, 3) if case == "huber_loops" else ())
        fac, fkeys, priors = [], [], [(0, T0[0], 1e10)]
        kw = dict(max_iterations=20)
    else:
        fr, packed, maps = keyframes
        spec = [(0, 1, 0.5), (0, 1, 1.0), (0, 2, 0.5), (1, 2, 0.5)]
        fac = [(maps[(t, r)],) + packed[s] for t, s, r in spec]
        fkeys = [(t, s) for t, s, _ in spec]
        rng = synth.rng_for(1310)
        T0 = [fr[0][2]] + [synth.perturb(fr[k][2], rng, 0.01, 0.1) for k in (1, 2)]
        priors = [(0, fr[0][2], 1e10)]
        bts = [(1, 2, synth.inv_pose(fr[1][2]) @ fr[2][2], 1e6, None), (2, 0, synth.inv_pose(fr[2][2]) @ fr[0][2], spd(rng, 1e3), 0.05)]
        if case == "degenerate":
            T0[1] = T0[1].copy()
            T0[1][:3, 3] += 1000.0
            T0[2] = T0[2].copy()
            T0[2][:3, 3] += (0.0, 1000.0, 0.0)
        elif case == "untouched_key":
            T0 = T0 + [synth.pose(3.0, 1.0, 0.0, 0.2)]
    bL = [(i, j, Z, np.asarray(L, float) * np.eye(6) if np.ndim(L) == 0 else L, k or 0.0) for i, j, Z, L, k in bts]
    ref = pgo.optimize(lambda f, d: (oracle.split122(oracle.linearize_gpumap(fac[f][0], *fac[f][1:], d)[0]), d),
                       lambda f, dl, d: oracle.error_gpumap(fac[f][0], *fac[f][1:], dl, d), fkeys, T0, priors, bL, kw)
    got = host_optimize(pm, fac, fkeys, T0, priors, bts, **kw)
    assert (got["iterations"], got["trials"], got["status"]) == (ref["iterations"], ref["trials"], ref["status"]), (got, ref)
    assert np.abs(got["T"] - ref["T"]).max() < 1e-8
    assert got["num_inliers"] == ref["num_inliers"]
    assert abs(got["error"] - ref["error"]) <= 1e-9 * max(ref["error"], 1.0)
    if case == "degenerate":
        assert ref["status"] == lm.ALIGN_DEGENERATE and np.array_equal(got["T"], np.stack(T0)) and got["trials"] == 0
    if case == "untouched_key":
        assert np.array_equal(got["T"][3], T0[3])
    if case == "huber_loops":
        w = pgo.huber_weights(got["T"], bL)
        assert w[-2] < 1.0 and w[-1] < 1.0, w[-4:]
    if case.startswith("pose_graph") or case == "huber_loops":
        assert ref["iterations"] >= 2


def test_between_terms_layout_and_mapping():
    """gpu.between_terms packs gb_between_term as the header lays it out: a scalar information is w I, a 6x6 goes column-major,
    huber_width None is 0, keys map through the local index"""
    dt = capi.BETWEEN_DTYPE
    assert dt.itemsize == 432 and [dt.fields[k][1] for k in ("key_i", "key_j", "Z", "information", "huber_width")] == [0, 4, 8, 136, 424]
    Z = synth.pose(1.0, 2.0, 3.0, 0.1, 0.2, 0.3)
    L = np.arange(36.0).reshape(6, 6)
    a = gpu.between_terms([("a", "b", Z, 4.0, None), ("b", "a", Z, L, 0.25)], {"a": 7, "b": 3})
    assert (a[0]["key_i"], a[0]["key_j"], a[1]["key_i"], a[1]["key_j"]) == (7, 3, 3, 7)
    assert np.array_equal(a[0]["Z"], Z.T.ravel()) and np.array_equal(a[0]["information"], (4.0 * np.eye(6)).ravel())
    assert np.array_equal(a[1]["information"].reshape(6, 6).T, L) and (a[0]["huber_width"], a[1]["huber_width"]) == (0.0, 0.25)


def test_binding_maps_keys_and_refuses_fixed_targets(monkeypatch):
    """optimize_pose_graph's arguments as the C call receives them (a recording stand-in for the library)"""
    seen = {}

    class Fake:
        def gb_align_default_params(self, p):
            return capi.lib().gb_align_default_params(p)

        def gb_pose_graph_optimize(self, ctx, K, T, F, fac, fk, Q, qk, qp, qw, B, bt, prm, Tout, res):
            seen.update(K=K, F=F, Q=Q, B=B, qk=np.ctypeslib.as_array(C.cast(qk, C.POINTER(C.c_int32)), shape=(Q,)).copy(),
                        bt=np.frombuffer((C.c_char * (432 * B)).from_address(bt.value), capi.BETWEEN_DTYPE).copy(),
                        T=np.ctypeslib.as_array(C.cast(T, C.POINTER(C.c_double)), shape=(K, 16)).copy())
            out = np.ctypeslib.as_array(C.cast(Tout, C.POINTER(C.c_double)), shape=(K, 16))
            out[:] = seen["T"]
            return 0

    class Ctx:
        h = None

    monkeypatch.setattr(gpu, "lib", lambda: Fake())
    vals = {10: synth.pose(1, 0, 0, 0), 20: synth.pose(2, 0, 0, 0), 30: synth.pose(3, 0, 0, 0)}
    Z = synth.pose(1, 0, 0, 0)
    r = gpu.optimize_pose_graph([], vals, priors=[(20, vals[20], 1e10)], betweens=[(10, 20, Z, 1e6, None), (30, 20, Z, np.eye(6), 0.5)], ctx=Ctx())
    assert (seen["K"], seen["F"], seen["Q"], seen["B"]) == (3, 0, 1, 2)
    assert list(seen["qk"]) == [1] and [(b["key_i"], b["key_j"]) for b in seen["bt"]] == [(0, 1), (2, 1)]
    assert np.array_equal(seen["T"], capi.pose16(np.stack(list(vals.values()))))
    assert set(r["values"]) == {10, 20, 30} and np.array_equal(r["values"][30], vals[30])
    with pytest.raises(capi.GlimB200Error):

        class Unary(gpu.IntegratedVGICPFactorGPU):
            def __init__(self):
                pass

            def is_binary(self):
                return False

        gpu.optimize_pose_graph([Unary()], vals, ctx=Ctx())


def test_refusals_without_factors_need_no_device():
    """every refusal that does not concern a factor, made by the library before it reads the context (a stand-in context
    block that is never entered); the refusals that concern factors are checked on the device"""
    L = capi.lib()
    fake = (C.c_char * 4096)()
    ctx = C.cast(fake, C.c_void_p)
    T0 = capi.pose16(np.stack([synth.pose(k, 0, 0, 0) for k in range(3)]))
    Z = capi.pose16(np.eye(4)[None])
    res = capi.GraphResult()
    Tout = np.zeros_like(T0)
    good = gpu.align_params()

    def bt(**kw):
        a = gpu.between_terms([(0, 1, synth.pose(1, 0, 0, 0), 1.0, None), (1, 2, synth.pose(1, 0, 0, 0), 1.0, 0.5)])
        for k, v in kw.items():
            a[1][k] = v
        return a

    def call(K=3, T=T0, qkeys=(0,), qposes=Z, qw=(1e10,), betweens=None, prm=good, out=Tout, c=ctx):
        b = bt() if betweens is None else betweens
        return L.gb_pose_graph_optimize(c, K, capi.ptr(T), 0, None, None, len(qkeys), capi.ptr(np.asarray(qkeys, np.int32)), capi.ptr(qposes),
                                        capi.ptr(np.asarray(qw, np.float64)), len(b), capi.ptr(b), C.byref(prm) if prm is not None else None,
                                        capi.ptr(out), C.byref(res))

    assert call(c=None) == 1
    assert call(out=None) == 1
    assert call(K=1) == 1 and call(K=1025) == 1
    assert call(betweens=bt()[:0]) == 1                                          # no factor and no between term
    assert call(betweens=bt(key_j=3)) == 1 and call(betweens=bt(key_i=-1)) == 1   # between key out of range
    assert call(betweens=bt(key_j=1)) == 1                                        # key_i == key_j
    Zb = np.eye(4).T.ravel().copy()
    Zb[13] = np.nan
    assert call(betweens=bt(Z=Zb)) == 1                                           # non-finite measurement
    Li = np.eye(6).ravel().copy()
    Li[1] = 1e-3
    assert call(betweens=bt(information=Li)) == 1                                 # not exactly symmetric
    Li = np.eye(6).ravel().copy()
    Li[7] = np.inf
    assert call(betweens=bt(information=Li)) == 1                                 # non-finite information
    assert call(betweens=bt(huber_width=-1.0)) == 1 and call(betweens=bt(huber_width=np.nan)) == 1
    bad = T0.copy()
    bad[2, 12] = np.inf
    assert call(T=bad) == 1                                                       # non-finite pose
    badZ = Z.copy()
    badZ[0, 5] = np.nan
    assert call(qposes=badZ) == 1                                                 # non-finite prior pose
    assert call(qw=(-1.0,)) == 1 and call(qw=(np.inf,)) == 1
    assert call(qkeys=(3,)) == 1 and call(qkeys=(-1,)) == 1                        # prior key out of range
    assert call(prm=None) == 1 and call(prm=gpu.align_params(max_iterations=0)) == 1 and call(prm=gpu.align_params(lambda_factor=1.0)) == 1
    assert "huber_width" in (call(betweens=bt(huber_width=-1.0)) and L.gb_last_error().decode())
