"""gb_pose_graph_optimize on the H100: Levenberg-Marquardt over one global map of up to 1024 poses, against the restatement of the
rule in tests/pose_graph_oracle.py (fed the fp64 oracle or the device's own records), against gb_graph_optimize and against
ground truth; GLIM's global-mapping and pose-graph graphs, determinism, launch counts and refusals."""
import ctypes as C

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth, workloads
from oracle import oracle
from tests import graph_oracle as go
from tests import lm_oracle as lm
from tests import pose_graph_oracle as pgo
from tests import solve_check as sc
from tests.util import cov_colmajor16

pytestmark = pytest.mark.gpu

PRIOR = 1e10  # init_pose_damping_scale: GLIM's LinearDampingFactor on X(0) as a prior at its initial pose
ODOM_SIGMA, LOOP_SIGMA, LOOP_HUBER = 1e-3, 0.1, 1.0  # global_mapping_pose_graph.cpp:53-55
GTSAM_LM = {"lambda_initial": 1e-5, "lambda_factor": 10.0, "lambda_upper_bound": 1e5, "relative_error_tol": 1e-5, "absolute_error_tol": 1e-5,
            "step_translation_tol": 0.0, "step_rotation_tol": 0.0}


def pose_error(T, T_ref):
    d = synth.inv_pose(T_ref) @ T
    return float(np.linalg.norm(d[:3, 3])), float(np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1)))


def rel(A, B):
    return synth.inv_pose(A) @ B


def random_between_graph(K, seed):
    """a chain plus random extra edges, random SPD information, starts off the measurements"""
    rng = np.random.default_rng(seed)
    gt = [synth.se3_exp(np.concatenate([rng.normal(size=3) * 0.5, rng.normal(size=3) * 20.0])) for _ in range(K)]
    edges = [(k, k + 1) for k in range(K - 1)] + [tuple(int(x) for x in rng.choice(K, 2, replace=False)) for _ in range(K // 2)]
    bts = []
    for m, (i, j) in enumerate(edges):
        A = rng.normal(size=(6, 6))
        L = A @ A.T + 6.0 * np.eye(6)
        L = np.triu(L) + np.triu(L, 1).T
        bts.append((i, j, synth.perturb(rel(gt[i], gt[j]), rng, 0.01, 0.05), L, 0.0 if m % 3 else 2.0))
    T0 = [gt[0]] + [synth.perturb(T, rng, 0.02, 0.2) for T in gt[1:]]
    return gt, T0, bts


def as_betweens(bts):
    return [(i, j, Z, L, k if k else None) for i, j, Z, L, k in bts]


def well_conditioned_graph(K, seed):
    """a chain plus 4 K random edges between poses within metres of each other, random SPD information, precision-100 priors
    on keys 0, K / 8, 2 K / 8, ...: the damped system's condition number stays below 1e6 at K <= 1024"""
    rng = np.random.default_rng(seed)
    gt = [synth.se3_exp(np.concatenate([rng.normal(size=3) * 0.3, rng.normal(size=3)])) for _ in range(K)]
    edges = [(k, k + 1) for k in range(K - 1)] + [tuple(int(x) for x in rng.choice(K, 2, replace=False)) for _ in range(4 * K)]
    bts = []
    for m, (i, j) in enumerate(edges):
        A = rng.normal(size=(6, 6))
        L = A @ A.T + 6.0 * np.eye(6)
        L = np.triu(L) + np.triu(L, 1).T
        bts.append((i, j, synth.perturb(rel(gt[i], gt[j]), rng, 0.01, 0.05), L, 0.0 if m % 3 else 2.0))
    T0 = [gt[0]] + [synth.perturb(T, rng, 0.02, 0.2) for T in gt[1:]]
    return T0, bts, [(k, T0[k], 100.0) for k in range(0, K, max(1, K // 8))]


def condition_1norm(T0, priors, bts, lam):
    """LAPACK's 1-norm condition estimate of the first damped system, from its Cholesky factor"""
    from scipy.linalg import lapack

    K = len(T0)
    recs = [pgo.between_record(T0[i], T0[j], Z, L, k) for i, j, Z, L, k in bts]
    qblocks = [go.prior_term(T0[k], Z, w)[1:] + (0.0,) for k, Z, w in priors]
    H, _, _, _ = pgo.assemble(K, [], [], [(i, j) for i, j, _, _, _ in bts], recs, [k for k, _, _ in priors], qblocks)
    A = H + lam * np.eye(6 * K)
    c, info = lapack.dpotrf(A, lower=1)
    assert info == 0
    rcond, info = lapack.dpocon(c, np.abs(A).sum(axis=0).max(), uplo="L")
    return 1.0 / rcond


@pytest.mark.parametrize("K", [33, 64, 341, 1024])
def test_one_round_between_only(ctx, K):
    """max_iterations = 1 on well-conditioned between-only graphs with random SPD information: the device's step against the
    restatement's.  Only the solve's order of operations differs (fp64 throughout), so the steps agree to about the condition
    number times the unit roundoff; 1e-9 relative holds with margin below a condition number of 1e6, which the test checks.
    The step's scaled backward error (tests/solve_check.py) is held to the restatement's, whatever the condition number."""
    T0, bts, priors = well_conditioned_graph(K, 500 + K)
    assert condition_1norm(T0, priors, bts, lm.ALIGN_DEFAULTS["lambda_initial"]) < 1e6
    got = gpu.optimize_pose_graph([], dict(enumerate(T0)), priors=priors, betweens=as_betweens(bts), params={"max_iterations": 1}, ctx=ctx)
    with sc.systems() as seen:
        ref = pgo.optimize(None, None, [], T0, priors, bts, {"max_iterations": 1})
    assert (got["iterations"], got["trials"], got["status"]) == (ref["iterations"], ref["trials"], ref["status"]) == (1, 1, lm.ALIGN_MAX_ITERATIONS)
    assert got["num_inliers"] == 0.0
    d_got = np.concatenate([go.se3_log(rel(T0[k], got["values"][k])) for k in range(K)])
    d_ref = np.concatenate([go.se3_log(rel(T0[k], ref["T"][k])) for k in range(K)])
    assert np.linalg.norm(d_got - d_ref) <= 1e-9 * np.linalg.norm(d_ref), np.linalg.norm(d_got - d_ref) / np.linalg.norm(d_ref)
    sc.check(f"pose graph K {K}, well conditioned", seen[0], d_got, d_ref, sc.pose_eps(T0, [got["values"][k] for k in range(K)]))
    assert abs(got["error"] - ref["error"]) <= 1e-9 * ref["error"]


@pytest.fixture(scope="module")
def gm64(ctx):
    """global mapping scaled down: 64 submaps on two laps, drifted starts, the fp64 oracle maps"""
    w = workloads.global_mapping(ctx, n_submaps=64, laps=2, n_rays=64 * 128)
    facs = w.gpu_factors(w.sets[0])
    rng = synth.rng_for(2100)
    drift = np.array([0.0, 0.0, 0.001, 0.01, -0.005, 0.0])
    n = len(w.poses)
    T0 = [w.poses[0]] + [synth.perturb(w.poses[k] @ synth.se3_exp(k * drift), rng, 0.002, 0.02) for k in range(1, n)]
    packed = [oracle.pack_cloud(p, cov_colmajor16(c)) for p, c in w.host_clouds]
    omaps = {(i, l): oracle.GpuMap(*packed[i], r) for i in range(n) for l, r in enumerate(w.resolutions)}
    fac = [(omaps[(f.target, f.level)],) + packed[f.source] for f in w.sets[0].factors]
    keys = [(f.target, f.source) for f in w.sets[0].factors]
    return dict(w=w, facs=facs, T0=T0, fac=fac, keys=keys)


def restated(g, priors, betweens, params):
    fac = g["fac"]
    return pgo.optimize(lambda f, d: (oracle.split122(oracle.linearize_gpumap(fac[f][0], *fac[f][1:], d)[0]), d),
                        lambda f, dl, d: oracle.error_gpumap(fac[f][0], *fac[f][1:], dl, d), g["keys"], g["T0"], priors, betweens, params)


def test_global_mapping_scaled_down(ctx, gm64):
    g = gm64
    w, T0 = g["w"], g["T0"]
    priors = [(0, T0[0], PRIOR)]
    prm = dict(GTSAM_LM, max_iterations=20)
    got = gpu.optimize_pose_graph(g["facs"], dict(enumerate(T0)), priors=priors, params=prm, ctx=ctx)
    ref = restated(g, priors, [], prm)
    print(f"global mapping 64: {len(g['facs'])} factors, device {got['iterations']}/{got['trials']}/{got['status_name']}, "
          f"restated {ref['iterations']}/{ref['trials']}/{ref['status']}")
    assert (got["iterations"], got["trials"], got["status"]) == (ref["iterations"], ref["trials"], ref["status"])
    bound = max(pose_error(ref["T"][k], w.poses[k])[0] for k in range(len(T0)))
    for k in range(len(T0)):
        et, er = pose_error(got["values"][k], w.poses[k])
        assert et <= 1.5 * bound + 1e-3, (k, et, bound)
        et, er = pose_error(got["values"][k], ref["T"][k])
        assert et < 2e-3 and er < 2e-3, (k, et, er)


def test_agrees_with_graph_optimize_at_32_keys(ctx, gm64):
    """the first 32 submaps as one problem of gb_graph_optimize and as a pose graph: the same rule, only the solve differs"""
    g = gm64
    sel = [f for f, (t, s) in zip(g["facs"], g["keys"]) if t < 32 and s < 32]
    vals = {k: g["T0"][k] for k in range(32)}
    priors = [(0, g["T0"][0], PRIOR)]
    a = gpu.optimize_graphs([dict(factors=sel, values=vals, priors=priors)], params={"max_iterations": 10})[0]
    b = gpu.optimize_pose_graph(sel, vals, priors=priors, params={"max_iterations": 10}, ctx=ctx)
    assert (a["iterations"], a["trials"], a["status"]) == (b["iterations"], b["trials"], b["status"])
    for k in range(32):
        assert np.abs(a["values"][k] - b["values"][k]).max() <= 1e-9, k
    assert a["num_inliers"] == b["num_inliers"]


def test_glim_between_recipes_mixed_with_vgicp(ctx, gm64):
    """global_mapping.cpp:475-481 (an isolated submap's between, 1e6 I) and create_between_factors with GICP (:379-428: L =
    the registration's Hessian block of X(1) + 1e6 I, the registration a two-key gb_graph_optimize) next to the VGICP factors,
    against the restatement on the fp64 oracle.  The registration's measurement carries its own error and L weighs it about
    1e7: the graph's optimum follows it, wherever ground truth is, so the device is held to the restatement's optimum."""
    g = gm64
    T0 = g["T0"]
    # the isolated submap: drop every factor that touches key 40 and tie it to 39 with the between of the starts
    keep = [i for i, (t, s) in enumerate(g["keys"]) if 40 not in (t, s)]
    facs = [g["facs"][i] for i in keep]
    iso = (39, 40, rel(T0[39], T0[40]), 1e6, None)
    # create_between_factors: register 20 -> 21 with a two-key problem, then take its Hessian block of X(1)
    pair = [g["facs"][i] for i, (t, s) in enumerate(g["keys"]) if (t, s) == (20, 21)]
    reg = gpu.optimize_graphs([dict(factors=pair, values={20: T0[20], 21: T0[21]}, priors=[(20, T0[20], 1e6)])], params={"max_iterations": 10})[0]
    H1 = sum(f.linearize(reg["values"])["H_ss"] for f in pair)
    L = 0.5 * (H1 + H1.T) + 1e6 * np.eye(6)
    gicp = (20, 21, rel(reg["values"][20], reg["values"][21]), L, None)
    prm = dict(GTSAM_LM, max_iterations=20)
    priors = [(0, T0[0], PRIOR)]
    got = gpu.optimize_pose_graph(facs, dict(enumerate(T0)), priors=priors, betweens=[iso, gicp], params=prm, ctx=ctx)
    sub = dict(g, fac=[g["fac"][i] for i in keep], keys=[g["keys"][i] for i in keep])
    bL = [(i, j, Z, np.asarray(Li, float) * np.eye(6) if np.ndim(Li) == 0 else Li, 0.0) for i, j, Z, Li, _ in (iso, gicp)]
    ref = restated(sub, priors, bL, prm)
    assert (got["iterations"], got["trials"], got["status"]) == (ref["iterations"], ref["trials"], ref["status"])
    assert got["iterations"] >= 2 and got["num_inliers"] == ref["num_inliers"]
    for k in range(len(T0)):
        et, er = pose_error(got["values"][k], ref["T"][k])
        assert et < 2e-3 and er < 2e-3, (k, et, er)
    # the isolated submap keeps its between, and the registration's between holds against the factors of the pair
    et, er = pose_error(rel(got["values"][39], got["values"][40]), iso[2])
    assert et < 1e-3 and er < 1e-3, (et, er)
    r_end = go.se3_log(rel(gicp[2], rel(got["values"][20], got["values"][21])))
    r_start = go.se3_log(rel(gicp[2], rel(T0[20], T0[21])))
    assert r_end @ L @ r_end < 0.01 * (r_start @ L @ r_start)


def test_pose_graph_back_end_with_huber_loops(ctx):
    """global_mapping_pose_graph.cpp: the anchor, an odometry chain (sigma 1e-3) and Huber loop factors (sigma 0.1, width 1.0),
    two of them wrong by metres: the restatement's path, the wrong loops down-weighted, the result near ground truth"""
    K = 48
    rng = np.random.default_rng(2200)
    gt = synth.loop_trajectory(K, 1, side=40.0)[:K]
    bts = [(k, k + 1, synth.perturb(rel(gt[k], gt[k + 1]), rng, 1e-4, 1e-3), np.eye(6) / ODOM_SIGMA**2, 0.0) for k in range(K - 1)]
    loops = [(0, K - 1), (2, K - 3), (5, K // 2), (7, K // 2 + 2)]
    for m, (i, j) in enumerate(loops):
        Z = rel(gt[i], gt[j])
        if m >= 2:
            Z = Z @ synth.pose(3.0, -2.0, 0.5, 0.5)
        bts.append((i, j, Z, np.eye(6) / LOOP_SIGMA**2, LOOP_HUBER))
    drift = np.array([0.0, 0.0, 0.002, 0.01, 0.005, 0.0])
    T0 = [gt[0]] + [gt[k] @ synth.se3_exp(k * drift) for k in range(1, K)]
    priors = [(0, T0[0], PRIOR)]
    prm = dict(GTSAM_LM, max_iterations=30)
    got = gpu.optimize_pose_graph([], dict(enumerate(T0)), priors=priors, betweens=as_betweens(bts), params=prm, ctx=ctx)
    ref = pgo.optimize(None, None, [], T0, priors, bts, prm)
    assert (got["iterations"], got["trials"], got["status"]) == (ref["iterations"], ref["trials"], ref["status"])
    Tg = [got["values"][k] for k in range(K)]
    for k in range(K):
        assert np.abs(Tg[k] - ref["T"][k]).max() < 1e-6, k
    w = pgo.huber_weights(Tg, bts)
    assert w[-1] < 1.0 and w[-2] < 1.0 and w[-4] == 1.0, w[-4:]
    bound = max(pose_error(ref["T"][k], gt[k])[0] for k in range(K))
    assert max(pose_error(Tg[k], gt[k])[0] for k in range(K)) <= bound + 1e-6 and bound < 0.5


def test_launches_per_round_do_not_depend_on_the_graph(ctx, gm64):
    per_round = []
    for K in (40, 1024):
        _, T0, bts = random_between_graph(K, 900 + K)
        before = ctx.kernel_launches
        r = gpu.optimize_pose_graph([], dict(enumerate(T0)), priors=[(0, T0[0], PRIOR)], betweens=as_betweens(bts), ctx=ctx)
        launches = ctx.kernel_launches - before
        assert launches == 2 * r["trials"], (K, launches, r)  # F = 0: no sweep, a step and an accept per round
        per_round.append(launches / r["trials"])
    assert per_round[0] == per_round[1]
    before = ctx.kernel_launches
    r = gpu.optimize_pose_graph(gm64["facs"], dict(enumerate(gm64["T0"])), priors=[(0, gm64["T0"][0], PRIOR)], ctx=ctx)
    assert ctx.kernel_launches - before <= 4 * r["trials"]


@pytest.fixture(scope="module")
def full(ctx):
    """the benchmark's global-mapping graph: 256 submaps on four laps, drifted starts"""
    w = workloads.global_mapping(ctx)
    facs = w.gpu_factors(w.sets[0])
    rng = synth.rng_for(2300)
    drift = np.array([0.0, 0.0, 0.0005, 0.005, -0.0025, 0.0])
    T0 = [w.poses[0]] + [synth.perturb(w.poses[k] @ synth.se3_exp(k * drift), rng, 0.002, 0.02) for k in range(1, len(w.poses))]
    return w, facs, T0


def test_benchmark_graph_converges_bit_identically(ctx, full):
    w, facs, T0 = full
    priors = [(0, T0[0], PRIOR)]
    prm = dict(GTSAM_LM, max_iterations=20)
    a = gpu.optimize_pose_graph(facs, dict(enumerate(T0)), priors=priors, params=prm, ctx=ctx)
    b = gpu.optimize_pose_graph(facs, dict(enumerate(T0)), priors=priors, params=prm, ctx=ctx)
    print(f"global mapping 256: {len(facs)} factors, {a['iterations']} iterations, {a['trials']} trials, {a['status_name']}")
    assert len(facs) > 6000
    assert a["status"] == lm.ALIGN_CONVERGED
    assert all(np.array_equal(a["values"][k], b["values"][k]) for k in a["values"]) and a["error"] == b["error"]
    start = max(pose_error(T0[k], w.poses[k])[0] for k in range(len(T0)))
    end = max(pose_error(a["values"][k], w.poses[k])[0] for k in range(len(T0)))
    print(f"largest translation error to ground truth: {start:.3f} m -> {end:.4f} m")
    assert end < 0.05 and end < 0.1 * start


def test_invalid_inputs_are_refused_before_any_launch(ctx, gm64):
    g = gm64
    L = capi.lib()
    facs = g["facs"][:2]
    keys = np.ascontiguousarray([[g["keys"][0][0], g["keys"][0][1]], [g["keys"][1][0], g["keys"][1][1]]], np.int32)
    arr = (C.c_void_p * 2)(*[f._handle() for f in facs])
    T0 = capi.pose16(np.stack(g["T0"]))
    res = capi.GraphResult()
    Tout = np.zeros_like(T0)
    good = gpu.align_params()
    Z = capi.pose16(np.eye(4)[None])
    bt = gpu.between_terms([(0, 1, np.eye(4), 1.0, None)])

    def call(K=len(g["T0"]), factors=arr, F=2, fkeys=keys, T=T0, betweens=bt):
        return L.gb_pose_graph_optimize(ctx.h, K, capi.ptr(T), F, C.cast(factors, C.c_void_p) if factors is not None else None, capi.ptr(np.ascontiguousarray(fkeys, np.int32)),
                                        1, capi.ptr(np.zeros(1, np.int32)), capi.ptr(Z), capi.ptr(np.ones(1)), len(betweens), capi.ptr(betweens), C.byref(good),
                                        capi.ptr(Tout), C.byref(res))

    src = g["w"].clouds[1]
    ivox = gpu.IVoxGPU(0.5, ctx=ctx)
    ivox.insert(g["w"].clouds[0])
    grid = gpu.PointGridGPU(g["w"].clouds[0], 1.05, ctx=ctx)
    gicp = gpu.IntegratedGICPFactorGPU(0, 1, grid, src, 1.0, ctx=ctx)  # held: the handles below must outlive the calls
    mixed = (C.c_void_p * 2)(arr[0], gicp._handle())
    ct_src = gpu.PointCloudGPU.clone(*g["w"].host_clouds[1], ctx=ctx)
    ct_src.add_times(np.linspace(0.0, 0.1, ct_src.size()))
    ctf = gpu.IntegratedCT_GICPFactorGPU(0, 1, ivox, ct_src, 1.0, ctx=ctx)
    ct = (C.c_void_p * 2)(arr[0], ctf._handle())
    vals = dict(enumerate(g["T0"]))
    before = [f.linearize(vals) for f in facs]
    launches = ctx.kernel_launches
    big = capi.pose16(np.stack([np.eye(4)] * 1025))
    assert call(K=1025, T=big) == 1                                          # K > 1024
    assert call(K=1) == 1
    assert call(F=0, factors=None, betweens=bt[:0]) == 1                     # nothing to optimize
    assert call(fkeys=[[0, 1], [1, len(g["T0"])]]) == 1                      # factor key out of range
    assert call(fkeys=[[0, 1], [2, 2]]) == 1                                 # target == source
    assert call(factors=(C.c_void_p * 2)(arr[0], None)) == 1                 # null factor
    assert call(factors=None) == 1
    assert call(factors=mixed) == 1                                          # two classes
    assert call(factors=ct) == 1                                             # a CT factor
    assert ctx.kernel_launches == launches
    after = [f.linearize(vals) for f in facs]
    for a, b in zip(before, after):
        assert a["num_inliers"] == b["num_inliers"] and np.array_equal(a["H_ss"], b["H_ss"]) and a["error"] == b["error"]
