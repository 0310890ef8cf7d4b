"""gb_graph_optimize on the H100: Levenberg-Marquardt over several poses per problem, many problems in one call, against the
restatement of the same rule in tests/graph_oracle.py (fed the fp64 oracles, or the device's own records), against ground truth
and against the fixed-target recipes of gb_vgicp_align; GLIM's three call sites, batches, launch counts and refusals."""
import ctypes as C

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth, workloads
from oracle import oracle
from tests import graph_oracle as gro
from tests import grid_oracle as go
from tests import lm_oracle as lm
from tests import solve_check as sc
from tests import voxelmap_oracle as vo
from tests.util import cov_colmajor16

pytestmark = pytest.mark.gpu

# GTSAM's LevenbergMarquardtParams defaults with no step test (sub_mapping.cpp:428-452, manual_loop_close_modal.cpp:476-517)
GTSAM_LM = {"lambda_initial": 1e-5, "lambda_factor": 10.0, "lambda_upper_bound": 1e5, "relative_error_tol": 1e-5, "absolute_error_tol": 1e-5,
            "step_translation_tol": 0.0, "step_rotation_tol": 0.0}
RECIPE_CELL = 1.05  # the point grid's cell per max correspondence distance (tests/test_point_grid_gpu.py)


def pose_error(T, T_ref):
    d = synth.inv_pose(T_ref) @ T
    return float(np.linalg.norm(d[:3, 3])), float(np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1)))


def rel(T0, T1):
    return synth.inv_pose(T0) @ T1


@pytest.fixture(scope="module")
def kf(ctx):
    """four hdl32 keyframes 1 m apart: device clouds and VGICP maps (0.5 / 1.0 m), oracle maps and packed clouds"""
    fr = vo.arc_frames(4, 32 * 200)
    clouds = [gpu.PointCloudGPU.clone(p, c, ctx=ctx) for p, c, _ in fr]
    maps = {(k, r): gpu.GaussianVoxelMapGPU(r, ctx=ctx).insert(clouds[k]) for k in range(4) for r in (0.5, 1.0)}
    packed = [oracle.pack_cloud(p, cov_colmajor16(c)) for p, c, _ in fr]
    omaps = {(k, r): oracle.GpuMap(*packed[k], r) for k in range(4) for r in (0.5, 1.0)}
    return dict(fr=fr, clouds=clouds, maps=maps, packed=packed, omaps=omaps, ctx=ctx)


def vgicp(kf, spec):
    """spec: (target, source, resolution) -> binary VGICP factors on keys (target, source)"""
    return [gpu.IntegratedVGICPFactorGPU(t, s, kf["maps"][(t, r)], kf["clouds"][s], ctx=kf["ctx"]) for t, s, r in spec]


def vgicp_restated(kf, spec, T0, priors, params):
    """the restatement on the fp64 oracle; keys are the spec's keys"""
    fac = [(kf["omaps"][(t, r)],) + kf["packed"][s] for t, s, r in spec]
    return gro.optimize(lambda f, d: (oracle.split122(oracle.linearize_gpumap(fac[f][0], *fac[f][1:], d)[0]), d),
                        lambda f, dl, d: oracle.error_gpumap(fac[f][0], *fac[f][1:], dl, d), [(t, s) for t, s, _ in spec], T0, priors, params)


SPEC3 = [(0, 1, 0.5), (0, 1, 1.0), (0, 2, 0.5), (1, 2, 0.5)]


def start3(kf, seed):
    rng = synth.rng_for(seed)
    return [kf["fr"][0][2]] + [synth.perturb(kf["fr"][k][2], rng, 0.01, 0.1) for k in (1, 2)]


def test_one_round_matches_downstream_of_the_records(kf, ctx):
    """max_iterations = 1: the device's poses against the restatement fed the records of a gpu.Sweep over the same factors in
    the same order at the same poses; everything after the sweep is fp64, so only the solve's order of operations differs.
    The step's scaled backward error (tests/solve_check.py) is held to the restatement's, a second sweep measuring the
    records' own spread."""
    T0 = start3(kf, 1400)
    priors = [(0, T0[0], 1e6)]
    facs = vgicp(kf, SPEC3)
    prob = dict(factors=facs, values=dict(enumerate(T0)), priors=priors)
    gpu.optimize_graphs([prob], params={"max_iterations": 1})  # the factors learn their inlier fractions, as in the call below
    rows0 = np.stack([rel(T0[t], T0[s]) for t, s, _ in SPEC3])
    recs = gpu.Sweep(ctx, facs).linearize(rows0)

    def lin(f, d):
        assert np.array_equal(d, rows0[f])
        return gpu.unpack_linearized(recs[f]), d

    def err(f, dl, d):
        return float(gpu.NonlinearFactorSetGPU(ctx).add([facs[f]]).error_deltas(dl[None], d[None])[0])

    with sc.systems() as seen:
        ref = gro.optimize(lin, err, [(t, s) for t, s, _ in SPEC3], T0, priors, {"max_iterations": 1})
    recs2 = gpu.Sweep(ctx, facs).linearize(rows0)
    with sc.systems() as again:
        gro.optimize(lambda f, d: (gpu.unpack_linearized(recs2[f]), d), err, [(t, s) for t, s, _ in SPEC3], T0, priors, {"max_iterations": 1})
    got = gpu.optimize_graphs([prob], params={"max_iterations": 1})[0]
    assert (got["iterations"], got["trials"], got["status"]) == (ref["iterations"], ref["trials"], ref["status"]) == (1, 1, lm.ALIGN_MAX_ITERATIONS)
    for k in range(3):
        step = np.linalg.norm(gro.se3_log(rel(T0[k], ref["T"][k])))
        diff = np.linalg.norm(gro.se3_log(rel(ref["T"][k], got["values"][k])))
        assert diff <= 1e-8 * max(step, 1e-3), (k, diff, step)
    Tg = [got["values"][k] for k in range(3)]
    sc.check("graph K 3", seen[0], sc.pose_steps(T0, Tg), sc.pose_steps(T0, ref["T"]), sc.pose_eps(T0, Tg), noise=again[0][:2])
    assert got["num_inliers"] == ref["num_inliers"]


def test_sub_mapping_lidar_only(ctx):
    """Sub-mapping's submap optimization (sub_mapping.cpp:428-452) with enable_imu false: 15 os1_64 keyframes built as
    workloads.sub_mapping_bundle builds them (levels 0.25 / 0.5 m, 105 pairs, 210 VGICP factors), drifted starts, a 1e8 prior on
    key 0 at its start pose, 20 iterations with GTSAM's default tolerances; then create_submap's merge of the keyframes."""
    w = workloads.sub_mapping_bundle(ctx, n_rays=64 * 256)
    n = len(w.poses)
    facs = w.gpu_factors(w.sets[0])
    assert len(facs) == 210
    rng = synth.rng_for(1500)
    drift = np.array([0.0, 0.0, 0.002, 0.01, -0.005, 0.0])
    T0 = [w.poses[0]] + [synth.perturb(w.poses[k] @ synth.se3_exp(k * drift), rng, 0.002, 0.02) for k in range(1, n)]
    prm = dict(GTSAM_LM, max_iterations=20)
    priors = [(0, T0[0], 1e8)]
    got = gpu.optimize_graphs([dict(factors=facs, values=dict(enumerate(T0)), priors=priors)], params=prm)[0]
    packed = [oracle.pack_cloud(p, cov_colmajor16(c)) for p, c in w.host_clouds]
    omaps = {(i, l): oracle.GpuMap(*packed[i], r) for i in range(n) for l, r in enumerate(w.resolutions)}
    fac = [(omaps[(f.target, f.level)],) + packed[f.source] for f in w.sets[0].factors]
    ref = gro.optimize(lambda f, d: (oracle.split122(oracle.linearize_gpumap(fac[f][0], *fac[f][1:], d)[0]), d),
                       lambda f, dl, d: oracle.error_gpumap(fac[f][0], *fac[f][1:], dl, d), [(f.target, f.source) for f in w.sets[0].factors], T0, priors, prm)
    assert got["status"] == ref["status"], (got, ref)
    for k in range(n):
        et, er = pose_error(got["values"][k], ref["T"][k])
        assert et < 2e-3 and er < 2e-3, (k, et, er)
        if k:
            assert pose_error(got["values"][k], w.poses[k])[0] < pose_error(T0[k], w.poses[k])[0], k
    d_got, d_ref = gro.se3_log(rel(T0[0], got["values"][0])), gro.se3_log(rel(T0[0], ref["T"][0]))
    assert np.linalg.norm(d_got - d_ref) <= 1e-3 * max(np.linalg.norm(d_ref), 1e-9) + 1e-9, (d_got, d_ref)
    print(f"sub-mapping: {got['iterations']} iterations, {got['trials']} trials, status {got['status_name']}, key 0 moved {np.linalg.norm(d_got):.3e}")
    pts, _, _ = gpu.merge_frames_gpu([got["values"][k] for k in range(n)], w.clouds, 0.25, 50000, ctx=ctx, host_outputs=True)
    assert len(pts) > 0 and np.isfinite(pts).all()


@pytest.fixture(scope="module")
def frames():
    return vo.arc_frames(8, 32 * 200)


def submap(ctx, frames, first, count=4, resolution=0.1):
    clouds = [gpu.PointCloudGPU.clone(frames[k][0], frames[k][1], ctx=ctx) for k in range(first, first + count)]
    poses = [rel(frames[first][2], frames[k][2]) for k in range(first, first + count)]
    return gpu.merge_frames_gpu(poses, clouds, resolution, ctx=ctx, host_outputs=False)[2]


def grid_restated(tgt, src, cell, r, T0, w, params):
    """the two-key problem (prior w on key 0 at T0[0], one GICP factor (0, 1)) on the fp64 grid oracle"""
    xt, ct = tgt.download()
    xs, cs = src.download()
    R = go.PointGrid(xt, ct, cell)
    return gro.optimize(lambda f, d: go.linearize(R, xs, cs, d, r), lambda f, corr, d: go.linearize(R, xs, cs, d, r, corr=corr)[0]["error"],
                        [(0, 1)], T0, [(0, T0[0], w)], params)


def test_global_mapping_between_factor(ctx, frames):
    """create_between_factors of global mapping (global_mapping.cpp:393-426): a 1e6 prior on X(0) plus a GICP point-grid factor
    (r = 0.5, lambdaInitial 1e-12, 10 iterations), solved exactly: X0^-1 X1 agrees with the fixed-target recipe within its
    test's tolerance and with the restatement, and X0's displacement -- what the fixed target neglects -- with the restatement's."""
    A, B = submap(ctx, frames, 0), submap(ctx, frames, 4)
    T_gt = rel(frames[0][2], frames[4][2])
    r = 0.5
    g = gpu.PointGridGPU(A, RECIPE_CELL * r, ctx=ctx)
    prm = {"lambda_initial": 1e-12, "max_iterations": 10}
    for k in range(2):
        X0 = synth.pose(2.0, -1.0, 0.3, 0.4)
        T0 = [X0, X0 @ synth.perturb(T_gt, synth.rng_for(960, k), 0.01, 0.1)]
        f = gpu.IntegratedGICPFactorGPU(0, 1, g, B, r, ctx=ctx)
        got = gpu.optimize_graphs([dict(factors=[f], values={0: T0[0], 1: T0[1]}, priors=[(0, X0, 1e6)])], params=prm)[0]
        fixed = gpu.align_vgicp([[gpu.IntegratedGICPFactorGPU(np.eye(4), 0, g, B, r, ctx=ctx)]], [rel(T0[0], T0[1])], params=prm)[0]
        d = rel(got["values"][0], got["values"][1])
        et, er = pose_error(d, fixed["T_target_source"])
        assert et < 0.02 and er < np.radians(0.1), (k, et, er)
        et, er = pose_error(d, T_gt)
        assert et < 0.02 and er < np.radians(0.1), (k, et, er)
        ref = grid_restated(A, B, RECIPE_CELL * r, r, T0, 1e6, prm)
        for key in (0, 1):
            et, er = pose_error(got["values"][key], ref["T"][key])
            assert et < 2e-3 and er < 2e-3, (k, key, et, er)
        d_got, d_ref = gro.se3_log(rel(X0, got["values"][0])), gro.se3_log(rel(X0, ref["T"][0]))
        assert np.linalg.norm(d_got - d_ref) <= 0.05 * np.linalg.norm(d_ref) + 1e-9, (d_got, d_ref)
        assert got["status"] == ref["status"]


@pytest.fixture(scope="module")
def modal(ctx):
    """a merged submap with covariances, its copy under a planted pose (covariances rotated with it), and the pose"""
    fr = vo.arc_frames(4, 32 * 300)
    clouds = [gpu.PointCloudGPU.clone(f[0], f[1], ctx=ctx) for f in fr]
    pts, covs, tgt = gpu.merge_frames_gpu([rel(fr[0][2], f[2]) for f in fr], clouds, 0.1, ctx=ctx)
    T_gt = synth.pose(0.4, -0.3, 0.05, np.radians(4), np.radians(1), np.radians(-1))
    Ti = synth.inv_pose(T_gt)
    moved = np.c_[pts[:, :3] @ Ti[:3, :3].T + Ti[:3, 3], np.ones(len(pts))]
    C4 = np.zeros((len(pts), 4, 4))
    C4[:, :3, :3] = np.einsum("ij,njk,lk->nil", Ti[:3, :3], np.asarray(covs).reshape(-1, 4, 4)[:, :3, :3], Ti[:3, :3])
    return tgt, gpu.PointCloudGPU.clone(moved, C4, ctx=ctx), T_gt


@pytest.mark.parametrize("kind", ["gicp", "icp"])
def test_manual_loop_closure(ctx, modal, kind):
    """the modal's align (manual_loop_close_modal.cpp:476-517): a 1e6 prior on key 0 plus GICP for 20 iterations, or ICP for
    200, on gb_merge_frames submaps, from 4 starts around a planted pose; against ground truth, the fixed-target recipe and
    (GICP) the restatement"""
    tgt, src, T_gt = modal
    r = 1.0
    g = gpu.PointGridGPU(tgt, RECIPE_CELL * r, ctx=ctx)
    make = gpu.IntegratedGICPFactorGPU if kind == "gicp" else gpu.IntegratedICPFactorGPU
    prm = dict(GTSAM_LM, max_iterations=20 if kind == "gicp" else 200)
    rng = synth.rng_for(1600)
    T0s = [[np.eye(4), synth.perturb(T_gt, rng, 0.01, 0.15)] for _ in range(4)]
    probs = [dict(factors=[make(0, 1, g, src, r, ctx=ctx)], values={0: T0[0], 1: T0[1]}, priors=[(0, np.eye(4), 1e6)]) for T0 in T0s]
    out = gpu.optimize_graphs(probs, params=prm)
    fixed = gpu.align_vgicp([[make(np.eye(4), 0, g, src, r, ctx=ctx)] for _ in T0s], [T0[1] for T0 in T0s], params=prm)
    for i, (res, fx) in enumerate(zip(out, fixed)):
        d = rel(res["values"][0], res["values"][1])
        et, er = pose_error(d, T_gt)
        assert et < 1e-3 and er < 1e-4 and res["num_inliers"] > 0.95 * src.size(), (i, et, er, res)
        et, er = pose_error(d, fx["T_target_source"])
        assert et < 1e-3 and er < 1e-4, (i, et, er)
    if kind == "gicp":
        ref = grid_restated(tgt, src, RECIPE_CELL * r, r, T0s[0], 1e6, prm)
        for key in (0, 1):
            et, er = pose_error(out[0]["values"][key], ref["T"][key])
            assert et < 2e-3 and er < 2e-3, (key, et, er)


def batch_specs(kf):
    """mixed problems: 3 keys / 4 factors / 2 levels, 2 keys / 1 level, 4 keys / 3 factors and two priors, and one problem whose
    source is 1 km away"""
    rng = synth.rng_for(1700)
    fr = kf["fr"]
    specs = []
    for i in range(12):
        kind = i % 3
        if kind == 0:
            spec, keys = SPEC3, (0, 1, 2)
        elif kind == 1:
            spec, keys = [(1, 2, 1.0)], (1, 2)
        else:
            spec, keys = [(0, 1, 0.5), (1, 2, 0.5), (2, 3, 1.0)], (0, 1, 2, 3)
        local = {k: j for j, k in enumerate(keys)}
        T0 = [fr[keys[0]][2]] + [synth.perturb(fr[k][2], rng, 0.01, 0.1) for k in keys[1:]]
        priors = [(0, T0[0], 1e6)] + ([(3, fr[3][2], 1e2)] if kind == 2 else [])
        specs.append(dict(spec=[(local[t], local[s], r) for t, s, r in spec], gkeys=keys, T0=T0, priors=priors))
    specs[4]["T0"][1] = specs[4]["T0"][1].copy()
    specs[4]["T0"][1][:3, 3] += 1000.0
    return specs, 4


def problem(kf, s):
    facs = [gpu.IntegratedVGICPFactorGPU(t, sk, kf["maps"][(s["gkeys"][t], r)], kf["clouds"][s["gkeys"][sk]], ctx=kf["ctx"]) for t, sk, r in s["spec"]]
    return dict(factors=facs, values=dict(enumerate(s["T0"])), priors=s["priors"])


def test_batch_matches_solo_runs(kf, ctx):
    specs, far = batch_specs(kf)
    probs = [problem(kf, s) for s in specs]
    launches = ctx.kernel_launches
    batch = gpu.optimize_graphs(probs)
    launches = ctx.kernel_launches - launches
    assert launches <= 4 * (max(r["trials"] for r in batch) + 1)
    d = batch[far]
    assert d["status"] == capi.ALIGN_DEGENERATE and (d["iterations"], d["trials"]) == (1, 0)
    assert all(np.array_equal(d["values"][k], specs[far]["T0"][k]) for k in d["values"])
    flipped = []
    for i, (s, r) in enumerate(zip(specs, batch)):
        if i == far:
            continue
        solo = gpu.optimize_graphs([probs[i]])[0]
        same = (r["iterations"], r["trials"], r["status"]) == (solo["iterations"], solo["trials"], solo["status"])
        for k in r["values"]:
            et, er = pose_error(r["values"][k], solo["values"][k])
            # the batch's sweep may sum a factor's fp32 partial sums in another order than the solo sweep: where a trial's error
            # ties with the current one to that rounding, the two runs may decide differently, at the noise floor only
            assert (et < 1e-6 and er < 1e-6) if same else (et < 2e-3 and er < 2e-3), (i, k, et, er, r, solo)
        if not same:
            flipped.append(i)
        assert r["status"] != capi.ALIGN_DEGENERATE
    assert len(flipped) <= len(specs) // 4, flipped
    # the 4-key problem with two priors against the restatement on the oracle
    s = specs[2]
    ref = vgicp_restated(kf, [(s["gkeys"][t], s["gkeys"][u], r) for t, u, r in s["spec"]], s["T0"], s["priors"], None)
    assert batch[2]["status"] == ref["status"]
    for k in range(4):
        et, er = pose_error(batch[2]["values"][k], ref["T"][k])
        assert et < 2e-3 and er < 2e-3, (k, et, er)


def test_launches_do_not_depend_on_the_number_of_problems(kf, ctx):
    s = batch_specs(kf)[0][0]
    counts = []
    for P in (1, 8):
        probs = [problem(kf, s) for _ in range(P)]
        launches = ctx.kernel_launches
        out = gpu.optimize_graphs(probs)
        counts.append(ctx.kernel_launches - launches)
        assert counts[-1] <= 4 * (max(r["trials"] for r in out) + 1)
        assert len({(r["iterations"], r["trials"], r["status"]) for r in out}) == 1
    assert counts[0] == counts[1], counts


def test_no_side_effects(kf):
    facs = vgicp(kf, SPEC3)
    T0 = start3(kf, 1800)
    vals = dict(enumerate(T0))
    before = [f.linearize(vals) for f in facs]
    gpu.optimize_graphs([dict(factors=facs, values=vals, priors=[(0, T0[0], 1e6)])])
    after = [f.linearize(vals) for f in facs]
    for a, b in zip(before, after):
        assert a["num_inliers"] == b["num_inliers"]
        for k in ("H_ss", "b_s", "H_tt", "b_t", "H_ts"):
            assert np.abs(a[k] - b[k]).max() <= 1e-12 * np.abs(b[k]).max(), k
        assert abs(a["error"] - b["error"]) <= 1e-12 * b["error"]


def test_invalid_inputs_are_refused_before_any_launch(kf, ctx, frames):
    L = capi.lib()
    facs = vgicp(kf, [(0, 1, 0.5), (1, 2, 0.5)])
    arr = (C.c_void_p * 2)(*[f._handle() for f in facs])
    T0 = capi.pose16(np.stack(start3(kf, 1900)))
    Z = capi.pose16(np.eye(4)[None])
    res = (capi.GraphResult * 1)()
    Tout = np.zeros_like(T0)
    good = gpu.align_params()
    keys = np.array([[0, 1], [1, 2]], np.int32)

    def call(koff=(0, 3), foff=(0, 2), fkeys=keys, factors=arr, T=T0, qoff=(0, 1), qkeys=(0,), qposes=Z, qw=(1e6,), prm=good):
        u = lambda a: np.asarray(a, np.uint64)
        return L.gb_graph_optimize(ctx.h, len(koff) - 1, capi.ptr(u(koff)), capi.ptr(T), capi.ptr(u(foff)), C.cast(factors, C.c_void_p) if factors is not None else None,
                                   capi.ptr(np.ascontiguousarray(fkeys, np.int32)), capi.ptr(u(qoff)), capi.ptr(np.asarray(qkeys, np.int32)), capi.ptr(qposes),
                                   capi.ptr(np.asarray(qw, np.float64)), C.byref(prm), capi.ptr(Tout), C.cast(res, C.c_void_p))

    grid = gpu.PointGridGPU(kf["clouds"][0], 1.05, ctx=ctx)
    mixed = (C.c_void_p * 2)(arr[0], gpu.IntegratedGICPFactorGPU(1, 2, grid, kf["clouds"][2], 1.0, ctx=ctx)._handle())
    ivox = gpu.IVoxGPU(0.5, ctx=ctx)
    ivox.insert(kf["clouds"][0])
    src = gpu.PointCloudGPU.clone(frames[1][0], frames[1][1], ctx=ctx)
    src.add_times(np.linspace(0.0, 0.1, src.size()))
    ct = (C.c_void_p * 2)(arr[0], gpu.IntegratedCT_GICPFactorGPU(1, 2, ivox, src, 1.0, ctx=ctx)._handle())
    launches = ctx.kernel_launches
    assert call(koff=(0, 1), fkeys=[[0, 0], [0, 0]]) == 1                 # K = 1
    big = capi.pose16(np.stack([np.eye(4)] * 33))
    assert call(koff=(0, 33), T=big) == 1                                  # K = 33
    assert call(foff=(0, 0)) == 1                                          # no factor
    assert call(fkeys=[[0, 1], [1, 3]]) == 1                               # key out of range
    assert call(fkeys=[[0, 1], [2, 2]]) == 1                               # target == source
    assert call(fkeys=[[0, 1], [-1, 2]]) == 1                              # negative key
    assert call(factors=(C.c_void_p * 2)(arr[0], None)) == 1               # null factor
    assert call(factors=None) == 1
    assert call(factors=mixed) == 1                                        # two classes
    assert call(factors=ct) == 1                                           # a CT factor
    bad = T0.copy()
    bad[1, 13] = np.nan
    assert call(T=bad) == 1                                                # non-finite pose
    badZ = Z.copy()
    badZ[0, 0] = np.inf
    assert call(qposes=badZ) == 1                                          # non-finite prior pose
    assert call(qw=(-1.0,)) == 1 and call(qw=(np.nan,)) == 1 and call(qw=(np.inf,)) == 1
    assert call(qkeys=(3,)) == 1                                           # prior key out of range
    assert call(prm=gpu.align_params(max_iterations=0)) == 1
    assert call(prm=gpu.align_params(lambda_factor=1.0)) == 1
    assert ctx.kernel_launches == launches
    assert call() == 0 and call(qoff=(0, 0)) == 0
    with pytest.raises(capi.GlimB200Error):
        gpu.optimize_graphs([dict(factors=[gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, kf["maps"][(0, 0.5)], kf["clouds"][1], ctx=ctx)], values={0: np.eye(4), 1: np.eye(4)})])
