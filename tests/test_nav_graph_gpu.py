"""gb_nav_graph_optimize on the H100: a call with poses only bit-identical to gb_pose_graph_optimize; one round against the
rule's restatement in tests/nav_graph_oracle.py fed the device's own sweep records; GLIM's global-mapping IMU recipe
(global_mapping.cpp:166-218) on a scaled-down global map and sub-mapping's IMU recipe (sub_mapping.cpp:218-243) against the
restatement fed the fp64 oracle; repeatability, launch counts and refusals."""
import ctypes as C

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth, workloads
from oracle import oracle
from tests import imu_oracle as io
from tests import nav_graph_oracle as ngo
from tests import solve_check as sc
from tests.util import cov_colmajor16

pytestmark = pytest.mark.gpu

PRIOR = 1e10
GTSAM_LM = {"lambda_initial": 1e-5, "lambda_factor": 10.0, "lambda_upper_bound": 1e5, "relative_error_tol": 1e-5, "absolute_error_tol": 1e-5,
            "step_translation_tol": 0.0, "step_rotation_tol": 0.0}


def between_graph(K, seed):
    rng = np.random.default_rng(seed)
    gt = [synth.se3_exp(np.concatenate([rng.normal(size=3) * 0.5, rng.normal(size=3) * 20.0])) for _ in range(K)]
    edges = [(k, k + 1) for k in range(K - 1)] + [tuple(int(x) for x in rng.choice(K, 2, replace=False)) for _ in range(K // 2)]
    bts = [(i, j, synth.perturb(synth.inv_pose(gt[i]) @ gt[j], rng, 0.01, 0.05), 100.0, None if m % 3 else 2.0) for m, (i, j) in enumerate(edges)]
    return [gt[0]] + [synth.perturb(T, rng, 0.02, 0.2) for T in gt[1:]], bts


@pytest.fixture(scope="module")
def gm32(ctx):
    """global mapping scaled down to 32 submaps, the fp64 oracle maps, and GLIM's IMU structure over an analytic trajectory"""
    w = workloads.global_mapping(ctx, n_submaps=32, laps=2, n_rays=64 * 128)
    facs = w.gpu_factors(w.sets[0])
    n = len(w.poses)
    packed = [oracle.pack_cloud(p, cov_colmajor16(c)) for p, c in w.host_clouds]
    omaps = {(i, l): oracle.GpuMap(*packed[i], r) for i in range(n) for l, r in enumerate(w.resolutions)}
    fac = [(omaps[(f.target, f.level)],) + packed[f.source] for f in w.sets[0].factors]
    keys = [(f.target, f.source) for f in w.sets[0].factors]
    return dict(w=w, facs=facs, fac=fac, keys=keys, n=n)


def glim_imu_graph(ctx, n, X_gt, seed=2200, fallback=5):
    """GLIM's enable_imu structure for n submaps: submap k has E(2k) (k > 0), E(2k+1), V(.), B(.) with the X -> E betweens, the
    rotate-velocity terms at 1e6, the bias priors and the bias between at 1e6; an ImuFactor E(2k-1), V(2k-1) -> E(2k), V(2k)
    with B(2k-1) per submap, or a velocity between at precision 1 where fewer than two samples were integrated (submap
    `fallback`).  The endpoints and velocities come from the analytic trajectory; drifted starts.
    -> (poses, velocities, biases, betweens, imu, vec, truth dicts)"""
    rng = np.random.default_rng(seed)
    bias = np.array([0.04, -0.03, 0.06, 0.003, -0.002, 0.002])
    tL = {k: 1.0 + 0.6 * k for k in range(n)}
    tR = {k: tL[k] + 0.4 for k in range(n)}
    s = io.samples(0.5, tR[n - 1] + 0.5, 200, bias)
    gap = (s[:, 0] > tR[fallback - 1] + 1e-9) & (s[:, 0] < tL[fallback] - 1e-9)
    s = s[~gap]  # no sample between submaps fallback - 1 and fallback
    ends = {}
    for k in range(n):
        for e, t in ((2 * k, tL[k]), (2 * k + 1, tR[k])):
            if e == 0:
                continue
            T, v, _, _ = io.truth(t)
            ends[e] = (T, v)
    est_bias = {e: bias + rng.normal(size=6) * 0.002 for e in ends}
    intervals = [(tR[k - 1], tL[k]) for k in range(1, n)]
    recs = gpu.imu_preintegrate(s, intervals, [est_bias[2 * k] for k in range(1, n)], ctx=ctx)  # imu_biasL, global_mapping.cpp:208
    poses_gt = {("X", k): X_gt[k] for k in range(n)}
    poses_gt.update({("E", e): T for e, (T, _) in ends.items()})
    vel_gt = {e: v for e, (_, v) in ends.items()}
    betweens, vec, imu = [], [], []
    for e in ends:
        k = e // 2
        betweens.append((("X", k), ("E", e), synth.inv_pose(X_gt[k]) @ ends[e][0], 1e6, None))
        vec.append(("rotate_velocity", ("X", k), e, X_gt[k][:3, :3].T @ ends[e][1], 1e6))
        vec.append(("bias_prior", e, None, est_bias[e], 1e6))
    for k in range(1, n):
        vec.append(("bias_between", 2 * k, 2 * k + 1, np.zeros(6), 1e6))
    for k in range(1, n):
        r = recs[k - 1]
        if r["num_integrated"] < 2:
            vec.append(("velocity_between", 2 * k - 1, 2 * k, np.zeros(3), 1.0))
        else:
            imu.append((("E", 2 * k - 1), 2 * k - 1, ("E", 2 * k), 2 * k, 2 * k - 1, r))
    assert sum(1 for v in vec if v[0] == "velocity_between") == 1 and len(imu) == n - 2
    drift = np.array([0.0, 0.0, 0.001, 0.01, -0.005, 0.0])
    poses = {("X", 0): X_gt[0]}
    poses.update({("X", k): synth.perturb(X_gt[k] @ synth.se3_exp(k * drift), rng, 0.002, 0.02) for k in range(1, n)})
    poses.update({("E", e): poses[("X", e // 2)] @ synth.inv_pose(X_gt[e // 2]) @ T for e, (T, _) in ends.items()})
    velocities = {e: v + rng.normal(size=3) * 0.05 for e, (_, v) in ends.items()}
    biases = {e: est_bias[e].copy() for e in ends}
    return poses, velocities, biases, betweens, imu, vec, (poses_gt, vel_gt, bias)


def restated(factors, poses, velocities, biases, priors, betweens, imu, vec, params):
    """the restatement on the same graph: local indices; factors = (pose keys (t, s) per factor, linearize, error) as
    nav_graph_oracle.optimize takes them"""
    lx = {k: i for i, k in enumerate(poses)}
    lv = {k: i for i, k in enumerate(velocities)}
    lb = {k: i for i, k in enumerate(biases)}
    kinds = capi.VECTOR_KINDS
    gvec = []
    for kind, a, b, z, w in vec:
        k = kinds[kind]
        da, db = {0: (lv, None), 1: (lb, None), 2: (lv, lv), 3: (lb, lb), 4: (lx, lv)}[k]
        gvec.append((k, da[a], db[b] if db is not None else None, np.asarray(z, float), w))
    graph = ngo.Graph(len(lx), len(lv), len(lb), [(lx[k], Z, w) for k, Z, w in priors],
                      [(lx[i], lx[j], Z, w * np.eye(6), 0.0) for i, j, Z, w, _ in betweens],
                      [(lx[a], lv[b], lx[c], lv[d], lb[e], io.record_of(r)) for a, b, c, d, e, r in imu], gvec)
    keys, lin, err = factors
    X0 = (np.stack(list(poses.values())), np.stack(list(velocities.values())), np.stack(list(biases.values())))
    return ngo.optimize(graph, X0, params, ([(lx[t], lx[s]) for t, s in keys], lin, err)), lx, lv, lb


def oracle_factors(fac, keys):
    """the fp64 oracle's linearization and error of each factor (fac[f] = (map, source xyz, cov6)) on pose keys (t, s)"""
    return (keys, lambda f, d: (oracle.split122(oracle.linearize_gpumap(fac[f][0], *fac[f][1:], d)[0]), d),
            lambda f, dl, d: oracle.error_gpumap(fac[f][0], *fac[f][1:], dl, d))


def recipe(ctx, g):
    """gm32's graph with GLIM's IMU structure, X keys as the factors name them -> (device arguments, restatement arguments,
    ground truth)"""
    n, w = g["n"], g["w"]
    poses, velocities, biases, betweens, imu, vec, truth = glim_imu_graph(ctx, n, w.poses)
    remap = {("X", k): k for k in range(n)}
    P = {remap.get(k, k): T for k, T in poses.items()}
    dev = dict(poses=P, velocities=velocities, biases=biases, priors=[(0, P[0], PRIOR)],
               betweens=[(remap.get(i, i), remap.get(j, j), Z, wt, h) for i, j, Z, wt, h in betweens],
               imu_terms=[(remap.get(a, a), b, remap.get(c, c), d, e, r) for a, b, c, d, e, r in imu],
               vector_terms=[(kind, remap.get(a, a) if kind == "rotate_velocity" else a, b, z, wt) for kind, a, b, z, wt in vec])
    ref = (poses, velocities, biases, [(("X", 0), poses[("X", 0)], PRIOR)], betweens, imu, vec)
    return dev, ref, truth, remap


def state_diffs(got, ref, lx, lv, lb, remap):
    """the largest pose (translation, rotation), velocity and bias differences of a device result from the restatement's"""
    dt = dr = 0.0
    for key, i in lx.items():
        d = synth.inv_pose(ref["x"][0][i]) @ got["poses"][remap.get(key, key)]
        dt, dr = max(dt, np.linalg.norm(d[:3, 3])), max(dr, np.linalg.norm(io.log3(d[:3, :3])))
    dv = max(np.linalg.norm(got["velocities"][k] - ref["x"][1][i]) for k, i in lv.items())
    db = max(np.linalg.norm(got["biases"][k] - ref["x"][2][i]) for k, i in lb.items())
    return dt, dr, dv, db


def test_poses_only_is_bit_identical_to_the_pose_graph(ctx, gm32):
    T0, bts = between_graph(40, 71)
    prm = dict(GTSAM_LM, max_iterations=20)
    a = gpu.optimize_pose_graph([], dict(enumerate(T0)), priors=[(0, T0[0], PRIOR)], betweens=bts, params=prm, ctx=ctx)
    b = gpu.optimize_nav_graph([], dict(enumerate(T0)), {}, {}, priors=[(0, T0[0], PRIOR)], betweens=bts, params=prm, ctx=ctx)
    assert (a["iterations"], a["trials"], a["status"], a["error"], a["lambda"]) == (b["iterations"], b["trials"], b["status"], b["error"], b["lambda"])
    assert all(np.array_equal(a["values"][k], b["poses"][k]) for k in a["values"])
    g = gm32
    T0 = [g["w"].poses[0]] + [synth.perturb(T, synth.rng_for(2101, k), 0.002, 0.02) for k, T in enumerate(g["w"].poses[1:])]
    a = gpu.optimize_pose_graph(g["facs"], dict(enumerate(T0)), priors=[(0, T0[0], PRIOR)], params=prm, ctx=ctx)
    b = gpu.optimize_nav_graph(g["facs"], dict(enumerate(T0)), {}, {}, priors=[(0, T0[0], PRIOR)], params=prm, ctx=ctx)
    assert (a["iterations"], a["trials"], a["status"], a["error"], a["num_inliers"]) == (b["iterations"], b["trials"], b["status"], b["error"], b["num_inliers"])
    assert all(np.array_equal(a["values"][k], b["poses"][k]) for k in a["values"])


def test_one_round_matches_downstream_of_the_records(ctx, gm32):
    """max_iterations = 1 on GLIM's global-mapping IMU recipe: the device's poses, velocities and biases against the restatement
    fed the records of a gpu.Sweep over the same factors at the same poses.  Everything after the sweep is fp64 (the IMU and
    vector terms, the pinned dofs, the solve), so only the order of operations differs: the steps agree to about the system's
    condition number times the unit roundoff, which the test computes from the restatement's first system.  The step's scaled
    backward error (tests/solve_check.py) is held to the restatement's whatever the condition number, a second sweep
    measuring the records' own spread."""
    g = gm32
    dev, refargs, _, remap = recipe(ctx, g)
    facs = g["facs"]
    call = lambda: gpu.optimize_nav_graph(facs, ctx=ctx, params={"max_iterations": 1}, **dev)
    call()  # the factors learn their inlier fractions, as in the call below
    rows0 = np.stack([synth.inv_pose(dev["poses"][t]) @ dev["poses"][s] for t, s in g["keys"]])
    recs = gpu.Sweep(ctx, facs).linearize(rows0)
    systems = []

    def lin(f, d):
        assert np.array_equal(d, rows0[f])
        return gpu.unpack_linearized(recs[f]), d

    def err(f, dl, d):
        return float(gpu.NonlinearFactorSetGPU(ctx).add([facs[f]]).error_deltas(dl[None], d[None])[0])

    keys = [(("X", t), ("X", s)) for t, s in g["keys"]]
    assemble = ngo.assemble

    def spy(*a):  # the restatement's first system, for its condition number
        out = assemble(*a)
        systems.append(out[0])
        return out

    ngo.assemble = spy
    try:
        with sc.systems() as seen:
            ref, lx, lv, lb = restated((keys, lin, err), *refargs, {"max_iterations": 1})
    finally:
        ngo.assemble = assemble
    got = call()
    assert (got["iterations"], got["trials"], got["status"]) == (ref["iterations"], ref["trials"], ref["status"]) == (1, 1, 1)
    live = [i for i in range(len(systems[0])) if np.any(systems[0][i])]  # the pinned velocity dofs have zero rows
    cond = np.linalg.cond(systems[0][np.ix_(live, live)] + 1e-5 * np.eye(len(live)))
    X0 = refargs  # each variable's step from the start, device and restatement

    def steps(res_poses, res_v, res_b):
        d = [synth_log(synth.inv_pose(X0[0][k]) @ res_poses(k)) for k in lx]
        d += [res_v(k) - X0[1][k] for k in lv]
        d += [res_b(k) - X0[2][k] for k in lb]
        return np.concatenate(d)

    d_ref = steps(lambda k: ref["x"][0][lx[k]], lambda k: ref["x"][1][lv[k]], lambda k: ref["x"][2][lb[k]])
    d_got = steps(lambda k: got["poses"][remap.get(k, k)], lambda k: got["velocities"][k], lambda k: got["biases"][k])
    err_rel = np.linalg.norm(d_got - d_ref) / np.linalg.norm(d_ref)
    vmove = max(np.linalg.norm(ref["x"][1][i] - X0[1][k]) for k, i in lv.items())
    bmove = max(np.linalg.norm(ref["x"][2][i] - X0[2][k]) for k, i in lb.items())
    print(f"one round: condition {cond:.3g}, relative step difference {err_rel:.3g}; restated velocity step {vmove:.3g}, bias step {bmove:.3g}")
    assert vmove > 1e-3 and bmove > 0.0
    assert err_rel <= max(1e-9, 1e-15 * cond), (err_rel, cond)
    recs2 = gpu.Sweep(ctx, facs).linearize(rows0)
    with sc.systems() as again:
        restated((keys, lambda f, d: (gpu.unpack_linearized(recs2[f]), d), err), *refargs, {"max_iterations": 1})
    mask = np.zeros(len(systems[0]), bool)
    mask[live] = True
    X0s = ([X0[0][k] for k in lx], [X0[1][k] for k in lv], [X0[2][k] for k in lb])
    Xg = ([got["poses"][remap.get(k, k)] for k in lx], [got["velocities"][k] for k in lv], [got["biases"][k] for k in lb])
    sc.check("nav graph gm32 IMU recipe", seen[0], sc.nav_steps(X0s, Xg), sc.nav_steps(X0s, ref["x"]), sc.nav_eps(X0s, Xg), live=mask, noise=again[0][:2])
    assert got["num_inliers"] == ref["num_inliers"]


def synth_log(T):
    return np.concatenate([io.log3(T[:3, :3]), T[:3, 3]])


def test_glim_global_mapping_imu_recipe(ctx, gm32):
    g = gm32
    n = g["n"]
    dev, refargs, (pgt, vgt, bias), remap = recipe(ctx, g)
    prm = dict(GTSAM_LM, max_iterations=20)
    before = ctx.kernel_launches
    got = gpu.optimize_nav_graph(g["facs"], params=prm, ctx=ctx, **dev)
    launches = ctx.kernel_launches - before
    assert launches <= 4 * got["trials"]
    # a second call: the solver's sums use no atomic, but the VGICP sweep's records may differ in the last bit from sweep to
    # sweep (its fp64 accumulators take the items' fp32 partial sums with atomics, exact only while their exponents stay close)
    again = gpu.optimize_nav_graph(g["facs"], params=prm, ctx=ctx, **dev)
    assert (got["iterations"], got["trials"], got["status"]) == (again["iterations"], again["trials"], again["status"])
    assert max(np.abs(got["poses"][k] - again["poses"][k]).max() for k in got["poses"]) < 1e-9
    assert max(np.abs(got["velocities"][k] - again["velocities"][k]).max() for k in got["velocities"]) < 1e-9
    assert max(np.abs(got["biases"][k] - again["biases"][k]).max() for k in got["biases"]) < 1e-9
    keys = [(("X", t), ("X", s)) for t, s in g["keys"]]
    ref, lx, lv, lb = restated(oracle_factors(g["fac"], keys), *refargs, prm)
    slots = len(dev["poses"]) + len(dev["velocities"]) + len(dev["biases"])
    dt, dr, dv, db = state_diffs(got, ref, lx, lv, lb, remap)
    vmove = max(np.linalg.norm(ref["x"][1][i] - refargs[1][k]) for k, i in lv.items())
    bmove = max(np.linalg.norm(ref["x"][2][i] - refargs[2][k]) for k, i in lb.items())
    print(f"global mapping 32 with IMU: {slots} slots, {len(g['facs'])} factors, {len(dev['imu_terms'])} IMU terms, device {got['iterations']}/"
          f"{got['trials']}/{got['status_name']}, restated {ref['iterations']}/{ref['trials']}/{ref['status']}, {launches} launches; device - restated: "
          f"pose {dt:.2g} m / {dr:.2g} rad, velocity {dv:.2g} m/s (restated moved {vmove:.2g}), bias {db:.2g} (restated moved {bmove:.2g})")
    assert slots == 4 + (n - 1) * 7
    assert (got["iterations"], got["trials"], got["status"]) == (ref["iterations"], ref["trials"], ref["status"])
    assert dt < 2e-3 and dr < 2e-3
    assert dv < 2e-3 and dv < 0.1 * vmove  # the velocities move, and as the restatement moves them
    assert db < 0.1 * bmove + 1e-7
    ev = max(np.linalg.norm(got["velocities"][e] - vgt[e]) for e in vgt)
    et = max(np.linalg.norm(got["poses"][remap.get(k, k)][:3, 3] - T[:3, 3]) for k, T in pgt.items())
    bound = max(np.linalg.norm(ref["x"][0][lx[k]][:3, 3] - T[:3, 3]) for k, T in pgt.items())
    print(f"against ground truth: translation {et:.4f} m (restated {bound:.4f} m), velocity {ev:.4f} m/s")
    assert et <= 1.5 * bound + 1e-3


def test_sub_mapping_imu_recipe(ctx):
    """sub_mapping.cpp:218-243 with enable_imu: X, V, B on each of 45 odometry frames at 5 Hz on the analytic trajectory, a 1e3
    velocity prior and a 1e6 bias prior on every frame, 1e6 bias betweens and an ImuFactor between consecutive frames (each
    integrated with the later frame's bias); 15 keyframes (every third frame) fully connected by VGICP factors at 0.25 / 0.5 m
    as workloads.sub_mapping_bundle connects them; a 1e8 prior on X(0); drifted starts.  The device against the restatement on
    the fp64 oracle."""
    off = synth.pose(0.0, -2.0, 0.0, 0.0)  # into the hall's clear corridor; a translation keeps gravity along -z
    rng = np.random.default_rng(2400)
    bias = np.array([0.05, -0.04, 0.03, 0.004, 0.002, -0.003])
    times = 1.0 + 0.2 * np.arange(45)
    T_gt = [off @ io.truth(t)[0] for t in times]
    V_gt = [io.truth(t)[1] for t in times]
    kfs = list(range(0, 45, 3))
    w = workloads.Workload("sub_mapping_imu", ctx)
    sc = synth.make_hall_scene()
    for j, i in enumerate(kfs):
        w.host_clouds.append(workloads.make_scan(sc, "os1_64", T_gt[i], synth.rng_for(311, j), n_rays=64 * 128, ctx=ctx))
        w.poses.append(T_gt[i])
    w.resolutions = [0.25, 0.5]
    w.upload()
    w.build_maps()
    factors = [workloads.Factor(a, l, cur, 0) for cur in range(1, len(kfs)) for a in range(cur) for l in range(2)]
    facs = w.gpu_factors(workloads.FactorSet(factors, np.zeros((len(factors), 4, 4))))
    assert len(facs) == 210
    key = {i: (kfs.index(i) if i in kfs else ("F", i)) for i in range(45)}  # keyframe j's pose is the factors' key j
    s = io.samples(times[0] - 0.05, times[-1] + 0.05, 200, bias)
    est_bias = [bias + rng.normal(size=6) * 0.002 for _ in times]
    recs = gpu.imu_preintegrate(s, list(zip(times[:-1], times[1:])), est_bias[1:], ctx=ctx)  # sub_mapping.cpp:231: the current frame's bias
    assert np.all(recs["num_integrated"] >= 2)
    v_est = [v + rng.normal(size=3) * 0.05 for v in V_gt]
    vec = [("velocity_prior", i, None, v_est[i], 1e3) for i in range(45)] + [("bias_prior", i, None, est_bias[i], 1e6) for i in range(45)]
    vec += [("bias_between", i - 1, i, np.zeros(6), 1e6) for i in range(1, 45)]
    imu = [(key[i - 1], i - 1, key[i], i, i - 1, recs[i - 1]) for i in range(1, 45)]
    drift = np.array([0.0, 0.0, 0.002, 0.01, -0.005, 0.0])
    poses = {key[0]: T_gt[0]}
    poses.update({key[i]: synth.perturb(T_gt[i] @ synth.se3_exp(i * drift), rng, 0.002, 0.02) for i in range(1, 45)})
    velocities = {i: v_est[i] for i in range(45)}
    biases = {i: est_bias[i].copy() for i in range(45)}
    priors = [(key[0], poses[key[0]], 1e8)]
    prm = dict(GTSAM_LM, max_iterations=20)
    got = gpu.optimize_nav_graph(facs, poses, velocities, biases, priors=priors, imu_terms=imu, vector_terms=vec, params=prm, ctx=ctx)
    packed = [oracle.pack_cloud(p, cov_colmajor16(c)) for p, c in w.host_clouds]
    omaps = {(i, l): oracle.GpuMap(*packed[i], r) for i in range(len(kfs)) for l, r in enumerate(w.resolutions)}
    fac = [(omaps[(f.target, f.level)],) + packed[f.source] for f in factors]
    ref, lx, lv, lb = restated(oracle_factors(fac, [(f.target, f.source) for f in factors]), poses, velocities, biases, priors, [], imu, vec, prm)
    dt, dr, dv, db = state_diffs(got, ref, lx, lv, lb, {})
    et = max(np.linalg.norm(got["poses"][key[i]][:3, 3] - T_gt[i][:3, 3]) for i in range(45))
    bound = max(np.linalg.norm(ref["x"][0][lx[key[i]]][:3, 3] - T_gt[i][:3, 3]) for i in range(45))
    ev = max(np.linalg.norm(got["velocities"][i] - V_gt[i]) for i in range(45))
    print(f"sub-mapping with IMU: 135 slots, 210 factors, 44 IMU terms, device {got['iterations']}/{got['trials']}/{got['status_name']}, restated "
          f"{ref['iterations']}/{ref['trials']}/{ref['status']}; device - restated: pose {dt:.2g} m / {dr:.2g} rad, velocity {dv:.2g}, bias {db:.2g}; "
          f"to ground truth: translation {et:.4f} m (restated {bound:.4f}), velocity {ev:.4f} m/s")
    assert (got["iterations"], got["trials"], got["status"]) == (ref["iterations"], ref["trials"], ref["status"])
    assert dt < 2e-3 and dr < 2e-3 and dv < 2e-3 and db < 1e-4
    assert et <= 1.5 * bound + 1e-3


def test_invalid_inputs_are_refused_before_any_launch(ctx):
    L = capi.lib()
    T0 = capi.pose16(np.stack([synth.pose(k, 0, 0, 0) for k in range(2)]))
    v0 = capi.f64(np.zeros((2, 3)))
    b0 = capi.f64(np.zeros((1, 6)))
    s = io.samples(0.0, 1.0, 200, np.zeros(6))
    rec = gpu.imu_preintegrate(s, [(0.1, 0.6)], [np.zeros(6)], ctx=ctx)
    res = capi.GraphResult()
    Tout, vout, bout = np.zeros_like(T0), np.zeros_like(v0), np.zeros_like(b0)
    good = gpu.align_params()

    def terms(**kw):
        it = gpu.imu_term_array([(0, 0, 1, 1, 0, rec[0])], {0: 0, 1: 1}, {0: 0, 1: 1}, {0: 0})
        for k, v in kw.items():
            if k.startswith("pim_"):
                it[0]["pim"][k[4:]] = v
            else:
                it[0][k] = v
        return it

    vt_good = gpu.vector_term_array([("velocity_prior", 0, None, np.zeros(3), 1.0)], {}, {0: 0, 1: 1}, {0: 0})

    def call(KX=2, KV=2, KB=1, it=None, vt=None):
        it = terms() if it is None else it
        vt = vt_good if vt is None else vt
        return L.gb_nav_graph_optimize(ctx.h, KX, capi.ptr(T0), KV, capi.ptr(v0), KB, capi.ptr(b0), 0, None, None, 0, None, None, None, 0, None,
                                       len(it), capi.ptr(it), len(vt), capi.ptr(vt), C.byref(good), capi.ptr(Tout), capi.ptr(vout), capi.ptr(bout), C.byref(res))

    before = ctx.kernel_launches
    assert call(KX=0) == 1 and call(KV=2100) == 1 and call(KX=2**64 - 1, KV=3) == 1  # a pose count that would wrap the slot sum
    assert call(it=terms(pose_j=0)) == 1 and call(it=terms(vel_j=0)) == 1 and call(it=terms(bias_i=1)) == 1 and call(it=terms(pose_i=-1)) == 1
    assert call(it=terms(pim_delta_t=0.0)) == 1
    cov = np.array(rec[0]["covariance"])
    asym = cov.copy()
    asym[0, 1] += 1e-12
    assert call(it=terms(pim_covariance=asym)) == 1 and "symmetric" in L.gb_last_error().decode()
    neg = cov.copy()
    neg[4, 4] = -1.0
    assert call(it=terms(pim_covariance=neg)) == 1 and "positive definite" in L.gb_last_error().decode()
    nan = np.array(rec[0]["preintegrated"])
    nan[2] = np.nan
    assert call(it=terms(pim_preintegrated=nan)) == 1
    bad = vt_good.copy()
    bad[0]["kind"] = 9
    assert call(vt=bad) == 1
    bad = vt_good.copy()
    bad[0]["precision"] = -1.0
    assert call(vt=bad) == 1
    bad = gpu.vector_term_array([("velocity_between", 0, 0, np.zeros(3), 1.0)], {}, {0: 0}, {})
    assert call(vt=bad) == 1
    assert ctx.kernel_launches == before
    assert call() == 0 and ctx.kernel_launches > before
