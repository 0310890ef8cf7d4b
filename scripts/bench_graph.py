"""gb_graph_optimize against the same Levenberg-Marquardt rule driven from the host, on two workloads:

  (a) sub-mapping: the sub_mapping_gpu workload (15 os1_64 keyframes, 105 pairs x 2 levels = 210 VGICP factors), every
      keyframe drifted from ground truth, a 1e8 prior on key 0, 20 iterations with GTSAM's default tolerances and no step test
      (sub_mapping.cpp:428-452): one gb_graph_optimize call versus the host-driven rule;
  (b) loop closures: 64 two-key problems (a 1e6 prior on key 0 and one GICP point-grid factor, r = 1.0, 20 iterations, as
      manual_loop_close_modal.cpp:476-517) in one call versus one call per problem.

The host-driven leg runs the rule of include/glim_b200.h in numpy around NonlinearFactorSetGPU.linearize_deltas /
error_deltas: one factor-set linearize per accepted step and one factor-set error per trial, each ending in a stream sync, the
6K x 6K system assembled and solved by numpy -- what GTSAM's LM does over the factor-set hook.  It reports its time per round
and the share of its dense solve.  Times are a host clock around synchronised calls after one warm-up pass, median of --repeats
passes.  Prints one JSON line per leg plus the card's name and power limit, read in the same run.

    python scripts/bench_graph.py [--repeats 5] [--n-rays 131072]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from glim_b200 import gpu, synth, workloads  # noqa: E402

GTSAM_LM = dict(lambda_initial=1e-5, lambda_factor=10.0, lambda_upper_bound=1e5, relative_error_tol=1e-5, absolute_error_tol=1e-5,
                step_translation_tol=0.0, step_rotation_tol=0.0)


def se3_log(T):
    from scipy.spatial.transform import Rotation

    w = Rotation.from_matrix(T[:3, :3]).as_rotvec()
    th = np.linalg.norm(w)
    K = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    Jl = np.eye(3) + K / 2.0 + K @ K / 6.0 if th < 1e-6 else np.eye(3) + (1 - np.cos(th)) / th**2 * K + (th - np.sin(th)) / th**3 * K @ K
    return np.concatenate([w, np.linalg.solve(Jl, T[:3, 3])])


def prior_terms(T, Z, w):
    r = se3_log(synth.inv_pose(Z) @ T)
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = -np.array([[0.0, -r[2], r[1]], [r[2], 0.0, -r[0]], [-r[1], r[0], 0.0]])
    A[3:, :3] = -np.array([[0.0, -r[5], r[4]], [r[5], 0.0, -r[3]], [-r[4], r[3], 0.0]])
    J, P, f = np.eye(6), np.eye(6), 1.0
    for k in range(1, 30):
        P, f = P @ A, f * (k + 1)
        J = J + P / f
    J = np.linalg.inv(J)
    return w * r @ r, w * J.T @ J, w * J.T @ r


def host_graph(fset, keys, T0, priors, prm):
    """the rule of include/glim_b200.h driven from the host -> (T, iterations, trials, seconds in the dense solve)"""
    K, F = len(T0), len(keys)
    T = [np.asarray(x, dtype=np.float64).copy() for x in T0]
    lam, need_lin, it, trials, t_solve = prm["lambda_initial"], True, 0, 0, 0.0
    rows = lambda Ts: np.stack([synth.inv_pose(Ts[t]) @ Ts[s] for t, s in keys])
    while True:
        if need_lin:
            lin_rows = rows(T)
            recs = fset.linearize_deltas(lin_rows)
            H, b = np.zeros((6 * K, 6 * K)), np.zeros(6 * K)
            for (t, s), r in zip(keys, recs):
                Tt, Ss = slice(6 * t, 6 * t + 6), slice(6 * s, 6 * s + 6)
                Htt, Hss, Hts = (np.asarray(r[k]).reshape(6, 6).T for k in ("H_tt", "H_ss", "H_ts"))
                H[Tt, Tt] += Htt
                H[Ss, Ss] += Hss
                H[Tt, Ss] += Hts
                H[Ss, Tt] += Hts.T
                b[Tt] += r["b_t"]
                b[Ss] += r["b_s"]
            e, n = float(recs["error"].sum()), float(recs["num_inliers"].sum())
            for k, Z, w in priors:
                ep, Hp, bp = prior_terms(T[k], Z, w)
                H[6 * k:6 * k + 6, 6 * k:6 * k + 6] += Hp
                b[6 * k:6 * k + 6] += bp
                e += ep
            it += 1
            need_lin = False
            if n == 0 and it == 1:
                return T, it, trials, t_solve
        trials += 1
        t0 = time.perf_counter()
        A = H + lam * np.eye(6 * K)
        try:
            L = np.linalg.cholesky(A)
            d = np.linalg.solve(L.T, np.linalg.solve(L, -b))
            ok = True
        except np.linalg.LinAlgError:
            ok = False
        t_solve += time.perf_counter() - t0
        status = None
        if ok:
            Tn = [T[k] @ synth.se3_exp(d[6 * k:6 * k + 6]) for k in range(K)]
            e_new = float(fset.error_deltas(lin_rows, rows(Tn)).sum()) + sum(prior_terms(Tn[k], Z, w)[0] for k, Z, w in priors)
        if ok and e_new < e:
            T, lam, need_lin = Tn, lam / prm["lambda_factor"], True
            if e - e_new <= prm["absolute_error_tol"] or (e - e_new) / e <= prm["relative_error_tol"] or it >= prm["max_iterations"]:
                status = 0
            e = e_new
        else:
            lam *= prm["lambda_factor"]
            if lam > prm["lambda_upper_bound"]:
                status = 2
        if status is not None:
            return T, it, trials, t_solve


def timed(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--n-rays", type=int, default=None, help="os1_64 rays per keyframe (default: the workload's 131072)")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    ctx = gpu.Context(0)

    # (a) sub-mapping
    w = workloads.sub_mapping_bundle(ctx, n_rays=a.n_rays)
    n = len(w.poses)
    facs = w.gpu_factors(w.sets[0])
    keys = [(f.target, f.source) for f in w.sets[0].factors]
    rng = synth.rng_for(1500)
    drift = np.array([0.0, 0.0, 0.002, 0.01, -0.005, 0.0])
    T0 = [w.poses[0]] + [synth.perturb(w.poses[k] @ synth.se3_exp(k * drift), rng, 0.002, 0.02) for k in range(1, n)]
    priors = [(0, T0[0], 1e8)]
    prm = dict(GTSAM_LM, max_iterations=20)
    prob = dict(factors=facs, values=dict(enumerate(T0)), priors=priors)
    l0 = ctx.kernel_launches
    gpu.optimize_graphs([prob], params=prm)
    launches = ctx.kernel_launches - l0
    ms, out = timed(lambda: gpu.optimize_graphs([prob], params=prm)[0], a.repeats)
    fset = gpu.NonlinearFactorSetGPU(ctx).add(facs)
    ms_host, (T_h, it_h, tr_h, t_solve) = timed(lambda: host_graph(fset, keys, T0, priors, prm), a.repeats)
    dev = max(np.abs(out["values"][k] - T_h[k]).max() for k in range(n))
    print(json.dumps({"leg": "sub_mapping", "keys": n, "factors": len(facs), "points_per_keyframe": int(np.mean([len(p) for p, _ in w.host_clouds])),
                      "graph_optimize_ms": round(ms, 3), "iterations": out["iterations"], "trials": out["trials"], "status": out["status_name"],
                      "launches": launches, "host_lm_ms": round(ms_host, 3), "host_iterations": it_h, "host_trials": tr_h,
                      "host_ms_per_round": round(ms_host / max(tr_h, 1), 3), "host_solve_share": round(t_solve * 1e3 / ms_host, 4),
                      "speedup": round(ms_host / ms, 2), "max_abs_pose_diff": float(dev), "card": card}))

    # (b) 64 two-key loop closures
    clouds = w.clouds[:8]
    probs = []
    r = 1.0
    grids = [gpu.PointGridGPU(clouds[k], 1.05 * r, ctx=ctx) for k in range(4)]
    rng = synth.rng_for(1600)
    for i in range(64):
        t, s = i % 4, 4 + (i // 4) % 4
        T_ts = synth.inv_pose(w.poses[t]) @ w.poses[s]
        f = gpu.IntegratedGICPFactorGPU(0, 1, grids[t], clouds[s], r, ctx=ctx)
        probs.append(dict(factors=[f], values={0: np.eye(4), 1: synth.perturb(T_ts, rng, 0.01, 0.1)}, priors=[(0, np.eye(4), 1e6)]))
    prm = dict(GTSAM_LM, max_iterations=20)
    l0 = ctx.kernel_launches
    batch = gpu.optimize_graphs(probs, params=prm)
    launches = ctx.kernel_launches - l0
    ms_b, batch = timed(lambda: gpu.optimize_graphs(probs, params=prm), a.repeats)
    ms_s, _ = timed(lambda: [gpu.optimize_graphs([p], params=prm) for p in probs], a.repeats)
    print(json.dumps({"leg": "loop_closures", "problems": len(probs), "batched_ms": round(ms_b, 3), "per_problem_calls_ms": round(ms_s, 3),
                      "speedup": round(ms_s / ms_b, 2), "launches": launches, "max_trials": max(x["trials"] for x in batch),
                      "max_iterations": max(x["iterations"] for x in batch), "card": card}))


if __name__ == "__main__":
    main()
