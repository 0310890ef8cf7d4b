"""gb_vgicp_align against the same Levenberg-Marquardt rule driven from the host, on two workloads:

  (a) single_pair: the 16 draws of the BASELINE single_pair workload (odometry_estimation_cpu.cpp:105-150, one 0.5 m level,
      the odometry_estimation_cpu LM settings), one problem per call;
  (b) loop candidates: the first 64 and 256 submap pairs of the global_mapping_gpu workload (two levels, 10 iterations and
      GTSAM's default tolerances as global_mapping_pose_graph.cpp:405-417 sets them, no step test), one call for the whole
      batch versus one call per candidate;
  (c) GICP on point grids (gb_point_grid_build, gb_gicp_grid_factor_create): the same 64 and 256 loop candidates with
      registration_type GICP (global_mapping_pose_graph.cpp:391-405): target = the whole submap (about 50 k points) as a
      point grid, source = 10 % of the candidate submap, r = 2.0, one factor per candidate, at the cell sizes that make the
      search half-width m = 1, 2 and 3 (the 64-candidate batch) and at the chosen one (both counts, batched versus one call
      per candidate); the grid build of one submap and of one hdl32 frame; one sub-mapping between-factor linearize
      (sub_mapping.cpp:189-211) from an hdl32 frame to the next.

The host-driven leg runs the rule of include/glim_b200.h in numpy around NonlinearFactorSetGPU.linearize_deltas / error_deltas
(one factor-set linearize and one factor-set error per round, each ending in a stream sync).  Times are a host clock around
synchronised calls after one warm-up pass, median of --repeats passes.  Prints one JSON line per leg plus the card's name
and power limit, read in the same run.

    python scripts/bench_align.py [--repeats 5] [--legs single_pair,loop,grid]
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

ODOMETRY = {}  # gb_align_default_params
LOOP = dict(max_iterations=10, absolute_error_tol=1e-5, relative_error_tol=1e-5, step_translation_tol=0.0, step_rotation_tol=0.0)


def host_align(fset, T0, P):
    """the rule of include/glim_b200.h, one factor-set linearize / error per round (the way a caller does it today)"""
    F = fset.size()
    T, lam, need_lin, it, trials = np.asarray(T0, dtype=np.float64).copy(), P.lambda_initial, True, 0, 0
    while True:
        if need_lin:
            recs = fset.linearize_deltas(np.stack([T] * F))
            H = sum(np.asarray(r["H_ss"]).reshape(6, 6).T for r in recs)
            b = sum(np.asarray(r["b_s"]) for r in recs)
            e, n = float(sum(r["error"] for r in recs)), float(sum(r["num_inliers"] for r in recs))
            it += 1
            need_lin = False
            if n == 0 and it == 1:
                return T, it, trials
        trials += 1
        A = H + lam * np.eye(6)
        try:
            np.linalg.cholesky(A)
            d = np.linalg.solve(A, -b)
            E = synth.se3_exp(d)
            Tn = T @ E
            e_new = float(fset.error_deltas(np.stack([T] * F), np.stack([Tn] * F)).sum())
            ok = e_new < e
        except np.linalg.LinAlgError:
            ok = False
        if ok:
            dt, dr = np.linalg.norm(E[:3, 3]), np.linalg.norm(d[:3])
            T, lam, need_lin, de = Tn, lam / P.lambda_factor, True, e - e_new
            done = (not (dt < 1e-10 and dr < 1e-10) and dt < P.step_translation_tol and dr < P.step_rotation_tol) or de <= P.absolute_error_tol or de / e <= P.relative_error_tol or it >= P.max_iterations
            e = e_new
        else:
            lam *= P.lambda_factor
            need_lin, done = False, lam > P.lambda_upper_bound
        if done:
            return T, it, trials


def timed(fn, repeats):
    fn()  # warm-up: module load, sweep blocks into the context's pool
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), [round(t * 1e3, 3) for t in ts]


def leg(name, ctx, fn, repeats, **extra):
    l0 = ctx.kernel_launches
    fn()
    launches = ctx.kernel_launches - l0
    med, all_ms = timed(fn, repeats)
    print(json.dumps(dict(leg=name, median_ms=round(med * 1e3, 3), runs_ms=all_ms, kernel_launches=launches, **extra)), flush=True)
    return med


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--legs", default="single_pair,loop,grid")
    args = ap.parse_args()
    legs = set(args.legs.split(","))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"card": card[0] if card else "unknown"}), flush=True)
    ctx = gpu.Context(0)

    if "single_pair" in legs:
        single_pair_leg(ctx, args)
    if legs & {"loop", "grid"}:
        g = workloads.global_mapping(ctx, use_gpu=True)
        if "loop" in legs:
            loop_leg(ctx, g, args)
        if "grid" in legs:
            grid_leg(ctx, g, args)


def single_pair_leg(ctx, args):
    # (a) single_pair
    w = workloads.single_pair(ctx, use_gpu=True)
    f = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, w.maps[0][0], w.clouds[1], ctx=ctx)
    T0s = [s.deltas[0] for s in w.sets]
    P = gpu.align_params(**ODOMETRY)
    fset = gpu.NonlinearFactorSetGPU(ctx).add([f])
    res = [gpu.align_vgicp([[f]], [T], params=P)[0] for T in T0s]
    rounds = sum(r["trials"] for r in res)
    dev = leg("single_pair/device_per_draw", ctx, lambda: [gpu.align_vgicp([[f]], [T], params=P) for T in T0s], args.repeats, problems=len(T0s), rounds=rounds)
    host = leg("single_pair/host_driven", ctx, lambda: [host_align(fset, T, P) for T in T0s], args.repeats, problems=len(T0s))
    print(json.dumps({"single_pair_speedup_device_vs_host": round(host / dev, 2)}), flush=True)


def loop_candidates(g):
    """the global-mapping graph's submap pairs in factor order -> list of [(factor, delta) per level]"""
    pairs = {}
    for fac, T in zip(g.sets[0].factors, g.sets[0].deltas):
        pairs.setdefault(fac.pair, []).append((fac, T))
    return list(pairs.values())


def loop_leg(ctx, g, args):
    # (b) loop candidates from the global-mapping graph
    P = gpu.align_params(**LOOP)
    for count in (64, 256):
        chosen = loop_candidates(g)[:count]
        problems = [[gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, g.maps[fac.target][fac.level], g.clouds[fac.source], ctx=ctx) for fac, _ in pr] for pr in chosen]
        T0 = [pr[0][1] for pr in chosen]
        sets = [gpu.NonlinearFactorSetGPU(ctx).add(pb) for pb in problems]
        res = gpu.align_vgicp(problems, T0, params=P)
        rounds = max(r["trials"] for r in res)
        st = {k: sum(r["status_name"] == k for r in res) for k in ("CONVERGED", "MAX_ITERATIONS", "LAMBDA_EXCEEDED", "DEGENERATE")}
        pts = sum(g.clouds[fac.source].n for pr in chosen for fac, _ in pr)
        batched = leg(f"loop{count}/device_batched", ctx, lambda: gpu.align_vgicp(problems, T0, params=P), args.repeats, problems=len(problems), point_factors=pts, rounds=rounds, status=st)
        seq = leg(f"loop{count}/device_sequential", ctx, lambda: [gpu.align_vgicp([pb], [T], params=P) for pb, T in zip(problems, T0)], args.repeats, problems=len(problems))
        host = leg(f"loop{count}/host_driven_sequential", ctx, lambda: [host_align(s, T, P) for s, T in zip(sets, T0)], args.repeats, problems=len(problems))
        print(json.dumps({f"loop{count}_speedup_batched_vs_sequential": round(seq / batched, 2), f"loop{count}_speedup_batched_vs_host": round(host / batched, 2)}), flush=True)


GRID_R = 2.0                               # gicp_max_correspondence_dist (config_global_mapping_pose_graph.json:40)
GRID_CELLS = {1: 2.1, 2: 1.05, 3: 0.7}     # cell size per search half-width m at r = 2.0
GRID_CHOSEN = 1                            # the m the recipes use (DESIGN.md 4.11)


def grid_leg(ctx, g, args):
    # (c) loop candidates with registration_type GICP on point grids; grid builds; a sub-mapping between factor
    P = gpu.align_params(**LOOP)
    cands = loop_candidates(g)
    rng = np.random.default_rng(0)
    sources = {}
    for pr in cands[:256]:
        s = pr[0][0].source
        if s not in sources:
            pts, cov = g.host_clouds[s]
            keep = rng.random(len(pts)) < 0.1
            sources[s] = gpu.PointCloudGPU.clone(pts[keep], cov[keep], ctx=ctx)

    def problems_for(count, cell):
        grids = {}
        probs = []
        for pr in cands[:count]:
            fac = pr[0][0]
            if fac.target not in grids:
                grids[fac.target] = gpu.PointGridGPU(g.clouds[fac.target], cell, ctx=ctx)
            probs.append([gpu.IntegratedGICPFactorGPU(np.eye(4), 0, grids[fac.target], sources[fac.source], GRID_R, ctx=ctx)])
        return probs, [pr[0][1] for pr in cands[:count]]

    for m, cell in sorted(GRID_CELLS.items()):
        problems, T0 = problems_for(64, cell)
        assert problems[0][0].search_half_width() == m
        res = gpu.align_vgicp(problems, T0, params=P)
        kept = sum(r["num_inliers"] / pb[0].source.n >= 0.5 for r, pb in zip(res, problems))
        leg(f"grid_loop64_m{m}/device_batched", ctx, lambda: gpu.align_vgicp(problems, T0, params=P), args.repeats, problems=64, cell_size=cell, half_width=m,
            rounds=max(r["trials"] for r in res), kept_at_inlier_fraction_0_5=int(kept))
    for count in (64, 256):
        problems, T0 = problems_for(count, GRID_CELLS[GRID_CHOSEN])
        res = gpu.align_vgicp(problems, T0, params=P)
        st = {k: sum(r["status_name"] == k for r in res) for k in ("CONVERGED", "MAX_ITERATIONS", "LAMBDA_EXCEEDED", "DEGENERATE")}
        pts = sum(pb[0].source.n for pb in problems)
        batched = leg(f"grid_loop{count}/device_batched", ctx, lambda: gpu.align_vgicp(problems, T0, params=P), args.repeats, problems=count, point_factors=pts,
                      rounds=max(r["trials"] for r in res), status=st, half_width=GRID_CHOSEN)
        seq = leg(f"grid_loop{count}/device_sequential", ctx, lambda: [gpu.align_vgicp([pb], [T], params=P) for pb, T in zip(problems, T0)], args.repeats, problems=count)
        print(json.dumps({f"grid_loop{count}_speedup_batched_vs_sequential": round(seq / batched, 2)}), flush=True)
    # grid builds: one submap, one hdl32 frame
    sc = synth.make_hall_scene()
    traj = synth.arc_trajectory(2)
    frames = [workloads.make_scan(sc, "hdl32", traj[k], synth.rng_for(990, k), ctx=ctx, use_gpu=True) for k in (0, 1)]
    clouds = [gpu.PointCloudGPU.clone(p, c, ctx=ctx) for p, c in frames]
    cell = GRID_CELLS[GRID_CHOSEN]
    leg("grid_build/submap", ctx, lambda: gpu.PointGridGPU(g.clouds[0], cell, ctx=ctx), args.repeats, points=g.clouds[0].n, cell_size=cell)
    leg("grid_build/hdl32_frame", ctx, lambda: gpu.PointGridGPU(clouds[0], cell, ctx=ctx), args.repeats, points=clouds[0].n, cell_size=cell)
    # one sub-mapping between factor: X(last) -> X(current), linearized once at the odometry delta
    r_sub = 1.0
    grid0 = gpu.PointGridGPU(clouds[0], r_sub * GRID_CELLS[GRID_CHOSEN] / GRID_R, ctx=ctx)
    f = gpu.IntegratedGICPFactorGPU(0, 1, grid0, clouds[1], r_sub, ctx=ctx)
    values = {0: traj[0], 1: traj[1]}
    leg("grid_sub_mapping_between/linearize", ctx, lambda: f.linearize(values), args.repeats, source_points=clouds[1].n, target_points=clouds[0].n, half_width=f.search_half_width())


if __name__ == "__main__":
    main()
