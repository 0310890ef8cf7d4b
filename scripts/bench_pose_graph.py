"""gb_pose_graph_optimize on two workloads:

  (a) global mapping: the benchmark's global_mapping_gpu graph (256 os1_64 submaps on four laps, VGICP factors at 0.5 / 1.0 m),
      every submap drifted from ground truth, GLIM's 1e10 anchor on X(0) as a prior, 20 iterations with GTSAM's default
      tolerances and no step test: one gb_pose_graph_optimize call versus the same rule driven from the host (bench_graph.py's
      host leg: gpu.NonlinearFactorSetGPU linearize / error per round, the dense system assembled and factored by numpy);
  (b) between-only graphs at K = 256 and 1024 (a chain plus K / 2 random edges, random SPD information): the time per round
      of the call, and k_pose_graph_step's kernel time from a torch.profiler pass of its own, with the factorization's fp64
      rate computed from n^3 / 3.

Times are a host clock around synchronised calls after one warm-up pass, median of --repeats passes.  Prints one JSON line per
leg with the card's name and power limit, read in the same run.

    python scripts/bench_pose_graph.py [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_graph import GTSAM_LM, host_graph, timed  # noqa: E402
from glim_b200 import gpu, synth, workloads  # noqa: E402


def between_graph(K, seed):
    rng = np.random.default_rng(seed)
    gt = [synth.se3_exp(np.concatenate([rng.normal(size=3) * 0.5, rng.normal(size=3) * 20.0])) for _ in range(K)]
    edges = [(k, k + 1) for k in range(K - 1)] + [tuple(int(x) for x in rng.choice(K, 2, replace=False)) for _ in range(K // 2)]
    bts = []
    for i, j in edges:
        A = rng.normal(size=(6, 6))
        L = A @ A.T + 6.0 * np.eye(6)
        bts.append((i, j, synth.perturb(synth.inv_pose(gt[i]) @ gt[j], rng, 0.01, 0.05), np.triu(L) + np.triu(L, 1).T, None))
    T0 = [gt[0]] + [synth.perturb(T, rng, 0.02, 0.2) for T in gt[1:]]
    return T0, bts


def step_kernel_ms(fn):
    """k_pose_graph_step's mean kernel time over one call, from torch.profiler's CUDA activities"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if "k_pose_graph_step" in e.name]
    return (float(np.mean(times)) / 1e3 if times else None), len(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--skip-global", action="store_true")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    ctx = gpu.Context(0)

    if not a.skip_global:  # (a) the benchmark's global-mapping graph
        w = workloads.global_mapping(ctx)
        facs = w.gpu_factors(w.sets[0])
        keys = [(f.target, f.source) for f in w.sets[0].factors]
        rng = synth.rng_for(2300)
        drift = np.array([0.0, 0.0, 0.0005, 0.005, -0.0025, 0.0])
        T0 = [w.poses[0]] + [synth.perturb(w.poses[k] @ synth.se3_exp(k * drift), rng, 0.002, 0.02) for k in range(1, len(w.poses))]
        priors = [(0, T0[0], 1e10)]
        prm = dict(GTSAM_LM, max_iterations=20)
        l0 = ctx.kernel_launches
        gpu.optimize_pose_graph(facs, dict(enumerate(T0)), priors=priors, params=prm, ctx=ctx)
        launches = ctx.kernel_launches - l0
        ms, out = timed(lambda: gpu.optimize_pose_graph(facs, dict(enumerate(T0)), priors=priors, params=prm, ctx=ctx), a.repeats)
        fset = gpu.NonlinearFactorSetGPU(ctx).add(facs)
        ms_host, (T_h, it_h, tr_h, t_solve) = timed(lambda: host_graph(fset, keys, T0, priors, prm), a.repeats)
        gt_err = max(float(np.linalg.norm((synth.inv_pose(w.poses[k]) @ out["values"][k])[:3, 3])) for k in range(len(T0)))
        print(json.dumps({"leg": "global_mapping", "keys": len(T0), "factors": len(facs), "pose_graph_optimize_ms": round(ms, 3),
                          "iterations": out["iterations"], "trials": out["trials"], "status": out["status_name"], "launches": launches,
                          "ms_per_round": round(ms / max(out["trials"], 1), 3), "max_gt_translation_error_m": round(gt_err, 5),
                          "host_lm_ms": round(ms_host, 3), "host_iterations": it_h, "host_trials": tr_h, "host_solve_share": round(t_solve * 1e3 / ms_host, 4),
                          "speedup": round(ms_host / ms, 2),
                          "max_abs_pose_diff_vs_host": float(max(np.abs(out["values"][k] - T_h[k]).max() for k in range(len(T0)))), "card": card}), flush=True)

    for K in (256, 1024):  # (b) between-only graphs
        T0, bts = between_graph(K, 700 + K)
        priors = [(0, T0[0], 1e10)]
        prm = dict(GTSAM_LM, max_iterations=5)
        call = lambda: gpu.optimize_pose_graph([], dict(enumerate(T0)), priors=priors, betweens=bts, params=prm, ctx=ctx)
        ms, out = timed(call, a.repeats)
        step_ms, steps = step_kernel_ms(call)
        n = 6 * K
        N = (n + 63) // 64 * 64
        flop = N**3 / 3.0
        print(json.dumps({"leg": "between_only", "keys": K, "betweens": len(bts), "call_ms": round(ms, 3), "trials": out["trials"], "status": out["status_name"],
                          "ms_per_round": round(ms / out["trials"], 3), "step_kernel_ms": round(step_ms, 3) if step_ms else None, "step_kernels": steps,
                          "factorization_gflop": round(flop / 1e9, 2), "fp64_tflops_over_step": round(flop / (step_ms * 1e-3) / 1e12, 2) if step_ms else None,
                          "card": card}), flush=True)


if __name__ == "__main__":
    main()
