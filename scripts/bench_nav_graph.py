"""gb_nav_graph_optimize and gb_imu_preintegrate:

  (a) the benchmark's global_mapping_gpu graph (256 os1_64 submaps on four laps, VGICP factors at 0.5 / 1.0 m) with GLIM's IMU
      structure (global_mapping.cpp:166-218: X / E / V / B per submap, 4 + 255 * 7 = 1789 slots, n = 10734), endpoints and
      velocities from an analytic trajectory, drifted starts, GLIM's 1e10 anchor on X(0): the time of one call, its time per
      round, and k_pose_graph_step's kernel time from a torch.profiler pass of its own with the factorization's fp64 rate
      computed from N^3 / 3;
  (b) a large preintegration batch: 4096 intervals of 0.1 s over 400 Hz samples.

Times are a host clock around synchronised calls after one warm-up pass, median of --repeats passes.  Prints one JSON line per
leg with the card's name and power limit, read in the same run.  The graph is built as tests/test_nav_graph_gpu.py builds its
scaled-down one.

    python scripts/bench_nav_graph.py [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_graph import GTSAM_LM, timed  # noqa: E402
from bench_pose_graph import step_kernel_ms  # noqa: E402
from glim_b200 import gpu, synth, workloads  # noqa: E402
from tests import imu_oracle as io  # noqa: E402
from tests.test_nav_graph_gpu import glim_imu_graph  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    ctx = gpu.Context(0)

    w = workloads.global_mapping(ctx)
    facs = w.gpu_factors(w.sets[0])
    n = len(w.poses)
    poses, velocities, biases, betweens, imu, vec, (pgt, vgt, bias) = glim_imu_graph(ctx, n, w.poses, fallback=n // 2)
    remap = {("X", k): k for k in range(n)}
    P = {remap.get(k, k): T for k, T in poses.items()}
    B_ = [(remap.get(i, i), remap.get(j, j), Z, wt, h) for i, j, Z, wt, h in betweens]
    I_ = [(remap.get(x, x), b, remap.get(c, c), d, e, r) for x, b, c, d, e, r in imu]
    V_ = [(kind, remap.get(x, x) if kind == "rotate_velocity" else x, b, z, wt) for kind, x, b, z, wt in vec]
    priors = [(0, P[0], 1e10)]
    prm = dict(GTSAM_LM, max_iterations=20)
    call = lambda: gpu.optimize_nav_graph(facs, P, velocities, biases, priors=priors, betweens=B_, imu_terms=I_, vector_terms=V_, params=prm, ctx=ctx)
    l0 = ctx.kernel_launches
    call()
    launches = ctx.kernel_launches - l0
    ms, out = timed(call, a.repeats)
    step_ms, steps = step_kernel_ms(call)
    slots = len(P) + len(velocities) + len(biases)
    N = (6 * slots + 63) // 64 * 64
    flop = N**3 / 3.0
    et = max(float(np.linalg.norm(out["poses"][remap.get(k, k)][:3, 3] - T[:3, 3])) for k, T in pgt.items())
    ev = max(float(np.linalg.norm(out["velocities"][e] - vgt[e])) for e in vgt)
    print(json.dumps({"leg": "global_mapping_imu", "slots": slots, "n": 6 * slots, "N": N, "factors": len(facs), "imu_terms": len(I_), "vector_terms": len(V_),
                      "call_ms": round(ms, 3), "iterations": out["iterations"], "trials": out["trials"], "status": out["status_name"], "launches": launches,
                      "ms_per_round": round(ms / max(out["trials"], 1), 3), "step_kernel_ms": round(step_ms, 3) if step_ms else None, "step_kernels": steps,
                      "factorization_gflop": round(flop / 1e9, 2), "fp64_tflops_over_step": round(flop / (step_ms * 1e-3) / 1e12, 2) if step_ms else None,
                      "max_gt_translation_error_m": round(et, 5), "max_gt_velocity_error_mps": round(ev, 5), "card": card}), flush=True)

    I = 4096
    s = io.samples(0.0, 0.1 * I + 0.2, 400, bias)
    intervals = [(0.1 * i, 0.1 * (i + 1)) for i in range(I)]
    bz = [bias] * I
    ms, recs = timed(lambda: gpu.imu_preintegrate(s, intervals, bz, ctx=ctx), a.repeats)
    print(json.dumps({"leg": "imu_preintegrate", "intervals": I, "samples": len(s), "integrated": int(recs["num_integrated"].sum()), "call_ms": round(ms, 3),
                      "card": card}), flush=True)


if __name__ == "__main__":
    main()
