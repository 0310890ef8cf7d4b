#!/usr/bin/env python
"""A/B of sweep-kernel configurations on the BASELINE workloads, one process, one workload build per workload.
usage: python scripts/ab_sweep.py [workload ...]   (configs are env-variable sets read by gb_sweep_create)"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

CONFIGS = [
    ("v3", {"GB_KERNEL": "3"}),
    ("auto", {}),
    ("v5", {"GB_KERNEL": "5"}),
]
KEYS = ["GB_KERNEL"]


def main():
    names = sys.argv[1:] or ["odometry_gpu", "single_pair", "sub_mapping_gpu", "livox_stress", "global_mapping_gpu"]
    cfgs = CONFIGS
    if os.environ.get("AB_CONFIGS"):
        want = os.environ["AB_CONFIGS"].split(",")
        cfgs = [c for c in CONFIGS if c[0] in want]
    env = bench.Env()
    from glim_b200 import gpu

    for name in names:
        t0 = time.time()
        w = bench.build_workload(name, env.ctx, 1.0, use_gpu=True)
        sizes = [len(c[0]) for c in w.host_clouds]
        small = sum(sizes) * 36 <= bench.L2_BYTES
        ref_inl = None
        for label, e in cfgs:
            for k in KEYS:
                os.environ.pop(k, None)
            os.environ.update(e)
            sweeps = []
            for fset in w.sets:
                sw = gpu.Sweep(env.ctx, w.gpu_factors(fset))
                sw.set_poses(fset.deltas)
                sweeps.append(sw)
            pf = sum(s.point_factors for s in sweeps)
            by = sum(s.algorithmic_bytes for s in sweeps)

            def step():
                for s in sweeps:
                    s.launch()

            step()
            for sw in sweeps:
                sw.fetch()
            for _ in range(5):
                step()
            steps = 30
            ms, _, _, _ = env.timed(step, steps, small)
            inl = np.concatenate([s.fetch()["num_inliers"] for s in sweeps])
            h = np.concatenate([s.fetch()["H_ss"].sum(axis=1) for s in sweeps])
            if ref_inl is None:
                ref_inl, ref_h = inl, h
            ok = bool(np.array_equal(inl, ref_inl)) and bool(np.allclose(h, ref_h, rtol=1e-4))
            per = ms / steps / len(sweeps)
            print(json.dumps({"workload": name, "config": label, "M_pf_s": round(pf / (ms / steps * 1e-3) / 1e6), "us_per_launch": round(per * 1e3, 2), "frac": round(by / len(sweeps) / (per * 1e-3) / 1e9 / 6582.8, 3),
                              "items_grid": [int(sweeps[0].num_tiles), int(sweeps[0].grid)], "same_as_first": ok}), flush=True)
            del sweeps
        print(f"# {name}: {time.time() - t0:.0f} s", flush=True)
        del w


if __name__ == "__main__":
    main()
