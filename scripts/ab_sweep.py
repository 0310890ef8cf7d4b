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
    ("auto notaper", {"GB_TAPER": "0"}),
    ("auto ipw10", {"GB_ITEMS_PER_WARP": "10"}),
    ("auto ipw16", {"GB_ITEMS_PER_WARP": "16"}),
    ("auto ipw24", {"GB_ITEMS_PER_WARP": "24"}),
    ("v5", {"GB_KERNEL": "5"}),
    ("v5 pipe1", {"GB_KERNEL": "5", "GB_PIPE": "1"}),
    ("v5 pipe2", {"GB_KERNEL": "5", "GB_PIPE": "2"}),
    ("v5 pipe3", {"GB_KERNEL": "5", "GB_PIPE": "3"}),
    ("v5 nostride", {"GB_KERNEL": "5", "GB_STRIDED": "0"}),
    ("v5 minrows1", {"GB_KERNEL": "5", "GB_MIN_ROWS": "1"}),
    ("v5 minrows8", {"GB_KERNEL": "5", "GB_MIN_ROWS": "8"}),
    ("v5 ipw2", {"GB_KERNEL": "5", "GB_STRIDED": "0", "GB_ITEMS_PER_WARP": "2"}),
    ("v4 T128 ipw4", {"GB_KERNEL": "4", "GB_STAGE": "128", "GB_ITEMS_PER_WARP": "4"}),
    ("v4 T128 ipw1", {"GB_KERNEL": "4", "GB_STAGE": "128", "GB_ITEMS_PER_WARP": "1"}),
    ("v4 T128 ipw2", {"GB_KERNEL": "4", "GB_STAGE": "128", "GB_ITEMS_PER_WARP": "2"}),
    ("v4 T128 ipw8", {"GB_KERNEL": "4", "GB_STAGE": "128", "GB_ITEMS_PER_WARP": "8"}),
    ("v4 T64 ipw4", {"GB_KERNEL": "4", "GB_STAGE": "64", "GB_ITEMS_PER_WARP": "4"}),
    ("v4 T64 ipw2", {"GB_KERNEL": "4", "GB_STAGE": "64", "GB_ITEMS_PER_WARP": "2"}),
]
KEYS = ["GB_KERNEL", "GB_STAGE", "GB_ITEMS_PER_WARP", "GB_TILE", "GB_STRIDED", "GB_MIN_ROWS", "GB_PIPE", "GB_TAPER"]


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
