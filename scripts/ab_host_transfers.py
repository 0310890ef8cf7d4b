#!/usr/bin/env python
"""Paired timing of the entry points that move host arrays, across two or more builds of libglim_b200.so loaded into one
process: every round calls each build once per workload, in a rotated order, on the same inputs, so the per-round ratio to
the first build resolves differences of a few percent that separate runs of the bench scripts cannot.  Workloads:
gb_preprocess with and without host products, gb_covariances, gb_find_neighbors, gb_voxelgrid_sampling and gb_deskew on
hdl32 (60 k), os1_64 (131 k) and mid360 (500 k) scans of the hall scene.  Prints one JSON line per scan and workload with
the card and its power limit: per build the median and IQR in ms, and the median and IQR of its per-round ratio to the first.

    python scripts/ab_host_transfers.py parent/libglim_b200.so glim_b200/libglim_b200.so [--rounds 30]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from glim_b200 import capi, gpu, preprocess, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+", help="builds of libglim_b200.so (the same C ABI); ratios are to the first")
    ap.add_argument("--rounds", type=int, default=30)
    a = ap.parse_args()
    libs = []
    for path in a.libs:
        L = C.CDLL(os.path.abspath(path))
        for name, (argtypes, restype) in capi._SIGNATURES.items():
            fn = getattr(L, name)
            fn.argtypes, fn.restype = argtypes, restype
        libs.append(L)
    # the Python mirror calls capi.lib(), which returns capi._lib: each call below runs with the build that made its context
    ctxs = []
    for L in libs:
        capi._lib = L
        ctxs.append(gpu.Context(0))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    sc, traj = synth.make_hall_scene(), synth.arc_trajectory(8)
    prm = preprocess.CloudPreprocessorParams(distance_near_thresh=0.5, distance_far_thresh=100.0, downsample_resolution=0.1, k_correspondences=10)
    for sensor in ("hdl32", "os1_64", "mid360"):
        pts, tms = synth.scan(sc, sensor, traj[3], synth.rng_for(700), backend="torch")
        capi._lib = libs[0]
        nb = preprocess.find_neighbors(pts, 10, ctx=ctxs[0])
        work = {
            "preprocess_host_products": lambda c: preprocess.FramePreprocessorGPU(prm, c).preprocess(0.0, tms, pts, host_outputs=True),
            "preprocess_device_cloud": lambda c: preprocess.FramePreprocessorGPU(prm, c).preprocess(0.0, tms, pts, host_outputs=False),
            "covariances": lambda c: preprocess.CloudCovarianceEstimation(ctx=c).estimate(pts, nb),
            "find_neighbors": lambda c: preprocess.find_neighbors(pts, 10, ctx=c),
            "voxelgrid": lambda c: preprocess.voxelgrid_sampling(pts, 0.1, times=tms, ctx=c),
            "deskew": lambda c: preprocess.CloudDeskewing(ctx=c).deskew(np.eye(4), tms, pts, linear_vel=np.array([1.0, 0, 0]), angular_vel=np.array([0, 0, 0.3])),
        }
        for wname, fn in work.items():
            ts = [[] for _ in libs]
            for r in range(a.rounds + 2):  # two warm-up rounds
                for k in [(r + j) % len(libs) for j in range(len(libs))]:
                    capi._lib = libs[k]
                    t0 = time.perf_counter()
                    fn(ctxs[k])  # its device cloud is released here, by the same build
                    if r >= 2:
                        ts[k].append((time.perf_counter() - t0) * 1e3)
            base = np.array(ts[0])
            out = {"card": card, "scan": sensor, "points": len(pts), "call": wname, "rounds": a.rounds, "builds": []}
            for path, t in zip(a.libs, ts):
                q, rq = np.percentile(t, [25, 50, 75]), np.percentile(np.array(t) / base, [25, 50, 75])
                out["builds"].append({"lib": path, "median_ms": round(q[1], 3), "iqr_ms": [round(q[0], 3), round(q[2], 3)],
                                      "ratio_median": round(rq[1], 4), "ratio_iqr": [round(rq[0], 4), round(rq[2], 4)]})
            print(json.dumps(out), flush=True)
    sys.stdout.flush()
    os._exit(0)  # the contexts belong to different builds: skip the mirror's destructors, which would call the last one


if __name__ == "__main__":
    main()
