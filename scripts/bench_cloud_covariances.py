"""Covariances and normals of a device cloud from its own k nearest neighbours (not a gate): gb_cloud_estimate_covariances
against the host round trip it replaces (gb_cloud_download, gb_find_neighbors, gb_covariances, gb_cloud_upload), on the three
inputs of GLIM's call sites:
  * submap:  SubMap::load (sub_map.cpp:192-196): a 50 k-point gb_merge_frames submap of hdl32 scans in the hall scene,
             k = 10, covariances;
  * modal:   ManualLoopCloseModal::preprocess_maps (manual_loop_close_modal.cpp:338-356): the iVox map of 10 arc frames
             (resolution 2.5 m, 50 points per cell, min distance 0.5 m) from voxel_data(), k = 10, covariances and normals;
  * editor:  PointsSelector::select_points_segmentation (points_selector.cpp:785-787): the min-cut participants (planes and a
             pole, 6 m of background_mask_radius + 1 around the picked point), k = 20, normals.
Each leg is the median of --reps calls after --warmup calls, timed with a host clock around calls that end in a stream
synchronisation.  Prints one JSON line per input with the card and its power limit.

    python scripts/bench_cloud_covariances.py [--reps 20] [--warmup 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from glim_b200 import gpu, preprocess, synth  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return name, limit


def arc_frames(n_frames, n_rays):
    sc = synth.make_hall_scene()
    out = []
    for i, T in enumerate(synth.arc_trajectory(n_frames)):
        pts, _ = synth.scan(sc, "hdl32", T, synth.rng_for(510, i), n_rays=n_rays)
        _, cov = synth.with_covariances(pts, 10)
        out.append((pts, cov, T))
    return out


def submap_input(ctx):
    fr = arc_frames(10, 32 * 1000)
    frames = [gpu.PointCloudGPU.clone(p, c, ctx=ctx) for p, c, _ in fr]
    T0 = synth.inv_pose(fr[0][2])
    pts, _, _ = gpu.merge_frames_gpu([T0 @ T for _, _, T in fr], frames, 0.1, target_num_points=50000, ctx=ctx)
    return gpu.PointCloudGPU.clone(pts, ctx=ctx)


def modal_input(ctx):
    iv = gpu.IVoxGPU(2.5, min_dist_in_cell=0.5, max_points_in_cell=50, lru_horizon=1000000, ctx=ctx)
    for pts, cov, T in arc_frames(16, 32 * 400)[:10]:
        iv.insert(gpu.PointCloudGPU.clone(pts, cov, ctx=ctx), T)
    return iv.voxel_data()


def editor_input(ctx):
    rng = np.random.default_rng(7)
    parts = []
    for x in np.arange(-6.0, 6.0, 0.05):  # a floor, a wall and a pole at 5 cm
        y = np.arange(-6.0, 6.0, 0.05)
        parts.append(np.c_[np.full_like(y, x), y, np.zeros_like(y)])
        if x < 3.0:
            parts.append(np.c_[np.full(40, x), np.full(40, 2.0), np.arange(40) * 0.05])
    a = np.linspace(0, 2 * np.pi, 24, endpoint=False)
    for z in np.arange(0.0, 2.0, 0.05):
        parts.append(np.c_[0.15 * np.cos(a), 0.15 * np.sin(a), np.full_like(a, z)])
    P = np.concatenate(parts) + rng.normal(scale=0.005, size=(sum(len(p) for p in parts), 3))
    cloud = gpu.PointCloudGPU.clone(np.c_[P, np.ones(len(P))], ctx=ctx)
    inside = gpu.select_radius(cloud, [0.15, 0.0, 1.0], "inside", radius=6.0)["selected"]
    rest = np.setdiff1d(np.arange(cloud.n), inside).astype(np.uint64)
    return gpu.remove_points([cloud], rest, ctx=ctx)["frames"][0]


def host_round_trip(ctx, cloud, k, covs, normals):
    xyz, cov6 = cloud.download()
    p4 = np.c_[xyz.astype(np.float64), np.ones(len(xyz))]
    nb = preprocess.find_neighbors(p4, k, ctx=ctx)
    n4, c44 = preprocess.CloudCovarianceEstimation(ctx=ctx).estimate(p4, nb)
    return gpu.PointCloudGPU.clone(p4, c44 if covs else None, n4 if normals else None, ctx=ctx)


def median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(t)), 1e3 * float(np.percentile(t, 75) - np.percentile(t, 25))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    name, limit = card()
    ctx = gpu.Context(0)
    for label, make, k, covs, normals in (("submap", submap_input, 10, True, False), ("modal", modal_input, 10, True, True), ("editor", editor_input, 20, False, True)):
        cloud = make(ctx)
        if covs:
            dev = lambda: cloud.estimate_covariances(k, normals=normals)  # noqa: E731
        else:
            dev = lambda: cloud.estimate_normals(k)  # noqa: E731
        dev_ms, dev_iqr = median_ms(dev, a.reps, a.warmup)
        host_ms, host_iqr = median_ms(lambda: host_round_trip(ctx, cloud, k, covs, normals).close(), a.reps, a.warmup)
        print(json.dumps({"card": name, "power_limit": limit, "input": label, "points": cloud.n, "k": k, "covariances": covs, "normals": normals,
                          "device_ms": round(dev_ms, 4), "device_iqr_ms": round(dev_iqr, 4), "host_round_trip_ms": round(host_ms, 4),
                          "host_round_trip_iqr_ms": round(host_iqr, 4), "speedup": round(host_ms / dev_ms, 2)}), flush=True)


if __name__ == "__main__":
    main()
