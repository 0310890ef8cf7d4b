"""GLIM's passthrough sub-mapping on the device (not a gate): one submap of 50 keyframes with the shipped parameters of
config_sub_mapping_passthrough.json, from synthetic OS1-64 scans raycast in the hall scene (glim_b200/synth.py) and preprocessed
by gb_preprocess (0.25 m voxel grid, k = 10 covariances), so that each keyframe is a realistic device cloud with covariances.

Legs, each timed with a host clock around calls that end in a stream synchronisation:
  * insert:  gb_ivox_insert of each keyframe at T_world_sensor into the module's iVox (0.5 m, 0.2 m, 64 points per cell, no
             eviction), against the number of points the map already stores (each insert regroups every stored point);
  * extract: IVoxGPU.voxel_data (gb_ivox_extract) of the 50-keyframe map at T_world_origin^-1, thinned to 50 000 points, median
             of --reps calls after a warm-up;
  * submap:  the module mirror (SubMappingPassthroughGPU) over the 50 frames, from the first insert to the submap's cloud.
There is no CPU iVox to compare against: gtsam_points is not vendored.  Prints one JSON line per leg with the card and its power
limit.

    python scripts/bench_passthrough.py [--keyframes 50] [--reps 10]"""
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
from glim_b200 import sub_mapping_passthrough as spt  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, default=50)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    name, limit = card()
    ctx = gpu.Context(0)
    params = spt.SubMappingPassthroughParams()
    assert a.keyframes <= params.max_num_keyframes
    sc = synth.make_hall_scene()
    traj = synth.arc_trajectory(a.keyframes, step=0.5)  # 0.5 m apart: every frame is a keyframe, and the voxels stay under 2.5x those of keyframe 3
    pre = preprocess.FramePreprocessorGPU(preprocess.CloudPreprocessorParams(downsample_resolution=0.25, k_correspondences=10), ctx)
    clouds = []
    for i, T in enumerate(traj):
        pts, times = synth.scan(sc, "os1_64", T, synth.rng_for(90, i))
        clouds.append(pre.preprocess(0.1 * i, times, pts, host_outputs=False)[3])
    base = {"card": name, "power_limit": limit, "keyframes": a.keyframes, "mean_frame_points": float(np.mean([c.n for c in clouds]))}

    def build_map():
        m = gpu.IVoxGPU(params.submap_voxel_resolution, params.min_dist_in_voxel, min(params.max_num_points_in_voxel, spt.IVOX_MAX_POINTS_IN_CELL), 1, 0, spt.INT_MAX,
                        ctx=ctx)
        rows = []
        for c, T in zip(clouds, traj):
            stored = m.num_points
            t0 = time.perf_counter()
            m.insert(c, T)
            rows.append((stored, time.perf_counter() - t0))
        return m, rows

    build_map()  # warm-up: module loads, scratch and pool growth
    m, rows = build_map()
    stored = np.array([r[0] for r in rows])
    ts = np.array([r[1] for r in rows])
    quart = np.array_split(np.arange(len(rows)), 4)
    print(json.dumps({**base, "leg": "insert", "median_ms": 1e3 * float(np.median(ts)), "final_points": m.num_points, "final_voxels": m.num_voxels,
                      "by_stored_points": [{"stored_points": [int(stored[q[0]]), int(stored[q[-1]])], "median_ms": 1e3 * float(np.median(ts[q]))} for q in quart]}),
          flush=True)

    T_origin_world = spt.inverse(traj[len(traj) // 2])
    seed = spt.submap_seed(0, m.num_points)
    m.voxel_data(T_origin_world, params.submap_target_num_points, seed)
    te = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        out = m.voxel_data(T_origin_world, params.submap_target_num_points, seed)
        te.append(time.perf_counter() - t0)
        out.close()
    te_all = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        out = m.voxel_data(T_origin_world)
        te_all.append(time.perf_counter() - t0)
        out.close()
    print(json.dumps({**base, "leg": "extract", "map_points": m.num_points, "target": params.submap_target_num_points,
                      "thinned_median_ms": 1e3 * float(np.median(te)), "all_points_median_ms": 1e3 * float(np.median(te_all))}), flush=True)

    tsub, submap = [], None
    for _ in range(3):
        mod = spt.SubMappingPassthroughGPU(params, ctx=ctx)
        t0 = time.perf_counter()
        for i, (c, T) in enumerate(zip(clouds, traj)):
            mod.insert_frame(i, c, T)
        got = mod.get_submaps()
        tsub.append(time.perf_counter() - t0)
        assert len(got) == 1 and len(got[0].keyframe_ids) == a.keyframes
        submap = got[0]
    print(json.dumps({**base, "leg": "submap", "median_ms": 1e3 * float(np.median(tsub)), "submap_points": submap.frame.n, "per_keyframe_ms": 1e3 * float(np.median(tsub)) / a.keyframes}),
          flush=True)


if __name__ == "__main__":
    main()
