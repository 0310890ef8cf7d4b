"""Map segmentation on the device (not a gate): an editor-sized window cut out of a synthetic map of a few hundred submaps
by gb_concat_frames, then gb_region_growing at the editor's typical settings, and gb_min_cut with the editor's defaults on the
same window, each against the host restatement (tests/segment_oracle.py, tests/mincut_oracle.py) on the
same input.  Prints one JSON line per leg with the card and its power limit.

    python scripts/bench_segment.py [--submaps 300] [--points 10000] [--reps 5]"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from glim_b200 import gpu  # noqa: E402
from tests import mincut_oracle as mo  # noqa: E402
from tests import segment_oracle as so  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--submaps", type=int, default=300)
    ap.add_argument("--points", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    name, limit = card()
    rng = np.random.default_rng(0)
    ctx = gpu.Context(0)
    side = int(math.ceil(math.sqrt(a.submaps)))
    poses, frames, host = [], [], []
    for k in range(a.submaps):
        T = np.eye(4)
        T[:3, 3] = [15.0 * (k % side), 15.0 * (k // side), 0.0]
        P = np.concatenate([rng.uniform(-10, 10, (a.points, 2)), rng.normal(scale=0.01, size=(a.points, 1))], axis=1).astype(np.float32)
        N = np.tile(np.array([0, 0, 1], np.float32), (a.points, 1))
        poses.append(T)
        host.append((P, None, N))
        frames.append(gpu.PointCloudGPU.clone(np.concatenate([P, np.ones((a.points, 1), np.float32)], axis=1).astype(np.float64), None,
                                              np.concatenate([N, np.zeros((a.points, 1), np.float32)], axis=1).astype(np.float64), ctx=ctx))
    picked = np.array([15.0 * (side // 2), 15.0 * (side // 2), 0.0])
    cell, w = 2.0, 5
    c = np.floor(picked / cell).astype(int)
    window = (cell, tuple(c - w), tuple(c + w))
    prm = dict(distance_threshold=0.5, angle_threshold=math.radians(10), dilation_radius=1.0)
    base = dict(card=name, power_limit=limit, submaps=a.submaps, map_points=a.submaps * a.points)

    def timed(fn):
        fn()
        ctx.synchronize()
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            r = fn()
            ctx.synchronize()
            ts.append(time.perf_counter() - t0)
        return r, float(np.median(ts)) * 1e3

    (cloud, ids), t_cat = timed(lambda: gpu.concat_frames(poses, frames, window=window, ctx=ctx))
    print(json.dumps(dict(base, leg="concat_frames", window_points=cloud.size(), ms=round(t_cat, 3))), flush=True)
    got, t_rg = timed(lambda: gpu.region_growing(cloud, picked, ctx=ctx, **prm))
    print(json.dumps(dict(base, leg="region_growing", window_points=cloud.size(), selected=int(got["num_selected"]), ms=round(t_rg, 3))), flush=True)
    t0 = time.perf_counter()
    ref_cat = so.concat_frames(poses, host, window)
    ref = so.region_growing(ref_cat["xyz"], ref_cat["normals"], picked, **prm)
    t_host = (time.perf_counter() - t0) * 1e3
    same = bool(np.array_equal(ids[got["selected"]], ref_cat["ids"][ref["selected"]]))
    print(json.dumps(dict(base, leg="host_oracle", window_points=len(ref_cat["xyz"]), ms=round(t_host, 3), identical=same)), flush=True)
    # the editor's default method on the same window, picked at the same point, with the editor's radii and weight
    mc, t_mc = timed(lambda: gpu.min_cut(cloud, picked, ctx=ctx))
    print(json.dumps(dict(base, leg="min_cut", window_points=cloud.size(), participants=int(mc["num_points"]), edges=int(mc["num_edges"]),
                          rounds=int(mc["rounds"]), selected=int(mc["num_selected"]), ms=round(t_mc, 3))), flush=True)
    t0 = time.perf_counter()
    ref_mc = mo.min_cut(ref_cat["xyz"], ref_cat["normals"], picked)
    t_host = (time.perf_counter() - t0) * 1e3
    same_mc = bool(np.array_equal(ids[mc["selected"]], ref_cat["ids"][ref_mc["selected"]]))
    print(json.dumps(dict(base, leg="min_cut_host_oracle", participants=int(ref_mc["num_points"]), ms=round(t_host, 3), identical=same_mc)), flush=True)
    if not (same and same_mc):
        sys.exit(1)


if __name__ == "__main__":
    main()
