"""The map editor's selection tools and point removal on the device (not a gate): a synthetic map of a few hundred submaps,
the gizmo over the whole map (gb_select_gizmo, box and sphere), the radius-outlier tool on an editor-sized window
(gb_concat_frames then gb_select_radius), and the removal of the selected points from the submaps they touch
(gb_remove_points).  Each leg's wall time is taken around calls that end in a stream synchronisation, after a warm-up call.
Prints one JSON line per leg with the card and its power limit.

    python scripts/bench_editor.py [--submaps 256] [--points 50000] [--reps 5]"""
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


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return name, limit


def timed(fn, reps):
    fn()  # warm-up: module loads, scratch growth
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return out, float(np.median(ts)), float(min(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--submaps", type=int, default=256)
    ap.add_argument("--points", type=int, default=50000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    name, limit = card()
    rng = np.random.default_rng(0)
    ctx = gpu.Context(0)
    side = int(math.ceil(math.sqrt(a.submaps)))
    frames, poses = [], []
    for k in range(a.submaps):
        # a 20 m x 20 m submap: a noisy floor and sprinkled points up to 3 m, on a grid of submaps 15 m apart
        n = a.points
        xyz = np.stack([rng.uniform(-10, 10, n), rng.uniform(-10, 10, n), rng.normal(scale=0.02, size=n)], 1)
        xyz[: n // 20, 2] = rng.uniform(0, 3, n // 20)
        T = np.eye(4)
        c, s = math.cos(0.3 * k), math.sin(0.3 * k)
        T[:2, :2] = [[c, -s], [s, c]]
        T[:3, 3] = [15.0 * (k % side), 15.0 * (k // side), 0.0]
        frames.append(gpu.PointCloudGPU.clone(np.concatenate([xyz, np.ones((n, 1))], 1), None, ctx=ctx))
        poses.append(T)
    total = a.submaps * a.points
    mid = np.array([15.0 * (side // 2), 15.0 * (side // 2), 0.0])
    base = {"card": name, "power_limit": limit, "submaps": a.submaps, "points_per_submap": a.points}

    # the gizmo: a 60 m x 40 m x 4 m box and a 25 m sphere around the middle of the map, rotated
    model = np.eye(4)
    c, s = math.cos(0.4), math.sin(0.4)
    model[:3, :3] = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]) @ np.diag([60.0, 40.0, 4.0])
    model[:3, 3] = mid
    A = np.linalg.inv(model)
    A[3] = [0, 0, 0, 1]
    for shape in ("box", "sphere"):
        B = A if shape == "box" else np.linalg.inv(np.diag([25.0, 25.0, 25.0, 1.0]) @ np.block([[np.eye(3), (mid / 25.0)[:, None]], [np.zeros((1, 3)), np.ones((1, 1))]]))
        B[3] = [0, 0, 0, 1]
        ids, med, best = timed(lambda: gpu.select_gizmo(poses, frames, B, shape, ctx=ctx), a.reps)
        touched = len(np.unique(ids >> np.uint64(32)))
        print(json.dumps({**base, "leg": f"gizmo_{shape}", "selected": int(len(ids)), "touched_submaps": touched, "median_s": med, "min_s": best,
                          "points_per_s": total / med}), flush=True)

    # the radius outliers on the window of the 3 x 3 submaps around the middle (gb_concat_frames' world-frame cloud)
    near = [k for k in range(a.submaps) if np.max(np.abs(poses[k][:2, 3] - mid[:2])) <= 15.0]
    window, wids = gpu.concat_frames([poses[k] for k in near], [frames[k] for k in near], ctx=ctx)
    for radius in (2.0, 8.0):
        r, med, best = timed(lambda: gpu.select_radius(window, mid + [0, 0, 0.5], "outliers", ctx=ctx, radius=radius), a.reps)
        print(json.dumps({**base, "leg": f"radius_outliers_r{radius:g}", "window_points": window.n, "participants": int(r["num_participants"]),
                          "selected": int(r["num_selected"]), "median_s": med, "min_s": best}), flush=True)

    # the removal of the box gizmo's selection: every submap it touches gets a new cloud (the inputs are kept)
    ids = gpu.select_gizmo(poses, frames, A, "box", ctx=ctx)
    res, med, best = timed(lambda: gpu.remove_points(frames, ids, ctx=ctx), a.reps)
    print(json.dumps({**base, "leg": "remove_points", "ids": int(len(ids)), "removed": int(res["num_removed"]), "changed_submaps": int(res["num_changed"]),
                      "touched_points": int(sum(frames[k].n for k in np.unique((ids >> np.uint64(32)).astype(np.int64)))), "median_s": med,
                      "min_s": best}), flush=True)


if __name__ == "__main__":
    main()
