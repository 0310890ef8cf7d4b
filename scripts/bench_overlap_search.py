"""gb_find_overlapping_submaps against the per-pair loop it replaces (GlobalMapping::find_overlapping_submaps through the shim:
one gb_overlap launch, one 4-byte read-back and one stream synchronise per gated pair):

  (a) the benchmark's global_mapping_gpu scene as bench.py builds it: 256 os1_64 submaps on four laps of a 300 m square;
  (b) 1024 submaps on 16 laps of the same loop (64 submaps per lap, as in (a)), built the same way.

Each scene uses the submaps' clouds, their coarsest voxel maps (1.0 m) and ground-truth poses, GLIM's max_implicit_loop_distance
100 m and min_implicit_loop_overlap 0.2, and first_source 0 (the viewer's "Find overlapping submaps").  After one warm-up call of
each path, the two are timed alternately in the same process, --repeats times, each call a host clock around work that ends in
a device synchronise.  Reports candidates tested, pairs found, source points probed, gb_ctx_kernel_launches per call of each
path, the median and all times, whether both paths return the same pair list and bit-identical overlaps, and the card's name and
power limit read in the same run.  One JSON file per scene under --out.

    python scripts/bench_overlap_search.py --out DIR [--repeats 3] [--scenes 256,1024]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from glim_b200 import gpu, workloads  # noqa: E402
from tests import overlap_search_oracle as oso  # noqa: E402


def scene(ctx, n_submaps):
    """(maps, clouds, poses) of bench.py's global_mapping_gpu scene (scale 1: 256 submaps on four laps), or of the same loop
    driven n_submaps / 64 times"""
    args = bench.workload_args("global_mapping_gpu", 1.0)
    args.update(n_submaps=n_submaps, laps=n_submaps // 64)
    w = workloads.global_mapping(ctx, use_gpu=True, **args)
    return [m[-1] for m in w.maps], list(w.clouds), np.stack(w.poses), args["params"]


def loop(ctx, maps, clouds, T, max_distance, min_overlap):
    """the per-pair loop of the shim: the gate on the host, then one gb_overlap per gated pair"""
    S = len(T)
    pairs, ovs = [], []
    for i in range(S):
        j = np.arange(i + 1, S)
        if not len(j):
            continue
        D = oso.deltas(T[i][None], T[j])
        for jj, d in zip(j[oso.gate(D, max_distance)], D[oso.gate(D, max_distance)]):
            ov = gpu.overlap_gpu(maps[i], clouds[jj], d, ctx=ctx)
            if ov >= min_overlap:
                pairs.append((i, int(jj)))
                ovs.append(ov)
    return np.array(pairs, np.int32).reshape(-1, 2), np.array(ovs)


def timed(ctx, fn):
    ctx.synchronize()
    l0 = ctx.kernel_launches
    t0 = time.perf_counter()
    out = fn()
    ctx.synchronize()
    return (time.perf_counter() - t0) * 1e3, ctx.kernel_launches - l0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--scenes", default="256,1024")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    ctx = gpu.Context(0)
    for S in (int(s) for s in a.scenes.split(",")):
        t_build = time.perf_counter()
        maps, clouds, T, prm = scene(ctx, S)
        md, mo = prm.max_implicit_loop_distance, prm.min_implicit_loop_overlap
        t_build = time.perf_counter() - t_build
        gated = [(i, int(j)) for i in range(S - 1) for j in np.arange(i + 1, S)[oso.gate(oso.deltas(T[i][None], T[i + 1:]), md)]]
        n = np.array([c.n for c in clouds])
        probed = int(sum(n[j] for _, j in gated))
        run_loop = lambda: loop(ctx, maps, clouds, T, md, mo)
        run_search = lambda: gpu.find_overlapping_submaps(maps, clouds, T, max_distance=md, min_overlap=mo, ctx=ctx)
        run_loop(), run_search()  # warm-up
        t_loop, t_search = [], []
        for _ in range(a.repeats):
            ms, l_loop, (p_loop, o_loop) = timed(ctx, run_loop)
            t_loop.append(ms)
            ms, l_search, (p_search, o_search) = timed(ctx, run_search)
            t_search.append(ms)
        identical = bool(np.array_equal(p_loop, p_search) and o_loop.tobytes() == o_search.tobytes())
        rec = {"scene": f"global_mapping_{S}", "submaps": S, "candidates": S * (S - 1) // 2, "gated": len(gated), "pairs_found": len(p_search),
               "source_points_probed": probed, "max_distance": md, "min_overlap": mo, "launches_loop": l_loop, "launches_search": l_search,
               "loop_ms": [round(x, 3) for x in t_loop], "search_ms": [round(x, 3) for x in t_search], "loop_ms_median": round(float(np.median(t_loop)), 3),
               "search_ms_median": round(float(np.median(t_search)), 3), "identical": identical, "scene_build_s": round(t_build, 1), "card": card}
        print(json.dumps(rec), flush=True)
        with open(os.path.join(a.out, f"overlap_search_{S}.json"), "w") as f:
            json.dump(rec, f, indent=1)
        if not identical:
            sys.exit(1)


if __name__ == "__main__":
    main()
