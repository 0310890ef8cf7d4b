"""The interactive viewer's plane bundle adjustment on the device (not a gate): Update (gb_plane_patch), Auto Radius
(gb_plane_auto_radius) and Create Factor (gb_plane_evm_factor_create) on 32 submaps x 250 k points around a picked corner of
a floor and a wall, and the linearization of 64 PlaneEVMFactors in one call, each timed with CUDA events on the context's
stream after a warm-up; the numpy restatement (tests/plane_ba_oracle.py) of each patch call runs beside it on the same input.
Prints one JSON line per leg with the card and its power limit.

    python scripts/bench_plane_ba.py [--submaps 32] [--points 250000] [--reps 10]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from glim_b200 import gpu, synth  # noqa: E402
from tests import plane_ba_oracle as po  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--submaps", type=int, default=32)
    ap.add_argument("--points", type=int, default=250000)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    name, limit = card()
    rng = np.random.default_rng(0)
    ctx = gpu.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    c = np.array([40.0, 20.0, 1.0])
    n = a.points
    frames, host, X = [], [], []
    for _ in range(a.submaps):
        T = np.eye(4)
        T[:3, :3] = synth.so3_exp([0, 0, rng.uniform(-np.pi, np.pi)])
        T[:3, 3] = c + np.array([rng.uniform(-20, 20), rng.uniform(-20, 20), 0.0])
        w = np.concatenate([np.column_stack([c[0] + rng.uniform(-25, 25, n // 2), c[1] + rng.uniform(-25, 25, n // 2), c[2] - 1.0 + rng.normal(0, 0.01, n // 2)]),
                            np.column_stack([c[0] + rng.normal(0, 0.01, n // 4), c[1] + rng.uniform(-25, 25, n // 4), c[2] + rng.uniform(-1, 3, n // 4)]),
                            c + rng.uniform(-25, 25, (n - n // 2 - n // 4, 3))])
        loc = ((w - T[:3, 3]) @ T[:3, :3]).astype(np.float32)
        host.append(loc)
        frames.append(gpu.PointCloudGPU.clone(np.column_stack([loc.astype(np.float64), np.ones(n)]), ctx=ctx))
        X.append(T)
    base = dict(card=name, power_limit=limit, submaps=a.submaps, map_points=a.submaps * n)

    def timed(fn):
        fn()
        ctx.synchronize()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.reps)]
        for s, e in ev:
            s.record(stream)
            r = fn()
            e.record(stream)
        ctx.synchronize()
        torch.cuda.synchronize()
        return r, float(np.median([s.elapsed_time(e) for s, e in ev]))

    def host_ms(fn):
        t0 = time.perf_counter()
        r = fn()
        return r, (time.perf_counter() - t0) * 1e3

    prm = po.params()
    got, t = timed(lambda: gpu.plane_patch(frames, X, c, ctx=ctx))
    ref, th = host_ms(lambda: po.stats(po.select(host, X, c, prm["radius"], prm["max_frame_distance"])[1]))
    same = got["num_points"] == ref[0] and bool(np.max(np.abs(got["eigenvalues"] - ref[1])) <= 1e-12 * ref[1][2])
    print(json.dumps(dict(base, leg="update", points=int(got["num_points"]), ms=round(t, 3), host_ms=round(th, 1), agrees=same)), flush=True)
    got, t = timed(lambda: gpu.plane_auto_radius(frames, X, c, ctx=ctx))
    ref, th = host_ms(lambda: po.auto_radius(host, X, c))
    same_a = got["radius"] == ref[0] and got["trials"] == ref[3]
    print(json.dumps(dict(base, leg="auto_radius", radius=got["radius"], trials=len(got["trials"]), ms=round(t, 3), host_ms=round(th, 1), agrees=same_a)), flush=True)
    f, t = timed(lambda: gpu.PlaneEVMFactorGPU(frames, X, c, ctx=ctx))
    ref, th = host_ms(lambda: po.factor_keys(host, X, c))
    same_f = f.keys.tolist() == ref[0] and f.key_points.tolist() == [len(p) for p in ref[1]]
    print(json.dumps(dict(base, leg="create_factor", keys=len(f.keys), points=int(f.num_points), ms=round(t, 3), host_ms=round(th, 1), agrees=same_f)), flush=True)
    facs = [gpu.PlaneEVMFactorGPU(frames, X, c + rng.uniform(-5, 5, 3) * [1, 1, 0], ctx=ctx, radius=float(rng.uniform(0.5, 2.0))) for _ in range(64)]
    poses = [[X[k] for k in fa.keys] for fa in facs]
    _, t = timed(lambda: gpu.linearize_plane_evm(facs, poses, ctx=ctx))
    print(json.dumps(dict(base, leg="linearize_64", keys=int(sum(len(fa.keys) for fa in facs)), ms=round(t, 3))), flush=True)
    if not (same and same_a and same_f):
        sys.exit(1)


if __name__ == "__main__":
    main()
