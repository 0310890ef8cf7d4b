#!/usr/bin/env python
"""What does ONE rank's share of the global-mapping sweep cost on its own?  Runs, on one GPU, the shard every rank of an
N-GPU job would run (same partition as bench.py, calibrated by measured inliers; plain slab instead of the peer slab) and
prints the per-shard kernel times next to T(N=1)/N.  Separates the size-regime loss of the sweep kernel from the cost of the
NVLink exchange in the multi-GPU numbers.
usage: python scripts/shard_emulate.py [N ...]   env: AB_CONFIGS="label=K1:V1;K2:V2,label2=..." for kernel knobs"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

KEYS = ["GB_KERNEL", "GB_ITEMS_PER_WARP", "GB_TILE", "GB_TAPER", "GB_TAPER_A", "GB_TAPER_B"]


def main():
    ncu_mode = len(sys.argv) > 1 and sys.argv[1] == "--one"  # --one WORLD RANK: launch that shard a few times (for ncu) and exit
    worlds = [int(a) for a in sys.argv[1:]] if not ncu_mode else [int(sys.argv[2])]
    worlds = worlds or [1, 8]
    cfgs = [("auto", {})]
    if os.environ.get("AB_CONFIGS"):
        cfgs = []
        for c in os.environ["AB_CONFIGS"].split(","):
            label, _, kv = c.partition("=")
            cfgs.append((label, dict(x.split(":") for x in kv.split(";") if x)))
    env = bench.Env()
    from glim_b200 import gpu, multi_gpu
    from glim_b200.capi import GB_SLAB_STRIDE

    w = bench.build_workload("global_mapping_gpu", env.ctx, 1.0, use_gpu=True)
    sizes = [len(c[0]) for c in w.host_clouds]
    fset = w.sets[0]
    num_pairs = max(f.pair for f in fset.factors) + 1

    def make(mine):
        sub = type(fset)([fset.factors[k] for k in mine], fset.deltas[mine])
        sw = gpu.Sweep(env.ctx, w.gpu_factors(sub), pair_index=[f.pair for f in sub.factors])
        slab = torch.zeros((num_pairs, GB_SLAB_STRIDE), dtype=torch.float32, device=env.dev)
        sw.attach_slab(slab.data_ptr(), num_pairs)
        sw.set_poses(sub.deltas)
        sw._slab = slab
        return sw

    full = make(list(range(len(fset.factors))))
    full.launch()
    inl = full.fetch()["num_inliers"]
    del full
    for label, e in cfgs:
        for k in KEYS:
            os.environ.pop(k, None)
        os.environ.update(e)
        t1 = None
        for world in worlds:
            f_rank, _ = multi_gpu.shard_factors(fset.factors, sizes, world, pair_cost=w.notes.get("_pair_overlap"), factor_inliers=inl if world > 1 else None) if world > 1 else (np.zeros(len(fset.factors), dtype=np.int64), None)
            times, items = [], []
            if ncu_mode:
                sw = make([k for k in range(len(fset.factors)) if f_rank[k] == int(sys.argv[3])])
                for _ in range(6):
                    sw.launch()
                torch.cuda.synchronize()
                return
            for r in range(world):
                sw = make([k for k in range(len(fset.factors)) if f_rank[k] == r])
                for _ in range(4):
                    sw.launch()
                ms, _, _, _ = env.timed(sw.launch, 20, False)
                times.append(ms / 20)
                items.append(int(sw.num_tiles))
                del sw
            if world == 1:
                t1 = times[0]
            print(json.dumps({"config": label, "world": world, "shard_ms": [round(t, 4) for t in times], "max": round(max(times), 4), "mean": round(float(np.mean(times)), 4),
                              "ideal": None if t1 is None else round(t1 / world, 4), "eff_max": None if t1 is None else round(t1 / world / max(times), 3),
                              "eff_mean": None if t1 is None else round(t1 / world / float(np.mean(times)), 3), "items": items[:2]}), flush=True)


if __name__ == "__main__":
    main()
