"""How the VGICP sweep's first hash probe ends, on the CPU: for sample pairs of the global-mapping workload (bench.py's default,
256 submaps x 50 k points, four laps of a 300 m loop), the target's voxel tables at both levels are built with the oracle
(oracle.GpuMap: the device table, bit for bit) and every source point, moved by the pair's perturbed relative pose and taken in
the device cloud's Morton order, is looked up the way phase A of k_vgicp_sweep3 / 5 does.  Per pair kind and level it prints the
fraction of points whose FIRST bucket holds their voxel (hit), is empty (miss) or holds another voxel (collision: the lane
gathers the second bucket), the fraction that needs a third bucket or more, and the fraction of 32-point warp rows with at
least one colliding lane (a row whose lanes all resolve on the first bucket skips the second gather round).

    python scripts/probe_stats.py [--anchors 3] [--seed 0]

Needs oracle/libglim_oracle.so (built by __graft_entry__.build()); no GPU.
"""
import argparse
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from glim_b200 import synth, workloads  # noqa: E402
from oracle import oracle  # noqa: E402

N_SUBMAPS, LAPS, SIDE = 256, 4, 300.0  # bench.py workload_args("global_mapping_gpu", 1.0)
PER_LAP = N_SUBMAPS // LAPS
KINDS = {"next submap": 1, "same place, next lap": PER_LAP, "two laps apart": 2 * PER_LAP}
M32 = np.uint64(0xFFFFFFFF)


def c16(cov):
    return np.ascontiguousarray(np.swapaxes(cov, 1, 2)).reshape(len(cov), 16)


def morton_order(xyz):
    """The device cloud's storage order (k_morton_keys + a stable radix sort): Morton key of the 1/16 m cell, non-finite last."""
    f = np.floor(xyz.astype(np.float32) * np.float32(16.0))
    ok = np.isfinite(xyz).all(1) & (np.abs(f) < 1048576.0).all(1)
    c = np.where(ok[:, None], f, 0).astype(np.int64) + (1 << 20)
    key = np.zeros(len(xyz), np.uint64)
    for bit in range(21):
        for axis, shift in ((0, 2), (1, 1), (2, 0)):
            key |= ((c[:, axis].astype(np.uint64) >> np.uint64(bit)) & np.uint64(1)) << np.uint64(3 * bit + shift)
    key[~ok] = np.uint64(0xFFFFFFFFFFFFFFFF)
    return np.argsort(key, kind="stable")


def gb_hash(c):
    x = c.astype(np.int64).astype(np.uint64) & M32
    return ((x[:, 0] * np.uint64(73856093)) & M32) ^ ((x[:, 1] * np.uint64(19349669)) & M32) ^ ((x[:, 2] * np.uint64(83492791)) & M32)


def probe(table, xyz, delta):
    """Per point: number of buckets gb_lookup reads before it stops (1 = resolved on the first), and whether it hit."""
    R, t = delta[:3, :3].astype(np.float32), delta[:3, 3].astype(np.float32)
    q = xyz @ R.T + t  # fp32; the kernel's FMA order can move a point on a voxel face: statistics only
    c = np.floor(q * (np.float32(1.0) / np.float32(table.resolution))).astype(np.int64)
    h = gb_hash(c)
    B = table.buckets
    mask = np.uint64(len(B) - 1)
    reads = np.zeros(len(xyz), np.int64)
    hit = np.zeros(len(xyz), bool)
    open_ = np.isfinite(q).all(1)
    for k in range(10):  # max_scan of GaussianVoxelMapGPU
        if not open_.any():
            break
        b = B[((h + np.uint64(k)) & mask).astype(np.int64)]
        reads[open_] += 1
        empty = b[:, 3] < 0
        match = ~empty & (b[:, :3] == c).all(1)
        hit |= open_ & match
        open_ &= ~(empty | match)
    return reads, hit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--anchors", type=int, default=3, help="pairs per kind (sources spread over the second lap)")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    t0 = time.time()
    p = workloads.GlobalMappingParams()
    resolutions = [p.submap_voxel_resolution * p.submap_voxelmap_scaling_factor**l for l in range(p.submap_voxelmap_levels)]
    sc = synth.make_blocks_scene()
    traj = synth.loop_trajectory(PER_LAP, LAPS, side=SIDE)
    rng = np.random.default_rng(args.seed)
    clouds, tables = {}, {}

    def cloud(i):
        if i not in clouds:
            pts, cov = workloads.make_scan(sc, "os1_64", traj[i], synth.rng_for(401, i), max_points=p.submap_target_num_points)
            xyz, cov6 = oracle.pack_cloud(pts, c16(cov))
            clouds[i] = (xyz, cov6)
        return clouds[i]

    print(f"{'pair kind':<22} {'level':>6} {'points':>8} {'hit':>6} {'empty':>6} {'collide':>8} {'>2 buckets':>11} {'rows w/ collision':>18}")
    for kind, gap in KINDS.items():
        sums = {}
        for a in range(args.anchors):
            src = PER_LAP + (a * PER_LAP) // max(1, args.anchors) + int(rng.integers(PER_LAP // max(1, args.anchors)))
            tgt = src - gap
            xyz = cloud(src)[0]
            xyz = xyz[morton_order(xyz)]
            delta = synth.perturb(synth.inv_pose(traj[tgt]) @ traj[src], synth.rng_for(402, tgt, src), 0.02, 0.2)
            for lvl, res in enumerate(resolutions):
                if (tgt, lvl) not in tables:
                    tables[(tgt, lvl)] = oracle.GpuMap(*cloud(tgt), res)
                reads, hit = probe(tables[(tgt, lvl)], xyz, delta)
                first_hit = hit & (reads == 1)
                empty = (reads == 1) & ~hit
                collide = reads >= 2
                nw = len(xyz) // 32
                rows = collide[: nw * 32].reshape(nw, 32).any(1)
                s = sums.setdefault(lvl, np.zeros(7))
                s += [len(xyz), first_hit.sum(), empty.sum(), collide.sum(), (reads >= 3).sum(), rows.sum(), nw]
        for lvl, s in sorted(sums.items()):
            n = s[0]
            print(f"{kind:<22} {resolutions[lvl]:>5.1f}m {int(n):>8d} {s[1] / n:>6.3f} {s[2] / n:>6.3f} {s[3] / n:>8.3f} {s[4] / n:>11.4f} {s[5] / max(1, s[6]):>18.3f}")
    print(f"({args.anchors} pair(s) per kind, {len(clouds)} clouds, {time.time() - t0:.0f} s)")


if __name__ == "__main__":
    main()
