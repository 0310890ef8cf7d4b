"""How the VGICP sweep's first hash probe ends, on the CPU: for sample pairs of the global-mapping workload (bench.py's default,
256 submaps x 50 k points, four laps of a 300 m loop), the target's voxel tables at both levels are built with the oracle
(oracle.GpuMap: the device table, bit for bit) and every source point, moved by the pair's perturbed relative pose and taken in
the device cloud's Morton order, is looked up the way phase A of k_vgicp_sweep3 / 5 does.  Per pair kind and level it prints the
fraction of points whose FIRST bucket holds their voxel (hit), is empty (miss) or holds another voxel (collision: the lane
gathers the second bucket), the fraction that needs a third bucket or more, and the fraction of 32-point warp rows with at
least one colliding lane (a row whose lanes all resolve on the first bucket skips the second gather round).

With --index it also builds each target's probe index (glim_b200/csrc/gb_probe_index.cuh, compiled for the host from
tests/cpp/probe_index_host.cpp) and compares, per 256-point lookup group of the Morton-ordered source (k_vgicp_sweep3's group),
the fraction of groups that need a second and a third dependent gather on the bucket table and on the index, the fraction of
points the index's box culls without a gather, and the bytes per voxel of both.

    python scripts/probe_stats.py [--anchors 3] [--seed 0] [--index]

Needs oracle/libglim_oracle.so (built by __graft_entry__.build()) and, for --index, g++; no GPU.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile
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


GROUP = 256  # points per lookup group of k_vgicp_sweep3 (8 probes per lane)
SET_SHIFT = 1  # kPiSetShift


def index_lib():
    so = os.path.join(tempfile.mkdtemp(), "libprobe_index_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-o", so, os.path.join(ROOT, "tests", "cpp", "probe_index_host.cpp")])
    L = C.CDLL(so)
    vp = C.c_void_p
    L.pih_build.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp, C.c_int, C.c_uint]
    L.pih_lookup.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def index_rounds(L, table, xyz, delta):
    """per point: the dependent set gathers of a probe-index lookup (0 = outside the box), and whether the index was built"""
    buckets = np.ascontiguousarray(table.buckets, np.int32)
    vcoord = np.zeros((table.num_voxels, 4), np.int32)
    vcoord[:, :3] = table.vcoord
    slots = np.empty(2 * (table.num_buckets >> SET_SHIFT), np.uint64)
    box = np.zeros(6, np.int32)
    if not L.pih_build(_p(buckets), table.num_buckets, _p(vcoord), table.num_voxels, _p(slots), _p(box), 0, 0):
        return None
    R, t = delta[:3, :3].astype(np.float32), delta[:3, 3].astype(np.float32)
    q = xyz @ R.T + t
    with np.errstate(invalid="ignore"):
        c = np.floor(q * (np.float32(1.0) / np.float32(table.resolution)))
    c = np.ascontiguousarray(np.where(np.isfinite(c), c, 0).astype(np.int32))
    out = np.empty(len(c), np.int32)
    rounds = np.empty(len(c), np.int32)
    L.pih_lookup(_p(slots), table.num_buckets, _p(box), len(c), _p(c), _p(out), _p(rounds))
    return rounds


def group_frac(x):
    ng = len(x) // GROUP
    return x[: ng * GROUP].reshape(ng, GROUP).any(1).sum(), ng


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--anchors", type=int, default=3, help="pairs per kind (sources spread over the second lap)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--index", action="store_true", help="also simulate the probe index and report per-group dependent gathers")
    args = ap.parse_args()
    L = index_lib() if args.index else None
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

    head = f"{'pair kind':<22} {'level':>6} {'points':>8} {'hit':>6} {'empty':>6} {'collide':>8} {'>2 buckets':>11} {'rows w/ collision':>18}"
    if L:
        head += f" | {'table: groups 2nd':>17} {'3rd':>6} {'index: groups 2nd':>17} {'3rd':>6} {'box culled':>10} {'B/voxel table':>13} {'index':>6}"
    print(head)
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
                s = sums.setdefault(lvl, np.zeros(15))
                s[:7] += [len(xyz), first_hit.sum(), empty.sum(), collide.sum(), (reads >= 3).sum(), rows.sum(), nw]
                if L:
                    tb = tables[(tgt, lvl)]
                    ir = index_rounds(L, tb, xyz, delta)
                    g2, ng = group_frac(reads >= 2)
                    g3, _ = group_frac(reads >= 3)
                    i2, _ = group_frac(ir >= 2)
                    i3, _ = group_frac(ir >= 3)
                    s[7:] += [ng, g2, g3, i2, i3, (ir == 0).sum(), 16 * tb.num_buckets / tb.num_voxels, 16 * (tb.num_buckets >> SET_SHIFT) / tb.num_voxels]
        for lvl, s in sorted(sums.items()):
            n = s[0]
            line = f"{kind:<22} {resolutions[lvl]:>5.1f}m {int(n):>8d} {s[1] / n:>6.3f} {s[2] / n:>6.3f} {s[3] / n:>8.3f} {s[4] / n:>11.4f} {s[5] / max(1, s[6]):>18.3f}"
            if L:
                ng = max(1, s[7])
                line += f" | {s[8] / ng:>17.3f} {s[9] / ng:>6.3f} {s[10] / ng:>17.3f} {s[11] / ng:>6.3f} {s[12] / n:>10.3f} {s[13] / args.anchors:>13.1f} {s[14] / args.anchors:>6.1f}"
            print(line)
    print(f"({args.anchors} pair(s) per kind, {len(clouds)} clouds, {time.time() - t0:.0f} s)")


if __name__ == "__main__":
    main()
