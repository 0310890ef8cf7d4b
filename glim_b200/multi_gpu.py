"""Sharding of a global-mapping relinearization sweep across the GPUs of one box (SURVEY.md 8(e)).

The reference has no multi-GPU notion (SURVEY 0.6); this is the multi-GPU addition north_star asks for.
Every rank holds all submap clouds and voxel maps (replicated at insert time, ~1.5 GB); the (target, source) PAIRS of the
factor graph are partitioned over the ranks -- both voxel levels of a pair stay together; by default `world` CONTIGUOUS chunks
of the reference's source-major factor order, cut at equal cost (measured inliers, then per-rank kernel-time feedback), so that
a rank keeps all factors of the source clouds it touches.  Each rank sweeps its factors with the fused kernel.  Result exchange,
two variants (DESIGN.md 8):
  * peer slab (default, `gpu.PeerSlab`): every pair is owned by one rank, whose kernel stores the finished fp32 row
    [GB_SLAB_STRIDE] into every rank's IPC-mapped slab over NVLink -- an all-gather done by the producers, no NCCL in the step;
  * local slab + one NCCL all-reduce (sum) of [num_pairs][GB_SLAB_STRIDE] (`ShardedSweep` below; `bench.py --collective nccl`,
    and the world-size-2 gloo test on the CPU-only box).
Either way every rank ends up with the complete block-sparse Hessian for its copy of the host solver.
"""
from __future__ import annotations

import numpy as np

from .capi import GB_SLAB_STRIDE


def lpt_partition(weights, n_parts: int):
    """Longest-processing-time-first: returns part index per item; deterministic (ties by index)."""
    weights = np.asarray(weights, dtype=np.float64)
    order = sorted(range(len(weights)), key=lambda i: (-weights[i], i))
    load = [0.0] * n_parts
    part = np.zeros(len(weights), dtype=np.int64)
    for i in order:
        p = min(range(n_parts), key=lambda k: (load[k], k))
        part[i] = p
        load[p] += weights[i]
    return part


def shard_factors(factors, source_sizes, world: int, pair_cost=None, contiguous=True, factor_inliers=None, factor_scale=None):
    """factors: objects with .pair and .source, in the order the reference creates them (source-major: all factors of one
    new submap are consecutive, global_mapping.cpp:441-470); -> (rank per factor, rank per pair).  Pairs are kept whole.

    pair_cost (optional): pair -> expected inlier fraction (the overlap the gate measured).  In the sweep kernel a hit costs
    ~2.2x a miss (fit to the measured sub-mapping / global-mapping throughputs), so a factor weighs n_source * (1 + 1.25 * overlap).

    factor_inliers (optional): measured inlier count per factor from a previous sweep (a relinearizing back-end has them for
    free): the weight becomes n_source + 1.25 * inliers, which replaces the overlap estimate.

    factor_scale (optional): multiplier per factor on top of either weight -- the time feedback of a back-end that re-linearizes
    the same factor set many times: after a sweep every rank knows its kernel time t_r (CUDA events); the factors it held get
    their weight scaled by t_r / mean(t), and the next partition evens out what the cost model missed (cache locality, ...).

    contiguous=True (default): cut the factor list into `world` consecutive chunks of equal total weight.  Every rank then
    keeps ALL factors of the source clouds it touches, so a source cloud is read from HBM once per rank-sweep and served from
    L2 to the ~26 factors that share it -- exactly the reuse a single GPU gets.  contiguous=False: longest-processing-time
    first (best balance, but scatters the factors of one source over all ranks)."""
    pairs = []
    seen = set()
    for f in factors:
        if f.pair not in seen:
            seen.add(f.pair)
            pairs.append(f.pair)
    index = {p: k for k, p in enumerate(pairs)}
    w = np.zeros(len(pairs))
    for k, f in enumerate(factors):
        sc = 1.0 if factor_scale is None else float(factor_scale[k])
        if factor_inliers is not None:
            w[index[f.pair]] += sc * (source_sizes[f.source] + 1.25 * float(factor_inliers[k]))
        else:
            c = 1.0 + 1.25 * float(pair_cost[f.pair]) if pair_cost is not None and f.pair in pair_cost else 1.0
            w[index[f.pair]] += sc * source_sizes[f.source] * c
    if contiguous:
        cum = np.cumsum(w) - 0.5 * w  # midpoint rule: a pair goes to the chunk its centre of mass falls in
        total = float(w.sum()) or 1.0
        pair_rank = np.minimum(world - 1, (cum / total * world).astype(np.int64))
    else:
        pair_rank = lpt_partition(w, world)
    return np.array([pair_rank[index[f.pair]] for f in factors], dtype=np.int64), {p: int(pair_rank[index[p]]) for p in pairs}


def unpack_slab_row(row):
    """fp32 slab row -> dict of 6x6 / 6 blocks (see GB_SLAB_STRIDE in include/glim_b200.h)."""
    row = np.asarray(row, dtype=np.float64)
    iu = np.triu_indices(6)

    def sym(v):
        M = np.zeros((6, 6))
        M[iu] = v
        return M + np.triu(M, 1).T

    return {
        "H_tt": sym(row[0:21]),
        "H_ts": row[21:57].reshape(6, 6).T.copy(),
        "H_ss": sym(row[57:78]),
        "b_t": row[78:84].copy(),
        "b_s": row[84:90].copy(),
        "error": float(row[90]),
        "num_inliers": float(row[91]),
    }


def pack_slab_row(rec: dict) -> np.ndarray:
    """Inverse of unpack_slab_row for [row, col] blocks (host-side reference used by the CPU tests)."""
    iu = np.triu_indices(6)
    row = np.zeros(GB_SLAB_STRIDE, dtype=np.float32)
    row[0:21] = rec["H_tt"][iu]
    row[21:57] = rec["H_ts"].T.reshape(36)
    row[57:78] = rec["H_ss"][iu]
    row[78:84] = rec["b_t"]
    row[84:90] = rec["b_s"]
    row[90] = rec["error"]
    row[91] = rec["num_inliers"]
    return row


class ShardedSweep:
    """One rank's share of a sweep + the slab all-reduce.  `launch` is a callable that enqueues this rank's kernel
    (adds into `slab`); on the GPU it is gpu.Sweep.launch, in the CPU (gloo) tests a host stand-in."""

    def __init__(self, slab, launch, world: int):
        self.slab = slab  # torch tensor [num_pairs, GB_SLAB_STRIDE] float32
        self.launch = launch
        self.world = world

    def step(self):
        import torch.distributed as dist

        self.slab.zero_()
        self.launch()
        if self.world > 1:
            dist.all_reduce(self.slab, op=dist.ReduceOp.SUM)
        return self.slab
