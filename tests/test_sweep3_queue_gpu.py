"""k_vgicp_sweep3's one-word queue entries, and its lookup on long collision chains, against the fp64 oracle
(go_vgicp_linearize_gpumap).

sweep3 queues a hit as one word: the point's offset within its item (11 bits) above the voxel index (21 bits).  So a sweep
whose target holds 2^21 voxels or more runs sweep5, whatever GB_KERNEL says.  A lookup gathers the first bucket of every
probe of a group, the second for the probes whose first bucket holds another voxel, and walks longer chains bucket by bucket.
"""
import numpy as np
import pytest

from tests import util
from tests.util import check_linearized

pytestmark = pytest.mark.gpu


def _hash(c):
    c = np.asarray(c, np.int64).astype(np.uint32)
    return (c[..., 0] * np.uint32(73856093)) ^ (c[..., 1] * np.uint32(19349669)) ^ (c[..., 2] * np.uint32(83492791))


def _cloud(pts, cov_diag):
    P = np.concatenate([pts, np.ones((len(pts), 1))], axis=1)
    Cv = np.tile(np.diag(list(cov_diag) + [0.0]), (len(P), 1, 1))
    return P, Cv


def _sweep_vs_oracle(ctx, tgt, src, res, T):
    """One factor on a built map of `tgt`, swept from `src` at pose T: -> (sweep, record, oracle record, corr, map, oracle map)"""
    from oracle import oracle
    from glim_b200 import gpu

    m = gpu.GaussianVoxelMapGPU(res, ctx=ctx).insert(gpu.PointCloudGPU.clone(*tgt, ctx=ctx))
    xyz0, cov0 = oracle.pack_cloud(tgt[0], util.cov_colmajor16(tgt[1]))
    xyz1, cov1 = oracle.pack_cloud(src[0], util.cov_colmajor16(src[1]))
    ref_map = oracle.GpuMap(xyz0, cov0, res)
    assert (m.num_voxels, m.num_buckets) == (ref_map.num_voxels, ref_map.num_buckets)
    sw = gpu.Sweep(ctx, [gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, m, gpu.PointCloudGPU.clone(*src, ctx=ctx), ctx=ctx)])
    sw.set_poses(np.stack([T]))
    sw.launch()
    got = gpu.unpack_linearized(sw.fetch()[0])
    ref, corr = oracle.linearize_gpumap(ref_map, xyz1, cov1, T)
    check_linearized(got, ref, hits=util.factor_hits(ref_map.vmean, ref_map.vcov, xyz1, cov1, T, corr))
    return sw, got, ref, corr, m, ref_map


def test_collision_chains_of_three_or_more_buckets(ctx, monkeypatch):
    """A target whose voxels collide on purpose: 8 groups of 6 voxels near the origin, each group's voxels hashing to the
    same bucket of the 16384-bucket table, so their lookups walk chains of up to 6 buckets."""
    from glim_b200 import synth

    monkeypatch.setenv("GB_KERNEL", "3")
    res, nb = 0.5, 16384
    g = np.stack(np.meshgrid(*[np.arange(-40, 40)] * 3, indexing="ij"), -1).reshape(-1, 3)
    slot = _hash(g) & np.uint32(nb - 1)
    order = np.argsort(slot, kind="stable")
    s_sorted = slot[order]
    starts = np.flatnonzero(np.r_[True, s_sorted[1:] != s_sorted[:-1]])
    bases, voxels = [], []
    for st in starts:
        if len(voxels) == 8:
            break
        b = int(s_sorted[st])
        if any(abs(b - x) < 16 for x in bases) or st + 6 > len(s_sorted) or s_sorted[st + 5] != b:
            continue
        bases.append(b)
        voxels.append(g[order[st:st + 6]])
    voxels = np.concatenate(voxels)
    assert len(voxels) == 48
    rng = synth.rng_for(901)
    pts = (np.repeat(voxels, 24, axis=0) + rng.uniform(0.1, 0.9, size=(48 * 24, 3))) * res
    tgt = _cloud(pts, (0.004, 0.003, 0.002))
    src = _cloud(pts + rng.normal(0, 0.01, size=pts.shape), (0.003, 0.004, 0.002))
    T = synth.pose(0.02, -0.01, 0.005, 0.01, 0.002, -0.003)
    sw, got, ref, corr, m, ref_map = _sweep_vs_oracle(ctx, tgt, src, res, T)
    assert sw.num_tiles > 1 and got["num_inliers"] > 0.5 * len(pts)
    buckets = m.download()[0]
    occ = buckets[:, 3] >= 0
    dist = (np.flatnonzero(occ) - _hash(buckets[occ, :3]).astype(np.int64)) & (nb - 1)
    dist_of_voxel = np.empty(m.num_voxels, np.int64)
    dist_of_voxel[buckets[occ, 3]] = dist
    hit_dist = dist_of_voxel[corr[corr >= 0]]
    assert (hit_dist >= 2).sum() > 0.4 * len(hit_dist)  # most hits took a chain of three or more buckets
    assert hit_dist.max() == 5


def test_target_of_2_21_voxels_or_more_runs_sweep5(ctx, monkeypatch):
    """A target of 2^21 voxels or more: its voxel indices do not fit sweep3's queue word, so the sweep runs sweep5 whatever
    GB_KERNEL says (its item count is sweep5's), and matches the oracle."""
    from glim_b200 import synth

    monkeypatch.setenv("GB_KERNEL", "3")
    res, side = 0.1, 130
    g = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3)
    pts = (g + 0.5) * res
    tgt = _cloud(pts, (4e-4, 3e-4, 2e-4))
    rng = synth.rng_for(903)
    n = 20000  # rows of 32: 625; sweep5 gives one factor 625 // 4 = 156 items, sweep3 ceil(20000 / 128) = 157
    sp = pts[rng.choice(len(pts), n, replace=False)] + rng.normal(0, 0.005, size=(n, 3))
    src = _cloud(sp, (3e-4, 4e-4, 2e-4))
    sw, got, _, _, m, _ = _sweep_vs_oracle(ctx, tgt, src, res, synth.pose(0.003, -0.002, 0.001, 0.002))
    assert m.num_voxels >= 1 << 21
    assert sw.num_tiles == 156
    assert got["num_inliers"] > 0.5 * n
