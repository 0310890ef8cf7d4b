"""k_vgicp_sweep3 probes each target's probe index (glim_b200/csrc/gb_probe_index.cuh), against the fp64 oracle
(go_vgicp_linearize_gpumap).

A built map gets the index when its voxels fit it: fewer than 2^21 of them and a coordinate box of at most 2^14 - 2 voxels per
axis past its minimum.  A sweep runs sweep3 only when every target has one; a target whose box is wider runs sweep5, whatever
GB_KERNEL says.
"""
import numpy as np
import pytest

from tests.test_probe_index_host import Index, dense_block, host_index_lib
from tests.test_sweep3_queue_gpu import _cloud, _sweep_vs_oracle

pytestmark = pytest.mark.gpu

N_SRC = 20000  # rows of 32: 625; sweep5 gives one factor 625 // 4 = 156 items, sweep3 ceil(20000 / 128) = 157


def _scene(res, offset, seed):
    """a 20^3 voxel block at the origin and another `offset` voxels along x, and a source sampled around both"""
    from glim_b200 import synth

    g = np.stack(np.meshgrid(*[np.arange(20)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    g = np.concatenate([g, g + [offset, 0, 0]])
    rng = synth.rng_for(seed)
    pts = (np.repeat(g, 3, axis=0) + rng.uniform(0.1, 0.9, size=(3 * len(g), 3))) * res
    sp = pts[rng.choice(len(pts), N_SRC, replace=False)] + rng.normal(0, 0.01 * res, size=(N_SRC, 3))
    return _cloud(pts, (4e-4, 3e-4, 2e-4)), _cloud(sp, (3e-4, 4e-4, 2e-4))


@pytest.mark.parametrize("offset,kernel_items", [(16382 - 19, 157), (16383 - 19, 156)])
def test_index_box_limit_picks_the_kernel(ctx, monkeypatch, offset, kernel_items):
    """A box of 16382 voxels along x still has an index (sweep3 under GB_KERNEL=3); one of 16383 has none and runs sweep5.
    Both match the oracle."""
    from glim_b200 import synth

    monkeypatch.setenv("GB_KERNEL", "3")
    res = 0.05
    tgt, src = _scene(res, offset, 911)
    sw, got, _, _, m, _ = _sweep_vs_oracle(ctx, tgt, src, res, synth.pose(0.003, -0.002, 0.001, 0.002))
    assert sw.num_tiles == kernel_items
    assert got["num_inliers"] > 0.5 * N_SRC


def test_dense_target_with_overflowing_sets(ctx, monkeypatch, tmp_path):
    """A dense 40^3 block of voxels: some index sets overflow, and some of the sweep's hits are voxels that a lookup finds only
    by walking past its home set (counted with the host build of the same index).  The sweep matches the oracle."""
    from glim_b200 import synth

    monkeypatch.setenv("GB_KERNEL", "3")
    res = 0.1
    pts, cov = dense_block(40, res)
    rng = synth.rng_for(912)
    sp = pts[rng.choice(len(pts), N_SRC, replace=False), :3] + rng.normal(0, 0.02, size=(N_SRC, 3))
    tgt = (pts, cov)
    sw, got, _, corr, m, ref_map = _sweep_vs_oracle(ctx, tgt, _cloud(sp, (3e-4, 4e-4, 2e-4)), res, synth.pose(0.003, -0.002, 0.001, 0.002))
    assert sw.num_tiles == 157
    assert got["num_inliers"] > 0.5 * N_SRC and (corr < 0).sum() > 0
    ix = Index(host_index_lib(tmp_path), ref_map)
    assert ix.fits and ix.overflowing_sets() > 0
    hit_voxels = np.unique(corr[corr >= 0])
    found, rounds = ix.lookup(ref_map.vcoord[hit_voxels], rounds=True)
    assert np.array_equal(found, hit_voxels)
    assert (rounds >= 2).sum() > 0  # hits resolved by the overflow walk


@pytest.mark.parametrize("init_buckets,kernel_items", [(1, 156), (16384, 157)])
def test_empty_target(ctx, monkeypatch, init_buckets, kernel_items):
    """A target without voxels (every point NaN).  A table of one bucket has no index set, so the sweep runs sweep5 under
    GB_KERNEL=3; a larger table gets an empty index and sweep3.  Source points in voxel (0, 0, 0) and NaN points (which land
    there) find nothing, as in the oracle."""
    from oracle import oracle
    from glim_b200 import gpu, synth
    from tests import util

    monkeypatch.setenv("GB_KERNEL", "3")
    res = 0.5
    tgt = _cloud(np.full((64, 3), np.nan), (4e-4, 3e-4, 2e-4))
    rng = synth.rng_for(913)
    sp = rng.uniform(0.0, 0.45, size=(N_SRC, 3))
    sp[::7] = np.nan
    src = _cloud(sp, (3e-4, 4e-4, 2e-4))
    m = gpu.GaussianVoxelMapGPU(res, init_num_buckets=init_buckets, ctx=ctx).insert(gpu.PointCloudGPU.clone(*tgt, ctx=ctx))
    ref_map = oracle.GpuMap(*oracle.pack_cloud(tgt[0], util.cov_colmajor16(tgt[1])), res, init_buckets=init_buckets)
    assert (m.num_voxels, m.num_buckets) == (ref_map.num_voxels, ref_map.num_buckets) == (0, init_buckets)
    sw = gpu.Sweep(ctx, [gpu.IntegratedVGICPFactorGPU(np.eye(4), 1, m, gpu.PointCloudGPU.clone(*src, ctx=ctx), ctx=ctx)])
    T = synth.pose(0.0, 0.0, 0.0, 0.0)
    sw.set_poses(np.stack([T]))
    sw.launch()
    got = gpu.unpack_linearized(sw.fetch()[0])
    xyz1, cov1 = oracle.pack_cloud(src[0], util.cov_colmajor16(src[1]))
    ref = oracle.split122(oracle.linearize_gpumap(ref_map, xyz1, cov1, T)[0])
    assert sw.num_tiles == kernel_items
    assert got["num_inliers"] == ref["num_inliers"] == 0
    for k in ("H_tt", "H_ss", "H_ts", "b_t", "b_s"):
        assert not np.any(got[k])
    assert got["error"] == 0.0
