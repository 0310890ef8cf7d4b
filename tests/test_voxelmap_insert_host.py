"""The numpy restatement of the incremental voxel map (tests/voxelmap_oracle.py) against the CPU oracle's GaussianVoxelMapCPU
(go_cpumap: incremental insert with the LRU horizon, SURVEY B.5), and its table against the oracle's map build.  No device."""
import numpy as np

from oracle import oracle
from tests import voxelmap_oracle as vo
from tests.util import cov_colmajor16

N_FRAMES = 22
NAN_FRAME = 9
EMPTY_INSERT = 14  # sampling keeps no point


def insert_rate(k):
    if k == EMPTY_INSERT:
        return 1e-9
    return 1.0 if k < 5 else 0.1  # update_target: 10 % from frame 5 on (odometry_estimation_cpu.cpp:181)


def test_sampling_pick():
    n = 1000
    h = vo.rg_hash(7, np.arange(n))
    assert len(np.unique(h)) == n  # a bijection of the index: no ties
    keep = vo.sample_mask(n, 0.1, 7)
    assert keep.sum() == 100 and h[keep].max() < h[~keep].min()
    assert vo.sample_mask(n, 1.0, 7).all() and not vo.sample_mask(n, 1e-9, 7).any()
    assert vo.sample_mask(999, 0.1, 3).sum() == 99  # (size_t)(n * rate), as random_sampling
    assert not np.array_equal(vo.sample_mask(n, 0.1, 7), vo.sample_mask(n, 0.1, 8))


def test_transform_matches_numpy():
    rng = np.random.default_rng(4)
    T = synth_pose(rng)
    xyz = rng.normal(size=(50, 3)).astype(np.float32) * 20
    A = rng.normal(size=(50, 3, 3))
    C = np.einsum("nij,nkj->nik", A, A)
    cov6 = C[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].astype(np.float32)
    q, c6 = vo.transform(T, xyz, cov6)
    assert np.allclose(q, xyz.astype(np.float64) @ T[:3, :3].T + T[:3, 3], rtol=0, atol=1e-12)
    Cf = cov6.astype(np.float64)[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3)
    RCR = np.einsum("ij,njk,lk->nil", T[:3, :3], Cf, T[:3, :3])
    assert np.allclose(c6, RCR[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]], rtol=1e-13, atol=1e-12)


def synth_pose(rng):
    from glim_b200 import synth

    return synth.se3_exp(np.concatenate([rng.normal(0, 0.3, 3), rng.normal(0, 5.0, 3)]))


def test_restatement_matches_cpu_voxelmap_with_lru():
    """>= 20 inserts at world poses along an arc, LRU horizon 6 / clear cycle 2 as in test_cpu_voxelmap_lru_horizon, one frame
    with NaN points and one insert that keeps no point: after every insert both maps hold the same voxels, and every mean and
    covariance agrees to 1e-12 relative (go_cpumap re-opens a voxel by mean *= n, the restatement keeps the sums)."""
    frames = vo.arc_frames(N_FRAMES, 32 * 60, nan_frame=NAN_FRAME)
    res = 0.5
    R = vo.IncrementalMap(res, lru_horizon=6, lru_clear_cycle=2)
    cm = oracle.CpuMap(float(np.float32(res)))
    cm.set_lru_horizon(6, clear_cycle=2)
    sizes, evicted = [], 0
    for k, (pts, cov, T) in enumerate(frames):
        xyz, cov6 = oracle.pack_cloud(pts, cov_colmajor16(cov))
        before = R.num_voxels
        R.insert(xyz, cov6, T, insert_rate(k), seed=100 + k)
        q, c6 = R.last_points
        if k == EMPTY_INSERT:
            assert len(q) == 0
        if k == NAN_FRAME:
            assert len(q) < int(len(pts) * insert_rate(k))  # the NaN points were sampled but skipped
        pts4 = np.concatenate([q, np.ones((len(q), 1))], 1)
        C = np.zeros((len(q), 4, 4))
        C[:, :3, :3] = c6[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3)
        cm.insert(pts4, cov_colmajor16(C))
        assert cm.num_voxels == R.num_voxels, k
        evicted += R.num_voxels < before
        sizes.append(R.num_voxels)
        m64, C64 = R.mean_cov64()
        centers = (R.vcoord + 0.5) * R.resolution
        for v in range(R.num_voxels):
            j, mean, cov_ref = cm.lookup(centers[v])
            assert j >= 0, (k, v)
            assert np.linalg.norm(mean[:3] - m64[v]) <= 1e-12 * np.linalg.norm(m64[v]), (k, v)
            assert np.linalg.norm(cov_ref[:3, :3] - C64[v]) <= 1e-12 * np.linalg.norm(C64[v]), (k, v)
    assert R.counter == N_FRAMES
    assert evicted > 0  # the LRU rule actually dropped voxels


def test_table_restatement_matches_oracle_build():
    """One insert at T = I, rate 1, at a power-of-two resolution (fp32 and fp64 keys agree): the restated table equals the
    oracle's GaussianVoxelMapGPU build (go_gpumap_build, the library's build rule), slot for slot."""
    pts, cov, _ = vo.arc_frames(N_FRAMES, 32 * 60, nan_frame=NAN_FRAME)[3]
    xyz, cov6 = oracle.pack_cloud(pts, cov_colmajor16(cov))
    for res in (0.25, 0.5):
        R = vo.IncrementalMap(res, init_buckets=16384).insert(xyz, cov6)
        ref = oracle.GpuMap(xyz, cov6, res, init_buckets=16384)
        assert R.num_voxels == ref.num_voxels
        assert np.array_equal(R.buckets, ref.buckets)
        assert np.array_equal(R.n, ref.vnum)
        assert np.allclose(R.means, ref.vmean, rtol=0, atol=1e-5)
