"""gb_find_overlapping_submaps on the H100, on a small global-mapping scene (48 submaps on two laps, reduced rays):
  * the pair list equals GLIM's loop restated in Python over gb_overlap with the numpy-restated deltas, for first_source
    0 and S - 1 and min_overlap 0 and 0.2, and the overlaps are equal (==, not a tolerance);
  * on a sample of pairs the overlaps equal the independent oracle on its own copy of each target map;
  * exclusion is ordered, the distance gate is exact (a bound no candidate lies within 1e-6 m of; 0; unbounded);
  * an empty source, sources with NaN points and an incremental voxel map as a target;
  * a capacity below the count writes the prefix and reports the full count; identical calls return identical bytes;
  * the launch count is the documented 8 for two different S, and gb_overlap stays one launch;
  * on the benchmark's 256-submap scene the pairs found at min_overlap 0.2 are the ones workloads.global_mapping chose."""
import ctypes as C

import numpy as np
import pytest

from glim_b200 import capi, gpu, workloads
from oracle import oracle
from tests import overlap_search_oracle as oso

pytestmark = pytest.mark.gpu
LAUNCHES = 8  # k_overlap_candidates, Select, k_overlap_queries, InclusiveSum, k_overlap, k_overlap_threshold, Select, k_overlap_emit


@pytest.fixture(scope="module")
def scene(ctx):
    w = workloads.global_mapping(ctx, n_submaps=48, laps=2, n_rays=64 * 128)
    maps = [m[-1] for m in w.maps]
    T = np.stack(w.poses)
    # a bound that no candidate's distance lies within 1e-6 m of
    d = np.array([np.linalg.norm(oso.deltas(T[i], T[j])[:3, 3]) for i, j in oso.slots(len(T), 0)])
    md = 60.0
    while np.abs(d - md).min() < 1e-6:
        md += 0.37
    return w, maps, list(w.clouds), T, md


def reference(maps, sources, T, first_source=0, existing=(), max_distance=100.0, min_overlap=0.2):
    """GLIM's loop: the gated candidates in order, one gb_overlap each, kept when overlap >= min_overlap"""
    pairs, ovs = [], []
    for i, j, D in oso.candidates(T, first_source, existing, max_distance):
        ov = gpu.overlap_gpu(maps[i], sources[j], D)
        if ov >= min_overlap:
            pairs.append((i, j))
            ovs.append(ov)
    return np.array(pairs, np.int32).reshape(-1, 2), np.array(ovs)


def search(ctx, maps, sources, T, **kw):
    return gpu.find_overlapping_submaps(maps, sources, T, ctx=ctx, **kw)


@pytest.mark.parametrize("min_overlap", [0.0, 0.2])
@pytest.mark.parametrize("last", [False, True])
def test_pairs_equal_the_reference_loop(ctx, scene, min_overlap, last):
    w, maps, sources, T, md = scene
    f = len(T) - 1 if last else 0
    want_p, want_o = reference(maps, sources, T, f, (), md, min_overlap)
    got_p, got_o = search(ctx, maps, sources, T, max_distance=md, min_overlap=min_overlap, first_source=f)
    assert len(want_p) > (2 if last else 40)
    assert np.array_equal(got_p, want_p)
    assert np.array_equal(got_o, want_o)  # bit-identical to gb_overlap
    if min_overlap == 0.0:
        assert len(got_p) == len(oso.candidates(T, f, (), md)) and (got_o < 0.2).any()


def test_overlaps_equal_the_oracle_on_a_sample(ctx, scene):
    w, maps, sources, T, md = scene
    pairs, ovs = search(ctx, maps, sources, T, max_distance=md, min_overlap=0.0)
    rng = np.random.default_rng(3)
    res = w.resolutions[-1]
    refs = {}
    for r in rng.choice(len(pairs), 12, replace=False):
        i, j = pairs[r]
        if i not in refs:
            xyz, cov = oracle.pack_cloud(w.host_clouds[i][0], np.ascontiguousarray(np.swapaxes(w.host_clouds[i][1], 1, 2)).reshape(-1, 16))
            refs[i] = oracle.GpuMap(xyz, cov, res)
        xyz_j, _ = oracle.pack_cloud(w.host_clouds[j][0])
        assert ovs[r] == oracle.overlap_gpumap([refs[i]], xyz_j, [oso.deltas(T[i], T[j])]), (i, j)


def test_exclusion_is_ordered(ctx, scene):
    w, maps, sources, T, md = scene
    pairs, ovs = search(ctx, maps, sources, T, max_distance=md, min_overlap=0.2)
    i, j = (int(x) for x in pairs[len(pairs) // 2])
    p2, o2 = search(ctx, maps, sources, T, existing=[(i, j)], max_distance=md, min_overlap=0.2)
    keep = ~((pairs[:, 0] == i) & (pairs[:, 1] == j))
    assert keep.sum() == len(pairs) - 1 and np.array_equal(p2, pairs[keep]) and np.array_equal(o2, ovs[keep])
    p3, o3 = search(ctx, maps, sources, T, existing=[(j, i)] + [(k, k) for k in range(len(T))], max_distance=md, min_overlap=0.2)
    assert np.array_equal(p3, pairs) and np.array_equal(o3, ovs)
    want_p, _ = reference(maps, sources, T, 0, list(map(tuple, pairs[:5])), md, 0.2)
    assert np.array_equal(search(ctx, maps, sources, T, existing=pairs[:5], max_distance=md, min_overlap=0.2)[0], want_p)


def test_distance_gate(ctx, scene):
    w, maps, sources, T, md = scene
    S = len(T)
    assert len(search(ctx, maps, sources, T, max_distance=0.0, min_overlap=0.0)[0]) == 0
    p, o = search(ctx, maps, sources, T, max_distance=1e300, min_overlap=0.0)
    assert [tuple(x) for x in p] == oso.slots(S, 0)
    near = search(ctx, maps, sources, T, max_distance=md, min_overlap=0.0)[0]
    assert 0 < len(near) < len(p)
    assert [tuple(x) for x in near] == [(i, j) for i, j, _ in oso.candidates(T, 0, (), md)]


def test_empty_and_nan_sources_and_an_incremental_target(ctx, scene):
    w, maps, sources, T, md = scene
    S = 8
    srcs = list(sources[:S])
    srcs[3] = gpu.PointCloudGPU.clone(np.zeros((0, 4)), ctx=ctx)
    pts, cov = w.host_clouds[5]
    pts = pts.copy()
    pts[::7, :3] = np.nan
    pts[::11, 1] = np.nan
    srcs[5] = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
    tg = list(maps[:S])
    inc = gpu.IncrementalVoxelMapGPU(w.resolutions[-1], ctx=ctx)
    inc.insert(sources[2])
    tg[2] = inc
    for mo in (0.0, 0.2, -1.0):
        want_p, want_o = reference(tg, srcs, T[:S], 0, (), md, mo)
        got_p, got_o = search(ctx, tg, srcs, T[:S], max_distance=md, min_overlap=mo)
        assert np.array_equal(got_p, want_p) and np.array_equal(got_o, want_o), mo
        empty = got_p[:, 1] == 3
        assert (got_o[empty] == 0.0).all() and empty.any() == (mo <= 0.0)
    assert ((got_p[:, 1] == 5) & (got_o > 0)).any() and ((got_p[:, 0] == 2) & (got_o > 0)).any()


def raw(ctx, maps, sources, T, capacity, **kw):
    S = len(maps)
    marr = (C.c_void_p * S)(*[m.h for m in maps])
    sarr = (C.c_void_p * S)(*[s.h for s in sources])
    T16 = capi.pose16(T)
    found = C.c_size_t()
    pairs, ovs = np.full((capacity, 2), -7, np.int32), np.full(capacity, -7.0)
    capi.check(capi.lib().gb_find_overlapping_submaps(ctx.h, S, C.cast(marr, C.c_void_p), C.cast(sarr, C.c_void_p), capi.ptr(T16), 0, 0, None,
                                                      kw.get("max_distance", 100.0), kw.get("min_overlap", 0.0), capacity, C.byref(found),
                                                      capi.ptr(pairs) if capacity else None, capi.ptr(ovs) if capacity else None))
    return found.value, pairs, ovs


def test_capacity_and_repeatability(ctx, scene):
    w, maps, sources, T, md = scene
    total, p_all, o_all = raw(ctx, maps, sources, T, 2000, max_distance=md)
    assert 30 < total < 2000
    n0, _, _ = raw(ctx, maps, sources, T, 0, max_distance=md)
    assert n0 == total
    n, p, o = raw(ctx, maps, sources, T, 17, max_distance=md)
    assert n == total and np.array_equal(p, p_all[:17]) and np.array_equal(o, o_all[:17])
    _, p2, o2 = raw(ctx, maps, sources, T, 2000, max_distance=md)
    assert p2.tobytes() == p_all.tobytes() and o2.tobytes() == o_all.tobytes()
    assert (p_all[total:] == -7).all() and (o_all[total:] == -7.0).all()


def test_launch_count_is_constant(ctx, scene):
    w, maps, sources, T, md = scene
    for S in (5, len(T)):
        before = ctx.kernel_launches
        search(ctx, maps[:S], sources[:S], T[:S], max_distance=md, min_overlap=0.2)
        assert ctx.kernel_launches - before == LAUNCHES, S
    before = ctx.kernel_launches
    gpu.overlap_gpu(maps[0], sources[1], oso.deltas(T[0], T[1]))
    assert ctx.kernel_launches - before == 1
    before = ctx.kernel_launches
    assert len(search(ctx, maps[:1], sources[:1], T[:1])[0]) == 0
    assert ctx.kernel_launches == before  # one submap: no pair, no launch


def test_a_point_grid_is_refused(ctx, scene):
    w, maps, sources, T, md = scene
    grid = gpu.PointGridGPU(sources[0], 1.0, ctx=ctx)
    before = ctx.kernel_launches
    with pytest.raises(capi.GlimB200Error, match="point grid"):
        search(ctx, [grid] + maps[1:4], sources[:4], T[:4])
    assert ctx.kernel_launches == before


def test_benchmark_scene_pairs_equal_the_workload_loop(ctx):
    """the benchmark's 256-submap graph, built as bench.py builds it: workloads.global_mapping chose its pairs with a per-pair
    loop over gb_overlap"""
    import bench

    args = bench.workload_args("global_mapping_gpu", 1.0)
    w = bench.build_workload("global_mapping_gpu", ctx, 1.0, use_gpu=True)
    p = args["params"]
    chosen = sorted({(f.target, f.source) for f in w.sets[0].factors})
    pairs, ovs = gpu.find_overlapping_submaps([m[-1] for m in w.maps], w.clouds, w.poses, max_distance=p.max_implicit_loop_distance,
                                              min_overlap=p.min_implicit_loop_overlap, ctx=ctx)
    assert len(w.poses) == 256 and len(chosen) == w.notes["num_pairs"] > 500
    assert [tuple(int(v) for v in x) for x in pairs] == chosen
    assert (ovs >= p.min_implicit_loop_overlap).all()
