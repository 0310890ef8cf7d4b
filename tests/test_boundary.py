"""The drop-in boundary without a GPU: libglim_b200.so loads, exports exactly what include/glim_b200.h declares, and
fails loudly (no CPU fallback) when there is no CUDA device.  Host logic of the multi-GPU sharding."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from glim_b200 import capi, multi_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "glim_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return re.findall(r"GB_API\s+[\w\s\*]+?\b(gb_\w+)\s*\(", src)


def test_library_exports_every_declared_symbol():
    L = capi.lib()
    declared = header_functions()
    assert len(declared) >= 30
    assert sorted(declared) == sorted(capi.SYMBOLS)
    for name in declared:
        assert hasattr(L, name), name


def test_library_is_sm90a_only_and_links_no_torch():
    out = os.popen(f"cuobjdump --list-elf {capi.SO_PATH} 2>/dev/null").read()
    if out.strip():
        archs = set(re.findall(r"sm_(\d+a?)", out))
        assert archs == {"90a"}, archs
    # library NAMES only: the load addresses ldd prints are random hex strings (ASLR) and may well contain "c10"
    libs = [line.split()[0] for line in os.popen(f"ldd {capi.SO_PATH}").read().splitlines() if line.strip()]
    assert libs and not [l for l in libs if "torch" in l or "c10" in l], libs


def test_product_never_touches_the_oracle():
    """oracle/ is test infrastructure: nothing under glim_b200/ or include/ may import, include or link it, and the library must
    not depend on libglim_oracle.so (only tests/, __graft_entry__.smoke() and bench.py's checker / CPU legs may use it)."""
    offenders = []
    for base in ("glim_b200", "include"):
        for d, _, files in os.walk(os.path.join(ROOT, base)):
            if "build" in d.split(os.sep) or "__pycache__" in d:
                continue
            for f in files:
                if not f.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cpp", "Makefile")):
                    continue
                txt = open(os.path.join(d, f), errors="replace").read()
                if re.search(r"^\s*(from|import)\s+oracle\b|#include\s*[<\"][^>\"]*oracle|libglim_oracle|-lglim_oracle|dlopen[^\n]*oracle", txt, flags=re.M):
                    offenders.append(os.path.join(d, f))
    assert not offenders, offenders
    needed = os.popen(f"readelf -d {capi.SO_PATH}").read()
    assert "NEEDED" in needed and "oracle" not in needed


def test_status_strings():
    L = capi.lib()
    assert L.gb_status_string(0) == b"ok"
    assert b"no CPU fallback" in L.gb_status_string(4)


def test_no_device_fails_loudly():
    L = capi.lib()
    if L.gb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    h = C.c_void_p()
    st = L.gb_ctx_create(0, C.byref(h))
    assert st == 4 and not h.value  # GB_ERR_NO_DEVICE
    assert b"no CPU fallback" in L.gb_last_error()
    from glim_b200 import gpu

    with pytest.raises(capi.GlimB200Error):
        gpu.Context(0)
    fr = C.c_size_t()
    assert L.gb_mem_info(0, C.byref(fr), C.byref(fr)) == 4


def test_null_arguments_are_rejected_not_crashed():
    L = capi.lib()
    assert L.gb_ctx_create(0, None) == 1
    assert L.gb_cloud_size(None, None) == 1
    assert L.gb_voxelmap_info(None, None, None, None) == 1
    assert L.gb_sweep_launch(None) == 1
    assert L.gb_ctx_destroy(None) == 0 and L.gb_cloud_destroy(None) == 0 and L.gb_vgicp_factor_destroy(None) == 0


def test_pose16_is_column_major():
    T = np.arange(16.0).reshape(4, 4)
    assert np.array_equal(capi.pose16(T), T.T.reshape(16))
    assert capi.pose16(np.stack([T, T])).shape == (2, 16)


def test_lpt_partition_balances_and_is_deterministic():
    rng = np.random.default_rng(0)
    w = rng.integers(1000, 60000, size=301)
    for parts in (1, 2, 4, 8):
        p = multi_gpu.lpt_partition(w, parts)
        loads = np.array([w[p == k].sum() for k in range(parts)])
        assert loads.sum() == w.sum() and loads.max() <= loads.mean() + w.max()
        assert np.array_equal(p, multi_gpu.lpt_partition(w, parts))


def test_shard_factors_keeps_pairs_whole():
    from glim_b200.workloads import Factor

    factors = [Factor(i, l, j, pair) for pair, (i, j) in enumerate([(0, 3), (1, 3), (2, 3), (0, 4), (1, 4)]) for l in (0, 1)]
    sizes = [50000, 40000, 30000, 50000, 20000]
    f_rank, p_rank = multi_gpu.shard_factors(factors, sizes, 2)
    for f, r in zip(factors, f_rank):
        assert r == p_rank[f.pair]
    assert set(f_rank) == {0, 1}


def test_slab_row_roundtrip():
    rng = np.random.default_rng(1)
    A = rng.normal(size=(6, 6))
    rec = {"H_tt": A @ A.T, "H_ss": A.T @ A, "H_ts": rng.normal(size=(6, 6)), "b_t": rng.normal(size=6), "b_s": rng.normal(size=6), "error": 3.5, "num_inliers": 42.0}
    back = multi_gpu.unpack_slab_row(multi_gpu.pack_slab_row(rec))
    for k in ("H_tt", "H_ss", "H_ts", "b_t", "b_s"):
        assert np.allclose(back[k], rec[k], rtol=1e-6, atol=1e-6)
    assert back["error"] == 3.5 and back["num_inliers"] == 42.0


def test_contiguous_partition_is_balanced_ordered_and_keeps_sources_together():
    """The committed multi-GPU partition: contiguous chunks of the source-major factor order, equal cost, pairs whole; with
    measured inlier counts the weights follow them."""
    from glim_b200.workloads import Factor

    rng = np.random.default_rng(3)
    factors, pair = [], 0
    for cur in range(1, 120):
        for i in rng.choice(cur, size=min(cur, int(rng.integers(1, 9))), replace=False):
            for l in (0, 1):
                factors.append(Factor(int(i), l, cur, pair))
            pair += 1
    sizes = [50000] * 120
    ov = {p: float(rng.uniform(0.2, 0.9)) for p in range(pair)}
    for world in (2, 4, 8):
        f_rank, p_rank = multi_gpu.shard_factors(factors, sizes, world, pair_cost=ov)
        assert (np.diff(f_rank) >= 0).all() and set(f_rank) == set(range(world))  # contiguous, every rank has work
        for f, r in zip(factors, f_rank):
            assert r == p_rank[f.pair]
        cost = np.array([sizes[f.source] * (1 + 1.25 * ov[f.pair]) for f in factors])
        loads = np.array([cost[f_rank == r].sum() for r in range(world)])
        assert loads.max() <= loads.mean() * 1.02 + cost.max() * 2
        # a source cloud is split over at most two neighbouring ranks
        by_src = {}
        for f, r in zip(factors, f_rank):
            by_src.setdefault(f.source, set()).add(int(r))
        assert max(len(v) for v in by_src.values()) <= 2
    inl = rng.uniform(0, 50000, size=len(factors))
    f_rank, _ = multi_gpu.shard_factors(factors, sizes, 4, factor_inliers=inl)
    cost = np.array([sizes[f.source] for f in factors]) + 1.25 * inl
    loads = np.array([cost[f_rank == r].sum() for r in range(4)])
    assert loads.max() <= loads.mean() * 1.02 + cost.max() * 2
    lpt, _ = multi_gpu.shard_factors(factors, sizes, 4, pair_cost=ov, contiguous=False)
    assert set(lpt) == {0, 1, 2, 3}


def test_time_feedback_moves_work_off_the_slow_rank():
    """bench.py's partition feedback: the factors of a rank that measured slow get heavier, the next cut gives it fewer."""
    from glim_b200.workloads import Factor

    rng = np.random.default_rng(5)
    factors, pair = [], 0
    for cur in range(1, 200):
        for i in rng.choice(cur, size=min(cur, 6), replace=False):
            for l in (0, 1):
                factors.append(Factor(int(i), l, cur, pair))
            pair += 1
    sizes = [50000] * 200
    inl = rng.uniform(1000, 40000, size=len(factors))
    base, _ = multi_gpu.shard_factors(factors, sizes, 4, factor_inliers=inl)
    t = np.array([1.08, 1.0, 1.0, 0.96])  # rank 0 measured 8 % slow, rank 3 fast
    scale = (t / t.mean())[base]
    fb, p_rank = multi_gpu.shard_factors(factors, sizes, 4, factor_inliers=inl, factor_scale=scale)
    assert (np.diff(fb) >= 0).all() and set(fb) == {0, 1, 2, 3}
    for f, r in zip(factors, fb):
        assert r == p_rank[f.pair]
    n0, n1 = np.bincount(base, minlength=4), np.bincount(fb, minlength=4)
    assert n1[0] < n0[0] and n1[3] > n0[3]
    # predicted times with the per-factor slowness carried along: the spread shrinks
    cost = (np.array([sizes[f.source] for f in factors]) + 1.25 * inl) * scale
    spread = lambda fr: np.ptp([cost[fr == r].sum() for r in range(4)])
    assert spread(fb) < 0.5 * spread(base)
