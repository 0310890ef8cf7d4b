"""CPU-only exactness of the probe index (glim_b200/csrc/gb_probe_index.cuh) that k_vgicp_sweep3 probes instead of a built
map's bucket table.

The SAME text the device builds the index with (k_table_finalize) and looks it up with (probe_issue / probe_resolve of
gb_sweep_steps.cuh) is compiled for the host with g++ (tests/cpp/probe_index_host.cpp).  The index is built from the buckets of
oracle.GpuMap (the device's table, bit for bit) and must answer every coordinate exactly as gb_lookup on those buckets does: the
sweep's hits, their queue order and so every output bit depend on it.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from glim_b200 import synth, workloads
from oracle import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SET_SHIFT = 1  # kPiSetShift
MAX_EXTENT = (1 << 14) - 2  # kPiMaxExtent


def host_index_lib(directory):
    """tests/cpp/probe_index_host.cpp compiled into `directory`"""
    so = os.path.join(str(directory), "libprobe_index_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-Wall", "-Werror", "-o", so, os.path.join(ROOT, "tests", "cpp", "probe_index_host.cpp")])
    L = C.CDLL(so)
    vp = C.c_void_p
    L.pih_build.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp, C.c_int, C.c_uint]
    L.pih_lookup.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp, vp]
    L.pih_gb_lookup.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp]
    return L


@pytest.fixture(scope="module")
def pih(tmp_path_factory):
    return host_index_lib(tmp_path_factory.mktemp("pih"))


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class Index:
    """the probe index of oracle map m, built sequentially (threads = 0) or by `threads` threads in a shuffled order"""

    def __init__(self, L, m, threads=0, seed=0):
        self.L, self.m = L, m
        nb = m.num_buckets
        self.buckets = np.ascontiguousarray(m.buckets, np.int32)
        vcoord = np.zeros((m.num_voxels, 4), np.int32)
        vcoord[:, :3] = m.vcoord[:, :3]
        self.slots = np.empty(2 * (nb >> SET_SHIFT), np.uint64)
        self.box = np.zeros(6, np.int32)
        self.fits = bool(L.pih_build(_p(self.buckets), nb, _p(vcoord), m.num_voxels, _p(self.slots), _p(self.box), threads, seed))

    def lookup(self, xyz, rounds=False):
        """the index's answers (and, with rounds, the dependent set gathers of each lookup)"""
        xyz = np.ascontiguousarray(xyz, np.int32)
        out = np.empty(len(xyz), np.int32)
        r = np.empty(len(xyz), np.int32)
        self.L.pih_lookup(_p(self.slots), self.m.num_buckets, _p(self.box), len(xyz), _p(xyz), _p(out), _p(r))
        return (out, r) if rounds else out

    def overflowing_sets(self):
        return int((self.slots[0::2] & np.uint64(1)).sum())

    def gb_lookup(self, xyz):
        xyz = np.ascontiguousarray(xyz, np.int32)
        out = np.empty(len(xyz), np.int32)
        self.L.pih_gb_lookup(_p(self.buckets), self.m.num_buckets, 10, len(xyz), _p(xyz), _p(out))
        return out


def c16(cov):
    return np.ascontiguousarray(np.swapaxes(cov, 1, 2)).reshape(len(cov), 16)


def dense_block(side=40, res=0.1):
    """a side^3 block of voxels, one point at each voxel's centre (homogeneous points, 4x4 covariances): dense enough that some
    index sets overflow"""
    g = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3)
    pts = np.concatenate([(g + 0.5) * res, np.ones((len(g), 1))], axis=1)
    cov = np.zeros((len(g), 4, 4))
    cov[:, :3, :3] = np.diag([4e-4, 3e-4, 2e-4])
    return pts, cov


@pytest.fixture(scope="module")
def maps():
    """bench.py's global-mapping submap at 0.5 and 1.0 m, and a MID-360 frame (livox_stress's sensor) at 0.1 m"""
    p = workloads.GlobalMappingParams()
    traj = synth.loop_trajectory(64, 4, side=300.0)
    pts, cov = workloads.make_scan(synth.make_blocks_scene(), "os1_64", traj[70], synth.rng_for(401, 70), max_points=p.submap_target_num_points)
    xyz, cov6 = oracle.pack_cloud(pts, c16(cov))
    out = [oracle.GpuMap(xyz, cov6, r) for r in (0.5, 1.0)]
    pts, cov = workloads.make_scan(synth.make_hall_scene(), "mid360", synth.arc_trajectory(2, step=0.5)[0], synth.rng_for(501, 0), n_rays=200_000)
    xyz, cov6 = oracle.pack_cloud(pts, c16(cov))
    out.append(oracle.GpuMap(xyz, cov6, 0.1))
    return out


def queries(m, box, rng):
    keys = np.asarray(m.buckets[m.buckets[:, 3] >= 0][:, :3], np.int64)
    d = np.stack(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1], indexing="ij"), -1).reshape(-1, 3)
    near = (keys[:, None, :] + d[None, :, :]).reshape(-1, 3)  # every key and its 26 neighbours
    rand = rng.integers(-(1 << 20), 1 << 20, size=(200_000, 3))
    lo, ext = box[:3].astype(np.int64), box[3:].astype(np.int64)
    corners = np.stack(np.meshgrid(*[[lo[k] - 1, lo[k], lo[k] + ext[k], lo[k] + ext[k] + 1] for k in range(3)], indexing="ij"), -1).reshape(-1, 3)
    inbox = lo + rng.integers(0, ext + 1, size=(200_000, 3))
    alias = keys[rng.integers(0, len(keys), 50_000)] + rng.integers(1, 1 << 10, size=(50_000, 3)) * (1 << 14) * rng.integers(0, 2, size=(50_000, 3))
    alias = np.concatenate([alias, keys[:5000] + (1 << 14), keys[:5000] - (1 << 14)])  # equal to a key in the low 14 bits of each axis
    return np.concatenate([near, rand, corners, inbox, alias, np.zeros((1, 3), np.int64)]).astype(np.int32)


def test_index_equals_gb_lookup(pih, maps):
    rng = np.random.default_rng(0)
    for m in maps:
        ix = Index(pih, m)
        assert ix.fits and m.num_dropped_points >= 0
        q = queries(m, ix.box, rng)
        got, want = ix.lookup(q), ix.gb_lookup(q)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (m.resolution, len(bad), q[bad[:5]], got[bad[:5]], want[bad[:5]])
        assert (want >= 0).sum() >= m.num_voxels - m.num_dropped_points  # every held key was asked for, and found


def test_index_is_a_fixed_point_of_insertion_order(pih, maps):
    """the index holds every key the buckets hold, in ascending-index slot order, and marks exactly the sets that overflowed"""
    m = maps[0]
    ix = Index(pih, m)
    nsets = m.num_buckets >> SET_SHIFT
    s = ix.slots
    full = s != np.uint64(0xFFFFFFFFFFFFFFFE)
    held = np.sort((s[full] >> np.uint64(43)).astype(np.int64))
    assert np.array_equal(held, np.sort(m.buckets[m.buckets[:, 3] >= 0][:, 3]))
    assert (s[1::2][~full[0::2]] == np.uint64(0xFFFFFFFFFFFFFFFE)).all()  # an empty entry 0 has an empty entry 1
    assert not (s[1::2] & np.uint64(1)).any()  # the overflow bit lives in entry 0
    assert nsets * 2 == len(s)


def test_box_that_does_not_fit(pih):
    """a map wider than 14 bits of voxels per axis gets no index (the sweep then runs sweep5)"""
    rng = np.random.default_rng(1)
    xyz = np.concatenate([rng.normal(0, 1, (2000, 4)), rng.normal(0, 1, (2000, 4)) + [MAX_EXTENT + 2, 0, 0, 0]])
    xyz[:, 3] = 1.0
    cov = np.zeros((len(xyz), 4, 4))
    cov[:, :3, :3] = np.eye(3) * 0.01
    assert not Index(pih, oracle.GpuMap(*oracle.pack_cloud(xyz, c16(cov)), 1.0)).fits
    assert Index(pih, oracle.GpuMap(*oracle.pack_cloud(xyz[:2000], c16(cov[:2000])), 1.0)).fits


def test_concurrent_insertion_builds_the_sequential_index(pih, maps):
    """k_table_finalize inserts every voxel at once with atomicCAS / atomicOr: 16 threads inserting in shuffled orders with the
    same atomics must leave every slot as the sequential insertion in ascending voxel index does"""
    for m in maps + [oracle.GpuMap(*oracle.pack_cloud(*(lambda p, c: (p, c16(c)))(*dense_block())), 0.1)]:
        seq = Index(pih, m)
        for seed in range(3):
            par = Index(pih, m, threads=16, seed=seed)
            assert par.fits == seq.fits
            assert np.array_equal(par.slots, seq.slots), (m.resolution, seed, int((par.slots != seq.slots).sum()))


def test_dense_block_overflows_and_walks(pih):
    """the dense block of test_probe_index_gpu.py: sets overflow, some keys are found only by the walk past their home set,
    and every answer is gb_lookup's"""
    pts, cov = dense_block()
    m = oracle.GpuMap(*oracle.pack_cloud(pts, c16(cov)), 0.1)
    ix = Index(pih, m)
    assert ix.fits and ix.overflowing_sets() > 100
    keys = m.buckets[m.buckets[:, 3] >= 0][:, :3]
    got, rounds = ix.lookup(keys, rounds=True)
    assert np.array_equal(got, ix.gb_lookup(keys)) and (got >= 0).all()
    assert (rounds >= 2).sum() > 100


@pytest.mark.parametrize("init_buckets,fits", [(1, False), (2, True), (16384, True)])
def test_empty_map(pih, init_buckets, fits):
    """a map without voxels: a table of one bucket has no set and gets no index; a larger one gets an empty index whose box
    holds only (0, 0, 0), where a NaN point lands, and every lookup misses"""
    pts = np.full((64, 4), np.nan)
    m = oracle.GpuMap(*oracle.pack_cloud(pts, c16(np.zeros((64, 4, 4)))), 0.5, init_buckets=init_buckets)
    assert (m.num_voxels, m.num_buckets) == (0, init_buckets)
    ix = Index(pih, m)
    assert ix.fits == fits
    if fits:
        q = np.array([[0, 0, 0], [1, 0, 0], [-1, -1, -1], [5, 7, 9]], np.int32)
        assert (ix.lookup(q) == -1).all() and (ix.gb_lookup(q) == -1).all()
