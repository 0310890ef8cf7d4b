"""CPU-only checks of the map segmentation (no GPU needed):
  * the per-point and per-pair functions of glim_b200/csrc/gb_segment_math.cuh, compiled for the host
    (tests/cpp/segment_math_host.cpp), against the numpy restatement (tests/segment_oracle.py) on seeded and adversarial inputs:
    NaN and zero normals, coincident points, d2 exactly at the bound, saturated keys;
  * the union-find hook run sequentially on random edge lists agrees with scipy's connected_components, whatever the order;
  * the oracle itself against a pure-Python breadth-first search on small scenes;
  * the arguments gb_region_growing and gb_concat_frames reject before they touch a device."""
import ctypes as C
import math
import os
import subprocess
from collections import deque

import numpy as np
import pytest

from tests import segment_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = np.float32, np.float64


@pytest.fixture(scope="module")
def hl(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("seg") / "libsegment_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", out,
                           os.path.join(ROOT, "tests", "cpp", "segment_math_host.cpp")])
    L = C.CDLL(out)
    vp = C.c_void_p
    L.keyed.argtypes = [C.c_int, vp, C.c_float, vp]
    L.edge.argtypes = [C.c_int, vp, vp, vp, vp, C.c_float, C.c_double, vp]
    L.seed_keys.argtypes = [C.c_int, vp, vp, vp]
    L.rotate_normals.argtypes = [C.c_int, vp, vp, vp]
    L.in_window.argtypes = [C.c_int, vp, C.c_double, vp, vp, vp]
    L.union_find.argtypes = [C.c_int, C.c_int, vp, vp, vp]
    return L


def p(a):
    return a.ctypes.data_as(C.c_void_p)


def c(a, dt):
    return np.ascontiguousarray(a, dtype=dt)


def unit(rng, n):
    v = rng.normal(size=(n, 3))
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(F32)


def test_keyed_matches_oracle(hl):
    rng = np.random.default_rng(1)
    cell = 0.21
    inv = F32(1.0 / cell)
    edge = float(1 << 20) / float(inv)
    xyz = np.concatenate([rng.uniform(-100, 100, (500, 3)), rng.uniform(-1, 1, (200, 3)) * edge * 1.5,
                          [[np.nan, 0, 0], [np.inf, 0, 0], [0, -np.inf, 0], [3e38, 0, 0], [-3e38, 1, 1]]]).astype(F32)
    xyz = c(xyz, F32)
    out = np.empty(len(xyz), np.int32)
    hl.keyed(len(xyz), p(xyz), inv, p(out))
    ref = so.keyed(xyz, cell)
    assert np.array_equal(out.astype(bool), ref)
    assert ref.sum() > 500 and (~ref).sum() > 50  # both sides of the range are exercised


def test_edge_matches_oracle(hl):
    rng = np.random.default_rng(2)
    n = 4000
    a = rng.uniform(-50, 50, (n, 3)).astype(F32)
    b = (a + rng.normal(scale=0.3, size=(n, 3))).astype(F32)
    na, nb = unit(rng, n), unit(rng, n)
    nb[: n // 4] = na[: n // 4]                        # parallel normals
    nb[n // 4: n // 4 + 50] = -na[n // 4: n // 4 + 50]  # opposite normals
    na[100:110] = np.nan                               # NaN normals never join
    na[110:120] = 0                                    # zero normals: dot 0
    b[200:220] = a[200:220]                            # coincident points
    dt = 0.5
    max_d2 = F32(dt * dt)
    d2 = so.point_d2(a, b)
    b[300] = a[300]
    b[300, 0] = a[300, 0] + F32(0.5)                   # d2 exactly at the bound: not joined
    assert so.point_d2(a[300], b[300]) == max_d2
    for ang in (0.0, 0.3, math.pi / 2, 2.5, math.pi):
        cos_t = math.cos(ang)
        out = np.empty(n, np.int32)
        hl.edge(n, p(c(a, F32)), p(c(na, F32)), p(c(b, F32)), p(c(nb, F32)), max_d2, cos_t, p(out))
        ref = (so.point_d2(a, b) < max_d2) & so.normals_join(na, nb, cos_t)
        assert np.array_equal(out.astype(bool), ref), ang
        assert not out[100:110].any() and not out[300]
    assert (d2 < max_d2).sum() > 100


def test_seed_keys_order_as_the_oracle(hl):
    rng = np.random.default_rng(3)
    xyz = rng.uniform(-5, 5, (3000, 3)).astype(F32)
    xyz[10] = xyz[20] = xyz[5]  # ties: the smaller index wins
    xyz[30] = np.nan
    xyz[31, 2] = np.inf
    for q in (xyz[5].astype(F64), np.array([100.0, -3.0, 2.0]), np.array([0.1, 0.2, 0.3])):
        keys = np.empty(len(xyz), np.uint64)
        qf = c(q, F32)
        hl.seed_keys(len(xyz), p(c(xyz, F32)), p(qf), p(keys))
        assert keys[30] == keys[31] == np.uint64(~0 & (2**64 - 1))
        assert int(np.argmin(keys)) == so.seed_of(xyz, q)
    bad = np.full((4, 3), np.nan, F32)
    assert so.seed_of(bad, [0, 0, 0]) == -1


def test_rotate_normals_and_window_match_oracle(hl):
    rng = np.random.default_rng(4)
    n = 2000
    nrm = unit(rng, n)
    nrm[:5] = 0
    nrm[5:8] = np.nan
    for _ in range(4):
        q = rng.normal(size=4)
        w, x, y, z = q / np.linalg.norm(q)
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                      [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        T = np.eye(4)
        T[:3, :3] = R
        T[:3, 3] = rng.uniform(-100, 100, 3)
        out = np.empty((n, 3), F32)
        hl.rotate_normals(n, p(c(R, F64)), p(c(nrm, F32)), p(out))
        ref = so.rotate_normals(T, nrm).astype(F32)
        assert np.array_equal(out, ref, equal_nan=True)
    cell = 2.0
    qq = np.concatenate([rng.uniform(-30, 30, (3000, 3)), [[np.nan, 0, 0], [np.inf, 1, 1], [4.0, 6.0, 8.0], [-10.0, -8.0, -6.0]]])
    lo, hi = np.array([-5, -4, -3], np.int32), np.array([2, 3, 4], np.int32)
    out = np.empty(len(qq), np.int32)
    hl.in_window(len(qq), p(c(qq, F64)), 1.0 / cell, p(lo), p(hi), p(out))
    ref = so.in_window(qq, cell, lo, hi)
    assert np.array_equal(out.astype(bool), ref)
    assert ref.sum() > 50 and not ref[-4] and not ref[-3] and ref[-2] and ref[-1]  # faces of the window are inclusive


@pytest.mark.parametrize("seed", range(5))
def test_union_find_agrees_with_connected_components(hl, seed):
    rng = np.random.default_rng(10 + seed)
    n = int(rng.integers(1, 3000))
    m = int(rng.integers(0, 2 * n))
    e = rng.integers(0, n, (m, 2))
    if seed == 0:  # a chain given from its far end: the worst order for a naive hook
        e = np.stack([np.arange(n - 1, 0, -1), np.arange(n - 2, -1, -1)], axis=1)
    e = e[e[:, 0] != e[:, 1]]
    lo, hi = np.minimum(e[:, 0], e[:, 1]), np.maximum(e[:, 0], e[:, 1])
    ref = so.component_labels(n, np.stack([lo, hi], axis=1), np.ones(n, bool))
    for order in (np.arange(len(e)), rng.permutation(len(e))):
        ee = c(np.stack([lo, hi], axis=1)[order], np.int32)
        parent, labels = np.empty(n, np.int32), np.empty(n, np.int32)
        hl.union_find(n, len(ee), p(ee), p(parent), p(labels))
        assert np.array_equal(labels, ref)
        assert (parent <= np.arange(n)).all()  # every parent is an ancestor with a smaller index


def bfs_region(xyz, nrm, seed_point, dt, ang, dil):
    """a plain breadth-first restatement over all pairs, for small scenes"""
    n = len(xyz)
    fin = so.finite(xyz)
    k = so.keyed(xyz, 1.05 * dt)
    cos_t = math.cos(ang)
    adj = [[] for _ in range(n)]
    for i in range(n):
        for j in range(i + 1, n):
            if k[i] and k[j] and so.point_d2(xyz[i], xyz[j]) < F32(dt * dt) and so.normals_join(nrm[i], nrm[j], cos_t):
                adj[i].append(j)
                adj[j].append(i)
    lab = np.full(n, -1)
    for s in range(n):
        if fin[s] and lab[s] < 0:
            lab[s] = s
            dq = deque([s])
            while dq:
                u = dq.popleft()
                for v in adj[u]:
                    if lab[v] < 0:
                        lab[v] = s
                        dq.append(v)
    best, seed = None, -1
    for i in range(n):
        if fin[i]:
            d = so.point_d2(xyz[i], np.asarray(seed_point, F64).astype(F32))
            if best is None or d < best:
                best, seed = d, i
    R = (lab == lab[seed]) & (lab >= 0) if seed >= 0 else np.zeros(n, bool)
    sel = R.copy()
    if dil > 0:
        kd = so.keyed(xyz, 1.05 * dil)
        for j in range(n):
            if not R[j] and kd[j]:
                sel[j] = any(R[i] and kd[i] and so.point_d2(xyz[i], xyz[j]) < F32(dil * dil) for i in range(n))
    return lab, seed, np.flatnonzero(sel)


@pytest.mark.parametrize("seed", range(3))
def test_oracle_against_breadth_first_search(seed):
    rng = np.random.default_rng(20 + seed)
    n = 150
    xyz = np.concatenate([rng.uniform(0, 3, (n // 2, 3)) * [1, 1, 0.02], rng.uniform(0, 3, (n - n // 2, 3)) * [0.02, 1, 1] + [4, 0, 0]]).astype(F32)
    nrm = np.concatenate([np.tile([0, 0, 1], (n // 2, 1)), np.tile([1, 0, 0], (n - n // 2, 1))]).astype(F32)
    nrm += rng.normal(scale=0.05, size=nrm.shape).astype(F32)
    xyz[3] = np.nan
    nrm[7] = np.nan
    xyz[8] = xyz[9]
    for dt, ang, dil in ((0.5, 0.3, 0.0), (0.4, 1.2, 1.2), (1.5, math.pi, 0.7)):
        sp = xyz[int(rng.integers(10, n))].astype(F64) + 0.01
        r = so.region_growing(xyz, nrm, sp, dt, ang, dil)
        lab, s, sel = bfs_region(xyz, nrm, sp, dt, ang, dil)
        assert np.array_equal(r["labels"], lab) and r["seed"] == s and np.array_equal(r["selected"], sel)
        assert r["num_components"] == len(set(lab[lab >= 0].tolist()))


def test_region_growing_refusals_before_any_device_work():
    from glim_b200 import capi

    L = capi.lib()
    prm = capi.RegionGrowingParams()
    assert L.gb_region_growing_default_params(C.byref(prm)) == 0
    assert (prm.distance_threshold, prm.dilation_radius) == (0.5, 0.0) and abs(prm.angle_threshold - math.radians(10)) < 1e-15
    res = capi.RegionGrowingResult()
    q = np.zeros(3)
    # a null context or cloud is refused before anything else (every other refusal needs a device and is checked there)
    assert L.gb_region_growing(None, None, p(q), C.byref(prm), C.byref(res), None, None) == 1
    ids = np.zeros(1, np.uint64)
    m = C.c_size_t()
    h = C.c_void_p()
    assert L.gb_concat_frames(None, 0, None, None, None, C.byref(h), p(ids), C.byref(m)) == 1
