"""CPU-only checks of the device iVox and its GICP factor (no GPU needed):
  * properties of the numpy restatement of the insert rule (tests/ivox_oracle.py) over an insert sequence with LRU eviction,
    NaN points and an empty insert, its eviction against the oracle's GaussianVoxelMapCPU (go_cpumap);
  * the fp64 GICP linearize of the restatement against finite differences of its error;
  * the correspondence search as k_gicp_sweep compiles it (glim_b200/csrc/gb_ivox_math.cuh, built here with g++) against the
    restatement, bit for bit;
  * host validation of every argument gb_ivox_create / gb_ivox_insert / gb_gicp_factor_create reject (these return before
    they touch a device)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from glim_b200 import synth
from oracle import oracle
from tests import ivox_oracle as io
from tests import voxelmap_oracle as vo
from tests.util import cov_colmajor16

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_FRAMES = 20
NAN_FRAME = 7
EMPTY_INSERT = 12


def rate_of(k):
    if k == EMPTY_INSERT:
        return 1e-9  # keeps no point
    return 1.0 if k < 5 else 0.1


@pytest.fixture(scope="module")
def frames():
    return vo.arc_frames(N_FRAMES, 32 * 120, nan_frame=NAN_FRAME)


def packed(frame):
    pts, cov, _ = frame
    return oracle.pack_cloud(pts, cov_colmajor16(cov))


def test_insert_properties_and_eviction(frames):
    """Over 20 inserts (LRU horizon 6, cycle 2): no voxel holds more than the cap, no two points of a voxel are closer than
    min_dist, and the surviving voxels are exactly those of GaussianVoxelMapCPU (go_cpumap)
    fed the same kept points with the same LRU setting."""
    res, min_dist, cap = 0.5, 0.1, 4
    iv = io.IVox(res, min_dist=min_dist, max_points=cap, mode=7, lru_horizon=6, lru_clear_cycle=2)
    cm = oracle.CpuMap(res)
    cm.set_lru_horizon(6, clear_cycle=2)
    shrank, full = 0, 0
    for k, frame in enumerate(frames):
        xyz, cov6 = packed(frame)
        T = frame[2]
        before = iv.num_voxels
        iv.insert(xyz, cov6, T, rate_of(k), seed=300 + k)
        keep = vo.sample_mask(len(xyz), rate_of(k), 300 + k)
        q, _ = vo.transform(T, xyz, cov6)
        _, ok = io.coords64(q, res)
        sel = keep & ok
        q4 = np.concatenate([q[sel], np.ones((int(sel.sum()), 1))], 1)
        cm.insert(q4, np.zeros((int(sel.sum()), 16)))
        shrank += iv.num_voxels < before
        full = max(full, int((iv.counts == cap).sum()))
        assert (iv.counts >= 1).all() and (iv.counts <= cap).all(), k
        for v in range(iv.num_voxels):
            f, n = int(iv.first[v]), int(iv.counts[v])
            p = iv.xyz[f:f + n].astype(np.float64)
            d2 = ((p[:, None, :] - p[None, :, :]) ** 2).sum(-1)
            assert (d2[~np.eye(n, dtype=bool)] >= min_dist ** 2).all(), (k, v)
        assert cm.num_voxels == iv.num_voxels, k
        for c in iv.vcoord:
            assert cm.lookup((c + 0.5) * res)[0] >= 0, (k, c)
    assert shrank > 0 and full > 0  # eviction happened, and voxels reached the cap
    assert iv.counter == N_FRAMES


def test_empty_insert_still_counts():
    iv = io.IVox(1.0, lru_horizon=1, lru_clear_cycle=1)
    iv.insert(np.zeros((1, 3), np.float32), np.zeros((1, 6), np.float32))
    assert iv.num_voxels == 1
    iv.insert(np.zeros((0, 3), np.float32), np.zeros((0, 6), np.float32))  # c = 2: stamp 0 + 1 < 2
    assert iv.num_voxels == 0 and iv.counter == 2


def test_fp64_linearize_matches_finite_differences(frames):
    """The restated GICP linearize: H_ss is J^T M J and b_s = J^T M r of the fixed correspondences, so along any tangent
    direction the error's central difference equals 2 b_s . xi (error = sum r^T M r, no 1/2)."""
    iv = io.IVox(1.0, mode=7)
    for k in (0, 1):
        xyz, cov6 = packed(frames[k])
        iv.insert(xyz, cov6, frames[k][2])
    xyz, cov6 = packed(frames[2])
    T = synth.perturb(frames[2][2], synth.rng_for(61), 0.02, 0.2)
    T = np.asarray(T, dtype=np.float32).astype(np.float64)  # the restatement evaluates at the fp32-cast pose
    lin, corr = io.linearize(iv, xyz, cov6, T, 2.0)
    assert lin["num_inliers"] > 100
    # the residual Jacobian J_s by central differences of r(T Exp(xi)) in fp64, correspondences and M fixed at T
    a, q, r, M = io.residuals(iv, xyz, cov6, T, corr)
    mu = iv.xyz[corr[corr >= 0]].astype(np.float64)

    def resid(xi):  # r at T Exp(xi), correspondences and M fixed at T
        Tq = T @ synth.se3_exp(xi)
        return mu - (a @ Tq[:3, :3].T + Tq[:3, 3])

    def err(xi):
        rr = resid(xi)
        return float(np.einsum("ni,nij,nj->", rr, M, rr))

    h = 1e-5
    J = np.stack([(resid(h * e) - resid(-h * e)) / (2 * h) for e in np.eye(6)], 2)  # (n, 3, 6)
    assert np.linalg.norm(np.einsum("nki,nkl,nlj->ij", J, M, J) - lin["H_ss"]) < 1e-6 * np.linalg.norm(lin["H_ss"])
    assert np.linalg.norm(np.einsum("nki,nkl,nl->i", J, M, r) - lin["b_s"]) < 1e-6 * np.linalg.norm(lin["b_s"])
    assert abs(err(np.zeros(6)) - lin["error"]) < 1e-9 * lin["error"]
    # error = sum r^T M r (no 1/2): its gradient along any direction is 2 b . xi
    rng = np.random.default_rng(5)
    for _ in range(3):
        xi = rng.normal(size=6)
        xi /= np.linalg.norm(xi)
        fd = (err(h * xi) - err(-h * xi)) / (2 * h)
        assert abs(fd - 2 * lin["b_s"] @ xi) < 1e-5 * np.linalg.norm(2 * lin["b_s"]) + 1e-6 * lin["error"], (fd, 2 * lin["b_s"] @ xi)
    assert np.linalg.eigvalsh(lin["H_ss"]).min() > 0


@pytest.fixture(scope="module")
def ivs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("ivs") / "libivox_search_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so, os.path.join(ROOT, "tests", "cpp", "ivox_search_host.cpp")])
    L = C.CDLL(so)
    vp = C.c_void_p
    L.ivs_search.argtypes = [C.c_int, vp, vp, vp, C.c_uint, C.c_int, vp, vp, C.c_int, C.c_float, C.c_float, vp]
    L.ivs_offset.argtypes = [C.c_int, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_search(L, m: io.IVox, xyz, T, max_corr):
    rec = np.zeros((m.num_points, 12), np.float32)
    rec[:, 0:3] = m.xyz
    rec[:, 3] = m.cov6[:, 0]
    rec[:, 4:8] = m.cov6[:, 1:5]
    rec[:, 8] = m.cov6[:, 5]
    rec[:, 9] = 1.0
    rec = np.ascontiguousarray(rec)
    cells = np.ascontiguousarray(np.stack([m.first, m.counts], 1).astype(np.int32).reshape(-1, 2))
    buckets = np.ascontiguousarray(m.buckets, dtype=np.int32)
    src = np.ascontiguousarray(xyz, dtype=np.float32)
    Tc = oracle.pose_colmajor(T)
    out = np.empty(len(src), np.int32)
    L.ivs_search(len(src), _p(src), _p(Tc), _p(buckets), len(buckets) - 1, io.MAX_SCAN, _p(cells), _p(rec), m.mode,
                 np.float32(1.0 / m.resolution), np.float32(max_corr * max_corr), _p(out))
    return out


def test_offset_order_matches_restatement(ivs):
    d = np.zeros(3, np.int32)
    got = []
    for k in range(27):
        ivs.ivs_offset(k, _p(d))
        got.append(tuple(int(x) for x in d))
    assert got == io.offsets(27)
    assert len(set(got)) == 27


@pytest.mark.parametrize("mode", [1, 7, 19, 27])
def test_host_build_of_the_search_matches_restatement(ivs, frames, mode):
    """Correspondences of the host-compiled search equal the restatement's exactly, at poses including identity, a 180 degree
    yaw and a map at negative coordinates; the NaN points of one frame find nothing."""
    iv = io.IVox(0.5 if mode > 1 else 1.0, mode=mode, max_points=6)
    shift = np.eye(4)
    shift[:3, 3] = [-40.0, -25.0, -3.0]  # the whole map at negative coordinates
    for k in (0, 1, 2):
        xyz, cov6 = packed(frames[k])
        iv.insert(xyz, cov6, shift @ frames[k][2])
    yaw = np.eye(4)
    yaw[:2, :2] = [[-1.0, 0.0], [0.0, -1.0]]
    xyz, _ = packed(frames[3])
    nan_xyz, _ = packed(frames[NAN_FRAME])
    poses = [np.eye(4), shift @ frames[3][2], shift @ synth.perturb(frames[3][2], synth.rng_for(62), 0.05, 0.5), shift @ frames[3][2] @ yaw]
    hits = 0
    for T in poses:
        for src in (xyz, nan_xyz):
            got = host_search(ivs, iv, src, T, 1.0)
            want = io.correspondences(iv, src, T, 1.0)
            assert np.array_equal(got, want)
            hits += int((got >= 0).sum())
            assert (got[~np.isfinite(src).all(1)] == -1).all()
    assert hits > 1000


def test_fmaf_emulation_is_correctly_rounded():
    """the restatement's fp32 fma against exact rational arithmetic on random and halfway-constructed inputs"""
    from fractions import Fraction
    rng = np.random.default_rng(9)
    a = rng.normal(size=400).astype(np.float32)
    b = rng.normal(size=400).astype(np.float32)
    c = rng.normal(size=400).astype(np.float32)
    c[:100] = (-(a[:100].astype(np.float64) * b[:100].astype(np.float64))).astype(np.float32)  # heavy cancellation
    got = io.fmaf(a, b, c)
    for x, y, z, g in zip(a, b, c, got):
        exact = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        lo = np.float32(float(exact))
        cands = {lo, np.nextafter(lo, np.float32(np.inf)), np.nextafter(lo, np.float32(-np.inf))}
        best = min(cands, key=lambda f: (abs(Fraction(float(f)) - exact), int(np.float32(f).view(np.int32)) & 1))
        assert g == best, (x, y, z, g, best)


def test_invalid_arguments_are_rejected_on_the_host():
    """Every rejected argument fails with GB_ERR_INVALID_ARGUMENT before the call looks for a device."""
    from glim_b200 import capi

    L = capi.lib()
    dummy = C.c_void_p(1)  # never dereferenced: validation comes first
    h = C.c_void_p()
    good = dict(resolution=1.0, min_dist=0.1, cap=10, mode=1, horizon=100, cycle=10)

    def create(**kw):
        a = dict(good, **kw)
        return L.gb_ivox_create(dummy, a["resolution"], a["min_dist"], a["cap"], a["mode"], a["horizon"], a["cycle"], C.byref(h))

    for r in (0.0, -1.0, float("nan"), float("inf")):
        assert create(resolution=r) == 1, r
    assert create(min_dist=-0.01) == 1
    assert create(min_dist=float("nan")) == 1
    for cap in (0, -1, 65):
        assert create(cap=cap) == 1, cap
    for mode in (0, 2, 6, 8, 26, 28):
        assert create(mode=mode) == 1, mode
    for cycle in (0, -3):
        assert create(cycle=cycle) == 1, cycle
    assert not h.value
    assert L.gb_ivox_create(None, 1.0, 0.1, 10, 1, 100, 10, C.byref(h)) == 1
    # insert: sampling rate and pose are checked before the handles are read
    T = capi.pose16(np.eye(4))
    for rate in (0.0, -0.5, 1.0000001, float("nan")):
        assert L.gb_ivox_insert(dummy, dummy, dummy, capi.ptr(T), rate, 0) == 1, rate
    for bad in (np.nan, np.inf):
        Tb = T.copy()
        Tb[13] = bad
        assert L.gb_ivox_insert(dummy, dummy, dummy, capi.ptr(Tb), 1.0, 0) == 1
    assert L.gb_ivox_insert(None, None, None, None, 1.0, 0) == 1
    for d in (0.0, -1.0, float("nan"), float("inf")):
        assert L.gb_gicp_factor_create(dummy, dummy, dummy, d, C.byref(h)) == 1, d
    assert L.gb_gicp_factor_create(None, None, None, 2.0, C.byref(h)) == 1
    assert not h.value
