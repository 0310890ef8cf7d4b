"""CPU-only checks of the device point grid and its GICP factor (no GPU needed):
  * the numpy restatement's correspondences (tests/grid_oracle.py) against an independent fp64 search (scipy's cKDTree) on
    every query but those within an explicit margin of a tie or of the bound, which are counted;
  * the restatement's fp64 linearize against finite differences of its error;
  * the correspondence search as k_gicp_grid_sweep compiles it (glim_b200/csrc/gb_grid_math.cuh, built here with g++) against
    the restatement, bit for bit, on adversarial inputs: points on cell faces, pairs at exactly the fp32 bound, equidistant
    ties, NaN / Inf / far queries, and search half-widths m = 1, 2, 3;
  * the bound: on those inputs every target point with d2 below the bound lies within m cells of its query;
  * host validation of the arguments gb_point_grid_build / gb_gicp_grid_factor_create reject before they touch a device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree

from glim_b200 import synth
from oracle import oracle
from tests import grid_oracle as go
from tests import voxelmap_oracle as vo
from tests.util import cov_colmajor16

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


@pytest.fixture(scope="module")
def frames():
    return vo.arc_frames(4, 32 * 150, nan_frame=2)


def packed(frame):
    pts, cov, _ = frame
    return oracle.pack_cloud(pts, cov_colmajor16(cov))


def delta(frames, a, b):
    return synth.inv_pose(frames[a][2]) @ frames[b][2]


def test_build_rule(frames):
    """Cells ascending by packed key, each cell's points ascending by original index and keyed to it by the fp32 rule, the
    keyless (NaN) points last, every point stored once, the table finding every cell."""
    xyz, cov6 = packed(frames[2])
    g = go.PointGrid(xyz, cov6, 0.5)
    assert g.num_points == len(xyz) and sorted(g.index) == list(range(len(xyz)))
    assert np.array_equal(g.xyz[np.argsort(g.index)], xyz, equal_nan=True) and np.array_equal(g.cov6[np.argsort(g.index)], cov6)
    nan = ~np.isfinite(xyz).all(1)
    assert nan.sum() > 0 and g.num_keyed == len(xyz) - nan.sum()
    assert set(g.index[g.num_keyed:]) == set(np.nonzero(nan)[0])
    assert (g.keys[1:] > g.keys[:-1]).all()
    for v in range(g.num_cells):
        f, n = int(g.first[v]), int(g.counts[v])
        assert (np.diff(g.index[f:f + n]) > 0).all()
        c = np.floor((g.xyz[f:f + n] * g.inv).astype(F32))
        assert (c == g.vcoord[v]).all()
    assert g.counts.sum() == g.num_keyed
    assert g.key_extent == int(np.maximum(-g.vcoord, g.vcoord + 1).max())
    empty = go.PointGrid(np.zeros((0, 3), F32), np.zeros((0, 6), F32), 1.0)
    assert empty.num_cells == 0 and empty.num_points == 0 and empty.key_extent == 0


@pytest.mark.parametrize("max_corr", [0.3, 1.0, 2.0])
def test_restatement_matches_an_exact_kdtree(frames, max_corr):
    """The restated correspondence is the nearest target point within the bound: on every query outside a 1e-6 relative margin
    of a tie (the two nearest distances) or of the bound, its original index is cKDTree's (fp64 on the same fp32 points and
    queries), and a query without a match has no target point within the bound.  The margin queries are counted: few."""
    xyz_t, cov_t = packed(frames[0])
    xyz_s, _ = packed(frames[1])
    g = go.PointGrid(xyz_t, cov_t, 1.0)
    T = synth.perturb(delta(frames, 0, 1), synth.rng_for(71), 0.01, 0.1)
    q = go.io.transform_f32(T, xyz_s)
    corr = go.nearest(g, q, go.max_d2(max_corr))
    tree = cKDTree(g.xyz[:g.num_keyed].astype(np.float64))
    dist, idx = tree.query(q.astype(np.float64), k=2)
    d1, d2 = dist[:, 0] ** 2, dist[:, 1] ** 2
    r2 = float(go.max_d2(max_corr))
    margin = 1e-6 * np.maximum(d1, 1e-6)
    near_tie = np.abs(d2 - d1) <= margin
    near_bound = np.abs(d1 - r2) <= 1e-6 * r2
    clear = ~(near_tie | near_bound)
    within = d1 < r2
    assert within.sum() > 1000
    got = np.where(corr >= 0, g.index[np.maximum(corr, 0)], -1)
    want = np.where(within, g.index[idx[:, 0]], -1)
    assert np.array_equal(got[clear], want[clear])
    assert (near_tie | near_bound).sum() <= 0.002 * len(q), (near_tie.sum(), near_bound.sum())


def test_fp64_linearize_matches_finite_differences(frames):
    """The restated grid linearize: along any tangent direction the error's central difference (correspondences and M fixed)
    equals 2 b_s . xi, and H_ss = J^T M J of the finite-difference Jacobian."""
    xyz_t, cov_t = packed(frames[0])
    xyz, cov6 = packed(frames[1])
    g = go.PointGrid(xyz_t, cov_t, 1.0)
    T = np.asarray(synth.perturb(delta(frames, 0, 1), synth.rng_for(72), 0.02, 0.2), dtype=F32).astype(np.float64)
    lin, corr = go.linearize(g, xyz, cov6, T, 1.0)
    assert lin["num_inliers"] > 100
    a, _, r, M = go.io.residuals(g, xyz, cov6, T, corr)
    mu = g.xyz[corr[corr >= 0]].astype(np.float64)

    def resid(xi):
        Tq = T @ synth.se3_exp(xi)
        return mu - (a @ Tq[:3, :3].T + Tq[:3, 3])

    def err(xi):
        rr = resid(xi)
        return float(np.einsum("ni,nij,nj->", rr, M, rr))

    h = 1e-5
    J = np.stack([(resid(h * e) - resid(-h * e)) / (2 * h) for e in np.eye(6)], 2)
    assert np.linalg.norm(np.einsum("nki,nkl,nlj->ij", J, M, J) - lin["H_ss"]) < 1e-6 * np.linalg.norm(lin["H_ss"])
    assert np.linalg.norm(np.einsum("nki,nkl,nl->i", J, M, r) - lin["b_s"]) < 1e-6 * np.linalg.norm(lin["b_s"])
    assert abs(err(np.zeros(6)) - lin["error"]) < 1e-9 * lin["error"]
    rng = np.random.default_rng(7)
    for _ in range(3):
        xi = rng.normal(size=6)
        xi /= np.linalg.norm(xi)
        fd = (err(h * xi) - err(-h * xi)) / (2 * h)
        assert abs(fd - 2 * lin["b_s"] @ xi) < 1e-5 * np.linalg.norm(2 * lin["b_s"]) + 1e-6 * lin["error"]
    # error(): correspondences of T_lin evaluated at T_eval
    Te = T @ synth.se3_exp(np.full(6, 1e-3))
    assert go.error(g, xyz, cov6, T, Te, 1.0) == go.linearize(g, xyz, cov6, Te, 1.0, corr=corr)[0]["error"]


# ---------------------------------------------------------------------------------------------------------------------
# the host-compiled search
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("gs") / "libgrid_search_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so, os.path.join(ROOT, "tests", "cpp", "grid_search_host.cpp")])
    L = C.CDLL(so)
    vp = C.c_void_p
    L.gs_search.argtypes = [C.c_int, vp, vp, vp, C.c_uint, C.c_int, vp, vp, C.c_int, C.c_float, C.c_float, vp]
    L.gs_search_q.argtypes = [C.c_int, vp, vp, C.c_uint, C.c_int, vp, vp, C.c_int, C.c_float, C.c_float, vp]
    L.gs_half_width.argtypes = [C.c_float, C.c_float, C.c_int]
    L.gs_half_width.restype = C.c_int
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def device_arrays(g: go.PointGrid):
    """the grid as the device holds it: 48-byte records (original index bits in slot 2.z), cells {first, count}, buckets"""
    rec = np.zeros((g.num_points, 12), F32)
    rec[:, 0:3] = g.xyz
    rec[:, 3] = g.cov6[:, 0]
    rec[:, 4:8] = g.cov6[:, 1:5]
    rec[:, 8] = g.cov6[:, 5]
    rec[:, 9] = 1.0
    rec[:, 10] = g.index.astype(np.int32).view(F32)
    cells = np.ascontiguousarray(np.stack([g.first, g.counts], 1).astype(np.int32).reshape(-1, 2))
    return np.ascontiguousarray(rec), cells, np.ascontiguousarray(g.buckets, dtype=np.int32)


def host_search_q(L, g: go.PointGrid, q, max_corr, m):
    rec, cells, buckets = device_arrays(g)
    q = np.ascontiguousarray(q, dtype=F32)
    out = np.empty(len(q), np.int32)
    L.gs_search_q(len(q), _p(q), _p(buckets), len(buckets) - 1, go.MAX_SCAN, _p(cells), _p(rec), m, g.inv, go.max_d2(max_corr), _p(out))
    return out


def adversarial(cell, max_corr, rng):
    """A target of points on cell faces and off them, with equidistant groups whose original order runs against the cell
    order, and queries: at the fp32 bound exactly and one ulp inside it, at tie centres, on faces, NaN / Inf / far away."""
    r2 = go.max_d2(max_corr)
    r = F32(np.sqrt(np.float64(r2)))
    base = np.array([3.0, -2.0, 1.0], F32) * F32(cell)  # a cell corner: every coordinate on a face
    pts = [base + F32(cell) * rng.integers(-4, 5, size=(200, 3)).astype(F32)]  # face points (exact multiples)
    pts.append(base + (rng.uniform(-4, 4, size=(300, 3)) * cell).astype(F32))
    queries = [base.copy()]
    # ties: a centre with points at the same fp32 offsets along +-x, +-y, +-z (distance 0.7 r: inside the bound)
    for k in range(6):
        c = base + F32(cell) * rng.integers(-3, 4, size=3).astype(F32) + F32(0.25 * cell)
        dd = F32(0.7) * r
        ring = np.array([[dd, 0, 0], [-dd, 0, 0], [0, dd, 0], [0, -dd, 0], [0, 0, dd], [0, 0, -dd]], F32)
        pts.append((c + ring[::-1] if k % 2 else c + ring).astype(F32))
        queries.append(c)
    # pairs at the bound: with r and q dyadic, p = q + (r, 0, 0) is exact and d2 = r * r = (float)(r^2) exactly; and one ulp
    # of r either side
    for k in range(8):
        qb = (base + rng.integers(-192, 193, size=3).astype(F32) / F32(64)).astype(F32)
        for dr in (r, np.nextafter(r, F32(0)), np.nextafter(r, F32(np.inf))):
            p = qb.copy()
            p[k % 3] = F32(p[k % 3] + dr)
            pts.append(p[None, :])
        queries.append(qb)
    queries += [np.array([np.nan, 0, 0], F32), np.array([np.inf, 1, 1], F32), np.array([-np.inf, np.inf, np.nan], F32),
                np.array([1e30, -1e30, 0], F32), np.array([1e8, 0, 0], F32), np.array([3e9, 3e9, 3e9], F32)]
    queries.append((base + (rng.uniform(-5, 5, size=(400, 3)) * cell)).astype(F32))
    P = np.concatenate([np.atleast_2d(x) for x in pts]).astype(F32)
    Q = np.concatenate([np.atleast_2d(x) for x in queries]).astype(F32)
    perm = rng.permutation(len(P))  # original indices in no relation to the cells
    return P[perm], Q


# r (dyadic, so that pairs can sit exactly at the bound) below, above and well above the 0.5 m cell
RADII = [(0.375, 1), (0.75, 2), (1.3125, 3)]


@pytest.mark.parametrize("max_corr,want_m", RADII)
def test_host_build_of_the_search_matches_restatement(gs, max_corr, want_m):
    """r below, above and well above the cell size (m = 1, 2, 3): the host-compiled grid_nearest equals the brute-force
    restatement bit for bit on the adversarial inputs; ties are decided by original index, a pair at exactly the bound does
    not match, NaN / Inf / far queries find nothing."""
    rng = np.random.default_rng(int(max_corr * 64))
    cell = 0.5
    P, Q = adversarial(cell, max_corr, rng)
    g = go.PointGrid(P, np.tile(np.arange(6, dtype=F32), (len(P), 1)), cell)
    m = go.half_width(g.inv, go.max_d2(max_corr), g.key_extent)
    assert m == want_m == gs.gs_half_width(g.inv, go.max_d2(max_corr), g.key_extent)
    got = host_search_q(gs, g, Q, max_corr, m)
    want = go.nearest(g, Q, go.max_d2(max_corr))
    assert np.array_equal(got, want)
    assert (got[~np.isfinite(Q).all(1)] == -1).all() and (got[np.abs(Q).max(1) >= 1e8] == -1).all()
    d2 = go.d2_matrix(Q, g.xyz)
    ties = ((d2 == d2.min(1, keepdims=True)) & (d2 < go.max_d2(max_corr))).sum(1) > 1
    assert ties.sum() >= 6  # the tie centres
    at_bound = (d2 == go.max_d2(max_corr)).any(1)
    assert at_bound.sum() >= 1
    # the same search through the sweep's transform, at a pose
    T = synth.pose(0.3, -0.2, 0.1, 0.4, 0.05, -0.02)
    src = (Q[np.isfinite(Q).all(1)] - np.array([0.3, -0.2, 0.1], F32)).astype(F32)
    rec, cells, buckets = device_arrays(g)
    out = np.empty(len(src), np.int32)
    gs.gs_search(len(src), _p(np.ascontiguousarray(src)), _p(oracle.pose_colmajor(T)), _p(buckets), len(buckets) - 1, go.MAX_SCAN, _p(cells), _p(rec), m,
                 g.inv, go.max_d2(max_corr), _p(out))
    assert np.array_equal(out, go.correspondences(g, src, T, max_corr))


@pytest.mark.parametrize("max_corr", [r for r, _ in RADII])
def test_half_width_bounds_every_match(gs, max_corr):
    """The proof of grid_half_width on the adversarial inputs and on pairs near the bound far from the origin (where the fp32
    products round most): every target point with d2 < (float)(r^2) is within m cells of its query's cell on every axis."""
    rng = np.random.default_rng(100 + int(max_corr * 64))
    cell = 0.5
    thr = go.max_d2(max_corr)
    P, Q = adversarial(cell, max_corr, rng)
    far = np.array([4.0e4, -3.0e4, 1.0e3], F32)  # about 2^17 cells out
    Qf = (far + rng.uniform(-1, 1, size=(300, 3)) * cell).astype(F32)
    u = rng.normal(size=(300, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    Pf = (Qf + (u * (max_corr * rng.uniform(0.97, 1.0, size=(300, 1))))).astype(F32)
    for P_, Q_ in ((P, Q), (np.concatenate([P, Pf]), Qf)):
        g = go.PointGrid(P_, np.zeros((len(P_), 6), F32), cell)
        m = go.half_width(g.inv, thr, g.key_extent)
        assert m == gs.gs_half_width(g.inv, thr, g.key_extent)
        fin = np.isfinite(Q_).all(1) & (np.abs(Q_).max(1) < 1e7)
        cq = go.io.fp32_coords(Q_[fin], g.inv)
        d2 = go.d2_matrix(Q_[fin], g.xyz[:g.num_keyed])
        qi, pi = np.nonzero(d2 < thr)
        assert len(qi) > 100
        cp = go.io.fp32_coords(g.xyz[:g.num_keyed], g.inv)
        assert np.abs(cp[pi] - cq[qi]).max() <= m
    # the width grows with the extent only by the rounding terms, and never below r / cell
    for K in (1, 100, 1 << 17, 1 << 20):
        for rr in (0.3, 0.49, 0.51, 0.99, 1.01, 2.0, 3.9):
            mm = go.half_width(F32(1.0 / cell), go.max_d2(rr), K)
            assert mm == gs.gs_half_width(F32(1.0 / cell), go.max_d2(rr), K)
            assert mm >= int(np.ceil(rr / cell - 1e-9))
    assert go.half_width(F32(2.0), go.max_d2(1.0), 1 << 20) == 3  # 2 cells plus 2 x 2^20 x 2^-24 of rounding
    assert gs.gs_half_width(F32(2.0), go.max_d2(4.5), 10) == go.MAX_HALF_WIDTH + 1


def test_invalid_arguments_are_rejected_on_the_host():
    """Every rejected value fails with GB_ERR_INVALID_ARGUMENT before the call looks for a device, creating nothing."""
    from glim_b200 import capi

    L = capi.lib()
    dummy = C.c_void_p(1)  # never dereferenced: validation comes first
    h = C.c_void_p()
    for cs in (0.0, -1.0, float("nan"), float("inf")):
        assert L.gb_point_grid_build(dummy, dummy, cs, C.byref(h)) == 1, cs
    for d in (0.0, -1.0, float("nan"), float("inf")):
        assert L.gb_gicp_grid_factor_create(dummy, dummy, dummy, d, C.byref(h)) == 1, d
    assert L.gb_point_grid_build(None, None, 1.0, C.byref(h)) == 1
    assert L.gb_gicp_grid_factor_create(None, None, None, 2.0, C.byref(h)) == 1
    assert L.gb_point_grid_info(None, None, None, None) == 1
    assert L.gb_point_grid_download(None, None, None, None, None, None) == 1
    assert L.gb_point_grid_destroy(None) == 0
    assert not h.value
