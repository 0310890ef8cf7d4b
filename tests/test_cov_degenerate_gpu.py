"""Covariance / normal estimation and k-NN on degenerate inputs, on the device, against the oracle and the exact reference.

The covariance kernels run the oracle's uncontracted fp64 arithmetic (glim_b200/csrc/gb_cov_math.cuh); what remains between
device and oracle are the ulps of atan2, cos and sin, which move the eigenvalues by a few u in the solver's scaled units and
the eigenvectors by that over the gaps.  So the device bar of a row is DEV_C u (1 / g01 + 1 / g12), with the gaps of the
scaled matrix the oracle's solver works on (numpy reproduces its A exactly).  The normal's sign is compared too, except
where p . n itself is within the bar.
"""
import collections
import ctypes as C

import numpy as np
import pytest

from glim_b200 import preprocess
from glim_b200.capi import Preprocessed, lib, ptr
from oracle import oracle
from tests import cov_reference as cr
from tests import util
from tests.test_gpu_parity import _cpu_frame

pytestmark = pytest.mark.gpu

DEV_C = 32.0
GB_ERR_INVALID_ARGUMENT = 1
KNN_KS = (1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 15, 16, 20, 24, 32)


def device_bar(A):
    g01, g12 = cr.solver_gaps(A)
    with np.errstate(divide="ignore"):
        return DEV_C * cr.U * (1 / g01 + 1 / g12)


def row_diff(P, n_d, c_d, n_o, c_o, bar):
    """per row: the largest entry difference of C and of the normal; either sign of the normal counts only where
    |p . n| <= |p| bar"""
    dc = np.abs(c_d - c_o).reshape(len(c_d), -1).max(axis=1)
    dn = np.abs(n_d - n_o).max(axis=1)
    with np.errstate(invalid="ignore"):  # p = 0 with an infinite bar: the sign is firm (p . n = 0 never flips)
        amb = np.abs(np.einsum("ni,ni->n", P[:, :3], n_o[:, :3])) <= np.linalg.norm(P[:, :3], axis=1) * bar
    dn = np.where(amb, np.minimum(dn, np.abs(n_d + n_o).max(axis=1)), dn)
    return np.maximum(dc, dn)


@pytest.fixture(scope="module")
def device_battery(ctx):
    """gb_covariances on every case of the battery: one call per (k_correspondences, k_neighbors), the cases concatenated"""
    cases = cr.battery()
    groups = collections.defaultdict(list)
    for c, case in enumerate(cases):
        groups[(case["kc"], case["k"])].append(c)
    out = [None] * len(cases)
    est = preprocess.CloudCovarianceEstimation(ctx=ctx)
    for (kc, k), members in groups.items():
        offs = np.cumsum([0] + [len(cases[c]["points"]) for c in members])
        P = np.concatenate([cases[c]["points"] for c in members])
        nb = np.concatenate([cases[c]["nb"] + o for c, o in zip(members, offs[:-1])])
        normals, covs = est.estimate(P, nb, k_neighbors=k)
        for c, a, b in zip(members, offs[:-1], offs[1:]):
            out[c] = (normals[a:b], covs[a:b])
    return cases, out


def test_gb_covariances_matches_oracle_on_the_battery(device_battery):
    cases, out = device_battery
    worst = collections.defaultdict(float)
    tight = 0
    for case, (n_d, c_d) in zip(cases, out):
        n_o, c_o = cr.oracle_outputs(case)
        bar = device_bar(cr.oracle_A(case))
        d = row_diff(case["points"], n_d, c_d, n_o, c_o, bar)
        worst[case["family"]] = max(worst[case["family"]], float(d.max()))
        tight += int((bar < 1e-12).sum())
        bad = np.nonzero(d > bar)[0]
        assert len(bad) == 0, (case["family"], case["kc"], case["k"], d[bad[:3]], bar[bad[:3]])
    print("\nworst |device - oracle| per family: " + ", ".join(f"{f} {w:.2g}" for f, w in sorted(worst.items())))
    assert tight > 0.5 * len(cr.rows(cases))  # the bar is at the rounding level on most rows


def test_gb_covariances_matches_exact_reference_and_invariants(device_battery):
    cases, out = device_battery
    posed = 0
    for case, (n_d, c_d) in zip(cases, out):
        assert not c_d[:, 3, :].any() and not c_d[:, :, 3].any() and not n_d[:, 3].any()
        tol = cr.invariant_tol(cr.oracle_A(case))
        C3 = c_d[:, :3, :3]
        assert (np.abs(np.linalg.eigvalsh(C3) - [1e-3, 1.0, 1.0]).max(axis=1) <= tol).all(), case["family"]
        assert (np.abs(C3 - C3.transpose(0, 2, 1)).max(axis=(1, 2)) <= tol).all(), case["family"]
        assert (np.abs(np.einsum("nij,nj->ni", C3, n_d[:, :3]) - 1e-3 * n_d[:, :3]).max(axis=1) <= tol).all(), case["family"]
        assert (np.abs(np.linalg.norm(n_d[:, :3], axis=1) - 1.0) <= 1e-12).all()
        P = case["points"]
        assert ((((P[:, 0] * n_d[:, 0] + P[:, 1] * n_d[:, 1]) + P[:, 2] * n_d[:, 2]) + P[:, 3] * n_d[:, 3]) <= 0.0).all(), case["family"]
        for i in range(len(P)):
            ex = cr.exact_row(case, i)
            bar = cr.posed_bar(ex)
            if bar >= cr.POSED_MAX:
                continue
            posed += 1
            en = np.abs(n_d[i, :3] - ex["n"]).max()
            if abs(ex["dot"]) <= bar:
                en = min(en, np.abs(n_d[i, :3] + ex["n"]).max())
            assert max(np.abs(C3[i] - ex["C"]).max(), en) <= bar, (case["family"], i)
    assert posed > 2000


def _frames(k):
    """(name, raw points (N, 4), times, params) of degenerate frames"""
    rng = np.random.default_rng(77)
    par = dict(distance_near_thresh=0.5, distance_far_thresh=50.0, downsample_resolution=0.0, k_correspondences=k)
    for m in sorted({1, 2, 3, k - 1, k} - {0}):
        inside = rng.normal(size=(m, 3)) * 0.3 + [5.0, -2.0, 1.0]
        far = rng.normal(size=(40, 3)) * 5.0 + [200.0, 0.0, 0.0]  # dropped by the range gate
        P = np.concatenate([np.concatenate([inside, far]), np.ones((m + 40, 1))], axis=1)
        yield f"{m}_points", P, rng.uniform(0, 0.1, len(P)), par
    base = rng.normal(size=(60, 3)) * [4.0, 4.0, 0.5] + [6.0, 0.0, 0.0]
    P = np.concatenate([np.repeat(base, 12, axis=0), np.ones((720, 1))], axis=1)  # every point 12 times
    yield "duplicates_x12", P, np.repeat(rng.uniform(0, 0.1, 60), 12), par
    x, y = np.meshgrid(np.arange(-20, 21) * 0.25, np.arange(-20, 21) * 0.25)
    P = np.stack([x.ravel() + 3.0, y.ravel(), np.full(x.size, -1.5), np.ones(x.size)], axis=1)  # a lattice floor
    yield "lattice_floor", P, np.linspace(0, 0.1, len(P)), dict(par, downsample_resolution=0.1)


@pytest.mark.parametrize("k", [5, 10, 20])
def test_gb_preprocess_degenerate_frames_match_oracle(ctx, k):
    for name, P, T, par in _frames(k):
        fr, normals, covs, cloud = preprocess.FramePreprocessorGPU(preprocess.CloudPreprocessorParams(**par), ctx).preprocess(1.0, T, P)
        res = par["downsample_resolution"]
        pts, tms, nb, n_ref, c_ref = _cpu_frame(P, T, res if res > 0 else None, par["distance_near_thresh"], par["distance_far_thresh"], k, mask=None if res > 0 else np.ones(len(P), bool))
        assert fr.size() == len(pts) > 0, name
        assert np.array_equal(fr.points, pts) and np.array_equal(fr.times, tms), name
        assert np.array_equal(fr.neighbors.reshape(-1, k), nb), name
        case = {"points": pts, "nb": nb, "kc": k, "k": k}
        d = row_diff(pts, normals, covs, n_ref, c_ref, device_bar(cr.oracle_A(case)))
        assert (d <= device_bar(cr.oracle_A(case))).all(), (name, d.max())
        gx, gc = cloud.download()
        xyz, cov6 = oracle.pack_cloud(fr.points, util.cov_colmajor16(covs))
        assert np.array_equal(gx, xyz) and np.array_equal(gc, cov6), name  # the planes are the fp32 cast of the fp64 products


def _knn_clouds():
    x, y, z = np.meshgrid(np.arange(6) * 0.5, np.arange(5) * 0.5, np.arange(3) * 0.5)
    lattice = np.stack([x.ravel(), y.ravel(), z.ravel(), np.ones(x.size)], axis=1)  # massive distance ties
    rng = np.random.default_rng(9)
    base = rng.normal(size=(40, 3))
    dup = np.concatenate([np.repeat(base, 5, axis=0), base[:7], np.tile(base[3], (40, 1))])
    dup = np.concatenate([dup, np.ones((len(dup), 1))], axis=1)
    return {"lattice": lattice, "duplicates": dup}


@pytest.mark.parametrize("name", ["lattice", "duplicates"])
def test_knn_is_exact_at_every_instantiated_k(ctx, name):
    cloud = _knn_clouds()[name]
    for k in KNN_KS:
        nb = preprocess.find_neighbors(cloud, k, ctx=ctx).reshape(len(cloud), k)
        ref, _ = oracle.knn_bruteforce(cloud, k)
        assert np.array_equal(nb, ref), (name, k)


@pytest.mark.parametrize("name", ["lattice", "duplicates"])
def test_uninstantiated_k_and_bad_indices_are_rejected_before_any_launch(ctx, name):
    P = _knn_clouds()[name]
    n = len(P)
    L = lib()
    before = ctx.kernel_launches
    out = np.zeros((n, 11), np.int32)
    assert L.gb_find_neighbors(ctx.h, n, ptr(P), 11, ptr(out)) == GB_ERR_INVALID_ARGUMENT
    g = preprocess.FramePreprocessorGPU(preprocess.CloudPreprocessorParams(downsample_resolution=0.0, k_correspondences=11), ctx)
    cp = g.c_params()
    res = Preprocessed()
    assert L.gb_preprocess(ctx.h, n, ptr(P), None, None, C.byref(cp), C.byref(res)) == GB_ERR_INVALID_ARGUMENT
    cp = preprocess.FramePreprocessorGPU(preprocess.CloudPreprocessorParams(downsample_resolution=0.0, enable_outlier_removal=True, outlier_removal_k=11), ctx).c_params()
    assert L.gb_preprocess(ctx.h, n, ptr(P), None, None, C.byref(cp), C.byref(res)) == GB_ERR_INVALID_ARGUMENT
    nb, _ = oracle.knn_bruteforce(P, 5)
    normals, covs = np.zeros((n, 4)), np.zeros((n, 16))
    for bad in (-1, n):
        b = nb.copy()
        b[n // 2, 3] = bad
        assert L.gb_covariances(ctx.h, n, ptr(P), ptr(b), 5, 5, ptr(normals), ptr(covs)) == GB_ERR_INVALID_ARGUMENT
    b = nb.copy()
    b[:, 4] = n + 7  # beyond k_neighbors: never read, accepted
    assert L.gb_covariances(ctx.h, n, ptr(P), ptr(b), 5, 4, ptr(normals), ptr(covs)) == 0
    assert ctx.kernel_launches == before + 1
