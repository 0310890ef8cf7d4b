"""Continuous-time GICP on the H100 (gb_cloud_add_times, gb_ct_gicp_factor_create / _linearize / _error, gb_ct_gicp_align,
gb_ct_deskew): the time table exactly, the factor and the solve against the numpy restatement (tests/ct_oracle.py) on
motion-distorted frames, the one-entry factor against the GICP factor, the deskewed frame, refusals before any launch, and
GLIM's LiDAR-only odometry loop as shipped end to end against ground truth."""
import ctypes as C

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth
from oracle import oracle
from tests import ct_oracle as co
from tests import ivox_oracle as io
from tests import voxelmap_oracle as vo
from tests import util
from tests.util import REL_TOL, cov_colmajor16, rel_err

pytestmark = pytest.mark.gpu

MAX_CORR = 2.0


def pose_error(T, T_ref):
    d = synth.inv_pose(T_ref) @ T
    return float(np.linalg.norm(d[:3, 3])), float(np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1)))


def distorted(k, n_rays, key=0):
    """distorted frame k with its PLANE covariances, neighbours (k = 10) and times"""
    pts, tms = co.distorted_frame(synth.make_hall_scene(), k, n_rays, synth.rng_for(4500, key, k))
    nb = synth.knn(pts, 10)
    nrm, cov = synth.plane_covariances(pts, nb)
    return pts, cov, nrm, nb, tms


@pytest.fixture(scope="module")
def scene(ctx):
    """an iVox (1.0 m, mode 7) of three undistorted arc frames on the device and restated, and a motion-distorted source
    placed in that map: its points, covariances, times, time table and ground-truth X / Y"""
    frames = vo.arc_frames(4, 32 * 200)
    m = gpu.IVoxGPU(1.0, 0.1, 10, 7, 100, 10, ctx=ctx)
    R = io.IVox(1.0, 0.1, 10, 7, 100, 10)
    for k in (0, 1, 2):
        cloud = gpu.PointCloudGPU.clone(frames[k][0], frames[k][1], ctx=ctx)
        xyz, cov6 = oracle.pack_cloud(frames[k][0], cov_colmajor16(frames[k][1]))
        m.insert(cloud, frames[k][2])
        R.insert(xyz, cov6, frames[k][2])
    pts, cov, _, nb, tms = distorted(21, 32 * 200)  # frame 21 of the distorted run: t in [2.1, 2.2) s
    starts, tau = co.time_table(tms)
    # the distorted run drives the arc of arc_frames: at 2.1 s it is among the map's frames
    X = co.gt_pose(2.1 + tms[0])
    Y = co.gt_pose(2.1 + tms[starts[-2]])
    src = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx).add_times(tms)
    xyz, cov6 = oracle.pack_cloud(pts, cov_colmajor16(cov))
    return m, R, src, xyz, cov6, pts, nb, tms, starts, tau, X, Y


def test_time_table_is_exact(ctx, scene):
    """gb_cloud_add_times against the restatement, exactly; setting times again replaces the table"""
    _, _, src, *_, tms, starts, tau, _, _ = scene
    s, t, t0, t1 = src.time_table()
    assert np.array_equal(s, starts) and np.array_equal(t, tau)
    assert (t0, t1) == (tms[0], tms[starts[-2]])
    assert 50 < len(tau) <= 101
    other = np.sort(synth.rng_for(4501).uniform(0.0, 0.05, len(tms)))
    src.add_times(other)
    s2, t2, _, _ = src.time_table()
    r2, rt2 = co.time_table(other)
    assert np.array_equal(s2, r2) and np.array_equal(t2, rt2)
    src.add_times(tms)
    assert np.array_equal(src.time_table()[0], starts)


def ct_record_check(got, ref, what):
    assert got["num_inliers"] == ref["num_inliers"] > 0, what
    H = np.block([[got["H_tt"], got["H_ts"]], [got["H_ts"].T, got["H_ss"]]])
    assert rel_err(H, ref["H"]) < REL_TOL, (what, rel_err(H, ref["H"]))
    b = np.concatenate([got["b_t"], got["b_s"]])
    scale = max(np.linalg.norm(ref["b"]), 0.1 * np.sqrt(np.trace(ref["H"]) * ref["error"]))
    assert np.linalg.norm(b - ref["b"]) < REL_TOL * scale, what
    assert abs(got["error"] - ref["error"]) < REL_TOL * ref["error"], what


def ct_scale(R, xyz, cov6, starts, tau, X, Y, corr):
    """the entry-wise scale of a CT record, through the kernel's chain: each entry's GICP sums at its fp32-cast pose T_b, its
    H_ss / b_s through |Ad(T_b)| as factor_epilogue forms them, then the 12 x 12 system through |[D0 D1]|"""
    A, B = {"H": np.zeros((12, 12)), "b": np.zeros(12), "error": 0.0}, {"H": np.zeros((12, 12)), "b": np.zeros(12), "error": 0.0}
    for idx, t, c in zip(co.entry_indices(starts), tau, corr):
        Tb = co.entry_pose(X, Y, t)
        P = np.abs(util.adjoint_f32(Tb))
        J = np.abs(np.concatenate(co.entry_blocks(X, Y, t), axis=1))
        for part, s in zip((A, B), util.hit_scale(util.factor_hits(R.xyz, R.cov6, xyz[idx], cov6[idx], Tb, c))):
            part["H"] += J.T @ P.T @ s["H_tt"] @ P @ J
            part["b"] += J.T @ P.T @ s["b_t"]
            part["error"] += s["error"]

    def blocks(p):
        return {"H_tt": p["H"][:6, :6], "H_ss": p["H"][6:, 6:], "H_ts": p["H"][:6, 6:], "b_t": p["b"][:6], "b_s": p["b"][6:], "error": p["error"]}

    return util.EntryScale(blocks(A), blocks(B))


def test_factor_matches_restatement_on_a_distorted_frame(ctx, scene):
    """linearize at several (X, Y) (the ground truth, perturbed poses, no motion): inlier counts exact, H and error within
    1e-4 relative, b by the project's criterion; error() with lin != eval likewise"""
    m, R, src, xyz, cov6, _, _, _, starts, tau, X, Y = scene
    rng = synth.rng_for(4502)
    cases = [(X, Y), (X, X)] + [(synth.perturb(X, rng, 0.01, 0.1), synth.perturb(Y, rng, 0.01, 0.1)) for _ in range(2)]
    f = gpu.IntegratedCT_GICPFactorGPU(0, 1, m, src, MAX_CORR, ctx=ctx)
    for i, (Xc, Yc) in enumerate(cases):
        got = f.linearize({0: Xc, 1: Yc})
        ref, corr = co.linearize(R, xyz, cov6, starts, tau, Xc, Yc, MAX_CORR)
        ct_record_check(got, ref, i)
        util.check_entrywise(got, ref, ct_scale(R, xyz, cov6, starts, tau, Xc, Yc, corr), what=("CT", i))
        assert np.allclose(got["H_tt"], got["H_tt"].T, rtol=0, atol=1e-9 * np.abs(got["H_tt"]).max())
    Xe, Ye = synth.perturb(X, rng, 0.005, 0.05), synth.perturb(Y, rng, 0.005, 0.05)
    f.linearize({0: X, 1: Y})
    e = f.error({0: Xe, 1: Ye})
    e_ref = co.error(R, xyz, cov6, starts, tau, X, Y, Xe, Ye, MAX_CORR)
    assert abs(e - e_ref) < REL_TOL * e_ref


def test_one_entry_equals_the_gicp_factor(ctx, scene):
    """all times equal: H_XX, b_X, error and inliers are gb_vgicp_linearize's of the GICP factor at X within 1e-6; the Y
    blocks are zero"""
    m, _, _, _, _, pts, _, _, _, _, X, Y = scene
    cov = synth.plane_covariances(pts, synth.knn(pts, 10))[1]
    src = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx).add_times(np.full(len(pts), 0.03))
    ct = gpu.IntegratedCT_GICPFactorGPU(0, 1, m, src, MAX_CORR, ctx=ctx).linearize({0: X, 1: Y})
    g = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, m, src, MAX_CORR, ctx=ctx).linearize({0: X})
    assert ct["num_inliers"] == g["num_inliers"] > 0
    assert rel_err(ct["H_tt"], g["H_ss"]) < 1e-6
    assert np.linalg.norm(ct["b_t"] - g["b_s"]) < 1e-6 * max(np.linalg.norm(g["b_s"]), 0.1 * np.sqrt(np.trace(g["H_ss"]) * g["error"]))
    assert abs(ct["error"] - g["error"]) < 1e-6 * g["error"]
    assert not ct["H_ss"].any() and not ct["H_ts"].any() and not ct["b_s"].any()


def test_align_matches_restatement_batch_equals_singles_and_launch_count(ctx, scene):
    """gb_ct_gicp_align from perturbed starts against the restatement's LM (2e-3 m / rad); a batch of 4 equals the problems
    run one at a time (bit-identical where the iteration path matches); launches = 3 per round + 1 per linearization"""
    m, R, src, xyz, cov6, _, _, _, starts, tau, X, Y = scene
    rng = synth.rng_for(4503)
    f = gpu.IntegratedCT_GICPFactorGPU(0, 1, m, src, MAX_CORR, ctx=ctx)
    inits = [(synth.perturb(X, rng, 0.005, 0.1), synth.perturb(Y, rng, 0.005, 0.1)) for _ in range(4)]
    Xp = [synth.perturb(X, rng, 0.002, 0.02) for _ in range(4)]
    batch = gpu.align_ct_gicp([f] * 4, [a for a, _ in inits], [b for _, b in inits], Xp)
    for p, ((X0, Y0), r) in enumerate(zip(inits, batch)):
        l0 = ctx.kernel_launches
        single = gpu.align_ct_gicp([f], [X0], [Y0], [Xp[p]])[0]
        launches = ctx.kernel_launches - l0
        assert launches == 3 * single["trials"] + single["iterations"], (launches, single)
        if (single["iterations"], single["trials"]) == (r["iterations"], r["trials"]):
            assert np.array_equal(single["X"], r["X"]) and np.array_equal(single["Y"], r["Y"]) and single["error"] == r["error"]
        ref = co.align(R, xyz, cov6, starts, tau, X0, Y0, Xp[p], MAX_CORR)
        for key in ("X", "Y"):
            et, er = pose_error(r[key], ref[key])
            assert et < 2e-3 and er < 2e-3, (p, key, et, er, r["status_name"], ref["status"])
        # near the minimum the fp32 sums decide e' < e, so a problem may also end by rejections (LAMBDA_EXCEEDED)
        assert r["status"] != capi.ALIGN_DEGENERATE, r
        print(f"problem {p}: {r['status_name']} after {r['iterations']} linearizations / {r['trials']} trials "
              f"(restatement {ref['iterations']} / {ref['trials']}), X off ground truth by {pose_error(r['X'], X)[0]:.4f} m")


def test_deskew_matches_restatement(ctx, scene):
    """points within 1e-9 m of Exp(tau_b xi) p; covariances and normals within 1e-9 of gb_covariances on those points where
    the neighbourhood's relative eigengap exceeds 1e-3; the output cloud is the frame gb_cloud_upload would make of them"""
    _, _, src, xyz, _, _, nb, _, starts, tau, X, Y = scene
    pts, cov, nrm, cloud = gpu.deskew_ct(src, X, Y, nb, 10)
    xi = co.motion(X, Y)
    ref = np.zeros((len(xyz), 4))
    for idx, t in zip(co.entry_indices(starts), tau):
        ref[idx] = (co.se3_exp(t * xi) @ np.concatenate([xyz[idx].astype(np.float64), np.ones((len(idx), 1))], axis=1).T).T
    assert np.abs(pts - ref).max() < 1e-9
    n = len(ref)
    nrm_ref, cov_ref = np.empty((n, 4)), np.empty((n, 16))
    capi.check(capi.lib().gb_covariances(ctx.h, n, capi.ptr(np.ascontiguousarray(ref)), capi.ptr(nb), 10, 10, capi.ptr(nrm_ref), capi.ptr(cov_ref)))
    P = ref[nb][:, :, :3]
    w = np.linalg.eigvalsh(np.einsum("nki,nkj->nij", P - P.mean(1, keepdims=True), P - P.mean(1, keepdims=True)) / 10)
    good = (w[:, 1] - w[:, 0]) > 1e-3 * np.maximum(w[:, 2], 1e-300)
    assert good.mean() > 0.9
    cov16 = cov_colmajor16(cov)
    assert np.abs(cov16[good] - cov_ref[good]).max() < 1e-9
    assert np.abs(nrm[good] - nrm_ref[good]).max() < 1e-9
    xyz_c, cov6_c = cloud.download()
    up = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx).download()
    assert np.array_equal(xyz_c, up[0]) and np.array_equal(cov6_c, up[1])
    assert cloud.time_table()[1].size == 0


def test_invalid_inputs_are_refused_before_any_launch(ctx, scene):
    L = capi.lib()
    m, _, src, _, _, pts, nb, tms, _, _, X, Y = scene
    plain = gpu.PointCloudGPU.clone(pts, synth.plane_covariances(pts, nb)[1], ctx=ctx)
    vmap = gpu.IncrementalVoxelMapGPU(1.0, ctx=ctx).insert(plain, X)
    ct = gpu.IntegratedCT_GICPFactorGPU(0, 1, m, src, MAX_CORR, ctx=ctx)
    g = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, m, plain, MAX_CORR, ctx=ctx)
    good, bad = capi.pose16(X), capi.pose16(X).copy()
    bad[13] = np.nan
    h = C.c_void_p()
    out = np.zeros(1, gpu.LIN_DTYPE)
    e = C.c_double()
    launches = ctx.kernel_launches
    # times: unsorted, NaN, wrong length
    for t in (tms[::-1].copy(), np.where(np.arange(len(tms)) == 5, np.nan, tms), tms[:-1].copy()):
        assert L.gb_cloud_add_times(ctx.h, plain.h, len(t), capi.ptr(np.ascontiguousarray(t))) == 1
    # a source without times, a non-iVox target, a bad distance
    assert L.gb_ct_gicp_factor_create(ctx.h, m.h, plain.h, MAX_CORR, C.byref(h)) == 1 and not h.value
    assert L.gb_ct_gicp_factor_create(ctx.h, vmap.h, src.h, MAX_CORR, C.byref(h)) == 1 and not h.value
    assert L.gb_ct_gicp_factor_create(ctx.h, m.h, src.h, -1.0, C.byref(h)) == 1 and not h.value
    # a CT factor in every existing consumer
    one = (C.c_void_p * 1)(ct._handle())
    assert L.gb_vgicp_linearize(ct._handle(), capi.ptr(good), capi.ptr(out)) == 1
    assert L.gb_vgicp_error(ct._handle(), capi.ptr(good), capi.ptr(good), C.byref(e)) == 1
    assert L.gb_factor_set_linearize(ctx.h, 1, C.cast(one, C.c_void_p), capi.ptr(good), capi.ptr(out)) == 1
    assert L.gb_factor_set_error(ctx.h, 1, C.cast(one, C.c_void_p), capi.ptr(good), capi.ptr(good), capi.ptr(np.zeros(1))) == 1
    assert L.gb_sweep_create(ctx.h, 1, C.cast(one, C.c_void_p), None, C.byref(h)) == 1 and not h.value
    off = np.array([0, 1], np.uint64)
    res = (capi.AlignResult * 1)()
    assert L.gb_vgicp_align(ctx.h, 1, capi.ptr(off), C.cast(one, C.c_void_p), capi.ptr(good), C.byref(gpu.align_params()), C.cast(res, C.c_void_p)) == 1
    # other factors in the CT entry points
    gone = (C.c_void_p * 1)(g._handle())
    cres = (capi.CtResult * 1)()
    prm = gpu.ct_params()
    assert L.gb_ct_gicp_linearize(g._handle(), capi.ptr(good), capi.ptr(good), capi.ptr(out)) == 1
    assert L.gb_ct_gicp_error(g._handle(), capi.ptr(good), capi.ptr(good), capi.ptr(good), capi.ptr(good), C.byref(e)) == 1
    assert L.gb_ct_gicp_align(ctx.h, 1, C.cast(gone, C.c_void_p), capi.ptr(good), capi.ptr(good), capi.ptr(good), C.byref(prm), C.cast(cres, C.c_void_p)) == 1
    # non-finite poses
    assert L.gb_ct_gicp_linearize(ct._handle(), capi.ptr(bad), capi.ptr(good), capi.ptr(out)) == 1
    assert L.gb_ct_gicp_error(ct._handle(), capi.ptr(good), capi.ptr(good), capi.ptr(good), capi.ptr(bad), C.byref(e)) == 1
    for a, b, c in ((bad, good, good), (good, bad, good), (good, good, bad)):
        assert L.gb_ct_gicp_align(ctx.h, 1, C.cast(one, C.c_void_p), capi.ptr(a), capi.ptr(b), capi.ptr(c), C.byref(prm), C.cast(cres, C.c_void_p)) == 1
    assert L.gb_ct_deskew(ctx.h, src.h, capi.ptr(bad), capi.ptr(good), capi.ptr(nb), 10, 10, None, None, None, C.byref(h)) == 1 and not h.value
    # out-of-range parameters and neighbour indices
    for kw in ({"max_iterations": 0}, {"lambda_factor": 1.0}, {"location_consistency_inf_scale": -1.0}, {"constant_velocity_inf_scale": np.inf}):
        assert L.gb_ct_gicp_align(ctx.h, 1, C.cast(one, C.c_void_p), capi.ptr(good), capi.ptr(good), capi.ptr(good), C.byref(gpu.ct_params(**kw)), C.cast(cres, C.c_void_p)) == 1
    nb_bad = nb.copy()
    nb_bad[7, 3] = len(pts)
    for arr, kc, k in ((nb_bad, 10, 10), (nb, 10, 11), (nb, 10, 0)):
        assert L.gb_ct_deskew(ctx.h, src.h, capi.ptr(good), capi.ptr(good), capi.ptr(arr), kc, k, None, None, None, C.byref(h)) == 1 and not h.value
    assert L.gb_ct_deskew(ctx.h, plain.h, capi.ptr(good), capi.ptr(good), capi.ptr(nb), 10, 10, None, None, None, C.byref(h)) == 1 and not h.value
    assert ctx.kernel_launches == launches


def test_shipped_ct_odometry_end_to_end(ctx):
    """GLIM's LiDAR-only odometry as shipped (odometry_estimation_ct.cpp:85-235) on 40 motion-distorted hdl32 frames (10 m/s,
    0.6 rad/s): twist prediction, gb_ct_gicp_align with the prior at the last Y and the default gb_ct_params, gb_ct_deskew,
    and the deskewed frame inserted at X into a 1.0 m iVox (min_dist 0.1, LRU 200, mode 1, max_correspondence_distance 2.0).
    X is scored against ground truth at t_0, Y at t_{B-1}.  The rigid GICP loop of test_shipped_gicp_odometry_end_to_end on
    the same frames (scored at mid-scan) is printed beside it.
    Bar: about twice the first H100 run's worst frame (X 0.074 m / 0.80 deg, Y 0.091 m / 0.73 deg; mean X error 0.032 m).
    That run's rigid loop: worst 0.69 m / 1.3 deg, mean 0.30 m at mid-scan."""
    n_frames, n_rays = 40, 32 * 1000
    world0 = synth.inv_pose(co.gt_pose(0.0))
    ivox = gpu.IVoxGPU(1.0, 0.1, 10, 1, 200, 10, ctx=ctx)
    rigid = gpu.IVoxGPU(1.0, 0.1, 10, 1, 100, 10, ctx=ctx)
    errs, rigid_errs, rigid_est = [], [], []
    X_last = Y_last = t_prev = None
    for k in range(n_frames):
        pts, cov, _, nb, tms = distorted(k, n_rays, key=1)
        cloud = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx).add_times(tms)
        starts, _, t0, t1 = cloud.time_table()
        t0, t1 = 0.1 * k + t0, 0.1 * k + t1
        X_gt, Y_gt = world0 @ co.gt_pose(t0), world0 @ co.gt_pose(t1)
        if k == 0:
            X, Y = X_gt, Y_gt  # the initial state
        else:
            v = co.motion(X_last, Y_last) / (t_prev[1] - t_prev[0])  # the last frame's twist (odometry_estimation_ct.cpp:126-155)
            X0 = Y_last @ co.se3_exp(v * (t0 - t_prev[1]))
            Y0 = X0 @ co.se3_exp(v * (t1 - t0))
            f = gpu.IntegratedCT_GICPFactorGPU(0, 1, ivox, cloud, 2.0, ctx=ctx)
            r = gpu.align_ct_gicp([f], [X0], [Y0], [Y_last])[0]
            X, Y = r["X"], r["Y"]
            errs.append(pose_error(X, X_gt) + pose_error(Y, Y_gt))
        _, _, _, desk = gpu.deskew_ct(cloud, X, Y, nb, 10, host_outputs=False)
        ivox.insert(desk, X, 1.0, seed=k)
        X_last, Y_last, t_prev = X, Y, (t0, t1)
        # the rigid loop on the raw frame, predicted with the last increment (the ground truth's for frame 1)
        T_mid = world0 @ co.gt_pose(0.1 * k + 0.05)
        if k == 0:
            rigid_est.append(T_mid)
        else:
            prev = rigid_est[-2] if k > 1 else world0 @ co.gt_pose(-0.05)
            fac = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, rigid, cloud, 2.0, ctx=ctx)
            init = rigid_est[-1] @ synth.inv_pose(prev) @ rigid_est[-1]
            rigid_est.append(gpu.align_vgicp([[fac]], [init], params={"max_iterations": 8})[0]["T_target_source"])
            rigid_errs.append(pose_error(rigid_est[-1], T_mid))
        rigid.insert(cloud, rigid_est[-1], sampling_rate=1.0 if k < 5 else 0.1, seed=k)
    e = np.array(errs)
    re_ = np.array(rigid_errs)
    print(f"CT odometry, {n_frames} frames: X max {e[:, 0].max():.4f} m / {np.degrees(e[:, 1].max()):.3f} deg, mean {e[:, 0].mean():.4f} m; "
          f"Y max {e[:, 2].max():.4f} m / {np.degrees(e[:, 3].max()):.3f} deg, mean {e[:, 2].mean():.4f} m")
    print(f"rigid GICP odometry on the same frames (mid-scan): max {re_[:, 0].max():.4f} m / {np.degrees(re_[:, 1].max()):.3f} deg, mean {re_[:, 0].mean():.4f} m")
    assert e[:, 0].max() < 0.15 and e[:, 2].max() < 0.18, (e[:, 0].max(), e[:, 2].max())
    assert e[:, 1].max() < np.radians(1.6) and e[:, 3].max() < np.radians(1.5), (e[:, 1].max(), e[:, 3].max())
