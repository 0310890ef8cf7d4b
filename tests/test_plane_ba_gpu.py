"""The interactive viewer's plane bundle adjustment on the H100 (gb_plane_patch, gb_plane_auto_radius, gb_plane_evm_*) against
the per-point restatement of tests/plane_ba_oracle.py: selection ids exactly, statistics within 1e-12 lambda_2, the auto-radius
path bit for bit on each of its exits, the factor's keys and counts exactly and its error, gradient and Hessian within 1e-10
lambda_2 / 1e-8 max |H|, batching and determinism bit for bit, a damped Newton loop that flattens a wall seen by several
submaps, refusals that launch nothing, and the launch counts the header states."""
import ctypes as C

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth
from tests import plane_ba_oracle as po

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    return gpu.Context(0)


# every radius a test here evaluates: its starting radii shrunk by 0.8 and grown by 1.1 up to 10 times, and max_radius
_RADII = np.log(np.unique([r0 * 0.8**i * 1.1**j for r0 in (0.3, 0.5, 0.9, 1.0, 1.5, 2.0, 2.5, 4.8, 5.0) for i in range(11) for j in range(11 - i)]))


def clear_shells(world, c):
    """the points of a scene farther than 1e-4 relative from every sphere about c a test evaluates: the stored fp32 local
    points then keep the device's and the oracle's selections out of their 1e-6 caveat"""
    d = np.log(np.linalg.norm(world - c, axis=1))
    i = np.clip(np.searchsorted(_RADII, d), 1, len(_RADII) - 1)
    return world[np.minimum(np.abs(d - _RADII[i]), np.abs(d - _RADII[i - 1])) > 1e-4]


def upload(ctx, local):
    return gpu.PointCloudGPU.clone(np.column_stack([local, np.ones(len(local))]), ctx=ctx)


def submaps(ctx, rng, world, K, spread=3.0, center=np.zeros(3), poses=None):
    """world points split among K submaps at random poses about `center`: (frames, host fp32 local points, poses)"""
    world = clear_shells(world, center)
    part = rng.integers(0, K, len(world))
    frames, host, X = [], [], []
    for k in range(K):
        if poses is not None:
            T = poses[k]
        else:
            T = np.eye(4)
            T[:3, :3] = synth.so3_exp(rng.normal(0, 0.6, 3))
            T[:3, 3] = center + rng.normal(0, spread, 3)
        loc = ((world[part == k] - T[:3, 3]) @ T[:3, :3]).astype(np.float32)
        frames.append(upload(ctx, loc.astype(np.float64)))
        host.append(loc)
        X.append(T)
    return frames, host, X


def wall(rng, n, center, half=3.0, thick=0.01, normal_rot=None):
    R = synth.so3_exp(rng.normal(0, 1, 3)) if normal_rot is None else normal_rot
    pts = np.column_stack([rng.uniform(-half, half, n), rng.uniform(-half, half, n), rng.normal(0, thick, n)])
    return pts @ R.T + center


def check_patch(ctx, frames, host, X, c, **kw):
    p = po.params(**kw)
    assert po.margin(host, X, c, p["radius"], p["max_frame_distance"]) > 1e-6
    got = gpu.plane_patch(frames, X, c, ids=True, ctx=ctx, **kw)
    ids, q, _ = po.select(host, X, c, p["radius"], p["max_frame_distance"])
    assert np.array_equal(got["ids"], ids)
    n, ev = po.stats(q)
    assert got["num_points"] == n
    if n:
        assert np.max(np.abs(got["eigenvalues"] - ev)) <= 1e-12 * ev[2]
    else:
        assert np.all(np.isnan(got["eigenvalues"]))
    return got


def test_selection_and_statistics(ctx):
    rng = np.random.default_rng(1)
    c = np.array([12.0, -4.0, 1.5])
    world = np.concatenate([wall(rng, 40000, c), c + rng.uniform(-4, 4, (20000, 3))])
    frames, host, X = submaps(ctx, rng, world, 6, center=c)
    for r in (0.3, 1.0, 2.5):
        got = check_patch(ctx, frames, host, X, c, radius=r)
        assert got["num_points"] > 100
    # nothing inside: n = 0, NaN eigenvalues
    check_patch(ctx, frames, host, X, c + 100.0, radius=0.5, max_frame_distance=np.inf)


def test_frame_filter_at_25_m(ctx):
    rng = np.random.default_rng(2)
    c = np.array([1.0, 2.0, 3.0])
    pts = (rng.uniform(-1, 1, (500, 3)) * 0.5).astype(np.float32)
    X = []
    for d in (24.9, 25.1):
        T = np.eye(4)
        T[:3, 3] = c + np.array([d, 0.0, 0.0])
        X.append(T)
    # the frames' points sit at the centre although their origins are 24.9 m and 25.1 m away
    local = [((c + pts.astype(np.float64)) - T[:3, 3]).astype(np.float32) for T in X]
    frames = [upload(ctx, l.astype(np.float64)) for l in local]
    got = check_patch(ctx, frames, local, X, c, radius=1.0)
    fr = got["ids"] >> np.uint64(32)
    assert set(fr.tolist()) == {0} and got["num_points"] == 500


def auto_case(ctx, frames, host, X, c, **kw):
    p = po.params(**kw)
    r, n, ev, trials = po.auto_radius(host, X, c, **kw)
    for t in [p["radius"]] + [t for t, _ in trials] + [max(p["radius"], p["max_radius"])]:
        assert po.margin(host, X, c, t, p["max_frame_distance"]) > 1e-6
    got = gpu.plane_auto_radius(frames, X, c, ctx=ctx, **kw)
    assert got["trials"] == trials
    assert got["radius"] == r and got["num_points"] == n
    if n:
        assert np.max(np.abs(got["eigenvalues"] - ev)) <= 1e-12 * ev[2]
    return r, n, trials


def test_auto_radius_every_exit(ctx):
    rng = np.random.default_rng(3)
    c = np.zeros(3)
    flat = wall(rng, 60000, c, half=6.0, thick=0.005)
    frames, host, X = submaps(ctx, rng, flat, 4)
    # planar everywhere: all 10 trials grow
    r, n, trials = auto_case(ctx, frames, host, X, c)
    assert len(trials) == 10 and r == trials[-1][0]
    # the next growth leaves [min_radius, max_radius]
    r, n, trials = auto_case(ctx, frames, host, X, c, radius=4.8)
    assert trials == [] and r == 4.8
    blob = rng.uniform(-1.5, 1.5, (200000, 3))
    frames_b, host_b, X_b = submaps(ctx, rng, blob, 3)
    # never planar: shrinks until the next radius is below min_radius
    r, n, trials = auto_case(ctx, frames_b, host_b, X_b, c, radius=0.5)
    assert 0 < len(trials) < 10 and r == trials[-1][0] and r * 0.8 < 0.1 and trials[-1][1] >= 10
    # fewer than 10 points at a shrunk radius: 12 points on a 0.85 m sphere
    u = rng.normal(0, 1, (12, 3))
    frames_s, host_s, X_s = submaps(ctx, rng, 0.85 * u / np.linalg.norm(u, axis=1)[:, None], 2)
    r, n, trials = auto_case(ctx, frames_s, host_s, X_s, c, radius=0.9)
    assert trials == [(0.9 * 0.8, 0)] and r == 0.9 and n == 12
    # grown past the start, then no longer planar: a 1.15 m disc of wall inside clutter
    disc = wall(rng, 60000, c, half=1.3, thick=0.003)
    disc = disc[np.linalg.norm(disc, axis=1) < 1.15]
    shell = rng.normal(0, 1, (100000, 3))
    shell = shell / np.linalg.norm(shell, axis=1)[:, None] * rng.uniform(1.15, 3.0, (100000, 1))
    frames_d, host_d, X_d = submaps(ctx, rng, np.concatenate([disc, shell]), 3)
    r, n, trials = auto_case(ctx, frames_d, host_d, X_d, c, radius=1.0)
    assert r == 1.1 and [t for t, _ in trials] == [1.1, 1.1 * 1.1] and trials[-1][1] >= 10


def factor_case(ctx, rng, K, c, thick, n_pts, radius, spread=3.0):
    world = wall(rng, n_pts, c, half=radius * 1.5, thick=thick)
    frames, host, X = submaps(ctx, rng, world, K, spread=spread, center=c)
    f = gpu.PlaneEVMFactorGPU(frames, X, c, ctx=ctx, radius=radius)
    keys, key_pts = po.factor_keys(host, X, c, radius=radius)
    assert f.keys.tolist() == keys
    assert f.key_points.tolist() == [len(a) for a in key_pts] and f.num_points == sum(len(a) for a in key_pts)
    return f, frames, host, X, keys, key_pts


@pytest.mark.parametrize("case", ["thin", "far", "many_keys"])
def test_factor_matches_the_oracle(ctx, case):
    rng = np.random.default_rng({"thin": 4, "far": 5, "many_keys": 6}[case])
    c = np.array([5000.0, -3000.0, 40.0]) if case == "far" else np.array([3.0, 1.0, 0.5])
    K = 40 if case == "many_keys" else 6
    f, frames, host, X, keys, key_pts = factor_case(ctx, rng, K, c, 1e-4 if case == "thin" else 0.02, 30000, 2.0)
    Xk = [X[k] for k in keys]
    worst = {}
    for step in range(3):
        Xe = po.perturbed(Xk, rng.normal(0, np.tile([0.01] * 3 + [0.05] * 3, len(keys))) * (step > 0))
        got = f.linearize(Xe)
        e, b, H, deg = po.linearize(key_pts, Xe, c)
        lam = np.linalg.eigvalsh(np.cov(np.concatenate(po.points_world(key_pts, Xe, c)).T, bias=True))
        assert got["status"] == 0 and not deg
        scale = np.max(np.abs(H))
        worst["error"] = max(worst.get("error", 0), abs(got["error"] - e) / lam[2])
        worst["H"] = max(worst.get("H", 0), np.max(np.abs(got["H"] - H)) / scale)
        worst["b"] = max(worst.get("b", 0), np.max(np.abs(got["b"] - b)) / scale)
        assert abs(f.error(Xe) - got["error"]) == 0.0
    print(f"plane factor {case}: K={len(keys)} N={f.num_points} worst |de|/lambda_2 {worst['error']:.2e}, |dH|/max|H| {worst['H']:.2e}, "
          f"|db|/max|H| {worst['b']:.2e}")
    assert worst["error"] <= 1e-10 and worst["H"] <= 1e-8 and worst["b"] <= 1e-8
    # the factor keeps no reference to its frames
    for fr in frames:
        fr.close()
    again = f.linearize(Xk)
    assert again["error"] == f.linearize(Xk)["error"]


def test_batch_is_bit_identical_to_single_calls(ctx):
    rng = np.random.default_rng(7)
    c = np.zeros(3)
    world = np.concatenate([wall(rng, 30000, c, half=4.0, thick=0.01), rng.uniform(-4, 4, (5000, 3))])
    frames, host, X = submaps(ctx, rng, world, 8)
    facs, poses = [], []
    for i in range(64):
        ci = rng.uniform(-2, 2, 3) * np.array([1, 1, 0])
        f = gpu.PlaneEVMFactorGPU(frames, X, ci, ctx=ctx, radius=float(rng.uniform(0.5, 1.5)))
        facs.append(f)
        poses.append(po.perturbed([X[k] for k in f.keys], rng.normal(0, 0.01, 6 * len(f.keys))))
    before = ctx.kernel_launches
    batch = gpu.linearize_plane_evm(facs, poses, ctx=ctx)
    assert ctx.kernel_launches - before == 1
    batch2 = gpu.linearize_plane_evm(facs, poses, ctx=ctx)
    for f, P, got, got2 in zip(facs, poses, batch, batch2):
        one = f.linearize(P)
        for k in ("H", "b"):
            assert np.array_equal(got[k], one[k]) and np.array_equal(got[k], got2[k])
        assert got["error"] == one["error"] == got2["error"] and got["status"] == one["status"]


def test_newton_flattens_a_wall(ctx):
    """several submaps see one wall; 0.5 deg and 5 cm pose errors; damped Newton on the device records, first key fixed"""
    rng = np.random.default_rng(8)
    c = np.zeros(3)
    world = wall(rng, 40000, c, half=3.0, thick=0.005, normal_rot=synth.so3_exp([0.3, 0.2, 0.0]))
    K = 5
    true = []
    for k in range(K):
        T = np.eye(4)
        T[:3, :3] = synth.so3_exp(rng.normal(0, 0.5, 3))
        T[:3, 3] = rng.normal(0, 3, 3)
        true.append(T)
    frames, host, _ = submaps(ctx, rng, world, K, poses=true)
    est = [true[0]] + [T @ synth.se3_exp(np.concatenate([rng.normal(0, 1, 3) / np.sqrt(3) * np.radians(0.5), rng.normal(0, 1, 3) / np.sqrt(3) * 0.05]))
                       for T in true[1:]]
    f = gpu.PlaneEVMFactorGPU(frames, est, c, ctx=ctx, radius=2.0)
    assert len(f.keys) == K
    e_true = f.error(true)
    e0 = f.error(est)
    lam = 1e-3
    for it in range(20):
        r = f.linearize(est)
        H, b = r["H"][6:, 6:], r["b"][6:]
        step = np.linalg.solve(H + lam * np.trace(H) / len(H) * np.eye(len(H)), -b)
        cand = [est[0]] + [T @ synth.se3_exp(step[6 * k:6 * k + 6]) for k, T in enumerate(est[1:])]
        if f.error(cand) < r["error"]:
            est, lam = cand, lam * 0.3
        else:
            lam *= 10
    e1 = f.error(est)
    print(f"plane Newton: error {e0:.3e} -> {e1:.3e} (true poses {e_true:.3e})")
    assert e1 <= 1.5 * e_true < e0


def test_refusals_launch_nothing(ctx):
    rng = np.random.default_rng(9)
    c = np.zeros(3)
    world = wall(rng, 5000, c)
    frames, host, X = submaps(ctx, rng, world, 3)
    L = capi.lib()
    arr = (C.c_void_p * 3)(*[fr.h for fr in frames])
    T = capi.pose16(np.stack(X))
    r = capi.PlanePatchResult()
    h = C.c_void_p()
    bad = [dict(radius=0.0), dict(radius=np.inf), dict(min_radius=0.0), dict(min_radius=2.0, max_radius=1.0), dict(max_radius=np.nan),
           dict(plane_eps=-1.0), dict(plane_eps=np.inf), dict(max_frame_distance=-1.0), dict(max_frame_distance=np.nan)]
    before = ctx.kernel_launches
    for kw in bad:
        p = gpu.plane_patch_params(c, **kw)
        assert L.gb_plane_patch(ctx.h, 3, arr, capi.ptr(T), C.byref(p), C.byref(r), None) == 1, kw
        assert L.gb_plane_auto_radius(ctx.h, 3, arr, capi.ptr(T), C.byref(p), C.byref(r)) == 1, kw
        assert L.gb_plane_evm_factor_create(ctx.h, 3, arr, capi.ptr(T), C.byref(p), C.byref(h)) == 1 and not h.value, kw
    p = gpu.plane_patch_params([np.nan, 0, 0])
    assert L.gb_plane_patch(ctx.h, 3, arr, capi.ptr(T), C.byref(p), C.byref(r), None) == 1
    Tn = T.copy()
    Tn[1, 5] = np.inf
    p = gpu.plane_patch_params(c)
    assert L.gb_plane_patch(ctx.h, 3, arr, capi.ptr(Tn), C.byref(p), C.byref(r), None) == 1
    assert ctx.kernel_launches == before
    # fewer than 3 points: refused after the selection, nothing created
    p = gpu.plane_patch_params(c + 50.0, max_frame_distance=np.inf)
    assert L.gb_plane_evm_factor_create(ctx.h, 3, arr, capi.ptr(T), C.byref(p), C.byref(h)) == 1 and not h.value
    # every existing factor entry point refuses a plane factor, and the plane calls refuse the other kinds
    pf = gpu.PlaneEVMFactorGPU(frames, X, c, ctx=ctx)
    vmap = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(frames[0])
    vf = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, vmap, frames[1], ctx=ctx)
    I16 = capi.pose16(np.eye(4))
    out = np.zeros(1, gpu.LIN_DTYPE)
    e = C.c_double()
    one = (C.c_void_p * 1)(pf.h)
    before = ctx.kernel_launches
    assert L.gb_vgicp_linearize(pf.h, capi.ptr(I16), capi.ptr(out)) == 1
    assert L.gb_vgicp_error(pf.h, capi.ptr(I16), capi.ptr(I16), C.byref(e)) == 1
    assert L.gb_factor_set_linearize(ctx.h, 1, C.cast(one, C.c_void_p), capi.ptr(I16), capi.ptr(out)) == 1
    assert L.gb_factor_set_error(ctx.h, 1, C.cast(one, C.c_void_p), capi.ptr(I16), capi.ptr(I16), capi.ptr(np.zeros(1))) == 1
    sw = C.c_void_p()
    assert L.gb_sweep_create(ctx.h, 1, C.cast(one, C.c_void_p), None, C.byref(sw)) == 1 and not sw.value
    ap = gpu.align_params()
    res = (C.c_byte * 4096)()
    assert L.gb_vgicp_align(ctx.h, 1, capi.ptr(np.array([0, 1], np.uint64)), C.cast(one, C.c_void_p), capi.ptr(I16), C.byref(ap), C.cast(res, C.c_void_p)) == 1
    assert L.gb_ct_gicp_linearize(pf.h, capi.ptr(I16), capi.ptr(I16), capi.ptr(out)) == 1
    assert L.gb_ct_gicp_error(pf.h, capi.ptr(I16), capi.ptr(I16), capi.ptr(I16), capi.ptr(I16), C.byref(e)) == 1
    vone = (C.c_void_p * 1)(vf.h)
    P16 = capi.pose16(np.stack([np.eye(4)] * 3))
    assert L.gb_plane_evm_error(ctx.h, 1, C.cast(vone, C.c_void_p), capi.ptr(P16), capi.ptr(np.zeros(1))) == 1
    assert L.gb_plane_evm_linearize(ctx.h, 1, C.cast(vone, C.c_void_p), capi.ptr(P16), capi.ptr(np.zeros(36 * 9)), capi.ptr(np.zeros(18)),
                                    capi.ptr(np.zeros(1)), None) == 1
    assert L.gb_plane_evm_factor_info(vf.h, None, None, None, None) == 1
    Pn = capi.pose16(np.stack([np.eye(4)] * len(pf.keys)))
    Pn[0, 0] = np.nan
    assert L.gb_plane_evm_error(ctx.h, 1, C.cast(one, C.c_void_p), capi.ptr(Pn), capi.ptr(np.zeros(1))) == 1
    assert ctx.kernel_launches == before


def test_launch_counts(ctx):
    rng = np.random.default_rng(10)
    c = np.zeros(3)
    frames, host, X = submaps(ctx, rng, wall(rng, 20000, c, half=5.0), 4)
    n0 = ctx.kernel_launches
    gpu.plane_patch(frames, X, c, ids=True, ctx=ctx)
    assert ctx.kernel_launches - n0 == 5
    n0 = ctx.kernel_launches
    got = gpu.plane_auto_radius(frames, X, c, ctx=ctx)
    assert ctx.kernel_launches - n0 == 4 + 1 + len(got["trials"])
    n0 = ctx.kernel_launches
    f = gpu.PlaneEVMFactorGPU(frames, X, c, ctx=ctx)
    assert ctx.kernel_launches - n0 == 5
    n0 = ctx.kernel_launches
    f.linearize([X[k] for k in f.keys])
    f.error([X[k] for k in f.keys])
    assert ctx.kernel_launches - n0 == 2
    # no participating frame: no launch
    n0 = ctx.kernel_launches
    got = gpu.plane_patch(frames, X, c + 1000.0, ctx=ctx)
    assert got["num_points"] == 0 and ctx.kernel_launches == n0


def test_large_map(ctx):
    rng = np.random.default_rng(11)
    K, n = 32, 250000
    c = np.array([40.0, 20.0, 1.0])
    frames, host, X = [], [], []
    for k in range(K):
        T = np.eye(4)
        T[:3, :3] = synth.so3_exp([0, 0, rng.uniform(-np.pi, np.pi)])
        T[:3, 3] = c + np.array([rng.uniform(-20, 20), rng.uniform(-20, 20), 0.0])
        # a floor and a wall through the picked point, plus clutter, in the submap's frame
        wpts = np.concatenate([np.column_stack([c[0] + rng.uniform(-25, 25, n // 2), c[1] + rng.uniform(-25, 25, n // 2), c[2] - 1.0 + rng.normal(0, 0.01, n // 2)]),
                               np.column_stack([c[0] + rng.normal(0, 0.01, n // 4), c[1] + rng.uniform(-25, 25, n // 4), c[2] + rng.uniform(-1, 3, n // 4)]),
                               c + rng.uniform(-25, 25, (n - n // 2 - n // 4, 3))])
        wpts = clear_shells(wpts, c)
        loc = ((wpts - T[:3, 3]) @ T[:3, :3]).astype(np.float32)
        host.append(loc)
        frames.append(upload(ctx, loc.astype(np.float64)))  # fewer than 250 k after clear_shells
        X.append(T)
    p = po.params(radius=1.5)
    got = check_patch(ctx, frames, host, X, c, radius=1.5)
    assert got["num_points"] > 10000
    auto_case(ctx, frames, host, X, c, radius=1.5)
    f = gpu.PlaneEVMFactorGPU(frames, X, c, ctx=ctx, radius=1.5)
    keys, key_pts = po.factor_keys(host, X, c, radius=p["radius"])
    assert f.keys.tolist() == keys and f.key_points.tolist() == [len(a) for a in key_pts]
    Xk = [X[k] for k in keys]
    r = f.linearize(Xk)
    e, b, H, _ = po.linearize(key_pts, Xk, c)
    lam = np.linalg.eigvalsh(np.cov(np.concatenate(po.points_world(key_pts, Xk, c)).T, bias=True))
    assert abs(r["error"] - e) <= 1e-10 * lam[2]
    assert np.max(np.abs(r["H"] - H)) <= 1e-8 * np.max(np.abs(H)) and np.max(np.abs(r["b"] - b)) <= 1e-8 * np.max(np.abs(H))
