"""Every work schedule of the device sweeps against the fp64 oracle.  The host rules (gb_sweep_create, build_items,
sweep_learn_inliers, graph_eligible, the ctr_base advance) choose a kernel, an item table, a grid and accumulator copies for
each sweep; tests/sweep_schedule.py restates them, and each test here asserts through gb_sweep_stats that the sweep it built
runs the regime it asks for, then checks that regime three ways:

  * linearize against the oracle: inlier counts exact, blocks within the 1e-4 bars of tests/util.check_linearized;
  * the error at T_eval != T_lin against the oracle's error with the correspondences of T_lin;
  * linearize, error, linearize, linearize on one cached sweep: inlier counts exact across the repeats and blocks within 1e-12
    (only the order of the fp64 accumulator atomics may differ).

Factors are made distinguishable: factor f takes source prefix f % len(cycle), pose f % 8 and voxel level f % 3, so an item
credited to the wrong factor, or a row skipped or counted twice, changes some factor's exact inlier count.  References are
computed once per distinct (level, prefix, pose).  Maps and poses stay within about 40 m of the origin."""
import ctypes as C

import numpy as np
import pytest
import torch

from glim_b200 import capi, gpu, multi_gpu, synth
from oracle import oracle
from tests import grid_oracle as go
from tests import icp_oracle as icp
from tests import ivox_oracle as io
from tests import sweep_schedule as ss
from tests import voxelmap_oracle as vo
from tests import util
from tests.util import REL_TOL, check_linearized, cov_colmajor16

pytestmark = pytest.mark.gpu

LEVELS = (0.25, 0.5, 1.0)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def stats(sw):
    """gb_sweep_stats now (Sweep.num_tiles / .grid are read once, at construction) -> (num_tiles, grid)"""
    nt, gs = C.c_uint32(), C.c_uint32()
    capi.check(capi.lib().gb_sweep_stats(sw.h, None, None, C.byref(nt), C.byref(gs)))
    return nt.value, gs.value


def assert_plan(sw, p, what):
    assert stats(sw) == (p["num_tiles"], p["grid"]), (what, stats(sw), p["num_tiles"], p["grid"])


def assert_repeat(a, b, what):
    """two records of the same sweep at the same poses: inliers exact, blocks equal up to the order of fp64 atomics"""
    assert np.array_equal(a["num_inliers"], b["num_inliers"]), what
    for k in ("H_tt", "H_ss", "H_ts", "b_t", "b_s"):
        x, y = np.asarray(a[k]).reshape(len(a), -1), np.asarray(b[k]).reshape(len(b), -1)
        scale = np.maximum(np.linalg.norm(y, axis=1), np.sqrt(np.abs(np.asarray(b["error"]) * np.linalg.norm(np.asarray(b["H_tt"]).reshape(len(b), -1), axis=1))))
        assert (np.linalg.norm(x - y, axis=1) <= 1e-12 * scale).all(), (what, k)
    assert np.allclose(a["error"], b["error"], rtol=1e-12, atol=0), what


# ---------------------------------------------------------------------------------------------------------------------
# VGICP data: one 131 k-point scan, its three voxel levels, source prefixes and eight poses
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scene(ctx):
    sc = synth.make_hall_scene()
    pts, _ = synth.scan(sc, "os1_64", synth.arc_trajectory(8)[3], synth.rng_for(55, 3))
    nrm, cov = synth.with_covariances(pts, 10)
    assert len(pts) > ss.MAX_PREFIX
    xyz, cov6 = oracle.pack_cloud(pts, cov_colmajor16(cov))
    whole = gpu.PointCloudGPU.clone(pts, cov, nrm, ctx=ctx)
    rng = synth.rng_for(1200)
    poses = [synth.perturb(np.eye(4), rng, 0.01, 0.05) for _ in range(ss.N_POSES)]
    evals = [synth.perturb(T, rng, 0.005, 0.02) for T in poses]
    return {
        "pts": pts, "cov": cov, "nrm": nrm, "xyz": xyz, "cov6": cov6, "nrm32": nrm[:, :3].astype(np.float32),
        "maps": [gpu.GaussianVoxelMapGPU(r, ctx=ctx).insert(whole) for r in LEVELS],
        "refmaps": [oracle.GpuMap(xyz, cov6, r) for r in LEVELS],
        "poses": poses, "evals": evals, "clouds": {}, "refs": {},
    }


def cloud(ctx, S, n):
    if n not in S["clouds"]:
        P, Cv, N = S["pts"][:n], S["cov"][:n], S["nrm"][:n]
        S["clouds"][n] = gpu.PointCloudGPU.clone(P, Cv, N if n else None, ctx=ctx)
    return S["clouds"][n]


def reference(S, level, n, T, Te, sv):
    """-> (122-double oracle record at T, error at Te with the correspondences of T, rejected by the gate, its entry-wise
    scale), cached"""
    key = (level, n, T.tobytes(), Te.tobytes(), sv)
    if key not in S["refs"]:
        m = S["refmaps"][level]
        nr = S["nrm32"][:n] if sv else None
        rec, corr = oracle.linearize_gpumap(m, S["xyz"][:n], S["cov6"][:n], T, normals=nr)
        err = oracle.error_gpumap(m, S["xyz"][:n], S["cov6"][:n], T, Te, normals=nr)
        scale = util.record_scale(util.factor_hits(m.vmean, m.vcov, S["xyz"][:n], S["cov6"][:n], T, corr))
        S["refs"][key] = (rec, err, int((corr == -2).sum()), scale)
    return S["refs"][key]


class VgicpSet:
    """a regime's factors: factor f on level f % 3, prefix sizes[f], pose f % 8 (or the given poses)"""

    def __init__(self, ctx, S, sizes, sv=None, poses=None):
        self.ctx, self.S, self.sizes = ctx, S, list(sizes)
        F = len(sizes)
        self.levels = [f % len(LEVELS) for f in range(F)]
        self.sv = [bool(sv and sv(f)) for f in range(F)]
        self.T = np.stack([S["poses"][f % ss.N_POSES] for f in range(F)]) if poses is None else np.stack(poses)
        self.Te = np.stack([S["evals"][f % ss.N_POSES] for f in range(F)]) if poses is None else np.stack([synth.perturb(T, synth.rng_for(1201, f), 0.005, 0.02) for f, T in enumerate(poses)])
        self.refs = [reference(S, self.levels[f], self.sizes[f], self.T[f], self.Te[f], self.sv[f]) for f in range(F)]

    def factors(self):
        """fresh factor objects (each learns its own inlier fraction)"""
        out = []
        for f, n in enumerate(self.sizes):
            fac = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, self.S["maps"][self.levels[f]], cloud(self.ctx, self.S, n), ctx=self.ctx)
            fac.set_enable_surface_validation(self.sv[f])
            out.append(fac)
        return out

    def check(self, rec, what):
        for f, r in enumerate(self.refs):
            try:
                check_linearized(gpu.unpack_linearized(rec[f]), r[0], hits=r[3])
            except AssertionError as e:
                raise AssertionError((what, "factor", f, "points", self.sizes[f])) from e

    def check_error(self, e, what):
        for f, r in enumerate(self.refs):
            assert abs(e[f] - r[1]) <= REL_TOL * abs(r[1]) + 1e-12, (what, f, e[f], r[1])


def run_regime(ctx, fset, p, what):
    """The three checks of a regime whose built plan is p: a Sweep (plain launch, its stats before and after the fetch), then
    linearize / error / linearize / linearize on the cached sweep of a factor set.  -> the Sweep's records"""
    facs = fset.factors()
    sw = gpu.Sweep(ctx, facs)
    assert_plan(sw, p, what)
    sw.set_poses(fset.T)
    sw.launch()
    rec = sw.fetch()
    fset.check(rec, what)
    learned, _ = ss.learn(p, rec["num_inliers"])
    assert_plan(sw, learned, (what, "after the fetch"))
    fs = gpu.NonlinearFactorSetGPU(ctx).add(facs)
    l1 = fs.linearize_deltas(fset.T)
    fset.check(l1, (what, "set"))
    fset.check_error(fs.error_deltas(fset.T, fset.Te), what)
    l2 = fs.linearize_deltas(fset.T)
    l3 = fs.linearize_deltas(fset.T)
    assert_repeat(l1, l2, what)
    assert_repeat(l2, l3, what)
    return rec


# ---------------------------------------------------------------------------------------------------------------------
# sweep5
# ---------------------------------------------------------------------------------------------------------------------
def test_r1_sweep5_with_and_without_descriptor_cache(ctx, scene):
    """F = 40 (descriptors and poses cached in shared memory) and F = 41 (read from the table), ragged sizes with 0, 1, 31
    and 33 points: one wave of strided items."""
    n = sms()
    plans = ss.plans_of("R1", n)
    ss.check_regime("R1", plans, n)
    for sizes, p in zip(ss.regimes(n)["R1"]["sizes"], plans):
        run_regime(ctx, VgicpSet(ctx, scene, sizes), p, ("R1", p["F"], "cached" if p["cached"] else "uncached"))


def test_r2_sweep5_queue_with_look_ahead(ctx, scene):
    """16 x SMs + 300 factors of 1-97 points: more items than warps, so sweep5 draws further items from the queue one item
    ahead; the repeated launches check the ctr_base advance (items + one look-ahead draw per warp)."""
    n = sms()
    (p,) = ss.plans_of("R2", n)
    ss.check_regime("R2", [p], n)
    fset = VgicpSet(ctx, scene, ss.regimes(n)["R2"]["sizes"][0])
    run_regime(ctx, fset, p, "R2")
    # five more launches of one sweep at alternating poses: a ctr_base behind the counter skips items from the second on
    facs = fset.factors()
    sw = gpu.Sweep(ctx, facs)
    other = VgicpSet(ctx, scene, fset.sizes, poses=[fset.Te[f] for f in range(len(fset.sizes))])
    for k in range(5):
        s = fset if k % 2 == 0 else other
        sw.set_poses(s.T)
        sw.launch()
        s.check(sw.fetch(), ("R2 launch", k))
        assert_plan(sw, p, ("R2 launch", k))


def test_r3_sweep5_accumulator_copies(ctx, scene):
    """Single factors whose item counts select 1, 2, 4, 8 and 16 accumulator copies (acc_slots)."""
    n = sms()
    plans = ss.plans_of("R3", n)
    ss.check_regime("R3", plans, n)
    for sizes, p in zip(ss.regimes(n)["R3"]["sizes"], plans):
        run_regime(ctx, VgicpSet(ctx, scene, sizes), p, ("R3", p["acc_slots"]))


def test_r4_sweep5_calibration(ctx, scene):
    """Factors with near-full and near-zero inlier rates: the first fetch re-sizes the item table from the measured inlier
    fractions.  Later linearizations against the oracle through a Sweep's plain launches, through gb_sweep_linearize and
    through a factor set (the captured graph, captured again for the new table)."""
    n = sms()
    (p,) = ss.plans_of("R4", n)
    ss.check_regime("R4", [p], n)
    sizes = ss.regimes(n)["R4"]["sizes"][0]
    far = [synth.pose(30.0 - 4.0 * f, 25.0, 0.5, 1.0 + 0.1 * f) for f in range(len(sizes))]  # off the scan: few or no hits
    poses = [scene["poses"][f % ss.N_POSES] if f % 2 == 0 else far[f] for f in range(len(sizes))]
    fset = VgicpSet(ctx, scene, sizes, poses=poses)
    inl = [r[0][121] / max(nn, 1) for r, nn in zip(fset.refs, sizes)]
    assert min(inl[0::2]) > ss.CALIB_FRACTIONS[0] and max(inl[1::2]) < ss.CALIB_FRACTIONS[1], inl
    # plain launches
    sw = gpu.Sweep(ctx, fset.factors())
    assert_plan(sw, p, "R4")
    sw.set_poses(fset.T)
    sw.launch()
    rec = sw.fetch()
    fset.check(rec, "R4 first")
    learned, _ = ss.learn(p, rec["num_inliers"])
    assert learned["num_tiles"] != p["num_tiles"] and learned["graph"]  # the calibration changed the table
    assert_plan(sw, learned, "R4 calibrated")
    for k in range(2):
        sw.launch()
        fset.check(sw.fetch(), ("R4 plain", k))
    assert_plan(sw, learned, "R4 calibrated once")
    # gb_sweep_linearize: the graph, captured again after the first call re-sized the table
    sw2 = gpu.Sweep(ctx, fset.factors())
    r1 = sw2.linearize(fset.T)
    fset.check(r1, "R4 graph first")
    learned2, _ = ss.learn(p, r1["num_inliers"])
    assert learned2["num_tiles"] != p["num_tiles"]
    assert_plan(sw2, learned2, "R4 graph calibrated")
    r2 = sw2.linearize(fset.T)
    r3 = sw2.linearize(fset.T)
    fset.check(r2, "R4 graph recaptured")
    assert_repeat(r2, r3, "R4 graph")
    # the factor set of fresh factors: the same, through the cached sweep
    fs = gpu.NonlinearFactorSetGPU(ctx).add(fset.factors())
    fset.check(fs.linearize_deltas(fset.T), "R4 set first")
    fset.check_error(fs.error_deltas(fset.T, fset.Te), "R4 set")
    l2 = fs.linearize_deltas(fset.T)
    fset.check(l2, "R4 set recaptured")
    assert_repeat(l2, fs.linearize_deltas(fset.T), "R4 set")


# ---------------------------------------------------------------------------------------------------------------------
# sweep3
# ---------------------------------------------------------------------------------------------------------------------
def test_r5_sweep3_static_items(ctx, scene, monkeypatch):
    """GB_KERNEL = 3 at a size where every item is 128 points and the grid holds them all (no queue): sources of 479 / 480 /
    481, 991 and 2047 / 2048 / 2049 points near the identity pose, where most points hit, so each item ends on a partial pass
    of its hit queue."""
    monkeypatch.setenv("GB_KERNEL", "3")
    n = sms()
    (p,) = ss.plans_of("R5", n)
    ss.check_regime("R5", [p], n)
    run_regime(ctx, VgicpSet(ctx, scene, ss.regimes(n)["R5"]["sizes"][0]), p, "R5")


def test_r6_sweep3_queue_of_128_point_items(ctx, scene, monkeypatch):
    """GB_KERNEL = 3 with more 128-point items than warps: the queue path."""
    monkeypatch.setenv("GB_KERNEL", "3")
    n = sms()
    (p,) = ss.plans_of("R6", n)
    ss.check_regime("R6", [p], n)
    run_regime(ctx, VgicpSet(ctx, scene, ss.regimes(n)["R6"]["sizes"][0]), p, "R6")


def test_r7_sweep3_tapered_tail(ctx, scene):
    """More than 6 x 16 x SMs x 2048 point-factors, no override: 2048-point items whose 480-point rounds carry their last
    partial pass into the next round (factors of 481 .. 2049 points), then the tail cut to 512- and 128-point items; empty
    factors and factors of 1, 31 and 33 points among them."""
    n = sms()
    (p,) = ss.plans_of("R7", n)
    ss.check_regime("R7", [p], n)
    run_regime(ctx, VgicpSet(ctx, scene, ss.regimes(n)["R7"]["sizes"][0]), p, "R7")


def test_r8_sweep3_surface_validation(ctx, scene):
    """Factors with and without surface validation in one large sweep (k_vgicp_sweep3's SV instantiation), linearize and the
    gated error, against the oracle's gate."""
    n = sms()
    (p,) = ss.plans_of("R8", n)
    ss.check_regime("R8", [p], n)
    fset = VgicpSet(ctx, scene, ss.regimes(n)["R8"]["sizes"][0], sv=lambda f: f % 2 == 0)
    assert sum(r[2] for r in fset.refs) > 0 and any(fset.sv) and not all(fset.sv)  # the gate rejects correspondences
    run_regime(ctx, fset, p, "R8")


def slab_rows_match(rows, rec, fset, pair, num_pairs, rtol_h, rtol_b, what):
    """each slab row against the fp64 sum of the oracle records of its pair (1e-4, and entry-wise: the members' bounds plus the
    fp32 rounding of each summed level and of each fp32 sum of them) and of the device records (fp32 bars)"""
    used = set(pair)
    for q in range(num_pairs):
        if q not in used:
            assert not rows[q].any(), (what, q)
            continue
        got = multi_gpu.unpack_slab_row(rows[q])
        members = [f for f in range(len(pair)) if pair[f] == q]
        refs = [oracle.split122(fset.refs[f][0]) for f in members]
        want = {k: sum(r[k] for r in refs) for k in refs[0]}
        scale = fset.refs[members[0]][3]
        for f in members[1:]:
            scale = scale + fset.refs[f][3]
        stored = {k: len(members) * util.U32 * sum(np.abs(gpu.unpack_linearized(rec[f])[k]) for f in members) for k in util.KEYS}
        check_linearized(got, want, hits=scale + util.EntryScale({k: np.zeros_like(v) for k, v in stored.items()}, stored))
        for k in ("H_tt", "H_ss", "H_ts", "b_t", "b_s"):
            dev = sum(gpu.unpack_linearized(rec[f])[k] for f in members)
            rtol = rtol_b if k[0] == "b" else rtol_h
            assert np.allclose(got[k], dev, rtol=rtol, atol=rtol_h * np.abs(dev).max()), (what, q, k)
        assert got["num_inliers"] == sum(rec[f]["num_inliers"] for f in members), (what, q)


def test_r9_sweep3_slabs(ctx, scene):
    """A large sweep with pair indices interleaved across its factors, with an atomic slab and with a peer slab of world 1:
    every row equals its pair's summed records, the unused row stays zero, repeated peer steps are bit-identical."""
    n = sms()
    (p,) = ss.plans_of("R9", n)
    ss.check_regime("R9", [p], n)
    fset = VgicpSet(ctx, scene, ss.regimes(n)["R9"]["sizes"][0])
    F, num_pairs = len(fset.sizes), 12
    pair = [(4 * f) % 11 for f in range(F)]  # row 11 is used by no factor
    # atomic slab
    sw = gpu.Sweep(ctx, fset.factors(), pair_index=pair)
    assert_plan(sw, p, "R9 atomic")
    slab = torch.zeros((num_pairs, capi.GB_SLAB_STRIDE), dtype=torch.float32, device="cuda:0")
    torch.cuda.synchronize()
    sw.attach_slab(slab.data_ptr(), num_pairs)
    sw.set_poses(fset.T)
    sw.launch()
    rec = sw.fetch()
    ctx.synchronize()
    fset.check(rec, "R9 atomic")
    slab_rows_match(slab.cpu().numpy(), rec, fset, pair, num_pairs, 1e-6, 1e-5, "R9 atomic")
    # peer slab, world 1
    sw2 = gpu.Sweep(ctx, fset.factors(), pair_index=pair)
    assert_plan(sw2, p, "R9 peer")
    ps = gpu.PeerSlab(ctx, num_pairs)
    sw2.attach_peer_slab(ps)
    sw2.set_poses(fset.T)
    rows = []
    for _ in range(3):
        sw2.launch()
        ps.signal_wait()
        rows.append(ps.fetch())
    rec2 = sw2.fetch()
    fset.check(rec2, "R9 peer")
    assert rows[0].tobytes() == rows[1].tobytes() == rows[2].tobytes()
    slab_rows_match(rows[0], rec2, fset, pair, num_pairs, 2e-7, 2e-7, "R9 peer")


# ---------------------------------------------------------------------------------------------------------------------
# the GICP and ICP sweeps
# ---------------------------------------------------------------------------------------------------------------------
GICP_MAX_CORR = 1.0
GRID_CELL = 1.05


@pytest.fixture(scope="module")
def gicp_data(ctx):
    """frames 0-2 of the arc in an iVox and frame 2 in a point grid, device and restated; frame 3 (NaN points included) as the
    source, eight poses about each target's ground truth"""
    frames = vo.arc_frames(4, 32 * 200, nan_frame=3)
    ivox = gpu.IVoxGPU(1.0, 0.1, 10, 1, 100, 10, ctx=ctx)
    R = io.IVox(1.0, 0.1, 10, 1, 100, 10)
    for k in (0, 1, 2):
        ivox.insert(gpu.PointCloudGPU.clone(frames[k][0], frames[k][1], ctx=ctx), frames[k][2])
        R.insert(*oracle.pack_cloud(frames[k][0], cov_colmajor16(frames[k][1])), frames[k][2])
    tgt = gpu.PointCloudGPU.clone(frames[2][0], frames[2][1], ctx=ctx)
    xt, ct = tgt.download()
    grid = gpu.PointGridGPU(tgt, GRID_CELL, ctx=ctx)
    P, Cv = frames[3][0], frames[3][1]
    xyz, cov6 = oracle.pack_cloud(P, cov_colmajor16(Cv))
    assert len(P) >= max(ss.GICP_WAVE)
    rng = synth.rng_for(1300)
    out = {"P": P, "Cv": Cv, "xyz": xyz, "cov6": cov6, "clouds": {}}
    for kind, target, restated, T0 in (("ivox", ivox, R, frames[3][2]), ("gicp_grid", grid, go.PointGrid(xt, ct, GRID_CELL), synth.inv_pose(frames[2][2]) @ frames[3][2]),
                                       ("icp_grid", grid, icp.grid(xt, GRID_CELL), synth.inv_pose(frames[2][2]) @ frames[3][2])):
        poses = [T0] + [synth.perturb(T0, rng, 0.01, 0.1) for _ in range(ss.N_POSES - 1)]
        evals = [synth.perturb(T, rng, 0.005, 0.05) for T in poses]
        out[kind] = {"target": target, "R": restated, "poses": poses, "evals": evals, "corr": {}, "refs": {}}
    return out


def gicp_reference(D, kind, n, k):
    """(record dict, error at the eval pose, 0, entry-wise scale) of prefix n at pose k; correspondences once per pose for the
    longest prefix"""
    K = D[kind]
    if (n, k) not in K["refs"]:
        m, T, Te = K["R"], K["poses"][k], K["evals"][k]
        top = max(ss.GICP_WAVE + ss.TINY)
        if k not in K["corr"]:
            xyz = D["xyz"][:top]
            corr = io.correspondences(m, xyz, T, GICP_MAX_CORR) if kind == "ivox" else go.correspondences(m, xyz, T, GICP_MAX_CORR)
            K["corr"][k] = corr
        corr = K["corr"][k][:n]
        xyz, cov6 = D["xyz"][:n], D["cov6"][:n]
        if kind == "icp_grid":
            rec = icp.linearize(m, xyz, T, GICP_MAX_CORR, corr=corr)[0]
            err = icp.linearize(m, xyz, Te, GICP_MAX_CORR, corr=corr)[0]["error"]
            scale = util.record_scale(util.factor_hits(m.xyz, None, xyz, None, T, corr))
        else:
            rec = io.linearize(m, xyz, cov6, T, GICP_MAX_CORR, corr=corr)[0]
            err = io.linearize(m, xyz, cov6, Te, GICP_MAX_CORR, corr=corr)[0]["error"]
            scale = util.record_scale(util.factor_hits(m.xyz, m.cov6, xyz, cov6, T, corr))
        K["refs"][(n, k)] = (rec, err, 0, scale)
    return K["refs"][(n, k)]


class GicpSet(VgicpSet):
    def __init__(self, ctx, D, kind, sizes):
        self.ctx, self.D, self.kind, self.sizes = ctx, D, kind, list(sizes)
        K = D[kind]
        F = len(sizes)
        self.T = np.stack([K["poses"][f % ss.N_POSES] for f in range(F)])
        self.Te = np.stack([K["evals"][f % ss.N_POSES] for f in range(F)])
        self.refs = [gicp_reference(D, kind, n, f % ss.N_POSES) for f, n in enumerate(sizes)]

    def factors(self):
        out = []
        for n in self.sizes:
            if n not in self.D["clouds"]:
                self.D["clouds"][n] = gpu.PointCloudGPU.clone(self.D["P"][:n], self.D["Cv"][:n], ctx=self.ctx)
            cls = gpu.IntegratedICPFactorGPU if self.kind == "icp_grid" else gpu.IntegratedGICPFactorGPU
            out.append(cls(np.eye(4), 0, self.D[self.kind]["target"], self.D["clouds"][n], GICP_MAX_CORR, ctx=self.ctx))
        return out


@pytest.mark.parametrize("kind", ["ivox", "gicp_grid", "icp_grid"])
def test_r10_gicp_and_icp_sweeps(ctx, gicp_data, kind):
    """k_gicp_sweep (iVox), k_gicp_grid_sweep and k_icp_grid_sweep (point grid): one wave of strided items, and the queue with
    more factors than warps, against tests/ivox_oracle.py, tests/grid_oracle.py and tests/icp_oracle.py."""
    n = sms()
    plans = ss.plans_of("R10", n)
    ss.check_regime("R10", plans, n)
    for sizes, p in zip(ss.regimes(n)["R10"]["sizes"], plans):
        fset = GicpSet(ctx, gicp_data, kind, sizes)
        assert sum(r[0]["num_inliers"] for r in fset.refs) > 0.2 * sum(sizes)
        run_regime(ctx, fset, p, ("R10", kind, "queue" if p["dynamic"] else "wave"))
