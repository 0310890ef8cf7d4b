"""gb_vgicp_align on the H100: Levenberg-Marquardt registration of many problems in one call, against the restatement
of the same rule in tests/align_oracle.py (align_gpumap, on the CPU oracle) and against ground truth."""
import ctypes as C

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth, workloads
from oracle import oracle
from tests import align_oracle
from tests import lm_oracle as lm
from tests.util import cov_colmajor16, scan_pair

pytestmark = pytest.mark.gpu


def pose_error(T, T_ref):
    d = synth.inv_pose(T_ref) @ T
    return float(np.linalg.norm(d[:3, 3])), float(np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1)))


class Scene:
    """one scan pair as device objects (clouds, maps at 0.5 / 1.0 m) and as oracle objects"""

    def __init__(self, ctx, pair, resolutions=(0.5, 1.0)):
        self.ctx = ctx
        P0, P1 = pair["points"]
        C0, C1 = pair["covs"]
        self.T_gt = synth.inv_pose(pair["poses"][0]) @ pair["poses"][1]
        self.normals = np.ascontiguousarray(pair["normals"][1][:, :4]) if pair.get("normals") else None
        tgt = gpu.PointCloudGPU.clone(P0, C0, ctx=ctx)
        self.sources = {}
        self.packed = {}
        self.gmaps = [gpu.GaussianVoxelMapGPU(r, ctx=ctx).insert(tgt) for r in resolutions]
        xyz0, cov0 = oracle.pack_cloud(P0, cov_colmajor16(C0))
        self.omaps = [oracle.GpuMap(xyz0, cov0, r) for r in resolutions]
        self.P1, self.C1 = P1, C1

    def source(self, step=1):
        """every step-th point of the source scan (with its normals)"""
        if step not in self.sources:
            P, Cv = np.ascontiguousarray(self.P1[::step]), np.ascontiguousarray(self.C1[::step])
            nr = np.ascontiguousarray(self.normals[::step]) if self.normals is not None else None
            self.sources[step] = gpu.PointCloudGPU.clone(P, Cv, nr, ctx=self.ctx)
            self.packed[step] = oracle.pack_cloud(P, cov_colmajor16(Cv)) + (nr,)
        return self.sources[step]

    def factors(self, levels=(0, 1), step=1, sv=False):
        out = []
        for l in levels:
            f = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, self.gmaps[l], self.source(step), ctx=self.ctx)
            f.set_enable_surface_validation(sv)
            out.append(f)
        return out

    def oracle(self, T0, levels=(0, 1), step=1, sv=False, params=None):
        self.source(step)
        xyz, cov6, nr = self.packed[step]
        return align_oracle.align_gpumap([self.omaps[l] for l in levels], xyz, cov6, T0, params=params, normals=nr if sv else None)


@pytest.fixture(scope="module")
def scene(ctx):
    return Scene(ctx, scan_pair(n_rays=32 * 200))


def start(scene, seed):
    return synth.perturb(scene.T_gt, synth.rng_for(seed), 0.02, 0.25)


def test_one_iteration_matches_oracle(scene):
    T0 = start(scene, 41)
    got = gpu.align_vgicp([scene.factors()], [T0], params={"max_iterations": 1})[0]
    ref = scene.oracle(T0, params={"max_iterations": 1})
    et, er = pose_error(got["T_target_source"], ref["T"])
    assert et < 1e-4 and er < 1e-5, (et, er)
    assert (got["iterations"], got["trials"], got["status"]) == (ref["iterations"], ref["trials"], ref["status"]) == (1, 1, lm.ALIGN_MAX_ITERATIONS)
    assert got["num_inliers"] == ref["num_inliers"]


@pytest.mark.parametrize("kernel", ["3", "5"])
def test_full_run_matches_oracle_and_ground_truth(scene, monkeypatch, kernel):
    monkeypatch.setenv("GB_KERNEL", kernel)
    for seed in (43, 44):
        T0 = start(scene, seed)
        got = gpu.align_vgicp([scene.factors()], [T0])[0]
        ref = scene.oracle(T0)
        et, er = pose_error(got["T_target_source"], ref["T"])
        assert et < 2e-3 and er < 2e-3, (seed, et, er, got, ref)
        gt, gr = pose_error(got["T_target_source"], scene.T_gt)
        assert gt < 0.03 and gr < 2e-3, (seed, gt, gr)
        assert got["status"] == ref["status"] == lm.ALIGN_CONVERGED, (seed, got, ref)
        assert got["iterations"] <= 8


def batch_problems(scene, count=66):
    """mixed problems: 2-level full scans, 1-level half scans, 2-level quarter scans, one with surface validation, one whose
    source starts 1 km away (no inlier at all)"""
    specs = []
    for i in range(count):
        kind = i % 3
        spec = dict(levels=(0, 1) if kind != 1 else (0,), step=(1, 2, 4)[kind], sv=False)
        spec["T0"] = start(scene, 600 + i)
        specs.append(spec)
    specs[5]["sv"] = True
    specs[7]["T0"] = specs[7]["T0"].copy()
    specs[7]["T0"][:3, 3] += 1000.0
    return specs, 7


def test_batch_matches_solo_runs_and_oracle(scene, ctx):
    specs, degenerate = batch_problems(scene)
    problems = [scene.factors(s["levels"], s["step"], s["sv"]) for s in specs]
    T0 = [s["T0"] for s in specs]
    launches = ctx.kernel_launches
    batch = gpu.align_vgicp(problems, T0)
    launches = ctx.kernel_launches - launches
    assert launches <= 4 * max(r["iterations"] + r["trials"] for r in batch)
    assert launches <= 4 * (max(r["trials"] for r in batch) + 1)
    d = batch[degenerate]
    assert d["status"] == capi.ALIGN_DEGENERATE and np.array_equal(d["T_target_source"], T0[degenerate])
    assert (d["iterations"], d["trials"], d["num_inliers"]) == (1, 0, 0.0)
    flipped, missed = [], []
    for i, (s, r) in enumerate(zip(specs, batch)):
        if i == degenerate:
            continue
        solo = gpu.align_vgicp([problems[i]], [T0[i]])[0]
        et, er = pose_error(r["T_target_source"], solo["T_target_source"])
        if (r["iterations"], r["trials"], r["status"]) == (solo["iterations"], solo["trials"], solo["status"]):
            assert et < 1e-6 and er < 1e-6, (i, et, er, r, solo)
        else:
            # the batch sums each factor's fp32 partial sums in another order than the solo sweep: where a trial's error
            # ties with the current one to that rounding, the two runs may decide differently -- only at the noise floor,
            # so the poses stay within one step shorter than the 1e-3 m step tolerance
            flipped.append(i)
            assert et < 1e-3 and er < 1e-4, (i, et, er, r, solo)
        ref = scene.oracle(s["T0"], s["levels"], s["step"], s["sv"])
        et, er = pose_error(r["T_target_source"], ref["T"])
        assert et < 2e-3 and er < 2e-3, (i, et, er, r, ref)
        # a one-level start on the half-density scan can stop in a local minimum away from ground truth; the oracle
        # stops there too, and the device must reach the bar wherever the oracle does
        gt, gr = pose_error(r["T_target_source"], scene.T_gt)
        ot, orr = pose_error(ref["T"], scene.T_gt)
        if ot < 0.025 and orr < 1.5e-3:
            assert gt < 0.03 and gr < 2e-3, (i, gt, gr)
        else:
            missed.append(i)
        assert r["status"] != capi.ALIGN_DEGENERATE and r["iterations"] <= 8
    assert len(flipped) <= len(specs) // 8, flipped
    assert len(missed) <= len(specs) // 8, missed


def test_dense_frame_on_the_queue_kernel(ctx, monkeypatch):
    """One MID-360-shaped 500 k-point frame against the previous one at 0.1 / 0.2 m, on k_vgicp_sweep3 (its queue head
    advances with every launch of every round)."""
    monkeypatch.setenv("GB_KERNEL", "3")
    sc = synth.make_hall_scene()
    traj = synth.arc_trajectory(2, step=0.5)
    frames = [workloads.make_scan(sc, "mid360", traj[i], synth.rng_for(701, i), n_rays=500_000, ctx=ctx, use_gpu=True) for i in (0, 1)]
    pair = {"points": [f[0] for f in frames], "covs": [f[1] for f in frames], "poses": list(traj)}
    big = Scene(ctx, pair, resolutions=(0.1, 0.2))
    assert len(pair["points"][1]) > 400_000
    T0 = synth.perturb(big.T_gt, synth.rng_for(702), 0.01, 0.1)
    got = gpu.align_vgicp([big.factors()], [T0])[0]
    ref = big.oracle(T0)
    et, er = pose_error(got["T_target_source"], ref["T"])
    assert et < 2e-3 and er < 2e-3, (et, er, got, ref)
    gt, gr = pose_error(got["T_target_source"], big.T_gt)
    assert gt < 0.03 and gr < 2e-3, (gt, gr)
    assert got["status"] in (capi.ALIGN_CONVERGED, capi.ALIGN_LAMBDA_EXCEEDED) and got["iterations"] <= 8


def test_factor_linearizes_as_before_after_align(scene):
    facs = scene.factors()
    T = start(scene, 45)
    before = [f.linearize({0: T}) for f in facs]
    gpu.align_vgicp([facs], [T])
    after = [f.linearize({0: T}) for f in facs]
    for a, b in zip(before, after):
        assert a["num_inliers"] == b["num_inliers"]
        for k in ("H_ss", "b_s", "H_tt", "b_t"):
            assert np.abs(a[k] - b[k]).max() <= 1e-12 * np.abs(b[k]).max(), k
        assert abs(a["error"] - b["error"]) <= 1e-12 * b["error"]


def test_invalid_inputs_are_rejected(scene, ctx):
    L = capi.lib()
    facs = scene.factors()
    arr = (C.c_void_p * 2)(*[f._handle() for f in facs])
    T0 = capi.pose16(np.stack([start(scene, 46)] * 2))
    res = (capi.AlignResult * 2)()
    good = gpu.align_params()

    def call(off, factors=arr, T=T0, prm=good, P=None):
        off = np.asarray(off, np.uint64)
        return L.gb_vgicp_align(ctx.h, len(off) - 1 if P is None else P, capi.ptr(off), C.cast(factors, C.c_void_p) if factors is not None else None, capi.ptr(T), C.byref(prm), C.cast(res, C.c_void_p))

    launches = ctx.kernel_launches
    assert call([1, 2]) == 1  # does not start at 0
    assert call([0, 2, 1]) == 1  # decreasing
    assert call([0, 1, 1]) == 1  # empty problem
    assert call([0, 2], factors=(C.c_void_p * 2)(arr[0], None)) == 1  # null factor
    assert call([0, 2], factors=None) == 1
    assert call([0, 2], prm=gpu.align_params(max_iterations=0)) == 1
    assert call([0, 2], prm=gpu.align_params(lambda_factor=1.0)) == 1
    assert call([0, 2], prm=gpu.align_params(lambda_initial=0.0)) == 1
    assert call([0, 2], prm=gpu.align_params(lambda_upper_bound=float("inf"))) == 1
    bad = T0.copy()
    bad[0, 13] = np.nan
    assert call([0, 1, 2], T=bad) == 1
    assert ctx.kernel_launches == launches  # validation precedes every launch
    assert call([0, 1, 2]) == 0 and call([0, 2]) == 0
