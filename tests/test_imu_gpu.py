"""gb_imu_preintegrate on the H100: a batch of intervals against the restatement in tests/imu_oracle.py, one launch per call,
and the refusals made before any launch."""
import ctypes as C

import numpy as np
import pytest

from glim_b200 import capi, gpu
from tests import imu_oracle as io

pytestmark = pytest.mark.gpu


def test_batch_matches_the_restatement(ctx):
    """consecutive intervals over the analytic trajectory's 400 Hz samples with duplicate stamps, an interval ending past the
    last sample and one before the first: about 1e-12 relative, num_integrated exact, one launch"""
    rng = np.random.default_rng(5)
    bias = np.array([0.05, -0.03, 0.08, 0.004, -0.002, 0.003])
    s = io.samples(0.0, 6.0, 400, bias)
    s[100, 0] = s[99, 0]
    edges = np.concatenate([[0.0], np.sort(rng.uniform(0.01, 5.9, size=40)), [5.95]])
    intervals = list(zip(edges[:-1], edges[1:])) + [(5.5, 6.5), (-1.0, -0.5)]
    biases = [bias + rng.normal(size=6) * 0.01 for _ in intervals]
    before = ctx.kernel_launches
    got = gpu.imu_preintegrate(s, intervals, biases, ctx=ctx)
    assert ctx.kernel_launches - before == 1
    for r, (a, b), bb in zip(got, intervals, biases):
        ref = io.preintegrate(s, a, b, bb)
        assert int(r["num_integrated"]) == ref["num_integrated"]
        assert abs(r["delta_t"] - ref["delta_t"]) <= 1e-14 * max(1.0, ref["delta_t"])
        for k in ("preintegrated", "H_bias_acc", "H_bias_omega", "covariance"):
            scale = np.abs(ref[k]).max()
            assert np.abs(r[k] - ref[k]).max() <= 1e-12 * max(scale, 1e-300), (a, b, k)
        assert np.array_equal(r["covariance"], r["covariance"].T)
        assert np.array_equal(r["bias_hat"], bb) and np.array_equal(r["gravity"], io.DEFAULT_PARAMS["gravity"])
    assert got[-1]["num_integrated"] == 0 and got[-1]["delta_t"] == 0.5  # before the first sample: one final step with the first
    again = gpu.imu_preintegrate(s, intervals, biases, ctx=ctx)
    assert again.tobytes() == got.tobytes()
    other = gpu.imu_preintegrate(s, intervals[:3], biases[:3], params={"acc_noise": 0.1, "gravity": (0.0, 0.0, -9.8)}, ctx=ctx)
    ref = io.preintegrate(s, *intervals[1], biases[1], dict(acc_noise=0.1, gravity=np.array([0.0, 0.0, -9.8])))
    assert np.abs(other[1]["covariance"] - ref["covariance"]).max() <= 1e-12 * np.abs(ref["covariance"]).max()


def test_invalid_inputs_are_refused_before_any_launch(ctx):
    L = capi.lib()
    s = capi.f64(io.samples(0.0, 1.0, 200, np.zeros(6)))
    itv = capi.f64([[0.1, 0.5], [0.5, 0.9]])
    bia = capi.f64(np.zeros((2, 6)))
    out = np.zeros(2, capi.PREINTEGRATED_DTYPE)
    good = gpu.imu_params()

    def call(samples=s, intervals=itv, biases=bia, prm=good):
        return L.gb_imu_preintegrate(ctx.h, len(samples), capi.ptr(samples), len(intervals), capi.ptr(intervals), capi.ptr(biases),
                                     C.byref(prm) if prm is not None else None, capi.ptr(out))

    before = ctx.kernel_launches
    unsorted = s.copy()
    unsorted[[3, 4]] = unsorted[[4, 3]]
    nan = s.copy()
    nan[7, 2] = np.nan
    assert call(samples=unsorted) == 1 and "decrease" in L.gb_last_error().decode()
    assert call(samples=nan) == 1
    assert call(intervals=capi.f64([[0.5, 0.1], [0.5, 0.9]])) == 1
    assert call(biases=capi.f64([[np.inf] + [0.0] * 5, [0.0] * 6])) == 1
    assert call(prm=None) == 1 and call(prm=gpu.imu_params(acc_noise=-1.0)) == 1 and call(prm=gpu.imu_params(gravity=(0.0, np.nan, 0.0))) == 1
    assert ctx.kernel_launches == before
    assert call() == 0 and ctx.kernel_launches == before + 1
