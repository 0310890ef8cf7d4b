"""CloudDeskewing (SURVEY 8(f) row 2; src/glim/common/cloud_deskewing.cpp).

CPU: the oracle's two overloads against an independent numpy / scipy implementation; the product's HOST half
(gb_deskew_pose_table: time table + pose per slot, needs no device) against the oracle.
GPU: the kernel (gb_deskew) against the oracle."""
import numpy as np
import pytest

from glim_b200 import synth
from oracle import oracle


def scan_like(n=20000, seed=0):
    rng = np.random.default_rng(seed)
    times = np.sort(rng.uniform(0.0, 0.1, n))
    times[:50] = 0.0  # several points share the first slot
    pts = np.concatenate([rng.normal(0, 15, (n, 3)), np.ones((n, 1))], axis=1)
    return times, pts


def numpy_table(times):
    tab, idx = [], []
    for t in times:
        if not tab or t - tab[-1] > 1e-4:
            tab.append(t)
        idx.append(len(tab) - 1)
    return np.array(tab), np.array(idx)


T_IL = synth.pose(0.1, -0.05, 0.2, 0.3, 0.02, -0.01)
V, W = np.array([3.0, 0.2, -0.1]), np.array([0.05, -0.1, 0.8])
IMU_T = 100.0 + np.arange(-0.02, 0.14, 0.01)
IMU_P = np.stack([synth.pose(1 + 3 * (t - 100), 0.2 * (t - 100), 0.0, 0.5 + 0.8 * (t - 100), 0.02 * np.sin(30 * (t - 100)), 0.01) for t in IMU_T])


def numpy_const_vel(times, pts):
    tab, idx = numpy_table(times)
    Ts = np.stack([synth.inv_pose(T_IL) @ synth.inv_pose(synth.se3_exp(np.concatenate([W, V]) * dt)) @ T_IL for dt in tab])
    return np.einsum("nij,nj->ni", Ts[idx], pts)


def numpy_imu(times, pts, imu_t=IMU_T, imu_p=IMU_P, stamp=100.0):
    from scipy.spatial.transform import Rotation as Rot, Slerp

    tab, idx = numpy_table(times)
    cursor, Ts, T0w = 0, [], None
    for i, t in enumerate(tab):
        time = stamp + t
        while cursor < len(imu_t) - 1 and imu_t[cursor + 1] < time:
            cursor += 1
        if i == 0:
            T0w = synth.inv_pose(imu_p[cursor])
        if cursor + 1 >= len(imu_t):
            T = imu_p[cursor]
        else:
            p = min(1.0, max(0.0, (time - imu_t[cursor]) / (imu_t[cursor + 1] - imu_t[cursor])))
            T = np.eye(4)
            T[:3, 3] = (1 - p) * imu_p[cursor][:3, 3] + p * imu_p[cursor + 1][:3, 3]
            T[:3, :3] = Slerp([0, 1], Rot.from_matrix([imu_p[cursor][:3, :3], imu_p[cursor + 1][:3, :3]]))([p])[0].as_matrix()
        Ts.append(synth.inv_pose(T_IL) @ T0w @ T @ T_IL)
    return np.einsum("nij,nj->ni", np.stack(Ts)[idx], pts)


def test_oracle_matches_numpy_scipy():
    times, pts = scan_like()
    assert np.allclose(oracle.deskew_const_vel(T_IL, V, W, times, pts), numpy_const_vel(times, pts), rtol=0, atol=1e-11)
    assert np.allclose(oracle.deskew_imu(T_IL, IMU_T, IMU_P, 100.0, times, pts), numpy_imu(times, pts), rtol=0, atol=1e-11)
    # fused second transform == transforming afterwards (odometry_estimation_imu.cpp:314-316)
    a = oracle.deskew_imu(T_IL, IMU_T, IMU_P, 100.0, times, pts, T_post=T_IL)
    b = oracle.deskew_imu(T_IL, IMU_T, IMU_P, 100.0, times, pts) @ T_IL.T
    assert np.allclose(a, b, rtol=0, atol=1e-12)
    # zero motion is the identity; an empty cloud stays empty; IMU poses that end early are held (:104-105)
    assert np.allclose(oracle.deskew_const_vel(T_IL, np.zeros(3), np.zeros(3), times, pts), pts, atol=1e-12)
    assert oracle.deskew_const_vel(T_IL, V, W, np.zeros(0), np.zeros((0, 4))).shape == (0, 4)
    short = oracle.deskew_imu(T_IL, IMU_T[:6], IMU_P[:6], 100.0, times, pts)
    assert np.allclose(short, numpy_imu(times, pts, IMU_T[:6], IMU_P[:6]), atol=1e-11)
    # no IMU poses at all -> zero-velocity model (:69-71)
    assert np.allclose(oracle.deskew_imu(T_IL, np.zeros(0), np.zeros((0, 4, 4)), 100.0, times, pts), pts, atol=1e-12)


def test_product_host_pose_table_matches_oracle():
    """gb_deskew_pose_table runs on the host (the reference builds the table on the host too); applying it in numpy must
    reproduce the oracle's deskewed points."""
    from glim_b200 import preprocess

    times, pts = scan_like(seed=1)
    tab, idx_ref = numpy_table(times)
    idx, Ts = preprocess.deskew_pose_table(T_IL, times, linear_vel=V, angular_vel=W)
    assert np.array_equal(idx, idx_ref) and len(Ts) == len(tab)
    assert np.allclose(np.einsum("nij,nj->ni", Ts[idx], pts), oracle.deskew_const_vel(T_IL, V, W, times, pts), rtol=0, atol=1e-11)
    idx, Ts = preprocess.deskew_pose_table(T_IL, times, imu_times=IMU_T, imu_poses=IMU_P, stamp=100.0)
    assert np.array_equal(idx, idx_ref)
    assert np.allclose(np.einsum("nij,nj->ni", Ts[idx], pts), oracle.deskew_imu(T_IL, IMU_T, IMU_P, 100.0, times, pts), rtol=0, atol=1e-11)
    for lv, av in ((V, None), (None, W)):  # either velocity may be omitted = zero (include/glim_b200.h)
        idx, Ts = preprocess.deskew_pose_table(T_IL, times, linear_vel=lv, angular_vel=av)
        want = oracle.deskew_const_vel(T_IL, np.zeros(3) if lv is None else lv, np.zeros(3) if av is None else av, times, pts)
        assert np.allclose(np.einsum("nij,nj->ni", Ts[idx], pts), want, rtol=0, atol=1e-11)
    idx, Ts = preprocess.deskew_pose_table(T_IL, times)  # neither velocities nor poses: identity table
    assert np.allclose(Ts, np.eye(4), atol=1e-15)
    idx, Ts = preprocess.deskew_pose_table(T_IL, np.zeros(0))
    assert len(idx) == 0 and len(Ts) == 0


GPU_CHECK = r"""
import sys, numpy as np
sys.path.insert(0, {root!r})
from glim_b200 import gpu, preprocess
from oracle import oracle
from tests.test_deskew import scan_like, T_IL, V, W, IMU_T, IMU_P
ctx = gpu.Context(0)
times, pts = scan_like(n=60000, seed=2)
d = preprocess.CloudDeskewing(ctx=ctx)
assert np.allclose(d.deskew(T_IL, times, pts, linear_vel=V, angular_vel=W), oracle.deskew_const_vel(T_IL, V, W, times, pts), rtol=0, atol=1e-11)
assert np.allclose(d.deskew(T_IL, times, pts, imu_times=IMU_T, imu_poses=IMU_P, stamp=100.0, T_post=T_IL), oracle.deskew_imu(T_IL, IMU_T, IMU_P, 100.0, times, pts, T_post=T_IL), rtol=0, atol=1e-11)
assert d.deskew(T_IL, np.zeros(0), np.zeros((0, 4))).shape == (0, 4)
print("deskew gpu ok")
"""


@pytest.mark.gpu
def test_gpu_deskew_matches_oracle():
    """Runs in a subprocess so that a fault in the never-executed kernel cannot poison the CUDA context of the other GPU tests."""
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", GPU_CHECK.format(root=root)], capture_output=True, text=True, timeout=300, cwd=root)
    assert out.returncode == 0 and "deskew gpu ok" in out.stdout, out.stderr[-1500:]
