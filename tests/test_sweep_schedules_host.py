"""The oracle of the gated VGICP error (go_vgicp_error_gpumap_sv) against the oracle's own linearization, and the restated sweep
schedule of tests/sweep_schedule.py: for the SM counts of the H100 PCIe (114) and SXM (132), the sizes that
tests/test_sweep_schedules_gpu.py computes reach every regime it names."""
import numpy as np
import pytest

from glim_b200 import synth
from oracle import oracle
from tests import sweep_schedule as ss
from tests import util


@pytest.fixture(scope="module")
def data():
    pair = util.scan_pair()
    xyz0, cov0 = oracle.pack_cloud(pair["points"][0], util.cov_colmajor16(pair["covs"][0]))
    xyz1, cov1 = oracle.pack_cloud(pair["points"][1], util.cov_colmajor16(pair["covs"][1]))
    T = synth.inv_pose(pair["poses"][0]) @ pair["poses"][1]
    m = oracle.GpuMap(xyz0, cov0, 0.5)
    return m, xyz1, cov1, pair["normals"][1], util.test_poses(T, 3, key=41)


def old_error(m, xyz, cov6, T_lin, T_eval):
    xyz, cov6 = np.ascontiguousarray(xyz, np.float32), np.ascontiguousarray(cov6, np.float32)
    return oracle.lib().go_vgicp_error_gpumap(m.h, len(xyz), oracle._p(xyz), oracle._p(cov6), oracle._p(oracle.pose_colmajor(T_lin)), oracle._p(oracle.pose_colmajor(T_eval)))


def test_error_without_normals_is_unchanged(data):
    m, xyz, cov6, _, poses = data
    for T_lin in poses:
        for T_eval in poses:
            assert oracle.error_gpumap(m, xyz, cov6, T_lin, T_eval) == old_error(m, xyz, cov6, T_lin, T_eval)


def test_gated_error_at_the_linearization_point_is_the_linearized_error(data):
    m, xyz, cov6, normals, poses = data
    for T in poses:
        rec, corr = oracle.linearize_gpumap(m, xyz, cov6, T, normals=normals)
        assert (corr == -2).any()
        assert oracle.error_gpumap(m, xyz, cov6, T, T, normals=normals) == rec[120]


def test_gated_error_drops_exactly_the_rejected_correspondences(data):
    """At T_eval != T_lin the gate decides at T_lin: the gated error is the plain error of the points the gate kept there."""
    m, xyz, cov6, normals, poses = data
    for T_lin, T_eval in zip(poses, poses[1:] + poses[:1]):
        _, corr = oracle.linearize_gpumap(m, xyz, cov6, T_lin, normals=normals)
        keep = corr != -2
        assert not keep.all()
        gated = oracle.error_gpumap(m, xyz, cov6, T_lin, T_eval, normals=normals)
        assert gated == oracle.error_gpumap(m, xyz[keep], cov6[keep], T_lin, T_eval)
        assert gated < oracle.error_gpumap(m, xyz, cov6, T_lin, T_eval)
        # deciding at T_eval instead would reject another set
        _, corr_e = oracle.linearize_gpumap(m, xyz, cov6, T_eval, normals=normals)
        assert not np.array_equal(corr_e == -2, corr == -2)


@pytest.mark.parametrize("sms", [114, 132])
@pytest.mark.parametrize("regime", [f"R{k}" for k in range(1, 11)])
def test_restated_schedule_reaches_every_regime(sms, regime):
    ss.check_regime(regime, ss.plans_of(regime, sms), sms)


def test_restated_schedule_follows_the_rules():
    """A few values of the rules worked by hand (132 SMs: 264 CTAs, 2112 warps)."""
    p = ss.plan([76800], 132)  # sweep5, one factor of 2400 rows: 600 items of 4 rows, 16 accumulator copies
    assert (p["kernel"], p["num_tiles"], p["grid"], p["acc_slots"]) == (5, 600, 75, 16)
    p = ss.plan([0, 1], 132)  # empty factors still get one item each
    assert (p["num_tiles"], p["grid"], p["dynamic"]) == (2, 1, False)
    p = ss.plan([128] * 2113, 132)  # one item more than warps: the queue, with sweep5's look-ahead draws
    assert p["dynamic"] and p["ctr_advance"] == 2113 + 2112
    p = ss.plan([2048] * 2113, 132)  # 2048 x 2113 > 2048 x 2112 points: sweep3, items of 4327424 / (2112 x 6) + 1 -> 352 points
    assert (p["kernel"], p["tile_size"]) == (3, 352) and p["ctr_advance"] == p["num_tiles"]
    p = ss.plan([128] * 2113, 132, gicp=True)
    assert p["kernel"] == 5 and p["ctr_advance"] == 2113 and not p["cached"]
    assert ss.plan([100] * 40, 132)["cached"] and not ss.plan([100] * 41, 132)["cached"]
