"""GLIM's passthrough sub-mapping without a GPU: glim_b200.sub_mapping_passthrough's parameters against the shipped configuration
(tests/golden/passthrough_config_values.json, from tests/golden/make_passthrough_config_fixture.py), and the module mirror's
decisions, run over the numpy iVox (tests/ivox_oracle.IVox) through its map_factory, against the restatement
tests/passthrough_oracle.py on scripted trajectories: keyframes, the cut under each criterion and at the end of the sequence,
the centre frame, the three poses and the seeds exactly, and the extracted points bit for bit."""
import json
import math
import os
import sys

import numpy as np
import pytest

from glim_b200 import sub_mapping_passthrough as spt
from glim_b200 import synth
from tests import ivox_oracle
from tests import passthrough_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = os.path.join(ROOT, "tests", "golden", "passthrough_config_values.json")


def test_params_are_the_shipped_config_converted():
    cfg = json.load(open(FIX))["config_sub_mapping_passthrough"]["sub_mapping"]
    p = spt.SubMappingPassthroughParams()
    assert p == spt.SubMappingPassthroughParams.from_config(cfg)
    assert p.keyframe_update_interval_rot == cfg["keyframe_update_interval_rot"] and p.keyframe_update_interval_trans == cfg["keyframe_update_interval_trans"]
    assert p.max_num_keyframes == cfg["max_num_keyframes"] == 50
    assert cfg["max_num_voxels"] == -1 and p.max_num_voxels == 2**31 - 1  # std::numeric_limits<int>::max()
    assert p.adaptive_max_num_voxels == cfg["adaptive_max_num_voxels"] == 2.5
    assert p.submap_target_num_points == cfg["submap_target_num_points"] and p.submap_voxel_resolution == cfg["submap_voxel_resolution"]
    assert p.min_dist_in_voxel == cfg["min_dist_in_voxel"] and p.max_num_points_in_voxel == cfg["max_num_points_in_voxel"]


def test_negative_limits_convert_as_the_constructor_does():
    p = spt.SubMappingPassthroughParams.from_config({"max_num_keyframes": -1, "max_num_voxels": -5, "adaptive_max_num_voxels": -1.0})
    assert p.max_num_keyframes == 2**31 - 1 and p.max_num_voxels == 2**31 - 1 and p.adaptive_max_num_voxels == sys.float_info.max
    d = spt.SubMappingPassthroughParams.from_config({})  # the code defaults of :16-35
    assert (d.max_num_keyframes, d.max_num_voxels, d.adaptive_max_num_voxels, d.submap_target_num_points, d.min_dist_in_voxel) == (50, 50000, 0.5, 40000, 0.1)


def test_count_rule():
    assert po.thin_count(65692, 50000) == 49999  # random_sampling's count at the module's rate, one short of the target
    assert po.thin_count(49, 1) == 0 and po.thin_count(50, 1) == 1
    assert po.thin_count(100, 0) == 100 and po.thin_count(100, -1) == 100 and po.thin_count(100, 100) == 100
    rng = np.random.default_rng(3)
    xyz = rng.uniform(-50, 50, (65692, 3)).astype(np.float32)
    q, c6 = po.extract(xyz, np.zeros((65692, 6), np.float32), None, 50000, 12345)
    assert len(q) == len(c6) == 49999


def test_rotation_angle_follows_eigen():
    rng = np.random.default_rng(5)
    for k in range(200):
        w = rng.normal(size=3)
        w *= (math.pi * rng.uniform(0, 1) if k % 2 else 1e-3 * rng.uniform()) / np.linalg.norm(w)
        R = synth.so3_exp(w)
        assert spt.rotation_angle(R) == po.angle(R)
        assert abs(spt.rotation_angle(R) - np.linalg.norm(w)) < 1e-9


class OracleMap:
    """The numpy iVox behind the mirror's map_factory: clouds are (xyz, cov6) fp32 pairs, voxel_data returns the restated
    extraction with its seed."""

    def __init__(self, resolution, min_dist_in_cell, max_points_in_cell, neighbor_voxel_mode, lru_horizon, lru_clear_cycle, ctx=None):
        assert (neighbor_voxel_mode, lru_horizon, lru_clear_cycle) == (1, 0, 2**31 - 1)
        self.m = ivox_oracle.IVox(resolution, min_dist_in_cell, max_points_in_cell, neighbor_voxel_mode, lru_horizon, lru_clear_cycle)

    def insert(self, cloud, T):
        self.m.insert(cloud[0], cloud[1], T)

    @property
    def num_voxels(self):
        return self.m.num_voxels

    @property
    def num_points(self):
        return self.m.num_points

    def voxel_data(self, T_out_map, target_num_points, seed):
        return seed, po.extract_ivox(self.m, T_out_map, target_num_points, seed)

    def close(self):
        self.m = None


def world_points(rng):
    """a floor, two walls and scattered posts along a corridor x in [-5, 40]"""
    n = 6000
    x = rng.uniform(-5, 40, n)
    kind = rng.integers(0, 4, n)
    y = np.where(kind == 1, -4.0, np.where(kind == 2, 4.0, rng.uniform(-4, 4, n)))
    z = np.where(kind == 0, -1.5, rng.uniform(-1.5, 2.5, n))
    return np.stack([x, y, z], 1)


def scripted_frames(seed=0, n_frames=40, step=0.35):
    """frames along the corridor: mostly steps of `step` m (keyframes), some standing still or turning slightly"""
    rng = np.random.default_rng(seed)
    W = world_points(rng)
    frames, x, yaw = [], 0.0, 0.0
    for i in range(n_frames):
        kind = i % 7
        if kind == 3:
            pass  # stands still: not a keyframe
        elif kind == 5:
            yaw += 0.02  # turns in place: a keyframe by rotation only
        elif kind == 6:
            x += 0.05  # creeps: not a keyframe
        else:
            x += step
        T = synth.pose(x, 0.1 * math.sin(0.3 * i), 0.0, yaw, 0.003 * i, 0.0)
        local = (W - T[:3, 3]) @ T[:3, :3]
        sel = np.nonzero(np.linalg.norm(local, axis=1) < 6.0)[0][:400]
        xyz = local[sel].astype(np.float32)
        A = rng.normal(scale=0.05, size=(len(sel), 3, 3))
        C = A @ np.swapaxes(A, 1, 2) + 1e-4 * np.eye(3)
        cov6 = np.stack([C[:, 0, 0], C[:, 0, 1], C[:, 0, 2], C[:, 1, 1], C[:, 1, 2], C[:, 2, 2]], 1).astype(np.float32)
        frames.append((100 + i, xyz, cov6, T))
    return frames


def mirror_run(params, frames):
    """the mirror over OracleMap: its submaps with the index of the frame whose insertion cut them (len(frames) at the end)"""
    mod = spt.SubMappingPassthroughGPU(params, map_factory=OracleMap)
    out = []
    for idx, (fid, xyz, cov6, T) in enumerate(frames):
        mod.insert_frame(fid, (xyz, cov6), T)
        out += [(s, idx) for s in mod.get_submaps()]
    out += [(s, len(frames)) for s in mod.submit_end_of_sequence()]
    return out


def assert_same(mine, ref):
    assert [after for _, after in mine] == [r["after"] for r in ref]
    for (s, _), r in zip(mine, ref):
        assert s.id == r["id"]
        assert s.odom_frame_ids == r["odom_frame_ids"] and s.keyframe_ids == r["keyframe_ids"]
        assert s.odom_frame_ids[len(s.odom_frame_ids) // 2] == r["odom_frame_ids"][r["center"]]
        for k in ("T_world_origin", "T_origin_endpoint_L", "T_origin_endpoint_R"):
            assert np.array_equal(getattr(s, k), r[k]), k
        seed, (q, c6) = s.frame
        assert seed == r["seed"]
        assert np.array_equal(q, r["q"]) and np.array_equal(c6, r["c6"])


INT_MAX, DBL_MAX = 2**31 - 1, sys.float_info.max


@pytest.mark.parametrize("criterion,overrides", [
    ("keyframes", dict(max_num_keyframes=6, max_num_voxels=INT_MAX, adaptive_max_num_voxels=DBL_MAX)),
    ("voxels", dict(max_num_keyframes=INT_MAX, max_num_voxels=450, adaptive_max_num_voxels=DBL_MAX)),
    ("adaptive", dict(max_num_keyframes=INT_MAX, max_num_voxels=INT_MAX, adaptive_max_num_voxels=1.3)),
    ("end", dict()),
])
def test_mirror_cuts_as_the_restatement(criterion, overrides):
    params = spt.SubMappingPassthroughParams(**{**dict(submap_target_num_points=500), **overrides})
    frames = scripted_frames()
    ref = po.run(params, frames)
    mine = mirror_run(params, frames)
    assert_same(mine, ref)
    reasons = [r["reason"] for r in ref]
    if criterion == "end":
        assert reasons == ["end"]
    else:
        assert reasons.count(criterion) >= 2 and set(reasons) <= {criterion, "end"}, reasons
    assert any(r["P"] > 500 for r in ref) and any(len(r["q"]) < r["P"] for r in ref)  # thinning took place
    # keyframes: the scripted stills and creeps are not keyframes, the turns in place are
    all_keys = [k for r in ref for k in r["keyframe_ids"]]
    assert 100 + 3 not in all_keys and 100 + 6 not in all_keys and 100 + 5 in all_keys


def test_seed_uses_the_count_before_its_increment():
    params = spt.SubMappingPassthroughParams(max_num_keyframes=4, submap_target_num_points=100)
    ref = po.run(params, scripted_frames(n_frames=20))
    assert len(ref) >= 3
    for k, r in enumerate(ref):
        assert r["id"] == k and r["seed"] == (k * 643145 + r["P"] * 4312) % 2**64 == spt.submap_seed(k, r["P"])


def test_capacity_clamp():
    params = spt.SubMappingPassthroughParams()
    made = []
    spt.SubMappingPassthroughGPU(params, map_factory=lambda *a, ctx=None: made.append(a) or OracleMap(*a))
    assert made == [(0.5, 0.2, 64, 1, 0, 2**31 - 1)]


def test_voxel_data_passes_any_target_without_wrapping(monkeypatch):
    """gb_ivox_extract takes an int target: IVoxGPU.voxel_data clamps a larger one to INT_MAX (every point stays either way, a
    map holding fewer than 2^30) and one at or below 0 to 0, where ctypes would wrap it silently; a seed outside [0, 2^64) is
    refused.  The library is replaced by a recorder."""
    from glim_b200 import gpu

    calls = []

    class Lib:
        def gb_ivox_extract(self, ctx, h, T, target, seed, out):
            calls.append((target, seed))
            out._obj.value = 0x1000
            return 0

        def gb_cloud_size(self, h, n):
            n._obj.value = 3
            return 0

        def gb_cloud_destroy(self, h):
            return 0

    monkeypatch.setattr(gpu, "lib", lambda: Lib())
    m = object.__new__(gpu.IVoxGPU)
    m.ctx, m.h = object.__new__(gpu.Context), None
    for target, sent in ((2**32 + 5, INT_MAX), (2**31, INT_MAX), (INT_MAX, INT_MAX), (50000, 50000), (1, 1), (0, 0), (-1, 0), (-2**40, 0)):
        c = m.voxel_data(None, target, 2**64 - 1)
        assert calls[-1] == (sent, 2**64 - 1) and c.n == 3
        c.h = None
    for seed in (-1, 2**64):
        with pytest.raises(ValueError):
            m.voxel_data(None, 10, seed)
    assert len(calls) == 8
