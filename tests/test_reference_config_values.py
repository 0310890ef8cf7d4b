"""SURVEY 8(c) item 3: GLIM's call sites and shipped configuration are authoritative for the constructor arguments, defaults and
flags of the path.  tests/golden/reference_config_values.json is extracted from GLIM's config/*.json by
tests/golden/make_reference_config_fixture.py; the product's defaults and the workload builders' parameters must equal it."""
import ctypes as C
import json
import os

from glim_b200 import capi, workloads

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = os.path.join(ROOT, "tests", "golden", "reference_config_values.json")


def fixture():
    return json.load(open(FIX))


def test_preprocess_defaults_are_the_shipped_config():
    """gb_preprocess_default_params (host-only entry point) = config/config_preprocess.json"""
    cfg = fixture()["config_preprocess"]["preprocess"]
    p = capi.PreprocessParams()
    assert capi.lib().gb_preprocess_default_params(C.byref(p)) == 0
    assert p.distance_near_thresh == cfg["distance_near_thresh"] and p.distance_far_thresh == cfg["distance_far_thresh"]
    assert bool(p.use_random_grid_downsampling) == cfg["use_random_grid_downsampling"]
    assert p.downsample_resolution == cfg["downsample_resolution"]
    assert p.downsample_target == cfg["random_downsample_target"] and p.downsample_rate == cfg["random_downsample_rate"]
    assert bool(p.enable_outlier_removal) == cfg["enable_outlier_removal"] and p.outlier_removal_k == cfg["outlier_removal_k"]
    assert p.outlier_std_mul_factor == cfg["outlier_std_mul_factor"]
    assert (p.crop_bbox_frame != 0) == cfg["enable_cropbox_filter"]
    assert p.k_correspondences == cfg["k_correspondences"]


def test_workload_builders_use_the_shipped_module_parameters():
    f = fixture()
    od = f["config_odometry_gpu"]["odometry_estimation"]
    p = workloads.OdometryParams()
    assert p.voxel_resolution == od["voxel_resolution"] and p.voxelmap_levels == od["voxelmap_levels"] and p.voxelmap_scaling_factor == od["voxelmap_scaling_factor"]
    assert p.full_connection_window_size == od["full_connection_window_size"] and p.max_num_keyframes == od["max_num_keyframes"]
    assert p.keyframe_min_overlap == od["keyframe_min_overlap"] and p.keyframe_max_overlap == od["keyframe_max_overlap"]
    assert p.smoother_lag_frames == int(od["smoother_lag"] * 10)  # 10 Hz stream
    assert od["keyframe_update_strategy"] == "OVERLAP"  # the rule odometry_stream emulates (odometry_estimation_gpu.cpp:212-295)
    gm = f["config_global_mapping_gpu"]["global_mapping"]
    sm = f["config_sub_mapping_gpu"]["sub_mapping"]
    g = workloads.GlobalMappingParams()
    assert g.submap_voxel_resolution == gm["submap_voxel_resolution"] and g.submap_voxelmap_levels == gm["submap_voxelmap_levels"]
    assert g.submap_voxelmap_scaling_factor == gm["submap_voxelmap_scaling_factor"]
    assert g.max_implicit_loop_distance == gm["max_implicit_loop_distance"] and g.min_implicit_loop_overlap == gm["min_implicit_loop_overlap"]
    assert g.submap_target_num_points == sm["submap_target_num_points"]
    assert gm["registration_error_factor_type"] == sm["registration_error_factor_type"] == "VGICP_GPU"
    # sub-mapping bundle: 15 keyframes, 2 levels from 0.25 m (workloads.sub_mapping_bundle); single pair: the CPU odometry's VGICP map
    assert sm["max_num_keyframes"] == 15 and sm["keyframe_voxel_resolution"] == 0.25 and sm["keyframe_voxelmap_levels"] == 2 and sm["keyframe_voxelmap_scaling_factor"] == 2.0
    oc = f["config_odometry_cpu"]["odometry_estimation"]
    assert oc["vgicp_resolution"] == 0.5 and oc["vgicp_voxelmap_levels"] == 1 and oc["num_threads"] == 2
    w = workloads.sub_mapping_bundle(None, n_keyframes=3, n_rays=64 * 64, use_gpu=False)
    assert w.resolutions == [sm["keyframe_voxel_resolution"] * sm["keyframe_voxelmap_scaling_factor"] ** l for l in range(sm["keyframe_voxelmap_levels"])]


def test_python_mirror_params_shipped_and_code_defaults():
    from glim_b200 import preprocess

    cfg = fixture()["config_preprocess"]["preprocess"]
    s = preprocess.CloudPreprocessorParams.from_shipped_config()
    assert (s.distance_near_thresh, s.distance_far_thresh, s.use_random_grid_downsampling, s.downsample_resolution, s.downsample_target, s.downsample_rate) == (
        cfg["distance_near_thresh"], cfg["distance_far_thresh"], cfg["use_random_grid_downsampling"], cfg["downsample_resolution"], cfg["random_downsample_target"], cfg["random_downsample_rate"])
    assert (s.enable_outlier_removal, s.outlier_removal_k, s.outlier_std_mul_factor, s.enable_cropbox_filter, s.crop_bbox_frame, s.k_correspondences) == (
        cfg["enable_outlier_removal"], cfg["outlier_removal_k"], cfg["outlier_std_mul_factor"], cfg["enable_cropbox_filter"], cfg["crop_bbox_frame"], cfg["k_correspondences"])
    assert list(s.crop_bbox_min) == cfg["crop_bbox_min"] and list(s.crop_bbox_max) == cfg["crop_bbox_max"]
    # the CODE defaults (cloud_preprocessor.cpp:27-36, :58 -- what tests/test_oracle_vs_reference_tu.py reads back from the reference's
    # own CloudPreprocessorParams constructor through an empty config)
    d = preprocess.CloudPreprocessorParams()
    assert (d.distance_near_thresh, d.distance_far_thresh, d.downsample_resolution, d.downsample_rate, d.outlier_std_mul_factor, d.k_correspondences) == (1.0, 100.0, 0.15, 0.3, 2.0, 8)
