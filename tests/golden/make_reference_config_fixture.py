"""Extracts the shipped parameter values the hot path's call sites are constructed with from the reference's own config files
(<GLIM source tree>/config/*.json, JSON with // comments) into tests/golden/reference_config_values.json;
tests/test_reference_config_values.py checks the product's defaults against it.
Run: python tests/golden/make_reference_config_fixture.py <GLIM source tree>"""
import json
import os
import re
import sys

REF = None  # <GLIM source tree>/config, from the command line
FILES = ["config_preprocess", "config_odometry_gpu", "config_odometry_cpu", "config_sub_mapping_gpu", "config_global_mapping_gpu"]
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_config_values.json")


def load(name):
    s = open(os.path.join(REF, name + ".json")).read()
    s = re.sub(r"/\*.*?\*/", "", s, flags=re.S)
    s = re.sub(r"//[^\n]*", "", s)
    return json.loads(s)


# only the parameters the hot path's call sites are constructed with (the rest of the files configures GLIM's optimizers, IMU
# handling, logging ... -- out of scope)
KEYS = {
    "config_preprocess": ("preprocess", ["distance_near_thresh", "distance_far_thresh", "use_random_grid_downsampling", "downsample_resolution", "random_downsample_target", "random_downsample_rate",
                                         "enable_outlier_removal", "outlier_removal_k", "outlier_std_mul_factor", "enable_cropbox_filter", "crop_bbox_frame", "crop_bbox_min", "crop_bbox_max", "k_correspondences"]),
    "config_odometry_gpu": ("odometry_estimation", ["voxel_resolution", "voxel_resolution_max", "voxel_resolution_dmin", "voxel_resolution_dmax", "voxelmap_levels", "voxelmap_scaling_factor",
                                                    "full_connection_window_size", "keyframe_update_strategy", "max_num_keyframes", "keyframe_min_overlap", "keyframe_max_overlap", "smoother_lag"]),
    "config_odometry_cpu": ("odometry_estimation", ["registration_type", "vgicp_resolution", "vgicp_voxelmap_levels", "vgicp_voxelmap_scaling_factor", "num_threads"]),
    "config_sub_mapping_gpu": ("sub_mapping", ["max_num_keyframes", "registration_error_factor_type", "keyframe_voxel_resolution", "keyframe_voxelmap_levels", "keyframe_voxelmap_scaling_factor",
                                               "submap_downsample_resolution", "submap_voxel_resolution", "submap_target_num_points"]),
    "config_global_mapping_gpu": ("global_mapping", ["registration_error_factor_type", "submap_voxel_resolution", "submap_voxel_resolution_max", "submap_voxelmap_levels", "submap_voxelmap_scaling_factor",
                                                     "max_implicit_loop_distance", "min_implicit_loop_overlap"]),
}


def extract():
    out = {}
    for n in FILES:
        section, keys = KEYS[n]
        d = load(n)[section]
        out[n] = {section: {k: d[k] for k in keys}}
    return out


if __name__ == "__main__":
    REF = os.path.join(sys.argv[1], "config")
    with open(OUT, "w") as f:
        json.dump(extract(), f, indent=1, sort_keys=True)
    print("wrote", OUT)
