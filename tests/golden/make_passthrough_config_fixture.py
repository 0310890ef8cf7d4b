"""Extracts the shipped parameters of GLIM's passthrough sub-mapping (<GLIM source tree>/config/config_sub_mapping_passthrough.json)
into tests/golden/passthrough_config_values.json; tests/test_passthrough_host.py checks glim_b200.sub_mapping_passthrough's
SubMappingPassthroughParams against it.  The JSON comments are stripped by make_reference_config_fixture.load.
Run: python tests/golden/make_passthrough_config_fixture.py <GLIM source tree>"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_reference_config_fixture as base  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "passthrough_config_values.json")
# every parameter SubMappingPassthroughParams reads (src/glim/mapping/sub_mapping_passthrough.cpp:16-35)
KEYS = ["keyframe_update_interval_rot", "keyframe_update_interval_trans", "max_num_keyframes", "max_num_voxels", "adaptive_max_num_voxels",
        "submap_target_num_points", "submap_voxel_resolution", "min_dist_in_voxel", "max_num_points_in_voxel"]


def extract():
    d = base.load("config_sub_mapping_passthrough")["sub_mapping"]
    return {"config_sub_mapping_passthrough": {"sub_mapping": {k: d[k] for k in KEYS}}}


if __name__ == "__main__":
    base.REF = os.path.join(sys.argv[1], "config")
    with open(OUT, "w") as f:
        json.dump(extract(), f, indent=1, sort_keys=True)
    print("wrote", OUT)
