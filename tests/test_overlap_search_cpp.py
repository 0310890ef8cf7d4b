"""glim_b200::find_overlapping_submaps (include/glim_b200/gtsam_points_compat.hpp) compiles as GlobalMapping's two pair loops
would call it: stand-alone, and with -DGLIM_B200_WITH_GTSAM against the GTSAM signature stubs and the Eigen stand-in
(tests/cpp/overlap_search_callsites.cpp).  GTSAM and Eigen are not needed: the check is compile-only."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = os.path.join(ROOT, "include")
CPP = os.path.join(ROOT, "tests", "cpp")
GXX = "/usr/bin/g++"


def test_compat_helper_compiles_standalone(tmp_path):
    subprocess.check_call([GXX, "-std=c++17", "-Wall", "-Wextra", "-Werror", f"-I{INC}", "-c", os.path.join(CPP, "overlap_search_callsites.cpp"), "-o", str(tmp_path / "a.o")])


def test_compat_helper_compiles_in_gtsam_mode_with_eigen_poses(tmp_path):
    subprocess.check_call([GXX, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-DGLIM_B200_WITH_GTSAM=1", f"-I{INC}", f"-I{os.path.join(CPP, 'gtsam_stub')}",
                           f"-I{os.path.join(ROOT, 'oracle', 'ref_shim')}", "-c", os.path.join(CPP, "overlap_search_callsites.cpp"), "-o", str(tmp_path / "b.o")])
