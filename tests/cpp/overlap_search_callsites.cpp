// overlap_search_callsites.cpp -- COMPILE-ONLY check of glim_b200::find_overlapping_submaps (gtsam_points_compat.hpp) as
// GlobalMapping's two pair loops would call it (src/glim/mapping/global_mapping.cpp:285-351, :430-481): the existing-factor set
// as GLIM keeps it, poses as glim_b200::Pose or, with Eigen, Eigen::Isometry3d.  Built stand-alone, and with
// -DGLIM_B200_WITH_GTSAM against the signature stubs of tests/cpp/gtsam_stub and the Eigen stand-in of oracle/ref_shim.
#ifdef GLIM_B200_WITH_GTSAM
#include <Eigen/Core>
#include <Eigen/Geometry>
#endif
#include "glim_b200/gtsam_points_compat.hpp"

#include <array>
#include <set>
#include <utility>

struct SubMap {  // the members of glim::SubMap the loops touch
  std::vector<gtsam_points::GaussianVoxelMap::Ptr> voxelmaps;
  glim_b200::Pose T_world_origin;
#ifdef GLIM_B200_WITH_GTSAM
  Eigen::Isometry3d T_world_origin_eigen;
#endif
};

double callsites(const std::vector<std::shared_ptr<SubMap>>& submaps, const std::vector<gtsam_points::PointCloud::ConstPtr>& subsampled_submaps,
                 const std::set<std::pair<int, int>>& existing_factors, double max_implicit_loop_distance, double min_overlap) {
  std::vector<gtsam_points::GaussianVoxelMap::ConstPtr> maps;
  std::vector<glim_b200::Pose> poses;
  for (const auto& s : submaps) {
    maps.push_back(s->voxelmaps.back());
    poses.push_back(s->T_world_origin);
  }
  double sum = 0.0;
  // ---- find_overlapping_submaps (:308-351): every pair without a factor
  for (const auto& [i, j, overlap] : glim_b200::find_overlapping_submaps(maps, subsampled_submaps, poses, existing_factors, max_implicit_loop_distance, min_overlap)) {
    sum += i + j + overlap;
  }
  // ---- create_matching_cost_factors (:441-481): the current submap against every earlier one; min_overlap 0 also returns the
  //      previous submap's overlap for the isolation check
  const std::size_t current = submaps.size() - 1;
  double previous_overlap = 0.0;
  for (const auto& [i, j, overlap] : glim_b200::find_overlapping_submaps(maps, subsampled_submaps, poses, std::vector<std::pair<int, int>>(), max_implicit_loop_distance, 0.0, current)) {
    if (static_cast<std::size_t>(i) == current - 1) previous_overlap = overlap;
    if (overlap >= min_overlap) sum += j;
  }
#ifdef GLIM_B200_WITH_GTSAM
  std::vector<Eigen::Isometry3d> iso;
  for (const auto& s : submaps) iso.push_back(s->T_world_origin_eigen);
  sum += glim_b200::find_overlapping_submaps(maps, subsampled_submaps, iso, existing_factors, max_implicit_loop_distance, min_overlap).size();
#endif
  // an indexable key type, as GLIM's Eigen::Vector3i (i, j, 0)
  const std::vector<std::array<int, 3>> ex3 = {{{0, 1, 0}}};
  sum += glim_b200::find_overlapping_submaps(maps, subsampled_submaps, poses, ex3, max_implicit_loop_distance, min_overlap).size();
  return sum + previous_overlap;
}
