// api_conformance.cpp -- COMPILE-ONLY: the reference's OWN headers (include/glim/preprocess/cloud_preprocessor.hpp,
// include/glim/common/cloud_covariance_estimation.hpp, include/glim/common/cloud_deskewing.hpp, found on the include path under
// a GLIM source tree and compiled against the Eigen stand-in of oracle/ref_shim/) and the shims of
// include/glim_b200/glim_preprocess_compat.hpp in ONE translation unit.  Every function template below is written once and
// instantiated twice -- with the reference's classes and with the shim's -- so it only compiles if the shim offers the same
// member names, overloads and argument order GLIM's call sites use (odometry_estimation_imu.cpp:313-328, sub_mapping.cpp:365,:376,
// cloud_preprocessor.cpp:77).  A manual check, not run by the test suite (GLIM's headers are not part of this repository):
//   g++ -std=c++17 -fsyntax-only -Ioracle/ref_shim -I<GLIM source tree>/include -Iinclude tests/cpp/api_conformance.cpp
#include <glim/common/cloud_covariance_estimation.hpp>
#include <glim/common/cloud_deskewing.hpp>
#include <glim/preprocess/cloud_preprocessor.hpp>

#include "glim_b200/glim_preprocess_compat.hpp"

namespace ref = ::glim;
namespace shim = ::glim_b200::glim;

template <class Params> void every_parameter(Params& p) {
  p.distance_near_thresh = 0.5; p.distance_far_thresh = 100.0; p.global_shutter = false; p.use_random_grid_downsampling = true;
  p.downsample_resolution = 1.0; p.downsample_target = 10000; p.downsample_rate = 0.1; p.enable_outlier_removal = false;
  p.outlier_removal_k = 10; p.outlier_std_mul_factor = 1.0; p.enable_cropbox_filter = true; p.crop_bbox_frame = std::string("imu");
  p.crop_bbox_min[0] = -1.0; p.crop_bbox_max[2] = 1.0; (void)sizeof(p.T_imu_lidar); p.k_correspondences = 10; p.num_threads = 2;
}

template <class Preprocessor, class Params, class Raw, class Frame> int preprocess_like_glim(const Params& params) {
  Preprocessor preprocessor(params);
  std::shared_ptr<Raw> raw(new Raw);
  raw->stamp = 1.0;
  raw->times.push_back(0.0);
  raw->intensities.push_back(1.0);
  raw->points.push_back(typename decltype(raw->points)::value_type());
  std::shared_ptr<const Raw> craw = raw;
  std::shared_ptr<Frame> f = preprocessor.preprocess(craw);
  const double end = f->scan_end_time - f->stamp;
  return f->size() + f->k_neighbors + (int)f->times.size() + (int)f->points.size() + (int)f->intensities.size() + (int)f->neighbors.size() + (end > 0.0);
}

template <class Estimator, class V4, class M4> std::size_t covariances_like_glim() {
  Estimator by_default, estimator(4);
  std::vector<V4> points(3), normals;
  std::vector<int> neighbors(9, 0);
  std::vector<M4> covs;
  estimator.estimate(points, neighbors, normals, covs);      // odometry_estimation_imu.cpp:322-328
  estimator.estimate(points, neighbors, 2, normals, covs);   // sub_mapping.cpp:376
  std::vector<M4> a = estimator.estimate(points, neighbors, 2), b = by_default.estimate(points, neighbors);
  return a.size() + b.size() + covs.size() + normals.size();
}

template <class Deskewing, class Iso, class V3, class V4> std::size_t deskew_like_glim(const Iso& T_imu_lidar, const V3& vel) {
  Deskewing deskewing;
  std::vector<double> times(2, 0.0), imu_times(2, 0.0);
  std::vector<V4> points(2);
  std::vector<Iso> imu_poses(2, T_imu_lidar);
  std::vector<V4> a = deskewing.deskew(T_imu_lidar, vel, vel, times, points);                       // cloud_deskewing.cpp:11
  std::vector<V4> b = deskewing.deskew(T_imu_lidar, imu_times, imu_poses, 10.0, times, points);      // odometry_estimation_imu.cpp:313, sub_mapping.cpp:365
  return a.size() + b.size();
}

// GLIM's call sites hand Eigen::Isometry3d (and vectors of them) to the gtsam_points functions: the statements of
// odometry_estimation_gpu.cpp:224-231, :247-248, :265, :279, sub_mapping.cpp:253, :486-496 and odometry_estimation_imu.cpp:313 with
// the Eigen stand-in's Isometry3d against the SHIM's functions (compile-only; nothing is called).
double eigen_typed_call_sites(const gtsam_points::GaussianVoxelMap::ConstPtr& voxelmap, const gtsam_points::PointCloud::ConstPtr& frame, CUstream_st* stream) {
  const Eigen::Isometry3d T_world_a = Eigen::Isometry3d::Identity(), T_world_b = Eigen::Isometry3d::Identity();
  std::vector<gtsam_points::GaussianVoxelMap::ConstPtr> keyframes_(2, voxelmap);
  std::vector<Eigen::Isometry3d> delta_from_keyframes(keyframes_.size());
  for (std::size_t i = 0; i < keyframes_.size(); i++) delta_from_keyframes[i] = T_world_a.inverse() * T_world_b;
  double overlap = gtsam_points::overlap_gpu(keyframes_, frame, delta_from_keyframes, stream);
  const Eigen::Isometry3d delta = T_world_a.inverse() * T_world_b;
  overlap += gtsam_points::overlap_gpu(voxelmap, frame, delta, stream);
  overlap += gtsam_points::overlap_gpu(voxelmap, frame, T_world_a.inverse() * T_world_b, stream);
  overlap += gtsam_points::overlap_auto(voxelmap, frame, T_world_a.inverse() * T_world_b);
  std::vector<Eigen::Isometry3d> poses_to_merge(2, T_world_a);
  std::vector<gtsam_points::PointCloud::ConstPtr> keyframes_to_merge(2, frame);
  gtsam_points::PointCloud::Ptr merged = gtsam_points::merge_frames(poses_to_merge, keyframes_to_merge, 0.1, 50000);
  gtsam_points::PointCloudGPU::Ptr merged_gpu = gtsam_points::merge_frames_gpu(poses_to_merge, keyframes_to_merge, 0.1);
  auto factor = std::make_shared<gtsam_points::IntegratedVGICPFactorGPU>(T_world_a, 1, voxelmap, frame, stream, nullptr);  // fixed target pose form (:161)
  shim::CloudDeskewing deskewing;
  const std::vector<double> times(2, 0.0);
  const std::vector<shim::Vector4d> points(2);
  const std::vector<Eigen::Isometry3d> pred_imu_poses(2, T_world_a);
  const std::vector<shim::Vector4d> deskewed = deskewing.deskew(T_world_a, times, pred_imu_poses, 10.0, times, points);
  return overlap + (double)merged->size() + (double)merged_gpu->size() + (double)deskewed.size() + (double)factor->dim();
}

template <class E> int regularization_names() { return (int)E::NONE + (int)E::PLANE + (int)E::NORMALIZED_MIN_EIG + (int)E::FROBENIUS; }

int api_conformance() {
  ref::CloudPreprocessorParams rp;
  shim::CloudPreprocessorParams sp;
  every_parameter(rp);
  every_parameter(sp);
  int s = preprocess_like_glim<ref::CloudPreprocessor, ref::CloudPreprocessorParams, ref::RawPoints, ref::PreprocessedFrame>(rp);
  s += preprocess_like_glim<shim::CloudPreprocessor, shim::CloudPreprocessorParams, shim::RawPoints, shim::PreprocessedFrame>(sp);
  s += (int)covariances_like_glim<ref::CloudCovarianceEstimation, Eigen::Vector4d, Eigen::Matrix4d>();
  s += (int)covariances_like_glim<shim::CloudCovarianceEstimation, shim::Vector4d, shim::Matrix4d>();
  s += (int)deskew_like_glim<ref::CloudDeskewing, Eigen::Isometry3d, Eigen::Vector3d, Eigen::Vector4d>(Eigen::Isometry3d::Identity(), Eigen::Vector3d::Zero());
  s += (int)deskew_like_glim<shim::CloudDeskewing, glim_b200::Pose, shim::Vector3d, shim::Vector4d>(glim_b200::Pose(), shim::Vector3d::Zero());
  s += regularization_names<ref::RegularizationMethod>() - regularization_names<shim::RegularizationMethod>();
  return s;
}
