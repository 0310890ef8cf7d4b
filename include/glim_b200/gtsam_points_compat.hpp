// gtsam_points_compat.hpp -- header-only C++17 shims that give libglim_b200.so the class surface GLIM's modules
// construct from gtsam_points (SURVEY.md 8(b) "inner boundary").  Same names, constructor arguments, defaults
// and call order as the reference call sites; every method forwards to the C-ABI of include/glim_b200.h.
//
//   gtsam_points::CUDAStream / StreamTempBufferRoundRobin     src/glim/odometry/odometry_estimation_gpu.cpp:76-77, :139-141
//   gtsam_points::PointCloud{,CPU,GPU} (points, covs, normals, times, intensities, *_gpu, has_*())
//                                                            src/glim/odometry/odometry_estimation_imu.cpp:322-328; src/glim/mapping/sub_mapping.cpp:165
//   gtsam_points::PointCloudGPU::clone(frame[, stream])      src/glim/odometry/odometry_estimation_gpu.cpp:96; src/glim/mapping/sub_mapping.cpp:168, :393
//   gtsam_points::GaussianVoxelMapGPU(res, 8192*2, 10, 1e-3, stream)::insert(frame)   odometry_estimation_gpu.cpp:103-104; global_mapping.cpp:265 (1 argument)
//   gtsam_points::IntegratedVGICPFactorGPU(key | pose, key, voxelmap, frame, stream, buffer)   odometry_estimation_gpu.cpp:144, :161
//   gtsam_points::NonlinearFactorSetGPU::add / linearize    odometry_estimation_gpu.cpp:383-386
//   gtsam_points::overlap_gpu / overlap_auto                 odometry_estimation_gpu.cpp:231, :248; src/glim/mapping/global_mapping.cpp:448
//   gtsam_points::median_distance                            odometry_estimation_gpu.cpp:91
//   glim_b200::find_overlapping_submaps (the pair loops of)   src/glim/mapping/global_mapping.cpp:285-351, :441-453
//
// Ownership and threading (what a drop-in must get right, and round 1 did not):
//   * PointCloudGPU OWNS its host data.  GLIM replaces the only owner of a frame with its clone
//     (`new_frame->frame = PointCloudGPU::clone(*new_frame->frame)`, odometry_estimation_gpu.cpp:96; sub_mapping.cpp:168;
//     global_mapping.cpp:253) and keeps reading frame->points afterwards (median_distance, deskewing, viewer): clone()
//     deep-copies points / covs / normals / times / intensities, as gtsam_points' own PointCloudGPU (a PointCloudCPU) does.
//   * Work is bound to the stream the CALLER passes.  CUDAStream and StreamTempBufferRoundRobin each own a context (= a
//     gb_ctx = one CUDA stream + scratch arena); the raw `CUstream_st*` they hand to GLIM is looked up again when GLIM passes
//     it back into clone() / GaussianVoxelMapGPU() / IntegratedVGICPFactorGPU() / overlap_gpu().  A call without a stream
//     (clone(frame), GaussianVoxelMapGPU(resolution), overlap_auto) runs on the calling thread's default context.
//   * Frames migrate between GLIM's module threads (odometry -> sub-mapping -> global mapping:
//     async_sub_mapping.cpp:8, async_global_mapping.cpp:24).  A factor may therefore combine a voxel map and a cloud that
//     were uploaded through different contexts, and a factor set may mix such factors: device memory is shared, every
//     upload / build call returns only after its stream has drained, and each gb_ctx serialises its callers with a mutex.
//
// Two build modes:
//   * default: self-contained.  Poses are `Pose` (16 doubles, column-major == Eigen::Isometry3d::data()), keys are
//     uint64_t, `Values` is std::map<Key, Pose>, points / covariances are the layout-compatible PODs Vector4d / Matrix4d
//     below, and linearize() returns the raw gb_linearized6 blocks.  This is what tests/cpp/ compiles and runs here
//     (GTSAM / Eigen are not installed in this environment).
//   * -DGLIM_B200_WITH_GTSAM: Vector4d / Matrix4d ARE Eigen's, IntegratedVGICPFactorGPU derives from
//     gtsam::NonlinearFactor, takes gtsam::Key / gtsam::Pose3 / gtsam::Values and returns gtsam::HessianFactor exactly
//     as the reference factor does (SURVEY A.3).  Compile-checked only against the signature stubs of tests/cpp/gtsam_stub.
#pragma once

#include <array>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <algorithm>
#include <map>
#include <memory>
#include <mutex>
#include <numeric>
#include <random>
#include <functional>
#include <string>
#include <stdexcept>
#include <type_traits>
#include <string>
#include <utility>
#include <vector>

#include "../glim_b200.h"

#ifdef GLIM_B200_WITH_GTSAM
#include <gtsam/geometry/Pose3.h>
#include <gtsam/linear/HessianFactor.h>
#include <gtsam/nonlinear/NonlinearFactor.h>
#include <gtsam/nonlinear/NonlinearFactorGraph.h>
#include <gtsam/nonlinear/Values.h>
#endif

struct CUstream_st;  // the reference passes raw CUDA stream handles around

// SURVEY Appendix E: whether gtsam_points' evaluate() carries a 1/2 in `error` is version dependent; the C-ABI returns
// the raw sum r^T M r and the shim applies this compile-time scale.
#ifndef GLIM_B200_ERROR_SCALE
#define GLIM_B200_ERROR_SCALE 1.0
#endif

namespace glim_b200 {

inline void check(gb_status st, const char* what) {
  if (st != GB_OK) throw std::runtime_error(std::string(what) + ": " + gb_status_string(st) + ": " + gb_last_error());
}

#if defined(GLIM_B200_WITH_GTSAM) && defined(EIGEN_WORLD_VERSION)
using Vector4d = Eigen::Vector4d;
using Matrix4d = Eigen::Matrix4d;
using Vector3f = Eigen::Vector3f;
using Matrix3f = Eigen::Matrix3f;
#else
/// Layout-compatible stand-ins for Eigen::Vector4d (32 B) / Eigen::Matrix4d (128 B, column-major) / Vector3f / Matrix3f
/// (standard_viewer_mem.cpp:34-58), with the accessors GLIM uses on frame->points[i] / frame->covs[i].
struct alignas(16) Vector4d {
  double v[4];
  double& operator[](int i) { return v[i]; }
  double operator[](int i) const { return v[i]; }
  double& operator()(int i) { return v[i]; }
  double operator()(int i) const { return v[i]; }
  double x() const { return v[0]; }
  double y() const { return v[1]; }
  double z() const { return v[2]; }
  double w() const { return v[3]; }
  const double* data() const { return v; }
  double* data() { return v; }
  double norm() const { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3]); }
};
struct alignas(16) Matrix4d {
  double v[16];
  double& operator()(int r, int c) { return v[c * 4 + r]; }
  double operator()(int r, int c) const { return v[c * 4 + r]; }
  const double* data() const { return v; }
  double* data() { return v; }
};
struct Vector3f { float v[3]; };
struct Matrix3f { float v[9]; };
#endif
static_assert(sizeof(Vector4d) == 32 && sizeof(Matrix4d) == 128, "host element layout (standard_viewer_mem.cpp:34-41)");

/// 4x4 rigid transform, 16 doubles column-major (bit-compatible with Eigen::Isometry3d::data()).
struct Pose {
  std::array<double, 16> m{{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}};
  Pose() = default;
  /// From Eigen::Isometry3d (what GLIM's call sites pass: `T_a.inverse() * T_b`, odometry_estimation_gpu.cpp:228, :247, :265;
  /// sub_mapping.cpp:253; global_mapping.cpp:320) or any transform whose .matrix() exposes 16 column-major doubles.
  template <class Iso, class = decltype(static_cast<const double*>(std::declval<const Iso&>().matrix().data()))>
  Pose(const Iso& iso) {
    const auto& M = iso.matrix();
    for (int e = 0; e < 16; e++) m[static_cast<std::size_t>(e)] = M.data()[e];
  }
  const double* data() const { return m.data(); }
  double& operator()(int r, int c) { return m[c * 4 + r]; }
  double operator()(int r, int c) const { return m[c * 4 + r]; }
  Pose inverse() const {
    Pose o;
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) o(r, c) = (*this)(c, r);
      o(r, 3) = -((*this)(0, r) * (*this)(0, 3) + (*this)(1, r) * (*this)(1, 3) + (*this)(2, r) * (*this)(2, 3));
    }
    return o;
  }
  Pose operator*(const Pose& b) const {
    Pose o;
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) {
        double s = 0;
        for (int k = 0; k < 4; k++) s += (*this)(r, k) * b(k, c);
        o(r, c) = s;
      }
    return o;
  }
};

/// A gb_ctx: one CUDA stream + scratch arena + sweep cache.  Thread-safe (the C-ABI serialises callers per context).
class Context {
public:
  explicit Context(int device = 0) {
    check(gb_ctx_create(device, &ctx_), "gb_ctx_create");
    std::lock_guard<std::mutex> lock(registry_mutex());
    registry()[gb_ctx_stream(ctx_)] = ctx_;
  }
  ~Context() {
    {
      std::lock_guard<std::mutex> lock(registry_mutex());
      registry().erase(gb_ctx_stream(ctx_));
    }
    gb_ctx_destroy(ctx_);
  }
  Context(const Context&) = delete;
  Context& operator=(const Context&) = delete;
  gb_ctx* get() const { return ctx_; }
  CUstream_st* stream() const { return static_cast<CUstream_st*>(gb_ctx_stream(ctx_)); }

  /// the calling thread's default context (calls that carry no stream)
  static gb_ctx* default_ctx() {
    static thread_local std::shared_ptr<Context> c = std::make_shared<Context>(0);
    return c->get();
  }
  /// the context that owns `stream` (a handle obtained from CUDAStream / StreamTempBufferRoundRobin), or the calling
  /// thread's default context for a null / foreign stream
  static gb_ctx* of_stream(CUstream_st* stream) {
    if (stream) {
      std::lock_guard<std::mutex> lock(registry_mutex());
      auto it = registry().find(static_cast<void*>(stream));
      if (it != registry().end()) return it->second;
    }
    return default_ctx();
  }

private:
  static std::mutex& registry_mutex() { static std::mutex m; return m; }
  static std::map<void*, gb_ctx*>& registry() { static std::map<void*, gb_ctx*> r; return r; }
  gb_ctx* ctx_ = nullptr;
};

}  // namespace glim_b200

namespace gtsam_points {

using glim_b200::Matrix3f;
using glim_b200::Matrix4d;
using glim_b200::Vector3f;
using glim_b200::Vector4d;

#ifdef GLIM_B200_WITH_GTSAM
using Key = gtsam::Key;
using Values = gtsam::Values;
#else
using Key = std::uint64_t;
using Values = std::map<Key, glim_b200::Pose>;
#endif

/// gtsam_points::CUDAStream: owns a stream (context); converts to the raw handle GLIM passes around (`*stream`).
class CUDAStream {
public:
  CUDAStream() : ctx_(std::make_shared<glim_b200::Context>(0)) {}
  operator CUstream_st*() const { return ctx_->stream(); }
  CUstream_st* get_stream() const { return ctx_->stream(); }
  void sync() const { glim_b200::check(gb_ctx_synchronize(ctx_->get()), "gb_ctx_synchronize"); }

private:
  std::shared_ptr<glim_b200::Context> ctx_;
};

/// gtsam_points::TempBufferManager: scratch is owned by the gb_ctx arena; the handle exists for the signature.
class TempBufferManager {
public:
  TempBufferManager() = default;
};

/// gtsam_points::StreamTempBufferRoundRobin(N): the reference hands out N (stream, buffer) pairs so that N factors
/// can run concurrently.  The fused sweep runs all factors of a graph in ONE launch, so every pair is the module's one
/// stream; N is accepted and ignored.
class StreamTempBufferRoundRobin {
public:
  explicit StreamTempBufferRoundRobin(int /*num_streams*/ = 8) : ctx_(std::make_shared<glim_b200::Context>(0)), buffer_(std::make_shared<TempBufferManager>()) {}
  std::pair<CUstream_st*, std::shared_ptr<TempBufferManager>> get_stream_buffer() { return {ctx_->stream(), buffer_}; }

private:
  std::shared_ptr<glim_b200::Context> ctx_;
  std::shared_ptr<TempBufferManager> buffer_;
};

/// gtsam_points::PointCloud: non-owning view with the members GLIM reads (include/glim/odometry/estimation_frame.hpp:103;
/// standard_viewer_mem.cpp:34-58).
struct PointCloud {
  using Ptr = std::shared_ptr<PointCloud>;
  using ConstPtr = std::shared_ptr<const PointCloud>;
  PointCloud() = default;
  virtual ~PointCloud() = default;
  std::size_t size() const { return num_points; }
  bool has_times() const { return times != nullptr; }
  bool has_points() const { return points != nullptr; }
  bool has_normals() const { return normals != nullptr; }
  bool has_covs() const { return covs != nullptr; }
  bool has_intensities() const { return intensities != nullptr; }
  bool has_times_gpu() const { return times_gpu != nullptr; }
  bool has_points_gpu() const { return points_gpu != nullptr; }
  bool has_normals_gpu() const { return normals_gpu != nullptr; }
  bool has_covs_gpu() const { return covs_gpu != nullptr; }
  bool has_intensities_gpu() const { return intensities_gpu != nullptr; }

  std::size_t num_points = 0;
  double* times = nullptr;
  Vector4d* points = nullptr;
  Vector4d* normals = nullptr;
  Matrix4d* covs = nullptr;
  double* intensities = nullptr;
  // Device side.  Non-null == "this frame has GPU data" (the only way GLIM uses them: sub_mapping.cpp:165,
  // global_mapping.cpp:252, :330, standard_viewer_mem.cpp:49-58).  They point into the gb_cloud's planes
  // ({x y z c00} float4 / {c01 c02 c11 c12} float4 / c22), NOT at dense Vector3f / Matrix3f arrays.
  float* times_gpu = nullptr;
  Vector3f* points_gpu = nullptr;
  Vector3f* normals_gpu = nullptr;
  Matrix3f* covs_gpu = nullptr;
  float* intensities_gpu = nullptr;
};

/// gtsam_points::PointCloudCPU: owns its arrays.
struct PointCloudCPU : public PointCloud {
  using Ptr = std::shared_ptr<PointCloudCPU>;
  using ConstPtr = std::shared_ptr<const PointCloudCPU>;
  PointCloudCPU() = default;
  /// deep copy of whatever attributes `frame` has
  explicit PointCloudCPU(const PointCloud& frame) { copy_host(frame); }
  PointCloudCPU(const PointCloudCPU& other) : PointCloud() { copy_host(other); }
  PointCloudCPU& operator=(const PointCloudCPU&) = delete;

  template <typename T>
  void add_points(const T* pts, std::size_t n) {  // N x 4 doubles (w = 1)
    points_storage.resize(n);
    if (n) std::memcpy(static_cast<void*>(points_storage.data()), pts, sizeof(Vector4d) * n);
    points = points_storage.data();
    num_points = n;
  }
  void add_covs(const double* c, std::size_t n) {  // N x 16 doubles, column-major 4x4
    covs_storage.resize(n);
    if (n) std::memcpy(static_cast<void*>(covs_storage.data()), c, sizeof(Matrix4d) * n);
    covs = covs_storage.data();
  }
  void add_normals(const double* nr, std::size_t n) {
    normals_storage.resize(n);
    if (n) std::memcpy(static_cast<void*>(normals_storage.data()), nr, sizeof(Vector4d) * n);
    normals = normals_storage.data();
  }
  void add_times(const double* t, std::size_t n) { times_storage.assign(t, t + n); times = times_storage.data(); }
  void add_intensities(const double* t, std::size_t n) { intensities_storage.assign(t, t + n); intensities = intensities_storage.data(); }

  std::vector<double> times_storage;
  std::vector<Vector4d> points_storage;
  std::vector<Vector4d> normals_storage;
  std::vector<Matrix4d> covs_storage;
  std::vector<double> intensities_storage;

protected:
  void copy_host(const PointCloud& frame) {
    num_points = frame.num_points;
    if (frame.points) add_points(reinterpret_cast<const double*>(frame.points), frame.num_points);
    if (frame.covs) add_covs(reinterpret_cast<const double*>(frame.covs), frame.num_points);
    if (frame.normals) add_normals(reinterpret_cast<const double*>(frame.normals), frame.num_points);
    if (frame.times) add_times(frame.times, frame.num_points);
    if (frame.intensities) add_intensities(frame.intensities, frame.num_points);
  }
};

/// gtsam_points::PointCloudGPU: a PointCloudCPU (owning deep copy of the host data) + the fp32 device copy.
class PointCloudGPU : public PointCloudCPU {
public:
  using Ptr = std::shared_ptr<PointCloudGPU>;
  using ConstPtr = std::shared_ptr<const PointCloudGPU>;
  ~PointCloudGPU() override { gb_cloud_destroy(cloud_); }
  PointCloudGPU(const PointCloudGPU&) = delete;
  PointCloudGPU& operator=(const PointCloudGPU&) = delete;

  /// clone(frame): odometry_estimation_gpu.cpp:96, global_mapping.cpp:253, :260.  clone(frame, stream): sub_mapping.cpp:168, :393.
  static Ptr clone(const PointCloud& frame, CUstream_st* stream = nullptr) {
    Ptr c(new PointCloudGPU);
    c->copy_host(frame);  // OWNING copy: the caller is about to drop `frame`
    gb_ctx* ctx = glim_b200::Context::of_stream(stream);
    glim_b200::check(gb_cloud_upload(ctx, c->num_points, reinterpret_cast<const double*>(c->points), reinterpret_cast<const double*>(c->covs), reinterpret_cast<const double*>(c->normals), &c->cloud_), "gb_cloud_upload");
    void *p0 = nullptr, *p1 = nullptr, *nr = nullptr;
    glim_b200::check(gb_cloud_device_ptrs(c->cloud_, &p0, &p1, nullptr, &nr), "gb_cloud_device_ptrs");
    c->points_gpu = static_cast<Vector3f*>(p0);
    c->covs_gpu = c->covs ? static_cast<Matrix3f*>(p1) : nullptr;
    c->normals_gpu = static_cast<Vector3f*>(nr);
    return c;
  }
  /// Wrap a device cloud that gb_preprocess / gb_merge_frames already built (takes ownership of `cloud`) together with an
  /// owning copy of the matching host arrays: the frame looks exactly like the result of clone(), without the upload.
  static Ptr adopt(const double* points4, const double* covs16, const double* normals4, const double* times, const double* intensities, std::size_t n, gb_cloud* cloud) {
    Ptr c(new PointCloudGPU);
    c->num_points = n;
    if (points4) c->add_points(points4, n);
    if (covs16) c->add_covs(covs16, n);
    if (normals4) c->add_normals(normals4, n);
    if (times) c->add_times(times, n);
    if (intensities) c->add_intensities(intensities, n);
    c->cloud_ = cloud;
    if (cloud) {
      void *p0 = nullptr, *p1 = nullptr, *nr = nullptr;
      glim_b200::check(gb_cloud_device_ptrs(cloud, &p0, &p1, nullptr, &nr), "gb_cloud_device_ptrs");
      c->points_gpu = static_cast<Vector3f*>(p0);
      c->covs_gpu = covs16 ? static_cast<Matrix3f*>(p1) : nullptr;
      c->normals_gpu = static_cast<Vector3f*>(nr);
    }
    return c;
  }
  gb_cloud* handle() const { return cloud_; }

private:
  PointCloudGPU() = default;
  gb_cloud* cloud_ = nullptr;
};

/// gtsam_points::sample(frame, indices): a PointCloudCPU holding the listed points with every attribute `frame` has.
inline PointCloudCPU::Ptr sample(const PointCloud::ConstPtr& frame, const std::vector<int>& indices) {
  auto out = std::make_shared<PointCloudCPU>();
  const std::size_t m = indices.size();
  out->num_points = m;
  if (frame->points) { out->points_storage.resize(m); for (std::size_t k = 0; k < m; k++) out->points_storage[k] = frame->points[indices[k]]; out->points = out->points_storage.data(); }
  if (frame->covs) { out->covs_storage.resize(m); for (std::size_t k = 0; k < m; k++) out->covs_storage[k] = frame->covs[indices[k]]; out->covs = out->covs_storage.data(); }
  if (frame->normals) { out->normals_storage.resize(m); for (std::size_t k = 0; k < m; k++) out->normals_storage[k] = frame->normals[indices[k]]; out->normals = out->normals_storage.data(); }
  if (frame->times) { out->times_storage.resize(m); for (std::size_t k = 0; k < m; k++) out->times_storage[k] = frame->times[indices[k]]; out->times = out->times_storage.data(); }
  if (frame->intensities) { out->intensities_storage.resize(m); for (std::size_t k = 0; k < m; k++) out->intensities_storage[k] = frame->intensities[indices[k]]; out->intensities = out->intensities_storage.data(); }
  return out;
}

/// gtsam_points::random_sampling(frame, sampling_rate, mt)  (sub_mapping.cpp:385; global_mapping.cpp:248, :734 -- host side,
/// BEFORE the frame is uploaded): sampling_rate * size() points drawn without replacement, in ascending index order
/// (std::sample over the index range [EXT]; the draw depends on the caller's generator exactly as in the reference).
template <typename Rng>
inline PointCloudCPU::Ptr random_sampling(const PointCloud::ConstPtr& frame, double sampling_rate, Rng& mt) {
  const std::size_t n = frame->size();
  if (sampling_rate >= 1.0) return std::make_shared<PointCloudCPU>(*frame);
  const std::size_t m = static_cast<std::size_t>(static_cast<double>(n) * std::max(0.0, sampling_rate));
  std::vector<int> all(n), picked;
  std::iota(all.begin(), all.end(), 0);
  picked.reserve(m);
  std::sample(all.begin(), all.end(), std::back_inserter(picked), m, mt);
  return sample(frame, picked);
}

/// gtsam_points::merge_frames_gpu(poses, frames, downsample_resolution[, target_num_points]) -- the call the reference left
/// commented out at src/glim/mapping/sub_mapping.cpp:491 (its CPU twin merge_frames is what :496 runs).  Frames must be
/// PointCloudGPU; the merged submap comes back as a PointCloudGPU (host points / covariances + device cloud).
inline PointCloudGPU::Ptr merge_frames_gpu(const std::vector<glim_b200::Pose>& poses, const std::vector<PointCloud::ConstPtr>& frames, double downsample_resolution, int target_num_points = 0, CUstream_st* stream = nullptr, std::uint64_t seed = 0) {
  if (poses.size() != frames.size()) throw std::runtime_error("merge_frames_gpu: poses / frames size mismatch");
  std::vector<const gb_cloud*> handles(frames.size());
  std::vector<double> T(16 * frames.size());
  std::size_t cap = 0;
  for (std::size_t i = 0; i < frames.size(); i++) {
    const auto* g = dynamic_cast<const PointCloudGPU*>(frames[i].get());
    if (!g || !g->handle()) throw std::runtime_error("merge_frames_gpu: frames must be PointCloudGPU");
    handles[i] = g->handle();
    std::copy(poses[i].m.begin(), poses[i].m.end(), T.begin() + 16 * i);
    cap += g->size();
  }
  std::vector<Vector4d> pts(cap);
  std::vector<Matrix4d> covs(cap);
  std::size_t m = 0;
  gb_cloud* cloud = nullptr;
  glim_b200::check(gb_merge_frames(glim_b200::Context::of_stream(stream), frames.size(), handles.data(), T.data(), downsample_resolution, target_num_points, seed, reinterpret_cast<double*>(pts.data()),
                                   reinterpret_cast<double*>(covs.data()), &m, &cloud),
                   "gb_merge_frames");
  return PointCloudGPU::adopt(reinterpret_cast<const double*>(pts.data()), reinterpret_cast<const double*>(covs.data()), nullptr, nullptr, nullptr, m, cloud);
}

/// gtsam_points::merge_frames(poses, frames, downsample_resolution, target_num_points)  (sub_mapping.cpp:496, the call that
/// runs today): with GPU keyframes -- what params.enable_gpu produces at sub_mapping.cpp:393 -- it is merge_frames_gpu.
/// There is no CPU path in this library: host-only frames are rejected.
inline PointCloud::Ptr merge_frames(const std::vector<glim_b200::Pose>& poses, const std::vector<PointCloud::ConstPtr>& frames, double downsample_resolution, int target_num_points = 0) {
  for (const auto& f : frames)
    if (!std::dynamic_pointer_cast<const PointCloudGPU>(f)) throw std::runtime_error("merge_frames: frames must be PointCloudGPU (clone them first); libglim_b200 has no CPU path");
  return merge_frames_gpu(poses, frames, downsample_resolution, target_num_points);
}
/// the same with the container GLIM passes: std::vector<Eigen::Isometry3d> poses_to_merge (sub_mapping.cpp:486-496)
template <class Iso, class Alloc, class = std::enable_if_t<!std::is_same<Iso, glim_b200::Pose>::value && std::is_constructible<glim_b200::Pose, const Iso&>::value>>
inline PointCloudGPU::Ptr merge_frames_gpu(const std::vector<Iso, Alloc>& poses, const std::vector<PointCloud::ConstPtr>& frames, double downsample_resolution, int target_num_points = 0, CUstream_st* stream = nullptr, std::uint64_t seed = 0) {
  return merge_frames_gpu(std::vector<glim_b200::Pose>(poses.begin(), poses.end()), frames, downsample_resolution, target_num_points, stream, seed);
}
template <class Iso, class Alloc, class = std::enable_if_t<!std::is_same<Iso, glim_b200::Pose>::value && std::is_constructible<glim_b200::Pose, const Iso&>::value>>
inline PointCloud::Ptr merge_frames(const std::vector<Iso, Alloc>& poses, const std::vector<PointCloud::ConstPtr>& frames, double downsample_resolution, int target_num_points = 0) {
  return merge_frames(std::vector<glim_b200::Pose>(poses.begin(), poses.end()), frames, downsample_resolution, target_num_points);
}

/// gtsam_points::VoxelBucket (standard_viewer_mem.cpp:77 takes its size): one 16-byte open-addressing slot {x, y, z, voxel index}
struct VoxelBucket { int coord[3]; int index; };
static_assert(sizeof(VoxelBucket) == 16, "bucket layout");

/// gtsam_points::cuda_mem_get_info(&free, &total)  (memory_monitor.cpp:39) on the default device
inline void cuda_mem_get_info(std::size_t* free_bytes, std::size_t* total_bytes) { glim_b200::check(gb_mem_info(0, free_bytes, total_bytes), "gb_mem_info"); }
/// gtsam_points::cuda_device_names()  (debug.cpp:84): one entry per visible device (the C-ABI reports the count, not the marketing name)
inline std::vector<std::string> cuda_device_names() {
  std::vector<std::string> names;
  for (int d = 0; d < gb_device_count(); d++) names.push_back("CUDA device " + std::to_string(d) + " (sm_90a)");
  return names;
}

struct VoxelMapInfo {
  int num_voxels = 0;
  int num_buckets = 0;
  int max_bucket_scan_count = 0;
  float voxel_resolution = 0.f;
};

struct GaussianVoxelMap {
  using Ptr = std::shared_ptr<GaussianVoxelMap>;
  using ConstPtr = std::shared_ptr<const GaussianVoxelMap>;
  virtual ~GaussianVoxelMap() = default;
  virtual double voxel_resolution() const = 0;
  virtual void insert(const PointCloud& frame) = 0;
};

/// gtsam_points::GaussianVoxelMapGPU(resolution, init_num_buckets, max_bucket_scan_count, target_points_drop_rate, stream)
class GaussianVoxelMapGPU : public GaussianVoxelMap {
public:
  using Ptr = std::shared_ptr<GaussianVoxelMapGPU>;
  using ConstPtr = std::shared_ptr<const GaussianVoxelMapGPU>;
  explicit GaussianVoxelMapGPU(float resolution, int init_num_buckets = 8192 * 2, int max_bucket_scan_count = 10, double target_points_drop_rate = 1e-3, CUstream_st* stream = nullptr)
  : resolution_(resolution), init_num_buckets_(init_num_buckets), max_bucket_scan_count_(max_bucket_scan_count), target_points_drop_rate_(target_points_drop_rate), stream_(stream) {}
  ~GaussianVoxelMapGPU() override { gb_voxelmap_destroy(map_); }
  GaussianVoxelMapGPU(const GaussianVoxelMapGPU&) = delete;
  GaussianVoxelMapGPU& operator=(const GaussianVoxelMapGPU&) = delete;

  /// insert(frame): `frame` must be (or is uploaded as) a PointCloudGPU; one insert per map, as at every GLIM call site.
  /// Runs on the stream given to the constructor (the caller's module stream), whatever context uploaded the cloud.
  void insert(const PointCloud& frame) override {
    if (map_) throw std::runtime_error("GaussianVoxelMapGPU::insert called twice");
    const auto* gpu = dynamic_cast<const PointCloudGPU*>(&frame);
    PointCloudGPU::Ptr tmp;
    if (!gpu) { tmp = PointCloudGPU::clone(frame, stream_); gpu = tmp.get(); }
    glim_b200::check(gb_voxelmap_build(glim_b200::Context::of_stream(stream_), gpu->handle(), resolution_, init_num_buckets_, max_bucket_scan_count_, target_points_drop_rate_, &map_), "gb_voxelmap_build");
    float r = 0.f;
    gb_voxelmap_info(map_, &voxelmap_info.num_voxels, &voxelmap_info.num_buckets, &r);
    voxelmap_info.voxel_resolution = r;
    voxelmap_info.max_bucket_scan_count = max_bucket_scan_count_;
  }
  double voxel_resolution() const override { return resolution_; }
  gb_voxelmap* handle() const { return map_; }
  VoxelMapInfo voxelmap_info;

private:
  float resolution_;
  int init_num_buckets_, max_bucket_scan_count_;
  double target_points_drop_rate_;
  CUstream_st* stream_;
  gb_voxelmap* map_ = nullptr;
};

/// Result of one linearization in the default (GTSAM-free) build.
struct LinearizedSystem6 {
  gb_linearized6 blocks;  // H_tt H_ss H_ts b_t b_s error num_inliers (column-major 6x6, [rot; trans])
  bool binary;
};

/// gtsam_points::IntegratedVGICPFactorGPU
class IntegratedVGICPFactorGPU
#ifdef GLIM_B200_WITH_GTSAM
: public gtsam::NonlinearFactor
#endif
{
public:
  using shared_ptr = std::shared_ptr<IntegratedVGICPFactorGPU>;

  /// binary: (target_key, source_key, target voxelmap, source frame, stream, buffer)   odometry_estimation_gpu.cpp:144
  IntegratedVGICPFactorGPU(Key target_key, Key source_key, const GaussianVoxelMap::ConstPtr& target, const PointCloud::ConstPtr& source, CUstream_st* stream = nullptr, std::shared_ptr<TempBufferManager> = nullptr)
#ifdef GLIM_B200_WITH_GTSAM
  : gtsam::NonlinearFactor(gtsam::KeyVector{target_key, source_key}),
#else
  :
#endif
    is_binary_(true), target_key_(target_key), source_key_(source_key) {
    init(target, source, stream);
  }
  /// unary: (fixed_target_pose, source_key, ...)   odometry_estimation_gpu.cpp:161
#ifdef GLIM_B200_WITH_GTSAM
  IntegratedVGICPFactorGPU(const gtsam::Pose3& fixed_target_pose, Key source_key, const GaussianVoxelMap::ConstPtr& target, const PointCloud::ConstPtr& source, CUstream_st* stream = nullptr, std::shared_ptr<TempBufferManager> = nullptr)
  : gtsam::NonlinearFactor(gtsam::KeyVector{source_key}), is_binary_(false), target_key_(0), source_key_(source_key) {
    const gtsam::Matrix4 M = fixed_target_pose.matrix();
    for (int c = 0; c < 4; c++) for (int r = 0; r < 4; r++) fixed_target_pose_(r, c) = M(r, c);
    init(target, source, stream);
  }
#else
  IntegratedVGICPFactorGPU(const glim_b200::Pose& fixed_target_pose, Key source_key, const GaussianVoxelMap::ConstPtr& target, const PointCloud::ConstPtr& source, CUstream_st* stream = nullptr, std::shared_ptr<TempBufferManager> = nullptr)
  : is_binary_(false), target_key_(0), source_key_(source_key), fixed_target_pose_(fixed_target_pose) {
    init(target, source, stream);
  }
#endif
  ~IntegratedVGICPFactorGPU() { gb_vgicp_factor_destroy(factor_); }
  IntegratedVGICPFactorGPU(const IntegratedVGICPFactorGPU&) = delete;

  /// set_enable_surface_validation(bool)   odometry_estimation_gpu.cpp:145
  void set_enable_surface_validation(bool enable) {
    if (enable != surface_validation_) {
      surface_validation_ = enable;
      recreate();
    }
  }
  std::size_t dim() const
#ifdef GLIM_B200_WITH_GTSAM
    override
#endif
  { return 6; }
  bool is_binary() const { return is_binary_; }
  Key target_key() const { return target_key_; }
  Key source_key() const { return source_key_; }
  const glim_b200::Pose& get_fixed_target_pose() const { return fixed_target_pose_; }  // standard_viewer_callbacks.cpp:283
  std::size_t memory_usage() const { return sizeof(*this); }                           // standard_viewer_mem.cpp:160
  std::size_t memory_usage_gpu() const { return 122 * sizeof(double) + 64; }           // standard_viewer_mem.cpp:161
  double inlier_fraction() const { return source_->size() ? last_num_inliers_ / static_cast<double>(source_->size()) : 0.0; }
  int num_inliers() const { return static_cast<int>(last_num_inliers_); }
  gb_factor* handle() const { return factor_; }
  gb_ctx* context() const { return ctx_; }

  /// delta = T_target^-1 * T_source (SURVEY A.1)
  glim_b200::Pose delta(const Values& values) const {
    const glim_b200::Pose Ts = pose_of(values, source_key_);
    const glim_b200::Pose Tt = is_binary_ ? pose_of(values, target_key_) : fixed_target_pose_;
    return Tt.inverse() * Ts;
  }

  /// raw linearization (GTSAM-free); the batched path stores its result through set_cached()
  LinearizedSystem6 linearize_raw(const Values& values) {
    const glim_b200::Pose d = delta(values);
    LinearizedSystem6 out;
    out.binary = is_binary_;
    glim_b200::check(gb_vgicp_linearize(factor_, d.data(), &out.blocks), "gb_vgicp_linearize");
    lin_point_ = d;
    have_lin_point_ = true;
    last_num_inliers_ = out.blocks.num_inliers;
    return out;
  }
  /// error(values): inlier set of the last linearization point, evaluated at `values` (SURVEY A.2 / A.5)
  double error(const Values& values) const
#ifdef GLIM_B200_WITH_GTSAM
    override
#endif
  {
    const glim_b200::Pose d = delta(values);
    double e = 0.0;
    glim_b200::check(gb_vgicp_error(factor_, have_lin_point_ ? lin_point_.data() : d.data(), d.data(), &e), "gb_vgicp_error");
    return GLIM_B200_ERROR_SCALE * e;
  }

#ifdef GLIM_B200_WITH_GTSAM
  /// linearize(values) -> gtsam::HessianFactor (SURVEY A.3); uses the cached batch result when NonlinearFactorSetGPU ran
  std::shared_ptr<gtsam::GaussianFactor> linearize(const gtsam::Values& values) const override {
    auto* self = const_cast<IntegratedVGICPFactorGPU*>(this);
    gb_linearized6 L;
    if (self->cached_valid_) { L = self->cached_; self->cached_valid_ = false; } else { L = self->linearize_raw(values).blocks; }
    gtsam::Matrix6 H_tt, H_ss, H_ts;
    gtsam::Vector6 g_t, g_s;
    // exactly the reference's hand-off (SURVEY A.3): gb_hessian_blocks negates the gradients and scales the constant term
    gb_hessian_blocks(&L, GLIM_B200_ERROR_SCALE, &H_tt(0, 0), &H_ts(0, 0), &g_t(0), &H_ss(0, 0), &g_s(0), &L.error);
    if (is_binary_) return std::make_shared<gtsam::HessianFactor>(target_key_, source_key_, H_tt, H_ts, g_t, H_ss, g_s, L.error);
    return std::make_shared<gtsam::HessianFactor>(source_key_, H_ss, g_s, L.error);
  }
  gtsam::NonlinearFactor::shared_ptr clone() const override {
    std::shared_ptr<IntegratedVGICPFactorGPU> f;
    if (is_binary_) {
      f = std::make_shared<IntegratedVGICPFactorGPU>(target_key_, source_key_, target_, source_, stream_);
    } else {
      gtsam::Matrix4 M;
      for (int c = 0; c < 4; c++) for (int r = 0; r < 4; r++) M(r, c) = fixed_target_pose_(r, c);
      f = std::make_shared<IntegratedVGICPFactorGPU>(gtsam::Pose3(M), source_key_, target_, source_, stream_);
    }
    f->set_enable_surface_validation(surface_validation_);
    return f;
  }
#endif

  // used by NonlinearFactorSetGPU
  void set_cached(const gb_linearized6& L, const glim_b200::Pose& lin_point) {
    cached_ = L; cached_valid_ = true; lin_point_ = lin_point; have_lin_point_ = true; last_num_inliers_ = L.num_inliers;
  }
  bool take_cached(gb_linearized6* out) { if (!cached_valid_) return false; *out = cached_; cached_valid_ = false; return true; }

private:
  static glim_b200::Pose pose_of(const Values& values, Key k) {
#ifdef GLIM_B200_WITH_GTSAM
    const gtsam::Matrix4 M = values.at<gtsam::Pose3>(k).matrix();
    glim_b200::Pose p;
    for (int c = 0; c < 4; c++) for (int r = 0; r < 4; r++) p(r, c) = M(r, c);
    return p;
#else
    return values.at(k);
#endif
  }
  void init(const GaussianVoxelMap::ConstPtr& target, const PointCloud::ConstPtr& source, CUstream_st* stream) {
    target_ = std::dynamic_pointer_cast<const GaussianVoxelMapGPU>(target);
    source_ = std::dynamic_pointer_cast<const PointCloudGPU>(source);
    if (!target_ || !target_->handle()) throw std::runtime_error("IntegratedVGICPFactorGPU: target is not a (built) GaussianVoxelMapGPU");
    if (!source_ || !source_->handle()) throw std::runtime_error("IntegratedVGICPFactorGPU: source has no GPU points (PointCloudGPU::clone it first)");
    stream_ = stream;
    ctx_ = glim_b200::Context::of_stream(stream);  // the CALLER's stream: the module that builds the graph also linearizes it
    recreate();
  }
  void recreate() {
    if (factor_) gb_vgicp_factor_destroy(factor_);
    factor_ = nullptr;
    glim_b200::check(gb_vgicp_factor_create(ctx_, target_->handle(), source_->handle(), surface_validation_ ? GB_FACTOR_SURFACE_VALIDATION : 0, &factor_), "gb_vgicp_factor_create");
  }

  bool is_binary_;
  Key target_key_, source_key_;
  glim_b200::Pose fixed_target_pose_;
  GaussianVoxelMapGPU::ConstPtr target_;  // kept alive, as the reference factor keeps shared_ptrs
  PointCloudGPU::ConstPtr source_;
  CUstream_st* stream_ = nullptr;
  gb_ctx* ctx_ = nullptr;
  gb_factor* factor_ = nullptr;
  bool surface_validation_ = false;
  glim_b200::Pose lin_point_;
  bool have_lin_point_ = false;
  double last_num_inliers_ = 0.0;
  gb_linearized6 cached_{};
  bool cached_valid_ = false;
};

/// gtsam_points::NonlinearFactorSetGPU: add(graph) collects the GPU factors; linearize(values) runs ONE fused sweep
/// (F x 128 B of poses down, F records up) and caches every factor's result for the GTSAM linearize() that follows
/// (odometry_estimation_gpu.cpp:383-386).  The sweep runs on the context of the first factor, i.e. on the stream the
/// module passed when it built its factors; the factors may reference clouds / maps uploaded through other contexts.
class NonlinearFactorSetGPU {
public:
  void clear() { factors_.clear(); }
  std::size_t size() const { return factors_.size(); }
  bool add(const std::shared_ptr<IntegratedVGICPFactorGPU>& f) {
    if (!f) return false;
    factors_.push_back(f);
    return true;
  }
#ifdef GLIM_B200_WITH_GTSAM
  void add(const gtsam::NonlinearFactorGraph& graph) {
    for (const auto& f : graph) add(std::dynamic_pointer_cast<IntegratedVGICPFactorGPU>(f));
  }
#else
  template <typename Container>
  void add(const Container& graph) {
    for (const auto& f : graph) add(f);
  }
#endif
  void linearize(const Values& values) {
    const std::size_t F = factors_.size();
    if (!F) return;
    std::vector<gb_factor*> handles(F);
    std::vector<glim_b200::Pose> deltas(F);
    std::vector<double> T(16 * F);
    for (std::size_t i = 0; i < F; i++) {
      handles[i] = factors_[i]->handle();
      deltas[i] = factors_[i]->delta(values);
      std::copy(deltas[i].m.begin(), deltas[i].m.end(), T.begin() + 16 * i);
    }
    results_.resize(F);
    glim_b200::check(gb_factor_set_linearize(factors_[0]->context(), F, handles.data(), T.data(), results_.data()), "gb_factor_set_linearize");
    for (std::size_t i = 0; i < F; i++) factors_[i]->set_cached(results_[i], deltas[i]);
  }
  const std::vector<gb_linearized6>& results() const { return results_; }

private:
  std::vector<std::shared_ptr<IntegratedVGICPFactorGPU>> factors_;
  std::vector<gb_linearized6> results_;
};

/// gtsam_points::create_nonlinear_factor_set_gpu() and LinearizationHook::register_hook(...)  (offline_viewer.cpp:29): the
/// optimizers of the reference ask the registered hooks for a factor set to batch-linearize the GPU factors of a graph; the
/// optimizers themselves are out of scope, the registry is here so that the call site compiles and the hook is retrievable.
inline std::shared_ptr<NonlinearFactorSetGPU> create_nonlinear_factor_set_gpu() { return std::make_shared<NonlinearFactorSetGPU>(); }
struct LinearizationHook {
  using Hook = std::function<std::shared_ptr<NonlinearFactorSetGPU>()>;
  static void register_hook(const Hook& hook) { std::lock_guard<std::mutex> lock(mutex()); hooks().push_back(hook); }
  static std::vector<std::shared_ptr<NonlinearFactorSetGPU>> create_factor_sets() {
    std::lock_guard<std::mutex> lock(mutex());
    std::vector<std::shared_ptr<NonlinearFactorSetGPU>> sets;
    for (const auto& h : hooks()) sets.push_back(h());
    return sets;
  }
private:
  static std::vector<Hook>& hooks() { static std::vector<Hook> h; return h; }
  static std::mutex& mutex() { static std::mutex m; return m; }
};

/// gtsam_points::overlap_gpu(voxelmap, source, delta, stream)   odometry_estimation_gpu.cpp:248
inline double overlap_gpu(const GaussianVoxelMap::ConstPtr& target, const PointCloud::ConstPtr& source, const glim_b200::Pose& delta, CUstream_st* stream = nullptr) {
  const auto t = std::dynamic_pointer_cast<const GaussianVoxelMapGPU>(target);
  const auto s = std::dynamic_pointer_cast<const PointCloudGPU>(source);
  if (!t || !s) throw std::runtime_error("overlap_gpu: GPU voxel map / GPU point cloud required");
  const gb_voxelmap* maps[1] = {t->handle()};
  double ov = 0.0;
  glim_b200::check(gb_overlap(glim_b200::Context::of_stream(stream), 1, maps, s->handle(), delta.data(), &ov), "gb_overlap");
  return ov;
}
/// gtsam_points::overlap_gpu(voxelmaps, source, deltas, stream)   odometry_estimation_gpu.cpp:231
inline double overlap_gpu(const std::vector<GaussianVoxelMap::ConstPtr>& targets, const PointCloud::ConstPtr& source, const std::vector<glim_b200::Pose>& deltas, CUstream_st* stream = nullptr) {
  const auto s = std::dynamic_pointer_cast<const PointCloudGPU>(source);
  if (!s || targets.size() != deltas.size()) throw std::runtime_error("overlap_gpu: bad arguments");
  std::vector<const gb_voxelmap*> maps(targets.size());
  std::vector<double> T(16 * targets.size());
  for (std::size_t i = 0; i < targets.size(); i++) {
    const auto t = std::dynamic_pointer_cast<const GaussianVoxelMapGPU>(targets[i]);
    if (!t) throw std::runtime_error("overlap_gpu: GPU voxel map required");
    maps[i] = t->handle();
    std::copy(deltas[i].m.begin(), deltas[i].m.end(), T.begin() + 16 * i);
  }
  double ov = 0.0;
  glim_b200::check(gb_overlap(glim_b200::Context::of_stream(stream), maps.size(), maps.data(), s->handle(), T.data(), &ov), "gb_overlap");
  return ov;
}
/// the same with the container GLIM passes: std::vector<Eigen::Isometry3d> (odometry_estimation_gpu.cpp:225-231, :279)
template <class Iso, class Alloc, class = std::enable_if_t<!std::is_same<Iso, glim_b200::Pose>::value && std::is_constructible<glim_b200::Pose, const Iso&>::value>>
inline double overlap_gpu(const std::vector<GaussianVoxelMap::ConstPtr>& targets, const PointCloud::ConstPtr& source, const std::vector<Iso, Alloc>& deltas, CUstream_st* stream = nullptr) {
  return overlap_gpu(targets, source, std::vector<glim_b200::Pose>(deltas.begin(), deltas.end()), stream);
}
/// gtsam_points::overlap_auto: GPU voxel maps dispatch to overlap_gpu (sub_mapping.cpp:252; global_mapping.cpp:322, :448)
inline double overlap_auto(const GaussianVoxelMap::ConstPtr& target, const PointCloud::ConstPtr& source, const glim_b200::Pose& delta) { return overlap_gpu(target, source, delta); }

/// gtsam_points::median_distance(frame, max_scan_count)   odometry_estimation_gpu.cpp:91  (256 strided samples: host)
inline double median_distance(const PointCloud::ConstPtr& frame, int max_scan_count) {
  const std::size_t n = frame->size();
  if (!n) return 0.0;
  const std::size_t step = std::max<std::size_t>(1, n / static_cast<std::size_t>(max_scan_count));
  std::vector<double> d;
  for (std::size_t i = 0; i < n; i += step) {
    const double* p = reinterpret_cast<const double*>(&frame->points[i]);
    d.push_back(std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]));
  }
  std::nth_element(d.begin(), d.begin() + d.size() / 2, d.end());
  return d[d.size() / 2];
}

}  // namespace gtsam_points

namespace glim_b200 {

/// The (i, j) key of an entry of the caller's set of existing factors: a std::pair, or anything indexable such as the
/// Eigen::Vector3i of GlobalMapping::find_overlapping_submaps (global_mapping.cpp:290).
template <class A, class B> inline std::array<int32_t, 2> existing_key(const std::pair<A, B>& e) { return {{static_cast<int32_t>(e.first), static_cast<int32_t>(e.second)}}; }
template <class V> inline std::array<int32_t, 2> existing_key(const V& e) { return {{static_cast<int32_t>(e[0]), static_cast<int32_t>(e[1])}}; }

/// The pair loops of GlobalMapping::find_overlapping_submaps (global_mapping.cpp:308-351: first_source 0) and
/// create_matching_cost_factors (:441-453: first_source = current, min_overlap 0 to read previous_overlap as well) as one
/// gb_find_overlapping_submaps call.  maps[k] = submaps[k]->voxelmaps.back(), sources[k] = subsampled_submaps[k] (or the
/// current submap's frame), T_world_submap[k] = submaps[k]->T_world_origin (glim_b200::Pose or Eigen::Isometry3d); `existing`
/// holds the (i, j) pairs that already have a factor.  Returns (i, j, overlap) for every candidate with overlap >= min_overlap
/// in lexicographic (i, j) order, the order of both loops.
template <class PoseT, class Alloc, class Existing>
inline std::vector<std::tuple<int, int, double>> find_overlapping_submaps(const std::vector<gtsam_points::GaussianVoxelMap::ConstPtr>& maps,
                                                                          const std::vector<gtsam_points::PointCloud::ConstPtr>& sources,
                                                                          const std::vector<PoseT, Alloc>& T_world_submap, const Existing& existing,
                                                                          double max_distance, double min_overlap, std::size_t first_source = 0,
                                                                          CUstream_st* stream = nullptr) {
  const std::size_t S = maps.size();
  if (sources.size() != S || T_world_submap.size() != S) throw std::runtime_error("find_overlapping_submaps: maps, sources and poses differ in size");
  std::vector<const gb_voxelmap*> m(S);
  std::vector<const gb_cloud*> c(S);
  std::vector<double> T(16 * S);
  for (std::size_t k = 0; k < S; k++) {
    const auto t = std::dynamic_pointer_cast<const gtsam_points::GaussianVoxelMapGPU>(maps[k]);
    const auto s = std::dynamic_pointer_cast<const gtsam_points::PointCloudGPU>(sources[k]);
    if (!t || !s) throw std::runtime_error("find_overlapping_submaps: GPU voxel maps / GPU point clouds required");
    m[k] = t->handle();
    c[k] = s->handle();
    const Pose P(T_world_submap[k]);
    std::copy(P.m.begin(), P.m.end(), T.begin() + 16 * k);
  }
  std::vector<int32_t> ex;
  for (const auto& e : existing) {
    const auto key = existing_key(e);
    ex.insert(ex.end(), key.begin(), key.end());
  }
  gb_ctx* ctx = Context::of_stream(stream);
  std::size_t found = 0, capacity = std::min<std::size_t>(S * (S > 0 ? S - 1 : 0) / 2, 1 << 18);  // a first guess; a second call only when more are found
  std::vector<int32_t> pairs;
  std::vector<double> overlaps;
  for (int attempt = 0; attempt < 2; attempt++) {
    pairs.resize(2 * capacity);
    overlaps.resize(capacity);
    check(gb_find_overlapping_submaps(ctx, S, m.data(), c.data(), T.data(), first_source, ex.size() / 2, ex.empty() ? nullptr : ex.data(), max_distance, min_overlap,
                                      capacity, &found, capacity ? pairs.data() : nullptr, capacity ? overlaps.data() : nullptr),
          "gb_find_overlapping_submaps");
    if (found <= capacity) break;
    capacity = found;
  }
  std::vector<std::tuple<int, int, double>> out(found);
  for (std::size_t r = 0; r < found; r++) out[r] = std::make_tuple(pairs[2 * r], pairs[2 * r + 1], overlaps[r]);
  return out;
}

}  // namespace glim_b200
