// gb_deskew.cu -- CloudDeskewing::deskew on the GPU (SURVEY 8(f) row 2: the per-point transform that sits between the
// preprocess and the covariance estimation of every frame, src/glim/odometry/odometry_estimation_imu.cpp:313-316).
//
// Replaces glim::CloudDeskewing::deskew (src/glim/common/cloud_deskewing.cpp:11-55 constant velocity, :57-133 predicted IMU
// poses).  The reference quantises the per-point times into a <= ~1000-entry table (0.1 ms) and builds one pose per entry on
// the host (gtsam::Pose3::Expmap, quaternion slerp); that part is a few hundred 4x4 products and stays on the host here too
// (gb_deskew_pose_table, also exported so it can be checked without a GPU).  The O(N) part -- one table lookup and one or two
// 4x4 * 4-vector products per point, fp64 -- is the kernel.  Oracle: go_deskew_const_vel / go_deskew_imu.
//
// The host table is verified on the CPU against the oracle, the kernel on the GPU (tests/test_deskew.py).
#include "gb_internal.cuh"

#include <math.h>
#include <string.h>

#include <vector>

namespace {

struct M4 { double m[16]; };  // column-major

inline M4 identity() { M4 r; memset(r.m, 0, sizeof(r.m)); r.m[0] = r.m[5] = r.m[10] = r.m[15] = 1.0; return r; }
inline M4 mul(const M4& a, const M4& b) {
  M4 r;
  for (int c = 0; c < 4; c++)
    for (int row = 0; row < 4; row++) {
      double s = 0.0;
      for (int k = 0; k < 4; k++) s += a.m[k * 4 + row] * b.m[c * 4 + k];
      r.m[c * 4 + row] = s;
    }
  return r;
}
inline M4 rigid_inverse(const M4& t) {
  M4 r = identity();
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) r.m[j * 4 + i] = t.m[i * 4 + j];
  for (int i = 0; i < 3; i++) r.m[12 + i] = -(t.m[i * 4 + 0] * t.m[12] + t.m[i * 4 + 1] * t.m[13] + t.m[i * 4 + 2] * t.m[14]);
  return r;
}
// gtsam::Pose3::Expmap([w; v])
M4 pose3_expmap(const double w[3], const double v[3]) {
  const double eps = 2.220446049250313e-16;
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  const double W[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
  double WW[9], R[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) WW[i * 3 + j] = W[i * 3] * W[j] + W[i * 3 + 1] * W[3 + j] + W[i * 3 + 2] * W[6 + j];
  double a = 1.0, b = 0.5;
  if (th2 > eps) { const double th = sqrt(th2); a = sin(th) / th; b = (1.0 - cos(th)) / th2; }
  for (int k = 0; k < 9; k++) R[k] = (k % 4 == 0 ? 1.0 : 0.0) + a * W[k] + b * WW[k];
  double t[3] = {v[0], v[1], v[2]};
  if (th2 > eps) {
    const double wv = w[0] * v[0] + w[1] * v[1] + w[2] * v[2];
    const double x[3] = {w[1] * v[2] - w[2] * v[1], w[2] * v[0] - w[0] * v[2], w[0] * v[1] - w[1] * v[0]};
    for (int i = 0; i < 3; i++) t[i] = (x[i] - (R[i * 3] * x[0] + R[i * 3 + 1] * x[1] + R[i * 3 + 2] * x[2]) + w[i] * wv) / th2;
  }
  M4 T = identity();
  for (int i = 0; i < 3; i++) { for (int j = 0; j < 3; j++) T.m[j * 4 + i] = R[i * 3 + j]; T.m[12 + i] = t[i]; }
  return T;
}
// Eigen::Quaterniond(Matrix3d) -> (x, y, z, w)
void quat_from_rotation(const M4& T, double q[4]) {
  auto m = [&](int r, int c) { return T.m[c * 4 + r]; };
  double t = m(0, 0) + m(1, 1) + m(2, 2);
  if (t > 0.0) {
    t = sqrt(t + 1.0);
    q[3] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m(2, 1) - m(1, 2)) * t; q[1] = (m(0, 2) - m(2, 0)) * t; q[2] = (m(1, 0) - m(0, 1)) * t;
  } else {
    int i = 0;
    if (m(1, 1) > m(0, 0)) i = 1;
    if (m(2, 2) > m(i, i)) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0);
    q[i] = 0.5 * t;
    t = 0.5 / t;
    q[3] = (m(k, j) - m(j, k)) * t; q[j] = (m(j, i) + m(i, j)) * t; q[k] = (m(k, i) + m(i, k)) * t;
  }
}
// Eigen slerp + toRotationMatrix into the rotation block of T
void slerp_to_rotation(const double a[4], const double b[4], double p, M4& T) {
  const double d = a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3];
  const double ad = fabs(d);
  double s0 = 1.0 - p, s1 = p;
  if (ad < 1.0 - 2.220446049250313e-16) {
    const double th = acos(ad), st = sin(th);
    s0 = sin((1.0 - p) * th) / st;
    s1 = sin(p * th) / st;
  }
  if (d < 0.0) s1 = -s1;
  const double x = s0 * a[0] + s1 * b[0], y = s0 * a[1] + s1 * b[1], z = s0 * a[2] + s1 * b[2], w = s0 * a[3] + s1 * b[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  T.m[0] = 1 - (tyy + tzz); T.m[4] = txy - twz; T.m[8] = txz + twy;
  T.m[1] = txy + twz; T.m[5] = 1 - (txx + tzz); T.m[9] = tyz - twx;
  T.m[2] = txz - twy; T.m[6] = tyz + twx; T.m[10] = 1 - (txx + tyy);
}

// out = T_post * (T[idx] * p), each product evaluated as Eigen does (linear combination of the columns, left to right), with
// explicit un-contracted fp64 operations so that the result is bit-identical to the host arithmetic of the reference / oracle
__device__ __forceinline__ double4 xform(const double* __restrict__ T, const double4 p) {
  double o[4];
#pragma unroll
  for (int r = 0; r < 4; r++)
    o[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[r], p.x), __dmul_rn(T[4 + r], p.y)), __dmul_rn(T[8 + r], p.z)), __dmul_rn(T[12 + r], p.w));
  return make_double4(o[0], o[1], o[2], o[3]);
}
__global__ void __launch_bounds__(256) k_deskew(int n, const double4* __restrict__ pts, const int* __restrict__ idx, const double* __restrict__ table, const double* __restrict__ T_post, double4* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double4 d = xform(table + 16 * (size_t)idx[i], pts[i]);
  if (T_post) d = xform(T_post, d);
  out[i] = d;
}

}  // namespace

// time table (cloud_deskewing.cpp:25-35 / :75-82) + one pose per entry; HOST ONLY (no device needed)
extern "C" gb_status gb_deskew_pose_table(const double T_imu_lidar[16], const double* linear_vel, const double* angular_vel, size_t n_imu, const double* imu_times,
                                          const double* imu_poses, double stamp, size_t n, const double* times, int32_t* time_indices, double* table_poses, size_t* table_size) {
  GB_REQUIRE(T_imu_lidar && table_size, "null argument");
  *table_size = 0;
  if (n == 0) return GB_OK;  // :16-18 / :65-67
  GB_REQUIRE(times && time_indices && table_poses, "null argument");
  std::vector<double> tab;
  const double time_eps = 1e-4;
  for (size_t i = 0; i < n; i++) {
    if (tab.empty() || times[i] - tab.back() > time_eps) tab.push_back(times[i]);
    time_indices[i] = (int32_t)tab.size() - 1;
  }
  M4 Til;
  memcpy(Til.m, T_imu_lidar, sizeof(Til.m));
  const M4 Tli = rigid_inverse(Til);
  const bool use_imu = n_imu > 0 && imu_times && imu_poses;  // :69-71: no IMU poses -> zero-velocity model
  size_t cursor = 0;
  M4 T_imu0_world = identity();
  for (size_t i = 0; i < tab.size(); i++) {
    M4 T_l0_l1;
    if (!use_imu) {
      const double dt = tab[i];
      double w[3] = {0, 0, 0}, v[3] = {0, 0, 0};
      if (n_imu == 0) for (int k = 0; k < 3; k++) { if (angular_vel) w[k] = dt * angular_vel[k]; if (linear_vel) v[k] = dt * linear_vel[k]; }  // either may be NULL = zero (glim_b200.h)
      T_l0_l1 = mul(mul(Tli, rigid_inverse(pose3_expmap(w, v))), Til);  // :41-42
    } else {
      const double time = stamp + tab[i];
      while (cursor + 1 < n_imu && imu_times[cursor + 1] < time) cursor++;  // :94-96
      auto pose_at = [&](size_t k) { M4 p; memcpy(p.m, imu_poses + 16 * k, sizeof(p.m)); return p; };
      if (i == 0) T_imu0_world = rigid_inverse(pose_at(cursor));  // :98-101
      M4 T_world_imu1 = identity();
      if (cursor + 1 >= n_imu) {
        T_world_imu1 = pose_at(cursor);  // :104-105
      } else {
        const double t0 = imu_times[cursor], t1 = imu_times[cursor + 1];
        const double p = fmax(0.0, fmin(1.0, (time - t0) / (t1 - t0)));  // :110
        const M4 L = pose_at(cursor), Rr = pose_at(cursor + 1);
        for (int k = 0; k < 3; k++) T_world_imu1.m[12 + k] = (1.0 - p) * L.m[12 + k] + p * Rr.m[12 + k];  // :117
        double ql[4], qr[4];
        quat_from_rotation(L, ql);
        quat_from_rotation(Rr, qr);
        slerp_to_rotation(ql, qr, p, T_world_imu1);  // :118
      }
      T_l0_l1 = mul(mul(Tli, mul(T_imu0_world, T_world_imu1)), Til);  // :121-122
    }
    memcpy(table_poses + 16 * i, T_l0_l1.m, sizeof(T_l0_l1.m));
  }
  *table_size = tab.size();
  return GB_OK;
}

extern "C" gb_status gb_deskew(gb_ctx* ctx, const double T_imu_lidar[16], const double* linear_vel, const double* angular_vel, size_t n_imu, const double* imu_times, const double* imu_poses,
                               double stamp, size_t n, const double* times, const double* xyzw, const double* T_post, double* out_xyzw) {
  GB_REQUIRE(ctx, "null ctx");
  if (n == 0) return GB_OK;
  GB_REQUIRE(xyzw && out_xyzw && times, "null argument");
  std::vector<int32_t> idx(n);
  std::vector<double> table(16 * n > 16 * 4096 ? 16 * 4096 : 16 * n);
  // the table has at most (t_max - t_min) / 1e-4 + 1 entries; size it for the worst case of this scan
  size_t worst = 1;
  {
    double last = times[0];
    for (size_t i = 1; i < n; i++) if (times[i] - last > 1e-4) { worst++; last = times[i]; }
  }
  table.resize(16 * worst);
  size_t m = 0;
  GB_CHECK(gb_deskew_pose_table(T_imu_lidar, linear_vel, angular_vel, n_imu, imu_times, imu_poses, stamp, n, times, idx.data(), table.data(), &m));
  GB_ENTER(ctx);
  double4 *d_pts, *d_out;
  int* d_idx;
  double* d_tab;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    d_pts = cv.take<double4>(n);
    d_out = cv.take<double4>(n);
    d_idx = cv.take<int>(n);
    d_tab = cv.take<double>(16 * (m + 1));  // the table, then T_post
  }));
  double* d_post = T_post ? d_tab + 16 * m : nullptr;
  GB_CHECK(gb_upload(ctx, {{d_pts, xyzw, sizeof(double4) * n}, {d_idx, idx.data(), sizeof(int) * n}, {d_tab, table.data(), sizeof(double) * 16 * m},
                           {d_post, T_post, sizeof(double) * 16}}));
  GB_CHECK(gb_launch(ctx, "k_deskew", k_deskew, (unsigned)((n + 255) / 256), 256, 0, (int)n, d_pts, d_idx, d_tab, d_post, d_out));
  return gb_download(ctx, {{out_xyzw, d_out, sizeof(double4) * n}});
}
