// mini_eigen.hpp -- a stand-in for the handful of Eigen types the reference's cloud_covariance_estimation.cpp and
// cloud_deskewing.cpp use, WRITTEN HERE (Eigen is not installed in this environment and nothing of it is copied).
//
// TEST INFRASTRUCTURE ONLY (see oracle/Makefile, target _ref): it lets those two reference translation units compile
// UNMODIFIED from a GLIM source tree so that their control flow and formulas -- not a restatement of them -- can be run against
// oracle/glim_oracle.c.  What this does NOT pin is Eigen's own arithmetic: fixed-size products are evaluated here as plain
// sequential sums, SelfAdjointEigenSolver<Matrix3d>::computeDirect, Quaterniond(Matrix3d) / slerp / toRotationMatrix follow
// Eigen's published algorithms as restated by us.  Every object is a plain value (no expression templates, no alignment tricks).
#pragma once
#include <algorithm>
#include <cassert>
#include <cmath>
#include <cstddef>
#include <limits>
#include <vector>

#define EIGEN_MAKE_ALIGNED_OPERATOR_NEW
#define EIGEN_WORLD_VERSION 3  // include/glim_b200/gtsam_points_compat.hpp keys its "points are Eigen types" branch on this macro

namespace Eigen {

template <int R, int C> struct Mat;

template <int N> struct DiagWrap { double d[N]; };
template <int N> struct BoolArray {
  bool b[N];
  bool any() const { for (int k = 0; k < N; k++) if (b[k]) return true; return false; }
  bool all() const { for (int k = 0; k < N; k++) if (!b[k]) return false; return true; }
};
template <int N> struct ArrayWrap {
  double v[N];
  Mat<N, 1> max(double m) const;
  BoolArray<N> operator>(const ArrayWrap& o) const { BoolArray<N> r; for (int k = 0; k < N; k++) r.b[k] = v[k] > o.v[k]; return r; }
  BoolArray<N> operator>=(const ArrayWrap& o) const { BoolArray<N> r; for (int k = 0; k < N; k++) r.b[k] = v[k] >= o.v[k]; return r; }
  BoolArray<N> operator<=(const ArrayWrap& o) const { BoolArray<N> r; for (int k = 0; k < N; k++) r.b[k] = v[k] <= o.v[k]; return r; }
};

// lvalue block of a matrix (c.block<3,3>(0,0) = ..., T.translation() = ..., T.linear() = ...)
template <int BR, int BC, int R, int C> struct BlockRef {
  Mat<R, C>* m;
  int i0, j0;
  BlockRef& operator=(const Mat<BR, BC>& v);
  operator Mat<BR, BC>() const;
};

template <int R, int C> struct CommaInit {
  Mat<R, C>* m;
  int pos;  // number of coefficients written (vectors only)
  CommaInit& operator,(double s) { m->a[pos++] = s; return *this; }
  template <int K> CommaInit& operator,(const Mat<K, 1>& v) { for (int k = 0; k < K; k++) m->a[pos++] = v.a[k]; return *this; }
  Mat<R, C> finished() const { return *m; }
};

template <int R, int C> struct Mat {
  double a[R * C];  // column-major, like Eigen's default
  Mat() {}           // uninitialised, like Eigen
  Mat(double x, double y, double z) { static_assert(R * C == 3, "3-vector"); a[0] = x; a[1] = y; a[2] = z; }
  template <int RR, int CC> Mat(const BlockRef<R, C, RR, CC>& b) { *this = (Mat<R, C>)b; }

  void setZero() { for (int k = 0; k < R * C; k++) a[k] = 0.0; }
  bool allFinite() const { for (int k = 0; k < R * C; k++) if (!std::isfinite(a[k])) return false; return true; }
  double* data() { return a; }
  const double* data() const { return a; }
  template <int K> Mat<K, 1> head() const { static_assert(C == 1 && K <= R, "vector"); Mat<K, 1> h; for (int k = 0; k < K; k++) h.a[k] = a[k]; return h; }
  static Mat Zero() { Mat m; for (int k = 0; k < R * C; k++) m.a[k] = 0.0; return m; }
  static Mat Identity() { Mat m = Zero(); for (int k = 0; k < (R < C ? R : C); k++) m(k, k) = 1.0; return m; }

  double& operator()(int i, int j) { return a[j * R + i]; }
  double operator()(int i, int j) const { return a[j * R + i]; }
  double& operator()(int i) { return a[i]; }
  double operator()(int i) const { return a[i]; }
  double& operator[](int i) { return a[i]; }
  double operator[](int i) const { return a[i]; }

  Mat<C, R> transpose() const { Mat<C, R> t; for (int i = 0; i < R; i++) for (int j = 0; j < C; j++) t(j, i) = (*this)(i, j); return t; }
  Mat& operator+=(const Mat& o) { for (int k = 0; k < R * C; k++) a[k] += o.a[k]; return *this; }
  Mat& operator-=(const Mat& o) { for (int k = 0; k < R * C; k++) a[k] -= o.a[k]; return *this; }
  Mat operator-() const { Mat m; for (int k = 0; k < R * C; k++) m.a[k] = -a[k]; return m; }
  Mat operator+(const Mat& o) const { Mat m; for (int k = 0; k < R * C; k++) m.a[k] = a[k] + o.a[k]; return m; }
  Mat operator-(const Mat& o) const { Mat m; for (int k = 0; k < R * C; k++) m.a[k] = a[k] - o.a[k]; return m; }
  Mat operator/(double s) const { Mat m; for (int k = 0; k < R * C; k++) m.a[k] = a[k] / s; return m; }
  Mat operator*(double s) const { Mat m; for (int k = 0; k < R * C; k++) m.a[k] = a[k] * s; return m; }
  friend Mat operator*(double s, const Mat& o) { Mat m; for (int k = 0; k < R * C; k++) m.a[k] = s * o.a[k]; return m; }
  template <int K> Mat<R, K> operator*(const Mat<C, K>& o) const {
    Mat<R, K> m;
    for (int i = 0; i < R; i++)
      for (int j = 0; j < K; j++) {
        double s = (*this)(i, 0) * o(0, j);
        for (int k = 1; k < C; k++) s += (*this)(i, k) * o(k, j);
        m(i, j) = s;
      }
    return m;
  }
  Mat operator*(const DiagWrap<C>& d) const { Mat m; for (int i = 0; i < R; i++) for (int j = 0; j < C; j++) m(i, j) = (*this)(i, j) * d.d[j]; return m; }

  double dot(const Mat& o) const { double s = a[0] * o.a[0]; for (int k = 1; k < R * C; k++) s += a[k] * o.a[k]; return s; }
  double squaredNorm() const { return dot(*this); }
  double norm() const { return std::sqrt(squaredNorm()); }
  Mat normalized() const { return *this / norm(); }
  Mat<3, 1> cross(const Mat<3, 1>& o) const {
    static_assert(R * C == 3, "3-vector");
    return Mat<3, 1>(a[1] * o.a[2] - a[2] * o.a[1], a[2] * o.a[0] - a[0] * o.a[2], a[0] * o.a[1] - a[1] * o.a[0]);
  }
  Mat<R, 1> col(int j) const { Mat<R, 1> v; for (int i = 0; i < R; i++) v.a[i] = (*this)(i, j); return v; }
  void setCol(int j, const Mat<R, 1>& v) { for (int i = 0; i < R; i++) (*this)(i, j) = v.a[i]; }

  template <int BR, int BC> BlockRef<BR, BC, R, C> block(int i, int j) { return BlockRef<BR, BC, R, C>{this, i, j}; }
  template <int BR, int BC> Mat<BR, BC> block(int i, int j) const {
    Mat<BR, BC> b;
    for (int r = 0; r < BR; r++) for (int c = 0; c < BC; c++) b(r, c) = (*this)(i + r, j + c);
    return b;
  }
  DiagWrap<R> asDiagonal() const { static_assert(C == 1, "vector"); DiagWrap<R> d; for (int k = 0; k < R; k++) d.d[k] = a[k]; return d; }
  ArrayWrap<R> array() const { static_assert(C == 1, "vector"); ArrayWrap<R> w; for (int k = 0; k < R; k++) w.v[k] = a[k]; return w; }

  Mat inverse() const {  // 3x3 by cofactors (what Eigen does for fixed sizes <= 4)
    static_assert(R == 3 && C == 3, "3x3");
    const Mat& m = *this;
    Mat c;
    c(0, 0) = m(1, 1) * m(2, 2) - m(1, 2) * m(2, 1); c(0, 1) = m(0, 2) * m(2, 1) - m(0, 1) * m(2, 2); c(0, 2) = m(0, 1) * m(1, 2) - m(0, 2) * m(1, 1);
    c(1, 0) = m(1, 2) * m(2, 0) - m(1, 0) * m(2, 2); c(1, 1) = m(0, 0) * m(2, 2) - m(0, 2) * m(2, 0); c(1, 2) = m(0, 2) * m(1, 0) - m(0, 0) * m(1, 2);
    c(2, 0) = m(1, 0) * m(2, 1) - m(1, 1) * m(2, 0); c(2, 1) = m(0, 1) * m(2, 0) - m(0, 0) * m(2, 1); c(2, 2) = m(0, 0) * m(1, 1) - m(0, 1) * m(1, 0);
    const double det = m(0, 0) * c(0, 0) + m(0, 1) * c(1, 0) + m(0, 2) * c(2, 0);
    return c / det;
  }

  template <int K> CommaInit<R, C> operator<<(const Mat<K, 1>& v) { CommaInit<R, C> ci{this, 0}; ci, v; return ci; }
  CommaInit<R, C> operator<<(double s) { CommaInit<R, C> ci{this, 0}; ci, s; return ci; }
};

template <int N> Mat<N, 1> ArrayWrap<N>::max(double m) const { Mat<N, 1> r; for (int k = 0; k < N; k++) r.a[k] = v[k] < m ? m : v[k]; return r; }
template <int BR, int BC, int R, int C> BlockRef<BR, BC, R, C>& BlockRef<BR, BC, R, C>::operator=(const Mat<BR, BC>& v) {
  for (int r = 0; r < BR; r++) for (int c = 0; c < BC; c++) (*m)(i0 + r, j0 + c) = v(r, c);
  return *this;
}
template <int BR, int BC, int R, int C> BlockRef<BR, BC, R, C>::operator Mat<BR, BC>() const {
  Mat<BR, BC> b;
  for (int r = 0; r < BR; r++) for (int c = 0; c < BC; c++) b(r, c) = (*m)(i0 + r, j0 + c);
  return b;
}

struct Vector3f { float a[3]; };  // device-side element types the shim only names (standard_viewer_mem.cpp:49-58)
struct Matrix3f { float a[9]; };
using Vector3d = Mat<3, 1>;
using Vector4d = Mat<4, 1>;
using Matrix3d = Mat<3, 3>;
using Matrix4d = Mat<4, 4>;

// SelfAdjointEigenSolver<Matrix3d>::computeDirect: Eigen's closed-form solver (shift by the mean eigenvalue, scale by the
// largest coefficient, trigonometric roots of the characteristic polynomial, eigenvectors from cross products of the rows of
// A - lambda I with the best-conditioned pair first), eigenvalues ascending.
template <typename M> class SelfAdjointEigenSolver;
template <> class SelfAdjointEigenSolver<Matrix3d> {
public:
  SelfAdjointEigenSolver& computeDirect(const Matrix3d& mat) {
    const double shift = (mat(0, 0) + mat(1, 1) + mat(2, 2)) / 3.0;
    Matrix3d s = mat;
    s(0, 1) = s(1, 0); s(0, 2) = s(2, 0); s(1, 2) = s(2, 1);  // the lower triangle is the one that is read
    for (int k = 0; k < 3; k++) s(k, k) -= shift;
    double scale = 0.0;
    for (int k = 0; k < 9; k++) scale = std::max(scale, std::fabs(s.a[k]));
    if (scale > 0.0) s = s / scale;
    roots(s, vals_);
    const double eps = std::numeric_limits<double>::epsilon();
    if (vals_[2] - vals_[0] <= eps) {
      vecs_ = Matrix3d::Identity();
    } else {
      double d0 = vals_[2] - vals_[1], d1 = vals_[1] - vals_[0];
      int k = 0, l = 2;
      if (d0 > d1) { std::swap(k, l); d0 = d1; }
      Vector3d vk, vl;
      {
        Matrix3d t = s;
        for (int i = 0; i < 3; i++) t(i, i) -= vals_[k];
        kernel(t, vk, vl);
      }
      if (d0 <= 2.0 * eps * d1) {
        vl = vl - vk * vk.dot(vl);
        vl = vl.normalized();
      } else {
        Matrix3d t = s;
        for (int i = 0; i < 3; i++) t(i, i) -= vals_[l];
        Vector3d dummy;
        kernel(t, vl, dummy);
      }
      vecs_.setCol(k, vk);
      vecs_.setCol(l, vl);
      vecs_.setCol(1, vecs_.col(2).cross(vecs_.col(0)).normalized());
    }
    for (int i = 0; i < 3; i++) vals_[i] = vals_[i] * scale + shift;
    return *this;
  }
  const Vector3d& eigenvalues() const { return vals_; }
  const Matrix3d& eigenvectors() const { return vecs_; }

private:
  static void roots(const Matrix3d& m, Vector3d& r) {
    const double inv3 = 1.0 / 3.0, sqrt3 = std::sqrt(3.0);
    const double c0 = m(0, 0) * m(1, 1) * m(2, 2) + 2.0 * m(1, 0) * m(2, 0) * m(2, 1) - m(0, 0) * m(2, 1) * m(2, 1) - m(1, 1) * m(2, 0) * m(2, 0) - m(2, 2) * m(1, 0) * m(1, 0);
    const double c1 = m(0, 0) * m(1, 1) - m(1, 0) * m(1, 0) + m(0, 0) * m(2, 2) - m(2, 0) * m(2, 0) + m(1, 1) * m(2, 2) - m(2, 1) * m(2, 1);
    const double c2 = m(0, 0) + m(1, 1) + m(2, 2);
    const double c2_3 = c2 * inv3;
    double a_3 = (c2 * c2_3 - c1) * inv3;
    a_3 = std::max(a_3, 0.0);
    const double half_b = 0.5 * (c0 + c2_3 * (2.0 * c2_3 * c2_3 - c1));
    double q = a_3 * a_3 * a_3 - half_b * half_b;
    q = std::max(q, 0.0);
    const double rho = std::sqrt(a_3);
    const double theta = std::atan2(std::sqrt(q), half_b) * inv3;
    const double ct = std::cos(theta), st = std::sin(theta);
    r[0] = c2_3 - rho * (ct + sqrt3 * st);
    r[1] = c2_3 - rho * (ct - sqrt3 * st);
    r[2] = c2_3 + 2.0 * rho * ct;
  }
  // res = a unit vector of the kernel of the (rank <= 2) symmetric matrix m; ref = the row it was built from, normalised
  static bool kernel(Matrix3d& m, Vector3d& res, Vector3d& ref) {
    int i0 = 0;
    double best = std::fabs(m(0, 0));
    for (int i = 1; i < 3; i++) if (std::fabs(m(i, i)) > best) { best = std::fabs(m(i, i)); i0 = i; }
    ref = m.col(i0);
    ref = ref / ref.norm();
    const Vector3d c0 = ref.cross(m.col((i0 + 1) % 3)), c1 = ref.cross(m.col((i0 + 2) % 3));
    const double n0 = c0.squaredNorm(), n1 = c1.squaredNorm();
    if (n0 > n1) res = c0 / std::sqrt(n0); else res = c1 / std::sqrt(n1);
    return true;
  }
  Vector3d vals_;
  Matrix3d vecs_;
};

// Quaternion<double>: coefficients (x, y, z, w); from a rotation matrix, slerp and toRotationMatrix as Eigen documents them
class Quaterniond {
public:
  double x, y, z, w;
  Quaterniond() {}
  Quaterniond(double w_, double x_, double y_, double z_) : x(x_), y(y_), z(z_), w(w_) {}
  explicit Quaterniond(const Matrix3d& m) {
    double t = m(0, 0) + m(1, 1) + m(2, 2);
    if (t > 0.0) {
      t = std::sqrt(t + 1.0);
      w = 0.5 * t;
      t = 0.5 / t;
      x = (m(2, 1) - m(1, 2)) * t; y = (m(0, 2) - m(2, 0)) * t; z = (m(1, 0) - m(0, 1)) * t;
    } else {
      int i = 0;
      if (m(1, 1) > m(0, 0)) i = 1;
      if (m(2, 2) > m(i, i)) i = 2;
      const int j = (i + 1) % 3, k = (j + 1) % 3;
      t = std::sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0);
      double q[3];
      q[i] = 0.5 * t;
      t = 0.5 / t;
      w = (m(k, j) - m(j, k)) * t;
      q[j] = (m(j, i) + m(i, j)) * t;
      q[k] = (m(k, i) + m(i, k)) * t;
      x = q[0]; y = q[1]; z = q[2];
    }
  }
  Quaterniond slerp(double t, const Quaterniond& o) const {
    const double one = 1.0 - std::numeric_limits<double>::epsilon();
    const double d = x * o.x + y * o.y + z * o.z + w * o.w, ad = std::fabs(d);
    double s0, s1;
    if (ad >= one) {
      s0 = 1.0 - t; s1 = t;
    } else {
      const double theta = std::acos(ad), st = std::sin(theta);
      s0 = std::sin((1.0 - t) * theta) / st;
      s1 = std::sin(t * theta) / st;
    }
    if (d < 0.0) s1 = -s1;
    return Quaterniond(s0 * w + s1 * o.w, s0 * x + s1 * o.x, s0 * y + s1 * o.y, s0 * z + s1 * o.z);
  }
  Matrix3d toRotationMatrix() const {
    Matrix3d r;
    const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    r(0, 0) = 1.0 - (tyy + tzz); r(0, 1) = txy - twz; r(0, 2) = txz + twy;
    r(1, 0) = txy + twz; r(1, 1) = 1.0 - (txx + tzz); r(1, 2) = tyz - twx;
    r(2, 0) = txz - twy; r(2, 1) = tyz + twx; r(2, 2) = 1.0 - (txx + tyy);
    return r;
  }
};

// Transform<double, 3, Isometry>: 4x4 storage, last row assumed (0 0 0 1)
class Isometry3d {
public:
  Isometry3d() {}
  explicit Isometry3d(const Matrix4d& mat) : m_(mat) {}
  static Isometry3d Identity() { return Isometry3d(Matrix4d::Identity()); }
  const Matrix4d& matrix() const { return m_; }
  Matrix3d linear() const { return m_.block<3, 3>(0, 0); }
  BlockRef<3, 3, 4, 4> linear() { return m_.block<3, 3>(0, 0); }
  Vector3d translation() const { return m_.block<3, 1>(0, 3); }
  BlockRef<3, 1, 4, 4> translation() { return m_.block<3, 1>(0, 3); }
  Isometry3d inverse() const {  // R^T, -R^T t
    const Matrix3d Rt = linear().transpose();
    Isometry3d r = Identity();
    r.linear() = Rt;
    r.translation() = -(Rt * translation());
    return r;
  }
  Isometry3d operator*(const Isometry3d& o) const {  // affine product: linear = R1 R2, translation = R1 t2 + t1
    Isometry3d r = Identity();
    r.linear() = linear() * o.linear();
    r.translation() = linear() * o.translation() + translation();
    return r;
  }
  Vector3d operator*(const Vector3d& p) const { return linear() * p + translation(); }  // R p + t
  Vector4d operator*(const Vector4d& v) const {  // (3x4 affine part) * v, last coefficient copied
    Vector4d r;
    for (int i = 0; i < 3; i++) {
      double s = m_(i, 0) * v[0];
      for (int k = 1; k < 4; k++) s += m_(i, k) * v[k];
      r[i] = s;
    }
    r[3] = v[3];
    return r;
  }

private:
  Matrix4d m_;
};

}  // namespace Eigen
