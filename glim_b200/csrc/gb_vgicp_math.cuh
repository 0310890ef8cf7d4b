// gb_vgicp_math.cuh -- the per-point arithmetic of the fused VGICP sweep kernels (gb_kernels_vgicp.cu), kept free of anything
// that only exists on the device so that the SAME TEXT also compiles for the host: tests/cpp/kernel_math_host.cpp builds it
// with g++ and tests/test_kernel_math_host.py checks it against the CPU oracle on the CPU-only box (-m "not gpu").  The
// product never runs this on the host: only the kernels include it in a device build.  Math: SURVEY.md Appendix A.
#pragma once
#ifdef __CUDACC__
#define GB_HD __device__ __forceinline__
#else
#include <math.h>
#include <stdint.h>
#define GB_HD static inline
struct float4 { float x, y, z, w; };
struct int4 { int x, y, z, w; };
static inline float __fdividef(float a, float b) { return a / b; }
// cvt.rmi.s32.f32: NaN -> 0, saturating
static inline int __float2int_rd(float v) {
  if (!(v == v)) return 0;
  const float f = floorf(v);
  if (f >= 2147483648.0f) return 2147483647;
  if (f < -2147483648.0f) return (-2147483647 - 1);
  return (int)f;
}
#endif

// canonical voxel coordinate (fp32): floorf(p * inv_res); oracle: voxel_coord_f32 (glim_oracle.c)
GB_HD int gb_coord(float p, float inv_res) { return __float2int_rd(p * inv_res); }
// XOR-of-primes hash (SURVEY B.2); low 32 bits == the u64 evaluation modulo a power-of-two table
GB_HD uint32_t gb_hash(int x, int y, int z) {
  return ((uint32_t)x * 73856093u) ^ ((uint32_t)y * 19349669u) ^ ((uint32_t)z * 83492791u);
}
// linear-probing lookup of voxel (cx, cy, cz) in a voxel table (SURVEY B.4): its index, -1 if absent
GB_HD int gb_lookup(const int4* __restrict__ buckets, uint32_t mask, int max_scan, int cx, int cy, int cz) {
  const uint32_t h = gb_hash(cx, cy, cz);
  for (int i = 0; i < max_scan; i++) {
    const int4 b = buckets[(h + (uint32_t)i) & mask];
    if (b.w < 0) return -1;
    if (b.x == cx && b.y == cy && b.z == cz) return b.w;
  }
  return -1;
}
// the project's fixed pseudo-random pick ([EXT]: the reference draws with std::mt19937): the points / voxels with the smallest
// rg_hash(seed, index) are kept (random-grid downsampling, frame-merge thinning, voxel-map insert sampling; the oracle shares it),
// and RANSAC draws its samples from it (gb_global_math.cuh)
GB_HD unsigned long long rg_hash(unsigned long long seed, unsigned i) {
  unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (unsigned long long)(i + 1u);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

#ifndef GB_MODE_LINEARIZE_VALUE
#define GB_MODE_LINEARIZE_VALUE 0  // == GB_MODE_LINEARIZE (gb_internal.cuh)
#endif

namespace {

struct PoseF {
  float r00, r01, r02, r10, r11, r12, r20, r21, r22, tx, ty, tz;
};

GB_HD PoseF load_pose(const float* s) {
  PoseF P;
  P.r00 = s[0]; P.r01 = s[1]; P.r02 = s[2];
  P.r10 = s[3]; P.r11 = s[4]; P.r12 = s[5];
  P.r20 = s[6]; P.r21 = s[7]; P.r22 = s[8];
  P.tx = s[9]; P.ty = s[10]; P.tz = s[11];
  return P;
}

// pose -> fp32 row-major R | t  (Isometry3f cast of the reference GPU factor, SURVEY A.1)
GB_HD PoseF pose_from_colmajor(const double* __restrict__ T) {
  PoseF P;
  P.r00 = (float)T[0]; P.r01 = (float)T[4]; P.r02 = (float)T[8];  P.tx = (float)T[12];
  P.r10 = (float)T[1]; P.r11 = (float)T[5]; P.r12 = (float)T[9];  P.ty = (float)T[13];
  P.r20 = (float)T[2]; P.r21 = (float)T[6]; P.r22 = (float)T[10]; P.tz = (float)T[14];
  return P;
}

// q = R a + t with the canonical FMA order (bit-exact with transform_f32 in the oracle)
GB_HD void transform(const PoseF& P, float ax, float ay, float az, float& qx, float& qy, float& qz) {
  qx = fmaf(P.r00, ax, fmaf(P.r01, ay, fmaf(P.r02, az, P.tx)));
  qy = fmaf(P.r10, ax, fmaf(P.r11, ay, fmaf(P.r12, az, P.ty)));
  qz = fmaf(P.r20, ax, fmaf(P.r21, ay, fmaf(P.r22, az, P.tz)));
}

// M = (C_B + R C_A R^T)^-1, symmetric 3x3 (xx xy xz yy yz zz).  Returns false when the fused covariance is singular or
// non-finite: such a point contributes nothing and is not counted (oracle: mat3_inv fails -> point skipped).
GB_HD bool fused_mahalanobis(
  const PoseF& P, float cxx, float cxy, float cxz, float cyy, float cyz, float czz,  // C_A
  float bxx, float bxy, float bxz, float byy, float byz, float bzz,                  // C_B
  float& mxx, float& mxy, float& mxz, float& myy, float& myz, float& mzz) {
  // T = R * C_A
  const float t00 = P.r00 * cxx + P.r01 * cxy + P.r02 * cxz;
  const float t01 = P.r00 * cxy + P.r01 * cyy + P.r02 * cyz;
  const float t02 = P.r00 * cxz + P.r01 * cyz + P.r02 * czz;
  const float t10 = P.r10 * cxx + P.r11 * cxy + P.r12 * cxz;
  const float t11 = P.r10 * cxy + P.r11 * cyy + P.r12 * cyz;
  const float t12 = P.r10 * cxz + P.r11 * cyz + P.r12 * czz;
  const float t20 = P.r20 * cxx + P.r21 * cxy + P.r22 * cxz;
  const float t21 = P.r20 * cxy + P.r21 * cyy + P.r22 * cyz;
  const float t22 = P.r20 * cxz + P.r21 * cyz + P.r22 * czz;
  // S = C_B + T R^T (upper triangle)
  const float sxx = bxx + (t00 * P.r00 + t01 * P.r01 + t02 * P.r02);
  const float sxy = bxy + (t00 * P.r10 + t01 * P.r11 + t02 * P.r12);
  const float sxz = bxz + (t00 * P.r20 + t01 * P.r21 + t02 * P.r22);
  const float syy = byy + (t10 * P.r10 + t11 * P.r11 + t12 * P.r12);
  const float syz = byz + (t10 * P.r20 + t11 * P.r21 + t12 * P.r22);
  const float szz = bzz + (t20 * P.r20 + t21 * P.r21 + t22 * P.r22);
  // inverse by cofactors
  const float c00 = syy * szz - syz * syz;
  const float c01 = sxz * syz - sxy * szz;
  const float c02 = sxy * syz - sxz * syy;
  const float c11 = sxx * szz - sxz * sxz;
  const float c12 = sxy * sxz - sxx * syz;
  const float c22 = sxx * syy - sxy * sxy;
  const float det = sxx * c00 + sxy * c01 + sxz * c02;
  const float id = __fdividef(1.0f, det);
  mxx = c00 * id; mxy = c01 * id; mxz = c02 * id; myy = c11 * id; myz = c12 * id; mzz = c22 * id;
  return det != 0.0f && fabsf(det) <= 3.0e38f;
}

// One inlier's contribution: source point (a0 = {x y z c00}, a1 = {c01 c02 c11 c12}, a2 = c22), target voxel record
// (v0 = {mx my mz c00}, v1 = {c01 c02 c11 c12}, v2.x = c22), evaluated at pose Pe.  acc[0..20] = upper triangle of H_tt
// (row-major), acc[21..26] = b_t, acc[27] = error, acc[28] = inlier count.
template <int MODE>
GB_HD void accumulate_hit(float (&acc)[32], const PoseF& Pe, const float4 a0, const float4 a1, const float a2, const float4 v0, const float4 v1, const float4 v2) {
  float qx, qy, qz;
  transform(Pe, a0.x, a0.y, a0.z, qx, qy, qz);
  float mxx, mxy, mxz, myy, myz, mzz;
  if (!fused_mahalanobis(Pe, a0.w, a1.x, a1.y, a1.z, a1.w, a2, v0.w, v1.x, v1.y, v1.z, v1.w, v2.x, mxx, mxy, mxz, myy, myz, mzz)) return;
  const float rx = v0.x - qx, ry = v0.y - qy, rz = v0.z - qz;
  // a NaN source point converts to voxel coordinate 0 and may "hit" voxel (0, ., .): it is rejected here, on the hit path only
  // (the oracle never finds a voxel for it) -- three instructions per HIT instead of per point
  const float fin = (rx + ry) + rz;
  if (!(fin == fin)) return;
  const float wx = mxx * rx + mxy * ry + mxz * rz;
  const float wy = mxy * rx + myy * ry + myz * rz;
  const float wz = mxz * rx + myz * ry + mzz * rz;
  acc[27] += rx * wx + ry * wy + rz * wz;
  acc[28] += 1.0f;
  if (MODE == GB_MODE_LINEARIZE_VALUE) {
    // G = hat(q) M   (rows: rotation, cols: translation block of H_tt)
    const float g00 = qy * mxz - qz * mxy, g01 = qy * myz - qz * myy, g02 = qy * mzz - qz * myz;
    const float g10 = qz * mxx - qx * mxz, g11 = qz * mxy - qx * myz, g12 = qz * mxz - qx * mzz;
    const float g20 = qx * mxy - qy * mxx, g21 = qx * myy - qy * mxy, g22 = qx * myz - qy * mxz;
    // H_rr = G hat(q)^T : row i = q x g_i   (upper triangle)
    acc[0] += qy * g02 - qz * g01;
    acc[1] += qz * g00 - qx * g02;
    acc[2] += qx * g01 - qy * g00;
    acc[3] += g00; acc[4] += g01; acc[5] += g02;
    acc[6] += qz * g10 - qx * g12;
    acc[7] += qx * g11 - qy * g10;
    acc[8] += g10; acc[9] += g11; acc[10] += g12;
    acc[11] += qx * g21 - qy * g20;
    acc[12] += g20; acc[13] += g21; acc[14] += g22;
    acc[15] += mxx; acc[16] += mxy; acc[17] += mxz; acc[18] += myy; acc[19] += myz; acc[20] += mzz;
    // b_t = [q x w ; w]
    acc[21] += qy * wz - qz * wy;
    acc[22] += qz * wx - qx * wz;
    acc[23] += qx * wy - qy * wx;
    acc[24] += wx; acc[25] += wy; acc[26] += wz;
  }
}

// One inlier of a point-to-point ICP factor (k_icp_grid_sweep): accumulate_hit with M = I, reading only the source point
// a0 = {x y z .} and the target point v0 = {x y z .}.  r = p - q, error += r^T r; G = hat(q), so H_rr = hat(q) hat(q)^T,
// H_rt = hat(q), H_tt = I and b_t = [q x r ; r].  The correspondence search (grid_nearest) only returns points with a finite
// d2 < max_d2, so r is finite here.
template <int MODE>
GB_HD void accumulate_icp_hit(float (&acc)[32], const PoseF& Pe, const float4 a0, const float4 v0) {
  float qx, qy, qz;
  transform(Pe, a0.x, a0.y, a0.z, qx, qy, qz);
  const float rx = v0.x - qx, ry = v0.y - qy, rz = v0.z - qz;
  acc[27] += rx * rx + ry * ry + rz * rz;
  acc[28] += 1.0f;
  if (MODE == GB_MODE_LINEARIZE_VALUE) {
    // the upper triangle of H_tt in accumulate_hit's order; the entries that are zero for M = I are left out
    acc[0] += qy * qy + qz * qz;
    acc[1] -= qx * qy;
    acc[2] -= qx * qz;
    acc[4] -= qz; acc[5] += qy;
    acc[6] += qz * qz + qx * qx;
    acc[7] -= qy * qz;
    acc[8] += qz; acc[10] -= qx;
    acc[11] += qx * qx + qy * qy;
    acc[12] -= qy; acc[13] += qx;
    acc[15] += 1.0f; acc[18] += 1.0f; acc[20] += 1.0f;
    acc[21] += qy * rz - qz * ry;
    acc[22] += qz * rx - qx * rz;
    acc[23] += qx * ry - qy * rx;
    acc[24] += rx; acc[25] += ry; acc[26] += rz;
  }
}

// Surface validation (set_enable_surface_validation(true), odometry_estimation_gpu.cpp:145, :162).  The reference rule lives
// in the un-vendored gtsam_points and is not recoverable here (SURVEY A.6): ours is an ORIENTATION-CONSISTENCY gate that needs
// no eigen-decomposition.  With n = R n_A (source normal, flipped towards the sensor by the covariance estimator, rotated into
// the target frame) a correspondence is kept iff   3 n^T C_B n <= tr(C_B),
// i.e. the voxel's spread along the source normal is at most its mean spread: for a planar voxel with normal m this is
// |n . m| >= 1/sqrt(3) (within ~55 degrees); voxels that mix surfaces (corners, thin walls seen from both sides) or face
// another way are rejected.  Canonical fp32 operation order (the oracle evaluates the same expression bit for bit).
GB_HD bool surface_ok(const PoseF& P, const float4 nr, float bxx, float bxy, float bxz, float byy, float byz, float bzz) {
  const float nx = fmaf(P.r00, nr.x, fmaf(P.r01, nr.y, P.r02 * nr.z));
  const float ny = fmaf(P.r10, nr.x, fmaf(P.r11, nr.y, P.r12 * nr.z));
  const float nz = fmaf(P.r20, nr.x, fmaf(P.r21, nr.y, P.r22 * nr.z));
  const float ux = fmaf(bxx, nx, fmaf(bxy, ny, bxz * nz));
  const float uy = fmaf(bxy, nx, fmaf(byy, ny, byz * nz));
  const float uz = fmaf(bxz, nx, fmaf(byz, ny, bzz * nz));
  const float s = fmaf(nx, ux, fmaf(ny, uy, nz * uz));
  const float tr = (bxx + byy) + bzz;
  return 3.0f * s <= tr;
}

// slab row element e (see GB_SLAB_STRIDE in include/glim_b200.h) -> index in the 122-double record
GB_HD int slab_to_record(int e) {
  if (e < 21 || (e >= 57 && e < 78)) {  // upper triangles of H_tt / H_ss, row-major (i <= j)
    int u = e < 21 ? e : e - 57, i = 0;
    while (u >= 6 - i) { u -= 6 - i; i++; }
    const int j = i + u;
    return (e < 21 ? 0 : 36) + j * 6 + i;
  }
  if (e < 57) return 72 + (e - 21);   // H_ts, column-major as in the record
  if (e < 84) return 108 + (e - 78);  // b_t
  if (e < 90) return 114 + (e - 84);  // b_s
  return 120 + (e - 90);              // error, num_inliers
}

}  // namespace
