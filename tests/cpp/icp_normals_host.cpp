// Host build of the ICP factor's per-hit arithmetic (accumulate_icp_hit, glim_b200/csrc/gb_vgicp_math.cuh, the text
// k_icp_grid_sweep compiles) and of the per-point normal of gb_cloud_estimate_normals (covariance_normal,
// glim_b200/csrc/gb_cov_math.cuh, the text k_cloud_normals compiles).  tests/test_icp_normals_host.py compiles this with
// g++ -ffp-contract=off and compares it with the numpy restatements (tests/icp_oracle.py, tests/normals_oracle.py).
#include "../../glim_b200/csrc/gb_vgicp_math.cuh"
#include "../../glim_b200/csrc/gb_cov_math.cuh"

extern "C" {

// One hit's 32 accumulators (all zero before), mode 0 = linearize, 1 = error: source point a (3), target point v (3), pose
// (row-major fp32 R | t, 12 floats).
void icp_hit(int mode, const float* pose12, const float* a, const float* v, float* acc) {
  for (int k = 0; k < 32; k++) acc[k] = 0.f;
  const PoseF P = load_pose(pose12);
  const float4 a0 = {a[0], a[1], a[2], 0.f}, v0 = {v[0], v[1], v[2], 0.f};
  float (&A)[32] = *reinterpret_cast<float (*)[32]>(acc);
  if (mode == 0) accumulate_icp_hit<0>(A, P, a0, v0);
  else accumulate_icp_hit<1>(A, P, a0, v0);
}

// n points: fp32 positions (n x 3) and covariances (n x 6: c00 c01 c02 c11 c12 c22) -> fp32 normals (n x 3)
void normals(int n, const float* xyz, const float* cov6, float* out) {
  for (int i = 0; i < n; i++) {
    const float* p = xyz + 3 * i;
    const float* c = cov6 + 6 * i;
    float v[3];
    covariance_normal(p[0], p[1], p[2], c[0], c[1], c[2], c[3], c[4], c[5], v);
    for (int k = 0; k < 3; k++) out[3 * i + k] = v[k];
  }
}

}  // extern "C"
