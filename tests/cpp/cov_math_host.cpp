// Host build of the covariance kernels' per-point arithmetic (glim_b200/csrc/gb_cov_math.cuh -- the SAME text k_covariances
// and k_covariances_planes compile), laid out like go_covariance_estimate.  TEST INFRASTRUCTURE: built by
// tests/test_cov_degenerate.py with g++ -ffp-contract=off and compared bit for bit with the CPU oracle; nothing in the product
// links it.
#include <stddef.h>

#include "../../glim_b200/csrc/gb_cov_math.cuh"

// pts4: n x 4, neighbors: n x kc; normals4: n x 4, covs16: n x 16 (column-major 4x4, last row / column zero)
extern "C" void cm_covariance_estimate(int n, const double* pts4, const int* neighbors, int kc, int k, double* normals4, double* covs16) {
  const double4* P = reinterpret_cast<const double4*>(pts4);
  for (int i = 0; i < n; i++) {
    double C[9], nrm[3];
    plane_covariance(i, P, neighbors, kc, k, C, nrm);
    double* Co = covs16 + 16 * (size_t)i;
    for (int e = 0; e < 16; e++) Co[e] = 0.0;
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) Co[c * 4 + r] = C[r * 3 + c];
    double* no = normals4 + 4 * (size_t)i;
    no[0] = nrm[0]; no[1] = nrm[1]; no[2] = nrm[2]; no[3] = 0.0;
  }
}
