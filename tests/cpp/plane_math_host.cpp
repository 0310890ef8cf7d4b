// Host build of the plane bundle adjustment's arithmetic (glim_b200/csrc/gb_plane_math.cuh, the text k_plane_reduce and
// k_plane_evm compile).  tests/test_plane_ba_host.py compiles this with g++ -ffp-contract=off and compares it with the
// per-point restatement of tests/plane_ba_oracle.py.
#include "../../glim_b200/csrc/gb_plane_math.cuh"

#include <vector>

extern "C" {

// the patch statistics of n points from s = sum q and S = sum q q^T (xx xy xz yy yz zz)
void patch_stats(double n, const double* s, const double* S, double* ev) { plane_stats(n, s, S, ev); }

// One factor of K keys (moments K x GB_PLANE_MOMENTS, poses K x 16 column-major, offset o) as k_plane_evm evaluates it:
// e, b (6K), H (6K x 6K, column-major); returns 1 when degenerate (H and b zero).
int plane_evm(int K, const double* mom, const double* X, const double* o, double* H, double* b, double* e) {
  double C[9], pbar[3], N, ev[3], U[9];
  plane_evm_cov(K, mom, X, o, C, pbar, &N);
  eigen_sym3_direct(C, ev, U);
  *e = ev[0];
  const int n6 = 6 * K;
  if (plane_evm_degenerate(ev)) {
    for (int i = 0; i < n6 * n6; i++) H[i] = 0.0;
    for (int i = 0; i < n6; i++) b[i] = 0.0;
    return 1;
  }
  std::vector<double> terms((size_t)GB_PLANE_KEY_TERMS * K);
  for (int k = 0; k < K; k++) {
    double g[6];
    plane_evm_key(mom + GB_PLANE_MOMENTS * k, X + 16 * k, o, pbar, N, U, terms.data() + GB_PLANE_KEY_TERMS * k, g);
    for (int r = 0; r < 6; r++) b[6 * k + r] = 0.5 * g[r];
  }
  for (int c = 0; c < n6; c++)
    for (int r = 0; r < n6; r++) H[(size_t)c * n6 + r] = plane_evm_entry(r, c, terms.data(), N, ev);
  return 0;
}

}  // extern "C"
