// Host build of the map segmentation's per-point and per-pair arithmetic (glim_b200/csrc/gb_segment_math.cuh, the text
// k_concat_flags, k_concat_emit and the k_rg_* kernels compile).  tests/test_segment_host.py compiles this with
// g++ -ffp-contract=off and compares it with the numpy restatement (tests/segment_oracle.py).
#include "../../glim_b200/csrc/gb_segment_math.cuh"

extern "C" {

// out[i] = seg_keyed of point i (n x 3 fp32) at the fp32 cell inverse inv
void keyed(int n, const float* xyz, float inv, int* out) {
  for (int i = 0; i < n; i++) out[i] = seg_keyed(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], inv) ? 1 : 0;
}

// out[i] = the edge test of points a_i, b_i (n x 3 positions and normals): fp32 point_d2 < max_d2 and the normal test
void edge(int n, const float* pa, const float* na, const float* pb, const float* nb, float max_d2, double cos_t, int* out) {
  for (int i = 0; i < n; i++) {
    const float4 b = {pb[3 * i], pb[3 * i + 1], pb[3 * i + 2], 0.f};
    const bool near = point_d2(b, pa[3 * i], pa[3 * i + 1], pa[3 * i + 2]) < max_d2;
    out[i] = near && seg_normals_join(na[3 * i], na[3 * i + 1], na[3 * i + 2], nb[3 * i], nb[3 * i + 1], nb[3 * i + 2], cos_t) ? 1 : 0;
  }
}

// out[i] = seg_seed_key of point i against q
void seed_keys(int n, const float* xyz, const float* q, unsigned long long* out) {
  for (int i = 0; i < n; i++) {
    const float4 p = {xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], 0.f};
    out[i] = seg_seed_key(p, q[0], q[1], q[2], i);
  }
}

// out (n x 3) = R (row-major 9) applied to the fp32 normals
void rotate_normals(int n, const double* R, const float* nrm, float* out) {
  for (int i = 0; i < n; i++) seg_rotate_normal(R, nrm[3 * i], nrm[3 * i + 1], nrm[3 * i + 2], out + 3 * i);
}

// out[i] = seg_in_window of fp64 q_i
void in_window(int n, const double* q, double inv, const int* lo, const int* hi, int* out) {
  for (int i = 0; i < n; i++) out[i] = seg_in_window(q + 3 * i, inv, lo, hi) ? 1 : 0;
}

// the union-find of k_rg_init / k_rg_hook / k_rg_label run sequentially: every parent its own index, each edge (m x 2)
// hooked in the given order, then every label found
void union_find(int n, int m, const int* edges, int* parent, int* labels) {
  for (int i = 0; i < n; i++) parent[i] = i;
  for (int e = 0; e < m; e++) seg_hook(parent, edges[2 * e], edges[2 * e + 1]);
  for (int i = 0; i < n; i++) labels[i] = seg_find(parent, i);
}

}  // extern "C"
