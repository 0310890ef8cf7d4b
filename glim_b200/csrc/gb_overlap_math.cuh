// gb_overlap_math.cuh -- the candidate enumeration, relative pose and distance gate of gb_find_overlapping_submaps
// (gb_overlap_search.cu), and the work-item lookup of k_overlap (gb_kernels_vgicp.cu).  Like gb_cov_math.cuh it holds nothing
// that only exists on the device, so the SAME TEXT compiles for the host: tests/cpp/overlap_math_host.cpp builds it with g++ -ffp-contract=off and tests/test_overlap_search_host.py checks it
// bit for bit against a numpy restatement.  The rule is written once, in include/glim_b200.h (gb_find_overlapping_submaps).
//
// Every fp64 multiply and add is an explicit round-to-nearest operation summed in index order, so nvcc cannot contract it
// into an FMA and the device, the host build and numpy agree to the bit.
#pragma once
#include "gb_cov_math.cuh"  // GB_CHD, dot3, the fp64 intrinsics' host shims

namespace {

// The candidate slots of S submaps with first source f (0 <= f < S): row i holds the pairs (i, j) with
// max(i + 1, f) <= j < S, rows in ascending i, so slot order is lexicographic (i, j) order.  The first slot of row i (i <= S):
// rows r < min(i, f) hold S - f pairs each, rows f <= r < i hold S - 1 - r.  overlap_row_begin(S, f, S) is the slot count.
GB_CHD long long overlap_row_begin(long long S, long long f, long long i) {
  const long long a = i < f ? i : f;
  long long k = a * (S - f);
  if (i > f) k += (i - f) * (S - 1) - (i - f) * (i + f - 1) / 2;  // sum over r in [f, i) of S - 1 - r
  return k;
}

// The pair (i, j) of slot k < overlap_row_begin(S, f, S): the last row i <= S - 2 that begins at or before k (every row
// below S - 1 holds at least one pair).
GB_CHD void overlap_slot_pair(long long S, long long f, long long k, int& i, int& j) {
  long long lo = 0, hi = S - 2;
  while (lo < hi) {
    const long long mid = (lo + hi + 1) / 2;
    if (overlap_row_begin(S, f, mid) <= k) lo = mid; else hi = mid - 1;
  }
  const long long j0 = lo + 1 > f ? lo + 1 : f;
  i = (int)lo;
  j = (int)(j0 + (k - overlap_row_begin(S, f, lo)));
}

// delta = T_i^-1 T_j (16 doubles, column-major, as Eigen's Isometry3d::inverse() * T): R = R_i^T R_j and
// t = R_i^T t_j + (-(R_i^T t_i)), every dot product ((a0 b0 + a1 b1) + a2 b2).  overlap_delta_entry gives R(r, c) for c < 3
// and t(r) for c = 3; overlap_delta writes the whole pose and returns whether the pair passes the distance gate
// (t0 t0 + t1 t1) + t2 t2 <= max_distance2.
GB_CHD double overlap_delta_entry(const double* Ti, const double* Tj, int r, int c) {
  // column r of R_i is row r of R_i^T
  return c < 3 ? dot3(Ti + 4 * r, Tj + 4 * c) : __dadd_rn(dot3(Ti + 4 * r, Tj + 12), -dot3(Ti + 4 * r, Ti + 12));
}
GB_CHD bool overlap_delta(const double* Ti, const double* Tj, double max_distance2, double* D) {
  double t[3];
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) D[c * 4 + r] = overlap_delta_entry(Ti, Tj, r, c);
    D[r * 4 + 3] = 0.0;
    t[r] = overlap_delta_entry(Ti, Tj, r, 3);
    D[12 + r] = t[r];
  }
  D[15] = 1.0;
  return dot3(t, t) <= max_distance2;
}

// k_overlap's work items are (query, chunk of kOverlapChunk consecutive source points), numbered query-major: query q owns
// the items [item_end[q - 1], item_end[q]), item_end the inclusive scan of the chunk counts.  Items are counted in 64 bits: a
// search over 4096 submaps of up to 2^30 points each can have more than 2^31 of them.
constexpr int kOverlapChunk = 256;
GB_CHD long long overlap_chunks(int n) { return ((long long)n + kOverlapChunk - 1) / kOverlapChunk; }
// The query of `item` (< item_end[nq - 1]): the first q >= lo with item_end[q] > item (lo: a query at or before it).
GB_CHD int overlap_item_query(const long long* item_end, int nq, int lo, long long item) {
  int hi = nq - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (item_end[mid] > item) hi = mid; else lo = mid + 1;
  }
  return lo;
}
// The first source point of `item` of query q: a point index of the query's own cloud, below 2^30.
GB_CHD int overlap_item_point(const long long* item_end, int q, long long item) {
  return (int)((item - (q ? item_end[q - 1] : 0)) * kOverlapChunk);
}

}  // namespace
