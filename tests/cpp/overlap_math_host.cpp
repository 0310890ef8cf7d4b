// Host build of the candidate enumeration, relative pose and gate of gb_find_overlapping_submaps
// (glim_b200/csrc/gb_overlap_math.cuh, the text the kernels of gb_overlap_search.cu compile): tests/test_overlap_search_host.py
// compiles this with g++ -ffp-contract=off and compares it with a numpy restatement.
#include "../../glim_b200/csrc/gb_overlap_math.cuh"

extern "C" {

// the candidate slot count of S submaps with first source f
long long om_num_slots(long long S, long long f) { return overlap_row_begin(S, f, S); }

// the pairs of slots k0 .. k0 + count - 1 (count x 2)
void om_pairs(long long S, long long f, long long k0, long long count, int* ij) {
  for (long long k = 0; k < count; k++) overlap_slot_pair(S, f, k0 + k, ij[2 * k], ij[2 * k + 1]);
}

// chunk counts of n source-cloud sizes
void om_chunks(int n, const int* sizes, long long* chunks) {
  for (int k = 0; k < n; k++) chunks[k] = overlap_chunks(sizes[k]);
}

// the query and first point of m items over nq queries (item_end: the inclusive scan of their chunk counts), as k_overlap
// looks them up: `lo` from the previous item, items ascending
void om_items(const long long* item_end, int nq, int m, const long long* items, int* query, int* point) {
  int lo = 0;
  for (int k = 0; k < m; k++) {
    lo = overlap_item_query(item_end, nq, lo, items[k]);
    query[k] = lo;
    point[k] = overlap_item_point(item_end, lo, items[k]);
  }
}

// delta (16, column-major) and gate of n pose pairs (n x 16 each, column-major)
void om_deltas(int n, const double* Ti, const double* Tj, double max_distance2, double* D, int* gate) {
  for (int k = 0; k < n; k++) gate[k] = overlap_delta(Ti + 16 * k, Tj + 16 * k, max_distance2, D + 16 * k) ? 1 : 0;
}

}
