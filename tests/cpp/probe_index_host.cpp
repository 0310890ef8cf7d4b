// Host build of glim_b200/csrc/gb_probe_index.cuh (tests/test_probe_index_host.py, scripts/probe_stats.py --index): the probe
// index of a voxel table built by the same text k_table_finalize runs, and looked up as k_vgicp_sweep3 looks it up.  The voxels
// are inserted one at a time in ascending voxel index (the table the device's concurrent insertion must converge to), or, to
// check that convergence, in a shuffled order by several threads with atomic compare-and-swap and or, as the device does.
#include "../../glim_b200/csrc/gb_probe_index.cuh"

#include <algorithm>
#include <climits>
#include <random>
#include <thread>
#include <vector>

extern "C" {

// The index of a table of nb buckets ({x, y, z, voxel}, voxel -1 = empty) over V voxels (vcoord: V x {x, y, z, points}, the
// box is reduced over all of them, as k_table_insert does): slots (2 (nb >> kPiSetShift) entries) and box (x y z ex ey ez).
// threads = 0: sequential insertion in ascending voxel index; else that many threads insert the voxels in an order shuffled
// by seed.  Returns whether the map gets an index (table_build's rule); the slots are filled only then.
int pih_build(const int* buckets, int nb, const int* vcoord, int V, unsigned long long* slots, int* box, int threads, unsigned seed) {
  int mm[6] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
  for (int v = 0; v < V; v++)
    for (int k = 0; k < 3; k++) {
      mm[k] = vcoord[4 * v + k] < mm[k] ? vcoord[4 * v + k] : mm[k];
      mm[3 + k] = vcoord[4 * v + k] > mm[3 + k] ? vcoord[4 * v + k] : mm[3 + k];
    }
  PiBox B;
  const bool fits = pi_box(mm, V, B);
  box[0] = B.x; box[1] = B.y; box[2] = B.z;
  box[3] = (int)B.ex; box[4] = (int)B.ey; box[5] = (int)B.ez;
  const int ns = nb >> kPiSetShift;
  for (int i = 0; i < 2 * ns; i++) slots[i] = kPiEmpty;
  if (!fits || ns == 0) return 0;
  std::vector<int> order;  // the voxels the table holds, in ascending index
  std::vector<int> at(V, -1);  // the bucket of each voxel the table holds
  for (int i = 0; i < nb; i++)
    if (buckets[4 * i + 3] >= 0) at[buckets[4 * i + 3]] = i;
  for (int v = 0; v < V; v++)
    if (at[v] >= 0) order.push_back(v);
  auto insert = [&](int v, auto&& cas, auto&& mark) {
    const int* b = buckets + 4 * at[v];
    pi_insert(B, (uint32_t)ns - 1u, v, b[0], b[1], b[2], cas, mark);
  };
  if (threads <= 0) {
    auto cas = [&](uint32_t k, unsigned long long expected, unsigned long long desired) {
      const unsigned long long prev = slots[k];
      if (prev == expected) slots[k] = desired;
      return prev;
    };
    auto mark = [&](uint32_t k) { slots[k] |= 1ull; };
    for (int v : order) insert(v, cas, mark);
    return 1;
  }
  std::shuffle(order.begin(), order.end(), std::mt19937(seed));
  auto cas = [&](uint32_t k, unsigned long long expected, unsigned long long desired) {
    __atomic_compare_exchange_n(&slots[k], &expected, desired, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
    return expected;  // the previous value, as atomicCAS returns it
  };
  auto mark = [&](uint32_t k) { __atomic_fetch_or(&slots[k], 1ull, __ATOMIC_SEQ_CST); };
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; t++)
    pool.emplace_back([&, t] {
      for (size_t i = (size_t)t; i < order.size(); i += (size_t)threads) insert(order[i], cas, mark);
    });
  for (auto& th : pool) th.join();
  return 1;
}

// per coordinate (xyz: n x 3): the index's answer and its dependent set gathers (rounds may be null)
void pih_lookup(const unsigned long long* slots, int nb, const int* box, int n, const int* xyz, int* out, int* rounds) {
  const PiBox B{box[0], box[1], box[2], (unsigned)box[3], (unsigned)box[4], (unsigned)box[5]};
  const uint4* sets = reinterpret_cast<const uint4*>(slots);
  const uint32_t set_mask = (uint32_t)(nb >> kPiSetShift) - 1u;
  for (int i = 0; i < n; i++) out[i] = pi_lookup(sets, set_mask, B, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], rounds ? rounds + i : nullptr);
}

// per coordinate: gb_lookup's answer on the bucket table
void pih_gb_lookup(const int* buckets, int nb, int max_scan, int n, const int* xyz, int* out) {
  const int4* b = reinterpret_cast<const int4*>(buckets);
  for (int i = 0; i < n; i++) out[i] = gb_lookup(b, (uint32_t)nb - 1u, max_scan, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
}

}  // extern "C"
