// gb_overlap_search.cu -- gb_find_overlapping_submaps: GlobalMapping::find_overlapping_submaps and the overlap test of
// GlobalMapping::create_matching_cost_factors (src/glim/mapping/global_mapping.cpp:285-351, :441-453) over every candidate pair
// of a global map in one call.  The rule is written once in include/glim_b200.h; the candidate enumeration, the relative pose
// and the gate are gb_overlap_math.cuh (also compiled for the host by the CPU test), and the counting is k_overlap
// (gb_kernels_vgicp.cu), the kernel of gb_overlap, with one query per candidate.
//
// Eight launches, whatever the number of submaps and candidates:
//   k_overlap_candidates   one thread per candidate slot: exclusion bit, relative pose, distance gate -> flag
//   cub Select::Flagged    the gated slots, in slot (= lexicographic) order
//   k_overlap_queries      one thread per gated pair: its query and its chunk count; zeroes its count
//   cub InclusiveSum       the chunk counts -> item_end (64-bit: the items of a large search exceed 2^31)
//   k_overlap              the hits of every query, each under the relative pose of its pair
//   k_overlap_threshold    overlap = count / n, flag = overlap >= min_overlap
//   cub Select::Flagged    the pairs found, in candidate order
//   k_overlap_emit         their (i, j) and overlaps, packed for the download
#include "gb_internal.cuh"
#include "gb_overlap_math.cuh"

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <algorithm>
#include <cmath>
#include <cstring>

namespace {

constexpr int kSlotThreads = 256;

// flags[k] = slot k's pair (i, j) has no bit i * S + j in `existing` and passes the distance gate
__global__ void __launch_bounds__(kSlotThreads) k_overlap_candidates(int S, int f, int N, const double* __restrict__ T, const unsigned* __restrict__ existing,
                                                                     double max_distance2, int* __restrict__ flags) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= N) return;
  int i, j;
  overlap_slot_pair(S, f, k, i, j);
  const long long bit = (long long)i * S + j;
  bool keep = !((existing[bit >> 5] >> (bit & 31)) & 1u);
  if (keep) {
    double D[16];
    keep = overlap_delta(T + 16 * (size_t)i, T + 16 * (size_t)j, max_distance2, D);
  }
  flags[k] = keep ? 1 : 0;
}

// gated pair q < *num (slot slots[q]): its query (source j, target i, the relative pose of the world poses), its chunk count and
// a zero count; chunks[q] = 0 for the slots beyond, so that the scan's tail repeats the total
__global__ void __launch_bounds__(kSlotThreads) k_overlap_queries(int S, int f, int N, const FactorDesc* __restrict__ descs, const int* __restrict__ num,
                                                                  const int* __restrict__ slots, OverlapQuery* __restrict__ queries, long long* __restrict__ chunks,
                                                                  int* __restrict__ counts) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= N) return;
  if (q >= *num) {
    chunks[q] = 0;
    return;
  }
  int i, j;
  overlap_slot_pair(S, f, slots[q], i, j);
  queries[q] = OverlapQuery{j, i, -1, 1};
  chunks[q] = overlap_chunks(descs[j].n);
  counts[q] = 0;
}

// overlap = count / n as gb_overlap divides it (0 for an empty source); flags[q] = overlap >= min_overlap (0 beyond *num)
__global__ void __launch_bounds__(kSlotThreads) k_overlap_threshold(int N, const int* __restrict__ num, const OverlapQuery* __restrict__ queries,
                                                                    const FactorDesc* __restrict__ descs, const int* __restrict__ counts, double min_overlap,
                                                                    double* __restrict__ overlaps, int* __restrict__ flags) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= N) return;
  if (q >= *num) {
    flags[q] = 0;
    return;
  }
  const int n = descs[queries[q].source].n;
  const double ov = n > 0 ? __ddiv_rn((double)counts[q], (double)n) : 0.0;
  overlaps[q] = ov;
  flags[q] = ov >= min_overlap ? 1 : 0;
}

// result r < *found: the pair and overlap of query sel[r]
__global__ void __launch_bounds__(kSlotThreads) k_overlap_emit(int N, const int* __restrict__ found, const int* __restrict__ sel, const OverlapQuery* __restrict__ queries,
                                                               const double* __restrict__ overlaps, int2* __restrict__ pairs, double* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= N || r >= *found) return;
  const int q = sel[r];
  pairs[r] = make_int2(queries[q].target, queries[q].source);
  out[r] = overlaps[q];
}

}  // namespace

extern "C" gb_status gb_find_overlapping_submaps(gb_ctx* ctx, size_t S, const gb_voxelmap* const* maps, const gb_cloud* const* sources, const double* T_world_submap,
                                                 size_t first_source, size_t E, const int32_t* existing, double max_distance, double min_overlap, size_t capacity,
                                                 size_t* num_found, int32_t* pairs, double* overlaps) {
  if (num_found) *num_found = 0;
  GB_REQUIRE(ctx, "null ctx");
  GB_REQUIRE(num_found, "null num_found");
  GB_REQUIRE(maps, "null maps");
  GB_REQUIRE(sources, "null sources");
  GB_REQUIRE(T_world_submap, "null T_world_submap");
  GB_REQUIRE(S >= 1 && S <= GB_OVERLAP_SEARCH_MAX_SUBMAPS, "num_submaps must be in [1, GB_OVERLAP_SEARCH_MAX_SUBMAPS]");
  GB_REQUIRE(first_source < S, "first_source must be below num_submaps");
  GB_REQUIRE(gb_all_finite(T_world_submap, 16 * S), "T_world_submap must be finite");
  GB_REQUIRE(std::isfinite(max_distance) && max_distance >= 0.0, "max_distance must be finite and >= 0");
  GB_REQUIRE(std::isfinite(min_overlap), "min_overlap must be finite");
  GB_REQUIRE(E == 0 || existing, "null existing");
  for (size_t e = 0; e < 2 * E; e++) GB_REQUIRE(existing[e] >= 0 && (size_t)existing[e] < S, "existing keys must be in [0, num_submaps)");
  GB_REQUIRE(capacity == 0 || (pairs && overlaps), "null pairs / overlaps with capacity > 0");
  for (size_t k = 0; k < S; k++) {
    GB_REQUIRE(maps[k], "null entry of maps");
    GB_REQUIRE(sources[k], "null entry of sources");
    GB_REQUIRE(maps[k]->kind != GB_MAP_POINTS, "maps: a point grid is not an occupancy target");
    GB_REQUIRE(maps[k]->device == ctx->device && sources[k]->device == ctx->device, "maps / sources on another device than ctx");
  }
  const int N = (int)((S * (S - 1) - first_source * (first_source - 1)) / 2);  // overlap_row_begin(S, first_source, S)
  if (N == 0) return GB_OK;  // one submap: no pair
  const double md2 = max_distance * max_distance;
  GB_ENTER(ctx);

  const size_t words = (S * S + 31) / 32;  // the exclusion bitmap: bit i * S + j
  size_t cub_b = 0, select_b = 0;
  cub::DeviceSelect::Flagged(nullptr, select_b, thrust::counting_iterator<int>(0), (const int*)nullptr, (int*)nullptr, (int*)nullptr, N);
  cub::DeviceScan::InclusiveSum(nullptr, cub_b, (const long long*)nullptr, (long long*)nullptr, N);
  cub_b = std::max(cub_b, select_b);
  struct Host { FactorDesc* descs; unsigned* bits; int* found; } h;
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) {
    h.descs = cv.take<FactorDesc>(S);
    h.bits = cv.take<unsigned>(words);
    h.found = cv.take<int>(1);
  }));
  struct Dev {
    FactorDesc* descs; double* T; unsigned* bits;
    int* flags; int* slots; int* num;  // num: gated pairs, pairs found
    OverlapQuery* queries; long long* chunks; long long* item_end; int* counts; double* ov;
    int2* pairs; double* out; void* cub;
  } d;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    d.descs = cv.take<FactorDesc>(S);
    d.T = cv.take<double>(16 * S);
    d.bits = cv.take<unsigned>(words);
    d.flags = cv.take<int>(N);
    d.slots = cv.take<int>(N);  // the gated slots, then the selected queries
    d.num = cv.take<int>(2);
    d.queries = cv.take<OverlapQuery>(N);
    d.chunks = cv.take<long long>(N);
    d.item_end = cv.take<long long>(N);
    d.counts = cv.take<int>(N);
    d.ov = cv.take<double>(N);
    d.pairs = cv.take<int2>(N);
    d.out = cv.take<double>(N);
    d.cub = cv.take<char>(cub_b);
  }));
  for (size_t k = 0; k < S; k++) {
    FactorDesc& D = h.descs[k];
    memset(&D, 0, sizeof(D));
    D.p0 = sources[k]->p0; D.p1 = sources[k]->p1; D.p2 = sources[k]->p2;
    D.n = (int)sources[k]->n;
    desc_target(D, maps[k]);
  }
  memset(h.bits, 0, words * sizeof(unsigned));
  for (size_t e = 0; e < E; e++) {
    const size_t bit = (size_t)existing[2 * e] * S + (size_t)existing[2 * e + 1];
    h.bits[bit >> 5] |= 1u << (bit & 31);
  }
  GB_CHECK(gb_upload(ctx, {{d.descs, h.descs, S * sizeof(FactorDesc)}, {d.T, T_world_submap, 16 * S * sizeof(double)}, {d.bits, h.bits, words * sizeof(unsigned)}}));

  const int blocks = (N + kSlotThreads - 1) / kSlotThreads, Si = (int)S, f = (int)first_source;
  GB_CHECK(gb_launch(ctx, "k_overlap_candidates", k_overlap_candidates, blocks, kSlotThreads, 0, Si, f, N, d.T, d.bits, md2, d.flags));
  GB_CUB(ctx, cub::DeviceSelect::Flagged, d.cub, cub_b, thrust::counting_iterator<int>(0), d.flags, d.slots, d.num, N);
  GB_CHECK(gb_launch(ctx, "k_overlap_queries", k_overlap_queries, blocks, kSlotThreads, 0, Si, f, N, d.descs, d.num, d.slots, d.queries, d.chunks, d.counts));
  GB_CUB(ctx, cub::DeviceScan::InclusiveSum, d.cub, cub_b, d.chunks, d.item_end, N);
  GB_CHECK(gb_launch_overlap(ctx, ctx->num_sms * 8, 1, d.queries, d.num, d.item_end, d.descs, nullptr, d.T, d.counts));
  GB_CHECK(gb_launch(ctx, "k_overlap_threshold", k_overlap_threshold, blocks, kSlotThreads, 0, N, d.num, d.queries, d.descs, d.counts, min_overlap, d.ov, d.flags));
  GB_CUB(ctx, cub::DeviceSelect::Flagged, d.cub, cub_b, thrust::counting_iterator<int>(0), d.flags, d.slots, d.num + 1, N);
  GB_CHECK(gb_launch(ctx, "k_overlap_emit", k_overlap_emit, blocks, kSlotThreads, 0, N, d.num + 1, d.slots, d.queries, d.ov, d.pairs, d.out));

  GB_CHECK(gb_download(ctx, {{h.found, d.num + 1, sizeof(int)}}));
  *num_found = (size_t)*h.found;
  const size_t m = std::min(*num_found, capacity);
  if (m > 0) GB_CHECK(gb_download(ctx, {{pairs, d.pairs, m * sizeof(int2)}, {overlaps, d.out, m * sizeof(double)}}));
  return GB_OK;
}
