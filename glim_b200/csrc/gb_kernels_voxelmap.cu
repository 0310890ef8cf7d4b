// gb_kernels_voxelmap.cu -- deterministic GPU build of the Gaussian voxel map (sm_90a).
//
// Replaces gtsam_points::GaussianVoxelMapGPU(resolution, 8192*2, 10, 1e-3, stream)::insert(cloud)
// (GLIM call sites: src/glim/odometry/odometry_estimation_gpu.cpp:103-104; src/glim/mapping/sub_mapping.cpp:398-399;
// src/glim/mapping/global_mapping.cpp:265-266).  Spec: SURVEY.md Appendix B; oracle: go_gpumap_build
// (oracle/glim_oracle.c) -- results are bit-exact with it (coordinates, voxel numbering, bucket
// placement, fp32 means / covariances).
//
// The reference inserts with atomicCAS, which makes bucket placement, voxel numbering and the
// fp32 atomic sums depend on thread timing.  Here the build is a deterministic pipeline:
//   1. k_point_keys      coord = floorf(p * inv_res) -> packed 63-bit key per point
//   2. radix sort        (key, point index) pairs, stable  [cub::DeviceRadixSort -- CUDA toolkit]
//   3. k_head_flags + inclusive scan -> voxel id per sorted slot; voxel v = v-th smallest key
//   4. k_voxel_reduce    one thread per voxel sums its points IN POINT ORDER in fp32, then / n
//                        (voxel covariance = mean of the member points' covariances, B.3)
//   5. k_table_insert    all voxels inserted concurrently with atomicMin-priority linear probing:
//                        a slot always ends up with the smallest voxel id that probed it, the loser
//                        moves on -- the fixed point is exactly the table a sequential first-free-slot
//                        insertion in ascending voxel id builds (Shun & Blelloch's phase-concurrent
//                        deterministic hashing), including which voxels run out of probes (<= max_scan)
//   6. host loop         num_buckets = init doubled until >= 8 V (load factor <= 1/8), then doubled again while
//                        dropped points > drop_rate * N
// Steps 2-3 (+ k_voxel_starts) are gb_group_by_key / gb_group_starts, shared with the voxel-grid downsampling and the frame
// merge of gb_kernels_preprocess.cu; the hash thinning of those paths and of the map insert (gb_thin) sits next to them.
// Steps 1-3 with the voxel count are group_cloud, shared with the point grid.  Step 6 (table_build) also serves the
// incremental maps and iVoxes, whose one insert pipeline is described below.  The map entry points (gb_voxelmap_*, gb_ivox_*) are defined here too.  This file also builds
// every device cloud (gb_cloud_build: Morton reorder of staged planes), for gb_cloud_upload, gb_preprocess and gb_merge_frames.
#include "gb_internal.cuh"

#include <cub/cub.cuh>

#include <cmath>
#include <cstring>
#include <new>
#include <vector>

namespace {

constexpr int kEmpty = 0x7fffffff;

// i runs over ORIGINAL point indices (so that voxel sums are accumulated in the caller's point order, like the oracle);
// inv_perm maps them to the Morton-ordered storage
__global__ void k_point_keys(int n, const float4* __restrict__ p0, const int* __restrict__ inv_perm, float inv_res, unsigned long long* __restrict__ keys, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 a = __ldg(&p0[inv_perm ? inv_perm[i] : i]);
  unsigned long long key = kInvalidKey;
  if (isfinite(a.x) && isfinite(a.y) && isfinite(a.z)) {
    unsigned long long k;
    if (gb_pack_key(gb_coord(a.x, inv_res), gb_coord(a.y, inv_res), gb_coord(a.z, inv_res), &k)) key = k;
  }
  keys[i] = key;
  idx[i] = i;
}

__global__ void k_head_flags(int n, const unsigned long long* __restrict__ keys, int* __restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  flags[i] = (k != kInvalidKey && (i == 0 || keys[i - 1] != k)) ? 1 : 0;
}

// starts[v] = first sorted slot of voxel v; starts[V] = number of valid points
__global__ void k_voxel_starts(int n, const unsigned long long* __restrict__ keys, const int* __restrict__ flags, const int* __restrict__ pos, int* __restrict__ starts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (flags[i]) starts[pos[i] - 1] = i;
  const bool valid = keys[i] != kInvalidKey;
  const bool next_valid = (i + 1 < n) && keys[i + 1] != kInvalidKey;
  if (valid && !next_valid) starts[pos[i]] = i + 1;
}

// the candidates of gb_thin: i with cand[i] != 0 (when given) and i < *count (when given)
__device__ __forceinline__ bool thin_candidate(int i, const int* cand, const int* count) { return (!cand || cand[i]) && (!count || i < *count); }
__global__ void k_thin_hash(int n, const int* __restrict__ cand, const int* __restrict__ count, unsigned long long seed, unsigned long long* __restrict__ hash) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) hash[i] = thin_candidate(i, cand, count) ? rg_hash(seed, (unsigned)i) : ~0ull;
}
// rg_hash is a bijection of the index for a fixed seed, so exactly the m smallest candidate hashes are <= sorted[m - 1]
// (cand and keep may be the same array)
__global__ void k_thin_keep(int n, const int* cand, const int* __restrict__ count, int m, unsigned long long seed, const unsigned long long* __restrict__ sorted, int* keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = count ? *count : n;
  keep[i] = thin_candidate(i, cand, count) && (m <= 0 || m >= c || rg_hash(seed, (unsigned)i) <= sorted[m - 1]);
}

__global__ void k_voxel_reduce(int V, const int* __restrict__ starts, const unsigned long long* __restrict__ keys, const int* __restrict__ idx,
                               const float4* __restrict__ p0, const float4* __restrict__ p1, const float* __restrict__ p2, const int* __restrict__ inv_perm,
                               float4* __restrict__ voxels, int4* __restrict__ vcoord) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int b = starts[v], e = starts[v + 1];
  float sx = 0.f, sy = 0.f, sz = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f, c4 = 0.f, c5 = 0.f;
  for (int s = b; s < e; s++) {
    const int i = inv_perm ? inv_perm[idx[s]] : idx[s];
    const float4 a0 = __ldg(&p0[i]);
    const float4 a1 = __ldg(&p1[i]);
    const float a2 = __ldg(&p2[i]);
    sx += a0.x; sy += a0.y; sz += a0.z;
    c0 += a0.w; c1 += a1.x; c2 += a1.y; c3 += a1.z; c4 += a1.w; c5 += a2;
  }
  const int cnt = e - b;
  const float fn = (float)cnt;
  voxels[3 * (size_t)v + 0] = make_float4(sx / fn, sy / fn, sz / fn, c0 / fn);
  voxels[3 * (size_t)v + 1] = make_float4(c1 / fn, c2 / fn, c3 / fn, c4 / fn);
  voxels[3 * (size_t)v + 2] = make_float4(c5 / fn, fn, 0.f, 0.f);
  int x, y, z;
  gb_unpack_key(keys[b], x, y, z);
  vcoord[v] = make_int4(x, y, z, cnt);
}

__global__ void k_table_clear(int nb, int4* __restrict__ buckets) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nb) buckets[i] = make_int4(0, 0, 0, kEmpty);
}

__global__ void k_table_insert(int V, const int4* __restrict__ vcoord, int4* __restrict__ buckets, uint32_t mask, int max_scan, int* __restrict__ dropped_points) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  int cur = v;
  int4 c = vcoord[cur];
  uint32_t s = gb_hash(c.x, c.y, c.z) & mask;
  int dist = 0;
  for (;;) {
    if (dist >= max_scan) { atomicAdd(dropped_points, c.w); break; }
    const int old = atomicMin(&buckets[s].w, cur);
    if (old == kEmpty) break;
    if (old > cur) {  // took the slot from a lower-priority voxel: carry it onward
      cur = old;
      c = vcoord[cur];
      const uint32_t home = gb_hash(c.x, c.y, c.z) & mask;
      dist = (int)((s - home) & mask) + 1;
    } else {
      dist++;
    }
    s = (s + 1u) & mask;
  }
}

__global__ void k_table_finalize(int nb, const int4* __restrict__ vcoord, int4* __restrict__ buckets) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nb) return;
  const int w = buckets[i].w;
  if (w == kEmpty) {
    buckets[i] = make_int4(0, 0, 0, -1);
  } else {
    const int4 c = vcoord[w];
    buckets[i] = make_int4(c.x, c.y, c.z, w);
  }
}

}  // namespace

gb_status gb_group_by_key(gb_ctx* ctx, int n, const gb_sort_tmp& t, int* flags, int* pos) {
  GB_CUB(ctx, cub::DeviceRadixSort::SortPairs, t.cub, t.cub_bytes, t.keys, t.keys_s, t.idx, t.idx_s, n, 0, 64);
  GB_CHECK(gb_launch(ctx, "k_head_flags", k_head_flags, (n + 255) / 256, 256, 0, n, t.keys_s, flags));
  GB_CUB(ctx, cub::DeviceScan::InclusiveSum, t.cub, t.cub_bytes, flags, pos, n);
  return GB_OK;
}

gb_status gb_group_starts(gb_ctx* ctx, int n, const gb_sort_tmp& t, const int* flags, const int* pos, int* starts) {
  return gb_launch(ctx, "k_voxel_starts", k_voxel_starts, (n + 255) / 256, 256, 0, n, t.keys_s, flags, pos, starts);
}

gb_status gb_thin(gb_ctx* ctx, int n, const int* cand, const int* count, int m, unsigned long long seed, const gb_sort_tmp& t, int* keep) {
  const int blocks = (n + 255) / 256;
  GB_CHECK(gb_launch(ctx, "k_thin_hash", k_thin_hash, blocks, 256, 0, n, cand, count, seed, t.keys));
  GB_CUB(ctx, cub::DeviceRadixSort::SortKeys, t.cub, t.cub_bytes, t.keys, t.keys_s, n, 0, 64);
  return gb_launch(ctx, "k_thin_keep", k_thin_keep, blocks, 256, 0, n, cand, count, m, seed, t.keys_s, keep);
}

// The hash table of V voxels (vcoord[v] = {x, y, z, points}; d_dropped: one int of scratch, unused when V = 0): num_buckets =
// init_buckets doubled until >= 8 V, then doubled again while more than drop_rate * total_points points fall out of it.
// One host synchronisation per attempt.  A rejected attempt's table goes back to the pool before the next one is taken.
static gb_status table_build(gb_ctx* ctx, int V, const int4* d_vcoord, int* d_dropped, int init_buckets, int max_scan, double drop_rate, double total_points,
                             gb_dev_block& table, int* num_buckets, int* num_dropped_points) {
  cudaStream_t st = ctx->stream;
  int nb = init_buckets;
  while ((long long)nb < 8ll * V) nb *= 2;  // load factor <= 1/8: the XOR-of-primes hash clusters, and lookups that
                                                             // MISS (most of them in global mapping) walk until the first empty slot;
                                                             // same rule as the oracle
  for (;; nb *= 2) {
    gb_dev_block attempt(ctx->device);
    int4* buckets = nullptr;
    GB_CHECK(gb_dev_carve(ctx, attempt, [&](Carver& cv) { buckets = cv.take<int4>((size_t)nb); }));
    GB_CHECK(gb_launch(ctx, "k_table_clear", k_table_clear, (nb + 255) / 256, 256, 0, nb, buckets));
    int dropped = 0;
    if (V > 0) {
      GB_CUDA(cudaMemsetAsync(d_dropped, 0, sizeof(int), st));
      GB_CHECK(gb_launch(ctx, "k_table_insert", k_table_insert, (V + 255) / 256, 256, 0, V, d_vcoord, buckets, (uint32_t)nb - 1u, max_scan, d_dropped));
    }
    GB_CHECK(gb_launch(ctx, "k_table_finalize", k_table_finalize, (nb + 255) / 256, 256, 0, nb, d_vcoord, buckets));
    GB_CHECK(gb_download(ctx, {{&dropped, d_dropped, V > 0 ? sizeof(int) : 0}}));
    *num_buckets = nb;
    *num_dropped_points = dropped;
    if ((double)dropped <= drop_rate * total_points || nb >= (1 << 28)) {
      table = std::move(attempt);
      return GB_OK;
    }
  }
}

// The grouping of a cloud of n > 0 points by the build's fp32 key at inv_res, for the voxel-map build and the point grid: the
// scratch, k_point_keys and gb_group_by_key, then the group count V read back (one host synchronisation).  starts is left for
// gb_group_starts; vcoord and dropped are table_build's, extent the point grid's.
struct CloudGroups {
  gb_sort_tmp t;
  int *flags, *pos, *starts, *dropped, *extent;
  int4* vcoord;
  int V = 0;
};
static gb_status group_cloud(gb_ctx* ctx, const gb_cloud* cloud, float inv_res, CloudGroups& g) {
  const int n = (int)cloud->n;
  const size_t cub_b = gb_cub_temp_bytes(n);
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    g.t = gb_take_sort_tmp(cv, n, cv.take<char>(cub_b), cub_b);
    g.flags = cv.take<int>(n + 1);
    g.pos = cv.take<int>(n + 1);
    g.starts = cv.take<int>(n + 1);
    g.vcoord = cv.take<int4>(n);
    g.dropped = cv.take<int>(1);
    g.extent = cv.take<int>(1);
  }));
  GB_CHECK(gb_launch(ctx, "k_point_keys", k_point_keys, (n + 255) / 256, 256, 0, n, cloud->p0, cloud->inv_perm, inv_res, g.t.keys, g.t.idx));
  GB_CHECK(gb_group_by_key(ctx, n, g.t, g.flags, g.pos));
  return gb_download(ctx, {{&g.V, g.pos + (n - 1), sizeof(int)}});
}

// (the caller has made the map's device current)
static void voxelmap_free(gb_voxelmap* m) {
  gb_dev_free(m->device, m->base);
  gb_dev_free(m->device, m->buckets);
  delete m;
}

extern "C" gb_status gb_voxelmap_build(gb_ctx* ctx, const gb_cloud* cloud, float resolution, int init_num_buckets, int max_bucket_scan_count, double target_points_drop_rate, gb_voxelmap** out) {
  GB_REQUIRE(ctx && cloud && out, "null argument");
  GB_REQUIRE(resolution > 0.f, "resolution must be positive");
  GB_REQUIRE(init_num_buckets > 0 && (init_num_buckets & (init_num_buckets - 1)) == 0, "init_num_buckets must be a power of two");
  GB_REQUIRE(max_bucket_scan_count > 0, "max_bucket_scan_count must be positive");
  *out = nullptr;
  GB_ENTER(ctx);
  gb_owned<gb_voxelmap> m(new (std::nothrow) gb_voxelmap(), voxelmap_free);
  if (!m) return GB_ERR_INTERNAL;
  const int n = (int)cloud->n;
  m->device = ctx->device;
  m->resolution = resolution;
  m->inv_res = 1.0f / resolution;
  m->max_scan = max_bucket_scan_count;

  CloudGroups g{};
  gb_dev_block records(ctx->device), table(ctx->device);
  if (n > 0) {
    GB_CHECK(group_cloud(ctx, cloud, m->inv_res, g));
    if (g.V > 0) {
      GB_CHECK(gb_dev_carve(ctx, records, [&](Carver& cv) { m->voxels = cv.take<float4>(3 * (size_t)g.V); }));
      GB_CHECK(gb_group_starts(ctx, n, g.t, g.flags, g.pos, g.starts));
      GB_CHECK(gb_launch(ctx, "k_voxel_reduce", k_voxel_reduce, (g.V + 127) / 128, 128, 0, g.V, g.starts, g.t.keys_s, g.t.idx_s, cloud->p0, cloud->p1, cloud->p2, cloud->inv_perm,
                         m->voxels, g.vcoord));
    }
  }
  m->num_voxels = g.V;
  GB_CHECK(table_build(ctx, g.V, g.vcoord, g.dropped, init_num_buckets, max_bucket_scan_count, target_points_drop_rate, (double)n, table, &m->num_buckets,
                       &m->num_dropped_points));
  records.hand_over(m->base);
  table.hand_over(m->buckets);
  *out = m.release();
  return GB_OK;
}

// ---------------------------------------------------------------------------------------------
// Incremental maps and iVoxes (gb_voxelmap_insert / gb_ivox_insert; both rules are written once in include/glim_b200.h).
// One insert is one pass over (the map's stored entries, the frame's points), the same steps for both kinds:
//   1. old keys            the stored entries, tagged old (idx = -1 - entry), ahead of the points: one per voxel
//                          (k_ins_old_keys) or one per stored iVox point (k_ivox_old_keys)
//   2. k_merge_transform   (gb_transform_frames, shared with gb_merge_frames) q = R a + t, R C R^T in un-contracted fp64
//   3. k_grid_keys         (gb_grid_keys) packed floor(q * key_inv_res) in fp64; with sampling_rate < 1, gb_thin first keeps
//                          the m points with the smallest rg_hash(seed, index) and the others get no key
//   4. gb_group_by_key     stable: a voxel's group is its old entries first, then its new points in index order
//   5. merge               one thread per merged voxel: the kind's per-voxel rule, then the LRU eviction (the same
//                          expression in both merge kernels: a shared helper changes k_ivox_merge's SASS)
//                            incremental  stored sums + the new points one at a time, n, stamp (k_ins_merge, a scan, k_ins_count)
//                            iVox         the stored points, then the sequential admission of the new ones (k_ivox_merge,
//                                         two scans, k_ivox_count)
//   6. read back           surviving points and voxels
//   7. emit                the survivors, in ascending key order, into a new state block of the kind's layout (k_ins_emit:
//                          keys, n, stamps, sums, fp32 records; k_ivox_emit: point records, cells, keys, stamps)
//   8. table_build         the build's table kernels and sizing rule; an iVox has drop rate 0 and fails if a voxel is left out
// Two host synchronisations (survivor count; dropped points of each table attempt).  The new blocks stay in their owners until
// every step has succeeded; then they replace the map's, and the old blocks go back to the pool through gb_dev_free, which
// waits for every stream of the device: a sweep of another context still reading them is safe.
// ---------------------------------------------------------------------------------------------
namespace {

__global__ void k_ins_old_keys(int V, const unsigned long long* __restrict__ vkeys, unsigned long long* __restrict__ keys, int* __restrict__ idx) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  keys[v] = vkeys[v];
  idx[v] = -1 - v;
}

__global__ void k_ins_merge(int N, const int* __restrict__ num_merged, const int* __restrict__ starts, const int* __restrict__ idx_s,
                            const int* __restrict__ on, const int* __restrict__ ostamp, const double* __restrict__ osums,
                            const double4* __restrict__ pts, const double* __restrict__ cov6, int counter, int horizon, int cycle,
                            int* __restrict__ mn, int* __restrict__ mstamp, double* __restrict__ msums, int* __restrict__ keep, unsigned long long* __restrict__ total) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N) return;
  if (v >= *num_merged) { keep[v] = 0; return; }
  const int b = starts[v], e = starts[v + 1];
  double s[9];
  int cnt = 0, stamp = counter, first = b;
  const int i0 = idx_s[b];
  if (i0 < 0) {
    const int o = -1 - i0;
    for (int k = 0; k < 9; k++) s[k] = osums[9 * (size_t)o + k];
    cnt = on[o];
    stamp = ostamp[o];
    first = b + 1;
  } else {
    for (int k = 0; k < 9; k++) s[k] = 0.0;
  }
  for (int j = first; j < e; j++) {
    const int i = idx_s[j];
    const double4 p = pts[i];
    const double* c = cov6 + 6 * (size_t)i;
    s[0] += p.x; s[1] += p.y; s[2] += p.z;
    for (int k = 0; k < 6; k++) s[3 + k] += c[k];
  }
  if (e > first) { cnt += e - first; stamp = counter; }
  const int c1 = counter + 1;
  const bool evict = horizon > 0 && c1 % cycle == 0 && stamp + horizon < c1;
  keep[v] = evict ? 0 : 1;
  mn[v] = cnt;
  mstamp[v] = stamp;
  for (int k = 0; k < 9; k++) msums[9 * (size_t)v + k] = s[k];
  if (!evict) atomicAdd(total, (unsigned long long)cnt);
}
__global__ void k_ins_count(int N, const int* __restrict__ kpos, unsigned long long* __restrict__ kept) { *kept = (unsigned long long)kpos[N - 1]; }

__global__ void k_ins_emit(int N, const int* __restrict__ num_merged, const int* __restrict__ keep, const int* __restrict__ kpos, const int* __restrict__ starts,
                           const unsigned long long* __restrict__ keys_s, const int* __restrict__ mn, const int* __restrict__ mstamp, const double* __restrict__ msums,
                           unsigned long long* __restrict__ vkeys, int* __restrict__ vn, int* __restrict__ vstamp, double* __restrict__ vsums,
                           float4* __restrict__ voxels, int4* __restrict__ vcoord) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N || v >= *num_merged || !keep[v]) return;
  const int o = kpos[v] - 1;
  const unsigned long long key = keys_s[starts[v]];
  const int cnt = mn[v];
  double s[9];
  for (int k = 0; k < 9; k++) s[k] = msums[9 * (size_t)v + k];
  vkeys[o] = key;
  vn[o] = cnt;
  vstamp[o] = mstamp[v];
  for (int k = 0; k < 9; k++) vsums[9 * (size_t)o + k] = s[k];
  const double dn = (double)cnt;
  voxels[3 * (size_t)o + 0] = make_float4((float)(s[0] / dn), (float)(s[1] / dn), (float)(s[2] / dn), (float)(s[3] / dn));
  voxels[3 * (size_t)o + 1] = make_float4((float)(s[4] / dn), (float)(s[5] / dn), (float)(s[6] / dn), (float)(s[7] / dn));
  voxels[3 * (size_t)o + 2] = make_float4((float)(s[8] / dn), (float)cnt, 0.f, 0.f);
  int x, y, z;
  gb_unpack_key(key, x, y, z);
  vcoord[o] = make_int4(x, y, z, cnt);
}

__global__ void k_ivox_old_keys(int V, const unsigned long long* __restrict__ vkeys, const int2* __restrict__ cells, unsigned long long* __restrict__ keys, int* __restrict__ idx) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int2 c = cells[v];
  const unsigned long long key = vkeys[v];
  for (int s = 0; s < c.y; s++) {
    keys[c.x + s] = key;
    idx[c.x + s] = -1 - (c.x + s);
  }
}

// the fp32 position of a group entry: a stored record (ref < 0) or a new point
__device__ __forceinline__ float3 ivox_entry_pos(int ref, const float4* __restrict__ opoints, const double4* __restrict__ pts) {
  if (ref < 0) {
    const float4 p = opoints[3 * (size_t)(-1 - ref)];
    return make_float3(p.x, p.y, p.z);
  }
  const double4 q = pts[ref];
  return make_float3((float)q.x, (float)q.y, (float)q.z);
}

// mref[b .. b + mcount[v]) = the entries voxel v keeps (stored ones first, then the admitted new points in index order)
__global__ void k_ivox_merge(int N, const int* __restrict__ num_merged, const int* __restrict__ starts, const unsigned long long* __restrict__ keys_s, const int* __restrict__ idx_s,
                             int Vo, const unsigned long long* __restrict__ ovkeys, const int* __restrict__ ostamp, const float4* __restrict__ opoints,
                             const double4* __restrict__ pts, int max_points, double min_d2, int counter, int horizon, int cycle,
                             int* __restrict__ mref, int* __restrict__ mcount, int* __restrict__ mstamp, int* __restrict__ keep) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N) return;
  if (v >= *num_merged) { keep[v] = 0; mcount[v] = 0; return; }
  const int b = starts[v], e = starts[v + 1];
  int cnt = 0, stamp = counter;
  bool touched = false;
  if (idx_s[b] < 0) {  // a stored voxel: its stamp (the stored keys are ascending)
    const unsigned long long key = keys_s[b];
    int lo = 0, hi = Vo;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (ovkeys[mid] < key) lo = mid + 1; else hi = mid;
    }
    stamp = ostamp[lo];
  }
  for (int j = b; j < e; j++) {
    const int i = idx_s[j];
    if (i < 0) { mref[b + cnt++] = i; continue; }
    touched = true;
    if (cnt >= max_points) continue;
    const float3 a = ivox_entry_pos(i, opoints, pts);
    bool ok = true;
    for (int k = 0; k < cnt && ok; k++) {
      const float3 p = ivox_entry_pos(mref[b + k], opoints, pts);
      const double dx = (double)p.x - (double)a.x, dy = (double)p.y - (double)a.y, dz = (double)p.z - (double)a.z;
      const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
      ok = d2 >= min_d2;
    }
    if (ok) mref[b + cnt++] = i;
  }
  if (touched) stamp = counter;
  const int c1 = counter + 1;
  const bool evict = horizon > 0 && c1 % cycle == 0 && stamp + horizon < c1;
  keep[v] = evict ? 0 : 1;
  mcount[v] = evict ? 0 : cnt;
  mstamp[v] = stamp;
}
__global__ void k_ivox_count(int N, const int* __restrict__ kpos, const int* __restrict__ ppos, unsigned long long* __restrict__ info) {
  info[0] = (unsigned long long)ppos[N - 1];
  info[1] = (unsigned long long)kpos[N - 1];
}

__global__ void k_ivox_emit(int N, const int* __restrict__ num_merged, const int* __restrict__ keep, const int* __restrict__ kpos, const int* __restrict__ ppos,
                            const int* __restrict__ starts, const unsigned long long* __restrict__ keys_s, const int* __restrict__ mref, const int* __restrict__ mcount,
                            const int* __restrict__ mstamp, const float4* __restrict__ opoints, const double4* __restrict__ pts, const double* __restrict__ cov6,
                            unsigned long long* __restrict__ vkeys, int* __restrict__ vstamp, int2* __restrict__ cells, float4* __restrict__ points, int4* __restrict__ vcoord) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N || v >= *num_merged || !keep[v]) return;
  const int o = kpos[v] - 1;
  const int cnt = mcount[v];
  const int first = ppos[v] - cnt;
  const int b = starts[v];
  const unsigned long long key = keys_s[b];
  vkeys[o] = key;
  vstamp[o] = mstamp[v];
  cells[o] = make_int2(first, cnt);
  int x, y, z;
  gb_unpack_key(key, x, y, z);
  vcoord[o] = make_int4(x, y, z, cnt);
  for (int k = 0; k < cnt; k++) {
    const int ref = mref[b + k];
    float4* dst = points + 3 * (size_t)(first + k);
    if (ref < 0) {
      const float4* src = opoints + 3 * (size_t)(-1 - ref);
      dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
    } else {
      const double4 q = pts[ref];
      const double* c = cov6 + 6 * (size_t)ref;
      dst[0] = make_float4((float)q.x, (float)q.y, (float)q.z, (float)c[0]);
      dst[1] = make_float4((float)c[1], (float)c[2], (float)c[3], (float)c[4]);
      dst[2] = make_float4((float)c[5], 1.f, 0.f, 0.f);
    }
  }
}

// The scratch of steps 1-8 that both kinds use: the grouping of N entries, the frame's fp64 points and covariances, the
// survivors' table coordinates and the read-back {points in the surviving voxels, surviving voxels}.
struct InsertScratch {
  gb_sort_tmp t;
  int *flags, *pos, *starts, *keep, *kpos, *dropped;
  int4* vcoord;
  unsigned long long* info;
  gb_frame* frame;
  double4* pts = nullptr;
  double* cov = nullptr;
};

// The per-voxel part of an incremental map: one stored entry per voxel, whose fp64 sums the new points continue.
struct VoxelRule {
  const gb_voxelmap* m;
  int *mn, *mstamp;
  double* msums;
  void scratch(Carver& cv, size_t N) {
    mn = cv.take<int>(N);
    mstamp = cv.take<int>(N);
    msums = cv.take<double>(9 * N);
  }
  gb_status old_keys(gb_ctx* ctx, const gb_sort_tmp& t) const {
    const int Vo = m->num_voxels;
    return gb_launch(ctx, "k_ins_old_keys", k_ins_old_keys, (Vo + 255) / 256, 256, 0, Vo, m->vkeys, t.keys, t.idx);
  }
  gb_status merge(gb_ctx* ctx, const InsertScratch& s, int N) const {
    GB_CUDA(cudaMemsetAsync(s.info, 0, 2 * sizeof(unsigned long long), ctx->stream));  // k_ins_merge adds up info[0]
    GB_CHECK(gb_launch(ctx, "k_ins_merge", k_ins_merge, (N + 127) / 128, 128, 0, N, s.pos + (N - 1), s.starts, s.t.idx_s, m->vn, m->vstamp, m->vsums, s.pts, s.cov,
                       m->lru_counter, m->lru_horizon, m->lru_clear_cycle, mn, mstamp, msums, s.keep, s.info));
    GB_CUB(ctx, cub::DeviceScan::InclusiveSum, s.t.cub, s.t.cub_bytes, s.keep, s.kpos, N);
    return gb_launch(ctx, "k_ins_count", k_ins_count, 1, 1, 0, N, s.kpos, s.info + 1);
  }
  // the state block: fp32 records first (gb_voxelmap::voxels), then keys, counts, stamps and sums
  static void layout(Carver& cv, gb_voxelmap* next) {
    const size_t V = (size_t)next->num_voxels;
    next->voxels = cv.take<float4>(3 * V);
    next->vkeys = cv.take<unsigned long long>(V);
    next->vn = cv.take<int>(V);
    next->vstamp = cv.take<int>(V);
    next->vsums = cv.take<double>(9 * V);
  }
  gb_status emit(gb_ctx* ctx, const InsertScratch& s, int N, const gb_voxelmap& next) const {
    return gb_launch(ctx, "k_ins_emit", k_ins_emit, (N + 255) / 256, 256, 0, N, s.pos + (N - 1), s.keep, s.kpos, s.starts, s.t.keys_s, mn, mstamp, msums,
                     next.vkeys, next.vn, next.vstamp, next.vsums, next.voxels, s.vcoord);
  }
  gb_status check_table(const gb_voxelmap&) const { return GB_OK; }
};

// The per-voxel part of an iVox: one stored entry per stored point; a voxel keeps its points and admits new ones.
struct IvoxRule {
  const gb_voxelmap* m;
  int *ppos, *mcount, *mstamp, *mref;
  void scratch(Carver& cv, size_t N) {
    ppos = cv.take<int>(N + 1);
    mcount = cv.take<int>(N + 1);
    mstamp = cv.take<int>(N);
    mref = cv.take<int>(N);
  }
  gb_status old_keys(gb_ctx* ctx, const gb_sort_tmp& t) const {
    const int Vo = m->num_voxels;
    return gb_launch(ctx, "k_ivox_old_keys", k_ivox_old_keys, (Vo + 255) / 256, 256, 0, Vo, m->vkeys, m->cells, t.keys, t.idx);
  }
  gb_status merge(gb_ctx* ctx, const InsertScratch& s, int N) const {
    GB_CHECK(gb_launch(ctx, "k_ivox_merge", k_ivox_merge, (N + 127) / 128, 128, 0, N, s.pos + (N - 1), s.starts, s.t.keys_s, s.t.idx_s, m->num_voxels, m->vkeys, m->vstamp,
                       m->voxels, s.pts, m->max_points, m->min_dist * m->min_dist, m->lru_counter, m->lru_horizon, m->lru_clear_cycle, mref, mcount, mstamp, s.keep));
    GB_CUB(ctx, cub::DeviceScan::InclusiveSum, s.t.cub, s.t.cub_bytes, s.keep, s.kpos, N);
    GB_CUB(ctx, cub::DeviceScan::InclusiveSum, s.t.cub, s.t.cub_bytes, mcount, ppos, N);
    return gb_launch(ctx, "k_ivox_count", k_ivox_count, 1, 1, 0, N, s.kpos, ppos, s.info);
  }
  // the state block of V voxels and P points: point records first (gb_voxelmap::voxels), then cells, keys and stamps
  static void layout(Carver& cv, gb_voxelmap* next) {
    const size_t V = (size_t)next->num_voxels;
    next->voxels = cv.take<float4>(3 * next->num_points);
    next->cells = cv.take<int2>(V);
    next->vkeys = cv.take<unsigned long long>(V);
    next->vstamp = cv.take<int>(V);
  }
  gb_status emit(gb_ctx* ctx, const InsertScratch& s, int N, const gb_voxelmap& next) const {
    return gb_launch(ctx, "k_ivox_emit", k_ivox_emit, (N + 255) / 256, 256, 0, N, s.pos + (N - 1), s.keep, s.kpos, ppos, s.starts, s.t.keys_s, mref, mcount, mstamp,
                     m->voxels, s.pts, s.cov, next.vkeys, next.vstamp, next.cells, next.voxels, s.vcoord);
  }
  gb_status check_table(const gb_voxelmap& next) const {
    if (next.num_dropped_points == 0) return GB_OK;
    gb_set_error("iVox table: %d points left out of a table of %d buckets", next.num_dropped_points, next.num_buckets);
    return GB_ERR_INTERNAL;
  }
};

// Steps 1-8 for either kind; `rule` is the kind's per-voxel part.
template <typename Rule>
gb_status map_insert(gb_ctx* ctx, gb_voxelmap* m, const gb_cloud* cloud, const double* T, double sampling_rate, unsigned long long seed, Rule rule) {
  const int n = (int)cloud->n;
  const int No = (int)gb_stored_entries(m);
  const int kept = sampling_rate < 1.0 ? (int)(size_t)((double)n * sampling_rate) : n;  // random_sampling's count
  const int np = kept > 0 ? n : 0;  // points that take part (the unsampled ones get no key)
  const int N = No + np;
  gb_voxelmap next = *m;  // the map after this insert; m is replaced only when every step has succeeded
  next.lru_counter = m->lru_counter + 1;
  next.version = m->version + 1;
  gb_dev_block table(ctx->device), base(ctx->device);  // the new blocks until the hand-over, then m's replaced ones (base ends first)
  if (N > 0) {
    const size_t cub_b = gb_cub_temp_bytes((size_t)N);
    const std::vector<gb_frame> frame = gb_frame_table(1, &cloud, T, nullptr);
    InsertScratch s;
    GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
      s.t = gb_take_sort_tmp(cv, (size_t)N, cv.take<char>(cub_b), cub_b);
      s.flags = cv.take<int>(N + 1);
      s.pos = cv.take<int>(N + 1);
      s.starts = cv.take<int>(N + 1);
      s.keep = cv.take<int>(N + 1);
      s.kpos = cv.take<int>(N + 1);
      s.vcoord = cv.take<int4>(N);
      s.dropped = cv.take<int>(1);
      s.info = cv.take<unsigned long long>(2);
      s.frame = cv.take<gb_frame>(1);
      if (np > 0) {
        s.pts = cv.take<double4>(np);
        s.cov = cv.take<double>(6 * (size_t)np);
      }
      rule.scratch(cv, (size_t)N);
    }));
    if (np > 0) GB_CHECK(gb_upload(ctx, {{s.frame, frame.data(), sizeof(gb_frame)}}));
    if (m->num_voxels > 0) GB_CHECK(rule.old_keys(ctx, s.t));
    if (np > 0) {
      GB_CHECK(gb_transform_frames(ctx, 1, s.frame, np, s.pts, s.cov));
      const int* sampled = nullptr;  // the sampling's keep flags (in s.keep until the merge writes it)
      if (kept < n) {
        gb_sort_tmp pt = s.t;  // the hashes pass through the points' keys, which k_grid_keys writes next
        pt.keys += No;
        GB_CHECK(gb_thin(ctx, np, nullptr, nullptr, kept, seed, pt, s.keep));
        sampled = s.keep;
      }
      GB_CHECK(gb_grid_keys(ctx, np, s.pts, m->key_inv_res, sampled, s.t.keys + No, s.t.idx + No));
    }
    GB_CHECK(gb_group_by_key(ctx, N, s.t, s.flags, s.pos));
    GB_CHECK(gb_group_starts(ctx, N, s.t, s.flags, s.pos, s.starts));
    GB_CHECK(rule.merge(ctx, s, N));
    unsigned long long info[2] = {0, 0};
    GB_CHECK(gb_download(ctx, {{info, s.info, sizeof(info)}}));
    const int V = (int)info[1];
    next.num_voxels = V;
    next.num_points = (size_t)info[0];
    Carver size;
    Rule::layout(size, &next);  // measures, and leaves every state pointer null: the layout of an empty map
    if (V > 0) {
      GB_CHECK(gb_dev_carve(ctx, base, [&](Carver& cv) { Rule::layout(cv, &next); }));
      GB_CHECK(rule.emit(ctx, s, N, next));
    }
    GB_CHECK(table_build(ctx, V, s.vcoord, s.dropped, m->init_buckets, m->max_scan, m->drop_rate, (double)info[0], table, &next.num_buckets, &next.num_dropped_points));
    GB_CHECK(rule.check_table(next));
    base.hand_over(next.base);  // next held m's blocks until here
    table.hand_over(next.buckets);
  }
  *m = next;
  return GB_OK;
}

}  // namespace

// an empty incremental map or iVox of the parameters in `init` (the caller has entered ctx)
static gb_status map_create_empty(gb_ctx* ctx, const gb_voxelmap& init, gb_voxelmap** out) {
  gb_owned<gb_voxelmap> m(new (std::nothrow) gb_voxelmap(init), voxelmap_free);
  if (!m) return GB_ERR_INTERNAL;
  m->device = ctx->device;
  gb_dev_block table(ctx->device);
  GB_CHECK(table_build(ctx, 0, nullptr, nullptr, m->init_buckets, m->max_scan, m->drop_rate, 0.0, table, &m->num_buckets, &m->num_dropped_points));
  table.hand_over(m->buckets);
  *out = m.release();
  return GB_OK;
}
// The checks both inserts make before any launch, the handles read last; *T is the pose to insert at.
static gb_status insert_args(gb_ctx* ctx, const gb_voxelmap* m, gb_map_kind kind, const gb_cloud* cloud, const double* T_map_cloud, double sampling_rate, const double** T) {
  GB_REQUIRE(ctx && m && cloud, "null argument");
  GB_REQUIRE(sampling_rate > 0.0 && sampling_rate <= 1.0, "sampling_rate must be in (0, 1]");
  static const double kIdentity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  *T = T_map_cloud ? T_map_cloud : kIdentity;
  for (int k = 0; k < 16; k++) GB_REQUIRE(std::isfinite((*T)[k]), "T_map_cloud must be finite");
  GB_REQUIRE(m->kind == kind, kind == GB_MAP_IVOX ? "the map is not an iVox: create it with gb_ivox_create"
                                                  : "the map is not incremental: create it with gb_voxelmap_create_incremental");
  GB_REQUIRE(m->device == ctx->device && cloud->device == ctx->device, "cloud / map live on another device");
  GB_REQUIRE((uint64_t)gb_stored_entries(m) + (uint64_t)cloud->n < (1ull << 31) - 1, "stored entries + cloud points exceed 2^31");
  return GB_OK;
}
// 48-byte records (a voxel's or a stored point's) to the host; any output may be null.  A plain copy, its direction taken
// from the unified address space: the map may live on another device than the current one, and every producer call
// returned after its stream had drained.
static gb_status download_records(const float4* records, size_t count, int32_t* num_points, float* xyz, float* cov6) {
  if (count == 0 || !(num_points || xyz || cov6)) return GB_OK;
  std::vector<float4> h(3 * count);
  GB_CUDA(cudaMemcpy(h.data(), records, sizeof(float4) * h.size(), cudaMemcpyDefault));
  for (size_t r = 0; r < count; r++) {
    const float4 a = h[3 * r], b = h[3 * r + 1], c = h[3 * r + 2];
    if (num_points) num_points[r] = (int32_t)c.y;
    if (xyz) { xyz[3 * r] = a.x; xyz[3 * r + 1] = a.y; xyz[3 * r + 2] = a.z; }
    if (cov6) { cov6[6 * r] = a.w; cov6[6 * r + 1] = b.x; cov6[6 * r + 2] = b.y; cov6[6 * r + 3] = b.z; cov6[6 * r + 4] = b.w; cov6[6 * r + 5] = c.x; }
  }
  return GB_OK;
}
// The cells of an iVox or a point grid to the host, as download_records copies: coords[3 v + a] decoded from the packed key,
// counts[v] = the cell's points; either may be null.
static gb_status download_cells(const gb_voxelmap* m, int32_t* coords, int32_t* counts) {
  const size_t V = (size_t)m->num_voxels;
  if (V == 0 || !(coords || counts)) return GB_OK;
  std::vector<unsigned long long> keys(V);
  std::vector<int2> cells(V);
  GB_CUDA(cudaMemcpy(keys.data(), m->vkeys, sizeof(unsigned long long) * V, cudaMemcpyDefault));
  GB_CUDA(cudaMemcpy(cells.data(), m->cells, sizeof(int2) * V, cudaMemcpyDefault));
  for (size_t v = 0; v < V; v++) {
    if (coords) gb_unpack_key(keys[v], coords[3 * v], coords[3 * v + 1], coords[3 * v + 2]);
    if (counts) counts[v] = cells[v].y;
  }
  return GB_OK;
}

extern "C" gb_status gb_voxelmap_create_incremental(gb_ctx* ctx, float resolution, int init_num_buckets, int max_bucket_scan_count, double target_points_drop_rate,
                                                    int lru_horizon, int lru_clear_cycle, gb_voxelmap** out) {
  GB_REQUIRE(ctx && out, "null argument");
  GB_REQUIRE(resolution > 0.f && std::isfinite(resolution), "resolution must be positive and finite");
  GB_REQUIRE(init_num_buckets > 0 && (init_num_buckets & (init_num_buckets - 1)) == 0, "init_num_buckets must be a power of two");
  GB_REQUIRE(max_bucket_scan_count > 0, "max_bucket_scan_count must be positive");
  GB_REQUIRE(lru_clear_cycle >= 1, "lru_clear_cycle must be at least 1");
  *out = nullptr;
  GB_ENTER(ctx);
  gb_voxelmap m;
  m.kind = GB_MAP_INCREMENTAL;
  m.resolution = resolution;
  m.inv_res = 1.0f / resolution;
  m.key_inv_res = 1.0 / (double)resolution;
  m.max_scan = max_bucket_scan_count;
  m.init_buckets = init_num_buckets;
  m.drop_rate = target_points_drop_rate;
  m.lru_horizon = lru_horizon;
  m.lru_clear_cycle = lru_clear_cycle;
  return map_create_empty(ctx, m, out);
}
extern "C" gb_status gb_voxelmap_insert(gb_ctx* ctx, gb_voxelmap* map, const gb_cloud* cloud, const double* T_map_cloud, double sampling_rate, uint64_t seed) {
  const double* T;
  GB_CHECK(insert_args(ctx, map, GB_MAP_INCREMENTAL, cloud, T_map_cloud, sampling_rate, &T));
  GB_ENTER(ctx);
  return map_insert(ctx, map, cloud, T, sampling_rate, (unsigned long long)seed, VoxelRule{map});
}
extern "C" gb_status gb_voxelmap_info(const gb_voxelmap* m, int* num_voxels, int* num_buckets, float* resolution) {
  GB_REQUIRE(m, "null map");
  if (num_voxels) *num_voxels = m->num_voxels;
  if (num_buckets) *num_buckets = m->num_buckets;
  if (resolution) *resolution = m->resolution;
  return GB_OK;
}
extern "C" gb_status gb_voxelmap_download(const gb_voxelmap* m, int32_t* buckets, int32_t* num_points, float* means, float* cov6) {
  GB_REQUIRE(m, "null map");
  GB_REQUIRE(m->kind != GB_MAP_IVOX, "an iVox holds points, not voxels: use gb_ivox_download");
  GB_REQUIRE(m->kind != GB_MAP_POINTS, "a point grid holds points, not voxels: use gb_point_grid_download");
  if (buckets) GB_CUDA(cudaMemcpy(buckets, m->buckets, sizeof(int4) * (size_t)m->num_buckets, cudaMemcpyDefault));
  return download_records(m->voxels, (size_t)m->num_voxels, num_points, means, cov6);
}
extern "C" gb_status gb_voxelmap_destroy(gb_voxelmap* m) {
  if (!m) return GB_OK;
  cudaSetDevice(m->device);
  voxelmap_free(m);
  return GB_OK;
}

// iVox: a gb_voxelmap of kind GB_MAP_IVOX (gb_internal.cuh); voxelmap_free and gb_voxelmap_destroy release it
extern "C" gb_status gb_ivox_create(gb_ctx* ctx, double resolution, double min_dist_in_cell, int max_points_in_cell, int neighbor_voxel_mode, int lru_horizon,
                                    int lru_clear_cycle, gb_ivox** out) {
  GB_REQUIRE(ctx && out, "null argument");
  GB_REQUIRE(std::isfinite(resolution) && resolution > 0.0, "resolution must be positive and finite");
  GB_REQUIRE(min_dist_in_cell >= 0.0, "min_dist_in_cell must be >= 0");
  GB_REQUIRE(max_points_in_cell >= 1 && max_points_in_cell <= 64, "max_points_in_cell must be in [1, 64]");
  GB_REQUIRE(neighbor_voxel_mode == 1 || neighbor_voxel_mode == 7 || neighbor_voxel_mode == 19 || neighbor_voxel_mode == 27, "neighbor_voxel_mode must be 1, 7, 19 or 27");
  GB_REQUIRE(lru_clear_cycle >= 1, "lru_clear_cycle must be at least 1");
  *out = nullptr;
  GB_ENTER(ctx);
  gb_voxelmap m;
  m.kind = GB_MAP_IVOX;
  m.ivox_resolution = resolution;
  m.min_dist = min_dist_in_cell;
  m.max_points = max_points_in_cell;
  m.mode = neighbor_voxel_mode;
  m.resolution = (float)resolution;
  m.inv_res = (float)(1.0 / resolution);
  m.key_inv_res = 1.0 / resolution;
  m.max_scan = 10;          // the build's table (16384 buckets doubled until >= 8 V, 10 probes) with drop rate 0
  m.init_buckets = 16384;
  m.lru_horizon = lru_horizon;
  m.lru_clear_cycle = lru_clear_cycle;
  gb_voxelmap* h = nullptr;
  GB_CHECK(map_create_empty(ctx, m, &h));
  *out = reinterpret_cast<gb_ivox*>(h);
  return GB_OK;
}
extern "C" gb_status gb_ivox_insert(gb_ctx* ctx, gb_ivox* map, const gb_cloud* cloud, const double* T_map_cloud, double sampling_rate, uint64_t seed) {
  gb_voxelmap* m = ivox_map(map);
  const double* T;
  GB_CHECK(insert_args(ctx, m, GB_MAP_IVOX, cloud, T_map_cloud, sampling_rate, &T));
  GB_ENTER(ctx);
  return map_insert(ctx, m, cloud, T, sampling_rate, (unsigned long long)seed, IvoxRule{m});
}
extern "C" gb_status gb_ivox_info(const gb_ivox* map, int* num_voxels, size_t* num_points, double* resolution) {
  const gb_voxelmap* m = ivox_map(map);
  GB_REQUIRE(m && m->kind == GB_MAP_IVOX, "null map, or not an iVox");
  if (num_voxels) *num_voxels = m->num_voxels;
  if (num_points) *num_points = m->num_points;
  if (resolution) *resolution = m->ivox_resolution;
  return GB_OK;
}
extern "C" gb_status gb_ivox_download(const gb_ivox* map, int32_t* voxel_coords, int32_t* voxel_counts, float* xyz, float* cov6) {
  const gb_voxelmap* m = ivox_map(map);
  GB_REQUIRE(m && m->kind == GB_MAP_IVOX, "null map, or not an iVox");
  GB_CHECK(download_cells(m, voxel_coords, voxel_counts));
  return download_records(m->voxels, m->num_points, nullptr, xyz, cov6);
}
extern "C" gb_status gb_ivox_destroy(gb_ivox* map) { return gb_voxelmap_destroy(ivox_map(map)); }

// ---------------------------------------------------------------------------------------------
// Point grid (gb_point_grid_build; the rule is written once in include/glim_b200.h): every point of a cloud, grouped by its
// fp32 lookup key.  group_cloud (the build's fp32 key per original index, grouped) and gb_group_starts (stable: a cell's
// points in original index order, the points without a key last), k_grid_emit (records, cells, keys, table coordinates and the
// key extent), table_build with drop rate 0.  One host synchronisation for the cell count, one per table attempt.
// ---------------------------------------------------------------------------------------------
namespace {

// one thread per sorted slot s: record s is the cloud point of original index idx_s[s]; the first slot of a cell writes the cell
__global__ void k_grid_emit(int n, const unsigned long long* __restrict__ keys_s, const int* __restrict__ idx_s, const int* __restrict__ flags, const int* __restrict__ pos,
                            const int* __restrict__ starts, const float4* __restrict__ p0, const float4* __restrict__ p1, const float* __restrict__ p2, const int* __restrict__ inv_perm,
                            float4* __restrict__ points, int2* __restrict__ cells, unsigned long long* __restrict__ vkeys, int4* __restrict__ vcoord, int* __restrict__ extent) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const int i = idx_s[s];
  const int j = inv_perm ? inv_perm[i] : i;
  const float4 a0 = __ldg(&p0[j]);
  float4* dst = points + 3 * (size_t)s;
  dst[0] = a0;
  dst[1] = __ldg(&p1[j]);
  dst[2] = make_float4(__ldg(&p2[j]), 1.f, __int_as_float(i), 0.f);
  if (!flags[s]) return;
  const int v = pos[s] - 1;
  const unsigned long long key = keys_s[s];
  const int cnt = starts[v + 1] - s;
  int x, y, z;
  gb_unpack_key(key, x, y, z);
  cells[v] = make_int2(s, cnt);
  vkeys[v] = key;
  vcoord[v] = make_int4(x, y, z, cnt);
  const int e = max(max(max(-x, x + 1), max(-y, y + 1)), max(-z, z + 1));
  atomicMax(extent, e);
}

// the grid's block of P points and V cells: point records first (gb_voxelmap::voxels), then cells and keys
void grid_layout(Carver& cv, gb_voxelmap* g) {
  g->voxels = cv.take<float4>(3 * g->num_points);
  g->cells = cv.take<int2>((size_t)g->num_voxels);
  g->vkeys = cv.take<unsigned long long>((size_t)g->num_voxels);
}

}  // namespace

extern "C" gb_status gb_point_grid_build(gb_ctx* ctx, const gb_cloud* cloud, double cell_size, gb_point_grid** out) {
  GB_REQUIRE(ctx && cloud && out, "null argument");
  *out = nullptr;
  GB_REQUIRE(std::isfinite(cell_size) && cell_size > 0.0, "cell_size must be positive and finite");
  GB_REQUIRE(cloud->device == ctx->device, "the cloud lives on another device");
  GB_ENTER(ctx);
  gb_owned<gb_voxelmap> g(new (std::nothrow) gb_voxelmap(), voxelmap_free);
  if (!g) return GB_ERR_INTERNAL;
  g->device = ctx->device;
  g->kind = GB_MAP_POINTS;
  g->cell_size = cell_size;
  g->resolution = (float)cell_size;
  g->inv_res = (float)(1.0 / cell_size);
  g->max_scan = 10;  // the build's table (16384 buckets doubled until >= 8 cells, 10 probes) with drop rate 0
  g->init_buckets = 16384;
  const int n = (int)cloud->n;
  cudaStream_t st = ctx->stream;
  CloudGroups c{};
  gb_dev_block points(ctx->device), table(ctx->device);
  if (n > 0) {
    GB_CHECK(group_cloud(ctx, cloud, g->inv_res, c));
    g->num_voxels = c.V;
    g->num_points = (size_t)n;
    GB_CHECK(gb_dev_carve(ctx, points, [&](Carver& cv) { grid_layout(cv, g.get()); }));
    GB_CUDA(cudaMemsetAsync(c.extent, 0, sizeof(int), st));
    GB_CHECK(gb_group_starts(ctx, n, c.t, c.flags, c.pos, c.starts));
    GB_CHECK(gb_launch(ctx, "k_grid_emit", k_grid_emit, (n + 255) / 256, 256, 0, n, c.t.keys_s, c.t.idx_s, c.flags, c.pos, c.starts, cloud->p0, cloud->p1, cloud->p2,
                       cloud->inv_perm, g->voxels, g->cells, g->vkeys, c.vcoord, c.extent));
    GB_CHECK(gb_download(ctx, {{&g->key_extent, c.extent, sizeof(int)}}));
  }
  GB_CHECK(table_build(ctx, c.V, c.vcoord, c.dropped, g->init_buckets, g->max_scan, 0.0, (double)n, table, &g->num_buckets, &g->num_dropped_points));
  if (g->num_dropped_points != 0) {
    gb_set_error("point grid table: %d points left out of a table of %d buckets", g->num_dropped_points, g->num_buckets);
    return GB_ERR_INTERNAL;
  }
  points.hand_over(g->base);
  table.hand_over(g->buckets);
  *out = reinterpret_cast<gb_point_grid*>(g.release());
  return GB_OK;
}
extern "C" gb_status gb_point_grid_info(const gb_point_grid* grid, int* num_cells, size_t* num_points, double* cell_size) {
  const gb_voxelmap* g = grid_map(grid);
  GB_REQUIRE(g && g->kind == GB_MAP_POINTS, "null grid, or not a point grid");
  if (num_cells) *num_cells = g->num_voxels;
  if (num_points) *num_points = g->num_points;
  if (cell_size) *cell_size = g->cell_size;
  return GB_OK;
}
extern "C" gb_status gb_point_grid_download(const gb_point_grid* grid, int32_t* cell_coords, int32_t* cell_counts, int32_t* indices, float* xyz, float* cov6) {
  const gb_voxelmap* g = grid_map(grid);
  GB_REQUIRE(g && g->kind == GB_MAP_POINTS, "null grid, or not a point grid");
  const size_t P = g->num_points;
  GB_CHECK(download_cells(g, cell_coords, cell_counts));
  if (P > 0 && indices) {
    std::vector<float4> h(3 * P);
    GB_CUDA(cudaMemcpy(h.data(), g->voxels, sizeof(float4) * h.size(), cudaMemcpyDefault));
    for (size_t r = 0; r < P; r++) memcpy(&indices[r], &h[3 * r + 2].z, sizeof(int32_t));
  }
  return download_records(g->voxels, P, nullptr, xyz, cov6);
}
extern "C" gb_status gb_point_grid_destroy(gb_point_grid* grid) { return gb_voxelmap_destroy(grid_map(grid)); }
void grid_release(gb_point_grid* g) { gb_point_grid_destroy(g); }

// ---------------------------------------------------------------------------------------------
// Morton reordering of a new cloud (PointCloudGPU::clone keeps the caller's order on the host side of the
// boundary: gb_cloud_download and the voxel-map sums un-permute; only the device storage order changes).
// ---------------------------------------------------------------------------------------------
namespace {
__global__ void k_morton_keys(int n, const float4* __restrict__ p0, unsigned long long* __restrict__ keys, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 a = p0[i];
  unsigned long long key = ~0ull;  // non-finite / far-away points go last
  if (isfinite(a.x) && isfinite(a.y) && isfinite(a.z)) {
    const float s = 16.0f;  // 1/16 m cells
    const float fx = floorf(a.x * s), fy = floorf(a.y * s), fz = floorf(a.z * s);
    if (fabsf(fx) < 1048576.f && fabsf(fy) < 1048576.f && fabsf(fz) < 1048576.f) {
      const unsigned long long x = (unsigned long long)((int)fx + (1 << 20)), y = (unsigned long long)((int)fy + (1 << 20)), z = (unsigned long long)((int)fz + (1 << 20));
      key = (gb_spread21(x) << 2) | (gb_spread21(y) << 1) | gb_spread21(z);
    }
  }
  keys[i] = key;
  idx[i] = i;
}
__global__ void k_permute_cloud(int n, const int* __restrict__ perm, const float4* __restrict__ s0, const float4* __restrict__ s1, const float* __restrict__ s2, const float4* __restrict__ s3,
                                float4* __restrict__ d0, float4* __restrict__ d1, float* __restrict__ d2, float4* __restrict__ d3, int* __restrict__ inv_perm) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int i = perm[j];
  d0[j] = s0[i];
  d1[j] = s1[i];
  d2[j] = s2[i];
  if (s3) d3[j] = s3[i];
  inv_perm[i] = j;
}
}  // namespace

gb_status gb_cloud_build(gb_ctx* ctx, gb_cloud* c, size_t n_, const gb_planes& s, const gb_sort_tmp& t) {
  const int n = (int)n_;
  gb_planes d;
  gb_dev_block block(ctx->device);
  GB_CHECK(gb_dev_carve(ctx, block, [&](Carver& cv) {
    d = gb_cloud_planes(cv, n_, s.normals != nullptr);
    c->perm = cv.take<int>(n_);
    c->inv_perm = cv.take<int>(n_);
  }));
  c->n = n_;
  c->p0 = d.p0; c->p1 = d.p1; c->p2 = d.p2; c->normals = d.normals;
  const int tb = 256, gb = (n + tb - 1) / tb;
  GB_CHECK(gb_launch(ctx, "k_morton_keys", k_morton_keys, gb, tb, 0, n, s.p0, t.keys, t.idx));
  GB_CUB(ctx, cub::DeviceRadixSort::SortPairs, t.cub, t.cub_bytes, t.keys, t.keys_s, t.idx, c->perm, n, 0, 64);
  GB_CHECK(gb_launch(ctx, "k_permute_cloud", k_permute_cloud, gb, tb, 0, n, c->perm, s.p0, s.p1, s.p2, s.normals, c->p0, c->p1, c->p2, c->normals, c->inv_perm));
  block.hand_over(c->base);
  return GB_OK;
}
