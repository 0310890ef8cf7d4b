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
#include "gb_internal.cuh"

#include <cub/cub.cuh>
#include <stdlib.h>

namespace {

constexpr unsigned long long kInvalidKey = ~0ull;
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

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

}  // namespace

gb_status gb_voxelmap_build_impl(gb_ctx* ctx, const gb_cloud* cloud, float resolution, int init_buckets, int max_scan, double drop_rate, gb_voxelmap* m) {
  const int n = (int)cloud->n;
  cudaStream_t st = ctx->stream;
  m->device = ctx->device;
  m->resolution = resolution;
  m->inv_res = 1.0f / resolution;
  m->max_scan = max_scan;
  m->num_voxels = 0;
  m->num_dropped_points = 0;
  m->voxels = nullptr;
  m->buckets = nullptr;
  m->base = nullptr;

  int V = 0;
  int4* d_vcoord = nullptr;
  int* d_dropped = nullptr;
  if (n > 0) {
    // scratch layout
    size_t cub_sort = 0, cub_scan = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, cub_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, n, 0, 64, st);
    cub::DeviceScan::InclusiveSum(nullptr, cub_scan, (int*)nullptr, (int*)nullptr, n, st);
    const size_t cub_bytes = align_up(cub_sort > cub_scan ? cub_sort : cub_scan, 256);
    const size_t keys_b = align_up(sizeof(unsigned long long) * (size_t)n, 256), idx_b = align_up(sizeof(int) * (size_t)(n + 1), 256);
    const size_t vcoord_b = align_up(sizeof(int4) * (size_t)n, 256);
    const size_t total = cub_bytes + 2 * keys_b + 5 * idx_b + vcoord_b + 256;
    char* base = nullptr;
    GB_CHECK(gb_ctx_scratch(ctx, total, (void**)&base));
    char* p = base;
    void* d_cub = p; p += cub_bytes;
    unsigned long long* d_keys = (unsigned long long*)p; p += keys_b;
    unsigned long long* d_keys_s = (unsigned long long*)p; p += keys_b;
    int* d_idx = (int*)p; p += idx_b;
    int* d_idx_s = (int*)p; p += idx_b;
    int* d_flags = (int*)p; p += idx_b;
    int* d_pos = (int*)p; p += idx_b;
    int* d_starts = (int*)p; p += idx_b;
    d_vcoord = (int4*)p; p += vcoord_b;
    d_dropped = (int*)p;

    const int tb = 256, gb = (n + tb - 1) / tb;
    k_point_keys<<<gb, tb, 0, st>>>(n, cloud->p0, cloud->inv_perm, m->inv_res, d_keys, d_idx);
    size_t tmp = cub_bytes;
    GB_CUDA(cub::DeviceRadixSort::SortPairs(d_cub, tmp, d_keys, d_keys_s, d_idx, d_idx_s, n, 0, 64, st));
    k_head_flags<<<gb, tb, 0, st>>>(n, d_keys_s, d_flags);
    tmp = cub_bytes;
    GB_CUDA(cub::DeviceScan::InclusiveSum(d_cub, tmp, d_flags, d_pos, n, st));
    GB_CUDA(cudaMemcpyAsync(&V, d_pos + (n - 1), sizeof(int), cudaMemcpyDeviceToHost, st));
    GB_CUDA(cudaStreamSynchronize(st));
    ctx->launches += 4;
    if (V > 0) {
      GB_CUDA(gb_dev_malloc(ctx->device, sizeof(float4) * 3 * (size_t)V, &m->base));
      m->voxels = (float4*)m->base;
      k_voxel_starts<<<gb, tb, 0, st>>>(n, d_keys_s, d_flags, d_pos, d_starts);
      k_voxel_reduce<<<(V + 127) / 128, 128, 0, st>>>(V, d_starts, d_keys_s, d_idx_s, cloud->p0, cloud->p1, cloud->p2, cloud->inv_perm, m->voxels, d_vcoord);
      ctx->launches += 2;
    }
  }
  m->num_voxels = V;
  m->bytes = sizeof(float4) * 3 * (size_t)V;

  // hash table: double until the dropped-point rate is acceptable
  int nb = init_buckets;
  static const int load_mult = getenv("GB_TABLE_MULT") ? atoi(getenv("GB_TABLE_MULT")) : 8;  // experiment knob; 8 = the oracle's rule
  while ((long long)nb < (long long)load_mult * V) nb *= 2;  // load factor <= 1/8: the XOR-of-primes hash clusters, and lookups that
                                                             // MISS (most of them in global mapping) walk until the first empty slot;
                                                             // same rule as the oracle
  for (;;) {
    GB_CUDA(gb_dev_malloc(ctx->device, sizeof(int4) * (size_t)nb, (void**)&m->buckets));
    k_table_clear<<<(nb + 255) / 256, 256, 0, st>>>(nb, m->buckets);
    ctx->launches++;
    int dropped = 0;
    if (V > 0) {
      GB_CUDA(cudaMemsetAsync(d_dropped, 0, sizeof(int), st));
      k_table_insert<<<(V + 255) / 256, 256, 0, st>>>(V, d_vcoord, m->buckets, (uint32_t)nb - 1u, max_scan, d_dropped);
      k_table_finalize<<<(nb + 255) / 256, 256, 0, st>>>(nb, d_vcoord, m->buckets);
      ctx->launches += 2;
      GB_CUDA(cudaMemcpyAsync(&dropped, d_dropped, sizeof(int), cudaMemcpyDeviceToHost, st));
    } else {
      k_table_finalize<<<(nb + 255) / 256, 256, 0, st>>>(nb, d_vcoord, m->buckets);
      ctx->launches++;
    }
    GB_CUDA(cudaStreamSynchronize(st));
    GB_CUDA(cudaGetLastError());
    m->num_buckets = nb;
    m->num_dropped_points = dropped;
    if ((double)dropped <= drop_rate * (double)n || nb >= (1 << 28)) break;
    gb_dev_free(ctx->device, m->buckets);
    m->buckets = nullptr;
    nb *= 2;
  }
  m->bytes += sizeof(int4) * (size_t)m->num_buckets;
  return GB_OK;
}


// ---------------------------------------------------------------------------------------------
// Morton reordering of a freshly uploaded cloud (PointCloudGPU::clone keeps the caller's order on the host side of the
// boundary: gb_cloud_download and the voxel-map sums un-permute; only the device storage order changes).
// ---------------------------------------------------------------------------------------------
namespace {
__device__ __forceinline__ unsigned long long spread21(unsigned long long v) {  // 21 bits -> every third bit
  v &= 0x1FFFFFull;
  v = (v | (v << 32)) & 0x1F00000000FFFFull;
  v = (v | (v << 16)) & 0x1F0000FF0000FFull;
  v = (v | (v << 8)) & 0x100F00F00F00F00Full;
  v = (v | (v << 4)) & 0x10C30C30C30C30C3ull;
  v = (v | (v << 2)) & 0x1249249249249249ull;
  return v;
}
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
      key = (spread21(x) << 2) | (spread21(y) << 1) | spread21(z);
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

gb_status gb_cloud_reorder_impl(gb_ctx* ctx, gb_cloud* c, const void* staged, size_t b0, size_t b1, size_t b2, size_t b3) {
  const int n = (int)c->n;
  cudaStream_t st = ctx->stream;
  const char* sp = (const char*)staged;
  const float4* s0 = (const float4*)sp;
  const float4* s1 = (const float4*)(sp + b0);
  const float* s2 = (const float*)(sp + b0 + b1);
  const float4* s3 = b3 ? (const float4*)(sp + b0 + b1 + b2) : nullptr;
  size_t cub_sort = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, n, 0, 64, st);
  const size_t cub_b = align_up(cub_sort, 256), key_b = align_up(sizeof(unsigned long long) * (size_t)n, 256), idx_b = align_up(sizeof(int) * (size_t)n, 256);
  // the staged planes live at the start of the ctx scratch buffer; our temporaries go behind them (the caller sized it)
  char* p = (char*)staged + align_up(b0 + b1 + b2 + b3, 256);
  void* d_cub = p; p += cub_b;
  unsigned long long* d_keys = (unsigned long long*)p; p += key_b;
  unsigned long long* d_keys_s = (unsigned long long*)p; p += key_b;
  int* d_idx = (int*)p; p += idx_b;
  const int tb = 256, gb = (n + tb - 1) / tb;
  k_morton_keys<<<gb, tb, 0, st>>>(n, s0, d_keys, d_idx);
  size_t tmp = cub_b;
  GB_CUDA(cub::DeviceRadixSort::SortPairs(d_cub, tmp, d_keys, d_keys_s, d_idx, c->perm, n, 0, 64, st));
  k_permute_cloud<<<gb, tb, 0, st>>>(n, c->perm, s0, s1, s2, s3, c->p0, c->p1, c->p2, c->normals, c->inv_perm);
  GB_CUDA(cudaGetLastError());
  ctx->launches += 3;
  return GB_OK;
}

size_t gb_cloud_reorder_scratch_bytes(size_t n, size_t staged_bytes) {
  size_t cub_sort = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, (int)n, 0, 64, (cudaStream_t)0);
  return align_up(staged_bytes, 256) + align_up(cub_sort, 256) + 2 * align_up(sizeof(unsigned long long) * n, 256) + align_up(sizeof(int) * n, 256) + 256;
}
