// gb_api.cu -- implementation of the C-ABI declared in include/glim_b200.h (host side of libglim_b200.so).
#include "gb_internal.cuh"

#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <map>
#include <mutex>
#include <new>
#include <thread>

// ---------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
void gb_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
extern "C" const char* gb_last_error(void) { return g_err; }
extern "C" const char* gb_status_string(gb_status s) {
  switch (s) {
    case GB_OK: return "ok";
    case GB_ERR_INVALID_ARGUMENT: return "invalid argument";
    case GB_ERR_CUDA: return "CUDA error";
    case GB_ERR_OUT_OF_MEMORY: return "out of device memory";
    case GB_ERR_NO_DEVICE: return "no CUDA device (this library has no CPU fallback)";
    case GB_ERR_INTERNAL: return "internal error";
  }
  return "unknown status";
}

extern "C" int gb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}
extern "C" gb_status gb_mem_info(int device, size_t* free_bytes, size_t* total_bytes) {
  GB_REQUIRE(free_bytes && total_bytes, "null output");
  if (gb_device_count() <= device) { gb_set_error("no CUDA device %d", device); return GB_ERR_NO_DEVICE; }
  GB_CUDA(cudaSetDevice(device));
  GB_CUDA(cudaMemGetInfo(free_bytes, total_bytes));
  return GB_OK;
}

// ---------------------------------------------------------------------------------------------
// pooled device blocks (clouds, voxel maps)
// ---------------------------------------------------------------------------------------------
namespace {
struct DevPool {
  std::mutex mu;
  std::map<void*, size_t> live;            // block -> capacity
  std::multimap<size_t, void*> free_list;  // capacity -> block
  size_t free_bytes = 0;
  std::vector<gb_ctx*> ctxs;               // live contexts of the device (their streams are drained before a block is recycled)
};
DevPool g_pools[16];
size_t pool_class(size_t bytes) {  // size classes: 64 KB granules below 1 MB, 1/8-octave steps above
  if (bytes <= ((size_t)1 << 20)) return (bytes + 65535) / 65536 * 65536;
  size_t step = (size_t)1 << 17;
  while (step * 16 < bytes) step <<= 1;
  return (bytes + step - 1) / step * step;
}
constexpr size_t kPoolMaxFreeBytes = (size_t)2 << 30;
}  // namespace

cudaError_t gb_dev_malloc(int device, size_t bytes, void** out) {
  DevPool& P = g_pools[device & 15];
  const size_t cap = pool_class(std::max<size_t>(bytes, 256));
  {
    std::lock_guard<std::mutex> lock(P.mu);
    auto it = P.free_list.find(cap);
    if (it != P.free_list.end()) {
      *out = it->second;
      P.free_bytes -= cap;
      P.free_list.erase(it);
      P.live[*out] = cap;
      return cudaSuccess;
    }
  }
  cudaError_t e = cudaMalloc(out, cap);
  if (e != cudaSuccess) {  // give the pooled blocks back to the driver and retry once
    std::vector<void*> drop;
    { std::lock_guard<std::mutex> lock(P.mu); for (auto& kv : P.free_list) drop.push_back(kv.second); P.free_list.clear(); P.free_bytes = 0; }
    cudaGetLastError();
    for (void* q : drop) cudaFree(q);
    e = cudaMalloc(out, cap);
    if (e != cudaSuccess) return e;
  }
  std::lock_guard<std::mutex> lock(P.mu);
  P.live[*out] = cap;
  return cudaSuccess;
}
void gb_dev_free(int device, void* p) {
  if (!p) return;
  DevPool& P = g_pools[device & 15];
  std::vector<cudaStream_t> streams;
  size_t cap = 0;
  {
    std::lock_guard<std::mutex> lock(P.mu);
    auto it = P.live.find(p);
    if (it != P.live.end()) { cap = it->second; P.live.erase(it); }
    for (gb_ctx* c : P.ctxs) streams.push_back(c->stream);
  }
  if (cap == 0) { cudaFree(p); return; }
  for (cudaStream_t st : streams) cudaStreamSynchronize(st);  // nobody may still be reading the block (cudaFree's implicit guarantee)
  std::lock_guard<std::mutex> lock(P.mu);
  if (P.free_bytes + cap > kPoolMaxFreeBytes) { cudaFree(p); return; }
  P.free_list.emplace(cap, p);
  P.free_bytes += cap;
}

// ---------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------
static void ctx_release(gb_ctx* ctx);
static gb_status ctx_create(int device, cudaStream_t stream, bool own, gb_ctx** out) {
  GB_REQUIRE(out, "null output");
  *out = nullptr;
  const int n = gb_device_count();
  if (n <= 0 || device < 0 || device >= n) {
    gb_set_error("no CUDA device %d (%d visible); libglim_b200 has no CPU fallback", device, n);
    return GB_ERR_NO_DEVICE;
  }
  GB_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  GB_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    gb_set_error("device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
    return GB_ERR_NO_DEVICE;
  }
  gb_owned<gb_ctx> c(new (std::nothrow) gb_ctx(), ctx_release);
  if (!c) return GB_ERR_INTERNAL;
  c->refs.store(1);
  c->device = device;
  c->stream = stream;
  if (own) {
    GB_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    c->own_stream = true;
  }
  c->num_sms = prop.multiProcessorCount;
  { DevPool& P = g_pools[device & 15]; std::lock_guard<std::mutex> lock(P.mu); P.ctxs.push_back(c.get()); }
  *out = c.release();
  return GB_OK;
}
extern "C" gb_status gb_ctx_create(int device, gb_ctx** out) { return ctx_create(device, nullptr, true, out); }
extern "C" gb_status gb_ctx_create_on_stream(int device, void* cuda_stream, gb_ctx** out) { return ctx_create(device, (cudaStream_t)cuda_stream, false, out); }

// Cross links factor <-> sweep (a factor may sit in cached sweeps of several contexts): guarded by one registry mutex.
static std::mutex g_registry_mu;
static std::atomic<uint64_t> g_next_factor_id{1};

static void pool_block_free(const gb_pool_block& b) {
  if (b.d) cudaFree(b.d);
  if (b.h) cudaFreeHost(b.h);
}

// Contexts are reference counted: factors, sweeps and peer slabs hold one; gb_ctx_destroy drops the owner's.  A module may
// therefore destroy its CUDAStream while factors created on it are still alive (member destruction order, thread exit).
static void ctx_retain(gb_ctx* ctx) { ctx->refs.fetch_add(1); }
static void ctx_release(gb_ctx* ctx) {
  if (ctx->refs.fetch_sub(1) != 1) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  { DevPool& P = g_pools[ctx->device & 15]; std::lock_guard<std::mutex> lock(P.mu); P.ctxs.erase(std::remove(P.ctxs.begin(), P.ctxs.end(), ctx), P.ctxs.end()); }
  for (const gb_pool_block& b : ctx->pool) pool_block_free(b);
  if (ctx->scratch.base) cudaFree(ctx->scratch.base);
  if (ctx->pinned.base) cudaFreeHost(ctx->pinned.base);
  if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}
extern "C" gb_status gb_ctx_destroy(gb_ctx* ctx) {
  if (!ctx) return GB_OK;
  {
    GB_LOCK(ctx);
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    std::vector<gb_sweep*> cache;
    cache.swap(ctx->sweep_cache);
    for (gb_sweep* s : cache) sweep_free(s);
  }
  ctx_release(ctx);
  return GB_OK;
}
extern "C" gb_status gb_ctx_synchronize(gb_ctx* ctx) {
  GB_REQUIRE(ctx, "null ctx");
  GB_ENTER(ctx);
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  return GB_OK;
}
extern "C" void* gb_ctx_stream(gb_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
extern "C" uint64_t gb_ctx_kernel_launches(gb_ctx* ctx) { return ctx ? ctx->launches : 0; }

gb_status gb_arena_reserve(gb_ctx* ctx, gb_arena& a, size_t bytes) {
  if (bytes <= a.cap) return GB_OK;
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (a.base) GB_CUDA(a.host ? cudaFreeHost(a.base) : cudaFree(a.base));
  a.base = nullptr;
  a.cap = 0;
  const size_t cap = bytes + bytes / 4;
  GB_CUDA(a.host ? cudaMallocHost(&a.base, cap) : cudaMalloc(&a.base, cap));
  a.cap = cap;
  return GB_OK;
}

// ---------------------------------------------------------------------------------------------
// clouds
// ---------------------------------------------------------------------------------------------
// the reference casts Vector4d / Matrix4d to float on the host before the copy (SURVEY K1); so do we, straight into the
// plane layout in pinned memory, then stage the planes in scratch and Morton-sort them into the cloud on the device
// (the caller has made the cloud's device current)
static void cloud_free(gb_cloud* c) {
  gb_dev_free(c->device, c->base);  // waits for every stream that may still read the cloud, then recycles the block
  delete c;
}

static gb_status cloud_upload(gb_ctx* ctx, size_t n, const double* xyzw, const double* cov4x4, const double* normals4, gb_cloud* c) {
  gb_planes h;
  size_t planes_b = 0;
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) {
    h = gb_cloud_planes(cv, n, normals4 != nullptr);
    planes_b = cv.off;
  }));
  // fp64 -> fp32 cast straight into the plane layout; split over a few host threads for large clouds (the single-threaded
  // loop was 1.6 ms for 60 k points and 25 ms for 500 k: more than everything the GPU does per frame)
  auto pack = [&](size_t i0, size_t i1) {
    for (size_t i = i0; i < i1; i++) {
      const double* p = xyzw + 4 * i;
      float c00 = 0, c01 = 0, c02 = 0, c11 = 0, c12 = 0, c22 = 0;
      if (cov4x4) {
        const double* C = cov4x4 + 16 * i;  // column-major 4x4: (r,c) at c*4+r; upper triangle
        c00 = (float)C[0]; c01 = (float)C[4]; c02 = (float)C[8]; c11 = (float)C[5]; c12 = (float)C[9]; c22 = (float)C[10];
      }
      h.p0[i] = make_float4((float)p[0], (float)p[1], (float)p[2], c00);
      h.p1[i] = make_float4(c01, c02, c11, c12);
      h.p2[i] = c22;
      if (normals4) h.normals[i] = make_float4((float)normals4[4 * i], (float)normals4[4 * i + 1], (float)normals4[4 * i + 2], 0.f);
    }
  };
  {
    const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
    const size_t nt = n >= 262144 ? std::min(8u, hw) : (n >= 32768 ? std::min(4u, hw) : 1u);
    if (nt <= 1) {
      pack(0, n);
    } else {
      std::vector<std::thread> th;
      const size_t per = (n + nt - 1) / nt;
      for (size_t t = 1; t < nt; t++) th.emplace_back(pack, std::min(n, t * per), std::min(n, (t + 1) * per));
      pack(0, std::min(n, per));
      for (auto& x : th) x.join();
    }
  }
  const size_t cub_b = gb_cub_temp_bytes(n);
  gb_planes staged;
  gb_sort_tmp t;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    staged = gb_cloud_planes(cv, n, normals4 != nullptr);
    t = gb_take_sort_tmp(cv, n, cv.take<char>(cub_b), cub_b);
  }));
  GB_CUDA(cudaMemcpyAsync(staged.p0, h.p0, planes_b, cudaMemcpyHostToDevice, ctx->stream));
  GB_CHECK(gb_cloud_build(ctx, c, n, staged, t));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));  // the pinned staging buffer is reused by the next call
  return GB_OK;
}

extern "C" gb_status gb_cloud_upload(gb_ctx* ctx, size_t n, const double* xyzw, const double* cov4x4, const double* normals4, gb_cloud** out) {
  GB_REQUIRE(ctx && out, "null ctx / output");
  GB_REQUIRE(n == 0 || xyzw, "null points");
  GB_REQUIRE(n < (size_t)1 << 30, "too many points");
  *out = nullptr;
  GB_ENTER(ctx);
  gb_owned<gb_cloud> c(new (std::nothrow) gb_cloud(), cloud_free);
  if (!c) return GB_ERR_INTERNAL;
  c->device = ctx->device;
  if (n > 0) GB_CHECK(cloud_upload(ctx, n, xyzw, cov4x4, normals4, c.get()));
  *out = c.release();
  return GB_OK;
}
extern "C" gb_status gb_cloud_size(const gb_cloud* cloud, size_t* n) {
  GB_REQUIRE(cloud && n, "null argument");
  *n = cloud->n;
  return GB_OK;
}
extern "C" gb_status gb_cloud_download(const gb_cloud* c, float* xyz, float* cov6) {
  GB_REQUIRE(c, "null cloud");
  if (c->n == 0) return GB_OK;
  std::vector<float4> h0(c->n), h1(c->n);
  std::vector<float> h2(c->n);
  GB_CUDA(cudaSetDevice(c->device));  // the upload returned after its stream had drained: plain synchronous copies are safe
  GB_CUDA(cudaMemcpy(h0.data(), c->p0, sizeof(float4) * c->n, cudaMemcpyDeviceToHost));
  GB_CUDA(cudaMemcpy(h1.data(), c->p1, sizeof(float4) * c->n, cudaMemcpyDeviceToHost));
  GB_CUDA(cudaMemcpy(h2.data(), c->p2, sizeof(float) * c->n, cudaMemcpyDeviceToHost));
  std::vector<int> perm;
  if (c->perm) { perm.resize(c->n); GB_CUDA(cudaMemcpy(perm.data(), c->perm, sizeof(int) * c->n, cudaMemcpyDeviceToHost)); }
  for (size_t j = 0; j < c->n; j++) {
    const size_t i = c->perm ? (size_t)perm[j] : j;  // stored slot j holds the caller's point i
    if (xyz) { xyz[3 * i] = h0[j].x; xyz[3 * i + 1] = h0[j].y; xyz[3 * i + 2] = h0[j].z; }
    if (cov6) { cov6[6 * i] = h0[j].w; cov6[6 * i + 1] = h1[j].x; cov6[6 * i + 2] = h1[j].y; cov6[6 * i + 3] = h1[j].z; cov6[6 * i + 4] = h1[j].w; cov6[6 * i + 5] = h2[j]; }
  }
  return GB_OK;
}
extern "C" gb_status gb_cloud_device_ptrs(const gb_cloud* c, void** p0, void** p1, void** p2, void** normals) {
  GB_REQUIRE(c, "null cloud");
  if (p0) *p0 = c->p0;
  if (p1) *p1 = c->p1;
  if (p2) *p2 = c->p2;
  if (normals) *normals = c->normals;
  return GB_OK;
}
extern "C" gb_status gb_cloud_destroy(gb_cloud* c) {
  if (!c) return GB_OK;
  cudaSetDevice(c->device);
  cloud_free(c);
  return GB_OK;
}

// ---------------------------------------------------------------------------------------------
// voxel maps
// ---------------------------------------------------------------------------------------------
// (the caller has made the map's device current)
static void voxelmap_free(gb_voxelmap* m) {
  gb_dev_free(m->device, m->base);
  gb_dev_free(m->device, m->buckets);
  delete m;
}
// an empty incremental map or iVox of the parameters in `init` (the caller has entered ctx)
static gb_status map_create_empty(gb_ctx* ctx, const gb_voxelmap& init, gb_voxelmap** out) {
  gb_owned<gb_voxelmap> m(new (std::nothrow) gb_voxelmap(init), voxelmap_free);
  if (!m) return GB_ERR_INTERNAL;
  GB_CHECK(gb_map_create_empty_impl(ctx, m.get()));
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

extern "C" gb_status gb_voxelmap_build(gb_ctx* ctx, const gb_cloud* cloud, float resolution, int init_num_buckets, int max_bucket_scan_count, double target_points_drop_rate, gb_voxelmap** out) {
  GB_REQUIRE(ctx && cloud && out, "null argument");
  GB_REQUIRE(resolution > 0.f, "resolution must be positive");
  GB_REQUIRE(init_num_buckets > 0 && (init_num_buckets & (init_num_buckets - 1)) == 0, "init_num_buckets must be a power of two");
  GB_REQUIRE(max_bucket_scan_count > 0, "max_bucket_scan_count must be positive");
  *out = nullptr;
  GB_ENTER(ctx);
  gb_owned<gb_voxelmap> m(new (std::nothrow) gb_voxelmap(), voxelmap_free);
  if (!m) return GB_ERR_INTERNAL;
  GB_CHECK(gb_voxelmap_build_impl(ctx, cloud, resolution, init_num_buckets, max_bucket_scan_count, target_points_drop_rate, m.get()));
  *out = m.release();
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
  return gb_map_insert_impl(ctx, map, cloud, T, sampling_rate, (unsigned long long)seed);
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
  if (buckets) GB_CUDA(cudaMemcpy(buckets, m->buckets, sizeof(int4) * (size_t)m->num_buckets, cudaMemcpyDefault));
  return download_records(m->voxels, (size_t)m->num_voxels, num_points, means, cov6);
}
extern "C" gb_status gb_voxelmap_destroy(gb_voxelmap* m) {
  if (!m) return GB_OK;
  cudaSetDevice(m->device);
  voxelmap_free(m);
  return GB_OK;
}

// ---------------------------------------------------------------------------------------------
// iVox: a gb_voxelmap of kind GB_MAP_IVOX (gb_internal.cuh); voxelmap_free and gb_voxelmap_destroy release it
// ---------------------------------------------------------------------------------------------
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
  return gb_map_insert_impl(ctx, m, cloud, T, sampling_rate, (unsigned long long)seed);
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
  const size_t V = (size_t)m->num_voxels;
  if (V > 0 && (voxel_coords || voxel_counts)) {
    std::vector<unsigned long long> keys(V);
    std::vector<int2> cells(V);
    GB_CUDA(cudaMemcpy(keys.data(), m->vkeys, sizeof(unsigned long long) * V, cudaMemcpyDefault));
    GB_CUDA(cudaMemcpy(cells.data(), m->cells, sizeof(int2) * V, cudaMemcpyDefault));
    for (size_t v = 0; v < V; v++) {
      if (voxel_coords)
        for (int a = 0; a < 3; a++) voxel_coords[3 * v + a] = (int32_t)((keys[v] >> (42 - 21 * a)) & 0x1FFFFF) - (1 << 20);
      if (voxel_counts) voxel_counts[v] = cells[v].y;
    }
  }
  return download_records(m->voxels, m->num_points, nullptr, xyz, cov6);
}
extern "C" gb_status gb_ivox_destroy(gb_ivox* map) { return gb_voxelmap_destroy(ivox_map(map)); }

// ---------------------------------------------------------------------------------------------
// factors and sweeps
// ---------------------------------------------------------------------------------------------
extern "C" gb_status gb_vgicp_factor_create(gb_ctx* ctx, const gb_voxelmap* target, const gb_cloud* source, int flags, gb_factor** out) {
  GB_REQUIRE(ctx && target && source && out, "null argument");
  GB_REQUIRE(target->kind != GB_MAP_IVOX, "the target is an iVox: GICP factors on it come from gb_gicp_factor_create");
  // clouds / voxel maps may have been uploaded through another context (another module thread): device memory is shared,
  // and every producer call returns only after its stream has drained, so only the DEVICE has to match
  GB_REQUIRE(target->device == ctx->device && source->device == ctx->device, "cloud / voxel map live on another device");
  if (flags & GB_FACTOR_SURFACE_VALIDATION)
    GB_REQUIRE(source->normals != nullptr, "surface validation needs the source frame's normals on the device (PointCloudGPU::clone of a frame that has normals)");
  gb_factor* f = new (std::nothrow) gb_factor();
  if (!f) return GB_ERR_INTERNAL;
  f->ctx = ctx; f->target = target; f->source = source; f->flags = flags; f->id = g_next_factor_id.fetch_add(1);
  ctx_retain(ctx);
  *out = f;
  return GB_OK;
}
extern "C" gb_status gb_gicp_factor_create(gb_ctx* ctx, const gb_ivox* target, const gb_cloud* source, double max_correspondence_distance, gb_factor** out) {
  GB_REQUIRE(ctx && target && source && out, "null argument");
  GB_REQUIRE(std::isfinite(max_correspondence_distance) && max_correspondence_distance > 0.0, "max_correspondence_distance must be positive and finite");
  const gb_voxelmap* m = ivox_map(target);
  GB_REQUIRE(m->kind == GB_MAP_IVOX, "the target is not an iVox: VGICP factors on voxel maps come from gb_vgicp_factor_create");
  GB_REQUIRE(m->device == ctx->device && source->device == ctx->device, "cloud / iVox live on another device");
  GB_ENTER(ctx);
  gb_factor* f = new (std::nothrow) gb_factor();
  if (!f) return GB_ERR_INTERNAL;
  f->ctx = ctx; f->target = m; f->source = source; f->id = g_next_factor_id.fetch_add(1);
  f->max_corr2 = (float)(max_correspondence_distance * max_correspondence_distance);
  ctx_retain(ctx);
  *out = f;
  return GB_OK;
}

// return a retired sweep's blocks to its context's pool (the caller holds the context lock and has drained the stream)
static void pool_put(gb_ctx* ctx, const gb_pool_block& b) {
  if (!b.d || !b.h) { pool_block_free(b); return; }  // no block, or half of one (its pinned allocation failed): not kept
  if (ctx->pool.size() >= 64) {  // bounded: drop the smallest block
    size_t k = 0;
    for (size_t i = 1; i < ctx->pool.size(); i++) if (ctx->pool[i].d_cap < ctx->pool[k].d_cap) k = i;
    pool_block_free(ctx->pool[k]);
    ctx->pool.erase(ctx->pool.begin() + k);
  }
  ctx->pool.push_back(b);
}
static bool pool_get(gb_ctx* ctx, size_t d_need, size_t h_need, gb_pool_block* out) {
  int best = -1;
  for (size_t i = 0; i < ctx->pool.size(); i++) {
    const gb_pool_block& b = ctx->pool[i];
    if (b.d_cap >= d_need && b.h_cap >= h_need && b.d_cap <= 4 * d_need + (1 << 16) && (best < 0 || b.d_cap < ctx->pool[best].d_cap)) best = (int)i;
  }
  if (best < 0) return false;
  *out = ctx->pool[best];
  ctx->pool.erase(ctx->pool.begin() + best);
  return true;
}

void sweep_free(gb_sweep* s) {
  if (!s) return;
  gb_ctx* ctx = s->ctx;
  {
    GB_LOCK(ctx);
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    {
      std::lock_guard<std::mutex> reg(g_registry_mu);
      for (gb_factor* f : s->factors) {
        if (!f) continue;  // already destroyed (the sweep is stale)
        auto it = std::find(f->users.begin(), f->users.end(), s);
        if (it != f->users.end()) f->users.erase(it);
      }
    }
    for (int k = 0; k < 2; k++) if (s->pose_ev[k]) cudaEventDestroy(s->pose_ev[k]);
    if (s->graph_exec) cudaGraphExecDestroy(s->graph_exec);
    if (s->d_pair_ptr) cudaFree(s->d_pair_ptr);
    pool_put(ctx, s->blk);
    delete s;
  }
  ctx_release(ctx);
}

extern "C" gb_status gb_vgicp_factor_destroy(gb_factor* f) {
  if (!f) return GB_OK;
  if (f->single) { sweep_free(f->single); f->single = nullptr; }
  // sweeps that reference this factor (cached ones of any context, or caller-owned ones) are stale from now on; they are
  // freed by their owners (lazily for cached sweeps).  Only THOSE sweeps: a frame's other factor sets stay cached.
  {
    std::lock_guard<std::mutex> reg(g_registry_mu);
    for (gb_sweep* s : f->users) {
      s->stale = true;
      for (auto& p : s->factors) if (p == f) p = nullptr;
    }
    f->users.clear();
  }
  gb_ctx* ctx = f->ctx;
  delete f;
  ctx_release(ctx);
  return GB_OK;
}

static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v && *v ? atoi(v) : dflt;
}

// The work-item table of a sweep (descs[f].num_tiles / first_tile and the (factor, offset) list); it follows the kernel.
//   sweep3: items of tile_size consecutive points, factor-major (drawn from the queue by the persistent warps);
//   sweep5: strided items, about one item per warp in total; factor f gets J_f items in proportion to its expected cost
//               n_f * (1 + 1.25 r_f) (r_f = inlier fraction of its last linearization, 0.5 if unknown; a hit costs ~2.2x a
//               miss), item j owning the 32-point rows j, j + J_f, ... of the source cloud.
static void build_items(gb_sweep* s, FactorDesc* descs, std::vector<int2>& tiles) {
  tiles.clear();
  const size_t F = s->F;
  if (s->kernel_version == 3) {
    // TAIL TAPERING (guided self-scheduling): the last wave of a sweep leaves warps idle for up to one 2048-point item time --
    // little of a single-GPU sweep but a large share of one of 8 ranks' shard.  The factors that
    // hold the last ~1.5 item-times of work per warp get items of a quarter of the size, the last 0.4 a sixteenth.
    constexpr double kTaperQuarter = 1.5, kTaperSixteenth = 0.4;  // item-times per warp
    const double warps = (double)s->capacity * 8.0;
    uint64_t total = 0;
    for (size_t f = 0; f < F; f++) total += (uint64_t)descs[f].n;
    const uint64_t tail16 = (uint64_t)(warps * s->tile_size * kTaperSixteenth);
    const uint64_t tail4 = (uint64_t)(warps * s->tile_size * kTaperQuarter);
    uint64_t before = 0;
    for (size_t f = 0; f < F; f++) {
      FactorDesc& D = descs[f];
      const uint64_t remaining = total - before;  // points from the start of this factor to the end of the sweep
      int chunk = s->tile_size;
      if (remaining <= tail16) chunk = std::max(128, s->tile_size / 16);
      else if (remaining <= tail4) chunk = std::max(128, s->tile_size / 4);
      if (total <= (uint64_t)(warps * s->tile_size * 3.0)) chunk = s->tile_size;  // fewer than 3 items per warp: the item size is already chosen for the sweep
      D.chunk = chunk;
      // a factor with no points still gets one (empty) item so that its epilogue runs and zeroes its record
      const int nt = std::max(1, (D.n + chunk - 1) / chunk);
      D.num_tiles = nt;
      for (int t = 0; t < nt; t++) tiles.push_back(make_int2((int)f, t * chunk));
      before += (uint64_t)D.n;
    }
    return;
  }
  const double warps = (double)s->capacity * 8.0;
  constexpr int kMinRows = 4;  // rows of 32 points per strided item, at least
  std::vector<double> cost(F);
  double tot = 0.0;
  for (size_t f = 0; f < F; f++) {
    const gb_factor* fa = s->factors[f];
    const double r = (fa && fa->inlier_frac >= 0.f) ? (double)fa->inlier_frac : 0.5;
    cost[f] = (double)descs[f].n * (1.0 + 1.25 * r) + 64.0;  // + a floor so that empty factors get their one item
    tot += cost[f];
  }
  std::vector<int> J(F);
  double budget = warps;
  for (int iter = 0; iter < 64; iter++) {
    long long sum = 0;
    for (size_t f = 0; f < F; f++) {
      const int rows = (descs[f].n + 31) / 32;
      const int jmax = std::max(1, rows / kMinRows);
      J[f] = std::min(jmax, std::max(1, (int)(cost[f] / tot * budget + 0.5)));
      sum += J[f];
    }
    if ((double)sum <= warps) break;
    budget *= 0.95;
  }
  for (size_t f = 0; f < F; f++) {
    descs[f].chunk = 0;
    descs[f].num_tiles = J[f];
    for (int j = 0; j < J[f]; j++) tiles.push_back(make_int2((int)f, j));
  }
}

// After results have been fetched (the stream is idle): remember every factor's inlier fraction, and -- once per sweep5
// sweep -- re-size its item table from them.
static gb_status sweep_learn_inliers(gb_sweep* s) {
  for (size_t f = 0; f < s->F; f++) {
    gb_factor* fa = s->factors[f];
    if (fa && fa->source->n) fa->inlier_frac = (float)(s->h_out[f * GB_OUT_DOUBLES + 121] / (double)fa->source->n);
  }
  if (s->kernel_version != 5 || s->calibrated || s->stale) return GB_OK;
  s->calibrated = true;
  std::vector<int> old(s->F);
  for (size_t f = 0; f < s->F; f++) old[f] = s->h_descs[f].num_tiles;
  std::vector<int2> tiles;
  build_items(s, s->h_descs, tiles);
  bool changed = false;
  for (size_t f = 0; f < s->F; f++) changed = changed || std::abs(old[f] - s->h_descs[f].num_tiles) * 8 > old[f];
  if (!changed || tiles.size() > s->tiles_cap) {  // keep the old table
    for (size_t f = 0; f < s->F; f++) s->h_descs[f].num_tiles = old[f];
    return GB_OK;
  }
  memcpy(s->h_tiles, tiles.data(), sizeof(int2) * tiles.size());
  GB_CUDA(cudaMemcpyAsync(s->d_descs, s->h_descs, sizeof(FactorDesc) * s->F, cudaMemcpyHostToDevice, s->ctx->stream));
  GB_CUDA(cudaMemcpyAsync(s->d_tiles, s->h_tiles, sizeof(int2) * tiles.size(), cudaMemcpyHostToDevice, s->ctx->stream));
  s->num_tiles = (int)tiles.size();
  s->grid = std::max(1, std::min((s->num_tiles + 7) / 8, s->capacity));
  if (s->graph_exec) { cudaGraphExecDestroy(s->graph_exec); s->graph_exec = nullptr; }
  if (s->graph_state == 1) s->graph_state = 0;  // the launch geometry changed: capture again
  return GB_OK;
}

// the target part of a factor descriptor
static void desc_target(FactorDesc& D, const gb_voxelmap* t) {
  D.buckets = t->buckets; D.voxels = t->voxels;
  D.mask = (uint32_t)t->num_buckets - 1u;
  D.max_scan = t->max_scan;
  D.inv_res = t->inv_res;
}
// a GICP factor's target part: the iVox's table and point records in the FactorDesc, the rest in its GicpDesc
static void desc_target_ivox(FactorDesc& D, GicpDesc& G, const gb_factor* fa) {
  desc_target(D, fa->target);
  G.cells = fa->target->cells;
  G.max_corr2 = fa->max_corr2;
  G.num_offsets = fa->target->mode;
}
// B_f of SURVEY 8(d): 48 B per source point, 48 B per target voxel, 16 B per bucket, pose in + record out.
// The bucket term is charged at the SMALLEST table that could hold the voxels (16384 doubled until >= V), not at
// our deliberately sparse table (>= 8 V): padding we added for speed must not inflate the achieved-GB/s figure.
// A GICP factor is charged 48 B per STORED target point in place of the voxel records (its voxels' buckets the same way).
static uint64_t factor_bytes(const gb_factor* fa) {
  const bool sv = (fa->flags & GB_FACTOR_SURFACE_VALIDATION) != 0;
  const uint64_t V = (uint64_t)fa->target->num_voxels;
  const uint64_t records = fa->target->kind == GB_MAP_IVOX ? (uint64_t)fa->target->num_points : V;
  uint64_t nb_ref = 16384;
  while (nb_ref < V) nb_ref *= 2;
  return (uint64_t)fa->source->n * (48 + (sv ? 12 : 0)) + records * 48 + nb_ref * 16 + 64 + 488;  // +12 B / point: the normals, when they are read
}

// Before every launch: a factor whose target is an incremental map that gb_voxelmap_insert changed (or an iVox that
// gb_ivox_insert changed) since its descriptor was written gets that descriptor re-written (buckets, records, mask; for
// GICP the cells too) and re-uploaded.  Sweeps over built maps return at once.
static gb_status sweep_follow_targets(gb_sweep* s) {
  if (!s->any_incremental) return GB_OK;
  bool synced = false;
  for (size_t f = 0; f < s->F; f++) {
    const gb_factor* fa = s->factors[f];
    if (!fa || fa->target->version == s->target_versions[f]) continue;
    if (!synced) {  // an earlier copy of the pinned descriptors may still be in flight
      GB_CUDA(cudaStreamSynchronize(s->ctx->stream));
      synced = true;
    }
    s->target_versions[f] = fa->target->version;
    if (fa->target->kind == GB_MAP_IVOX) {
      desc_target_ivox(s->h_descs[f], s->h_gdescs[f], fa);
      GB_CUDA(cudaMemcpyAsync(s->d_gdescs + f, s->h_gdescs + f, sizeof(GicpDesc), cudaMemcpyHostToDevice, s->ctx->stream));
    } else {
      desc_target(s->h_descs[f], fa->target);
    }
    GB_CUDA(cudaMemcpyAsync(s->d_descs + f, s->h_descs + f, sizeof(FactorDesc), cudaMemcpyHostToDevice, s->ctx->stream));
  }
  if (synced) {
    s->algorithmic_bytes = 0;
    for (size_t f = 0; f < s->F; f++) if (s->factors[f]) s->algorithmic_bytes += factor_bytes(s->factors[f]);
  }
  return GB_OK;
}

// The sweep's device and pinned blocks (a pooled block may be larger than this layout measures).  The accumulators, tickets
// and queue head are adjacent: one memset zeroes them at creation, over the byte count returned.
static size_t sweep_layout(gb_sweep* s, Carver& d, Carver& h) {
  const size_t F = s->F;
  s->d_descs = d.take<FactorDesc>(F);
  s->d_tiles = d.take<int2>(s->tiles_cap);
  s->d_poses = d.take<double>(16 * F);
  s->d_poses_eval = d.take<double>(16 * F);
  const size_t zero_from = d.off;
  s->d_accum = d.take<double>(GB_ACC_STRIDE * F * s->acc_slots);
  s->d_done = d.take<unsigned>(F);
  s->d_tile_ctr = d.take<unsigned long long>(1);
  const size_t zero_bytes = d.off - zero_from;
  s->d_out = d.take<double>(GB_OUT_DOUBLES * F);
  s->h_pose_slot[0] = h.take<double>(16 * F);
  s->h_pose_slot[1] = h.take<double>(16 * F);
  s->h_poses_eval = h.take<double>(16 * F);
  s->h_out = h.take<double>(GB_OUT_DOUBLES * F);
  s->h_descs = h.take<FactorDesc>(F);
  s->h_tiles = h.take<int2>(s->tiles_cap);
  s->d_gdescs = s->gicp ? d.take<GicpDesc>(F) : nullptr;
  s->h_gdescs = s->gicp ? h.take<GicpDesc>(F) : nullptr;
  return zero_bytes;
}

extern "C" gb_status gb_sweep_create(gb_ctx* ctx, size_t F, gb_factor* const* factors, const int32_t* pair_index, gb_sweep** out) {
  GB_REQUIRE(ctx && out, "null argument");
  GB_REQUIRE(F == 0 || factors, "null factor list");
  *out = nullptr;
  // validate before anything is allocated
  uint64_t total_pts = 0;
  for (size_t f = 0; f < F; f++) {
    GB_REQUIRE(factors[f], "null factor");
    GB_REQUIRE(factors[f]->source->device == ctx->device && factors[f]->target->device == ctx->device, "factor lives on another device");
    GB_REQUIRE((factors[f]->target->kind == GB_MAP_IVOX) == (factors[0]->target->kind == GB_MAP_IVOX), "the factors of one sweep must all be VGICP or all GICP factors");
    total_pts += factors[f]->source->n;
  }
  const bool gicp = F > 0 && factors[0]->target->kind == GB_MAP_IVOX;
  GB_REQUIRE(!gicp || !pair_index, "GICP sweeps take no pair_index (no slab can be attached to them)");
  GB_ENTER(ctx);
  gb_owned<gb_sweep> s(new (std::nothrow) gb_sweep(), sweep_free);
  if (!s) return GB_ERR_INTERNAL;
  ctx_retain(ctx);
  s->ctx = ctx; s->F = F; s->factors.assign(factors, factors + F);
  s->gicp = gicp;

  // kernel generation and work-item policy
  // Kernel policy (A/B runs of the kernels, scripts/ab_sweep.py): small sweeps -- about one item per warp: an odometry
  // frame, a single pair -- run k_vgicp_sweep5 with one wave of equally expensive STRIDED items (faster on the odometry
  // workload); large sweeps run k_vgicp_sweep3 with contiguous 2048-point items drawn from the queue (its simpler hot loops
  // are faster there).  GB_KERNEL = 3 / 5 forces one kernel, with its own kind of items.
  const int kv = env_int("GB_KERNEL", 0);
  s->capacity = ctx->num_sms * 2;
  const uint64_t warps = (uint64_t)s->capacity * 8;
  const bool small = F > 0 && total_pts <= warps * 2048;
  s->kernel_version = (kv == 3 || kv == 5) ? kv : (small ? 5 : 3);
  if (gicp) s->kernel_version = 5;  // k_gicp_sweep runs sweep5's strided items at every size
  {
    // sweep3's items: ~6 items per warp (first one static, the rest drawn dynamically), between 128 and 2048 points each,
    // in whole rows of 32 points
    constexpr uint64_t kItemsPerWarp = 6, kMinItem = 128, kMaxItem = 2048;
    const uint64_t want = total_pts / (warps * kItemsPerWarp) + 1;
    const int tile = (int)std::min(kMaxItem, std::max(kMinItem, want));
    s->tile_size = (tile + 31) / 32 * 32;
  }

  std::vector<FactorDesc> descs(F);
  std::vector<GicpDesc> gdescs(gicp ? F : 0);
  std::vector<int2> tiles;
  bool any_sv = false;
  for (size_t f = 0; f < F; f++) {
    const gb_factor* fa = factors[f];
    FactorDesc& D = descs[f];
    D.p0 = fa->source->p0; D.p1 = fa->source->p1; D.p2 = fa->source->p2;
    const bool sv = (fa->flags & GB_FACTOR_SURFACE_VALIDATION) != 0;
    D.normals = sv ? fa->source->normals : nullptr;
    any_sv = any_sv || sv;
    if (gicp) desc_target_ivox(D, gdescs[f], fa); else desc_target(D, fa->target);
    s->target_versions.push_back(fa->target->version);
    s->any_incremental = s->any_incremental || fa->target->kind != GB_MAP_BUILT;
    D.n = (int)fa->source->n;
    D.pair = pair_index ? pair_index[f] : (int)f;
    s->h_pair.push_back(D.pair);
    D.flags = fa->flags;
    D.num_tiles = 1; D.chunk = s->tile_size;
    s->point_factors += (uint64_t)D.n;
    s->algorithmic_bytes += factor_bytes(fa);
  }
  s->any_sv = any_sv;
  build_items(s.get(), descs.data(), tiles);
  s->num_tiles = (int)tiles.size();
  s->grid = std::max(1, std::min((s->num_tiles + 7) / 8, s->capacity));
  // ~64 items per accumulator copy: sweeps with few factors (an odometry frame, a single pair) would otherwise
  // serialise hundreds of fp64 reductions on the same addresses
  s->acc_slots = 1;
  while (F > 0 && s->acc_slots < 16 && (uint64_t)s->num_tiles > (uint64_t)F * 64 * s->acc_slots) s->acc_slots *= 2;

  if (F > 0) {
    // one device block, one pinned block -- taken from the context's pool when a retired sweep left a fitting one
    s->tiles_cap = std::max<size_t>(tiles.size(), s->kernel_version == 5 ? (size_t)warps + F : 0);
    Carver d, h;
    sweep_layout(s.get(), d, h);
    if (!pool_get(ctx, d.off, h.off, &s->blk)) {
      GB_CUDA(cudaMalloc(&s->blk.d, d.off));
      s->blk.d_cap = d.off;
      GB_CUDA(cudaMallocHost(&s->blk.h, h.off));
      s->blk.h_cap = h.off;
    }
    d = Carver{(char*)s->blk.d};
    h = Carver{(char*)s->blk.h};
    const size_t zero_bytes = sweep_layout(s.get(), d, h);
    memcpy(s->h_descs, descs.data(), sizeof(FactorDesc) * F);
    memcpy(s->h_tiles, tiles.data(), sizeof(int2) * tiles.size());
    cudaStream_t st = ctx->stream;
    GB_CUDA(cudaMemcpyAsync(s->d_descs, s->h_descs, sizeof(FactorDesc) * F, cudaMemcpyHostToDevice, st));
    if (gicp) {
      memcpy(s->h_gdescs, gdescs.data(), sizeof(GicpDesc) * F);
      GB_CUDA(cudaMemcpyAsync(s->d_gdescs, s->h_gdescs, sizeof(GicpDesc) * F, cudaMemcpyHostToDevice, st));
    }
    GB_CUDA(cudaMemcpyAsync(s->d_tiles, s->h_tiles, sizeof(int2) * tiles.size(), cudaMemcpyHostToDevice, st));
    GB_CUDA(cudaMemsetAsync(s->d_accum, 0, zero_bytes, st));
    for (int k = 0; k < 2; k++) GB_CUDA(cudaEventCreateWithFlags(&s->pose_ev[k], cudaEventDisableTiming));
    // no synchronisation: the staging lives in the sweep's own pinned block, and everything that follows is stream ordered
  }
  {
    std::lock_guard<std::mutex> reg(g_registry_mu);
    for (gb_factor* f : s->factors) f->users.push_back(s.get());
  }
  *out = s.release();
  return GB_OK;
}
extern "C" gb_status gb_sweep_destroy(gb_sweep* s) { sweep_free(s); return GB_OK; }

extern "C" gb_status gb_sweep_attach_slab(gb_sweep* s, void* device_slab_f32, size_t num_pairs) {
  GB_REQUIRE(s, "null sweep");
  GB_REQUIRE(!s->gicp || !device_slab_f32, "no slab can be attached to a GICP sweep");
  for (size_t f = 0; f < s->F && device_slab_f32; f++)
    GB_REQUIRE(s->h_pair[f] >= 0 && (size_t)s->h_pair[f] < num_pairs, "pair index out of range for this slab");
  s->d_slab = (float*)device_slab_f32;
  s->num_pairs = num_pairs;
  return GB_OK;
}

extern "C" gb_status gb_sweep_set_poses(gb_sweep* s, const double* T) {
  GB_REQUIRE(s && (s->F == 0 || T), "null argument");
  if (s->F == 0) return GB_OK;
  GB_ENTER(s->ctx);
  // double-buffered pinned staging: wait only for the H2D that read THIS slot two calls ago (normally long finished)
  const int k = s->pose_slot;
  s->pose_slot ^= 1;
  GB_CUDA(cudaEventSynchronize(s->pose_ev[k]));
  memcpy(s->h_pose_slot[k], T, sizeof(double) * 16 * s->F);
  GB_CUDA(cudaMemcpyAsync(s->d_poses, s->h_pose_slot[k], sizeof(double) * 16 * s->F, cudaMemcpyHostToDevice, s->ctx->stream));
  GB_CUDA(cudaEventRecord(s->pose_ev[k], s->ctx->stream));
  return GB_OK;
}
static gb_status sweep_launch(gb_sweep* s, int mode) {
  if (s->stale) { gb_set_error("a factor of this sweep has been destroyed"); return GB_ERR_INVALID_ARGUMENT; }
  GB_CHECK(sweep_follow_targets(s));
  return gb_launch_sweep(s, mode);
}
// errors[f] = factor f's error at T_eval[f], with its correspondences found at T_lin[f] (F > 0)
static gb_status sweep_error(gb_sweep* s, const double* T_lin, const double* T_eval, double* errors) {
  GB_CHECK(gb_sweep_set_poses(s, T_lin));
  // the eval poses are only used by this blocking call (it ends with a stream sync): single buffer is safe
  memcpy(s->h_poses_eval, T_eval, sizeof(double) * 16 * s->F);
  GB_CUDA(cudaMemcpyAsync(s->d_poses_eval, s->h_poses_eval, sizeof(double) * 16 * s->F, cudaMemcpyHostToDevice, s->ctx->stream));
  GB_CHECK(sweep_launch(s, GB_MODE_ERROR));
  GB_CUDA(cudaMemcpyAsync(s->h_out, s->d_out, sizeof(double) * GB_OUT_DOUBLES * s->F, cudaMemcpyDeviceToHost, s->ctx->stream));
  GB_CUDA(cudaStreamSynchronize(s->ctx->stream));
  for (size_t f = 0; f < s->F; f++) errors[f] = s->h_out[f * GB_OUT_DOUBLES + 120];
  return GB_OK;
}
extern "C" gb_status gb_sweep_launch(gb_sweep* s) {
  GB_REQUIRE(s, "null sweep");
  GB_ENTER(s->ctx);
  return sweep_launch(s, GB_MODE_LINEARIZE);
}
extern "C" gb_status gb_sweep_fetch(gb_sweep* s, gb_linearized6* out) {
  GB_REQUIRE(s && (s->F == 0 || out), "null argument");
  if (s->F == 0) return GB_OK;
  GB_ENTER(s->ctx);
  static_assert(sizeof(gb_linearized6) == sizeof(double) * GB_OUT_DOUBLES, "gb_linearized6 layout");
  GB_CUDA(cudaMemcpyAsync(s->h_out, s->d_out, sizeof(double) * GB_OUT_DOUBLES * s->F, cudaMemcpyDeviceToHost, s->ctx->stream));
  GB_CUDA(cudaStreamSynchronize(s->ctx->stream));
  memcpy(out, s->h_out, sizeof(double) * GB_OUT_DOUBLES * s->F);
  return sweep_learn_inliers(s);
}
extern "C" gb_status gb_sweep_results_device(gb_sweep* s, void** device_ptr) {
  GB_REQUIRE(s && device_ptr, "null argument");
  *device_ptr = s->d_out;
  return GB_OK;
}
extern "C" gb_status gb_sweep_stats(const gb_sweep* s, uint64_t* point_factors, uint64_t* algorithmic_bytes, uint32_t* num_tiles, uint32_t* grid_size) {
  GB_REQUIRE(s, "null sweep");
  if (point_factors) *point_factors = s->point_factors;
  if (algorithmic_bytes) *algorithmic_bytes = s->algorithmic_bytes;
  if (num_tiles) *num_tiles = (uint32_t)s->num_tiles;
  if (grid_size) *grid_size = (uint32_t)s->grid;
  return GB_OK;
}

// cached sweep for (ctx, factor list): NonlinearFactorSetGPU keeps its factor list between linearize calls
static gb_status cached_sweep(gb_ctx* ctx, size_t F, gb_factor* const* factors, gb_sweep** out) {
  uint64_t key = 1469598103934665603ull;
  for (size_t f = 0; f < F; f++) {
    GB_REQUIRE(factors[f], "null factor");
    key = (key ^ factors[f]->id) * 1099511628211ull;
  }
  key ^= (uint64_t)F << 48;
  // drop the sweeps whose factors died since (only those)
  for (size_t i = 0; i < ctx->sweep_cache.size();) {
    if (ctx->sweep_cache[i]->stale) { sweep_free(ctx->sweep_cache[i]); ctx->sweep_cache.erase(ctx->sweep_cache.begin() + i); } else i++;
  }
  for (gb_sweep* s : ctx->sweep_cache)
    if (s->key == key && s->F == F && std::equal(s->factors.begin(), s->factors.end(), factors)) { *out = s; return GB_OK; }
  gb_sweep* s = nullptr;
  GB_CHECK(gb_sweep_create(ctx, F, factors, nullptr, &s));
  s->key = key;
  if (ctx->sweep_cache.size() >= 64) { sweep_free(ctx->sweep_cache.front()); ctx->sweep_cache.erase(ctx->sweep_cache.begin()); }
  ctx->sweep_cache.push_back(s);
  *out = s;
  return GB_OK;
}

// A small sweep (one wave, no queue, no exchange) has a fixed topology: poses H2D -> kernel -> records D2H.  Captured once
// as a CUDA graph, every linearization is then ONE launch call instead of three API calls (the online odometry path calls this
// ~10 times per frame: odometry_estimation_gpu.cpp:383-386).
static bool graph_eligible(const gb_sweep* s) {
  return s->graph_state >= 0 && s->kernel_version == 5 && !s->peer && !s->d_slab && (unsigned long long)s->num_tiles <= (unsigned long long)s->grid * 8ull && s->F > 0;
}
static gb_status sweep_linearize(gb_sweep* s, const double* T, gb_linearized6* out) {
  if (!graph_eligible(s)) {
    GB_CHECK(gb_sweep_set_poses(s, T));
    GB_CHECK(sweep_launch(s, GB_MODE_LINEARIZE));
    return gb_sweep_fetch(s, out);
  }
  if (s->stale) { gb_set_error("a factor of this sweep has been destroyed"); return GB_ERR_INVALID_ARGUMENT; }
  gb_ctx* ctx = s->ctx;
  GB_CHECK(sweep_follow_targets(s));  // the graph's kernel reads the descriptors from HBM
  cudaStream_t st = ctx->stream;
  const size_t pose_bytes = sizeof(double) * 16 * s->F, out_bytes = sizeof(double) * GB_OUT_DOUBLES * s->F;
  if (s->graph_state == 0) {
    GB_CUDA(cudaStreamSynchronize(st));  // nothing of this sweep may be in flight while its work is captured
    cudaGraph_t graph = nullptr;
    bool ok = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
    if (ok) {
      ok = cudaMemcpyAsync(s->d_poses, s->h_pose_slot[0], pose_bytes, cudaMemcpyHostToDevice, st) == cudaSuccess;
      const uint64_t launches = ctx->launches;
      ok = ok && gb_launch_sweep(s, GB_MODE_LINEARIZE) == GB_OK;
      ctx->launches = launches;  // counted per graph launch below
      ok = ok && cudaMemcpyAsync(s->h_out, s->d_out, out_bytes, cudaMemcpyDeviceToHost, st) == cudaSuccess;
      ok = (cudaStreamEndCapture(st, &graph) == cudaSuccess) && ok && graph != nullptr;
    }
    if (ok) ok = cudaGraphInstantiate(&s->graph_exec, graph, 0) == cudaSuccess;
    if (graph) cudaGraphDestroy(graph);
    if (!ok) {
      cudaGetLastError();
      s->graph_exec = nullptr;
      s->graph_state = -1;
      return sweep_linearize(s, T, out);  // plain launches from now on
    }
    s->graph_state = 1;
  }
  GB_CUDA(cudaEventSynchronize(s->pose_ev[0]));  // an earlier gb_sweep_set_poses may still be reading slot 0
  memcpy(s->h_pose_slot[0], T, pose_bytes);  // (the previous graph launch was synchronised below)
  GB_CUDA(cudaGraphLaunch(s->graph_exec, st));
  ctx->launches++;
  GB_CUDA(cudaStreamSynchronize(st));
  memcpy(out, s->h_out, out_bytes);
  return sweep_learn_inliers(s);
}

extern "C" gb_status gb_sweep_linearize(gb_sweep* s, const double* T, gb_linearized6* out) {
  GB_REQUIRE(s && (s->F == 0 || (T && out)), "null argument");
  if (s->F == 0) return GB_OK;
  GB_ENTER(s->ctx);
  return sweep_linearize(s, T, out);
}

extern "C" gb_status gb_factor_set_linearize(gb_ctx* ctx, size_t F, gb_factor* const* factors, const double* T, gb_linearized6* out) {
  GB_REQUIRE(ctx, "null ctx");
  if (F == 0) return GB_OK;
  GB_REQUIRE(factors && T && out, "null argument");
  GB_ENTER(ctx);
  gb_sweep* s = nullptr;
  GB_CHECK(cached_sweep(ctx, F, factors, &s));
  return sweep_linearize(s, T, out);
}

extern "C" gb_status gb_factor_set_error(gb_ctx* ctx, size_t F, gb_factor* const* factors, const double* T_lin, const double* T_eval, double* errors) {
  GB_REQUIRE(ctx, "null ctx");
  if (F == 0) return GB_OK;
  GB_REQUIRE(factors && T_lin && T_eval && errors, "null argument");
  GB_ENTER(ctx);
  gb_sweep* s = nullptr;
  GB_CHECK(cached_sweep(ctx, F, factors, &s));
  return sweep_error(s, T_lin, T_eval, errors);
}

static gb_status single_sweep(gb_factor* f, gb_sweep** out) {
  if (!f->single) GB_CHECK(gb_sweep_create(f->ctx, 1, &f, nullptr, &f->single));
  *out = f->single;
  return GB_OK;
}
extern "C" gb_status gb_vgicp_linearize(gb_factor* f, const double T[16], gb_linearized6* out) {
  GB_REQUIRE(f && T && out, "null argument");
  GB_ENTER(f->ctx);
  gb_sweep* s = nullptr;
  GB_CHECK(single_sweep(f, &s));
  return sweep_linearize(s, T, out);
}
extern "C" gb_status gb_vgicp_error(gb_factor* f, const double T_lin[16], const double T_eval[16], double* error) {
  GB_REQUIRE(f && T_lin && T_eval && error, "null argument");
  GB_ENTER(f->ctx);
  gb_sweep* s = nullptr;
  GB_CHECK(single_sweep(f, &s));
  return sweep_error(s, T_lin, T_eval, error);
}

// ---------------------------------------------------------------------------------------------
// solver hand-off: gtsam::HessianFactor blocks (SURVEY A.3; global_mapping.cpp:492-501)
// ---------------------------------------------------------------------------------------------
extern "C" gb_status gb_hessian_blocks(const gb_linearized6* L, double error_scale, double* G11, double* G12, double* g1, double* G22, double* g2, double* f) {
  GB_REQUIRE(L, "null record");
  if (G11) memcpy(G11, L->H_tt, sizeof(double) * 36);
  if (G12) memcpy(G12, L->H_ts, sizeof(double) * 36);
  if (G22) memcpy(G22, L->H_ss, sizeof(double) * 36);
  for (int k = 0; k < 6; k++) {
    if (g1) g1[k] = -L->b_t[k];  // HessianFactor takes the NEGATED gradients
    if (g2) g2[k] = -L->b_s[k];
  }
  if (f) *f = error_scale * L->error;
  return GB_OK;
}
extern "C" gb_status gb_slab_row_hessian_blocks(const float* row, double error_scale, double* G11, double* G12, double* g1, double* G22, double* g2, double* f, double* num_inliers) {
  GB_REQUIRE(row, "null slab row");
  // row: H_tt upper (21, row-major i <= j) | H_ts (36, column-major) | H_ss upper (21) | b_t (6) | b_s (6) | error | num_inliers
  int u = 0;
  for (int i = 0; i < 6; i++)
    for (int j = i; j < 6; j++, u++) {
      if (G11) { G11[j * 6 + i] = row[u]; G11[i * 6 + j] = row[u]; }
      if (G22) { G22[j * 6 + i] = row[57 + u]; G22[i * 6 + j] = row[57 + u]; }
    }
  if (G12) for (int e = 0; e < 36; e++) G12[e] = row[21 + e];
  for (int k = 0; k < 6; k++) {
    if (g1) g1[k] = -(double)row[78 + k];
    if (g2) g2[k] = -(double)row[84 + k];
  }
  if (f) *f = error_scale * (double)row[90];
  if (num_inliers) *num_inliers = (double)row[91];
  return GB_OK;
}

// ---------------------------------------------------------------------------------------------
// fused multi-GPU result exchange (peer slabs over CUDA IPC)
// ---------------------------------------------------------------------------------------------
static void peer_slab_free(gb_peer_slab* ps) {
  gb_ctx* ctx = ps->ctx;
  {
    GB_LOCK(ctx);
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (int p = 0; p < ps->world; p++)
      if (ps->opened[p]) cudaIpcCloseMemHandle(ps->peer[p]);
    if (ps->local) cudaFree(ps->local);
    if (ps->d_my_pairs) cudaFree(ps->d_my_pairs);
    if (ps->h_pinned) cudaFreeHost(ps->h_pinned);
    delete ps;
  }
  ctx_release(ctx);  // outside the lock: it may delete the context
}

extern "C" gb_status gb_peer_slab_create(gb_ctx* ctx, size_t num_pairs, int world, int rank, gb_peer_slab** out) {
  GB_REQUIRE(ctx && out, "null argument");
  GB_REQUIRE(world >= 1 && world <= GB_MAX_PEERS && rank >= 0 && rank < world, "world must be 1..8 and rank < world");
  GB_REQUIRE(num_pairs > 0, "num_pairs must be positive");
  *out = nullptr;
  GB_ENTER(ctx);
  gb_owned<gb_peer_slab> ps(new (std::nothrow) gb_peer_slab(), peer_slab_free);
  if (!ps) return GB_ERR_INTERNAL;
  ctx_retain(ctx);
  ps->ctx = ctx; ps->num_pairs = num_pairs; ps->world = world; ps->rank = rank;
  ps->connected = (world == 1);
  // fused: the sweep's epilogue stores every finished row straight into all peers; deferred: rows go to the local buffer and
  // the exchange kernel pushes them (see gb_launch_peer_signal_wait).  The peer stores' cost to the sweep grows with the
  // rank count faster than the exchange kernel's extra time -> fused up to 4 ranks, deferred above.  GB_PEER_PUSH=fused|deferred forces one.
  {
    const char* e = getenv("GB_PEER_PUSH");
    ps->deferred = world > 4;
    if (e && !strcmp(e, "fused")) ps->deferred = false;
    if (e && !strcmp(e, "deferred")) ps->deferred = true;
  }
  Carver size;
  gb_peer_layout(size, num_pairs, world);
  GB_CUDA(cudaMalloc((void**)&ps->local, size.off));
  ps->peer[rank] = ps->local;
  GB_CUDA(cudaMemsetAsync(ps->local, 0, size.off, ctx->stream));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  GB_CUDA(cudaMallocHost((void**)&ps->h_pinned, num_pairs * GB_SLAB_STRIDE * sizeof(float) + 64));
  *out = ps.release();
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_export(gb_peer_slab* ps, void* handle) {
  GB_REQUIRE(ps && handle, "null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == GB_IPC_HANDLE_BYTES, "IPC handle size");
  GB_ENTER(ps->ctx);
  cudaIpcMemHandle_t h;
  GB_CUDA(cudaIpcGetMemHandle(&h, ps->local));
  memcpy(handle, &h, sizeof(h));
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_connect(gb_peer_slab* ps, const void* handles) {
  GB_REQUIRE(ps && handles, "null argument");
  GB_ENTER(ps->ctx);
  for (int p = 0; p < ps->world; p++) {
    if (p == ps->rank || ps->opened[p]) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, (const char*)handles + (size_t)p * GB_IPC_HANDLE_BYTES, sizeof(h));
    void* ptr = nullptr;
    GB_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
    ps->peer[p] = (char*)ptr;
    ps->opened[p] = true;
  }
  ps->connected = true;
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_destroy(gb_peer_slab* ps) {
  if (ps) peer_slab_free(ps);
  return GB_OK;
}

// Replaces the device block *block (nullptr: none yet; the stream has drained) with a fresh cudaMalloc block of the layout.
// *block is the layout's first array: measuring sets it to nullptr, so it never points at a freed block.
template <typename Layout> static gb_status dev_block_realloc(void** block, Layout&& layout) {
  if (*block) GB_CUDA(cudaFree(*block));
  Carver size;
  layout(size);
  Carver cv;
  GB_CUDA(cudaMalloc((void**)&cv.base, size.off));
  layout(cv);
  return GB_OK;
}

extern "C" gb_status gb_sweep_attach_peer_slab(gb_sweep* s, gb_peer_slab* ps) {
  GB_REQUIRE(s, "null sweep");
  if (!ps) { s->peer = nullptr; return GB_OK; }
  GB_REQUIRE(!s->gicp, "no peer slab can be attached to a GICP sweep");
  GB_REQUIRE(ps->ctx == s->ctx, "peer slab belongs to another context");
  GB_REQUIRE(ps->connected, "connect the peer slab (gb_peer_slab_connect) before attaching it");
  // CSR: global pair id -> this sweep's factor indices
  const size_t P = ps->num_pairs;
  std::vector<int> ptr(P + 1, 0), fac(s->F);
  for (size_t f = 0; f < s->F; f++) {
    GB_REQUIRE(s->h_pair[f] >= 0 && (size_t)s->h_pair[f] < P, "pair index out of range for this peer slab");
    ptr[s->h_pair[f] + 1]++;
  }
  for (size_t k = 0; k < P; k++) ptr[k + 1] += ptr[k];
  std::vector<int> fill(ptr.begin(), ptr.end() - 1);
  for (size_t f = 0; f < s->F; f++) fac[fill[s->h_pair[f]]++] = (int)f;
  // the pairs this sweep owns (one sweep per peer slab): the rows the exchange kernel copies to the peers
  std::vector<int> mine;
  for (size_t k = 0; k < P; k++) if (ptr[k + 1] > ptr[k]) mine.push_back((int)k);
  GB_ENTER(s->ctx);
  GB_CUDA(cudaStreamSynchronize(s->ctx->stream));
  GB_CHECK(dev_block_realloc((void**)&s->d_pair_ptr, [&](Carver& cv) {
    s->d_pair_ptr = cv.take<int>(P + 1);
    s->d_pair_factors = cv.take<int>(std::max<size_t>(1, s->F));
    s->d_pair_done = cv.take<unsigned>(P);
    s->d_peer_tables = cv.take<PeerPush>(2);
  }));
  GB_CHECK(dev_block_realloc((void**)&ps->d_my_pairs, [&](Carver& cv) { ps->d_my_pairs = cv.take<int>(std::max<size_t>(1, mine.size())); }));
  PeerPush tabs[2];
  memset(tabs, 0, sizeof(tabs));
  for (int par = 0; par < 2; par++) {
    if (ps->deferred) {  // the sweep writes this rank's buffer only
      tabs[par].world = 1;
      tabs[par].base[0] = gb_peer_regions_of(ps, ps->rank).buf[par];
    } else {
      tabs[par].world = ps->world;
      for (int p = 0; p < ps->world; p++) tabs[par].base[p] = gb_peer_regions_of(ps, p).buf[par];
    }
    tabs[par].pair_ptr = s->d_pair_ptr; tabs[par].pair_factors = s->d_pair_factors; tabs[par].pair_done = s->d_pair_done;
  }
  GB_CUDA(cudaMemcpy(s->d_peer_tables, tabs, sizeof(tabs), cudaMemcpyHostToDevice));
  GB_CUDA(cudaMemcpy(s->d_pair_ptr, ptr.data(), sizeof(int) * (P + 1), cudaMemcpyHostToDevice));
  if (s->F) GB_CUDA(cudaMemcpy(s->d_pair_factors, fac.data(), sizeof(int) * s->F, cudaMemcpyHostToDevice));
  GB_CUDA(cudaMemset(s->d_pair_done, 0, sizeof(unsigned) * P));
  ps->num_my_pairs = (int)mine.size();
  if (!mine.empty()) GB_CUDA(cudaMemcpy(ps->d_my_pairs, mine.data(), sizeof(int) * mine.size(), cudaMemcpyHostToDevice));
  s->peer = ps;
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_signal_wait(gb_peer_slab* ps) {
  GB_REQUIRE(ps, "null peer slab");
  GB_REQUIRE(ps->connected, "gb_peer_slab_connect has not been called");
  GB_ENTER(ps->ctx);
  ps->step++;
  GB_CHECK(gb_launch_peer_signal_wait(ps));
  ps->completed_parity = ps->parity;
  ps->parity ^= 1;
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_device_ptr(gb_peer_slab* ps, void** device_ptr) {
  GB_REQUIRE(ps && device_ptr, "null argument");
  *device_ptr = gb_peer_regions_of(ps, ps->rank).buf[ps->completed_parity];
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_fetch_async(gb_peer_slab* ps, const float** host_ptr) {
  GB_REQUIRE(ps, "null peer slab");
  GB_ENTER(ps->ctx);
  const size_t bytes = ps->num_pairs * GB_SLAB_STRIDE * sizeof(float);
  const gb_peer_regions r = gb_peer_regions_of(ps, ps->rank);
  GB_CUDA(cudaMemcpyAsync(ps->h_pinned, r.buf[ps->completed_parity], bytes, cudaMemcpyDeviceToHost, ps->ctx->stream));
  GB_CUDA(cudaMemcpyAsync((char*)ps->h_pinned + bytes, r.timeout, sizeof(int), cudaMemcpyDeviceToHost, ps->ctx->stream));
  if (host_ptr) *host_ptr = ps->h_pinned;
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_fetch(gb_peer_slab* ps, float* host) {
  GB_REQUIRE(ps && host, "null argument");
  GB_ENTER(ps->ctx);
  const size_t bytes = ps->num_pairs * GB_SLAB_STRIDE * sizeof(float);
  GB_CHECK(gb_peer_slab_fetch_async(ps, nullptr));
  GB_CUDA(cudaStreamSynchronize(ps->ctx->stream));
  int timeout = 0;
  memcpy(&timeout, (char*)ps->h_pinned + bytes, sizeof(int));
  if (timeout) { gb_set_error("peer slab: a peer did not publish its completion flag within the timeout"); return GB_ERR_INTERNAL; }
  memcpy(host, ps->h_pinned, bytes);
  return GB_OK;
}

// ---------------------------------------------------------------------------------------------
// overlap
// ---------------------------------------------------------------------------------------------
extern "C" gb_status gb_overlap(gb_ctx* ctx, size_t T, const gb_voxelmap* const* targets, const gb_cloud* source, const double* deltas, double* overlap) {
  GB_REQUIRE(ctx && source && overlap, "null argument");
  *overlap = 0.0;
  if (T == 0 || source->n == 0) return GB_OK;
  GB_REQUIRE(targets && deltas, "null targets / deltas");
  GB_ENTER(ctx);
  // the same layout in pinned staging and in scratch: descriptors | poses | count
  struct Staging { FactorDesc* descs; double* poses; int* count; } h, d;
  auto layout = [&](Carver& cv, Staging& b) {
    b.descs = cv.take<FactorDesc>(T);
    b.poses = cv.take<double>(16 * T);
    b.count = cv.take<int>(1);
  };
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) { layout(cv, h); }));
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) { layout(cv, d); }));
  for (size_t t = 0; t < T; t++) {
    GB_REQUIRE(targets[t], "null target");
    FactorDesc& D = h.descs[t];
    memset(&D, 0, sizeof(D));
    D.p0 = source->p0; D.p1 = source->p1; D.p2 = source->p2;
    desc_target(D, targets[t]);
    D.n = (int)source->n;
  }
  memcpy(h.poses, deltas, sizeof(double) * 16 * T);
  GB_CUDA(cudaMemcpyAsync(d.descs, h.descs, (char*)h.count - (char*)h.descs, cudaMemcpyHostToDevice, ctx->stream));  // descriptors and poses
  GB_CUDA(cudaMemsetAsync(d.count, 0, sizeof(int), ctx->stream));
  GB_CHECK(gb_launch_overlap(ctx, (int)T, d.descs, d.poses, (int)source->n, d.count));
  GB_CUDA(cudaMemcpyAsync(h.count, d.count, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  *overlap = (double)*h.count / (double)source->n;
  return GB_OK;
}

// ---------------------------------------------------------------------------------------------
// preprocess
// ---------------------------------------------------------------------------------------------
extern "C" gb_status gb_covariances(gb_ctx* ctx, size_t n, const double* xyzw, const int32_t* neighbors, int k_correspondences, int k_neighbors, double* normals4, double* cov4x4) {
  GB_REQUIRE(ctx, "null ctx");
  if (n == 0) return GB_OK;
  GB_REQUIRE(xyzw && neighbors && normals4 && cov4x4, "null argument");
  GB_REQUIRE(k_neighbors > 0 && k_neighbors <= k_correspondences, "k_neighbors must be in [1, k_correspondences]");
  GB_REQUIRE(n < (size_t)1 << 30, "too many points");
  // the kernel gathers the points of the first k_neighbors entries of every row: an index outside [0, n) would be an
  // out-of-bounds device read
  for (size_t i = 0; i < n; i++)
    for (int j = 0; j < k_neighbors; j++) {
      const int32_t q = neighbors[i * (size_t)k_correspondences + j];
      GB_REQUIRE(q >= 0 && (size_t)q < n, "neighbour index out of range [0, n)");
    }
  GB_ENTER(ctx);
  return gb_covariances_impl(ctx, n, xyzw, neighbors, k_correspondences, k_neighbors, normals4, cov4x4);
}
extern "C" gb_status gb_find_neighbors(gb_ctx* ctx, size_t n, const double* xyzw, int k, int32_t* neighbors) {
  GB_REQUIRE(ctx, "null ctx");
  if (n == 0) return GB_OK;
  GB_REQUIRE(xyzw && neighbors && k > 0, "null argument");
  GB_REQUIRE(gb_knn_instantiated(k), "k is not an instantiated neighbour count (1-10, 12, 15, 16, 20, 24, 32)");
  GB_ENTER(ctx);
  // >= 4096 points: exact search on a pyramid of hash grids (one Morton sort, cell size 0.25 m x 4^level); fewer: the tiled
  // brute force.  GB_KNN=pyramid / brute forces one.
  const char* mode = getenv("GB_KNN");
  const bool pyramid = mode ? (strcmp(mode, "pyramid") == 0) : (n >= 4096);
  if (pyramid) return gb_find_neighbors_pyramid_impl(ctx, n, xyzw, k, neighbors);
  return gb_find_neighbors_impl(ctx, n, xyzw, k, neighbors);
}

extern "C" gb_status gb_merge_frames(gb_ctx* ctx, size_t K, const gb_cloud* const* frames, const double* poses, double resolution, int target, uint64_t seed, double* out_xyzw, double* out_cov4x4, size_t* num_out, gb_cloud** out_cloud) {
  GB_REQUIRE(ctx && num_out, "null argument");
  *num_out = 0;
  if (out_cloud) *out_cloud = nullptr;
  if (K == 0) return GB_OK;
  GB_REQUIRE(frames && poses, "null frames / poses");
  GB_REQUIRE(resolution > 0.0, "downsample_resolution must be positive");
  size_t total = 0;
  for (size_t k = 0; k < K; k++) {
    GB_REQUIRE(frames[k] && frames[k]->device == ctx->device, "null frame / frame on another device");
    total += frames[k]->n;
  }
  GB_REQUIRE(total < (size_t)1 << 30 && K < 65536, "too many points / frames");
  GB_ENTER(ctx);
  gb_owned<gb_cloud> c(out_cloud ? new (std::nothrow) gb_cloud() : nullptr, cloud_free);
  if (out_cloud && !c) return GB_ERR_INTERNAL;
  if (c) c->device = ctx->device;
  GB_CHECK(gb_merge_frames_impl(ctx, (int)K, frames, poses, resolution, target, seed, out_xyzw, out_cov4x4, num_out, c.get()));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (out_cloud) *out_cloud = c.release();
  return GB_OK;
}

extern "C" gb_status gb_preprocess_default_params(gb_preprocess_params* p) {
  GB_REQUIRE(p, "null params");
  memset(p, 0, sizeof(*p));
  p->distance_near_thresh = 0.5;      // config_preprocess.json:20
  p->distance_far_thresh = 100.0;     // :21
  p->use_random_grid_downsampling = 1;  // :22
  p->downsample_resolution = 1.0;     // :23
  p->downsample_target = 10000;       // :24
  p->downsample_rate = 0.1;           // :25
  p->seed = 0;
  p->outlier_removal_k = 10;          // :27
  p->outlier_std_mul_factor = 1.0;    // :28
  p->k_correspondences = 10;          // :33
  p->estimate_covariances = 1;
  for (int i = 0; i < 4; i++) p->T_imu_lidar[i * 5] = 1.0;
  return GB_OK;
}
extern "C" gb_status gb_preprocess(gb_ctx* ctx, size_t n, const double* xyzw, const double* times, const double* intensities, const gb_preprocess_params* P, gb_preprocessed* out) {
  GB_REQUIRE(ctx && P && out, "null argument");
  out->num_points = 0; out->last_time = 0.0; out->cloud = nullptr;
  GB_REQUIRE(n < (size_t)1 << 30, "too many points");
  GB_REQUIRE(gb_knn_instantiated(P->k_correspondences), "k_correspondences is not an instantiated neighbour count (1-10, 12, 15, 16, 20, 24, 32)");
  GB_REQUIRE(P->k_neighbors_cov >= 0 && P->k_neighbors_cov <= P->k_correspondences, "k_neighbors_cov must be in [0, k_correspondences]");
  GB_REQUIRE(!P->enable_outlier_removal || gb_knn_instantiated(P->outlier_removal_k), "outlier_removal_k is not an instantiated neighbour count (1-10, 12, 15, 16, 20, 24, 32)");
  GB_REQUIRE(P->crop_bbox_frame >= 0 && P->crop_bbox_frame <= 2, "crop_bbox_frame must be 0 (off), 1 (lidar) or 2 (imu)");
  if (n == 0) return GB_OK;
  GB_REQUIRE(xyzw, "null points");
  GB_ENTER(ctx);
  gb_owned<gb_cloud> c(P->estimate_covariances ? new (std::nothrow) gb_cloud() : nullptr, cloud_free);
  if (P->estimate_covariances && !c) return GB_ERR_INTERNAL;
  if (c) c->device = ctx->device;
  GB_CHECK(gb_preprocess_impl(ctx, n, xyzw, times, intensities, P, out, c.get()));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));  // the cloud is complete when the call returns (it may be used from another context)
  out->cloud = c.release();
  return GB_OK;
}
extern "C" gb_status gb_voxelgrid_sampling(gb_ctx* ctx, size_t n, const double* xyzw, const double* times, const double* intensities, double resolution, double* out_xyzw, double* out_times, double* out_intensities, size_t* num_out) {
  GB_REQUIRE(ctx && num_out, "null argument");
  *num_out = 0;
  if (n == 0) return GB_OK;
  GB_REQUIRE(xyzw && out_xyzw && resolution > 0.0, "null argument");
  GB_ENTER(ctx);
  return gb_voxelgrid_sampling_impl(ctx, n, xyzw, times, intensities, resolution, out_xyzw, out_times, out_intensities, num_out);
}
