// gb_api.cu -- the shared host side of the C-ABI declared in include/glim_b200.h: errors, the device pool, contexts and
// arenas, clouds, factors, sweeps and overlap.  The map, preprocess and peer-slab entry points are defined next to their
// work, in gb_kernels_voxelmap.cu, gb_kernels_preprocess.cu and gb_peer.cu.
#include "gb_internal.cuh"
#include "gb_grid_math.cuh"  // grid_half_width
#include "gb_overlap_math.cuh"  // kOverlapChunk

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
  // Lock order: a context's mu, then drain_mu, then mu.  drain_mu is held while a free drains the streams of ctxs, while a
  // context leaves ctxs (so its stream is never synchronised after ctx_release destroys it), and while the library captures
  // a sweep graph on a context's stream (so a free never synchronises a stream the library is capturing on).
  std::mutex drain_mu;
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
// Before the block is recycled, nobody may still be reading it (cudaFree's implicit guarantee): every live context's stream
// is drained.  A stream with a capture in progress is skipped: synchronising it would invalidate that capture, and a capture
// begins on a drained stream (the library's own under drain_mu, right after a synchronise; a caller's as the header asks).
// Whatever fails here is not the caller's error: the calling thread's last-error slot is left clear, and a block whose
// drain failed goes back to the driver instead of the pool.
void gb_dev_free(int device, void* p) {
  if (!p) return;
  DevPool& P = g_pools[device & 15];
  size_t cap = 0;
  {
    std::lock_guard<std::mutex> lock(P.mu);
    auto it = P.live.find(p);
    if (it != P.live.end()) { cap = it->second; P.live.erase(it); }
  }
  bool drained = cap != 0;
  if (drained) {
    std::lock_guard<std::mutex> drain(P.drain_mu);
    std::vector<cudaStream_t> streams;
    { std::lock_guard<std::mutex> lock(P.mu); for (gb_ctx* c : P.ctxs) streams.push_back(c->stream); }
    for (cudaStream_t st : streams) {
      cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
      if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) { (void)cudaGetLastError(); continue; }  // the legacy stream beside a capture
      if (cs != cudaStreamCaptureStatusNone) continue;
      if (cudaStreamSynchronize(st) != cudaSuccess) { (void)cudaGetLastError(); drained = false; }
    }
  }
  if (drained) {
    std::lock_guard<std::mutex> lock(P.mu);
    if (P.free_bytes + cap <= kPoolMaxFreeBytes) {
      P.free_list.emplace(cap, p);
      P.free_bytes += cap;
      return;
    }
  }
  if (cudaFree(p) != cudaSuccess) (void)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------
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
void ctx_retain(gb_ctx* ctx) { ctx->refs.fetch_add(1); }
void ctx_release(gb_ctx* ctx) {
  if (ctx->refs.fetch_sub(1) != 1) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  {  // under drain_mu: a free that listed this stream has finished synchronising it before the stream can be destroyed
    DevPool& P = g_pools[ctx->device & 15];
    std::lock_guard<std::mutex> drain(P.drain_mu);
    std::lock_guard<std::mutex> lock(P.mu);
    P.ctxs.erase(std::remove(P.ctxs.begin(), P.ctxs.end(), ctx), P.ctxs.end());
  }
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

gb_status gb_upload(gb_ctx* ctx, std::initializer_list<gb_xfer> parts) {
  for (const gb_xfer& p : parts)
    if (p.src && p.bytes) GB_CUDA(cudaMemcpyAsync(p.dst, p.src, p.bytes, cudaMemcpyHostToDevice, ctx->stream));
  return GB_OK;
}
gb_status gb_download(gb_ctx* ctx, std::initializer_list<gb_xfer> parts) {
  for (const gb_xfer& p : parts)
    if (p.dst && p.bytes) GB_CUDA(cudaMemcpyAsync(p.dst, p.src, p.bytes, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  return GB_OK;
}

// ---------------------------------------------------------------------------------------------
// clouds
// ---------------------------------------------------------------------------------------------
// the reference casts Vector4d / Matrix4d to float on the host before the copy (SURVEY K1); so do we, straight into the
// plane layout in pinned memory, then stage the planes in scratch and Morton-sort them into the cloud on the device
// (the caller has made the cloud's device current)
void cloud_free(gb_cloud* c) {
  gb_dev_free(c->device, c->base);  // waits for every stream that may still read the cloud, then recycles the block
  gb_dev_free(c->device, c->t_base);
  for (void* b : {c->n_base, c->f_base}) gb_dev_free(c->device, b);  // what gb_cloud_estimate_normals / _fpfh estimated
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
  c->covs = cov4x4 != nullptr;
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
// factors and sweeps
// ---------------------------------------------------------------------------------------------
gb_factor* factor_new(gb_ctx* ctx, gb_factor_kind kind, const gb_voxelmap* target, const gb_cloud* source) {
  gb_factor* f = new (std::nothrow) gb_factor();
  if (!f) return nullptr;
  f->kind = kind;
  f->ctx = ctx; f->target = target; f->source = source; f->id = g_next_factor_id.fetch_add(1);
  ctx_retain(ctx);
  return f;
}

extern "C" gb_status gb_vgicp_factor_create(gb_ctx* ctx, const gb_voxelmap* target, const gb_cloud* source, int flags, gb_factor** out) {
  GB_REQUIRE(ctx && target && source && out, "null argument");
  *out = nullptr;
  GB_REQUIRE(target->kind != GB_MAP_IVOX, "the target is an iVox: GICP factors on it come from gb_gicp_factor_create");
  GB_REQUIRE(target->kind != GB_MAP_POINTS, "the target is a point grid: GICP factors on it come from gb_gicp_grid_factor_create");
  // clouds / voxel maps may have been uploaded through another context (another module thread): device memory is shared,
  // and every producer call returns only after its stream has drained, so only the DEVICE has to match
  GB_REQUIRE(target->device == ctx->device && source->device == ctx->device, "cloud / voxel map live on another device");
  if (flags & GB_FACTOR_SURFACE_VALIDATION)
    GB_REQUIRE(source->normals != nullptr, "surface validation needs the source frame's normals on the device (PointCloudGPU::clone of a frame that has normals)");
  gb_factor* f = factor_new(ctx, GB_FACTOR_POSE, target, source);
  if (!f) return GB_ERR_INTERNAL;
  f->flags = flags;
  *out = f;
  return GB_OK;
}
extern "C" gb_status gb_gicp_factor_create(gb_ctx* ctx, const gb_ivox* target, const gb_cloud* source, double max_correspondence_distance, gb_factor** out) {
  GB_REQUIRE(ctx && target && source && out, "null argument");
  *out = nullptr;
  GB_REQUIRE(std::isfinite(max_correspondence_distance) && max_correspondence_distance > 0.0, "max_correspondence_distance must be positive and finite");
  const gb_voxelmap* m = ivox_map(target);
  GB_REQUIRE(m->kind == GB_MAP_IVOX, "the target is not an iVox: VGICP factors on voxel maps come from gb_vgicp_factor_create");
  GB_REQUIRE(m->device == ctx->device && source->device == ctx->device, "cloud / iVox live on another device");
  GB_ENTER(ctx);
  gb_factor* f = factor_new(ctx, GB_FACTOR_POSE, m, source);
  if (!f) return GB_ERR_INTERNAL;
  f->max_corr2 = (float)(max_correspondence_distance * max_correspondence_distance);
  *out = f;
  return GB_OK;
}

// The argument checks of a GICP (icp = false) or ICP factor on a point grid, and the factor's correspondence bound and search
// half-width.  Only the GICP factor reads the source's covariances.
static gb_status grid_factor_args(const gb_ctx* ctx, const gb_point_grid* target, const gb_cloud* source, double max_correspondence_distance, bool icp, gb_factor** out,
                                  float* max_corr2, int* half_width) {
  GB_REQUIRE(ctx && target && source && out, "null argument");
  *out = nullptr;
  GB_REQUIRE(std::isfinite(max_correspondence_distance) && max_correspondence_distance > 0.0, "max_correspondence_distance must be positive and finite");
  const gb_voxelmap* m = grid_map(target);
  GB_REQUIRE(m->kind == GB_MAP_POINTS, "the target is not a point grid (gb_point_grid_build)");
  GB_REQUIRE(m->device == ctx->device && source->device == ctx->device, "cloud / point grid live on another device");
  GB_REQUIRE(icp || source->covs, "the source carries no covariances");
  *max_corr2 = (float)(max_correspondence_distance * max_correspondence_distance);
  *half_width = grid_half_width(m->inv_res, *max_corr2, m->key_extent);
  GB_REQUIRE(*half_width <= kGridMaxHalfWidth, "max_correspondence_distance / cell_size too large: the search would span more than 17^3 cells");
  return GB_OK;
}
extern "C" gb_status gb_gicp_grid_factor_create(gb_ctx* ctx, const gb_point_grid* target, const gb_cloud* source, double max_correspondence_distance, gb_factor** out) {
  float max_corr2 = 0.f;
  int half_width = 0;
  GB_CHECK(grid_factor_args(ctx, target, source, max_correspondence_distance, false, out, &max_corr2, &half_width));
  GB_ENTER(ctx);
  gb_factor* f = factor_new(ctx, GB_FACTOR_POSE, grid_map(target), source);
  if (!f) return GB_ERR_INTERNAL;
  f->max_corr2 = max_corr2;
  f->grid_m = half_width;
  *out = f;
  return GB_OK;
}
extern "C" gb_status gb_icp_grid_factor_create(gb_ctx* ctx, const gb_point_grid* target, const gb_cloud* source, double max_correspondence_distance, gb_factor** out) {
  float max_corr2 = 0.f;
  int half_width = 0;
  GB_CHECK(grid_factor_args(ctx, target, source, max_correspondence_distance, true, out, &max_corr2, &half_width));
  GB_ENTER(ctx);
  gb_factor* f = factor_new(ctx, GB_FACTOR_POSE, grid_map(target), source);
  if (!f) return GB_ERR_INTERNAL;
  f->max_corr2 = max_corr2;
  f->grid_m = half_width;
  f->icp = true;
  *out = f;
  return GB_OK;
}
extern "C" gb_status gb_gicp_grid_factor_half_width(const gb_factor* f, int* m) {
  GB_REQUIRE(f && m, "null argument");
  GB_ENTER(f->ctx);
  *m = f->grid_m;
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

void desc_target(FactorDesc& D, const gb_voxelmap* t) {
  D.buckets = t->buckets; D.voxels = t->voxels;
  D.mask = (uint32_t)t->num_buckets - 1u;
  D.max_scan = t->max_scan;
  D.inv_res = t->inv_res;
}
void desc_target_gicp(FactorDesc& D, GicpDesc& G, const gb_factor* fa) {
  desc_target(D, fa->target);
  G.cells = fa->target->cells;
  G.max_corr2 = fa->max_corr2;
  G.num_offsets = fa->target->kind == GB_MAP_POINTS ? fa->grid_m : fa->target->mode;
}
// B_f of SURVEY 8(d): 48 B per source point, 48 B per target voxel, 16 B per bucket, pose in + record out.
// The bucket term is charged at the SMALLEST table that could hold the voxels (16384 doubled until >= V), not at
// our deliberately sparse table (>= 8 V): padding we added for speed must not inflate the achieved-GB/s figure.
// A GICP factor is charged 48 B per STORED target point in place of the voxel records (its voxels' or cells' buckets the
// same way); an ICP factor reads one float4 of each: 16 B per source point and per stored target point.
static uint64_t factor_bytes(const gb_factor* fa) {
  const bool sv = (fa->flags & GB_FACTOR_SURFACE_VALIDATION) != 0;
  const uint64_t V = (uint64_t)fa->target->num_voxels;
  const uint64_t records = gb_target_class(fa->target) != 0 ? (uint64_t)fa->target->num_points : V;
  uint64_t nb_ref = 16384;
  while (nb_ref < V) nb_ref *= 2;
  if (fa->icp) return ((uint64_t)fa->source->n + records + nb_ref) * 16 + 64 + 488;
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
    if (s->gicp) {
      desc_target_gicp(s->h_descs[f], s->h_gdescs[f], fa);
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
  s->d_idescs = s->kernel_version == 3 ? d.take<IndexDesc>(F) : nullptr;
  s->h_idescs = s->kernel_version == 3 ? h.take<IndexDesc>(F) : nullptr;
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
    GB_REQUIRE(factors[f]->kind == GB_FACTOR_POSE,
               "not a pose factor: a CT factor has two poses (the gb_ct_* entry points), a plane factor one per key (gb_plane_evm_*)");
    GB_REQUIRE(factors[f]->source->device == ctx->device && factors[f]->target->device == ctx->device, "factor lives on another device");
    GB_REQUIRE(gb_factor_class(factors[f]) == gb_factor_class(factors[0]),
               "the factors of one sweep must all be VGICP factors, all GICP factors on iVoxes, all GICP factors on point grids or all ICP factors");
    total_pts += factors[f]->source->n;
  }
  const int factor_class = F > 0 ? gb_factor_class(factors[0]) : 0;
  const bool gicp = factor_class != 0;
  GB_REQUIRE(!gicp || !pair_index, "GICP sweeps take no pair_index (no slab can be attached to them)");
  GB_ENTER(ctx);
  gb_owned<gb_sweep> s(new (std::nothrow) gb_sweep(), sweep_free);
  if (!s) return GB_ERR_INTERNAL;
  ctx_retain(ctx);
  s->ctx = ctx; s->F = F; s->factors.assign(factors, factors + F);
  s->gicp = gicp;
  s->point_grid = factor_class >= 2;
  s->icp = factor_class == 3;

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
  if (gicp) s->kernel_version = 5;  // k_gicp_sweep, k_gicp_grid_sweep and k_icp_grid_sweep run sweep5's strided items at every size
  // sweep3 probes each target's probe index (gb_probe_index.cuh) and queues a hit's voxel index in 21 bits (gb_sweep_steps.cuh),
  // so it runs a sweep only when every target is a built map with an index -- fewer than 2^21 voxels and a box that fits 14 bits
  // per axis -- whatever GB_KERNEL says.  An incremental map may grow past that after the sweep is made.
  for (size_t f = 0; f < F; f++) {
    const gb_voxelmap* t = factors[f]->target;
    if (t->kind != GB_MAP_BUILT || !t->index) s->kernel_version = 5;
  }
  {
    // sweep3's items: ~6 items per warp (first one static, the rest drawn dynamically), between 128 and 2048 points each,
    // in whole rows of 32 points (sweep3 queues a point's offset within its item in 11 bits)
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
    if (gicp) desc_target_gicp(D, gdescs[f], fa); else desc_target(D, fa->target);
    s->target_versions.push_back(fa->target->version);
    s->any_incremental = s->any_incremental || (fa->target->kind != GB_MAP_BUILT && fa->target->kind != GB_MAP_POINTS);
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
    if (s->kernel_version == 3) {  // every target is a built map with a probe index
      for (size_t f = 0; f < F; f++) {
        const gb_voxelmap* t = factors[f]->target;
        s->h_idescs[f] = IndexDesc{t->index, ((uint32_t)t->num_buckets >> kPiSetShift) - 1u, t->box};
      }
      GB_CUDA(cudaMemcpyAsync(s->d_idescs, s->h_idescs, sizeof(IndexDesc) * F, cudaMemcpyHostToDevice, st));
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
    cudaGraph_t graph = nullptr;
    bool ok;
    {
      // under the pool's drain lock: no gb_dev_free of another thread synchronises the stream during the capture
      std::lock_guard<std::mutex> drain(g_pools[ctx->device & 15].drain_mu);
      GB_CUDA(cudaStreamSynchronize(st));  // nothing of this sweep may be in flight while its work is captured
      ok = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess;  // refused on the legacy stream
      if (ok) {
        ok = cudaMemcpyAsync(s->d_poses, s->h_pose_slot[0], pose_bytes, cudaMemcpyHostToDevice, st) == cudaSuccess;
        const uint64_t launches = ctx->launches;
        ok = ok && gb_launch_sweep(s, GB_MODE_LINEARIZE) == GB_OK;
        ctx->launches = launches;  // counted per graph launch below
        ok = ok && cudaMemcpyAsync(s->h_out, s->d_out, out_bytes, cudaMemcpyDeviceToHost, st) == cudaSuccess;
        ok = (cudaStreamEndCapture(st, &graph) == cudaSuccess) && ok && graph != nullptr;
      }
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
// overlap
// ---------------------------------------------------------------------------------------------
extern "C" gb_status gb_overlap(gb_ctx* ctx, size_t T, const gb_voxelmap* const* targets, const gb_cloud* source, const double* deltas, double* overlap) {
  GB_REQUIRE(ctx && source && overlap, "null argument");
  *overlap = 0.0;
  if (T == 0 || source->n == 0) return GB_OK;
  GB_REQUIRE(targets && deltas, "null targets / deltas");
  for (size_t t = 0; t < T; t++) GB_REQUIRE(!targets[t] || targets[t]->kind != GB_MAP_POINTS, "a point grid is not an occupancy target");
  GB_ENTER(ctx);
  // the same layout in pinned staging and in scratch: descriptors | poses | the query | its item count | count.  One query of
  // T targets: the source is descriptor 0's.
  struct Staging { FactorDesc* descs; double* poses; OverlapQuery* query; int* num_queries; long long* item_end; int* count; } h, d;
  auto layout = [&](Carver& cv, Staging& b) {
    b.descs = cv.take<FactorDesc>(T);
    b.poses = cv.take<double>(16 * T);
    b.query = cv.take<OverlapQuery>(1);
    b.num_queries = cv.take<int>(1);
    b.item_end = cv.take<long long>(1);
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
  const long long items = ((long long)source->n + kOverlapChunk - 1) / kOverlapChunk;  // overlap_chunks(n)
  *h.query = OverlapQuery{0, 0, 0, (int)T};
  *h.num_queries = 1;
  *h.item_end = items;
  GB_CUDA(cudaMemcpyAsync(d.descs, h.descs, (char*)h.count - (char*)h.descs, cudaMemcpyHostToDevice, ctx->stream));  // all but the count
  GB_CUDA(cudaMemsetAsync(d.count, 0, sizeof(int), ctx->stream));
  GB_CHECK(gb_launch_overlap(ctx, (int)std::min<long long>(items, ctx->num_sms * 8), (int)T, d.query, d.num_queries, d.item_end, d.descs, d.poses, nullptr, d.count));
  GB_CUDA(cudaMemcpyAsync(h.count, d.count, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  *overlap = (double)*h.count / (double)source->n;
  return GB_OK;
}
