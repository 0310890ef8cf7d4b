// gb_api.cu -- implementation of the C-ABI declared in include/glim_b200.h (host side of libglim_b200.so).
#include "gb_internal.cuh"

#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
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
  if (cap == 0 || getenv("GB_NO_POOL")) { cudaFree(p); return; }
  for (cudaStream_t st : streams) cudaStreamSynchronize(st);  // nobody may still be reading the block (cudaFree's implicit guarantee)
  std::lock_guard<std::mutex> lock(P.mu);
  if (P.free_bytes + cap > kPoolMaxFreeBytes) { cudaFree(p); return; }
  P.free_list.emplace(cap, p);
  P.free_bytes += cap;
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
  gb_ctx* c = new (std::nothrow) gb_ctx();
  if (!c) return GB_ERR_INTERNAL;
  c->device = device;
  c->own_stream = own;
  c->stream = stream;
  if (own) {
    cudaError_t e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) { delete c; gb_set_error("cudaStreamCreate: %s", cudaGetErrorString(e)); return GB_ERR_CUDA; }
  }
  c->num_sms = prop.multiProcessorCount;
  c->scratch = nullptr; c->scratch_cap = 0;
  c->pinned = nullptr; c->pinned_cap = 0;
  c->launches = 0;
  c->refs.store(1);
  { DevPool& P = g_pools[device & 15]; std::lock_guard<std::mutex> lock(P.mu); P.ctxs.push_back(c); }
  *out = c;
  return GB_OK;
}
extern "C" gb_status gb_ctx_create(int device, gb_ctx** out) { return ctx_create(device, nullptr, true, out); }
extern "C" gb_status gb_ctx_create_on_stream(int device, void* cuda_stream, gb_ctx** out) { return ctx_create(device, (cudaStream_t)cuda_stream, false, out); }

static void sweep_free(gb_sweep* s);

// Cross links factor <-> sweep (a factor may sit in cached sweeps of several contexts): guarded by one registry mutex.
static std::mutex g_registry_mu;
static std::atomic<uint64_t> g_next_factor_id{1};

// Contexts are reference counted: factors, sweeps and peer slabs hold one; gb_ctx_destroy drops the owner's.  A module may
// therefore destroy its CUDAStream while factors created on it are still alive (member destruction order, thread exit).
static void ctx_retain(gb_ctx* ctx) { ctx->refs.fetch_add(1); }
static void ctx_release(gb_ctx* ctx) {
  if (ctx->refs.fetch_sub(1) != 1) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  { DevPool& P = g_pools[ctx->device & 15]; std::lock_guard<std::mutex> lock(P.mu); P.ctxs.erase(std::remove(P.ctxs.begin(), P.ctxs.end(), ctx), P.ctxs.end()); }
  for (gb_pool_block& b : ctx->pool) { if (b.d) cudaFree(b.d); if (b.h) cudaFreeHost(b.h); }
  ctx->pool.clear();
  if (ctx->scratch) cudaFree(ctx->scratch);
  if (ctx->pinned) cudaFreeHost(ctx->pinned);
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
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  return GB_OK;
}
extern "C" void* gb_ctx_stream(gb_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
extern "C" uint64_t gb_ctx_kernel_launches(gb_ctx* ctx) { return ctx ? ctx->launches : 0; }

gb_status gb_ctx_scratch(gb_ctx* ctx, size_t bytes, void** out) {
  if (bytes > ctx->scratch_cap) {
    GB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (ctx->scratch) GB_CUDA(cudaFree(ctx->scratch));
    ctx->scratch = nullptr; ctx->scratch_cap = 0;
    const size_t cap = bytes + bytes / 4;
    GB_CUDA(cudaMalloc(&ctx->scratch, cap));
    ctx->scratch_cap = cap;
  }
  *out = ctx->scratch;
  return GB_OK;
}
gb_status gb_ctx_pinned(gb_ctx* ctx, size_t bytes, void** out) {
  if (bytes > ctx->pinned_cap) {
    GB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (ctx->pinned) GB_CUDA(cudaFreeHost(ctx->pinned));
    ctx->pinned = nullptr; ctx->pinned_cap = 0;
    const size_t cap = bytes + bytes / 4;
    GB_CUDA(cudaMallocHost(&ctx->pinned, cap));
    ctx->pinned_cap = cap;
  }
  *out = ctx->pinned;
  return GB_OK;
}

// ---------------------------------------------------------------------------------------------
// clouds
// ---------------------------------------------------------------------------------------------
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

extern "C" gb_status gb_cloud_upload(gb_ctx* ctx, size_t n, const double* xyzw, const double* cov4x4, const double* normals4, gb_cloud** out) {
  GB_REQUIRE(ctx && out, "null ctx / output");
  GB_REQUIRE(n == 0 || xyzw, "null points");
  GB_REQUIRE(n < (size_t)1 << 30, "too many points");
  *out = nullptr;
  GB_CUDA(cudaSetDevice(ctx->device));
  gb_cloud* c = new (std::nothrow) gb_cloud();
  if (!c) return GB_ERR_INTERNAL;
  c->device = ctx->device; c->n = n; c->base = nullptr; c->bytes = 0;
  c->p0 = nullptr; c->p1 = nullptr; c->p2 = nullptr; c->normals = nullptr; c->perm = nullptr; c->inv_perm = nullptr;
  if (n == 0) { *out = c; return GB_OK; }
  // the reference casts Vector4d / Matrix4d to float on the host before the copy (SURVEY K1); so do we,
  // straight into the device plane layout, staged through pinned memory
  const size_t b0 = align_up(sizeof(float4) * n, 256), b1 = b0, b2 = align_up(sizeof(float) * n, 256), b3 = normals4 ? b0 : 0;
  const size_t total = b0 + b1 + b2 + b3;
  char* h = nullptr;
  gb_status st = gb_ctx_pinned(ctx, total, (void**)&h);
  if (st != GB_OK) { delete c; return st; }
  float4* h0 = (float4*)h;
  float4* h1 = (float4*)(h + b0);
  float* h2 = (float*)(h + b0 + b1);
  float4* h3 = (float4*)(h + b0 + b1 + b2);
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
      h0[i] = make_float4((float)p[0], (float)p[1], (float)p[2], c00);
      h1[i] = make_float4(c01, c02, c11, c12);
      h2[i] = c22;
      if (normals4) h3[i] = make_float4((float)normals4[4 * i], (float)normals4[4 * i + 1], (float)normals4[4 * i + 2], 0.f);
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
  static const bool reorder = !(getenv("GB_NO_REORDER") && atoi(getenv("GB_NO_REORDER")));
  const size_t bperm = reorder ? align_up(sizeof(int) * n, 256) : 0;
  cudaError_t e = gb_dev_malloc(ctx->device, total + 2 * bperm, &c->base);
  if (e != cudaSuccess) { delete c; gb_set_error("cudaMalloc(%zu): %s", total + 2 * bperm, cudaGetErrorString(e)); return GB_ERR_OUT_OF_MEMORY; }
  c->bytes = total + 2 * bperm;
  char* d = (char*)c->base;
  c->p0 = (float4*)d; c->p1 = (float4*)(d + b0); c->p2 = (float*)(d + b0 + b1); c->normals = normals4 ? (float4*)(d + b0 + b1 + b2) : nullptr;
  if (reorder) { c->perm = (int*)(d + total); c->inv_perm = (int*)(d + total + bperm); }
  st = GB_OK;
  if (reorder) {
    // stage the planes in the caller's order in scratch, then Morton-sort them into place on the device
    char* scratch = nullptr;
    st = gb_ctx_scratch(ctx, gb_cloud_reorder_scratch_bytes(n, total), (void**)&scratch);
    if (st == GB_OK) {
      e = cudaMemcpyAsync(scratch, h, total, cudaMemcpyHostToDevice, ctx->stream);
      if (e != cudaSuccess) { gb_set_error("upload: %s", cudaGetErrorString(e)); st = GB_ERR_CUDA; }
    }
    if (st == GB_OK) st = gb_cloud_reorder_impl(ctx, c, scratch, b0, b1, b2, b3);
  } else {
    e = cudaMemcpyAsync(c->base, h, total, cudaMemcpyHostToDevice, ctx->stream);
    if (e != cudaSuccess) { gb_set_error("upload: %s", cudaGetErrorString(e)); st = GB_ERR_CUDA; }
  }
  if (st == GB_OK) {
    e = cudaStreamSynchronize(ctx->stream);  // the pinned staging buffer is reused by the next call
    if (e != cudaSuccess) { gb_set_error("upload: %s", cudaGetErrorString(e)); st = GB_ERR_CUDA; }
  }
  if (st != GB_OK) { gb_dev_free(ctx->device, c->base); delete c; return st; }
  *out = c;
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
  gb_dev_free(c->device, c->base);  // waits for every stream that may still read the cloud, then recycles the block
  delete c;
  return GB_OK;
}

// ---------------------------------------------------------------------------------------------
// voxel maps
// ---------------------------------------------------------------------------------------------
extern "C" gb_status gb_voxelmap_build(gb_ctx* ctx, const gb_cloud* cloud, float resolution, int init_num_buckets, int max_bucket_scan_count, double target_points_drop_rate, gb_voxelmap** out) {
  GB_REQUIRE(ctx && cloud && out, "null argument");
  GB_REQUIRE(resolution > 0.f, "resolution must be positive");
  GB_REQUIRE(init_num_buckets > 0 && (init_num_buckets & (init_num_buckets - 1)) == 0, "init_num_buckets must be a power of two");
  GB_REQUIRE(max_bucket_scan_count > 0, "max_bucket_scan_count must be positive");
  *out = nullptr;
  GB_CUDA(cudaSetDevice(ctx->device));
  gb_voxelmap* m = new (std::nothrow) gb_voxelmap();
  if (!m) return GB_ERR_INTERNAL;
  gb_status st = gb_voxelmap_build_impl(ctx, cloud, resolution, init_num_buckets, max_bucket_scan_count, target_points_drop_rate, m);
  if (st != GB_OK) {
    gb_dev_free(ctx->device, m->base);
    gb_dev_free(ctx->device, m->buckets);
    delete m;
    return st;
  }
  *out = m;
  return GB_OK;
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
  GB_CUDA(cudaSetDevice(m->device));
  if (buckets) GB_CUDA(cudaMemcpy(buckets, m->buckets, sizeof(int4) * (size_t)m->num_buckets, cudaMemcpyDeviceToHost));
  if ((num_points || means || cov6) && m->num_voxels > 0) {
    std::vector<float4> h(3 * (size_t)m->num_voxels);
    GB_CUDA(cudaMemcpy(h.data(), m->voxels, sizeof(float4) * h.size(), cudaMemcpyDeviceToHost));
    for (size_t v = 0; v < (size_t)m->num_voxels; v++) {
      const float4 a = h[3 * v], b = h[3 * v + 1], c = h[3 * v + 2];
      if (num_points) num_points[v] = (int32_t)c.y;
      if (means) { means[3 * v] = a.x; means[3 * v + 1] = a.y; means[3 * v + 2] = a.z; }
      if (cov6) { cov6[6 * v] = a.w; cov6[6 * v + 1] = b.x; cov6[6 * v + 2] = b.y; cov6[6 * v + 3] = b.z; cov6[6 * v + 4] = b.w; cov6[6 * v + 5] = c.x; }
    }
  }
  return GB_OK;
}
extern "C" gb_status gb_voxelmap_destroy(gb_voxelmap* m) {
  if (!m) return GB_OK;
  cudaSetDevice(m->device);
  gb_dev_free(m->device, m->base);
  gb_dev_free(m->device, m->buckets);
  delete m;
  return GB_OK;
}

// ---------------------------------------------------------------------------------------------
// factors and sweeps
// ---------------------------------------------------------------------------------------------
extern "C" gb_status gb_vgicp_factor_create(gb_ctx* ctx, const gb_voxelmap* target, const gb_cloud* source, int flags, gb_factor** out) {
  GB_REQUIRE(ctx && target && source && out, "null argument");
  // clouds / voxel maps may have been uploaded through another context (another module thread): device memory is shared,
  // and every producer call returns only after its stream has drained, so only the DEVICE has to match
  GB_REQUIRE(target->device == ctx->device && source->device == ctx->device, "cloud / voxel map live on another device");
  if (flags & GB_FACTOR_SURFACE_VALIDATION)
    GB_REQUIRE(source->normals != nullptr, "surface validation needs the source frame's normals on the device (PointCloudGPU::clone of a frame that has normals)");
  gb_factor* f = new (std::nothrow) gb_factor();
  if (!f) return GB_ERR_INTERNAL;
  f->ctx = ctx; f->target = target; f->source = source; f->flags = flags; f->single = nullptr; f->inlier_frac = -1.f; f->id = g_next_factor_id.fetch_add(1);
  ctx_retain(ctx);
  *out = f;
  return GB_OK;
}

// return a retired sweep's blocks to its context's pool (the caller holds the context lock and has drained the stream)
static void pool_put(gb_ctx* ctx, void* d, size_t d_cap, void* h, size_t h_cap) {
  if (!d && !h) return;
  if (ctx->pool.size() >= 64) {  // bounded: drop the smallest block
    size_t k = 0;
    for (size_t i = 1; i < ctx->pool.size(); i++) if (ctx->pool[i].d_cap < ctx->pool[k].d_cap) k = i;
    if (ctx->pool[k].d) cudaFree(ctx->pool[k].d);
    if (ctx->pool[k].h) cudaFreeHost(ctx->pool[k].h);
    ctx->pool.erase(ctx->pool.begin() + k);
  }
  ctx->pool.push_back({d, d_cap, h, h_cap});
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

static void sweep_free(gb_sweep* s) {
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
    pool_put(ctx, s->pool_d, s->pool_d_cap, s->pool_h, s->pool_h_cap);
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

// The work-item table of a sweep (descs[f].num_tiles / first_tile and the (factor, offset) list).
//   contiguous: items of tile_size consecutive points, factor-major (drawn from the queue by the persistent warps);
//   strided   : about one item per warp in total; factor f gets J_f items in proportion to its expected cost
//               n_f * (1 + 1.25 r_f) (r_f = inlier fraction of its last linearization, 0.5 if unknown; a hit costs ~2.2x a
//               miss), item j owning the 32-point rows j, j + J_f, ... of the source cloud.
static void build_items(gb_sweep* s, FactorDesc* descs, std::vector<int2>& tiles) {
  tiles.clear();
  const size_t F = s->F;
  if (!s->strided) {
    // TAIL TAPERING (guided self-scheduling): the last wave of a sweep leaves warps idle for up to one 2048-point item time --
    // little of a single-GPU sweep but a large share of one of 8 ranks' shard.  The factors that
    // hold the last ~1.5 item-times of work per warp get items of a quarter of the size, the last 0.4 a sixteenth.
    const double warps = (double)s->capacity * 8.0;
    uint64_t total = 0;
    for (size_t f = 0; f < F; f++) total += (uint64_t)descs[f].n;
    const bool taper = env_int("GB_TAPER", 1) != 0;
    const double ta = env_int("GB_TAPER_A", 150) * 0.01, tb = env_int("GB_TAPER_B", 40) * 0.01;
    const uint64_t tail16 = taper ? (uint64_t)(warps * s->tile_size * tb) : 0;  // last 0.4 item-times per warp: 1/16 items
    const uint64_t tail4 = taper ? (uint64_t)(warps * s->tile_size * ta) : 0;   // last 1.5 item-times per warp: 1/4 items
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
  const int min_rows = std::max(1, env_int("GB_MIN_ROWS", 4));
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
      const int jmax = std::max(1, rows / min_rows);
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

// After results have been fetched (the stream is idle): remember every factor's inlier fraction, and -- once per strided
// sweep -- re-size its item table from them.
static gb_status sweep_learn_inliers(gb_sweep* s) {
  for (size_t f = 0; f < s->F; f++) {
    gb_factor* fa = s->factors[f];
    if (fa && fa->source->n) fa->inlier_frac = (float)(s->h_out[f * GB_OUT_DOUBLES + 121] / (double)fa->source->n);
  }
  if (!s->strided || s->calibrated || s->stale) return GB_OK;
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

extern "C" gb_status gb_sweep_create(gb_ctx* ctx, size_t F, gb_factor* const* factors, const int32_t* pair_index, gb_sweep** out) {
  GB_REQUIRE(ctx && out, "null argument");
  GB_REQUIRE(F == 0 || factors, "null factor list");
  *out = nullptr;
  // validate before anything is allocated
  uint64_t total_pts = 0;
  for (size_t f = 0; f < F; f++) {
    GB_REQUIRE(factors[f], "null factor");
    GB_REQUIRE(factors[f]->source->device == ctx->device && factors[f]->target->device == ctx->device, "factor lives on another device");
    total_pts += factors[f]->source->n;
  }
  GB_LOCK(ctx);
  GB_CUDA(cudaSetDevice(ctx->device));
  gb_sweep* s = new (std::nothrow) gb_sweep();
  if (!s) return GB_ERR_INTERNAL;
  ctx_retain(ctx);
  s->ctx = ctx; s->F = F; s->factors.assign(factors, factors + F);
  s->d_descs = nullptr; s->d_tiles = nullptr; s->d_poses = nullptr; s->d_poses_eval = nullptr; s->d_accum = nullptr; s->d_done = nullptr; s->d_out = nullptr;
  s->h_poses_eval = nullptr; s->h_out = nullptr; s->d_slab = nullptr; s->num_pairs = 0;
  s->d_tile_ctr = nullptr; s->ctr_base = 0;
  s->peer = nullptr; s->d_pair_ptr = nullptr; s->d_pair_factors = nullptr; s->d_pair_done = nullptr; s->d_peer_tables = nullptr;
  s->num_tiles = 0; s->point_factors = 0; s->algorithmic_bytes = 0; s->key = 0; s->stale = false;
  s->h_pose_slot[0] = s->h_pose_slot[1] = nullptr; s->pose_ev[0] = s->pose_ev[1] = nullptr; s->pose_slot = 0;
  s->pool_d = nullptr; s->pool_d_cap = 0; s->pool_h = nullptr; s->pool_h_cap = 0;
  s->graph_exec = nullptr; s->graph_state = 0;

  // kernel generation and work-item policy
  // Kernel policy (A/B runs of the kernels, scripts/ab_sweep.py): small sweeps -- about one item per warp: an odometry
  // frame, a single pair -- run k_vgicp_sweep5 with one wave of equally expensive STRIDED items (faster on the odometry
  // workload); large sweeps run k_vgicp_sweep3 with contiguous 2048-point items drawn from the queue (its simpler hot loops
  // are faster there).  GB_KERNEL = 3 / 4 / 5 forces one kernel (4 = the bulk-async staged experiment).
  const int kv = env_int("GB_KERNEL", 0);
  s->stage_points = env_int("GB_STAGE", 128) == 64 ? 64 : 128;
  const int ctas_per_sm = (kv == 4 && s->stage_points == 64) ? 3 : 2;
  s->capacity = ctx->num_sms * ctas_per_sm;
  const uint64_t warps = (uint64_t)s->capacity * 8;
  const bool small = F > 0 && total_pts <= warps * 2048;
  s->kernel_version = (kv == 3 || kv == 4 || kv == 5) ? kv : (small ? 5 : 3);
  s->strided = (s->kernel_version == 5 && small && env_int("GB_STRIDED", 1)) ? 1 : 0;
  s->calibrated = false;
  s->pipe = env_int("GB_PIPE", 0) & 3;
  s->h_descs = nullptr; s->h_tiles = nullptr; s->tiles_cap = 0;
  {
    const int T = s->kernel_version == 4 ? s->stage_points : 32;
    int tile = env_int("GB_TILE", 0);
    if (tile <= 0) {
      // contiguous items: ~GB_ITEMS_PER_WARP items per warp (first one static, the rest drawn dynamically), between 128 and
      // 2048 points each
      const uint64_t ipw = (uint64_t)std::max(1, env_int("GB_ITEMS_PER_WARP", s->kernel_version == 4 ? 4 : 6));
      const uint64_t want = total_pts / (warps * ipw) + 1;
      tile = (int)std::min<uint64_t>(2048, std::max<uint64_t>(s->kernel_version == 4 ? T : 128, want));
    }
    s->tile_size = std::min(1 << 20, std::max(T, (tile + T - 1) / T * T));
  }

  std::vector<FactorDesc> descs(F);
  std::vector<int2> tiles;
  bool any_sv = false;
  for (size_t f = 0; f < F; f++) {
    const gb_factor* fa = factors[f];
    FactorDesc& D = descs[f];
    D.p0 = fa->source->p0; D.p1 = fa->source->p1; D.p2 = fa->source->p2;
    const bool sv = (fa->flags & GB_FACTOR_SURFACE_VALIDATION) != 0;
    D.normals = sv ? fa->source->normals : nullptr;
    any_sv = any_sv || sv;
    D.buckets = fa->target->buckets; D.voxels = fa->target->voxels;
    D.mask = (uint32_t)fa->target->num_buckets - 1u;
    D.max_scan = fa->target->max_scan;
    D.inv_res = fa->target->inv_res;
    D.n = (int)fa->source->n;
    D.pair = pair_index ? pair_index[f] : (int)f;
    s->h_pair.push_back(D.pair);
    D.flags = fa->flags;
    D.num_tiles = 1; D.chunk = s->tile_size;
    s->point_factors += (uint64_t)D.n;
    // B_f of SURVEY 8(d): 48 B per source point, 48 B per target voxel, 16 B per bucket, pose in + record out.
    // The bucket term is charged at the SMALLEST table that could hold the voxels (16384 doubled until >= V), not at
    // our deliberately sparse table (>= 8 V): padding we added for speed must not inflate the achieved-GB/s figure.
    uint64_t nb_ref = 16384;
    while (nb_ref < (uint64_t)fa->target->num_voxels) nb_ref *= 2;
    s->algorithmic_bytes += (uint64_t)D.n * (48 + (sv ? 12 : 0)) + (uint64_t)fa->target->num_voxels * 48 + nb_ref * 16 + 64 + 488;  // +12 B / point: the normals, when they are read
  }
  s->any_sv = any_sv;
  if (any_sv && s->kernel_version == 4) s->kernel_version = s->strided ? 5 : 3;  // the staged experiment does not carry normals
  build_items(s, descs.data(), tiles);
  s->num_tiles = (int)tiles.size();
  s->grid = std::max(1, std::min((s->num_tiles + 7) / 8, s->capacity));
  // ~64 items per accumulator copy: sweeps with few factors (an odometry frame, a single pair) would otherwise
  // serialise hundreds of fp64 reductions on the same addresses
  s->acc_slots = 1;
  while (F > 0 && s->acc_slots < 16 && (uint64_t)s->num_tiles > (uint64_t)F * 64 * s->acc_slots) s->acc_slots *= 2;

  if (F > 0) {
    // one device block, one pinned block -- taken from the context's pool when a retired sweep left a fitting one
    s->tiles_cap = std::max<size_t>(tiles.size(), s->strided ? (size_t)warps + F : 0);
    const size_t b_desc = align_up(sizeof(FactorDesc) * F, 256), b_tiles = align_up(sizeof(int2) * s->tiles_cap, 256), b_pose = align_up(sizeof(double) * 16 * F, 256);
    const size_t b_acc = align_up(sizeof(double) * GB_ACC_STRIDE * F * s->acc_slots, 256), b_done = align_up(sizeof(unsigned) * F + 16, 256), b_out = align_up(sizeof(double) * GB_OUT_DOUBLES * F, 256);
    const size_t total = b_desc + b_tiles + 2 * b_pose + b_acc + b_done + b_out;
    const size_t h_total = 3 * b_pose + b_out + b_desc + b_tiles;
    gb_pool_block blk{nullptr, 0, nullptr, 0};
    if (!pool_get(ctx, total, h_total, &blk)) {
      cudaError_t e = cudaMalloc(&blk.d, total);
      if (e != cudaSuccess) { delete s; ctx_release(ctx); gb_set_error("cudaMalloc(%zu): %s", total, cudaGetErrorString(e)); return GB_ERR_OUT_OF_MEMORY; }
      blk.d_cap = total;
      e = cudaMallocHost(&blk.h, h_total);
      if (e != cudaSuccess) { cudaFree(blk.d); delete s; ctx_release(ctx); gb_set_error("cudaMallocHost: %s", cudaGetErrorString(e)); return GB_ERR_OUT_OF_MEMORY; }
      blk.h_cap = h_total;
    }
    s->pool_d = blk.d; s->pool_d_cap = blk.d_cap; s->pool_h = blk.h; s->pool_h_cap = blk.h_cap;
    char* d = (char*)blk.d;
    s->d_descs = (FactorDesc*)d; d += b_desc;
    s->d_tiles = (int2*)d; d += b_tiles;
    s->d_poses = (double*)d; d += b_pose;
    s->d_poses_eval = (double*)d; d += b_pose;
    s->d_accum = (double*)d; d += b_acc;
    s->d_done = (unsigned*)d;
    s->d_tile_ctr = (unsigned long long*)(d + align_up(sizeof(unsigned) * F, 8));
    d += b_done;
    s->d_out = (double*)d;
    char* h = (char*)blk.h;
    s->h_pose_slot[0] = (double*)h; s->h_pose_slot[1] = (double*)(h + b_pose); s->h_poses_eval = (double*)(h + 2 * b_pose); s->h_out = (double*)(h + 3 * b_pose);
    s->h_descs = (FactorDesc*)(h + 3 * b_pose + b_out);
    s->h_tiles = (int2*)(h + 3 * b_pose + b_out + b_desc);
    memcpy(s->h_descs, descs.data(), sizeof(FactorDesc) * F);
    memcpy(s->h_tiles, tiles.data(), sizeof(int2) * tiles.size());
    cudaStream_t st = ctx->stream;
    cudaError_t e = cudaMemcpyAsync(s->d_descs, s->h_descs, sizeof(FactorDesc) * F, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(s->d_tiles, s->h_tiles, sizeof(int2) * tiles.size(), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(s->d_accum, 0, b_acc + b_done, st);
    for (int k = 0; k < 2 && e == cudaSuccess; k++) e = cudaEventCreateWithFlags(&s->pose_ev[k], cudaEventDisableTiming);
    if (e != cudaSuccess) { sweep_free(s); gb_set_error("sweep setup: %s", cudaGetErrorString(e)); return GB_ERR_CUDA; }
    // no synchronisation: the staging lives in the sweep's own pinned block, and everything that follows is stream ordered
  }
  {
    std::lock_guard<std::mutex> reg(g_registry_mu);
    for (gb_factor* f : s->factors) f->users.push_back(s);
  }
  *out = s;
  return GB_OK;
}
extern "C" gb_status gb_sweep_destroy(gb_sweep* s) { sweep_free(s); return GB_OK; }

extern "C" gb_status gb_sweep_attach_slab(gb_sweep* s, void* device_slab_f32, size_t num_pairs) {
  GB_REQUIRE(s, "null sweep");
  for (size_t f = 0; f < s->F && device_slab_f32; f++)
    GB_REQUIRE(s->h_pair[f] >= 0 && (size_t)s->h_pair[f] < num_pairs, "pair index out of range for this slab");
  s->d_slab = (float*)device_slab_f32;
  s->num_pairs = num_pairs;
  return GB_OK;
}

extern "C" gb_status gb_sweep_set_poses(gb_sweep* s, const double* T) {
  GB_REQUIRE(s && (s->F == 0 || T), "null argument");
  if (s->F == 0) return GB_OK;
  GB_LOCK(s->ctx);
  // double-buffered pinned staging: wait only for the H2D that read THIS slot two calls ago (normally long finished)
  const int k = s->pose_slot;
  s->pose_slot ^= 1;
  GB_CUDA(cudaEventSynchronize(s->pose_ev[k]));
  memcpy(s->h_pose_slot[k], T, sizeof(double) * 16 * s->F);
  GB_CUDA(cudaMemcpyAsync(s->d_poses, s->h_pose_slot[k], sizeof(double) * 16 * s->F, cudaMemcpyHostToDevice, s->ctx->stream));
  GB_CUDA(cudaEventRecord(s->pose_ev[k], s->ctx->stream));
  return GB_OK;
}
static gb_status sweep_set_eval_poses(gb_sweep* s, const double* T) {
  if (s->F == 0) return GB_OK;
  // the eval poses are only used by the blocking error calls (each ends with a stream sync): single buffer is safe
  memcpy(s->h_poses_eval, T, sizeof(double) * 16 * s->F);
  GB_CUDA(cudaMemcpyAsync(s->d_poses_eval, s->h_poses_eval, sizeof(double) * 16 * s->F, cudaMemcpyHostToDevice, s->ctx->stream));
  return GB_OK;
}
static gb_status sweep_launch(gb_sweep* s, int mode) {
  if (s->stale) { gb_set_error("a factor of this sweep has been destroyed"); return GB_ERR_INVALID_ARGUMENT; }
  GB_CUDA(cudaSetDevice(s->ctx->device));
  return gb_launch_sweep(s, mode);
}
extern "C" gb_status gb_sweep_launch(gb_sweep* s) {
  GB_REQUIRE(s, "null sweep");
  GB_LOCK(s->ctx);
  return sweep_launch(s, GB_MODE_LINEARIZE);
}
extern "C" gb_status gb_sweep_fetch(gb_sweep* s, gb_linearized6* out) {
  GB_REQUIRE(s && (s->F == 0 || out), "null argument");
  if (s->F == 0) return GB_OK;
  GB_LOCK(s->ctx);
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
  static const bool enabled = env_int("GB_GRAPH", 1) != 0;
  return enabled && s->graph_state >= 0 && s->strided && !s->peer && !s->d_slab && (unsigned long long)s->num_tiles <= (unsigned long long)s->grid * 8ull && s->F > 0;
}
static gb_status sweep_linearize(gb_sweep* s, const double* T, gb_linearized6* out) {
  if (!graph_eligible(s)) {
    GB_CHECK(gb_sweep_set_poses(s, T));
    GB_CHECK(sweep_launch(s, GB_MODE_LINEARIZE));
    return gb_sweep_fetch(s, out);
  }
  if (s->stale) { gb_set_error("a factor of this sweep has been destroyed"); return GB_ERR_INVALID_ARGUMENT; }
  gb_ctx* ctx = s->ctx;
  GB_CUDA(cudaSetDevice(ctx->device));
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
  GB_LOCK(s->ctx);
  return sweep_linearize(s, T, out);
}

extern "C" gb_status gb_factor_set_linearize(gb_ctx* ctx, size_t F, gb_factor* const* factors, const double* T, gb_linearized6* out) {
  GB_REQUIRE(ctx, "null ctx");
  if (F == 0) return GB_OK;
  GB_REQUIRE(factors && T && out, "null argument");
  GB_LOCK(ctx);
  gb_sweep* s = nullptr;
  GB_CHECK(cached_sweep(ctx, F, factors, &s));
  return sweep_linearize(s, T, out);
}

extern "C" gb_status gb_factor_set_error(gb_ctx* ctx, size_t F, gb_factor* const* factors, const double* T_lin, const double* T_eval, double* errors) {
  GB_REQUIRE(ctx, "null ctx");
  if (F == 0) return GB_OK;
  GB_REQUIRE(factors && T_lin && T_eval && errors, "null argument");
  GB_LOCK(ctx);
  gb_sweep* s = nullptr;
  GB_CHECK(cached_sweep(ctx, F, factors, &s));
  GB_CHECK(gb_sweep_set_poses(s, T_lin));
  GB_CHECK(sweep_set_eval_poses(s, T_eval));
  GB_CHECK(sweep_launch(s, GB_MODE_ERROR));
  GB_CUDA(cudaMemcpyAsync(s->h_out, s->d_out, sizeof(double) * GB_OUT_DOUBLES * F, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  for (size_t f = 0; f < F; f++) errors[f] = s->h_out[f * GB_OUT_DOUBLES + 120];
  return GB_OK;
}

static gb_status single_sweep(gb_factor* f, gb_sweep** out) {
  if (!f->single) GB_CHECK(gb_sweep_create(f->ctx, 1, &f, nullptr, &f->single));
  *out = f->single;
  return GB_OK;
}
extern "C" gb_status gb_vgicp_linearize(gb_factor* f, const double T[16], gb_linearized6* out) {
  GB_REQUIRE(f && T && out, "null argument");
  GB_LOCK(f->ctx);
  gb_sweep* s = nullptr;
  GB_CHECK(single_sweep(f, &s));
  return sweep_linearize(s, T, out);
}
extern "C" gb_status gb_vgicp_error(gb_factor* f, const double T_lin[16], const double T_eval[16], double* error) {
  GB_REQUIRE(f && T_lin && T_eval && error, "null argument");
  GB_LOCK(f->ctx);
  gb_sweep* s = nullptr;
  GB_CHECK(single_sweep(f, &s));
  GB_CHECK(gb_sweep_set_poses(s, T_lin));
  GB_CHECK(sweep_set_eval_poses(s, T_eval));
  GB_CHECK(sweep_launch(s, GB_MODE_ERROR));
  GB_CUDA(cudaMemcpyAsync(s->h_out, s->d_out, sizeof(double) * GB_OUT_DOUBLES, cudaMemcpyDeviceToHost, f->ctx->stream));
  GB_CUDA(cudaStreamSynchronize(f->ctx->stream));
  *error = s->h_out[120];
  return GB_OK;
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
static size_t peer_alloc_bytes(size_t num_pairs, int world) {
  return 2 * align_up(num_pairs * GB_SLAB_STRIDE * sizeof(float), 256) + align_up(sizeof(unsigned) * (size_t)world, 256);
}

extern "C" gb_status gb_peer_slab_create(gb_ctx* ctx, size_t num_pairs, int world, int rank, gb_peer_slab** out) {
  GB_REQUIRE(ctx && out, "null argument");
  GB_REQUIRE(world >= 1 && world <= GB_MAX_PEERS && rank >= 0 && rank < world, "world must be 1..8 and rank < world");
  GB_REQUIRE(num_pairs > 0, "num_pairs must be positive");
  *out = nullptr;
  GB_CUDA(cudaSetDevice(ctx->device));
  gb_peer_slab* ps = new (std::nothrow) gb_peer_slab();
  if (!ps) return GB_ERR_INTERNAL;
  ps->ctx = ctx; ps->num_pairs = num_pairs; ps->world = world; ps->rank = rank;
  ps->buf_floats = align_up(num_pairs * GB_SLAB_STRIDE * sizeof(float), 256) / sizeof(float);
  ps->local = nullptr; ps->step = 0; ps->parity = 0; ps->completed_parity = 0; ps->d_timeout = nullptr; ps->connected = (world == 1);
  // fused: the sweep's epilogue stores every finished row straight into all peers; deferred: rows go to the local buffer and
  // the exchange kernel pushes them (see gb_launch_peer_signal_wait).  The peer stores' cost to the sweep grows with the
  // rank count faster than the exchange kernel's extra time -> fused up to 4 ranks, deferred above.  GB_PEER_PUSH=fused|deferred forces one.
  {
    const char* e = getenv("GB_PEER_PUSH");
    ps->deferred = world > 4;
    if (e && !strcmp(e, "fused")) ps->deferred = false;
    if (e && !strcmp(e, "deferred")) ps->deferred = true;
  }
  ps->d_my_pairs = nullptr; ps->num_my_pairs = 0;
  for (int p = 0; p < GB_MAX_PEERS; p++) { ps->peer[p] = nullptr; ps->opened[p] = false; }
  const size_t bytes = peer_alloc_bytes(num_pairs, world);
  cudaError_t e = cudaMalloc((void**)&ps->local, bytes + 256);
  if (e != cudaSuccess) { delete ps; gb_set_error("cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e)); return GB_ERR_OUT_OF_MEMORY; }
  e = cudaMemsetAsync(ps->local, 0, bytes + 256, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) { cudaFree(ps->local); delete ps; gb_set_error("peer slab init: %s", cudaGetErrorString(e)); return GB_ERR_CUDA; }
  ps->d_timeout = (int*)(ps->local + bytes);
  ps->peer[rank] = ps->local;
  ps->h_pinned = nullptr;
  e = cudaMallocHost((void**)&ps->h_pinned, num_pairs * GB_SLAB_STRIDE * sizeof(float) + 64);
  if (e != cudaSuccess) { cudaFree(ps->local); delete ps; gb_set_error("cudaMallocHost: %s", cudaGetErrorString(e)); return GB_ERR_OUT_OF_MEMORY; }
  ctx_retain(ctx);
  *out = ps;
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_export(gb_peer_slab* ps, void* handle) {
  GB_REQUIRE(ps && handle, "null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == GB_IPC_HANDLE_BYTES, "IPC handle size");
  cudaIpcMemHandle_t h;
  GB_CUDA(cudaIpcGetMemHandle(&h, ps->local));
  memcpy(handle, &h, sizeof(h));
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_connect(gb_peer_slab* ps, const void* handles) {
  GB_REQUIRE(ps && handles, "null argument");
  GB_CUDA(cudaSetDevice(ps->ctx->device));
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
  if (!ps) return GB_OK;
  cudaSetDevice(ps->ctx->device);
  cudaStreamSynchronize(ps->ctx->stream);
  for (int p = 0; p < ps->world; p++)
    if (ps->opened[p]) cudaIpcCloseMemHandle(ps->peer[p]);
  if (ps->local) cudaFree(ps->local);
  if (ps->d_my_pairs) cudaFree(ps->d_my_pairs);
  if (ps->h_pinned) cudaFreeHost(ps->h_pinned);
  gb_ctx* ctx = ps->ctx;
  delete ps;
  ctx_release(ctx);
  return GB_OK;
}

extern "C" gb_status gb_sweep_attach_peer_slab(gb_sweep* s, gb_peer_slab* ps) {
  GB_REQUIRE(s, "null sweep");
  if (!ps) { s->peer = nullptr; return GB_OK; }
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
  GB_CUDA(cudaSetDevice(s->ctx->device));
  GB_CUDA(cudaStreamSynchronize(s->ctx->stream));
  if (s->d_pair_ptr) { GB_CUDA(cudaFree(s->d_pair_ptr)); s->d_pair_ptr = nullptr; }
  const size_t b_ptr = align_up(sizeof(int) * (P + 1), 256), b_fac = align_up(sizeof(int) * std::max<size_t>(1, s->F), 256), b_done = align_up(sizeof(unsigned) * P, 256);
  char* d = nullptr;
  GB_CUDA(cudaMalloc((void**)&d, b_ptr + b_fac + b_done + 2 * sizeof(PeerPush)));
  s->d_pair_ptr = (int*)d; s->d_pair_factors = (int*)(d + b_ptr); s->d_pair_done = (unsigned*)(d + b_ptr + b_fac);
  s->d_peer_tables = (PeerPush*)(d + b_ptr + b_fac + b_done);
  PeerPush tabs[2];
  memset(tabs, 0, sizeof(tabs));
  for (int par = 0; par < 2; par++) {
    if (ps->deferred) {  // the sweep writes this rank's buffer only
      tabs[par].world = 1;
      tabs[par].base[0] = reinterpret_cast<float*>(ps->local) + (size_t)par * ps->buf_floats;
    } else {
      tabs[par].world = ps->world;
      for (int p = 0; p < ps->world; p++) tabs[par].base[p] = reinterpret_cast<float*>(ps->peer[p]) + (size_t)par * ps->buf_floats;
    }
    tabs[par].pair_ptr = s->d_pair_ptr; tabs[par].pair_factors = s->d_pair_factors; tabs[par].pair_done = s->d_pair_done;
  }
  GB_CUDA(cudaMemcpy(s->d_peer_tables, tabs, sizeof(tabs), cudaMemcpyHostToDevice));
  GB_CUDA(cudaMemcpy(s->d_pair_ptr, ptr.data(), sizeof(int) * (P + 1), cudaMemcpyHostToDevice));
  if (s->F) GB_CUDA(cudaMemcpy(s->d_pair_factors, fac.data(), sizeof(int) * s->F, cudaMemcpyHostToDevice));
  GB_CUDA(cudaMemset(s->d_pair_done, 0, b_done));
  // the pairs this sweep owns (one sweep per peer slab): the rows the exchange kernel copies to the peers
  std::vector<int> mine;
  for (size_t k = 0; k < P; k++) if (ptr[k + 1] > ptr[k]) mine.push_back((int)k);
  if (ps->d_my_pairs) { GB_CUDA(cudaFree(ps->d_my_pairs)); ps->d_my_pairs = nullptr; }
  ps->num_my_pairs = (int)mine.size();
  if (!mine.empty()) {
    GB_CUDA(cudaMalloc((void**)&ps->d_my_pairs, sizeof(int) * mine.size()));
    GB_CUDA(cudaMemcpy(ps->d_my_pairs, mine.data(), sizeof(int) * mine.size(), cudaMemcpyHostToDevice));
  }
  s->peer = ps;
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_signal_wait(gb_peer_slab* ps) {
  GB_REQUIRE(ps, "null peer slab");
  GB_REQUIRE(ps->connected, "gb_peer_slab_connect has not been called");
  GB_CUDA(cudaSetDevice(ps->ctx->device));
  ps->step++;
  GB_CHECK(gb_launch_peer_signal_wait(ps));
  ps->completed_parity = ps->parity;
  ps->parity ^= 1;
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_device_ptr(gb_peer_slab* ps, void** device_ptr) {
  GB_REQUIRE(ps && device_ptr, "null argument");
  *device_ptr = ps->local + (size_t)ps->completed_parity * ps->buf_floats * sizeof(float);
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_fetch_async(gb_peer_slab* ps, const float** host_ptr) {
  GB_REQUIRE(ps, "null peer slab");
  const size_t bytes = ps->num_pairs * GB_SLAB_STRIDE * sizeof(float);
  GB_CUDA(cudaMemcpyAsync(ps->h_pinned, ps->local + (size_t)ps->completed_parity * ps->buf_floats * sizeof(float), bytes, cudaMemcpyDeviceToHost, ps->ctx->stream));
  GB_CUDA(cudaMemcpyAsync((char*)ps->h_pinned + bytes, ps->d_timeout, sizeof(int), cudaMemcpyDeviceToHost, ps->ctx->stream));
  if (host_ptr) *host_ptr = ps->h_pinned;
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_fetch(gb_peer_slab* ps, float* host) {
  GB_REQUIRE(ps && host, "null argument");
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
  GB_CUDA(cudaSetDevice(ctx->device));
  const size_t b_desc = align_up(sizeof(FactorDesc) * T, 256), b_pose = align_up(sizeof(double) * 16 * T, 256);
  char* h = nullptr;
  char* d = nullptr;
  GB_CHECK(gb_ctx_pinned(ctx, b_desc + b_pose + 256, (void**)&h));
  GB_CHECK(gb_ctx_scratch(ctx, b_desc + b_pose + 256, (void**)&d));
  FactorDesc* hd = (FactorDesc*)h;
  for (size_t t = 0; t < T; t++) {
    GB_REQUIRE(targets[t], "null target");
    FactorDesc& D = hd[t];
    memset(&D, 0, sizeof(D));
    D.p0 = source->p0; D.p1 = source->p1; D.p2 = source->p2;
    D.buckets = targets[t]->buckets; D.voxels = targets[t]->voxels;
    D.mask = (uint32_t)targets[t]->num_buckets - 1u; D.max_scan = targets[t]->max_scan; D.inv_res = targets[t]->inv_res; D.n = (int)source->n;
  }
  memcpy(h + b_desc, deltas, sizeof(double) * 16 * T);
  int* h_count = (int*)(h + b_desc + b_pose);
  int* d_count = (int*)(d + b_desc + b_pose);
  GB_CUDA(cudaMemcpyAsync(d, h, b_desc + b_pose, cudaMemcpyHostToDevice, ctx->stream));
  GB_CUDA(cudaMemsetAsync(d_count, 0, sizeof(int), ctx->stream));
  GB_CHECK(gb_launch_overlap(ctx, (int)T, (const FactorDesc*)d, (const double*)(d + b_desc), (int)source->n, d_count));
  GB_CUDA(cudaMemcpyAsync(h_count, d_count, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  *overlap = (double)*h_count / (double)source->n;
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
  GB_CUDA(cudaSetDevice(ctx->device));
  return gb_covariances_impl(ctx, n, xyzw, neighbors, k_correspondences, k_neighbors, normals4, cov4x4);
}
extern "C" gb_status gb_find_neighbors(gb_ctx* ctx, size_t n, const double* xyzw, int k, int32_t* neighbors) {
  GB_REQUIRE(ctx, "null ctx");
  if (n == 0) return GB_OK;
  GB_REQUIRE(xyzw && neighbors && k > 0, "null argument");
  GB_LOCK(ctx);
  GB_CUDA(cudaSetDevice(ctx->device));
  // >= 4096 points: exact search on a pyramid of hash grids (one Morton sort, cell size 0.25 m x 4^level);
  // GB_KNN=grid selects the round-1 single-level grid, GB_KNN=brute the tiled brute force
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
  GB_LOCK(ctx);
  GB_CUDA(cudaSetDevice(ctx->device));
  gb_cloud* c = nullptr;
  if (out_cloud) {
    c = new (std::nothrow) gb_cloud();
    if (!c) return GB_ERR_INTERNAL;
    c->device = ctx->device; c->n = 0; c->base = nullptr; c->bytes = 0;
    c->p0 = nullptr; c->p1 = nullptr; c->p2 = nullptr; c->normals = nullptr; c->perm = nullptr; c->inv_perm = nullptr;
  }
  gb_status st = gb_merge_frames_impl(ctx, (int)K, frames, poses, resolution, target, seed, out_xyzw, out_cov4x4, num_out, c);
  if (st == GB_OK) {
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { gb_set_error("gb_merge_frames: %s", cudaGetErrorString(e)); st = GB_ERR_CUDA; }
  }
  if (st != GB_OK) { if (c) { gb_dev_free(ctx->device, c->base); delete c; } return st; }
  if (out_cloud) *out_cloud = c;
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
  GB_REQUIRE(P->k_correspondences > 0, "k_correspondences must be positive");
  GB_REQUIRE(P->k_neighbors_cov >= 0 && P->k_neighbors_cov <= P->k_correspondences, "k_neighbors_cov must be in [0, k_correspondences]");
  GB_REQUIRE(!P->enable_outlier_removal || (P->outlier_removal_k > 0 && P->outlier_removal_k <= 32), "outlier_removal_k must be in [1, 32]");
  GB_REQUIRE(P->crop_bbox_frame >= 0 && P->crop_bbox_frame <= 2, "crop_bbox_frame must be 0 (off), 1 (lidar) or 2 (imu)");
  if (n == 0) return GB_OK;
  GB_REQUIRE(xyzw, "null points");
  GB_LOCK(ctx);
  GB_CUDA(cudaSetDevice(ctx->device));
  gb_cloud* c = nullptr;
  if (P->estimate_covariances) {
    c = new (std::nothrow) gb_cloud();
    if (!c) return GB_ERR_INTERNAL;
    c->device = ctx->device; c->n = 0; c->base = nullptr; c->bytes = 0;
    c->p0 = nullptr; c->p1 = nullptr; c->p2 = nullptr; c->normals = nullptr; c->perm = nullptr; c->inv_perm = nullptr;
  }
  gb_status st = gb_preprocess_impl(ctx, n, xyzw, times, intensities, P, out, c);
  if (st == GB_OK) {
    cudaError_t e = cudaStreamSynchronize(ctx->stream);  // the cloud is complete when the call returns (it may be used from another context)
    if (e != cudaSuccess) { gb_set_error("gb_preprocess: %s", cudaGetErrorString(e)); st = GB_ERR_CUDA; }
  }
  if (st != GB_OK) { if (c) { gb_dev_free(ctx->device, c->base); delete c; } return st; }
  out->cloud = c;
  return GB_OK;
}
extern "C" gb_status gb_voxelgrid_sampling(gb_ctx* ctx, size_t n, const double* xyzw, const double* times, const double* intensities, double resolution, double* out_xyzw, double* out_times, double* out_intensities, size_t* num_out) {
  GB_REQUIRE(ctx && num_out, "null argument");
  *num_out = 0;
  if (n == 0) return GB_OK;
  GB_REQUIRE(xyzw && out_xyzw && resolution > 0.0, "null argument");
  GB_CUDA(cudaSetDevice(ctx->device));
  return gb_voxelgrid_sampling_impl(ctx, n, xyzw, times, intensities, resolution, out_xyzw, out_times, out_intensities, num_out);
}
