// gb_internal.cuh -- shared declarations of libglim_b200.so (not part of the public boundary).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <cassert>
#include <atomic>
#include <initializer_list>
#include <memory>
#include <mutex>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "../../include/glim_b200.h"
#include "gb_segment_math.cuh"  // gb_frame, gb_frame_of (shared with the host-compiled CPU test of the segmentation arithmetic)

// ---------------------------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------------------------
void gb_set_error(const char* fmt, ...);
#define GB_CUDA(expr)                                                                         \
  do {                                                                                        \
    cudaError_t e__ = (expr);                                                                 \
    if (e__ != cudaSuccess) {                                                                 \
      gb_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return e__ == cudaErrorMemoryAllocation ? GB_ERR_OUT_OF_MEMORY : GB_ERR_CUDA;           \
    }                                                                                         \
  } while (0)
#define GB_CHECK(st)                 \
  do {                               \
    gb_status s__ = (st);            \
    if (s__ != GB_OK) return s__;    \
  } while (0)
#define GB_REQUIRE(cond, msg)                       \
  do {                                              \
    if (!(cond)) {                                  \
      gb_set_error("invalid argument: %s", msg);    \
      return GB_ERR_INVALID_ARGUMENT;               \
    }                                               \
  } while (0)

// ---------------------------------------------------------------------------------------------
// HBM data layout (DESIGN.md "Data layout")
// ---------------------------------------------------------------------------------------------
// Source cloud: three planes, 36 B / point, every warp access fully coalesced:
//   p0[i] = {x, y, z, c00}   p1[i] = {c01, c02, c11, c12}   p2[i] = c22
// Voxel map: open-addressing table of 16-byte buckets {cx, cy, cz, voxel index (-1 = empty)} and
// 48-byte voxel records (3 x float4): {mx, my, mz, c00} {c01, c02, c11, c12} {c22, num_points, 0, 0}.
struct gb_cloud {
  int device = 0;   // clouds / voxel maps do NOT keep their creating context: they outlive it when frames migrate between threads
  size_t n = 0;
  float4* p0 = nullptr;
  float4* p1 = nullptr;
  float* p2 = nullptr;
  float4* normals = nullptr;  // {nx, ny, nz, 0} or nullptr: in `base` when uploaded with the cloud, else in `n_base`
  void* n_base = nullptr;     // the normals of gb_cloud_estimate_normals on a cloud built without them: a pool block of their own
  // Points are stored in Morton order of their 1/16 m cell (gather locality of the sweep kernel: lanes of a warp
  // then hit the same few voxels).  perm[j] = original index of stored point j, inv_perm = its inverse; nullptr = identity.
  int* perm = nullptr;
  int* inv_perm = nullptr;
  void* base = nullptr;       // one allocation
  // The time table of gb_cloud_add_times (gb_kernels_ct.cu), or none (num_entries == 0).  Entry b holds the original indices
  // [t_starts[b], t_starts[b + 1]) at normalized time t_tau[b]; the stored slots are reached through inv_perm.  The device
  // copy is one block of its own (ct_table_layout), from the device pool; only the CT factor reads it.
  int num_entries = 0;
  double t_first = 0.0, t_last = 0.0;  // t_0 and t_{B-1}
  std::vector<int> h_starts;           // host copies
  std::vector<double> h_tau;
  int* t_starts = nullptr;
  double* t_tau = nullptr;
  void* t_base = nullptr;
  bool covs = false;  // the cloud carries covariances (an upload with cov4x4, a preprocessed, merged or deskewed frame)
  // The FPFH features of gb_cloud_estimate_fpfh (gb_kernels_global.cu), or none (fpfh == nullptr): N x 33 fp32 in the caller's
  // point order, one block of their own from the device pool; only the global registration entry points read them.
  float* fpfh = nullptr;
  void* f_base = nullptr;
};

// A map is one of four kinds, fixed at creation.  Every entry point that takes a map checks the kind it accepts.
enum gb_map_kind {
  GB_MAP_BUILT,        // gb_voxelmap_build: records and table only
  GB_MAP_INCREMENTAL,  // gb_voxelmap_create_incremental / gb_voxelmap_insert
  GB_MAP_IVOX,         // gb_ivox_create / gb_ivox_insert: the gb_ivox handle is the map itself
  GB_MAP_POINTS,       // gb_point_grid_build: every point of a cloud; the gb_point_grid handle is the map itself
};
struct gb_voxelmap {
  int device = 0;
  gb_map_kind kind = GB_MAP_BUILT;
  float resolution = 0.f, inv_res = 0.f;  // the fp32 lookup rule of every sweep and overlap
  int max_scan = 0;
  int num_voxels = 0, num_buckets = 0;
  int num_dropped_points = 0;
  int4* buckets = nullptr;
  float4* voxels = nullptr;   // 3 float4 per record: one record per voxel, or per stored point of an iVox
  void* base = nullptr;
  // Incremental maps and iVoxes also keep, in `base` behind the records, each voxel's packed key and the insert that last
  // touched it.  An incremental map adds each voxel's point count and fp64 sums (Sigma q: 3, Sigma C: 6 unique entries).  An
  // iVox's records are its stored points ({x y z c00} {c01 c02 c11 c12} {c22, 1, 0, 0}), voxel-major in ascending packed-key
  // order, and it adds each voxel's cell {first point, count}.  A built map keeps none of this and its version stays 0.
  uint64_t version = 0;        // bumped by every insert: sweeps re-read the target's buckets / records when it changed
  double key_inv_res = 0.0;    // an insert's fp64 key rule floor(q * key_inv_res), fixed at creation
  int init_buckets = 0;
  double drop_rate = 0.0;      // 0 for an iVox: every voxel is found
  int lru_horizon = 0, lru_clear_cycle = 10, lru_counter = 0;
  size_t num_points = 0;       // the points the voxels hold
  unsigned long long* vkeys = nullptr;  // ascending: the voxel numbering
  int* vstamp = nullptr;
  int* vn = nullptr;           // incremental
  double* vsums = nullptr;     // incremental, 9 per voxel: q.x q.y q.z c00 c01 c02 c11 c12 c22
  int2* cells = nullptr;       // iVox
  // iVox parameters: resolution and inv_res are (float)ivox_resolution and (float)(1 / ivox_resolution)
  double ivox_resolution = 0.0, min_dist = 0.0;
  int max_points = 10, mode = 1;
  // A point grid's records are every point of its cloud ({x y z c00} {c01 c02 c11 c12} {c22, 1, original index bits, 0}) in
  // ascending (packed key, original index) order, the points without a key last; it keeps cells and keys like an iVox (in
  // `base`, laid out by grid_layout) and is never inserted into: its version stays 0.  resolution and inv_res are
  // (float)cell_size and (float)(1 / cell_size).
  double cell_size = 0.0;
  int key_extent = 0;          // max over cells and axes of max(|k|, |k + 1|): bounds |q * inv_res| for the search width
};
// the stored entries an insert groups ahead of the frame's points: one per voxel, or one per stored point of an iVox
inline size_t gb_stored_entries(const gb_voxelmap* m) { return m->kind == GB_MAP_IVOX ? m->num_points : (size_t)m->num_voxels; }
// the handle of an iVox is its gb_voxelmap (gb_ivox stays an incomplete type)
inline gb_voxelmap* ivox_map(gb_ivox* h) { return reinterpret_cast<gb_voxelmap*>(h); }
inline const gb_voxelmap* ivox_map(const gb_ivox* h) { return reinterpret_cast<const gb_voxelmap*>(h); }
// likewise for a point grid (gb_point_grid stays an incomplete type)
inline gb_voxelmap* grid_map(gb_point_grid* h) { return reinterpret_cast<gb_voxelmap*>(h); }
inline const gb_voxelmap* grid_map(const gb_point_grid* h) { return reinterpret_cast<const gb_voxelmap*>(h); }
// The target class of a pose factor: a sweep or call holds one.  0: voxel maps (VGICP), 1: iVoxes (GICP), 2: point grids (GICP).
inline int gb_target_class(const gb_voxelmap* m) { return m->kind == GB_MAP_IVOX ? 1 : (m->kind == GB_MAP_POINTS ? 2 : 0); }

// device-side factor descriptor (80 B)
struct FactorDesc {
  const float4* p0;
  const float4* p1;
  const float* p2;
  const float4* normals;  // source normals, non-null only when surface validation is on for this factor
  const int4* buckets;
  const float4* voxels;
  uint32_t mask;
  int max_scan;
  float inv_res;
  int n;
  int pair;
  int flags;
  int num_tiles;
  int chunk;       // sweep3: points per item of THIS factor (the last factors of a sweep get smaller items: tail tapering)
};
static_assert(sizeof(FactorDesc) == 80, "FactorDesc size");
// The rest of a GICP factor's descriptor (k_gicp_sweep, k_gicp_grid_sweep): its FactorDesc carries the iVox's or point grid's
// table (buckets, mask, max_scan, inv_res) and its point records (voxels); this adds the cells, the correspondence bound and
// the searched offsets.
struct GicpDesc {
  const int2* cells;
  float max_corr2;   // (float)(max_correspondence_distance^2)
  int num_offsets;   // neighbor_voxel_mode (iVox), or the search half-width m (point grid)
};
static_assert(sizeof(GicpDesc) == 16, "GicpDesc size");
// a GICP factor's target part (gb_api.cu): the iVox's or point grid's table and point records in D, the rest in G
void desc_target_gicp(FactorDesc& D, GicpDesc& G, const gb_factor* fa);

// A factor is one of three kinds, fixed at creation.  A pose factor (gb_vgicp_factor_create, gb_gicp_factor_create) has one
// unknown pose and goes through sweeps; a CT factor (gb_ct_gicp_factor_create) has two and only the gb_ct_* entry points
// take it; a plane factor (gb_plane_evm_factor_create) has one per key and only the gb_plane_evm_* entry points take it.
// gb_sweep_create takes pose factors only, and so every consumer of sweeps refuses the other kinds.
enum gb_factor_kind {
  GB_FACTOR_POSE,
  GB_FACTOR_CT,
  GB_FACTOR_PLANE_EVM,
};
struct gb_factor {
  gb_factor_kind kind = GB_FACTOR_POSE;
  gb_ctx* ctx = nullptr;
  const gb_voxelmap* target = nullptr;  // a built or incremental map (VGICP), an iVox or a point grid (GICP)
  float max_corr2 = 0.f;                // GICP: (float)(max_correspondence_distance^2)
  int grid_m = 0;                       // GICP or ICP on a point grid: the search half-width m (grid_half_width)
  bool icp = false;                     // a point-to-point ICP factor on a point grid (gb_icp_grid_factor_create)
  const gb_cloud* source = nullptr;
  int flags = 0;
  gb_sweep* single = nullptr;  // lazily created 1-factor sweep
  float inlier_frac = -1.f;    // inlier fraction of the last linearization (< 0: unknown) -- sizes the work items of the next sweep
  uint64_t id = 0;             // process-wide unique
  std::vector<gb_sweep*> users;  // sweeps (of any context) that reference this factor; guarded by the registry mutex
  // A plane factor keeps everything on the host and borrows no cloud: per key the caller's frame index and the moments
  // {N, mean, scatter} (GB_PLANE_MOMENTS doubles, gb_plane_math.cuh) of its points, the offset o and the point count.
  std::vector<int32_t> plane_frames;
  std::vector<double> plane_moments;
  double plane_offset[3] = {0.0, 0.0, 0.0};
  size_t plane_points = 0;
};
// The class of a pose factor: a sweep or call holds one.  gb_target_class's 0 (VGICP), 1 and 2 (GICP), or 3: ICP on point grids.
inline int gb_factor_class(const gb_factor* f) { return f->icp ? 3 : gb_target_class(f->target); }

#define GB_MAX_PEERS 8
// device-resident parameter block of the fused result exchange (one per step parity)
struct PeerPush {
  int world;                      // 0 = disabled
  float* base[GB_MAX_PEERS];      // every rank's slab buffer of the current step parity, as mapped on THIS device
  const int* pair_ptr;            // CSR over global pair ids -> local factor indices (empty for pairs owned elsewhere)
  const int* pair_factors;
  unsigned* pair_done;            // per-pair tickets, self-cleaning
};

struct gb_peer_slab {
  gb_ctx* ctx = nullptr;
  size_t num_pairs = 0;
  int world = 0, rank = 0;
  char* local = nullptr;          // cudaMalloc, laid out by gb_peer_layout
  char* peer[GB_MAX_PEERS] = {};  // every rank's allocation as mapped here (peer[rank] == local)
  bool opened[GB_MAX_PEERS] = {};
  unsigned step = 0;              // last launched step
  int parity = 0;                 // buffer written by the NEXT launch
  int completed_parity = 0;       // buffer completed by the last signal_wait
  float* h_pinned = nullptr;      // the rows and the timeout word of the fetches (peer_fetch_layout, gb_peer.cu)
  bool connected = false;
  // deferred exchange (default): the sweep stores finished pair rows into the LOCAL buffer only; the exchange kernel that
  // follows it copies this rank's rows to every peer (one CTA per peer) before it publishes the completion flags
  bool deferred = false;
  int* d_my_pairs = nullptr;      // pair ids owned by the attached sweep
  int num_my_pairs = 0;
};

#define GB_ACC_STRIDE 32      // doubles per factor in the accumulation buffer (29 used)
#define GB_OUT_DOUBLES 122    // gb_linearized6

struct gb_pool_block { void* d = nullptr; size_t d_cap = 0; void* h = nullptr; size_t h_cap = 0; };

struct gb_sweep {
  gb_ctx* ctx = nullptr;
  size_t F = 0;
  std::vector<gb_factor*> factors;
  FactorDesc* d_descs = nullptr;
  int2* d_tiles = nullptr;          // work items {factor, first point}, factor-major
  double* d_poses = nullptr;        // F x 16 (T_lin)
  double* d_poses_eval = nullptr;   // F x 16 (error mode)
  double* d_accum = nullptr;        // F x acc_slots x GB_ACC_STRIDE, zero between sweeps (self-cleaning)
  int acc_slots = 0;                // power of two: copies of each factor's accumulator (spreads same-address atomics of few-factor sweeps)
  unsigned* d_done = nullptr;       // F tickets, zero between sweeps
  unsigned long long* d_tile_ctr = nullptr;  // dynamic tile queue head, monotonic across launches
  unsigned long long ctr_base = 0;           // value of the counter at the start of the next launch
  double* d_out = nullptr;          // F x 122
  double* h_poses_eval = nullptr;   // pinned
  double* h_out = nullptr;          // pinned
  float* d_slab = nullptr;
  size_t num_pairs = 0;
  gb_peer_slab* peer = nullptr;     // fused exchange target (or nullptr)
  int* d_pair_ptr = nullptr;        // CSR pair -> factors (device), built when a peer slab is attached
  int* d_pair_factors = nullptr;
  unsigned* d_pair_done = nullptr;
  PeerPush* d_peer_tables = nullptr;  // [2]: one per step parity
  std::vector<int> h_pair;            // pair id per factor
  int num_tiles = 0, tile_size = 0, grid = 0;  // work items, points per sweep3 item, CTAs
  // 5 = small sweeps: strided items, item j of a factor owns its rows j, j + J, ... (about one item per warp; see k_vgicp_sweep5);
  // 3 = large sweeps: a queue of contiguous items.  GB_KERNEL=3/5 forces one; the item table follows the kernel.
  int kernel_version = 0;
  bool any_sv = false;              // some factor of the sweep has surface validation on
  bool calibrated = false;          // sweep5: the item table has been re-sized from measured inlier fractions
  int capacity = 0;                 // CTAs of a full grid
  FactorDesc* h_descs = nullptr;    // pinned copies (re-uploaded when the item table is re-sized)
  int2* h_tiles = nullptr;
  size_t tiles_cap = 0;
  uint64_t point_factors = 0, algorithmic_bytes = 0;
  uint64_t key = 0;                 // cache key
  bool stale = false;               // a factor of this sweep was destroyed: it can no longer be launched
  double* h_pose_slot[2] = {};      // pinned pose staging, double buffered (no stream sync in gb_sweep_set_poses)
  cudaEvent_t pose_ev[2] = {};      // recorded after the H2D that read the slot
  int pose_slot = 0;
  cudaGraphExec_t graph_exec = nullptr;  // small sweeps: poses H2D -> kernel -> records D2H as ONE graph launch (gb_factor_set_linearize)
  int graph_state = 0;              // 0 = not built, 1 = valid, -1 = capture failed (plain launches from then on)
  gb_pool_block blk;                // the device and pinned blocks, laid out by sweep_layout; back to the context's pool at the end
  bool any_incremental = false;     // some target is not a built map: its descriptor may go stale (gb_voxelmap_insert, gb_ivox_insert)
  std::vector<uint64_t> target_versions;  // per factor: the target version its descriptor was written from
  // GICP sweeps (every factor on an iVox, or every factor on a point grid; a sweep holds one target class): k_gicp_sweep or
  // k_gicp_grid_sweep over sweep5's strided items, with the GICP half of each descriptor next to the FactorDesc table
  bool gicp = false;
  bool point_grid = false;          // a GICP or ICP sweep over point grids
  bool icp = false;                 // an ICP sweep (k_icp_grid_sweep; every factor from gb_icp_grid_factor_create)
  GicpDesc* d_gdescs = nullptr;
  GicpDesc* h_gdescs = nullptr;
};

// A context's grow-only buffer: device scratch or pinned host staging.  What it holds is valid until the next gb_carve on it.
struct gb_arena {
  bool host = false;  // cudaMallocHost, else cudaMalloc
  void* base = nullptr;
  size_t cap = 0;
};

struct gb_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  int num_sms = 0;
  gb_arena scratch;
  gb_arena pinned{true};
  uint64_t launches = 0;     // gb_ctx_kernel_launches: written by gb_launch, GB_CUB and the graph path of sweep_linearize only
  std::atomic<int> refs{0};  // owner + live factors / sweeps / peer slabs; the context is torn down when the last one lets go
  std::vector<gb_sweep*> sweep_cache;
  std::vector<gb_pool_block> pool;  // device + pinned blocks of retired sweeps, reused by the next gb_sweep_create
  // A context may be driven from more than one host thread (a frame cloned by the odometry thread is later used by the
  // sub-mapping thread): every entry point that touches the stream, the scratch arena, the caches or the launch counter
  // enters through GB_ENTER, which takes this lock.  Recursive: an entry point may call another (gb_vgicp_align creates a
  // sweep).  No entry point holds the locks of two contexts.
  std::recursive_mutex mu;
};
#define GB_LOCK(ctx) std::lock_guard<std::recursive_mutex> gb_lock__((ctx)->mu)
// The first statement of an entry point after its argument checks: the context's lock for the rest of the call, and the
// context's device as the thread's current device.
#define GB_ENTER(ctx) \
  GB_LOCK(ctx);       \
  GB_CUDA(cudaSetDevice((ctx)->device))

// Every kernel launch of the library: kernel<<<grid, block, smem, ctx->stream>>>(args...), its launch error read at once
// (an invalid configuration or a missing image is reported by the call that made it, naming the kernel) and, on success,
// one count in ctx->launches.  The triple-chevron launch converts each argument to the kernel's parameter type, as a
// direct launch would.
template <typename... P, typename... A>
gb_status gb_launch(gb_ctx* ctx, const char* name, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A&&... args) {
  kernel<<<grid, block, smem, ctx->stream>>>(std::forward<A>(args)...);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    gb_set_error("launch of %s failed: %s", name, cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? GB_ERR_OUT_OF_MEMORY : GB_ERR_CUDA;
  }
  ctx->launches++;
  return GB_OK;
}
// The same for a cooperative kernel (one that synchronises its whole grid with cooperative_groups' grid.sync()): launched by
// cudaLaunchCooperativeKernel, which refuses a grid larger than can be resident at once instead of letting it deadlock.  The
// arguments are converted to the kernel's parameter types first, as a direct launch would.
struct gb_cooperative_t {};
constexpr gb_cooperative_t gb_cooperative{};
template <typename... P, typename... A>
gb_status gb_launch(gb_ctx* ctx, const char* name, gb_cooperative_t, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A&&... args) {
  std::tuple<P...> params(std::forward<A>(args)...);
  const cudaError_t e = std::apply([&](auto&... p) {
    void* argv[] = {(void*)&p..., nullptr};
    return cudaLaunchCooperativeKernel((const void*)kernel, grid, block, argv, smem, ctx->stream);
  }, params);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    gb_set_error("cooperative launch of %s failed: %s", name, cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? GB_ERR_OUT_OF_MEMORY : GB_ERR_CUDA;
  }
  ctx->launches++;
  return GB_OK;
}
// Every cub device-wide call of the library with temporary storage: fn(storage, bytes, args..., ctx->stream), counted as
// one launch (a radix sort is several kernels; the counter's unit is the call).  The size queries of gb_cub_temp_bytes
// launch nothing and do not come here.
#define GB_CUB(ctx, fn, storage, bytes, ...)                         \
  do {                                                               \
    size_t cub_bytes__ = (bytes);                                    \
    GB_CUDA(fn(storage, cub_bytes__, __VA_ARGS__, (ctx)->stream));   \
    (ctx)->launches++;                                               \
  } while (0)

// Device blocks of clouds / voxel maps come from a process-wide pool (a frame costs one cloud + two maps = five allocations;
// cudaMalloc / cudaFree are 50-200 us each and cudaFree synchronises the device).  gb_dev_free waits for the streams of
// every live context of the device (what the implicit synchronisation of cudaFree used to guarantee) and keeps the block.
cudaError_t gb_dev_malloc(int device, size_t bytes, void** out);
void gb_dev_free(int device, void* p);
// A pool block is taken only by gb_dev_carve, into an owner made for its device, which returns it to the pool on every exit
// before hand_over(field).  That swaps it into a handle's field on the same device, and the owner returns the field's old block
// instead.  Only cloud_free and voxelmap_free return a handle's blocks.  An owner assigned to returns the block it held.
struct gb_dev_block {
  int device;
  void* base = nullptr;
  explicit gb_dev_block(int device) : device(device) {}
  gb_dev_block(gb_dev_block&& o) noexcept : device(o.device), base(std::exchange(o.base, nullptr)) {}
  gb_dev_block& operator=(gb_dev_block o) noexcept { std::swap(device, o.device); std::swap(base, o.base); return *this; }  // o returns the old block
  ~gb_dev_block() { gb_dev_free(device, base); }
  template <typename T> void hand_over(T*& field) { void* old = field; field = (T*)base; base = old; }
};
gb_status gb_arena_reserve(gb_ctx* ctx, gb_arena& a, size_t bytes);  // a.base holds at least `bytes` afterwards
// The host transfers of an entry point: gb_xfer parts, each one copy on ctx->stream straight between a device array and a
// host array (skipped when the host pointer is null or the size zero).  gb_upload makes the H2D copies and does not
// synchronise; gb_download makes the D2H copies, then one cudaStreamSynchronize.  A call that uploads ends with a download,
// whose synchronisation is the last read of its host arrays: a pinned caller array is read after gb_upload has returned.
// A call that fails between the two leaves those copies pending until gb_ctx_synchronize or the context's next call that
// synchronises.  Staging through ctx->pinned instead was slower: see DESIGN.md §2 (scripts/ab_host_transfers.py).
struct gb_xfer { void* dst; const void* src; size_t bytes; };
gb_status gb_upload(gb_ctx* ctx, std::initializer_list<gb_xfer> parts);
gb_status gb_download(gb_ctx* ctx, std::initializer_list<gb_xfer> parts);
// the parameter bounds of gb_vgicp_align (gb_align.cu), shared by gb_ct_gicp_align
gb_status gb_align_params_check(const gb_align_params* prm);
// The round loop of gb_vgicp_align and gb_ct_gicp_align.  round(need_lin) launches one round for every problem: the
// linearize sweep when need_lin, the step kernel, the error sweep and the accept kernel, which leave the status word (active
// problems | those that need a linearization) in d_ctr.  After each round one 8-byte copy of it into h_ctr (pinned) and a
// stream sync; the loop ends when no problem is active.
template <typename Round>
gb_status gb_align_rounds(gb_ctx* ctx, const unsigned* d_ctr, unsigned* h_ctr, Round&& round) {
  bool need_lin = true;
  for (;;) {
    GB_CHECK(round(need_lin));
    GB_CUDA(cudaMemcpyAsync(h_ctr, d_ctr, 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
    GB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (h_ctr[0] == 0) return GB_OK;
    need_lin = h_ctr[1] > 0;
  }
}

// The one free function of each handle that owns memory (cloud_free, voxelmap_free, sweep_free, peer_slab_free,
// ctx_release): it releases everything the handle owns, never returns early, and ends with the delete.  A creation holds
// its partial handle in a gb_owned with that function, so that every failure exit frees it, and releases it on success.
template <typename T> using gb_owned = std::unique_ptr<T, void (*)(T*)>;
void cloud_free(gb_cloud* c);
void sweep_free(gb_sweep* s);
void ctx_retain(gb_ctx* ctx);
void ctx_release(gb_ctx* ctx);
void grid_release(gb_point_grid* g);  // gb_point_grid_destroy, as the free function of a gb_owned point grid
// A new factor of `kind` on (target, source) with its context retained and a process-wide unique id; nullptr when out of
// host memory.  Every *_factor_create calls it after its own argument checks.
gb_factor* factor_new(gb_ctx* ctx, gb_factor_kind kind, const gb_voxelmap* target, const gb_cloud* source);

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Carves 256-byte aligned arrays out of one buffer.  Without a base it only measures: every block the host lays out is
// written once, as a function of a Carver, and run first to size the buffer and then to hand out the pointers (gb_carve).
struct Carver {
  char* base = nullptr;
  size_t off = 0;
  template <typename T> T* take(size_t count) {
    T* p = base ? (T*)(base + off) : nullptr;
    off += align_up(sizeof(T) * count, 256);
    return p;
  }
};
// A layout carved out of one of the context's arenas (ctx->scratch or ctx->pinned).
template <typename Layout> gb_status gb_carve(gb_ctx* ctx, gb_arena& arena, Layout&& layout) {
  Carver size;
  layout(size);
  GB_CHECK(gb_arena_reserve(ctx, arena, size.off));
  Carver cv{(char*)arena.base};
  layout(cv);
  return GB_OK;
}
// A layout carved out of a new block of the device pool, which `block` (an empty owner of ctx's device) owns afterwards.
template <typename Layout> gb_status gb_dev_carve(gb_ctx* ctx, gb_dev_block& block, Layout&& layout) {
  assert(!block.base && block.device == ctx->device);
  Carver size;
  layout(size);
  void* base = nullptr;
  GB_CUDA(gb_dev_malloc(ctx->device, size.off, &base));
  block.base = base;
  Carver cv{(char*)base};
  layout(cv);
  return GB_OK;
}

// The peer slab's allocation, the same on every rank (so a peer's regions are found at the same offsets of its mapping).
// All of it is zero at creation.
struct gb_peer_regions {
  float* buf[2];       // the step-parity buffers: num_pairs x GB_SLAB_STRIDE floats each
  unsigned* flags;     // [world] completion flags, written by the peers
  int* timeout;        // set by the exchange kernels when a peer misses its flag
  unsigned* arrivals;  // [world] CTA arrival counters of the deferred exchange (self-cleaning)
};
inline gb_peer_regions gb_peer_layout(Carver& cv, size_t num_pairs, int world) {
  gb_peer_regions r;
  r.buf[0] = cv.take<float>(num_pairs * GB_SLAB_STRIDE);
  r.buf[1] = cv.take<float>(num_pairs * GB_SLAB_STRIDE);
  r.flags = cv.take<unsigned>((size_t)world);
  r.timeout = cv.take<int>(1);
  r.arrivals = cv.take<unsigned>((size_t)world);
  return r;
}
// rank p's regions as mapped on this device
inline gb_peer_regions gb_peer_regions_of(const gb_peer_slab* ps, int p) {
  Carver cv{ps->peer[p]};
  return gb_peer_layout(cv, ps->num_pairs, ps->world);
}

// The largest temporary storage of the cub calls the library makes on n items (radix sorts of 64-bit keys with or
// without int values, inclusive int scans, double sums): one buffer of this size serves them all.
size_t gb_cub_temp_bytes(size_t n);

// Temporaries of a (key, index) radix sort: the cub storage (shared with the caller's other cub calls) and the arrays.
struct gb_sort_tmp {
  void* cub;
  size_t cub_bytes;
  unsigned long long* keys;
  unsigned long long* keys_s;
  int* idx;
  int* idx_s;
};
inline gb_sort_tmp gb_take_sort_tmp(Carver& cv, size_t n, void* cub, size_t cub_bytes) {
  gb_sort_tmp t;
  t.cub = cub;
  t.cub_bytes = cub_bytes;
  t.keys = cv.take<unsigned long long>(n);
  t.keys_s = cv.take<unsigned long long>(n);
  t.idx = cv.take<int>(n + 1);
  t.idx_s = cv.take<int>(n + 1);
  return t;
}

// Voxel grouping (gb_kernels_voxelmap.cu), shared by the map build, the voxel-grid downsampling and the frame merge.  The
// caller writes one packed key per point (~0 = no voxel) and idx[i] = i; gb_group_by_key sorts the pairs into keys_s /
// idx_s, flags the first slot of every voxel and scans the flags: pos[s] = number of voxels up to sorted slot s, so
// pos[n - 1] is the voxel count.  gb_group_starts then writes starts[v] = first sorted slot of voxel v and
// starts[V] = number of valid points.
gb_status gb_group_by_key(gb_ctx* ctx, int n, const gb_sort_tmp& t, int* flags, int* pos);
gb_status gb_group_starts(gb_ctx* ctx, int n, const gb_sort_tmp& t, const int* flags, const int* pos, int* starts);
// Hash thinning (gb_kernels_voxelmap.cu), shared by the random-grid cap, the frame-merge thinning and the map-insert sampling:
// of the candidates among n items (i with cand[i] != 0 when cand is given, and i < *count when count is given), the m with
// the smallest rg_hash(seed, i) stay.  keep[i] = candidate(i) && rg_hash(seed, i) <= sorted[m - 1], where sorted holds the
// candidates' hashes (~0 for the others) in ascending order; every candidate stays when m <= 0 or m >= *count (n without a
// count).  keep may be cand itself.  The hashes go through t.keys into t.keys_s (t.cub for the sort), which it overwrites.
// Three launches: k_thin_hash, cub SortKeys, k_thin_keep.
gb_status gb_thin(gb_ctx* ctx, int n, const int* cand, const int* count, int m, unsigned long long seed, const gb_sort_tmp& t, int* keep);

// Device cloud construction.  gb_cloud_planes lays out the planes of n points (p0, p1, p2, optional normals) at the
// carver's position; the planes staged in the caller's point order use the same layout as the cloud's own.
// gb_cloud_build takes c's block (planes, perm, inv_perm) from the device pool and fills it with the Morton reorder of the
// staged planes; it uses t.cub, t.keys, t.keys_s and t.idx for n points.
struct gb_planes {
  float4* p0;
  float4* p1;
  float* p2;
  float4* normals;
};
inline gb_planes gb_cloud_planes(Carver& cv, size_t n, bool normals) {
  gb_planes p;
  p.p0 = cv.take<float4>(n);
  p.p1 = cv.take<float4>(n);
  p.p2 = cv.take<float>(n);
  p.normals = normals ? cv.take<float4>(n) : nullptr;
  return p;
}
gb_status gb_cloud_build(gb_ctx* ctx, gb_cloud* c, size_t n, const gb_planes& staged, const gb_sort_tmp& t);
// The covariance stage of gb_preprocess (gb_kernels_preprocess.cu), shared with gb_ct_deskew and gb_covariances:
// plane_covariance of the first *d_count of M points (pts, neighbors[i * kc + j], the first k of each row) into the fp64
// normals (M x double4) and covs (M x 16, column-major), and, when staged.p0 is given, the fp32 planes staged for the cloud;
// then, when cloud_out is given, the cloud (gb_cloud_build with t).  One launch plus the build's.
gb_status gb_covariance_cloud(gb_ctx* ctx, int M, const int* d_count, const double4* pts, const int* neighbors, int kc, int k, double4* normals, double* covs,
                              const gb_planes& staged, const gb_sort_tmp& t, gb_cloud* cloud_out);

// kernel launchers (gb_kernels_*.cu)
enum { GB_MODE_LINEARIZE = 0, GB_MODE_ERROR = 1 };
gb_status gb_launch_sweep(gb_sweep* s, int mode);
gb_status gb_launch_gicp_sweep(gb_sweep* s, int mode);  // gb_launch_sweep of a GICP sweep
gb_status gb_launch_overlap(gb_ctx* ctx, int num_targets, const FactorDesc* d_descs, const double* d_poses, int n, int* d_count);
// The posed frame list of gb_merge_frames (gb_kernels_preprocess.cu), shared with the map insert, gb_concat_frames
// (gb_kernels_segment.cu) and the plane selection (gb_kernels_plane.cu): K device clouds and their poses (K x 16,
// column-major).  gb_frame_list_check refuses, before any launch, a null list when K > 0, a null frame, a frame on another
// device than ctx's, a frame of 2^32 points or more and 2^30 points or more in all, and gives the total; it does not look at
// the poses' values (gb_all_finite says whether n doubles are all finite).  gb_frame_table writes the list's descriptors
// (gb_frame, gb_segment_math.cuh) on the host, index[k] as the caller's index of frame k (k without index); the caller
// uploads them to d_table, which the kernels search with gb_frame_of.  gb_transform_frames writes the points q = R a + t and
// covariances R C R^T in un-contracted fp64, frame-major and each frame in its original point order (pts: total x double4,
// cov6: total x 6 upper triangle; nullptr: no covariances): one launch, none when total is 0.
gb_status gb_frame_list_check(const gb_ctx* ctx, size_t K, const gb_cloud* const* frames, const double* poses, size_t* total);
bool gb_all_finite(const double* v, size_t n);
std::vector<gb_frame> gb_frame_table(size_t K, const gb_cloud* const* frames, const double* poses, const int* index);
gb_status gb_transform_frames(gb_ctx* ctx, size_t K, const gb_frame* d_table, int total, double4* pts, double* cov6);
// The exact k-NN of gb_preprocess and gb_find_neighbors (gb_kernels_preprocess.cu), shared with gb_min_cut: the k nearest of
// the first *d_count points of d_pts (device resident, n slots) to each of them, by un-contracted fp64 d2 with ties to the
// smaller index, the query included, in neighbors[i * k + j]; the row of a point whose cell of h0 leaves the 21-bit range, or
// of a slot at or beyond *d_count, is i itself k times, and such a point is nobody's neighbour.  Six launches.  Its
// temporaries for up to n points come from take_knn_tmp (the cub storage is the caller's); gb_knn_instantiated(k) tells
// whether k is one of the instantiated neighbour counts (1-10, 12, 15, 16, 20, 24, 32), which entry points check before any
// launch.
struct KnnTmp {
  gb_sort_tmp s;
  double4* pts_s;
  void* tables;  // the per-level cell hash tables
  unsigned ts;   // hash table size per level
};
KnnTmp take_knn_tmp(Carver& cv, int n, void* cub, size_t cub_bytes);
gb_status knn_device(gb_ctx* ctx, int n, const int* d_count, const double4* d_pts, int k, double h0, int* neighbors, const KnnTmp& t);
bool gb_knn_instantiated(int k);
// k_grid_keys of the voxel-grid paths: key = packed floor(p * inv_res) in fp64 (~0 for non-finite / out-of-range points,
// and for every point with keep[i] == 0 when keep is given), idx[i] = i.  One launch.
gb_status gb_grid_keys(gb_ctx* ctx, int n, const double4* pts, double inv_res, const int* keep, unsigned long long* keys, int* idx);

// ---------------------------------------------------------------------------------------------
// device helpers shared by kernels
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__
#include "gb_vgicp_math.cuh"  // gb_coord, gb_hash, gb_lookup (shared with the host-compiled CPU test of the kernel arithmetic)
// packed 3 x 21-bit voxel key (ascending key = canonical voxel order); false if out of range
#define GB_KEY_OFFSET (1 << 20)
constexpr unsigned long long kInvalidKey = ~0ull;  // the key of a point in no voxel: sorts last
__device__ __forceinline__ bool gb_pack_key(int x, int y, int z, unsigned long long* key) {
  if (x < -GB_KEY_OFFSET || x >= GB_KEY_OFFSET || y < -GB_KEY_OFFSET || y >= GB_KEY_OFFSET || z < -GB_KEY_OFFSET || z >= GB_KEY_OFFSET) return false;
  *key = ((unsigned long long)(x + GB_KEY_OFFSET) << 42) | ((unsigned long long)(y + GB_KEY_OFFSET) << 21) | (unsigned long long)(z + GB_KEY_OFFSET);
  return true;
}
__host__ __device__ __forceinline__ void gb_unpack_key(unsigned long long key, int& x, int& y, int& z) {
  x = (int)((key >> 42) & 0x1FFFFF) - GB_KEY_OFFSET;
  y = (int)((key >> 21) & 0x1FFFFF) - GB_KEY_OFFSET;
  z = (int)(key & 0x1FFFFF) - GB_KEY_OFFSET;
}
// 21 bits -> every third bit (Morton interleaving)
__device__ __forceinline__ unsigned long long gb_spread21(unsigned long long v) {
  v &= 0x1FFFFFull;
  v = (v | (v << 32)) & 0x1F00000000FFFFull;
  v = (v | (v << 16)) & 0x1F0000FF0000FFull;
  v = (v | (v << 8)) & 0x100F00F00F00F00Full;
  v = (v | (v << 4)) & 0x10C30C30C30C30C3ull;
  v = (v | (v << 2)) & 0x1249249249249249ull;
  return v;
}
#endif
