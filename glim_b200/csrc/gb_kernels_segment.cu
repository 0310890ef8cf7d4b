// gb_kernels_segment.cu -- the map editor's segmentation on the device (sm_90a): submaps concatenated into one world-frame
// cloud (gb_concat_frames) and region growing from a picked point (gb_region_growing).  The rules are written once in
// include/glim_b200.h; the per-point and per-pair arithmetic is gb_segment_math.cuh, which the host test build compiles as well.
//
//   gb_concat_frames    k_merge_transform over every frame through one descriptor table (gb_transform_frames, shared with
//                       gb_merge_frames), k_concat_flags (the window), a cub inclusive scan of the flags, k_concat_emit (the
//                       kept points' fp32 planes, rotated normals and ids in output order), one copy of the kept count and a
//                       stream synchronisation, then gb_cloud_build and the copy of the ids.
//   gb_region_growing   the point grids of the cloud (gb_point_grid_build at 1.05 distance_threshold, and at 1.05
//                       dilation_radius), then k_rg_init (every parent its own index; the seed by a 64-bit atomicMin of
//                       seg_seed_key), k_rg_hook (one thread per grid record: each join (i, j > i) hooked once, ECL-CC),
//                       k_rg_label (the labels, which also compress the parents, the region and the counts), k_rg_dilate,
//                       and one cub compaction of the selection; one copy back and one stream synchronisation.
//   gb_min_cut          k_mc_flags (the participants, and the seed by the same 64-bit atomicMin of seg_seed_key), a cub scan,
//                       k_mc_nodes (the fp64 node positions, normals, original indices and roles, in ascending original
//                       index), knn_device on the nodes (6 launches), k_mc_arcs (each row's arcs both ways), a cub radix sort
//                       on (u << 32 | v), k_mc_unique and a cub scan of its packed (arc, edge) counts, k_mc_csr (the unique
//                       arcs), k_mc_graph (heads, reverse arcs, capacities, rows and the exported edges), the cooperative
//                       k_mc_solve (push-relabel, gb_mincut_math.cuh) and one cub compaction of the selection; one copy back
//                       and one stream synchronisation.
#include "gb_internal.cuh"
#include "gb_segment_math.cuh"
#include "gb_mincut_math.cuh"

#include <cooperative_groups.h>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <cmath>
#include <cstring>
#include <new>

namespace {

constexpr int kSegThreads = 256;
constexpr int kHookThreads = 128;

// flags[g] = 1 iff point g of the concatenation (fp64 q) is kept: always without a window
__global__ void k_concat_flags(int n, const double4* __restrict__ pts, int windowed, double inv, int3 lo, int3 hi, int* __restrict__ flags) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  const double4 p = pts[g];
  const double q[3] = {p.x, p.y, p.z};
  const int l[3] = {lo.x, lo.y, lo.z}, h[3] = {hi.x, hi.y, hi.z};
  flags[g] = !windowed || seg_in_window(q, inv, l, h) ? 1 : 0;
}

// one thread per point g of the concatenation: a kept point goes to slot pos[g] - 1 as fp32 planes (zero covariances unless
// every frame has them), its rotated normal and its id
__global__ void k_concat_emit(int n, int K, const gb_frame* __restrict__ frames, const int* __restrict__ flags,
                              const int* __restrict__ pos, const double4* __restrict__ pts, const double* __restrict__ cov6, int covs, float4* __restrict__ s0,
                              float4* __restrict__ s1, float* __restrict__ s2, float4* __restrict__ sn, unsigned long long* __restrict__ ids) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n || !flags[g]) return;
  const gb_frame& F = frames[gb_frame_of(frames, K, g)];
  const int i = g - F.offset, o = pos[g] - 1;
  const double4 p = pts[g];
  const double* c = cov6 + 6 * (size_t)g;
  s0[o] = make_float4((float)p.x, (float)p.y, (float)p.z, covs ? (float)c[0] : 0.f);
  s1[o] = covs ? make_float4((float)c[1], (float)c[2], (float)c[3], (float)c[4]) : make_float4(0.f, 0.f, 0.f, 0.f);
  s2[o] = covs ? (float)c[5] : 0.f;
  if (sn) {
    const float4 nr = F.normals[F.inv_perm ? F.inv_perm[i] : i];
    float v[3];
    seg_rotate_normal(F.T, nr.x, nr.y, nr.z, v);
    sn[o] = make_float4(v[0], v[1], v[2], 0.f);
  }
  ids[o] = ((unsigned long long)F.index << 32) | (unsigned)i;
}

// What gb_region_growing leaves for the host, ahead of the selection and the labels in one copy.
struct RgOut {
  unsigned long long seed_key;  // seg_seed_key of the seed, ~0 for none
  int num_region, num_components, num_selected, pad;
};

__device__ __forceinline__ void warp_count(bool c, int* counter) {
  const unsigned b = __ballot_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(counter, __popc(b));
}

// one thread per stored slot: parent[i] = i for its original index i, and the seed's key (the warp's minimum, then one atomic)
__global__ void __launch_bounds__(kSegThreads) k_rg_init(int n, const float4* __restrict__ p0, const int* __restrict__ perm, float qx, float qy, float qz,
                                                         int* __restrict__ parent, RgOut* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long key = ~0ull;
  if (j < n) {
    const int i = perm ? perm[j] : j;
    parent[i] = i;
    key = seg_seed_key(p0[j], qx, qy, qz, i);
  }
  for (int o = 16; o > 0; o >>= 1) key = min(key, __shfl_xor_sync(0xffffffffu, key, o));
  if ((threadIdx.x & 31) == 0 && key != ~0ull) atomicMin(&out->seed_key, key);
}

// one thread per record of the connectivity grid (point i): every join (i, j) with j > i, hooked
__global__ void __launch_bounds__(kHookThreads) k_rg_hook(int n, const int4* __restrict__ buckets, uint32_t mask, int max_scan, const int2* __restrict__ cells,
                                                          const float4* __restrict__ points, int m, float inv, float max_d2, const float4* __restrict__ normals,
                                                          const int* __restrict__ inv_perm, double cos_t, int* __restrict__ parent) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const float4 a = points[3 * (size_t)r];
  if (!seg_keyed(a.x, a.y, a.z, inv)) return;
  const int i = grid_record_index(points, r);
  const float4 ni = normals[inv_perm ? inv_perm[i] : i];
  grid_within(buckets, mask, max_scan, cells, points, m, inv, max_d2, a.x, a.y, a.z, [&](int q) {
    const int j = grid_record_index(points, q);
    if (j <= i) return;
    const float4 nj = normals[inv_perm ? inv_perm[j] : j];
    if (seg_normals_join(ni.x, ni.y, ni.z, nj.x, nj.y, nj.z, cos_t)) seg_hook(parent, i, j);
  });
}

// one thread per stored slot (original index i): labels[i] = its root (the component's minimum index, also written back as
// its parent) or -1, region[i] = label == the seed's label, and the component and region counts
__global__ void __launch_bounds__(kSegThreads) k_rg_label(int n, const float4* __restrict__ p0, const int* __restrict__ perm, int* __restrict__ parent,
                                                          int* __restrict__ labels, int* __restrict__ region, RgOut* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  bool root = false, in = false;
  if (j < n) {
    const int i = perm ? perm[j] : j;
    const float4 a = p0[j];
    int label = -1;
    if (isfinite(a.x) && isfinite(a.y) && isfinite(a.z)) {
      label = seg_find(parent, i);
      parent[i] = label;
    }
    const unsigned long long key = out->seed_key;
    in = label >= 0 && key != ~0ull && label == seg_find(parent, (int)(uint32_t)key);
    root = label == i;
    labels[i] = label;
    region[i] = in ? 1 : 0;
  }
  warp_count(root, &out->num_components);
  warp_count(in, &out->num_region);
}

// one thread per record of the dilation grid (point j): sel[j] = j in R, or j finite and keyed with a point of R within the
// dilation radius
__global__ void __launch_bounds__(kHookThreads) k_rg_dilate(int n, const int4* __restrict__ buckets, uint32_t mask, int max_scan, const int2* __restrict__ cells,
                                                            const float4* __restrict__ points, int m, float inv, float max_d2, const int* __restrict__ region,
                                                            int* __restrict__ sel) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const int j = grid_record_index(points, r);
  int s = region[j];
  if (!s) {
    const float4 a = points[3 * (size_t)r];
    s = seg_keyed(a.x, a.y, a.z, inv) && seg_grid_any(buckets, mask, max_scan, cells, points, m, inv, max_d2, a.x, a.y, a.z, region) ? 1 : 0;
  }
  sel[j] = s;
}

// a point grid of the cloud at 1.05 r and its search half-width for (float)(r^2)
gb_status rg_grid(gb_ctx* ctx, const gb_cloud* cloud, double r, gb_owned<gb_point_grid>& grid, int& m, float& max_d2) {
  gb_point_grid* gh = nullptr;
  const gb_status st = gb_point_grid_build(ctx, cloud, 1.05 * r, &gh);
  grid.reset(gh);
  GB_CHECK(st);
  const gb_voxelmap* g = grid_map(gh);
  max_d2 = (float)(r * r);
  m = grid_half_width(g->inv_res, max_d2, g->key_extent);
  if (m > kGridMaxHalfWidth) {
    gb_set_error("region growing search half-width %d exceeds %d", m, kGridMaxHalfWidth);
    return GB_ERR_INTERNAL;
  }
  return GB_OK;
}

// ---- gb_min_cut ----
constexpr int kMcThreads = 256;

// What gb_min_cut leaves for the host, ahead of the selection and the exported graph in one copy.
struct McOut {
  unsigned long long seed_key;  // seg_seed_key of the seed among the participants, ~0 for none
  long long cut_value;
  int num_points, num_foreground, num_background, num_arcs, num_edges, num_selected, rounds, status, seed_node, pad;
};

// one thread per stored slot: flags[i] = point i (original index) takes part, and the seed's key among the participants
__global__ void __launch_bounds__(kSegThreads) k_mc_flags(int n, const float4* __restrict__ p0, const int* __restrict__ perm, double cx, double cy, double cz, double r2,
                                                          int* __restrict__ flags, McOut* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long key = ~0ull;
  if (j < n) {
    const int i = perm ? perm[j] : j;
    const float4 p = p0[j];
    const bool in = isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && mc_d2(p.x, p.y, p.z, cx, cy, cz) < r2;
    flags[i] = in ? 1 : 0;
    if (in) key = seg_seed_key(p, (float)cx, (float)cy, (float)cz, i);
  }
  for (int o = 16; o > 0; o >>= 1) key = min(key, __shfl_xor_sync(0xffffffffu, key, o));
  if ((threadIdx.x & 31) == 0 && key != ~0ull) atomicMin(&out->seed_key, key);
}

// one thread per original index i: participant i becomes node pos[i] - 1 with its fp64 position, normal, index and role
__global__ void __launch_bounds__(kSegThreads) k_mc_nodes(int n, const float4* __restrict__ p0, const float4* __restrict__ normals, const int* __restrict__ inv_perm,
                                                          const int* __restrict__ flags, const int* __restrict__ pos, double cx, double cy, double cz, double fg2, double bg2,
                                                          double4* __restrict__ pts, float4* __restrict__ nrm, int* __restrict__ orig, int* __restrict__ role,
                                                          McOut* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool fg = false, bg = false;
  if (i < n && flags[i]) {
    const int u = pos[i] - 1, j = inv_perm ? inv_perm[i] : i;
    const float4 p = p0[j];
    pts[u] = make_double4(p.x, p.y, p.z, 1.0);
    nrm[u] = normals[j];
    orig[u] = i;
    const bool seed = (unsigned long long)(uint32_t)i == (out->seed_key & 0xffffffffull) && out->seed_key != ~0ull;
    const int r = seed ? MC_SEED : mc_role(mc_d2(p.x, p.y, p.z, cx, cy, cz), fg2, bg2);
    role[u] = r;
    if (seed) out->seed_node = u;
    fg = r == MC_FOREGROUND;
    bg = r == MC_BACKGROUND;
  }
  if (i == n - 1) out->num_points = pos[n - 1];
  warp_count(fg, &out->num_foreground);
  warp_count(bg, &out->num_background);
}

// one thread per k-NN slot (u, j): the arcs u -> v and v -> u of neighbour v != u, else two empty keys.  The rows of slots
// past the participants, and of nodes without a key, hold only the node itself.
__global__ void k_mc_arcs(int nk, int k, const int* __restrict__ nb, unsigned long long* __restrict__ keys) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nk) return;
  const unsigned long long u = (unsigned)(t / k), v = (unsigned)nb[t];
  const bool ok = u != v;
  keys[2 * (size_t)t] = ok ? (u << 32 | v) : ~0ull;
  keys[2 * (size_t)t + 1] = ok ? (v << 32 | u) : ~0ull;
}

__device__ __forceinline__ bool mc_first(const unsigned long long* keys_s, int s) {
  const unsigned long long k = keys_s[s];
  return k != ~0ull && (s == 0 || keys_s[s - 1] != k);
}

// one thread per sorted slot: 1 for the first copy of an arc, plus 2^32 when it is an edge's arc u -> v with u < v
__global__ void k_mc_unique(int na, const unsigned long long* __restrict__ keys_s, unsigned long long* __restrict__ flags) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= na) return;
  const unsigned long long k = keys_s[s];
  flags[s] = mc_first(keys_s, s) ? (1ull | ((k >> 32) < (k & 0xffffffffull) ? 1ull << 32 : 0ull)) : 0ull;
}

// one thread per sorted slot: the unique arcs in (u, v) order, each with its edge's rank (u < v) or -1, and their counts
__global__ void k_mc_csr(int na, const unsigned long long* __restrict__ keys_s, const unsigned long long* __restrict__ pos, unsigned long long* __restrict__ ukeys,
                         int* __restrict__ eidx, McOut* __restrict__ out) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= na) return;
  const unsigned long long k = keys_s[s], p = pos[s];
  if (mc_first(keys_s, s)) {
    const int a = (int)(uint32_t)p - 1;
    ukeys[a] = k;
    eidx[a] = (k >> 32) < (k & 0xffffffffull) ? (int)(p >> 32) - 1 : -1;
  }
  if (s == na - 1) {
    out->num_arcs = (int)(uint32_t)p;
    out->num_edges = (int)(p >> 32);
  }
}

// the first index of keys[0, n) (ascending) that is >= x
__device__ __forceinline__ int mc_lower_bound(const unsigned long long* keys, int n, unsigned long long x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (keys[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// one thread per arc a and per row start: head, reverse arc, capacity (and the exported edge row), row[u] = first arc of u
__global__ void k_mc_graph(int slots, const unsigned long long* __restrict__ ukeys, const int* __restrict__ eidx, const double4* __restrict__ pts, const float4* __restrict__ nrm,
                           const int* __restrict__ orig, double s2d, double s2a, const McOut* __restrict__ out, int* __restrict__ head, int* __restrict__ rev,
                           int* __restrict__ cap, int* __restrict__ row, int* __restrict__ edges, int* __restrict__ ecap) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= slots) return;
  const int A = out->num_arcs, m = out->num_points;
  if (t < A) {
    const unsigned long long k = ukeys[t];
    const int u = (int)(k >> 32), v = (int)(uint32_t)k;
    head[t] = v;
    rev[t] = mc_lower_bound(ukeys, A, (unsigned long long)v << 32 | (unsigned)u);
    const double4 a = pts[u], b = pts[v];
    const float4 na = nrm[u], nb = nrm[v];
    const int q = mc_edge_capacity((float)a.x, (float)a.y, (float)a.z, na.x, na.y, na.z, (float)b.x, (float)b.y, (float)b.z, nb.x, nb.y, nb.z, s2d, s2a);
    cap[t] = q;
    const int e = eidx[t];
    if (edges && e >= 0) {
      edges[2 * (size_t)e] = orig[u];
      edges[2 * (size_t)e + 1] = orig[v];
      ecap[e] = q;
    }
  }
  if (t <= m) row[t] = mc_lower_bound(ukeys, A, (unsigned long long)t << 32);
}

// The flow network and the solver's state (gb_mincut_math.cuh): m nodes of n slots, CSR rows, arcs with their heads, reverse
// arcs and capacities.  e, incoming and cnt are zero at launch.
struct McSolve {
  int n;
  int fg_cap;
  const int* row;
  const int* head;
  const int* rev;
  const int* cap;
  const int* role;
  int* res;
  int* fg_res;
  int* h0;  // the heights, double-buffered
  int* h1;
  long long* e;
  long long* incoming;
  int* cnt;  // [3]: the rotating grid-wide counters
  int* sel;
  McOut* out;
};

__device__ __forceinline__ bool mc_inner(int r) { return r == MC_FREE || r == MC_FOREGROUND; }

// The whole solve in one cooperative grid (grid.sync() between steps; every thread runs every loop the same number of
// times).  Initialise (every arc out of the background saturated), a global relabel, then rounds of push / relabel with a
// global relabel every kMcRelabelPeriod rounds, until no node is active or kMcMaxRounds rounds have run.  A global relabel
// is a level-synchronous breadth-first search from the seed over reverse residual arcs: exact distances, H for the nodes
// that cannot reach the seed.  The last one labels the selection.
__global__ void __launch_bounds__(kMcThreads, 4) k_mc_solve(McSolve g) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  const int t0 = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
  for (int u = t0; u < g.n; u += stride) g.sel[u] = 0;
  const int m = g.out->num_points;
  if (m == 0) return;  // every thread alike
  const int seed = g.out->seed_node, H = m + 2;
  for (int u = t0; u < m; u += stride) {
    const int ru = g.role[u];
    g.fg_res[u] = ru == MC_FOREGROUND ? g.fg_cap : 0;
    for (int a = g.row[u]; a < g.row[u + 1]; a++) {
      const int rv = g.role[g.head[a]];
      g.res[a] = mc_initial_residual(ru, rv, g.cap[a]);
      if (ru == MC_BACKGROUND && rv != MC_BACKGROUND) mc_add(&g.e[g.head[a]], g.cap[a]);
    }
  }
  grid.sync();
  int phase = 0;
  // the grid-wide sum of every thread's x (a grid barrier): counter phase % 3 collects it while the next one is cleared
  const auto total = [&](int x) {
    int* c = g.cnt + phase % 3;
    if (t0 == 0) g.cnt[(phase + 1) % 3] = 0;
    x = __reduce_add_sync(0xffffffffu, x);
    if ((threadIdx.x & 31) == 0 && x) atomicAdd(c, x);
    grid.sync();
    phase++;
    return *(volatile int*)c;
  };
  const auto global_relabel = [&](int* h) {
    for (int u = t0; u < m; u += stride) h[u] = u == seed ? 0 : H;
    grid.sync();
    volatile int* vh = h;
    for (int d = 0; d < m; d++) {
      int added = 0;
      for (int v = t0; v < m; v += stride) {
        if (d == 0 && g.role[v] == MC_FOREGROUND && g.fg_res[v] > 0 && vh[v] == H) {
          vh[v] = 1;
          added++;
        }
        if (vh[v] != d) continue;
        for (int a = g.row[v]; a < g.row[v + 1]; a++) {
          const int u = g.head[a];
          if (vh[u] == H && g.role[u] != MC_BACKGROUND && g.res[g.rev[a]] > 0) {
            vh[u] = d + 1;
            added++;
          }
        }
      }
      if (total(added) == 0) break;
    }
  };
  const auto active = [&](const int* h) {
    int x = 0;
    for (int u = t0; u < m; u += stride) x += mc_inner(g.role[u]) && h[u] < H && g.e[u] > 0;
    return total(x);
  };
  int *h = g.h0, *hn = g.h1, rounds = 0;
  global_relabel(h);
  int act = active(h);
  while (act > 0 && rounds < kMcMaxRounds) {
    rounds++;
    for (int u = t0; u < m; u += stride)
      if (mc_inner(g.role[u]) && h[u] < H && g.e[u] > 0) g.e[u] = mc_push_node(u, g.e[u], g.row, g.head, g.rev, g.res, g.fg_res, h, g.incoming, seed);
    grid.sync();
    int x = 0;
    for (int u = t0; u < m; u += stride) {
      const int ru = g.role[u];
      long long ex = g.e[u];
      int hu = h[u];
      if (mc_inner(ru) && hu < H && ex > 0) hu = mc_relabel_node(u, ru, g.row, g.head, g.res, g.fg_res, h, H);
      hn[u] = hu;
      ex += g.incoming[u];
      g.incoming[u] = 0;
      g.e[u] = ex;
      x += mc_inner(ru) && hu < H && ex > 0;
    }
    int* t = h;
    h = hn;
    hn = t;
    act = total(x);
    if (act > 0 && rounds % kMcRelabelPeriod == 0) {
      global_relabel(h);
      act = active(h);
    }
  }
  if (act > 0) {  // the round cap: nothing selected
    if (t0 == 0) {
      g.out->status = GB_MINCUT_NOT_CONVERGED;
      g.out->rounds = rounds;
    }
    return;
  }
  global_relabel(h);
  for (int u = t0; u < m; u += stride) g.sel[u] = h[u] < H && g.role[u] != MC_BACKGROUND ? 1 : 0;
  if (t0 == 0) {
    g.out->cut_value = g.e[seed];
    g.out->rounds = rounds;
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// entry points
// ---------------------------------------------------------------------------------------------
extern "C" gb_status gb_concat_frames(gb_ctx* ctx, size_t K, const gb_cloud* const* frames, const double* poses, const gb_cell_window* window, gb_cloud** out_cloud,
                                      uint64_t* ids, size_t* num_out) {
  GB_REQUIRE(ctx && out_cloud && num_out, "null argument");
  *out_cloud = nullptr;
  *num_out = 0;
  size_t total = 0;
  GB_CHECK(gb_frame_list_check(ctx, K, frames, poses, &total));
  GB_REQUIRE(gb_all_finite(poses, 16 * K), "a non-finite pose");
  bool covs = K > 0, normals = K > 0;
  for (size_t k = 0; k < K; k++) {
    covs = covs && frames[k]->covs;
    normals = normals && (frames[k]->normals || frames[k]->n == 0);
  }
  if (window) {
    GB_REQUIRE(std::isfinite(window->cell_size) && window->cell_size > 0.0, "cell_size must be positive and finite");
    for (int a = 0; a < 3; a++) GB_REQUIRE(window->lo[a] <= window->hi[a], "lo > hi");
  }
  GB_ENTER(ctx);
  gb_owned<gb_cloud> c(new (std::nothrow) gb_cloud(), cloud_free);
  if (!c) return GB_ERR_INTERNAL;
  c->device = ctx->device;
  c->covs = covs;
  if (total == 0) {
    *out_cloud = c.release();
    return GB_OK;
  }
  const int n = (int)total;
  const size_t N = total, cub_b = gb_cub_temp_bytes(N);
  const std::vector<gb_frame> table = gb_frame_table(K, frames, poses, nullptr);
  gb_planes staged;
  gb_sort_tmp t;
  gb_frame* d_table;
  int *d_flags, *d_pos;
  double4* d_pts;
  double* d_cov;
  unsigned long long* d_ids;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    staged = gb_cloud_planes(cv, N, normals);
    t = gb_take_sort_tmp(cv, N, cv.take<char>(cub_b), cub_b);
    d_table = cv.take<gb_frame>(K);
    d_flags = cv.take<int>(N);
    d_pos = cv.take<int>(N);
    d_pts = cv.take<double4>(N);
    d_cov = cv.take<double>(6 * N);
    d_ids = cv.take<unsigned long long>(N);
  }));
  GB_CHECK(gb_upload(ctx, {{d_table, table.data(), sizeof(gb_frame) * K}}));
  GB_CHECK(gb_transform_frames(ctx, K, d_table, n, d_pts, d_cov));
  const int gb = (n + kSegThreads - 1) / kSegThreads;
  const double inv = window ? 1.0 / window->cell_size : 0.0;
  const int3 lo = window ? make_int3(window->lo[0], window->lo[1], window->lo[2]) : make_int3(0, 0, 0);
  const int3 hi = window ? make_int3(window->hi[0], window->hi[1], window->hi[2]) : make_int3(0, 0, 0);
  GB_CHECK(gb_launch(ctx, "k_concat_flags", k_concat_flags, gb, kSegThreads, 0, n, d_pts, window ? 1 : 0, inv, lo, hi, d_flags));
  GB_CUB(ctx, cub::DeviceScan::InclusiveSum, t.cub, cub_b, d_flags, d_pos, n);
  GB_CHECK(gb_launch(ctx, "k_concat_emit", k_concat_emit, gb, kSegThreads, 0, n, (int)K, d_table, d_flags, d_pos, d_pts, d_cov, covs ? 1 : 0,
                     staged.p0, staged.p1, staged.p2, staged.normals, d_ids));
  int count = 0;
  GB_CHECK(gb_download(ctx, {{&count, d_pos + (n - 1), sizeof(int)}}));
  const size_t M = (size_t)count;
  if (M > 0) {
    GB_CHECK(gb_cloud_build(ctx, c.get(), M, staged, t));
    GB_CHECK(gb_download(ctx, {{ids, d_ids, sizeof(uint64_t) * M}}));
  }
  *num_out = M;
  *out_cloud = c.release();
  return GB_OK;
}

extern "C" gb_status gb_region_growing_default_params(gb_region_growing_params* p) {
  GB_REQUIRE(p, "null argument");
  p->distance_threshold = 0.5;
  p->angle_threshold = 10.0 * 3.141592653589793 / 180.0;
  p->dilation_radius = 0.0;
  return GB_OK;
}

extern "C" gb_status gb_region_growing(gb_ctx* ctx, const gb_cloud* cloud, const double seed_point[3], const gb_region_growing_params* prm,
                                       gb_region_growing_result* result, int32_t* selected, int32_t* labels) {
  GB_REQUIRE(ctx && cloud && seed_point && prm && result, "null argument");
  GB_REQUIRE(cloud->device == ctx->device, "the cloud lives on another device");
  GB_REQUIRE(cloud->n == 0 || cloud->normals, "region growing needs the cloud's normals");
  GB_REQUIRE(std::isfinite(seed_point[0]) && std::isfinite(seed_point[1]) && std::isfinite(seed_point[2]), "a non-finite seed point");
  GB_REQUIRE(std::isfinite(prm->distance_threshold) && prm->distance_threshold > 0.0, "distance_threshold must be positive and finite");
  GB_REQUIRE(prm->angle_threshold >= 0.0 && prm->angle_threshold <= 3.141592653589793, "angle_threshold must be in [0, pi]");
  GB_REQUIRE(std::isfinite(prm->dilation_radius) && prm->dilation_radius >= 0.0, "dilation_radius must be finite and non-negative");
  GB_ENTER(ctx);
  memset(result, 0, sizeof(*result));
  result->seed = -1;
  result->status = GB_REGION_NO_SEED;
  const size_t N = cloud->n;
  if (N == 0) return GB_OK;
  const int n = (int)N;
  const bool dilate = prm->dilation_radius > 0.0;
  // the grids first: their builds carve the context's scratch, which then holds this call's arrays
  gb_owned<gb_point_grid> conn(nullptr, grid_release), dil(nullptr, grid_release);
  int mc = 0, md = 0;
  float d2c = 0.f, d2d = 0.f;
  GB_CHECK(rg_grid(ctx, cloud, prm->distance_threshold, conn, mc, d2c));
  if (dilate) GB_CHECK(rg_grid(ctx, cloud, prm->dilation_radius, dil, md, d2d));
  size_t cub_b = 0;
  cub::DeviceSelect::Flagged(nullptr, cub_b, thrust::counting_iterator<int>(0), (const int*)nullptr, (int*)nullptr, (int*)nullptr, n);
  void* d_cub;
  int *d_parent, *d_region, *d_sel, *d_selected, *d_labels;
  RgOut* d_out;
  // out, selected and labels are adjacent: one copy brings them back, into the same layout of the pinned arena
  const auto tail = [&](Carver& cv, RgOut*& o, int*& s, int*& l) {
    o = cv.take<RgOut>(1);
    s = cv.take<int>(N);
    l = cv.take<int>(N);
  };
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    d_cub = cv.take<char>(cub_b);
    d_parent = cv.take<int>(N);
    d_region = cv.take<int>(N);
    d_sel = dilate ? cv.take<int>(N) : nullptr;
    tail(cv, d_out, d_selected, d_labels);
  }));
  RgOut* h_out;
  int *h_selected, *h_labels;
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) { tail(cv, h_out, h_selected, h_labels); }));
  cudaStream_t st = ctx->stream;
  GB_CUDA(cudaMemsetAsync(d_out, 0, sizeof(RgOut), st));
  GB_CUDA(cudaMemsetAsync(&d_out->seed_key, 0xff, sizeof(unsigned long long), st));
  const int gb = (n + kSegThreads - 1) / kSegThreads, hb = (n + kHookThreads - 1) / kHookThreads;
  GB_CHECK(gb_launch(ctx, "k_rg_init", k_rg_init, gb, kSegThreads, 0, n, cloud->p0, cloud->perm, (float)seed_point[0], (float)seed_point[1], (float)seed_point[2],
                     d_parent, d_out));
  const gb_voxelmap* g = grid_map(conn.get());
  GB_CHECK(gb_launch(ctx, "k_rg_hook", k_rg_hook, hb, kHookThreads, 0, n, g->buckets, (uint32_t)(g->num_buckets - 1), g->max_scan, g->cells, g->voxels, mc,
                     g->inv_res, d2c, cloud->normals, cloud->inv_perm, cos(prm->angle_threshold), d_parent));
  GB_CHECK(gb_launch(ctx, "k_rg_label", k_rg_label, gb, kSegThreads, 0, n, cloud->p0, cloud->perm, d_parent, d_labels, d_region, d_out));
  if (dilate) {
    const gb_voxelmap* h = grid_map(dil.get());
    GB_CHECK(gb_launch(ctx, "k_rg_dilate", k_rg_dilate, hb, kHookThreads, 0, n, h->buckets, (uint32_t)(h->num_buckets - 1), h->max_scan, h->cells, h->voxels, md,
                       h->inv_res, d2d, d_region, d_sel));
  }
  GB_CUB(ctx, cub::DeviceSelect::Flagged, d_cub, cub_b, thrust::counting_iterator<int>(0), dilate ? d_sel : d_region, d_selected, &d_out->num_selected, n);
  const char* end = labels ? (const char*)(d_labels + N) : (const char*)(d_selected + N);
  GB_CUDA(cudaMemcpyAsync(h_out, d_out, (size_t)(end - (const char*)d_out), cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  if (h_out->seed_key != ~0ull) {
    result->seed = (int32_t)(uint32_t)h_out->seed_key;
    result->status = GB_REGION_FOUND;
  }
  result->num_region = (size_t)h_out->num_region;
  result->num_selected = (size_t)h_out->num_selected;
  result->num_components = (size_t)h_out->num_components;
  if (selected) memcpy(selected, h_selected, sizeof(int32_t) * result->num_selected);
  if (labels) memcpy(labels, h_labels, sizeof(int32_t) * N);
  return GB_OK;
}

extern "C" gb_status gb_min_cut_default_params(gb_min_cut_params* p) {
  GB_REQUIRE(p, "null argument");
  p->distance_sigma = 0.25;
  p->angle_sigma = 10.0 * 3.141592653589793 / 180.0;
  p->foreground_mask_radius = 0.5;
  p->background_mask_radius = 5.0;
  p->foreground_weight = 10.0;
  p->k_neighbors = 20;
  return GB_OK;
}

extern "C" gb_status gb_min_cut(gb_ctx* ctx, const gb_cloud* cloud, const double c[3], const gb_min_cut_params* prm, gb_min_cut_result* result, int32_t* selected,
                                int32_t* edges, int32_t* capacities) {
  GB_REQUIRE(ctx && cloud && c && prm && result, "null argument");
  GB_REQUIRE(cloud->device == ctx->device, "the cloud lives on another device");
  GB_REQUIRE(cloud->n == 0 || cloud->normals, "min cut needs the cloud's normals");
  GB_REQUIRE(std::isfinite(c[0]) && std::isfinite(c[1]) && std::isfinite(c[2]), "a non-finite picked point");
  GB_REQUIRE(std::isfinite(prm->distance_sigma) && prm->distance_sigma > 0.0, "distance_sigma must be positive and finite");
  GB_REQUIRE(prm->angle_sigma > 0.0 && prm->angle_sigma <= 3.141592653589793, "angle_sigma must be in (0, pi]");
  GB_REQUIRE(std::isfinite(prm->foreground_mask_radius) && prm->foreground_mask_radius > 0.0, "foreground_mask_radius must be positive and finite");
  GB_REQUIRE(std::isfinite(prm->background_mask_radius) && prm->background_mask_radius > prm->foreground_mask_radius,
             "background_mask_radius must be finite and larger than foreground_mask_radius");
  GB_REQUIRE(prm->foreground_weight >= 0.0 && prm->foreground_weight <= 1000.0, "foreground_weight must be in [0, 1000]");
  GB_REQUIRE(gb_knn_instantiated(prm->k_neighbors), "k_neighbors is not an instantiated neighbour count (1-10, 12, 15, 16, 20, 24, 32)");
  GB_REQUIRE(cloud->n * (size_t)prm->k_neighbors < ((size_t)1 << 30), "N * k_neighbors must be below 2^30");
  GB_ENTER(ctx);
  memset(result, 0, sizeof(*result));
  result->seed = -1;
  result->status = GB_MINCUT_NO_SEED;
  const size_t N = cloud->n;
  if (N == 0) return GB_OK;
  const int n = (int)N, k = prm->k_neighbors, nk = n * k, na = 2 * nk;
  const bool graph = edges || capacities;
  int end_bit = 33;  // the arc keys (u << 32 | v) with u, v < n, and ~0 for none, which sorts last on these bits too
  while (end_bit < 64 && ((size_t)1 << (end_bit - 32)) < N) end_bit++;
  size_t cub_b = gb_cub_temp_bytes(N), b = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, b, (unsigned long long*)nullptr, (unsigned long long*)nullptr, na, 0, end_bit);
  cub_b = std::max(cub_b, b);
  cub::DeviceScan::InclusiveSum(nullptr, b, (unsigned long long*)nullptr, (unsigned long long*)nullptr, na);
  cub_b = std::max(cub_b, b);
  cub::DeviceSelect::Flagged(nullptr, b, (const int*)nullptr, (const int*)nullptr, (int*)nullptr, (int*)nullptr, n);
  cub_b = std::max(cub_b, b);
  KnnTmp knn;
  void* d_cub;
  int *d_flags, *d_pos, *d_orig, *d_role, *d_nb, *d_eidx, *d_head, *d_rev, *d_cap, *d_res, *d_row, *d_fg, *d_h0, *d_h1, *d_cnt, *d_sel, *d_selected, *d_edges, *d_ecap;
  double4* d_pts;
  float4* d_nrm;
  unsigned long long *d_keys, *d_keys_s, *d_apos;
  long long *d_e, *d_in;
  McOut* d_out;
  // out, selected and the graph are adjacent: one copy brings them back, into the same layout of the pinned arena
  const auto tail = [&](Carver& cv, McOut*& o, int*& s, int*& e, int*& q) {
    o = cv.take<McOut>(1);
    s = cv.take<int>(N);
    e = graph ? cv.take<int>(2 * (size_t)nk) : nullptr;
    q = graph ? cv.take<int>((size_t)nk) : nullptr;
  };
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    d_cub = cv.take<char>(cub_b);
    knn = take_knn_tmp(cv, n, d_cub, cub_b);
    d_flags = cv.take<int>(N);
    d_pos = cv.take<int>(N);
    d_pts = cv.take<double4>(N);
    d_nrm = cv.take<float4>(N);
    d_orig = cv.take<int>(N);
    d_role = cv.take<int>(N);
    d_nb = cv.take<int>((size_t)nk);
    d_keys = cv.take<unsigned long long>((size_t)na);  // the arcs, then the unique flags, then the unique arcs
    d_keys_s = cv.take<unsigned long long>((size_t)na);
    d_apos = cv.take<unsigned long long>((size_t)na);
    d_eidx = cv.take<int>((size_t)na);
    d_head = cv.take<int>((size_t)na);
    d_rev = cv.take<int>((size_t)na);
    d_cap = cv.take<int>((size_t)na);
    d_res = cv.take<int>((size_t)na);
    d_row = cv.take<int>(N + 1);
    d_fg = cv.take<int>(N);
    d_h0 = cv.take<int>(N);
    d_h1 = cv.take<int>(N);
    d_sel = cv.take<int>(N);
    d_e = cv.take<long long>(2 * N);  // excess, then incoming
    d_cnt = cv.take<int>(3);
    tail(cv, d_out, d_selected, d_edges, d_ecap);
  }));
  d_in = d_e + N;
  McOut* h_out;
  int *h_selected, *h_edges, *h_ecap;
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) { tail(cv, h_out, h_selected, h_edges, h_ecap); }));
  cudaStream_t st = ctx->stream;
  GB_CUDA(cudaMemsetAsync(d_out, 0, sizeof(McOut), st));
  GB_CUDA(cudaMemsetAsync(&d_out->seed_key, 0xff, sizeof(unsigned long long), st));
  GB_CUDA(cudaMemsetAsync(d_e, 0, sizeof(long long) * 2 * N, st));
  GB_CUDA(cudaMemsetAsync(d_cnt, 0, sizeof(int) * 3, st));
  const double r1 = prm->background_mask_radius + 1.0;
  const double fg = prm->foreground_mask_radius, bg = prm->background_mask_radius, sd = prm->distance_sigma, sa = prm->angle_sigma;
  const int gb = (n + kSegThreads - 1) / kSegThreads;
  GB_CHECK(gb_launch(ctx, "k_mc_flags", k_mc_flags, gb, kSegThreads, 0, n, cloud->p0, cloud->perm, c[0], c[1], c[2], r1 * r1, d_flags, d_out));
  GB_CUB(ctx, cub::DeviceScan::InclusiveSum, d_cub, cub_b, d_flags, d_pos, n);
  GB_CHECK(gb_launch(ctx, "k_mc_nodes", k_mc_nodes, gb, kSegThreads, 0, n, cloud->p0, cloud->normals, cloud->inv_perm, d_flags, d_pos, c[0], c[1], c[2], fg * fg, bg * bg,
                     d_pts, d_nrm, d_orig, d_role, d_out));
  GB_CHECK(knn_device(ctx, n, &d_out->num_points, d_pts, k, 0.25, d_nb, knn));
  GB_CHECK(gb_launch(ctx, "k_mc_arcs", k_mc_arcs, (nk + kSegThreads - 1) / kSegThreads, kSegThreads, 0, nk, k, d_nb, d_keys));
  GB_CUB(ctx, cub::DeviceRadixSort::SortKeys, d_cub, cub_b, d_keys, d_keys_s, na, 0, end_bit);
  const int ga = (na + kSegThreads - 1) / kSegThreads;
  GB_CHECK(gb_launch(ctx, "k_mc_unique", k_mc_unique, ga, kSegThreads, 0, na, d_keys_s, d_keys));
  GB_CUB(ctx, cub::DeviceScan::InclusiveSum, d_cub, cub_b, d_keys, d_apos, na);
  GB_CHECK(gb_launch(ctx, "k_mc_csr", k_mc_csr, ga, kSegThreads, 0, na, d_keys_s, d_apos, d_keys, d_eidx, d_out));
  const int slots = std::max(na, n + 1);
  GB_CHECK(gb_launch(ctx, "k_mc_graph", k_mc_graph, (slots + kSegThreads - 1) / kSegThreads, kSegThreads, 0, slots, d_keys, d_eidx, d_pts, d_nrm, d_orig, 2.0 * sd * sd,
                     2.0 * sa * sa, d_out, d_head, d_rev, d_cap, d_row, d_edges, d_ecap));
  McSolve S;
  S.n = n;
  S.fg_cap = (int)floor(prm->foreground_weight * kMcScale);
  S.row = d_row;
  S.head = d_head;
  S.rev = d_rev;
  S.cap = d_cap;
  S.role = d_role;
  S.res = d_res;
  S.fg_res = d_fg;
  S.h0 = d_h0;
  S.h1 = d_h1;
  S.e = d_e;
  S.incoming = d_in;
  S.cnt = d_cnt;
  S.sel = d_sel;
  S.out = d_out;
  // a persistent grid: as many CTAs as can be resident at once (the runtime refuses more), and no more than the slots need
  int per_sm = 0;
  GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_mc_solve, kMcThreads, 0));
  const int blocks = std::max(1, std::min(per_sm * ctx->num_sms, (n + kMcThreads - 1) / kMcThreads));
  GB_CHECK(gb_launch(ctx, "k_mc_solve", gb_cooperative, k_mc_solve, blocks, kMcThreads, 0, S));
  GB_CUB(ctx, cub::DeviceSelect::Flagged, d_cub, cub_b, d_orig, d_sel, d_selected, &d_out->num_selected, n);
  const char* end = graph ? (const char*)(d_ecap + nk) : (const char*)(d_selected + N);
  GB_CUDA(cudaMemcpyAsync(h_out, d_out, (size_t)(end - (const char*)d_out), cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  result->num_points = (size_t)h_out->num_points;
  result->num_foreground = (size_t)h_out->num_foreground;
  result->num_background = (size_t)h_out->num_background;
  result->num_edges = (size_t)h_out->num_edges;
  if (h_out->seed_key == ~0ull) return GB_OK;
  result->seed = (int32_t)(uint32_t)h_out->seed_key;
  result->status = h_out->status;
  result->num_selected = (size_t)h_out->num_selected;
  result->cut_value = h_out->cut_value;
  result->rounds = h_out->rounds;
  if (selected) memcpy(selected, h_selected, sizeof(int32_t) * result->num_selected);
  if (edges) memcpy(edges, h_edges, sizeof(int32_t) * 2 * result->num_edges);
  if (capacities) memcpy(capacities, h_ecap, sizeof(int32_t) * result->num_edges);
  return GB_OK;
}
