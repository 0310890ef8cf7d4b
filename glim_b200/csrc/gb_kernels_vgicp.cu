// gb_kernels_vgicp.cu -- the fused VGICP linearize / error sweep and the overlap kernel (sm_90a).
//
// Replaces gtsam_points::IntegratedVGICPFactorGPU::linearize / ::error as driven by
// NonlinearFactorSetGPU (GLIM call sites: src/glim/odometry/odometry_estimation_gpu.cpp:144,161,383-386;
// src/glim/mapping/sub_mapping.cpp:307; src/glim/mapping/global_mapping.cpp:466) and
// gtsam_points::overlap_gpu (odometry_estimation_gpu.cpp:231,248).  Math: SURVEY.md Appendix A;
// oracle: go_vgicp_linearize_gpumap / go_vgicp_error_gpumap / go_overlap_gpumap (oracle/glim_oracle.c).
//
// One launch covers a whole factor set.  Work unit = an item: a set of source points of one factor (consecutive points
// in sweep3, strided rows in sweep5, below); items are laid out factor-major and processed by the warps of a persistent
// grid (first item = warp index, further items from a global queue), so at any instant the grid works on a
// window of a few consecutive factors whose source cloud and voxel tables stay L2 resident.
// Both kernels run the same steps, written once in gb_sweep_steps.cuh (k_gicp_sweep of gb_kernels_gicp.cu runs them too): phase A (probe_issue, probe_resolve, probe_compact) resolves a round of points
// into the warp's shared-memory queue of hits, phase B (accumulate_queue) accumulates them, then reduce_item and the
// item's ticket (ticket_last); the warp that draws a factor's last ticket retires it (retire_factor).
// Per inlier (one lane):
//   q = R a + t -> voxel coord -> hash probe (sweep3: one 16-byte set of the target's probe index, gb_probe_index.cuh;
//   sweep5: 16-byte buckets) -> 48-byte voxel record ->
//   S = C_B + R C_A R^T, M = S^-1 (symmetric 3x3) -> accumulate the 21 unique entries of
//   H_tt = J_t^T M J_t (J_t = [-hat(q) | I]), the 6 of b_t = J_t^T M r, the error r^T M r and the
//   inlier count: 29 registers.
// Per item: transposing warp reduce-scatter (31 shuffles for 32 values) and 29 fp64 reductions (RED) into the
// factor's accumulator.  The warp that retires a factor's last item runs the fp64 epilogue:
// H_ts = -H_tt Ad, H_ss = Ad^T H_tt Ad, b_s = -Ad^T b_t with Ad = AdjointMap(delta) (SURVEY A.4),
// writes the 122-double record (and pushes the finished pair row to every rank's slab when one is attached),
// and re-zeroes the accumulator for the next sweep.
//
// Two sweep kernels live here; gb_sweep_create picks by sweep size (GB_KERNEL = 3 / 5 forces one):
//   k_vgicp_sweep3  large sweeps (sub mapping, global mapping): contiguous items of up to 2048 points from a global queue,
//                   register-staged loads, lazily published release tickets, tapered items at the tail of the sweep.
//   k_vgicp_sweep5  small sweeps (an odometry frame, a single pair -- about one item per warp): one wave of STRIDED items
//                   sized by each factor's last inlier fraction, descriptor / pose cache in shared memory.
#include "gb_internal.cuh"
#include "gb_vgicp_math.cuh"  // PoseF, transform, fused_mahalanobis, accumulate_hit, surface_ok, slab_to_record (also compiled for the host by the CPU test)
#include "gb_overlap_math.cuh"  // overlap_delta and k_overlap's item lookup (also compiled for the host by the CPU test)

#include "gb_sweep_steps.cuh"  // the steps every sweep kernel runs (shared with k_gicp_sweep, gb_kernels_gicp.cu)

namespace {

// =============================================================================================
// k_vgicp_sweep3 -- the large-sweep kernel: register-staged loads, contiguous items drawn from a global queue (the atomic
// for the next item is issued at the start of the current one).  An item's completion ticket is published LAZILY: an
// atom.release issued while the next item's first loads are in flight (no __threadfence, i.e. no MEMBAR.SC + L1
// invalidation per item), and a factor's epilogue runs after the next item's reduction.  Measured on the global-mapping
// sweep and its 1/8 shards: faster than a fence + ticket per item.
// An item's 29 accumulators are in registers only while a round's hits are accumulated (phase B); between rounds each lane
// parks them in its column of the warp's shared memory, so that phase A has those registers for probes in flight.  A lane
// adds its hits in the same order as with the accumulators live across the item, so the results are bit-identical.
// Tried and dropped: reading the queue one item ahead in registers (slower: the kernel sits at the 128-register
// cap); copying the next item's descriptor / pose to shared memory with cp.async during the current item (slower: the
// three dependent L2 round trips between two items are already covered by the other 15 warps of the SM); folding each
// round's accumulators over the warp (warp_reduce_scatter32) into one running float per lane instead of parking them
// (some 150 instructions per round; slower than the live accumulators at every probe count tried, DESIGN.md 4.1).
// =============================================================================================
// sweep3's shared memory per warp: the queue (a round's hits and the up to 31 carried from the previous round, one word
// each: probe_compact) and the parked accumulators.  Four 256-point lookup groups per round: 63.5 KB of dynamic shared
// memory per CTA, 127 KB per SM at 2 CTAs / SM.  Rounds of two groups in 48 KB per CTA (more L1) measured 1.2 % slower on
// the global-mapping sweep, and rounds of a whole 2048-point item (96 KB per CTA) 3 % slower (DESIGN.md 4.1).  The block is
// 16-byte aligned: the retiring warp reuses its queue as double / float4 scratch (retire_factor).
constexpr int kQueue3 = 4 * 256 + 31;
struct __align__(16) Sweep3Warp {
  unsigned q[kQueue3];
  float acc[29][32];  // acc[k][lane]: conflict-free
};
constexpr size_t kSmem3 = sizeof(Sweep3Warp) * kWarps;
// Probes per lane in flight.  Linearize: 8 (6 or 7 measured no faster than 5 with live accumulators on the global-mapping
// sweep, 8 is 4.7 % faster), four groups per 1024-point round.  Error: 7 (8 spills).  With surface validation (a dense odometry
// frame, livox_stress): 5, which measured 1.2 % faster than 8 there (7: 0.8 %, 6: 0.5 %), one group per round (three
// groups, 480 points, measured 0.5 % slower there).
template <int MODE, bool SV> constexpr int kLookupUnroll3 = SV ? 5 : MODE == GB_MODE_LINEARIZE ? 8 : 7;
template <int MODE, bool SV> constexpr int kRound3 = 32 * kLookupUnroll3<MODE, SV> * (SV ? 1 : (kQueue3 - 31) / (32 * kLookupUnroll3<MODE, SV>));  // points per round: whole lookup groups
static_assert(kRound3<GB_MODE_LINEARIZE, false> > 0 && kRound3<GB_MODE_ERROR, false> > 0 && kRound3<GB_MODE_LINEARIZE, true> > 0,
              "a round's hits and the up to 31 carried from the previous round fit the queue");

template <int MODE, bool PEER, bool SV>
__global__ void __launch_bounds__(kThreads, 2) k_vgicp_sweep3(
  const FactorDesc* __restrict__ descs, const IndexDesc* __restrict__ idescs, const double* __restrict__ poses, const double* __restrict__ poses_eval,
  const int2* __restrict__ items, int num_items,
  unsigned long long* __restrict__ item_ctr, unsigned long long ctr_base,
  double* __restrict__ accum, int acc_slots, unsigned* __restrict__ done, double* __restrict__ out, float* __restrict__ slab, const PeerPush* __restrict__ peer) {
  extern __shared__ __align__(16) unsigned char s_sweep3[];  // kSmem3 bytes
  Sweep3Warp* const s_w = reinterpret_cast<Sweep3Warp*>(s_sweep3);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  unsigned* __restrict__ q = s_w[warp].q;
  float (*__restrict__ parked)[32] = s_w[warp].acc;
  auto desc_of = [&](int f) { return descs[f]; };  // a copy, for retire_factor
  constexpr int U = kLookupUnroll3<MODE, SV>, kRound = kRound3<MODE, SV>;

  // first item: static (warp id); further items (only when there are more items than warps) come from the global queue
  const int total_warps = gridDim.x * kWarps;
  const bool dynamic = num_items > total_warps;
  int item = blockIdx.x * kWarps + warp;
  if (item >= num_items) return;
  int2 it = __ldg(&items[item]);
  int pend_f = -1, pend_last = 0, pend_tiles = 0;  // the previous item: its factor, whether it was the last, the factor's items
  auto pend_count = [&] { return pend_tiles; };

  while (true) {
    int next_item = 0x7fffffff;
    if (dynamic && lane == 0) next_item = (int)(atomicAdd(item_ctr, 1ull) - ctr_base) + total_warps;  // latency hidden behind the item
    const int f = it.x;
    const FactorDesc D = descs[f];
    const IndexDesc I = idescs[f];
    const PoseF P = pose_from_colmajor(poses + (size_t)f * 16);
    PoseF Pe = P;
    if (MODE == GB_MODE_ERROR) Pe = pose_from_colmajor(poses_eval + (size_t)f * 16);
    const int item_end = min(it.y + D.chunk, D.n);  // per-factor item size (the tail of a sweep is tapered)
    bool published = pend_f < 0;
    bool held = false;  // warp-uniform: the item's accumulators are parked (else they are all zero)
    auto unpark = [&](float (&acc)[32]) {
#pragma unroll
      for (int k = 0; k < 32; k++) acc[k] = held && k < 29 && (MODE == GB_MODE_LINEARIZE || k >= 27) ? parked[k][lane] : 0.f;
    };

    int nq = 0;  // warp-uniform queue length
    for (int wb = it.y; wb < item_end; wb += kRound) {
      const int we = min(wb + kRound, item_end);
      for (int i0 = wb; i0 < we; i0 += 32 * U) {
        IndexProbe p[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          const float4 a0 = __ldg(&D.p0[min(i0 + u * 32 + lane, we - 1)]);
          probe_issue(D, I, P, a0.x, a0.y, a0.z, p[u]);
        }
        if (!published) {  // the MEMBAR of the release overlaps with the loads above
          published = true;
          __syncwarp();
          if (lane == 0) pend_last = ticket_last(done, pend_f, pend_count);
        }
        int v[U];
        probe_resolve(I, p, v);
#pragma unroll
        for (int u = 0; u < U; u++) probe_compact(v[u], i0 + u * 32 + lane, we, it.y, q, nq, lt_mask);
      }
      __syncwarp();
      // Whole passes of 32 hits only: the last nq % 32 hits are carried to the front of the queue for the next round (a
      // pass costs a round trip however few lanes it fills), except in the item's last round.
      const int nacc = we == item_end ? nq : (nq & ~31);
      if (nacc > 0) {
        float acc[32];
        unpark(acc);
        // surface validation is a compile-time variant here (GLIM enables it for odometry factors only, which run sweep5)
        accumulate_queue<MODE, SV>(acc, D, P, Pe, q, nacc, lane, it.y);
#pragma unroll
        for (int k = 0; k < 29; k++)
          if (MODE == GB_MODE_LINEARIZE || k >= 27) parked[k][lane] = acc[k];
        held = true;
      }
      __syncwarp();  // the queue is overwritten by the next round
      nq -= nacc;
      if (nacc > 0 && lane < nq) q[lane] = q[nacc + lane];  // nacc >= 32 > nq: the ranges do not overlap
      __syncwarp();
    }
    if (!published) {  // the item had no lookup group (empty factor)
      __syncwarp();
      if (lane == 0) pend_last = ticket_last(done, pend_f, pend_count);
    }

    float acc[32];
    unpark(acc);
    reduce_item<MODE>(acc, accum, f, acc_slots, item, lane);
    if (pend_f >= 0 && __shfl_sync(0xffffffffu, pend_last, 0)) {  // the PREVIOUS item completed its factor
      fence_acquire();
      retire_factor<MODE, PEER>(pend_f, desc_of(pend_f), poses, poses_eval, accum, acc_slots, out, slab, peer, q);
      __syncwarp();
    }
    pend_f = f; pend_tiles = D.num_tiles; pend_last = 0;
    item = __shfl_sync(0xffffffffu, next_item, 0);
    if (item >= num_items) break;
    it = __ldg(&items[item]);
  }
  __syncwarp();
  if (lane == 0) pend_last = ticket_last(done, pend_f, pend_count);
  if (__shfl_sync(0xffffffffu, pend_last, 0)) {
    fence_acquire();
    retire_factor<MODE, PEER>(pend_f, desc_of(pend_f), poses, poses_eval, accum, acc_slots, out, slab, peer, q);
  }
}

constexpr int kSubMax = 512;  // queue capacity per warp (points per round)
constexpr int kLookupUnroll5 = 4;  // probes per lane in flight (5 spills)
constexpr int kDescCache = 40;  // factors whose descriptor + fp32 pose are cached in shared memory (an odometry graph has <= 34)
struct CtaCache {
  FactorDesc desc[kDescCache];
  PoseF pose[kDescCache];
  PoseF pose_eval[kDescCache];
};

// =============================================================================================
// k_vgicp_sweep5 -- the small-sweep kernel: register-staged like sweep3 (no large shared-memory carve-out: L1 stays big),
// with the per-item latency chain cut and the one-wave regime balanced:
//   * descriptor / fp32-pose cache in shared memory for small factor sets (an odometry graph), one-item look-ahead of the
//     work queue, lazily published release tickets (atom.release: no __threadfence, no L1 flush per item);
//   * STRIDED items, about one per warp in a small sweep (odometry, single pair): item j of a factor with J items owns
//     the 32-point rows j, j + J, j + 2J, ... of the source cloud, so every item of a factor samples the whole (Morton-
//     ordered) cloud and sees the same inlier rate; the host sizes J per factor from the factor's last inlier fraction
//     (a hit costs ~2.2x a miss).  One wave of equally expensive items instead of a tail of all-inlier items.
// =============================================================================================
template <int MODE, bool PEER>
__global__ void __launch_bounds__(kThreads, 2) k_vgicp_sweep5(
  const FactorDesc* __restrict__ descs, int num_factors, const double* __restrict__ poses, const double* __restrict__ poses_eval,
  const int2* __restrict__ items, int num_items,
  unsigned long long* __restrict__ item_ctr, unsigned long long ctr_base,
  double* __restrict__ accum, int acc_slots, unsigned* __restrict__ done, double* __restrict__ out, float* __restrict__ slab, const PeerPush* __restrict__ peer) {
  __shared__ __align__(16) uint2 s_q[kWarps][kSubMax];
  __shared__ CtaCache cache_s;
  CtaCache* const cache = &cache_s;
  constexpr int U = kLookupUnroll5;
  constexpr int kGroupsPerRound = kSubMax / (32 * U);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  uint2* __restrict__ q = s_q[warp];

  const bool cached = num_factors <= kDescCache;
  if (cached) {
    for (int f = threadIdx.x; f < num_factors; f += kThreads) {
      cache->desc[f] = descs[f];
      cache->pose[f] = pose_from_colmajor(poses + (size_t)f * 16);
      if (MODE == GB_MODE_ERROR) cache->pose_eval[f] = pose_from_colmajor(poses_eval + (size_t)f * 16);
    }
    __syncthreads();  // the only block-level barrier of the kernel
  }
  // descriptor reads keep their address space (LDS from the cache or LDG from the table)
  auto desc_of = [&](int f) -> FactorDesc { FactorDesc d; if (cached) d = cache->desc[f]; else d = descs[f]; return d; };

  const int total_warps = gridDim.x * kWarps;
  const bool dynamic = num_items > total_warps;
  int item = blockIdx.x * kWarps + warp;  // first item: static
  if (item >= num_items) return;
  int nxt = 0x7fffffff;  // one-item look-ahead of the queue
  if (dynamic) {
    if (lane == 0) nxt = (int)(atomicAdd(item_ctr, 1ull) - ctr_base) + total_warps;
    nxt = __shfl_sync(0xffffffffu, nxt, 0);
  }
  int2 it = __ldg(&items[item]);
  int pend_f = -1, pend_last = 0;
  auto pend_count = [&] { return desc_of(pend_f).num_tiles; };

  while (true) {
    int nxt2 = 0x7fffffff;
    if (dynamic && lane == 0) nxt2 = (int)(atomicAdd(item_ctr, 1ull) - ctr_base) + total_warps;
    int2 it_next = make_int2(0, 0);
    if (nxt < num_items) it_next = __ldg(&items[nxt]);  // the next item's identity travels while this item is processed
    const int f = it.x;
    const FactorDesc D = desc_of(f);
    PoseF P;
    if (cached) P = cache->pose[f]; else P = pose_from_colmajor(poses + (size_t)f * 16);
    PoseF Pe = P;
    if (MODE == GB_MODE_ERROR) { if (cached) Pe = cache->pose_eval[f]; else Pe = pose_from_colmajor(poses_eval + (size_t)f * 16); }

    // the item's points: the rows it.y, it.y + J, ... (32 points each) of the cloud, J = the factor's item count
    const int limit = D.n;
    const int row_stride = D.num_tiles * 32;
    const int first = it.y * 32;
    int ngroups = 0;
    if (first < limit) {
      const int rows = (limit - first + row_stride - 1) / row_stride;  // ceil((R - j) / J)
      ngroups = (rows + U - 1) / U;
    }

    float acc[32];
#pragma unroll
    for (int k = 0; k < 32; k++) acc[k] = 0.f;
    bool published = (pend_f < 0);

    for (int g0 = 0; g0 < ngroups; g0 += kGroupsPerRound) {
      const int g1 = min(g0 + kGroupsPerRound, ngroups);
      int nq = 0;  // warp-uniform queue length
      // ---------------- phase A: lookup + compaction ----------------
      float ax[U], ay[U], az[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const int i = first + (g0 * U + u) * row_stride + lane;
        const float4 a0 = __ldg(&D.p0[i < limit ? i : 0]);
        ax[u] = a0.x; ay[u] = a0.y; az[u] = a0.z;
      }
      for (int g = g0; g < g1; g++) {
        Probe p[U];
#pragma unroll
        for (int u = 0; u < U; u++) probe_issue(D, P, ax[u], ay[u], az[u], p[u]);
        if (!published) {  // the previous item's ticket: the MEMBAR of the release overlaps with the loads above
          published = true;
          __syncwarp();
          if (lane == 0) pend_last = ticket_last(done, pend_f, pend_count);
        }
        int v[U];
        probe_resolve(D, p, v);
#pragma unroll
        for (int u = 0; u < U; u++) probe_compact(v[u], first + (g * U + u) * row_stride + lane, limit, q, nq, lt_mask);
        if (g + 1 < g1) {  // the next group's points, loaded after this group is resolved
#pragma unroll
          for (int u = 0; u < U; u++) {
            const int i = first + ((g + 1) * U + u) * row_stride + lane;
            const float4 a0 = __ldg(&D.p0[i < limit ? i : 0]);
            ax[u] = a0.x; ay[u] = a0.y; az[u] = a0.z;
          }
        }
      }
      __syncwarp();
      accumulate_queue<MODE, true>(acc, D, P, Pe, q, nq, lane);
      __syncwarp();  // the queue is overwritten by the next round
    }
    if (!published) {  // empty item
      __syncwarp();
      if (lane == 0) pend_last = ticket_last(done, pend_f, pend_count);
    }

    reduce_item<MODE>(acc, accum, f, acc_slots, item, lane);
    // epilogue of the PREVIOUS item's factor, if that item was its last
    if (pend_f >= 0 && __shfl_sync(0xffffffffu, pend_last, 0)) {
      fence_acquire();
      retire_factor<MODE, PEER>(pend_f, desc_of(pend_f), poses, poses_eval, accum, acc_slots, out, slab, peer, q);
      __syncwarp();
    }
    pend_f = f;
    pend_last = 0;
    item = nxt;
    it = it_next;
    nxt = __shfl_sync(0xffffffffu, nxt2, 0);
    if (item >= num_items) break;
  }
  __syncwarp();
  if (lane == 0) pend_last = ticket_last(done, pend_f, pend_count);
  if (__shfl_sync(0xffffffffu, pend_last, 0)) {
    fence_acquire();
    retire_factor<MODE, PEER>(pend_f, desc_of(pend_f), poses, poses_eval, accum, acc_slots, out, slab, peer, q);
  }
}

// overlap: the source points of each query that hit an occupied voxel of any of its targets.  A query (OverlapQuery) is a
// source cloud and a range of (target descriptor, pose); gb_overlap is one query of T targets, gb_find_overlapping_submaps
// P queries of one target each, whose relative pose is computed here from the world poses of the pair.  Work items are
// (query, chunk of kOverlapChunk consecutive points), numbered query-major in 64 bits (gb_overlap_math.cuh).  A block takes
// items from a static grid stride, one point per thread, and adds the item's hits to the query's int count with one atomic:
// the counts do not depend on the order.
__global__ void __launch_bounds__(kOverlapChunk) k_overlap(const OverlapQuery* __restrict__ queries, const int* __restrict__ num_queries, const long long* __restrict__ item_end,
                                                           const FactorDesc* __restrict__ descs, const double* __restrict__ poses, const double* __restrict__ world,
                                                           int* __restrict__ counts) {
  extern __shared__ float s_poses[];  // the item's query: num_targets x 12
  __shared__ int s_q;
  const int nq = *num_queries;
  if (nq <= 0) return;
  const long long items = item_end[nq - 1];
  int q_lo = 0;  // a block's items ascend, and so do their queries
  for (long long item = blockIdx.x; item < items; item += gridDim.x) {
    if (threadIdx.x == 0) s_q = overlap_item_query(item_end, nq, q_lo, item);
    __syncthreads();
    const int q = s_q;
    q_lo = q;
    const OverlapQuery Q = queries[q];
    for (int k = threadIdx.x; k < Q.num_targets * 12; k += blockDim.x) {
      const int t = k / 12, e = k % 12;
      const int r = e < 9 ? e / 3 : e - 9, c = e < 9 ? e % 3 : 3;
      // a query with pose < 0 (one target): the relative pose of the pair (target, source), one entry per thread
      const double v = Q.pose < 0 ? overlap_delta_entry(world + 16 * (size_t)Q.target, world + 16 * (size_t)Q.source, r, c) : poses[(size_t)(Q.pose + t) * 16 + c * 4 + r];
      s_poses[k] = (float)v;
    }
    __syncthreads();
    const int i = overlap_item_point(item_end, q, item) + threadIdx.x;
    const int n = descs[Q.source].n;
    bool hit = false;
    if (i < n) {
      const float4 a0 = __ldg(&descs[Q.source].p0[i]);
      for (int t = 0; t < Q.num_targets && !hit; t++) {
        const PoseF P = load_pose(s_poses + 12 * t);
        float qx, qy, qz;
        transform(P, a0.x, a0.y, a0.z, qx, qy, qz);
        const float sum = (qx + qy) + qz;
        if (!(sum == sum)) continue;  // NaN point: no voxel
        const FactorDesc& D = descs[Q.target + t];
        const float inv_res = D.inv_res;
        hit = gb_lookup(D.buckets, D.mask, D.max_scan, gb_coord(qx, inv_res), gb_coord(qy, inv_res), gb_coord(qz, inv_res)) >= 0;
      }
    }
    const int c = __syncthreads_count(hit);  // also the barrier before s_q and s_poses are rewritten
    if (threadIdx.x == 0 && c) atomicAdd(&counts[q], c);
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------
template <int MODE, bool PEER>
static gb_status launch5(gb_sweep* s, const double* poses_eval, float* slab, const PeerPush* pp) {
  return gb_launch(s->ctx, "k_vgicp_sweep5", k_vgicp_sweep5<MODE, PEER>, s->grid, kThreads, 0, s->d_descs, (int)s->F, s->d_poses, poses_eval, s->d_tiles, s->num_tiles, s->d_tile_ctr,
                   s->ctr_base, s->d_accum, s->acc_slots, s->d_done, s->d_out, slab, pp);
}

template <int MODE, bool PEER, bool SV>
static gb_status launch3(gb_sweep* s, const double* poses_eval, float* slab, const PeerPush* pp) {
  // above 48 KB of dynamic shared memory a kernel must opt in, per device: set at every launch (a host-side attribute write)
  GB_CUDA(cudaFuncSetAttribute(k_vgicp_sweep3<MODE, PEER, SV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem3));
  return gb_launch(s->ctx, "k_vgicp_sweep3", k_vgicp_sweep3<MODE, PEER, SV>, s->grid, kThreads, kSmem3, s->d_descs, s->d_idescs, s->d_poses, poses_eval, s->d_tiles, s->num_tiles, s->d_tile_ctr,
                   s->ctr_base, s->d_accum, s->acc_slots, s->d_done, s->d_out, slab, pp);
}

gb_status gb_launch_sweep(gb_sweep* s, int mode) {
  if (s->num_tiles == 0) return GB_OK;
  if (s->gicp) return gb_launch_gicp_sweep(s, mode);  // gb_kernels_gicp.cu
  // the table for the buffer of the current step parity (both were written to the device when the slab was attached)
  const bool peer = (mode == GB_MODE_LINEARIZE) && s->peer != nullptr;
  const PeerPush* pp = peer ? s->d_peer_tables + s->peer->parity : nullptr;
  float* slab = mode == GB_MODE_LINEARIZE ? s->d_slab : nullptr;
  const double* pe = mode == GB_MODE_ERROR ? s->d_poses_eval : nullptr;
  gb_status st;
  if (s->kernel_version == 3) {
    if (s->any_sv) {
      if (mode == GB_MODE_LINEARIZE) st = peer ? launch3<GB_MODE_LINEARIZE, true, true>(s, pe, slab, pp) : launch3<GB_MODE_LINEARIZE, false, true>(s, pe, slab, pp);
      else st = launch3<GB_MODE_ERROR, false, true>(s, pe, slab, pp);
    } else {
      if (mode == GB_MODE_LINEARIZE) st = peer ? launch3<GB_MODE_LINEARIZE, true, false>(s, pe, slab, pp) : launch3<GB_MODE_LINEARIZE, false, false>(s, pe, slab, pp);
      else st = launch3<GB_MODE_ERROR, false, false>(s, pe, slab, pp);
    }
  } else {
    if (mode == GB_MODE_LINEARIZE) st = peer ? launch5<GB_MODE_LINEARIZE, true>(s, pe, slab, pp) : launch5<GB_MODE_LINEARIZE, false>(s, pe, slab, pp);
    else st = launch5<GB_MODE_ERROR, false>(s, pe, slab, pp);
  }
  GB_CHECK(st);
  // queue bookkeeping: a sweep with more items than warps draws one ticket per processed item, plus, for sweep5, one per warp
  // for its one-item look-ahead
  const unsigned long long warps = (unsigned long long)s->grid * kWarps;
  if ((unsigned long long)s->num_tiles > warps) s->ctr_base += (s->kernel_version == 3 ? 0ull : warps) + (unsigned long long)s->num_tiles;
  return GB_OK;
}

gb_status gb_launch_overlap(gb_ctx* ctx, int grid, int max_targets, const OverlapQuery* d_queries, const int* d_num_queries, const long long* d_item_end,
                            const FactorDesc* d_descs, const double* d_poses, const double* d_world, int* d_counts) {
  if (grid <= 0 || max_targets <= 0) return GB_OK;
  return gb_launch(ctx, "k_overlap", k_overlap, grid, kOverlapChunk, (size_t)max_targets * 12 * sizeof(float), d_queries, d_num_queries, d_item_end, d_descs, d_poses,
                   d_world, d_counts);
}
