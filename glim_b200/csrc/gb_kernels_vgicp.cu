// gb_kernels_vgicp.cu -- the fused VGICP linearize / error sweep and the overlap kernel (sm_90a).
//
// Replaces gtsam_points::IntegratedVGICPFactorGPU::linearize / ::error as driven by
// NonlinearFactorSetGPU (GLIM call sites: src/glim/odometry/odometry_estimation_gpu.cpp:144,161,383-386;
// src/glim/mapping/sub_mapping.cpp:307; src/glim/mapping/global_mapping.cpp:466) and
// gtsam_points::overlap_gpu (odometry_estimation_gpu.cpp:231,248).  Math: SURVEY.md Appendix A;
// oracle: go_vgicp_linearize_gpumap / go_vgicp_error_gpumap / go_overlap_gpumap (oracle/glim_oracle.c).
//
// One launch covers a whole factor set.  Work unit = an item of up to `chunk` consecutive source
// points of one factor; items are laid out factor-major and processed by the warps of a persistent grid
// (first item = warp index, further items from a global queue), so at any instant the grid works on a
// window of a few consecutive factors whose source cloud and voxel tables stay L2 resident.
// Per inlier (one lane):
//   q = R a + t -> voxel coord -> hash probe (16-byte buckets) -> 48-byte voxel record ->
//   S = C_B + R C_A R^T, M = S^-1 (symmetric 3x3) -> accumulate the 21 unique entries of
//   H_tt = J_t^T M J_t (J_t = [-hat(q) | I]), the 6 of b_t = J_t^T M r, the error r^T M r and the
//   inlier count: 29 registers.
// Per item: transposing warp reduce-scatter (31 shuffles for 32 values) and 29 fp64 reductions (RED) into the
// factor's accumulator.  The warp that retires a factor's last item runs the fp64 epilogue:
// H_ts = -H_tt Ad, H_ss = Ad^T H_tt Ad, b_s = -Ad^T b_t with Ad = AdjointMap(delta) (SURVEY A.4),
// writes the 122-double record (and pushes the finished pair row to every rank's slab when one is attached),
// and re-zeroes the accumulator for the next sweep.
//
// Three sweep kernels live here; gb_sweep_create picks by sweep size (GB_KERNEL = 3 / 4 / 5 forces one):
//   k_vgicp_sweep3  large sweeps (sub mapping, global mapping): contiguous items of up to 2048 points from a global queue,
//                   register-staged loads, lazily published release tickets, tapered items at the tail of the sweep.
//   k_vgicp_sweep5  small sweeps (an odometry frame, a single pair -- about one item per warp): one wave of STRIDED items
//                   sized by each factor's last inlier fraction, descriptor / pose cache in shared memory.
//   k_vgicp_sweep4  experiment, never the default: source tiles staged into shared memory by bulk async copies
//                   (cp.async.bulk / UBLKCP + mbarrier).  Slower than sweep3 when it was measured: the
//                   carve-out shrinks L1 and the path is latency-, not issue-bound.  Kept as the measured negative result.
#include "gb_internal.cuh"
#include "gb_vgicp_math.cuh"  // PoseF, transform, fused_mahalanobis, accumulate_hit, surface_ok, slab_to_record (also compiled for the host by the CPU test)

#include <stdlib.h>
#include <string.h>

namespace {

static_assert(GB_MODE_LINEARIZE == GB_MODE_LINEARIZE_VALUE, "gb_vgicp_math.cuh mirrors the mode constant");
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// probe result of one point given its first two buckets (b, b1 fetched together: adjacent 16-byte slots, one round trip)
__device__ __forceinline__ int resolve_probe(const FactorDesc& D, const int4 b, const int4 b1, uint32_t h, int cx, int cy, int cz) {
  int v = -1;
  if (b.w >= 0) {
    if (b.x == cx && b.y == cy && b.z == cz) {
      v = b.w;
    } else if (D.max_scan > 1 && b1.w >= 0) {
      if (b1.x == cx && b1.y == cy && b1.z == cz) {
        v = b1.w;
      } else {
        for (int k = 2; k < D.max_scan; k++) {  // rare: longer collision chain
          const int4 bb = __ldg(&D.buckets[(h + (uint32_t)k) & D.mask]);
          if (bb.w < 0) break;
          if (bb.x == cx && bb.y == cy && bb.z == cz) { v = bb.w; break; }
        }
      }
    }
  }
  return v;
}

// Transposing warp reduction: on return lane l holds sum over the warp of v[l] (in v[0]).
__device__ __forceinline__ float warp_reduce_scatter32(float (&v)[32], int lane) {
#pragma unroll
  for (int step = 16; step >= 1; step >>= 1) {
    const bool upper = (lane & step) != 0;
#pragma unroll
    for (int j = 0; j < step; j++) {
      const float send = upper ? v[j] : v[j + step];
      const float keep = upper ? v[j + step] : v[j];
      v[j] = keep + __shfl_xor_sync(0xffffffffu, send, step);
    }
  }
  return v[0];
}

// release / acquire building blocks of the per-factor and per-pair tickets.  atom.release = MEMBAR.ALL.GPU + ATOMG: it does
// NOT invalidate L1 (a __threadfence() is MEMBAR.SC.GPU + CCTL.IVALL, i.e. an L1 flush of the whole SM per item).
__device__ __forceinline__ unsigned ticket_release(unsigned* p) {
  unsigned r;
  asm volatile("atom.add.release.gpu.global.u32 %0, [%1], 1;" : "=r"(r) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void fence_acquire() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }

// Fused result exchange: executed by the warp that completed factor f.  If f was the LAST factor of its pair, sum the
// pair's records (fp64, fixed order -> deterministic), and store the fp32 row into every rank's slab (128-bit stores;
// peers are reached through their IPC-mapped addresses over NVLink).
__device__ __noinline__ void pair_push(const FactorDesc& D, const double* __restrict__ out, const PeerPush* __restrict__ peer_tab, float* row /* 96 floats of shared memory */) {
  const PeerPush& peer = *peer_tab;
  const int lane = threadIdx.x & 31;
  __syncwarp();  // this factor's record (written by all lanes) happens-before the release below
  int last = 0;
  const int pb = peer.pair_ptr[D.pair], pe = peer.pair_ptr[D.pair + 1];
  if (lane == 0) {
    const unsigned t = ticket_release(&peer.pair_done[D.pair]);
    last = (t == (unsigned)(pe - pb) - 1u);
    if (last) peer.pair_done[D.pair] = 0u;
  }
  last = __shfl_sync(0xffffffffu, last, 0);
  if (!last) return;
  fence_acquire();
  for (int e = lane; e < GB_SLAB_STRIDE; e += 32) {
    double s = 0.0;
    if (e < 92) {
      const int r = slab_to_record(e);
      for (int k = pb; k < pe; k++) s += __ldcg(&out[(size_t)peer.pair_factors[k] * GB_OUT_DOUBLES + r]);
    }
    row[e] = (float)s;
  }
  __syncwarp();
  if (lane < GB_SLAB_STRIDE / 4) {
    const float4 v = reinterpret_cast<const float4*>(row)[lane];
    for (int p = 0; p < peer.world; p++) reinterpret_cast<float4*>(peer.base[p] + (size_t)D.pair * GB_SLAB_STRIDE)[lane] = v;
  }
}

// fp64 epilogue of one factor, executed (all 32 lanes in parallel) by the warp that retired the factor's last item.
// sm: >= 104 doubles of shared memory (A[32] | Ad[36] | X[36]).
constexpr int kEpilogueDoubles = 104;
__device__ __noinline__ void factor_epilogue(int f, const FactorDesc& D, const double* __restrict__ poses, double* __restrict__ accum, int acc_slots, double* __restrict__ out, float* __restrict__ slab, double* sm) {
  const int lane = threadIdx.x & 31;
  double* A = sm;        // 32 accumulators
  double* Ad = sm + 32;  // 6x6 adjoint, row-major
  double* X = sm + 68;   // H_tt * Ad, row-major
  // the accumulators were produced by L2 reductions of other CTAs: read them past L1
  // (a factor's accumulator is replicated over acc_slots copies so that the items of a sweep with FEW factors do not all
  //  serialise on the same 29 addresses in L2; summed here in slot order)
  if (lane < 29) {
    double a = 0.0;
    for (int sl = 0; sl < acc_slots; sl++) {
      double* slot = &accum[((size_t)f * acc_slots + sl) * GB_ACC_STRIDE + lane];
      a += __ldcg(slot);
      *slot = 0.0;  // re-zero for the next sweep (self-cleaning; nobody touches this factor again in this launch)
    }
    A[lane] = a;
  }
  // Ad = [[R, 0], [hat(t) R, R]] from the fp32-cast pose the kernel used
  const double* T = poses + (size_t)f * 16;
  for (int e = lane; e < 36; e += 32) {
    const int i = e / 6, j = e % 6;
    double v = 0.0;
    if (j < 3 || i >= 3) {
      const int ri = i % 3, cj = j % 3;
      if ((i < 3) == (j < 3)) {
        v = (double)(float)T[cj * 4 + ri];  // R(ri, cj)
      } else {  // i >= 3, j < 3: (hat(t) R)(ri, cj) = (t x R(:, cj))(ri)
        const double t0 = (double)(float)T[12], t1 = (double)(float)T[13], t2 = (double)(float)T[14];
        const double r0 = (double)(float)T[cj * 4 + 0], r1 = (double)(float)T[cj * 4 + 1], r2 = (double)(float)T[cj * 4 + 2];
        v = ri == 0 ? t1 * r2 - t2 * r1 : (ri == 1 ? t2 * r0 - t0 * r2 : t0 * r1 - t1 * r0);
      }
    }
    Ad[e] = v;
  }
  __syncwarp();
  // H(i, j) = A[index of (min, max) in the row-major upper triangle]
  auto H = [&](int i, int j) -> double {
    const int a = i < j ? i : j, b = i < j ? j : i;
    return A[a * 6 - (a * (a - 1)) / 2 + (b - a)];
  };
  for (int e = lane; e < 36; e += 32) {
    const int i = e / 6, j = e % 6;
    double s = 0;
    for (int k = 0; k < 6; k++) s += H(i, k) * Ad[k * 6 + j];
    X[e] = s;
  }
  __syncwarp();
  double* o = out + (size_t)f * GB_OUT_DOUBLES;
  float* srow = slab ? slab + (size_t)D.pair * GB_SLAB_STRIDE : nullptr;
  for (int e = lane; e < 36; e += 32) {
    const int i = e / 6, j = e % 6;  // output element (row i, col j), stored column-major
    double ss = 0;
    for (int k = 0; k < 6; k++) ss += Ad[k * 6 + i] * X[k * 6 + j];
    const double hij = H(i, j);
    o[j * 6 + i] = hij;                      // H_tt
    o[36 + j * 6 + i] = ss;                  // H_ss = Ad^T H_tt Ad
    o[72 + j * 6 + i] = -X[i * 6 + j];       // H_ts = -H_tt Ad
    if (srow) {
      atomicAdd(&srow[21 + j * 6 + i], (float)(-X[i * 6 + j]));
      if (j >= i) {
        const int u = i * 6 - (i * (i - 1)) / 2 + (j - i);  // index in the row-major upper triangle
        atomicAdd(&srow[u], (float)hij);
        atomicAdd(&srow[57 + u], (float)ss);
      }
    }
  }
  if (lane < 6) {
    double bs = 0;
    for (int k = 0; k < 6; k++) bs += Ad[k * 6 + lane] * A[21 + k];
    o[108 + lane] = A[21 + lane];
    o[114 + lane] = -bs;
    if (srow) { atomicAdd(&srow[78 + lane], (float)A[21 + lane]); atomicAdd(&srow[84 + lane], (float)(-bs)); }
  }
  if (lane == 6) { o[120] = A[27]; if (srow) atomicAdd(&srow[90], (float)A[27]); }
  if (lane == 7) { o[121] = A[28]; if (srow) atomicAdd(&srow[91], (float)A[28]); }
  __syncwarp();
}

// =============================================================================================
// k_vgicp_sweep4 -- bulk-async staged source tiles, lazy release tickets, carry-over hit queue
// =============================================================================================
//
// Per warp, in dynamic shared memory:
//   two stage buffers { float4 p0[T + 32]; float4 p1[T + 32]; float p2[T + 32]; }  -- the three planes of up to T consecutive
//       source points, filled by three cp.async.bulk (1-D TMA) copies that complete on the buffer's mbarrier; the last
//       32 slots of every plane are the CARRY area (see below);
//   a hit queue uint2 q[T + 32] = (slot in the current stage buffer, voxel index).
// The stream of stages of a warp (the stages of its items, one item after the other) is double buffered: while stage s is
// being processed, the copy of stage s + 1 -- possibly the first stage of the NEXT item, whose identity is known one item
// ahead -- is in flight.  Nothing in the lookup phase waits for a global load of the source cloud any more, and the
// derivative phase reads the point from shared memory instead of gathering 36 bytes from L2.
//   phase A (lookup, all lanes): LDS {x,y,z,c00} -> transform -> voxel coordinate -> hash -> first two buckets (LDG.128 x2,
//       T/32 points per lane in flight) -> compaction of the hits into q with ballot + popc, in point order.
//   phase B (derivatives): lanes walk q in groups of 32.  Only FULL groups are processed; the < 32 left-over hits are
//       copied (36 bytes each) into the carry area of the OTHER stage buffer and head the queue of the next stage, so the
//       ~200-instruction derivative pass always runs with 32 active lanes whatever the inlier rate.  The last stage of an
//       item flushes the partial group.
// Item end: transposing warp reduce-scatter (31 shuffles), 29 fp64 REDs into the factor's accumulator.  The ticket that
// counts the factor's finished items is published LAZILY with a release atomic (no fence, no L1 invalidation): while the
// first bucket loads of the warp's next item are in flight, the MEMBAR that the release implies waits for nothing that
// the warp was not going to wait for anyway.  The warp that draws a factor's last ticket runs the epilogue (acquire fence
// there only) at the end of the item in which it found out.
template <int T>
struct StageBuf {
  float4 p0[T + 32];
  float4 p1[T + 32];
  float p2[T + 32];
};
template <int T>
struct WarpSmem {
  StageBuf<T> buf[2];
  uint2 q[T + 32];
  unsigned long long mbar[2];
};
constexpr int kDescCache = 40;  // factors whose descriptor + fp32 pose are cached in shared memory (an odometry graph has <= 34)
struct CtaCache {
  FactorDesc desc[kDescCache];
  PoseF pose[kDescCache];
  PoseF pose_eval[kDescCache];
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, int count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
    "{\n"
    ".reg .pred P1;\n"
    "LAB_WAIT:\n"
    "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
    "@P1 bra DONE;\n"
    "bra LAB_WAIT;\n"
    "DONE:\n"
    "}\n" ::"r"(bar), "r"(parity) : "memory");
}

// lane 0: start the copy of `cnt` points [first, first + cnt) of a cloud into stage buffer `sb`
template <int T>
__device__ __forceinline__ void issue_stage(StageBuf<T>* sb, uint32_t bar, const float4* p0, const float4* p1, const float* p2, int first, int cnt) {
  const uint32_t b0 = (uint32_t)cnt * 16u, b2 = ((uint32_t)cnt * 4u + 15u) & ~15u;  // the p2 plane is padded to 256 B: reading <= 12 B past the item is safe
  mbar_expect_tx(bar, 2u * b0 + b2);
  bulk_g2s(smem_u32(sb->p0), p0 + first, b0, bar);
  bulk_g2s(smem_u32(sb->p1), p1 + first, b0, bar);
  bulk_g2s(smem_u32(sb->p2), p2 + first, b2, bar);
}

template <int MODE, int T, bool PEER, int MINB>
__global__ void __launch_bounds__(kThreads, MINB) k_vgicp_sweep4(
  const FactorDesc* __restrict__ descs, int num_factors, const double* __restrict__ poses, const double* __restrict__ poses_eval,
  const int2* __restrict__ items, int num_items, int chunk,
  unsigned long long* __restrict__ item_ctr, unsigned long long ctr_base,
  double* __restrict__ accum, int acc_slots, unsigned* __restrict__ done, double* __restrict__ out, float* __restrict__ slab, const PeerPush* __restrict__ peer) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int U = T / 32;  // points per lane per stage
  static_assert(sizeof(StageBuf<T>) >= (kEpilogueDoubles * 8 + GB_SLAB_STRIDE * 4), "a stage buffer doubles as the epilogue scratch");
  WarpSmem<T>* const ws_all = reinterpret_cast<WarpSmem<T>*>(smem_raw);
  CtaCache* const cache = reinterpret_cast<CtaCache*>(smem_raw + sizeof(WarpSmem<T>) * kWarps);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  WarpSmem<T>& ws = ws_all[warp];
  uint2* __restrict__ q = ws.q;
  const uint32_t bar0 = smem_u32(&ws.mbar[0]), bar1 = smem_u32(&ws.mbar[1]);

  // ---- CTA prologue: descriptor / pose cache (small factor sets), mbarriers ----
  const bool cached = num_factors <= kDescCache;
  if (cached) {
    for (int f = threadIdx.x; f < num_factors; f += kThreads) {
      cache->desc[f] = descs[f];
      cache->pose[f] = pose_from_colmajor(poses + (size_t)f * 16);
      if (MODE == GB_MODE_ERROR) cache->pose_eval[f] = pose_from_colmajor(poses_eval + (size_t)f * 16);
    }
  }
  if (lane == 0) {
    mbar_init(bar0, 1);
    mbar_init(bar1, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();  // the only block-level barrier of the kernel

  const int total_warps = gridDim.x * kWarps;
  const bool dynamic = num_items > total_warps;
  int item = blockIdx.x * kWarps + warp;  // first item: static
  if (item >= num_items) return;
  // second item: drawn now so that its identity is known one item ahead (its first stage is prefetched during the current item)
  int nxt = 0x7fffffff;
  if (dynamic) {
    if (lane == 0) nxt = (int)(atomicAdd(item_ctr, 1ull) - ctr_base) + total_warps;
    nxt = __shfl_sync(0xffffffffu, nxt, 0);
  }

  // Descriptor reads keep their address space (LDS from the cache or LDG from the table): a merged generic pointer made the
  // compiler re-load D.mask / D.inv_res with generic LD.E inside the stage loop (a large share of the stall samples of the first version).
  auto desc_of = [&](int f) -> FactorDesc { FactorDesc d; if (cached) d = cache->desc[f]; else d = descs[f]; return d; };
  auto tiles_of = [&](int f) -> int { return cached ? cache->desc[f].num_tiles : descs[f].num_tiles; };
  // lane 0: start the copy of `cnt` points of factor f's source cloud
  auto issue_factor_stage = [&](int f, int b, int first, int cnt) {
    const float4 *p0, *p1;
    const float* p2;
    if (cached) { p0 = cache->desc[f].p0; p1 = cache->desc[f].p1; p2 = cache->desc[f].p2; } else { p0 = descs[f].p0; p1 = descs[f].p1; p2 = descs[f].p2; }
    issue_stage<T>(&ws.buf[b], b ? bar1 : bar0, p0, p1, p2, first, cnt);
  };
  // lane 0: start the copy of the first stage of item `it_idx` into buffer `b` (the item itself is re-read at its start)
  auto prefetch_item = [&](int it_idx, int b) {
    const int2 it = __ldg(&items[it_idx]);
    const int n = cached ? cache->desc[it.x].n : descs[it.x].n;
    const int fchunk = cached ? cache->desc[it.x].chunk : descs[it.x].chunk;
    const int cnt = min(min(fchunk, n - it.y), T);
    (void)chunk;
    if (cnt > 0) issue_factor_stage(it.x, b, it.y, cnt);
  };
  // lane 0 (after a __syncwarp): publish the ticket of the previous item's factor; is that factor complete now?
  auto publish = [&](int pf) -> int {
    const unsigned t = ticket_release(&done[pf]);
    const int last = (t == (unsigned)tiles_of(pf) - 1u);
    if (last) done[pf] = 0u;  // self-cleaning: nobody draws this ticket again in this launch
    return last;
  };

  int cur = 0;                   // stage buffer of the next stage to be processed
  uint32_t par0 = 0, par1 = 0;   // mbarrier phase parities
  if (lane == 0) prefetch_item(item, 0);
  int pend_f = -1;               // factor of the previous item: its ticket has not been published yet
  int pend_last = 0;             // (lane 0) the previous item turned out to be its factor's last

  while (true) {
    int nxt2 = 0x7fffffff;
    if (dynamic && lane == 0) nxt2 = (int)(atomicAdd(item_ctr, 1ull) - ctr_base) + total_warps;  // consumed at the end of the item
    const int2 it = __ldg(&items[item]);
    const int f = it.x;
    // only what the lookup / derivative phases need stays in registers; the plane pointers are re-read by lane 0 when it
    // issues a copy
    const FactorDesc D = desc_of(f);
    PoseF P;
    if (cached) P = cache->pose[f]; else P = pose_from_colmajor(poses + (size_t)f * 16);
    PoseF Pe = P;
    if (MODE == GB_MODE_ERROR) { if (cached) Pe = cache->pose_eval[f]; else Pe = pose_from_colmajor(poses_eval + (size_t)f * 16); }
    const int item_end = min(it.y + D.chunk, D.n);
    const int nstages = (max(0, item_end - it.y) + T - 1) / T;  // 0: factor without points (its epilogue still runs)

    float acc[32];
#pragma unroll
    for (int k = 0; k < 32; k++) acc[k] = 0.f;
    int nq = 0;  // warp-uniform queue length (carried hits first)
    bool published = (pend_f < 0);

    if (nstages == 0 && lane == 0 && nxt < num_items) prefetch_item(nxt, cur);
    for (int s = 0; s < nstages; s++) {
      const int wb = it.y + s * T;
      const int cnt = min(T, item_end - wb);
      const bool last_stage = (s == nstages - 1);
      // ---- keep the copy engine one stage ahead ----
      if (lane == 0) {
        if (!last_stage) issue_factor_stage(f, cur ^ 1, wb + T, min(T, item_end - wb - T));
        else if (nxt < num_items) prefetch_item(nxt, cur ^ 1);
      }
      StageBuf<T>& sb = ws.buf[cur];
      StageBuf<T>& ob = ws.buf[cur ^ 1];
      mbar_wait(cur ? bar1 : bar0, cur ? par1 : par0);
      if (cur) par1 ^= 1u; else par0 ^= 1u;

      // ---------------- phase A: lookup + compaction ----------------
      {
        int cx[U], cy[U], cz[U];
        uint32_t h[U];
        int4 b[U], b1[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          if (u * 32 < cnt) {  // warp-uniform: rows beyond the stage's points are skipped
            const float4 a0 = sb.p0[u * 32 + lane];
            float qx, qy, qz;
            transform(P, a0.x, a0.y, a0.z, qx, qy, qz);
            cx[u] = gb_coord(qx, D.inv_res); cy[u] = gb_coord(qy, D.inv_res); cz[u] = gb_coord(qz, D.inv_res);
            h[u] = gb_hash(cx[u], cy[u], cz[u]);
            b[u] = __ldg(&D.buckets[h[u] & D.mask]);
            b1[u] = __ldg(&D.buckets[(h[u] + 1u) & D.mask]);
          }
        }
        // the previous item's ticket: its REDs were issued a stage ago, and the MEMBAR of the release overlaps with the
        // bucket loads above
        if (!published) {
          published = true;
          __syncwarp();
          if (lane == 0) pend_last = publish(pend_f);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          if (u * 32 < cnt) {
            int v = resolve_probe(D, b[u], b1[u], h[u], cx[u], cy[u], cz[u]);
            if (u * 32 + lane >= cnt) v = -1;
            const unsigned m = __ballot_sync(0xffffffffu, v >= 0);
            if (v >= 0) q[nq + __popc(m & lt_mask)] = make_uint2((unsigned)(u * 32 + lane), (unsigned)v);
            nq += __popc(m);
          }
        }
      }
      __syncwarp();

      // ---------------- phase B: derivative pass over full groups of 32 hits ----------------
      // software pipelined: the voxel record of the lane's NEXT hit is in flight while the current one is processed
      const int nproc = last_stage ? nq : (nq & ~31);
      {
        int k = lane;
        uint2 e = make_uint2(0u, 0u);
        float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0, v2 = v0;
        if (k < nproc) {
          e = q[k];
          v0 = __ldg(&D.voxels[3 * (size_t)e.y + 0]); v1 = __ldg(&D.voxels[3 * (size_t)e.y + 1]); v2 = __ldg(&D.voxels[3 * (size_t)e.y + 2]);
        }
#pragma unroll 1
        while (k < nproc) {
          const int kn = k + 32;
          uint2 en = e;
          float4 n0 = v0, n1 = v1, n2 = v2;
          if (kn < nproc) {
            en = q[kn];
            n0 = __ldg(&D.voxels[3 * (size_t)en.y + 0]); n1 = __ldg(&D.voxels[3 * (size_t)en.y + 1]); n2 = __ldg(&D.voxels[3 * (size_t)en.y + 2]);
          }
          accumulate_hit<MODE>(acc, Pe, sb.p0[e.x], sb.p1[e.x], sb.p2[e.x], v0, v1, v2);
          e = en; v0 = n0; v1 = n1; v2 = n2;
          k = kn;
        }
      }
      // ---------------- carry the partial group over to the next stage ----------------
      if (!last_stage) {
        const int rem = nq - nproc;
        uint2 e = make_uint2(0u, 0u);
        float4 c0 = make_float4(0.f, 0.f, 0.f, 0.f), c1 = c0;
        float c2 = 0.f;
        if (lane < rem) {
          e = q[nproc + lane];
          c0 = sb.p0[e.x]; c1 = sb.p1[e.x]; c2 = sb.p2[e.x];
        }
        __syncwarp();
        if (lane < rem) {
          ob.p0[T + lane] = c0; ob.p1[T + lane] = c1; ob.p2[T + lane] = c2;
          q[lane] = make_uint2((unsigned)(T + lane), e.y);
        }
        nq = rem;
      }
      __syncwarp();  // every lane is done with this stage buffer and the queue before the next copy / compaction
      cur ^= 1;
    }
    if (!published) {  // item without a lookup phase (empty factor)
      __syncwarp();
      if (lane == 0) pend_last = publish(pend_f);
    }

    // ---------------- item reduction: warp -> 29 fp64 reductions ----------------
    double* __restrict__ my_acc = accum + ((size_t)f * acc_slots + (size_t)(item & (acc_slots - 1))) * GB_ACC_STRIDE;
    if (MODE == GB_MODE_LINEARIZE) {
      const float r = warp_reduce_scatter32(acc, lane);
      if (lane < 29) atomicAdd(&my_acc[lane], (double)r);
    } else {
      float e = acc[27], n = acc[28];
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) { e += __shfl_xor_sync(0xffffffffu, e, o); n += __shfl_xor_sync(0xffffffffu, n, o); }
      if (lane == 27) atomicAdd(&my_acc[27], (double)e);
      if (lane == 28) atomicAdd(&my_acc[28], (double)n);
    }

    // ---------------- epilogue of the PREVIOUS item's factor, if that item was its last ----------------
    // scratch: the stage buffer that was consumed last (the other one may be receiving the next item's first stage)
    if (pend_f >= 0 && __shfl_sync(0xffffffffu, pend_last, 0)) {
      fence_acquire();
      const FactorDesc Dp = desc_of(pend_f);
      double* scratch = reinterpret_cast<double*>(&ws.buf[cur ^ 1]);
      factor_epilogue(pend_f, Dp, MODE == GB_MODE_ERROR ? poses_eval : poses, accum, acc_slots, out, slab, scratch);
      if (PEER && MODE == GB_MODE_LINEARIZE) pair_push(Dp, out, peer, reinterpret_cast<float*>(scratch + kEpilogueDoubles));
      __syncwarp();
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic writes of the scratch before the next bulk copy into it
    }
    pend_f = f;
    pend_last = 0;

    item = nxt;
    nxt = __shfl_sync(0xffffffffu, nxt2, 0);
    if (item >= num_items) break;
  }

  // ---- drain: publish the last item's ticket ----
  __syncwarp();
  if (lane == 0) pend_last = publish(pend_f);
  if (__shfl_sync(0xffffffffu, pend_last, 0)) {
    fence_acquire();
    const FactorDesc Dp = desc_of(pend_f);
    double* scratch = reinterpret_cast<double*>(&ws.buf[cur ^ 1]);
    factor_epilogue(pend_f, Dp, MODE == GB_MODE_ERROR ? poses_eval : poses, accum, acc_slots, out, slab, scratch);
    if (PEER && MODE == GB_MODE_LINEARIZE) pair_push(Dp, out, peer, reinterpret_cast<float*>(scratch + kEpilogueDoubles));
  }
}

// =============================================================================================
// k_vgicp_sweep3 -- the large-sweep kernel: register-staged loads, contiguous items drawn from a global queue (the atomic
// for the next item is issued at the start of the current one).  An item's completion ticket is published LAZILY: an
// atom.release issued while the next item's first loads are in flight (no __threadfence, i.e. no MEMBAR.SC + L1
// invalidation per item), and a factor's epilogue runs after the next item's reduction.  Measured on the global-mapping
// sweep and its 1/8 shards: faster than a fence + ticket per item.
// Tried and dropped: reading the queue one item ahead in registers (slower: the kernel sits at the 128-register
// cap) and copying the next item's descriptor / pose to shared memory with cp.async during the current item (slower: the
// three dependent L2 round trips between two items are already covered by the other 15 warps of the SM).
// =============================================================================================
constexpr int kSubMax = 512;   // queue capacity per warp (points per round)
constexpr int kLookupUnroll = 4;

template <int MODE, bool PEER, bool SV>
__global__ void __launch_bounds__(kThreads, 2) k_vgicp_sweep3(
  const FactorDesc* __restrict__ descs, const double* __restrict__ poses, const double* __restrict__ poses_eval,
  const int2* __restrict__ items, int num_items, int chunk,
  unsigned long long* __restrict__ item_ctr, unsigned long long ctr_base,
  double* __restrict__ accum, int acc_slots, unsigned* __restrict__ done, double* __restrict__ out, float* __restrict__ slab, const PeerPush* __restrict__ peer) {
  __shared__ __align__(16) uint2 s_q[kWarps][kSubMax];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  uint2* __restrict__ q = s_q[warp];
  (void)chunk;

  // first item: static (warp id); further items (only when there are more items than warps) come from the global queue
  const int total_warps = gridDim.x * kWarps;
  const bool dynamic = num_items > total_warps;
  int item = blockIdx.x * kWarps + warp;
  if (item >= num_items) return;
  int2 it = __ldg(&items[item]);
  int pend_f = -1, pend_last = 0, pend_tiles = 0;
  auto publish = [&]() {  // lane 0, after a __syncwarp: the previous item's ticket
    const unsigned t = ticket_release(&done[pend_f]);
    pend_last = (t == (unsigned)pend_tiles - 1u);
    if (pend_last) done[pend_f] = 0u;  // self-cleaning
  };

  while (true) {
    int next_item = 0x7fffffff;
    if (dynamic && lane == 0) next_item = (int)(atomicAdd(item_ctr, 1ull) - ctr_base) + total_warps;  // latency hidden behind the item
    const int f = it.x;
    const FactorDesc D = descs[f];
    const PoseF P = pose_from_colmajor(poses + (size_t)f * 16);
    PoseF Pe = P;
    if (MODE == GB_MODE_ERROR) Pe = pose_from_colmajor(poses_eval + (size_t)f * 16);
    const int item_end = min(it.y + D.chunk, D.n);  // per-factor item size (the tail of a sweep is tapered)
    bool published = pend_f < 0;
    float acc[32];
#pragma unroll
    for (int k = 0; k < 32; k++) acc[k] = 0.f;

    for (int wb = it.y; wb < item_end; wb += kSubMax) {
      const int we = min(wb + kSubMax, item_end);
      int nq = 0;  // warp-uniform queue length
      for (int i0 = wb; i0 < we; i0 += 32 * kLookupUnroll) {
        int cx[kLookupUnroll], cy[kLookupUnroll], cz[kLookupUnroll];
        uint32_t h[kLookupUnroll];
        int4 b[kLookupUnroll], b1[kLookupUnroll];
#pragma unroll
        for (int u = 0; u < kLookupUnroll; u++) {
          const int i = i0 + u * 32 + lane;
          const float4 a0 = __ldg(&D.p0[min(i, we - 1)]);
          float qx, qy, qz;
          transform(P, a0.x, a0.y, a0.z, qx, qy, qz);
          cx[u] = gb_coord(qx, D.inv_res); cy[u] = gb_coord(qy, D.inv_res); cz[u] = gb_coord(qz, D.inv_res);
          h[u] = gb_hash(cx[u], cy[u], cz[u]);
          b[u] = __ldg(&D.buckets[h[u] & D.mask]);
          b1[u] = __ldg(&D.buckets[(h[u] + 1u) & D.mask]);
        }
        if (!published) {  // the MEMBAR of the release overlaps with the loads above
          published = true;
          __syncwarp();
          if (lane == 0) publish();
        }
#pragma unroll
        for (int u = 0; u < kLookupUnroll; u++) {
          const int i = i0 + u * 32 + lane;
          int v = resolve_probe(D, b[u], b1[u], h[u], cx[u], cy[u], cz[u]);
          if (i >= we) v = -1;
          const unsigned m = __ballot_sync(0xffffffffu, v >= 0);
          if (v >= 0) q[nq + __popc(m & lt_mask)] = make_uint2((unsigned)i, (unsigned)v);
          nq += __popc(m);
        }
      }
      __syncwarp();
#pragma unroll 2
      for (int k = lane; k < nq; k += 32) {
        const uint2 e = q[k];
        const int i = (int)e.x;
        const float4 a0 = __ldg(&D.p0[i]);
        const float4 a1 = __ldg(&D.p1[i]);
        const float a2 = __ldg(&D.p2[i]);
        const float4 v0 = __ldg(&D.voxels[3 * (size_t)e.y + 0]);
        const float4 v1 = __ldg(&D.voxels[3 * (size_t)e.y + 1]);
        const float4 v2 = __ldg(&D.voxels[3 * (size_t)e.y + 2]);
        // surface validation is a compile-time variant here (GLIM enables it for odometry factors only, which run sweep5)
        if (!SV || D.normals == nullptr || surface_ok(P, __ldg(&D.normals[i]), v0.w, v1.x, v1.y, v1.z, v1.w, v2.x)) accumulate_hit<MODE>(acc, Pe, a0, a1, a2, v0, v1, v2);
      }
      __syncwarp();  // the queue is overwritten by the next round
    }
    if (!published) {  // the item had no lookup group (empty factor)
      __syncwarp();
      if (lane == 0) publish();
    }

    double* __restrict__ my_acc = accum + ((size_t)f * acc_slots + (size_t)(item & (acc_slots - 1))) * GB_ACC_STRIDE;
    if (MODE == GB_MODE_LINEARIZE) {
      const float r = warp_reduce_scatter32(acc, lane);
      if (lane < 29) atomicAdd(&my_acc[lane], (double)r);
    } else {
      float e = acc[27], n = acc[28];
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) { e += __shfl_xor_sync(0xffffffffu, e, o); n += __shfl_xor_sync(0xffffffffu, n, o); }
      if (lane == 27) atomicAdd(&my_acc[27], (double)e);
      if (lane == 28) atomicAdd(&my_acc[28], (double)n);
    }
    if (pend_f >= 0 && __shfl_sync(0xffffffffu, pend_last, 0)) {  // the PREVIOUS item completed its factor
      fence_acquire();
      const FactorDesc Dp = descs[pend_f];
      factor_epilogue(pend_f, Dp, MODE == GB_MODE_ERROR ? poses_eval : poses, accum, acc_slots, out, slab, reinterpret_cast<double*>(q));
      if (PEER && MODE == GB_MODE_LINEARIZE) pair_push(Dp, out, peer, reinterpret_cast<float*>(q) + 512);
      __syncwarp();
    }
    pend_f = f; pend_tiles = D.num_tiles; pend_last = 0;
    item = __shfl_sync(0xffffffffu, next_item, 0);
    if (item >= num_items) break;
    it = __ldg(&items[item]);
  }
  __syncwarp();
  if (lane == 0) publish();
  if (__shfl_sync(0xffffffffu, pend_last, 0)) {
    fence_acquire();
    const FactorDesc Dp = descs[pend_f];
    factor_epilogue(pend_f, Dp, MODE == GB_MODE_ERROR ? poses_eval : poses, accum, acc_slots, out, slab, reinterpret_cast<double*>(q));
    if (PEER && MODE == GB_MODE_LINEARIZE) pair_push(Dp, out, peer, reinterpret_cast<float*>(q) + 512);
  }
}

// =============================================================================================
// k_vgicp_sweep5 (default) -- register-staged like v3 (no large shared-memory carve-out: L1 stays big), with the per-item
// latency chain cut and the one-wave regime balanced:
//   * descriptor / fp32-pose cache in shared memory for small factor sets (an odometry graph), one-item look-ahead of the
//     work queue, lazily published release tickets (atom.release: no __threadfence, no L1 flush per item);
//   * software-pipelined lookup (the next group's points are loaded while the current group's buckets are in flight) and
//     software-pipelined derivative pass (the lane's next hit -- 36-byte point + 48-byte voxel record -- is in flight
//     while the current one is processed);
//   * STRIDED items for sweeps of about one item per warp (odometry, single pair): item j of a factor with J items owns
//     the 32-point rows j, j + J, j + 2J, ... of the source cloud, so every item of a factor samples the whole (Morton-
//     ordered) cloud and sees the same inlier rate; the host sizes J per factor from the factor's last inlier fraction
//     (a hit costs ~2.2x a miss).  One wave of equally expensive items instead of a tail of all-inlier items.
// =============================================================================================
template <int MODE, bool PEER, int PIPE>
__global__ void __launch_bounds__(kThreads, 2) k_vgicp_sweep5(
  const FactorDesc* __restrict__ descs, int num_factors, const double* __restrict__ poses, const double* __restrict__ poses_eval,
  const int2* __restrict__ items, int num_items, int chunk, int strided,
  unsigned long long* __restrict__ item_ctr, unsigned long long ctr_base,
  double* __restrict__ accum, int acc_slots, unsigned* __restrict__ done, double* __restrict__ out, float* __restrict__ slab, const PeerPush* __restrict__ peer) {
  __shared__ __align__(16) uint2 s_q[kWarps][kSubMax];
  __shared__ CtaCache cache_s;
  CtaCache* const cache = &cache_s;
  constexpr int U = kLookupUnroll;
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
  auto publish = [&](int pf) -> int {  // lane 0, after a __syncwarp
    const unsigned t = ticket_release(&done[pf]);
    const int last = (t == (unsigned)(cached ? cache->desc[pf].num_tiles : descs[pf].num_tiles) - 1u);
    if (last) done[pf] = 0u;
    return last;
  };

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

    // the item's points: contiguous [it.y, it.y + chunk) or the rows it.y, it.y + J, ... (32 points each) of the cloud
    const int limit = strided ? D.n : min(it.y + D.chunk, D.n);
    (void)chunk;
    const int row_stride = strided ? D.num_tiles * 32 : 32;
    const int first = strided ? it.y * 32 : it.y;
    int ngroups = 0;
    if (first < limit) {
      const int rows = (limit - first + row_stride - 1) / row_stride;  // strided: ceil((R - j) / J); contiguous: ceil(len / 32)
      ngroups = (rows + U - 1) / U;
    }

    float acc[32];
#pragma unroll
    for (int k = 0; k < 32; k++) acc[k] = 0.f;
    bool published = (pend_f < 0);

    for (int g0 = 0; g0 < ngroups; g0 += kGroupsPerRound) {
      const int g1 = min(g0 + kGroupsPerRound, ngroups);
      int nq = 0;  // warp-uniform queue length
      // ---------------- phase A, software pipelined: group g's buckets and group g+1's points are in flight together ----
      float ax[U], ay[U], az[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const int i = first + (g0 * U + u) * row_stride + lane;
        const float4 a0 = __ldg(&D.p0[i < limit ? i : 0]);
        ax[u] = a0.x; ay[u] = a0.y; az[u] = a0.z;
      }
      for (int g = g0; g < g1; g++) {
        int cx[U], cy[U], cz[U];
        uint32_t h[U];
        int4 b[U], b1[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          float qx, qy, qz;
          transform(P, ax[u], ay[u], az[u], qx, qy, qz);
          cx[u] = gb_coord(qx, D.inv_res); cy[u] = gb_coord(qy, D.inv_res); cz[u] = gb_coord(qz, D.inv_res);
          h[u] = gb_hash(cx[u], cy[u], cz[u]);
          b[u] = __ldg(&D.buckets[h[u] & D.mask]);
          b1[u] = __ldg(&D.buckets[(h[u] + 1u) & D.mask]);
        }
        if ((PIPE & 1) && g + 1 < g1) {
#pragma unroll
          for (int u = 0; u < U; u++) {
            const int i = first + ((g + 1) * U + u) * row_stride + lane;
            const float4 a0 = __ldg(&D.p0[i < limit ? i : 0]);
            ax[u] = a0.x; ay[u] = a0.y; az[u] = a0.z;
          }
        }
        if (!published) {  // the previous item's ticket: the MEMBAR of the release overlaps with the loads above
          published = true;
          __syncwarp();
          if (lane == 0) pend_last = publish(pend_f);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          const int i = first + (g * U + u) * row_stride + lane;
          int v = resolve_probe(D, b[u], b1[u], h[u], cx[u], cy[u], cz[u]);
          if (i >= limit) v = -1;
          const unsigned m = __ballot_sync(0xffffffffu, v >= 0);
          if (v >= 0) q[nq + __popc(m & lt_mask)] = make_uint2((unsigned)i, (unsigned)v);
          nq += __popc(m);
        }
        if (!(PIPE & 1) && g + 1 < g1) {  // not pipelined: the next group's points are loaded after this group is resolved
#pragma unroll
          for (int u = 0; u < U; u++) {
            const int i = first + ((g + 1) * U + u) * row_stride + lane;
            const float4 a0 = __ldg(&D.p0[i < limit ? i : 0]);
            ax[u] = a0.x; ay[u] = a0.y; az[u] = a0.z;
          }
        }
      }
      __syncwarp();
      // ---------------- phase B ----------------
      if (!(PIPE & 2)) {
#pragma unroll 2
        for (int k = lane; k < nq; k += 32) {
          const uint2 e = q[k];
          const float4 a0 = __ldg(&D.p0[e.x]);
          const float4 a1 = __ldg(&D.p1[e.x]);
          const float a2 = __ldg(&D.p2[e.x]);
          const float4 v0 = __ldg(&D.voxels[3 * (size_t)e.y + 0]);
          const float4 v1 = __ldg(&D.voxels[3 * (size_t)e.y + 1]);
          const float4 v2 = __ldg(&D.voxels[3 * (size_t)e.y + 2]);
          if (D.normals == nullptr || surface_ok(P, __ldg(&D.normals[e.x]), v0.w, v1.x, v1.y, v1.z, v1.w, v2.x)) accumulate_hit<MODE>(acc, Pe, a0, a1, a2, v0, v1, v2);
        }
      } else {  // software pipelined: the lane's next hit is in flight while the current one is processed
        int k = lane;
        float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, v0 = a0, v1 = a0, v2 = a0;
        float a2 = 0.f;
        unsigned cur_i = 0;
        if (k < nq) {
          const uint2 e = q[k];
          cur_i = e.x;
          a0 = __ldg(&D.p0[e.x]); a1 = __ldg(&D.p1[e.x]); a2 = __ldg(&D.p2[e.x]);
          v0 = __ldg(&D.voxels[3 * (size_t)e.y + 0]); v1 = __ldg(&D.voxels[3 * (size_t)e.y + 1]); v2 = __ldg(&D.voxels[3 * (size_t)e.y + 2]);
        }
#pragma unroll 1
        while (k < nq) {
          const int kn = k + 32;
          float4 na0 = a0, na1 = a1, nv0 = v0, nv1 = v1, nv2 = v2;
          float na2 = a2;
          unsigned next_i = cur_i;
          if (kn < nq) {
            const uint2 e = q[kn];
            next_i = e.x;
            na0 = __ldg(&D.p0[e.x]); na1 = __ldg(&D.p1[e.x]); na2 = __ldg(&D.p2[e.x]);
            nv0 = __ldg(&D.voxels[3 * (size_t)e.y + 0]); nv1 = __ldg(&D.voxels[3 * (size_t)e.y + 1]); nv2 = __ldg(&D.voxels[3 * (size_t)e.y + 2]);
          }
          if (D.normals == nullptr || surface_ok(P, __ldg(&D.normals[cur_i]), v0.w, v1.x, v1.y, v1.z, v1.w, v2.x)) accumulate_hit<MODE>(acc, Pe, a0, a1, a2, v0, v1, v2);
          a0 = na0; a1 = na1; a2 = na2; v0 = nv0; v1 = nv1; v2 = nv2;
          cur_i = next_i;
          k = kn;
        }
      }
      __syncwarp();  // the queue is overwritten by the next round
    }
    if (!published) {  // empty item
      __syncwarp();
      if (lane == 0) pend_last = publish(pend_f);
    }

    double* __restrict__ my_acc = accum + ((size_t)f * acc_slots + (size_t)(item & (acc_slots - 1))) * GB_ACC_STRIDE;
    if (MODE == GB_MODE_LINEARIZE) {
      const float r = warp_reduce_scatter32(acc, lane);
      if (lane < 29) atomicAdd(&my_acc[lane], (double)r);
    } else {
      float e = acc[27], n = acc[28];
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) { e += __shfl_xor_sync(0xffffffffu, e, o); n += __shfl_xor_sync(0xffffffffu, n, o); }
      if (lane == 27) atomicAdd(&my_acc[27], (double)e);
      if (lane == 28) atomicAdd(&my_acc[28], (double)n);
    }
    // epilogue of the PREVIOUS item's factor, if that item was its last
    if (pend_f >= 0 && __shfl_sync(0xffffffffu, pend_last, 0)) {
      fence_acquire();
      const FactorDesc Dp = desc_of(pend_f);
      factor_epilogue(pend_f, Dp, MODE == GB_MODE_ERROR ? poses_eval : poses, accum, acc_slots, out, slab, reinterpret_cast<double*>(q));
      if (PEER && MODE == GB_MODE_LINEARIZE) pair_push(Dp, out, peer, reinterpret_cast<float*>(q) + 2 * kEpilogueDoubles);
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
  if (lane == 0) pend_last = publish(pend_f);
  if (__shfl_sync(0xffffffffu, pend_last, 0)) {
    fence_acquire();
    const FactorDesc Dp = desc_of(pend_f);
    factor_epilogue(pend_f, Dp, MODE == GB_MODE_ERROR ? poses_eval : poses, accum, acc_slots, out, slab, reinterpret_cast<double*>(q));
    if (PEER && MODE == GB_MODE_LINEARIZE) pair_push(Dp, out, peer, reinterpret_cast<float*>(q) + 2 * kEpilogueDoubles);
  }
}

// overlap: one thread per source point, count points that hit an occupied voxel of any target
__global__ void __launch_bounds__(256) k_overlap(int num_targets, const FactorDesc* __restrict__ descs, const double* __restrict__ poses, int n, int* __restrict__ count) {
  extern __shared__ float s_poses[];  // num_targets x 12
  for (int k = threadIdx.x; k < num_targets * 12; k += blockDim.x) {
    const int t = k / 12, e = k % 12;
    const int r = e < 9 ? e / 3 : e - 9, c = e < 9 ? e % 3 : 3;
    s_poses[k] = (float)poses[(size_t)t * 16 + c * 4 + r];
  }
  __syncthreads();
  int local = 0;
  const FactorDesc D0 = descs[0];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 a0 = __ldg(&D0.p0[i]);
    for (int t = 0; t < num_targets; t++) {
      const PoseF P = load_pose(s_poses + 12 * t);
      float qx, qy, qz;
      transform(P, a0.x, a0.y, a0.z, qx, qy, qz);
      const float sum = (qx + qy) + qz;
      if (!(sum == sum)) continue;  // NaN point: no voxel
      const float inv_res = descs[t].inv_res;
      const int v = gb_lookup(descs[t].buckets, descs[t].mask, descs[t].max_scan, gb_coord(qx, inv_res), gb_coord(qy, inv_res), gb_coord(qz, inv_res));
      if (v >= 0) { local++; break; }
    }
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0 && local) atomicAdd(count, local);
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------
template <int T>
static constexpr size_t sweep4_smem_bytes() { return sizeof(WarpSmem<T>) * kWarps + sizeof(CtaCache); }

size_t gb_sweep4_smem_bytes(int stage_points) { return stage_points == 64 ? sweep4_smem_bytes<64>() : sweep4_smem_bytes<128>(); }

template <int MODE, int T, bool PEER, int MINB>
static cudaError_t launch4(gb_sweep* s, const double* poses_eval, float* slab, const PeerPush* pp) {
  static bool attr_set[16] = {};  // per device
  auto kern = k_vgicp_sweep4<MODE, T, PEER, MINB>;
  const size_t smem = sweep4_smem_bytes<T>();
  const int dev = s->ctx->device & 15;
  if (!attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr_set[dev] = true;
  }
  kern<<<s->grid, kThreads, smem, s->ctx->stream>>>(s->d_descs, (int)s->F, s->d_poses, poses_eval, s->d_tiles, s->num_tiles, s->tile_size, s->d_tile_ctr, s->ctr_base, s->d_accum, s->acc_slots, s->d_done, s->d_out, slab, pp);
  return cudaGetLastError();
}

template <int MODE, bool PEER, int PIPE>
static cudaError_t launch5(gb_sweep* s, const double* poses_eval, float* slab, const PeerPush* pp) {
  k_vgicp_sweep5<MODE, PEER, PIPE><<<s->grid, kThreads, 0, s->ctx->stream>>>(s->d_descs, (int)s->F, s->d_poses, poses_eval, s->d_tiles, s->num_tiles, s->tile_size, s->strided, s->d_tile_ctr, s->ctr_base, s->d_accum, s->acc_slots, s->d_done, s->d_out, slab, pp);
  return cudaGetLastError();
}

template <int MODE, bool PEER, bool SV>
static cudaError_t launch3(gb_sweep* s, const double* poses_eval, float* slab, const PeerPush* pp) {
  k_vgicp_sweep3<MODE, PEER, SV><<<s->grid, kThreads, 0, s->ctx->stream>>>(s->d_descs, s->d_poses, poses_eval, s->d_tiles, s->num_tiles, s->tile_size, s->d_tile_ctr, s->ctr_base, s->d_accum, s->acc_slots, s->d_done, s->d_out, slab, pp);
  return cudaGetLastError();
}

// completion flags of the fused exchange: one thread per rank publishes this rank's step to that peer, then waits for the
// peer's flag.  The preceding sweep kernel has completed (stream order), so all its peer stores have been performed.
struct PeerFlags { unsigned* flags[GB_MAX_PEERS]; };
__global__ void k_peer_signal_wait(PeerFlags pf, int world, int rank, unsigned step, int* timeout) {
  const int t = threadIdx.x;
  if (t >= world) return;
  __threadfence_system();
  volatile unsigned* remote = pf.flags[t] + rank;
  *remote = step;
  __threadfence_system();
  volatile unsigned* mine = pf.flags[rank] + t;
  const long long t0 = clock64();
  while ((int)(*mine - step) < 0) {
    __nanosleep(200);
    if (clock64() - t0 > 4000000000ll) { *timeout = 1; break; }  // ~2 s: a peer died; do not hold the GPU
  }
  __threadfence_system();
}

gb_status gb_launch_sweep(gb_sweep* s, int mode) {
  if (s->num_tiles == 0) return GB_OK;
  gb_ctx* ctx = s->ctx;
  // the table for the buffer of the current step parity (both were written to the device when the slab was attached)
  const bool peer = (mode == GB_MODE_LINEARIZE) && s->peer != nullptr;
  const PeerPush* pp = peer ? s->d_peer_tables + s->peer->parity : nullptr;
  float* slab = mode == GB_MODE_LINEARIZE ? s->d_slab : nullptr;
  const double* pe = mode == GB_MODE_ERROR ? s->d_poses_eval : nullptr;
  cudaError_t e;
  if (s->kernel_version == 3) {
    if (s->any_sv) {
      if (mode == GB_MODE_LINEARIZE) e = peer ? launch3<GB_MODE_LINEARIZE, true, true>(s, pe, slab, pp) : launch3<GB_MODE_LINEARIZE, false, true>(s, pe, slab, pp);
      else e = launch3<GB_MODE_ERROR, false, true>(s, pe, slab, pp);
    } else {
      if (mode == GB_MODE_LINEARIZE) e = peer ? launch3<GB_MODE_LINEARIZE, true, false>(s, pe, slab, pp) : launch3<GB_MODE_LINEARIZE, false, false>(s, pe, slab, pp);
      else e = launch3<GB_MODE_ERROR, false, false>(s, pe, slab, pp);
    }
  } else if (s->kernel_version == 5) {
    if (mode == GB_MODE_ERROR) e = launch5<GB_MODE_ERROR, false, 0>(s, pe, slab, pp);
    else if (peer) e = launch5<GB_MODE_LINEARIZE, true, 0>(s, pe, slab, pp);
    else if (s->pipe == 1) e = launch5<GB_MODE_LINEARIZE, false, 1>(s, pe, slab, pp);
    else if (s->pipe == 2) e = launch5<GB_MODE_LINEARIZE, false, 2>(s, pe, slab, pp);
    else if (s->pipe == 3) e = launch5<GB_MODE_LINEARIZE, false, 3>(s, pe, slab, pp);
    else e = launch5<GB_MODE_LINEARIZE, false, 0>(s, pe, slab, pp);
  } else if (s->stage_points == 64) {
    if (mode == GB_MODE_LINEARIZE) e = peer ? launch4<GB_MODE_LINEARIZE, 64, true, 3>(s, pe, slab, pp) : launch4<GB_MODE_LINEARIZE, 64, false, 3>(s, pe, slab, pp);
    else e = launch4<GB_MODE_ERROR, 64, false, 3>(s, pe, slab, pp);
  } else {
    if (mode == GB_MODE_LINEARIZE) e = peer ? launch4<GB_MODE_LINEARIZE, 128, true, 2>(s, pe, slab, pp) : launch4<GB_MODE_LINEARIZE, 128, false, 2>(s, pe, slab, pp);
    else e = launch4<GB_MODE_ERROR, 128, false, 2>(s, pe, slab, pp);
  }
  if (e != cudaSuccess) { gb_set_error("sweep launch failed: %s", cudaGetErrorString(e)); return GB_ERR_CUDA; }
  // queue bookkeeping: a sweep with more items than warps draws one ticket per processed item, plus (v4, v5) one per warp for
  // the one-item look-ahead
  const unsigned long long warps = (unsigned long long)s->grid * kWarps;
  if ((unsigned long long)s->num_tiles > warps) s->ctr_base += (s->kernel_version == 3 ? 0ull : warps) + (unsigned long long)s->num_tiles;
  ctx->launches++;
  return GB_OK;
}

// Deferred exchange: the four CTAs of peer p copy this rank's finished rows (written by the sweep into the local buffer of the step
// parity) into peer p's buffer -- 128-bit stores through the IPC mapping, ~164 KB per peer at 8 ranks -- then publishes this
// rank's step to that peer and waits for the peer's flag.  The CTAs are independent (one per peer): no ordering between them.
// Why not from the sweep's epilogue (GB_PEER_PUSH=fused, the round-1 design): stores to peer memory issued from all the busy
// SMs slow the sweep down at 8 ranks (against the same shard without the peer stores) while the whole exchange is ~1 MB per rank
// and step.
struct PeerExchange {
  float* dst[GB_MAX_PEERS];   // every rank's buffer of the step parity, as mapped here
  unsigned* flags[GB_MAX_PEERS];
  const float* src;           // this rank's buffer of the step parity
  const int* my_pairs;
  int num_my_pairs;
  unsigned* arrivals;         // [world] CTA arrival counters (self-cleaning)
};
constexpr int kExchangeCtasPerPeer = 4;
constexpr int kExchangeThreads = 512;
__global__ void __launch_bounds__(kExchangeThreads) k_peer_exchange(PeerExchange px, int world, int rank, unsigned step, int* timeout) {
  const int p = blockIdx.x / kExchangeCtasPerPeer, c = blockIdx.x % kExchangeCtasPerPeer;
  if (p != rank) {
    float4* __restrict__ dst = reinterpret_cast<float4*>(px.dst[p]);
    const float4* __restrict__ src = reinterpret_cast<const float4*>(px.src);
    constexpr int kVec = GB_SLAB_STRIDE / 4;
    const int total = px.num_my_pairs * kVec;
    const int stride = kExchangeCtasPerPeer * kExchangeThreads;
    // four independent 16-byte loads in flight per thread: the copy is latency-, not bandwidth-bound (~1 MB per rank and step)
    for (int e0 = c * kExchangeThreads + threadIdx.x; e0 < total; e0 += 4 * stride) {
      float4 v[4];
      size_t at[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int e = min(e0 + u * stride, total - 1);
        at[u] = (size_t)px.my_pairs[e / kVec] * kVec + (size_t)(e % kVec);
        v[u] = __ldcg(&src[at[u]]);
      }
#pragma unroll
      for (int u = 0; u < 4; u++)
        if (e0 + u * stride < total) dst[at[u]] = v[u];
    }
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x != 0) return;
  // the last of this peer's CTAs publishes the flag and waits for the peer's
  const unsigned arrived = atomicAdd(&px.arrivals[p], 1u);
  if (arrived != (unsigned)kExchangeCtasPerPeer - 1u) return;
  px.arrivals[p] = 0u;
  __threadfence_system();
  volatile unsigned* remote = px.flags[p] + rank;
  *remote = step;
  volatile unsigned* mine = px.flags[rank] + p;
  const long long t0 = clock64();
  while ((int)(*mine - step) < 0) {
    __nanosleep(100);
    if (clock64() - t0 > 4000000000ll) { *timeout = 1; break; }  // ~2 s: a peer died; do not hold the GPU
  }
  __threadfence_system();
}

gb_status gb_launch_peer_signal_wait(gb_peer_slab* ps) {
  if (ps->deferred) {
    PeerExchange px;
    memset(&px, 0, sizeof(px));
    for (int p = 0; p < ps->world; p++) {
      px.dst[p] = reinterpret_cast<float*>(ps->peer[p]) + (size_t)ps->parity * ps->buf_floats;
      px.flags[p] = reinterpret_cast<unsigned*>(ps->peer[p] + 2 * ps->buf_floats * sizeof(float));
    }
    px.src = reinterpret_cast<const float*>(ps->local) + (size_t)ps->parity * ps->buf_floats;
    px.my_pairs = ps->d_my_pairs;
    px.num_my_pairs = ps->num_my_pairs;
    px.arrivals = reinterpret_cast<unsigned*>(ps->d_timeout) + 16;  // zeroed at creation, self-cleaning
    k_peer_exchange<<<ps->world * kExchangeCtasPerPeer, kExchangeThreads, 0, ps->ctx->stream>>>(px, ps->world, ps->rank, ps->step, ps->d_timeout);
    GB_CUDA(cudaGetLastError());
    ps->ctx->launches++;
    return GB_OK;
  }
  PeerFlags pf;
  memset(&pf, 0, sizeof(pf));
  for (int p = 0; p < ps->world; p++) pf.flags[p] = reinterpret_cast<unsigned*>(ps->peer[p] + 2 * ps->buf_floats * sizeof(float));
  k_peer_signal_wait<<<1, 32, 0, ps->ctx->stream>>>(pf, ps->world, ps->rank, ps->step, ps->d_timeout);
  GB_CUDA(cudaGetLastError());
  ps->ctx->launches++;
  return GB_OK;
}

gb_status gb_launch_overlap(gb_ctx* ctx, int num_targets, const FactorDesc* d_descs, const double* d_poses, int n, int* d_count) {
  if (n <= 0 || num_targets <= 0) return GB_OK;
  const int grid = min((n + 255) / 256, ctx->num_sms * 8);
  k_overlap<<<grid, 256, (size_t)num_targets * 12 * sizeof(float), ctx->stream>>>(num_targets, d_descs, d_poses, n, d_count);
  GB_CUDA(cudaGetLastError());
  ctx->launches++;
  return GB_OK;
}
