// gb_sweep_steps.cuh -- the steps of the fused sweep kernels, written once: phase A's probe, phase B's accumulation, the item
// reduction, the tickets and the fp64 epilogue (see gb_kernels_vgicp.cu).  Included by gb_kernels_vgicp.cu (k_vgicp_sweep3 / 5)
// and gb_kernels_gicp.cu (k_gicp_sweep): each translation unit compiles its own copy.
#pragma once
#include "gb_internal.cuh"
#include "gb_vgicp_math.cuh"

namespace {

static_assert(GB_MODE_LINEARIZE == GB_MODE_LINEARIZE_VALUE, "gb_vgicp_math.cuh mirrors the mode constant");
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// A point's hash probe in flight: its voxel coordinates, hash and the last bucket gathered for it.
struct Probe {
  int cx, cy, cz;
  uint32_t h;
  int4 b;
};

__device__ __forceinline__ bool bucket_holds(const int4 b, const Probe& p) { return b.w >= 0 && b.x == p.cx && b.y == p.cy && b.z == p.cz; }

// phase A of sweep5 and the GICP sweeps, issue: transform one source point and gather its first bucket.  The second bucket is gathered by probe_resolve,
// only for the lanes whose first bucket holds another voxel: 12-35 % of the points of the global-mapping sweep, by level and
// pair kind (scripts/probe_stats.py), so gathering it up front for every point wasted a 16-byte gather on most of them.
__device__ __forceinline__ void probe_issue(const FactorDesc& D, const PoseF& P, float ax, float ay, float az, Probe& p) {
  float qx, qy, qz;
  transform(P, ax, ay, az, qx, qy, qz);
  p.cx = gb_coord(qx, D.inv_res); p.cy = gb_coord(qy, D.inv_res); p.cz = gb_coord(qz, D.inv_res);
  p.h = gb_hash(p.cx, p.cy, p.cz);
  p.b = __ldg(&D.buckets[p.h & D.mask]);
}

// phase A, resolve: the voxel index of each probe of a group (as gb_lookup: -1 for a miss), from the first buckets issued by
// probe_issue.  The lanes whose first bucket holds another voxel gather their second bucket in ONE predicated round for the
// whole group, so a group waits for at most one more round trip; inactive lanes issue no wavefronts.  Chains longer than two
// buckets are walked one bucket at a time (rare: tables are at most 1/8 full).
template <int U>
__device__ __forceinline__ void probe_resolve(const FactorDesc& D, Probe (&p)[U], int (&v)[U]) {
  bool next[U];
#pragma unroll
  for (int u = 0; u < U; u++) {
    v[u] = bucket_holds(p[u].b, p[u]) ? p[u].b.w : -1;
    next[u] = p[u].b.w >= 0 && v[u] < 0 && D.max_scan > 1;
  }
#pragma unroll
  for (int u = 0; u < U; u++)
    if (next[u]) p[u].b = __ldg(&D.buckets[(p[u].h + 1u) & D.mask]);
#pragma unroll
  for (int u = 0; u < U; u++) {
    if (next[u] && p[u].b.w >= 0) {
      if (bucket_holds(p[u].b, p[u])) {
        v[u] = p[u].b.w;
      } else {
        for (int k = 2; k < D.max_scan; k++) {  // rare: longer collision chain
          const int4 bb = __ldg(&D.buckets[(p[u].h + (uint32_t)k) & D.mask]);
          if (bb.w < 0) break;
          if (bucket_holds(bb, p[u])) { v[u] = bb.w; break; }
        }
      }
    }
  }
}

// sweep3's probe in flight: the key (the bits of key << 1 as two words: pi_key), the home set and the set gathered for it.
struct IndexProbe {
  uint32_t lo, hi, s;
  uint4 e;
};

// phase A of sweep3, issue: transform one source point and gather its home set of the target's probe index
// (gb_probe_index.cuh).  A point outside the target's box gathers nothing: it is a miss (hi = 0 matches no empty entry).
__device__ __forceinline__ void probe_issue(const FactorDesc& D, const IndexDesc& I, const PoseF& P, float ax, float ay, float az, IndexProbe& p) {
  float qx, qy, qz;
  transform(P, ax, ay, az, qx, qy, qz);
  const int cx = gb_coord(qx, D.inv_res), cy = gb_coord(qy, D.inv_res), cz = gb_coord(qz, D.inv_res);
  const bool in = pi_key(I.box, cx, cy, cz, p.lo, p.hi);
  p.s = pi_home(cx, cy, cz) & I.set_mask;
  constexpr uint32_t lo = (uint32_t)kPiEmpty, hi = (uint32_t)(kPiEmpty >> 32);
  p.e = make_uint4(lo, hi, lo, hi);
  if (in) p.e = __ldg(&I.sets[p.s]);
  else p.hi = 0u;
}

// phase A of sweep3, resolve: the voxel index of each probe of a group, as gb_lookup gives it.  A key absent from its home set
// is a miss unless the set's overflow bit is set; those few probes walk the following sets after the whole group is compared.
template <int U>
__device__ __forceinline__ void probe_resolve(const IndexDesc& I, IndexProbe (&p)[U], int (&v)[U]) {
#pragma unroll
  for (int u = 0; u < U; u++) v[u] = pi_match_set(p[u].e, p[u].lo, p[u].hi);
#pragma unroll
  for (int u = 0; u < U; u++)
    if (v[u] < 0 && (p[u].e.x & 1u)) v[u] = pi_walk(I.sets, I.set_mask, p[u].s, p[u].lo, p[u].hi);
}

// phase A, compaction: a hit v >= 0 of point i (none when i >= limit) is appended to the warp's queue as (point, voxel), in
// lane order.  nq: the warp-uniform queue length.
__device__ __forceinline__ void probe_compact(int v, int i, int limit, uint2* __restrict__ q, int& nq, unsigned lt_mask) {
  if (i >= limit) v = -1;
  const unsigned m = __ballot_sync(0xffffffffu, v >= 0);
  if (v >= 0) q[nq + __popc(m & lt_mask)] = make_uint2((unsigned)i, (unsigned)v);
  nq += __popc(m);
}

// sweep3's queue entry: one word, the point's offset within its item (< 2048: 11 bits) above the voxel index (21 bits).
// gb_sweep_create runs a sweep on sweep3 only when every voxel index of its targets is below 2^21.
constexpr int kQueueVoxelBits = 21;
constexpr unsigned kQueueVoxelMask = (1u << kQueueVoxelBits) - 1u;

// phase A, compaction (sweep3): as probe_compact, queueing offset i - base
__device__ __forceinline__ void probe_compact(int v, int i, int limit, int base, unsigned* __restrict__ q, int& nq, unsigned lt_mask) {
  if (i >= limit) v = -1;
  const unsigned m = __ballot_sync(0xffffffffu, v >= 0);
  if (v >= 0) q[nq + __popc(m & lt_mask)] = ((unsigned)(i - base) << kQueueVoxelBits) | (unsigned)v;
  nq += __popc(m);
}

// a queue entry -> (point, voxel): a (point, voxel) pair as it is, or sweep3's word, whose point is base + its offset
__device__ __forceinline__ uint2 queue_hit(const uint2 e, int) { return e; }
__device__ __forceinline__ uint2 queue_hit(const unsigned e, int base) { return make_uint2((unsigned)base + (e >> kQueueVoxelBits), e & kQueueVoxelMask); }

// One stage of warp_reduce_scatter32: lanes STEP apart swap halves of v[0, 2 STEP) and keep the sums in v[0, STEP).
// STEP is a template argument so that every v[] index is a compile-time constant: with a runtime step the inner loop is not
// unrolled and acc[32] lives on the stack (an LDL -> SHFL -> STL chain per item and the stack copy zeroed at every item start).
template <int STEP>
__device__ __forceinline__ void reduce_scatter_stage(float (&v)[32], int lane) {
  const bool upper = (lane & STEP) != 0;
#pragma unroll
  for (int j = 0; j < STEP; j++) {
    const float send = upper ? v[j] : v[j + STEP];
    const float keep = upper ? v[j + STEP] : v[j];
    v[j] = keep + __shfl_xor_sync(0xffffffffu, send, STEP);
  }
}

// Transposing warp reduction: on return lane l holds sum over the warp of v[l] (in v[0]).
__device__ __forceinline__ float warp_reduce_scatter32(float (&v)[32], int lane) {
  reduce_scatter_stage<16>(v, lane);
  reduce_scatter_stage<8>(v, lane);
  reduce_scatter_stage<4>(v, lane);
  reduce_scatter_stage<2>(v, lane);
  reduce_scatter_stage<1>(v, lane);
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
constexpr int kPairRowOffset = 2 * kEpilogueDoubles;  // floats: pair_push's row follows the epilogue's scratch in the warp's queue
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

// phase B: the lanes walk the nq queued hits, so the warp stays full whatever the inlier rate.  SV = false compiles the
// surface validation out (no factor of the sweep has it on).  QE: the queue's entry type (queue_hit); base: sweep3's item start.
template <int MODE, bool SV, class QE>
__device__ __forceinline__ void accumulate_queue(float (&acc)[32], const FactorDesc& D, const PoseF& P, const PoseF& Pe, const QE* __restrict__ q, int nq, int lane, int base = 0) {
#pragma unroll 2
  for (int k = lane; k < nq; k += 32) {
    const uint2 e = queue_hit(q[k], base);
    const int i = (int)e.x;
    const float4 a0 = __ldg(&D.p0[i]);
    const float4 a1 = __ldg(&D.p1[i]);
    const float a2 = __ldg(&D.p2[i]);
    const float4 v0 = __ldg(&D.voxels[3 * (size_t)e.y + 0]);
    const float4 v1 = __ldg(&D.voxels[3 * (size_t)e.y + 1]);
    const float4 v2 = __ldg(&D.voxels[3 * (size_t)e.y + 2]);
    if (!SV || D.normals == nullptr || surface_ok(P, __ldg(&D.normals[i]), v0.w, v1.x, v1.y, v1.z, v1.w, v2.x)) accumulate_hit<MODE>(acc, Pe, a0, a1, a2, v0, v1, v2);
  }
}

// phase B of an ICP sweep (k_icp_grid_sweep): as accumulate_queue, but a hit reads only the source point's first plane and the
// target record's first float4 (16 + 16 B instead of 36 + 48 B).
template <int MODE>
__device__ __forceinline__ void accumulate_icp_queue(float (&acc)[32], const FactorDesc& D, const PoseF& Pe, const uint2* __restrict__ q, int nq, int lane) {
#pragma unroll 2
  for (int k = lane; k < nq; k += 32) {
    const uint2 e = q[k];
    accumulate_icp_hit<MODE>(acc, Pe, __ldg(&D.p0[e.x]), __ldg(&D.voxels[3 * (size_t)e.y]));
  }
}

// An item's sums into its factor's accumulator copy (item mod acc_slots): all 29 (linearize) or the error and the inlier
// count (error).
template <int MODE>
__device__ __forceinline__ void reduce_item(float (&acc)[32], double* __restrict__ accum, int f, int acc_slots, int item, int lane) {
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
}

// Lane 0, after a __syncwarp: publishes the completion of one of factor f's items.  Returns whether it was the last of the
// factor's num_tiles() items; its drawer re-zeroes the ticket for the next sweep (self-cleaning).  num_tiles() is evaluated
// after the release: sweep5 reads it from its descriptors, and reading it ahead of the release measured slower there.
template <class NumTiles>
__device__ __forceinline__ int ticket_last(unsigned* __restrict__ done, int f, const NumTiles& num_tiles) {
  const unsigned t = ticket_release(&done[f]);
  const int last = (t == (unsigned)num_tiles() - 1u);
  if (last) done[f] = 0u;
  return last;
}

// Retires factor f, by the warp that drew its last ticket: fp64 epilogue, then the pair push when a peer slab is attached.
// The warp's queue q is free at this point and serves as scratch.  The caller issues fence_acquire() and then copies D: a
// copy taken in here lands ahead of acc[] in sweep3's stack frame, which changed its code and measured slower.
template <int MODE, bool PEER>
__device__ __forceinline__ void retire_factor(int f, const FactorDesc& D, const double* __restrict__ poses, const double* __restrict__ poses_eval,
                                              double* __restrict__ accum, int acc_slots, double* __restrict__ out, float* __restrict__ slab, const PeerPush* __restrict__ peer, void* q) {
  factor_epilogue(f, D, MODE == GB_MODE_ERROR ? poses_eval : poses, accum, acc_slots, out, slab, static_cast<double*>(q));
  if (PEER && MODE == GB_MODE_LINEARIZE) pair_push(D, out, peer, static_cast<float*>(q) + kPairRowOffset);
}

}  // namespace
