// gb_kernels_gicp.cu -- the GICP linearize / error sweep on a device iVox (sm_90a).
//
// Replaces IntegratedGICPFactor_<iVox, PointCloud>::linearize / ::error as GLIM's CPU odometry drives it with
// registration_type "GICP" (src/glim/odometry/odometry_estimation_cpu.cpp:95-104).  The rule is written once, in
// include/glim_b200.h (gb_gicp_factor_create); the correspondence search is gb_ivox_math.cuh's (also compiled for the host by
// the CPU test), everything after it is the VGICP sweep's steps (gb_sweep_steps.cuh).
#include "gb_internal.cuh"
#include "gb_sweep_steps.cuh"
#include "gb_ivox_math.cuh"

namespace {

constexpr int kGicpQueue = 512;  // queue capacity per warp (points per round)

// =============================================================================================
// k_gicp_sweep -- GICP factors on a device iVox (gb_gicp_factor_create).  sweep5's strided items and accumulator machinery;
// only the lookup differs: a lane's point is transformed, ivox_nearest finds its nearest stored point, and the hit is queued
// as (point, point record) -- the records have the voxel-record layout, so accumulate_queue reads them as voxels.  The next
// item is drawn after the current one (draws = items, as sweep3's queue); no descriptor cache, no look-ahead.
// =============================================================================================
template <int MODE>
__global__ void __launch_bounds__(kThreads, 2) k_gicp_sweep(
  const FactorDesc* __restrict__ descs, const GicpDesc* __restrict__ gdescs, const double* __restrict__ poses, const double* __restrict__ poses_eval,
  const int2* __restrict__ items, int num_items, unsigned long long* __restrict__ item_ctr, unsigned long long ctr_base,
  double* __restrict__ accum, int acc_slots, unsigned* __restrict__ done, double* __restrict__ out) {
  __shared__ __align__(16) uint2 s_q[kWarps][kGicpQueue];
  constexpr int kRowsPerRound = kGicpQueue / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  uint2* __restrict__ q = s_q[warp];
  const int total_warps = gridDim.x * kWarps;
  const bool dynamic = num_items > total_warps;
  int item = blockIdx.x * kWarps + warp;  // first item: static
  if (item >= num_items) return;
  while (true) {
    const int2 it = __ldg(&items[item]);
    const int f = it.x;
    const FactorDesc D = descs[f];
    const GicpDesc G = gdescs[f];
    const PoseF P = pose_from_colmajor(poses + (size_t)f * 16);
    PoseF Pe = P;
    if (MODE == GB_MODE_ERROR) Pe = pose_from_colmajor(poses_eval + (size_t)f * 16);
    // the item's points: the rows it.y, it.y + J, ... (32 points each) of the cloud, J = the factor's item count
    const int row_stride = D.num_tiles * 32;
    float acc[32];
#pragma unroll
    for (int k = 0; k < 32; k++) acc[k] = 0.f;
    for (int r0 = it.y * 32; r0 < D.n; r0 += kRowsPerRound * row_stride) {
      int nq = 0;  // warp-uniform queue length
      for (int r = 0; r < kRowsPerRound; r++) {
        const int i = r0 + r * row_stride + lane;
        int v = -1;
        if (i < D.n) {
          const float4 a0 = __ldg(&D.p0[i]);
          float qx, qy, qz;
          transform(P, a0.x, a0.y, a0.z, qx, qy, qz);
          v = ivox_nearest(D.buckets, D.mask, D.max_scan, G.cells, D.voxels, G.num_offsets, D.inv_res, G.max_corr2, qx, qy, qz);
        }
        const unsigned m = __ballot_sync(0xffffffffu, v >= 0);
        if (v >= 0) q[nq + __popc(m & lt_mask)] = make_uint2((unsigned)i, (unsigned)v);
        nq += __popc(m);
      }
      __syncwarp();
      accumulate_queue<MODE, false>(acc, D, P, Pe, q, nq, lane);
      __syncwarp();  // the queue is overwritten by the next round
    }
    reduce_item<MODE>(acc, accum, f, acc_slots, item, lane);
    __syncwarp();
    int last = 0;
    if (lane == 0) last = ticket_last(done, f, [&] { return D.num_tiles; });
    if (__shfl_sync(0xffffffffu, last, 0)) {
      fence_acquire();
      retire_factor<MODE, false>(f, D, poses, poses_eval, accum, acc_slots, out, nullptr, nullptr, q);
      __syncwarp();
    }
    if (!dynamic) break;
    int nxt = 0;
    if (lane == 0) nxt = (int)(atomicAdd(item_ctr, 1ull) - ctr_base) + total_warps;
    item = __shfl_sync(0xffffffffu, nxt, 0);
    if (item >= num_items) break;
  }
}

}  // namespace

gb_status gb_launch_gicp_sweep(gb_sweep* s, int mode) {
  if (s->num_tiles == 0) return GB_OK;
  const bool lin = mode == GB_MODE_LINEARIZE;
  GB_CHECK(gb_launch(s->ctx, "k_gicp_sweep", lin ? k_gicp_sweep<GB_MODE_LINEARIZE> : k_gicp_sweep<GB_MODE_ERROR>, s->grid, kThreads, 0, s->d_descs, s->d_gdescs, s->d_poses,
                     lin ? nullptr : s->d_poses_eval, s->d_tiles, s->num_tiles, s->d_tile_ctr, s->ctr_base, s->d_accum, s->acc_slots, s->d_done, s->d_out));
  // one draw per item when there are more items than warps
  if ((unsigned long long)s->num_tiles > (unsigned long long)s->grid * kWarps) s->ctr_base += (unsigned long long)s->num_tiles;
  return GB_OK;
}
