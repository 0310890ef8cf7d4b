// gb_kernels_gicp.cu -- the GICP linearize / error sweeps on a device iVox and on a device point grid (sm_90a).
//
// Replaces IntegratedGICPFactor_<iVox, PointCloud>::linearize / ::error as GLIM's CPU odometry drives it with
// registration_type "GICP" (src/glim/odometry/odometry_estimation_cpu.cpp:95-104), and IntegratedGICPFactor between two whole
// frames with a KdTree over the target (sub_mapping.cpp:189-211, global_mapping.cpp:379-428, global_mapping_pose_graph.cpp:391-405),
// and the point-to-point IntegratedICPFactor of the manual loop closure's fallback (manual_loop_close_modal.cpp:479-492).
// The rules are written once, in include/glim_b200.h (gb_gicp_factor_create, gb_gicp_grid_factor_create, gb_icp_grid_factor_create); the correspondence
// searches are gb_ivox_math.cuh's and gb_grid_math.cuh's (also compiled for the host by the CPU tests), everything after them is
// the VGICP sweep's steps (gb_sweep_steps.cuh).
#include "gb_internal.cuh"
#include "gb_sweep_steps.cuh"
#include "gb_ivox_math.cuh"
#include "gb_grid_math.cuh"

namespace {

constexpr int kGicpQueue = 512;  // queue capacity per warp (points per round)

// =============================================================================================
// The GICP sweeps -- GICP factors on a device iVox (k_gicp_sweep, gb_gicp_factor_create) or on a device point grid
// (k_gicp_grid_sweep, gb_gicp_grid_factor_create).  sweep5's strided items and accumulator machinery; only the lookup differs:
// a lane's point is transformed, the kind's search (ivox_nearest, grid_nearest) finds its nearest stored point, and the hit is
// queued as (point, point record) -- the records have the voxel-record layout, so accumulate_queue reads them as voxels.  The
// next item is drawn after the current one (draws = items, as sweep3's queue); no descriptor cache, no look-ahead.
// =============================================================================================
template <int MODE, bool ICP, class Nearest>
__device__ __forceinline__ void gicp_sweep(
  uint2 (*s_q)[kGicpQueue], const FactorDesc* __restrict__ descs, const GicpDesc* __restrict__ gdescs, const double* __restrict__ poses, const double* __restrict__ poses_eval,
  const int2* __restrict__ items, int num_items, unsigned long long* __restrict__ item_ctr, unsigned long long ctr_base,
  double* __restrict__ accum, int acc_slots, unsigned* __restrict__ done, double* __restrict__ out, const Nearest& nearest) {
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
          v = nearest(D, G, qx, qy, qz);
        }
        const unsigned m = __ballot_sync(0xffffffffu, v >= 0);
        if (v >= 0) q[nq + __popc(m & lt_mask)] = make_uint2((unsigned)i, (unsigned)v);
        nq += __popc(m);
      }
      __syncwarp();
      if (ICP) accumulate_icp_queue<MODE>(acc, D, Pe, q, nq, lane);
      else accumulate_queue<MODE, false>(acc, D, P, Pe, q, nq, lane);
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

// iVox: the mode's neighbour voxels (FactorDesc: the iVox's table and point records; GicpDesc: cells, bound, mode)
template <int MODE>
__global__ void __launch_bounds__(kThreads, 2) k_gicp_sweep(
  const FactorDesc* __restrict__ descs, const GicpDesc* __restrict__ gdescs, const double* __restrict__ poses, const double* __restrict__ poses_eval,
  const int2* __restrict__ items, int num_items, unsigned long long* __restrict__ item_ctr, unsigned long long ctr_base,
  double* __restrict__ accum, int acc_slots, unsigned* __restrict__ done, double* __restrict__ out) {
  __shared__ __align__(16) uint2 s_q[kWarps][kGicpQueue];
  gicp_sweep<MODE, false>(s_q, descs, gdescs, poses, poses_eval, items, num_items, item_ctr, ctr_base, accum, acc_slots, done, out,
                   [](const FactorDesc& D, const GicpDesc& G, float qx, float qy, float qz) {
                     return ivox_nearest(D.buckets, D.mask, D.max_scan, G.cells, D.voxels, G.num_offsets, D.inv_res, G.max_corr2, qx, qy, qz);
                   });
}

// Point grid: the cells within the search half-width m (FactorDesc: the grid's table and point records; GicpDesc: cells,
// bound, m in num_offsets)
template <int MODE>
__global__ void __launch_bounds__(kThreads, 2) k_gicp_grid_sweep(
  const FactorDesc* __restrict__ descs, const GicpDesc* __restrict__ gdescs, const double* __restrict__ poses, const double* __restrict__ poses_eval,
  const int2* __restrict__ items, int num_items, unsigned long long* __restrict__ item_ctr, unsigned long long ctr_base,
  double* __restrict__ accum, int acc_slots, unsigned* __restrict__ done, double* __restrict__ out) {
  __shared__ __align__(16) uint2 s_q[kWarps][kGicpQueue];
  gicp_sweep<MODE, false>(s_q, descs, gdescs, poses, poses_eval, items, num_items, item_ctr, ctr_base, accum, acc_slots, done, out,
                   [](const FactorDesc& D, const GicpDesc& G, float qx, float qy, float qz) {
                     return grid_nearest(D.buckets, D.mask, D.max_scan, G.cells, D.voxels, G.num_offsets, D.inv_res, G.max_corr2, qx, qy, qz);
                   });
}

// Point-to-point ICP on a point grid: k_gicp_grid_sweep's search, the ICP accumulation (accumulate_icp_queue)
template <int MODE>
__global__ void __launch_bounds__(kThreads, 2) k_icp_grid_sweep(
  const FactorDesc* __restrict__ descs, const GicpDesc* __restrict__ gdescs, const double* __restrict__ poses, const double* __restrict__ poses_eval,
  const int2* __restrict__ items, int num_items, unsigned long long* __restrict__ item_ctr, unsigned long long ctr_base,
  double* __restrict__ accum, int acc_slots, unsigned* __restrict__ done, double* __restrict__ out) {
  __shared__ __align__(16) uint2 s_q[kWarps][kGicpQueue];
  gicp_sweep<MODE, true>(s_q, descs, gdescs, poses, poses_eval, items, num_items, item_ctr, ctr_base, accum, acc_slots, done, out,
                         [](const FactorDesc& D, const GicpDesc& G, float qx, float qy, float qz) {
                           return grid_nearest(D.buckets, D.mask, D.max_scan, G.cells, D.voxels, G.num_offsets, D.inv_res, G.max_corr2, qx, qy, qz);
                         });
}

}  // namespace

gb_status gb_launch_gicp_sweep(gb_sweep* s, int mode) {
  if (s->num_tiles == 0) return GB_OK;
  const bool lin = mode == GB_MODE_LINEARIZE;
  const auto kernel = s->icp          ? (lin ? k_icp_grid_sweep<GB_MODE_LINEARIZE> : k_icp_grid_sweep<GB_MODE_ERROR>)
                      : s->point_grid ? (lin ? k_gicp_grid_sweep<GB_MODE_LINEARIZE> : k_gicp_grid_sweep<GB_MODE_ERROR>)
                                      : (lin ? k_gicp_sweep<GB_MODE_LINEARIZE> : k_gicp_sweep<GB_MODE_ERROR>);
  GB_CHECK(gb_launch(s->ctx, s->icp ? "k_icp_grid_sweep" : (s->point_grid ? "k_gicp_grid_sweep" : "k_gicp_sweep"), kernel, s->grid, kThreads, 0, s->d_descs, s->d_gdescs, s->d_poses,
                     lin ? nullptr : s->d_poses_eval, s->d_tiles, s->num_tiles, s->d_tile_ctr, s->ctr_base, s->d_accum, s->acc_slots, s->d_done, s->d_out));
  // one draw per item when there are more items than warps
  if ((unsigned long long)s->num_tiles > (unsigned long long)s->grid * kWarps) s->ctr_base += (unsigned long long)s->num_tiles;
  return GB_OK;
}
