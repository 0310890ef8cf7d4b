// gb_kernels_ct.cu -- continuous-time GICP on a device iVox (sm_90a): the time table of a cloud (gb_cloud_add_times), the CT
// factor (gb_ct_gicp_factor_create / _linearize / _error), the per-frame Levenberg-Marquardt solve (gb_ct_gicp_align) and the
// deskewed frame (gb_ct_deskew).
//
// Replaces IntegratedCT_GICPFactor_<iVox, PointCloud> and the LevenbergMarquardtOptimizerExt loop around it in GLIM's
// LiDAR-only odometry (src/glim/odometry/odometry_estimation_ct.cpp:100-182).  The rule is written once, in include/glim_b200.h;
// the per-problem arithmetic lives in gb_ct_math.cuh (also compiled for the host by the CPU test), the correspondence search is
// gb_ivox_math.cuh's and the per-point accumulation the sweeps' (gb_sweep_steps.cuh).
//
// One call covers P problems (one CT factor each).  Its work items are (problem, time-table entry, up to kCtChunk points of the
// entry in original order).  k_ct_sweep gives each item one warp: the entry's pose T_b = X Exp(tau_b Log(X^-1 Y)) in fp64, its
// fp32 cast as the lookup transform, ivox_nearest and the GICP sweep's accumulation; the item's warp-reduced sums go to its own
// slot with plain stores.  ct_reduce (one CTA per problem) then chains the entries' 6x6 blocks to the 12x12 system in fp64, in
// a fixed order: no float atomics, so results are deterministic and a batch equals its problems run alone.
#include "gb_internal.cuh"
#include "gb_sweep_steps.cuh"
#include "gb_ivox_math.cuh"
#include "gb_ct_math.cuh"

#include <math.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <new>

namespace {

constexpr int kCtChunk = 128;       // points per work item
constexpr int kCtThreads = 256;     // ct_reduce: one CTA per problem, 8 warps over its entries
constexpr int kCtSystem = 158;      // H (144, row-major over [X; Y]) | b (12) | error | num_inliers

// The device descriptor of one problem.
struct CtDesc {
  FactorDesc D;             // source planes, the iVox's table and point records
  GicpDesc G;               // cells, correspondence bound, searched offsets
  const int* inv_perm;      // original index -> stored slot (nullptr = identity)
  const double* tau;        // the source's normalized entry times
  const int* entry_items;   // the problem's items of entry b: [entry_items[b], entry_items[b + 1])
  int num_entries;
  int pad;
};

// the pose of entry `tau` for poses XY = X (16) | Y (16)
__device__ __forceinline__ PoseF entry_pose_f(const double* XY, double tau) {
  double xi[6], T[16];
  ct_motion(XY, XY + 16, xi);
  ct_entry_pose(XY, xi, tau, T);
  return pose_from_colmajor(T);
}

// One warp per item: correspondences at the entry pose of XY, residuals at that of XYe (error mode), sums into slot `item`.
template <int MODE>
__global__ void __launch_bounds__(kThreads, 2) k_ct_sweep(const CtDesc* __restrict__ descs, const int4* __restrict__ items, int num_items, const double* __restrict__ XY,
                                                          const double* __restrict__ XYe, double* __restrict__ slots) {
  __shared__ __align__(16) uint2 s_q[kWarps][kCtChunk];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  uint2* __restrict__ q = s_q[warp];
  for (int item = blockIdx.x * kWarps + warp; item < num_items; item += gridDim.x * kWarps) {
    const int4 it = __ldg(&items[item]);  // {problem, entry, first original index, count}
    const FactorDesc D = descs[it.x].D;
    const GicpDesc G = descs[it.x].G;
    const int* __restrict__ inv_perm = descs[it.x].inv_perm;
    const double tau = descs[it.x].tau[it.y];
    const PoseF P = entry_pose_f(XY + (size_t)it.x * 32, tau);
    PoseF Pe = P;
    if (MODE == GB_MODE_ERROR) Pe = entry_pose_f(XYe + (size_t)it.x * 32, tau);
    float acc[32];
#pragma unroll
    for (int k = 0; k < 32; k++) acc[k] = 0.f;
    int nq = 0;  // warp-uniform queue length
    for (int r = 0; r < it.w; r += 32) {
      int i = -1, v = -1;
      if (r + lane < it.w) {
        const int j = it.z + r + lane;
        i = inv_perm ? __ldg(&inv_perm[j]) : j;
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
    double* __restrict__ slot = slots + (size_t)item * GB_ACC_STRIDE;
    if (MODE == GB_MODE_LINEARIZE) {
      const float s = warp_reduce_scatter32(acc, lane);
      if (lane < 29) slot[lane] = (double)s;
    } else {
      float e = acc[27], n = acc[28];
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) { e += __shfl_xor_sync(0xffffffffu, e, o); n += __shfl_xor_sync(0xffffffffu, n, o); }
      if (lane == 0) { slot[27] = (double)e; slot[28] = (double)n; }
    }
    __syncwarp();  // the queue is overwritten by the next item
  }
}

// Per-warp scratch of ct_reduce (doubles).
struct CtWarpScratch {
  double A[32];   // the entry's summed accumulators
  double Ad[36];  // Ad of the fp32-cast entry pose (row-major)
  double M[36];   // H_q Ad
  double Hb[36];  // the entry's H_ss
  double bb[6];   // the entry's b_s
  double J[72];   // [D0 D1], 6 x 12 row-major
  double W[72];   // Hb J
};

// The 12x12 system (MODE == LINEARIZE) or the error and inlier count of problem p, by the whole CTA (kCtThreads), into
// sys[kCtSystem] (shared).  Entry b is handled by warp b % 8, which sums its items' slots in item order, forms the entry's
// H_ss / b_s as factor_epilogue does for the pose T_b and chains them with [D0 D1]; the warps' partial sums are added in
// warp order.
template <int MODE>
__device__ void ct_reduce(const CtDesc& C, const double* X, const double* Y, const double* __restrict__ slots, double* sys) {
  __shared__ CtWarpScratch ws[kCtThreads / 32];
  __shared__ double part[kCtThreads / 32][160];
  __shared__ double prob[6 + 36 + 36];  // xi | J_r^-1(xi) | Ad(Y^-1 X)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (MODE == GB_MODE_LINEARIZE && threadIdx.x == 0) ct_problem_blocks(X, Y, prob, prob + 6, prob + 42);
  __syncthreads();
  CtWarpScratch& s = ws[warp];
  double acc[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int b = warp; b < C.num_entries; b += kCtThreads / 32) {
    const int i0 = C.entry_items[b], i1 = C.entry_items[b + 1];
    if (lane < 29 && (MODE == GB_MODE_LINEARIZE || lane >= 27)) {
      double a = 0.0;
      for (int it = i0; it < i1; it++) a += slots[(size_t)it * GB_ACC_STRIDE + lane];
      s.A[lane] = a;
    }
    if (MODE == GB_MODE_LINEARIZE && lane == 0) {
      const double tau = C.tau[b];
      double T[16], Tc[16], D0[36], D1[36];
      ct_entry_pose(X, prob, tau, T);
      for (int k = 0; k < 16; k++) Tc[k] = (double)(float)T[k];
      ct_adjoint(Tc, s.Ad);  // of the fp32-cast pose the lookup used, as factor_epilogue
      ct_entry_blocks(prob, prob + 6, prob + 42, tau, D0, D1);
      for (int i = 0; i < 6; i++)
        for (int j = 0; j < 6; j++) { s.J[i * 12 + j] = D0[i * 6 + j]; s.J[i * 12 + 6 + j] = D1[i * 6 + j]; }
    }
    __syncwarp();
    if (MODE == GB_MODE_LINEARIZE) {
      auto Hq = [&](int i, int j) -> double {
        const int a = i < j ? i : j, c = i < j ? j : i;
        return s.A[a * 6 - (a * (a - 1)) / 2 + (c - a)];
      };
      for (int e = lane; e < 36; e += 32) {
        const int i = e / 6, j = e % 6;
        double v = 0.0;
        for (int k = 0; k < 6; k++) v += Hq(i, k) * s.Ad[k * 6 + j];
        s.M[e] = v;
      }
      __syncwarp();
      for (int e = lane; e < 36; e += 32) {
        const int i = e / 6, j = e % 6;
        double v = 0.0;
        for (int k = 0; k < 6; k++) v += s.Ad[k * 6 + i] * s.M[k * 6 + j];
        s.Hb[e] = v;
      }
      if (lane < 6) {
        double v = 0.0;
        for (int k = 0; k < 6; k++) v += s.Ad[k * 6 + lane] * s.A[21 + k];
        s.bb[lane] = -v;
      }
      __syncwarp();
      for (int e = lane; e < 72; e += 32) {
        const int i = e / 12, j = e % 12;
        double v = 0.0;
        for (int k = 0; k < 6; k++) v += s.Hb[i * 6 + k] * s.J[k * 12 + j];
        s.W[e] = v;
      }
      __syncwarp();
#pragma unroll
      for (int k = 0; k < 5; k++) {
        const int e = lane + 32 * k;
        double v = 0.0;
        if (e < 144) {
          const int i = e / 12, j = e % 12;
          for (int m = 0; m < 6; m++) v += s.J[m * 12 + i] * s.W[m * 12 + j];
        } else if (e < 156) {
          for (int m = 0; m < 6; m++) v += s.J[m * 12 + (e - 144)] * s.bb[m];
        } else if (e == 156) {
          v = s.A[27];
        } else if (e == 157) {
          v = s.A[28];
        }
        acc[k] += v;
      }
    } else {
      if (lane == 28) acc[4] += s.A[27];  // element 156 of the system
      if (lane == 29) acc[4] += s.A[28];  // element 157
    }
    __syncwarp();  // the scratch is overwritten by the warp's next entry
  }
#pragma unroll
  for (int k = 0; k < 5; k++) part[warp][lane + 32 * k] = acc[k];
  __syncthreads();
  for (int e = threadIdx.x; e < kCtSystem; e += blockDim.x) {
    double v = 0.0;
    for (int w = 0; w < kCtThreads / 32; w++) v += part[w][e];
    sys[e] = v;
  }
  __syncthreads();
}

// One CTA per problem: the problem's record (gb_linearized6 with X in the target slot, Y in the source slot), or its error
// and inlier count.
template <int MODE>
__global__ void __launch_bounds__(kCtThreads) k_ct_record(const CtDesc* __restrict__ descs, const double* __restrict__ XY, const double* __restrict__ slots, double* __restrict__ out) {
  __shared__ double sys[kCtSystem];
  const int p = blockIdx.x;
  const double* X = XY + (size_t)p * 32;
  ct_reduce<MODE>(descs[p], X, X + 16, slots, sys);
  double* o = out + (size_t)p * GB_OUT_DOUBLES;
  for (int e = threadIdx.x; e < GB_OUT_DOUBLES; e += blockDim.x) {
    double v;
    if (e < 108) {  // H_tt | H_ss | H_ts, column-major 6x6 blocks
      const int blk = e / 36, c = (e % 36) / 6, r = e % 6;
      const int i = (blk == 1 ? 6 : 0) + r, j = (blk == 0 ? 0 : 6) + c;
      v = sys[i * 12 + j];
    } else {
      v = sys[144 + (e - 108)];  // b_t | b_s | error | num_inliers
    }
    o[e] = MODE == GB_MODE_LINEARIZE || e >= 120 ? v : 0.0;
  }
}

// rule steps 1-2 for every active problem (one CTA each): a fresh linearization into the state, then the trial poses into XYe.
// Block 0 clears the status word.
__global__ void __launch_bounds__(kCtThreads) k_ct_step(CtState* __restrict__ st, const CtDesc* __restrict__ descs, const double* __restrict__ slots, double* __restrict__ XYe,
                                                        double w_prior, double w_between, unsigned* __restrict__ counters) {
  __shared__ double sys[kCtSystem];
  __shared__ int active;
  align_status_clear(counters);
  const int p = blockIdx.x;
  CtState& s = st[p];
  if (s.a.status != GB_ALIGN_ACTIVE) return;
  if (s.a.need_lin) {
    ct_reduce<GB_MODE_LINEARIZE>(descs[p], s.a.T, s.Y, slots, sys);
    if (threadIdx.x == 0) {
      for (int k = 0; k < 144; k++) s.H[k] = sys[k];
      for (int k = 0; k < 12; k++) s.b[k] = sys[144 + k];
      s.a.e = sys[156] + ct_small_terms(s.a.T, s.Y, s.Xp, w_prior, w_between, s.H, s.b);
      s.a.n = sys[157];
      align_linearized(s.a);
      active = s.a.status == GB_ALIGN_ACTIVE;
    }
    __syncthreads();
    if (!active) return;
  }
  if (threadIdx.x == 0) {
    ct_trial(s);
    for (int k = 0; k < 16; k++) { XYe[(size_t)p * 32 + k] = s.a.Tn[k]; XYe[(size_t)p * 32 + 16 + k] = s.Yn[k]; }
  }
}

// rule steps 4-5 for every active problem (one CTA each): the objective at the trial poses with the inliers of the current
// ones, align_conclude, the accepted poses into XY; then count active problems and those that need a linearization.
__global__ void __launch_bounds__(kCtThreads) k_ct_accept(CtState* __restrict__ st, const CtDesc* __restrict__ descs, const double* __restrict__ slots, double* __restrict__ XY,
                                                          gb_align_params prm, double w_prior, double w_between, unsigned* __restrict__ counters) {
  __shared__ double sys[kCtSystem];
  const int p = blockIdx.x;
  CtState& s = st[p];
  if (s.a.status != GB_ALIGN_ACTIVE) return;
  ct_reduce<GB_MODE_ERROR>(descs[p], s.a.Tn, s.Yn, slots, sys);
  if (threadIdx.x == 0) {
    const double e_new = sys[156] + ct_small_terms(s.a.Tn, s.Yn, s.Xp, w_prior, w_between, nullptr, nullptr);
    ct_conclude(s, prm, e_new);
    if (align_status_tally(s.a, counters) & 1)
      for (int k = 0; k < 16; k++) { XY[(size_t)p * 32 + k] = s.a.T[k]; XY[(size_t)p * 32 + 16 + k] = s.Y[k]; }
  }
}

// gb_ct_deskew's points: one thread per stored slot j of the source; its entry b (the last with starts[b] <= its original
// index), Exp(tau_b xi) p in fp64 from the fp32 position, written at the original index.  Thread 0 writes the point count the
// covariance stage reads.
__global__ void k_ct_deskew(int n, const float4* __restrict__ p0, const int* __restrict__ perm, const int* __restrict__ starts, const double* __restrict__ tau, int B,
                            const double* __restrict__ XY, double4* __restrict__ out, int* __restrict__ count) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j == 0) *count = n;
  if (j >= n) return;
  const int i = perm ? perm[j] : j;
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (starts[mid] <= i) lo = mid; else hi = mid - 1;
  }
  double xi[6], E[16];
  ct_motion(XY, XY + 16, xi);
  for (int k = 0; k < 6; k++) xi[k] *= tau[lo];
  ct_exp(xi, E);
  const float4 a = p0[j];
  const double x = a.x, y = a.y, z = a.z;
  out[i] = make_double4(E[0] * x + E[4] * y + E[8] * z + E[12], E[1] * x + E[5] * y + E[9] * z + E[13], E[2] * x + E[6] * y + E[10] * z + E[14], 1.0);
}

// The device block of a cloud's time table: starts (B + 1) | tau (B).
struct CtTable { int* starts; double* tau; };
CtTable ct_table_layout(Carver& cv, int B) {
  CtTable t;
  t.starts = cv.take<int>((size_t)B + 1);
  t.tau = cv.take<double>((size_t)B);
  return t;
}

// The per-call block of P problems, the same layout in scratch and in pinned staging (the staged prefix is copied in one go):
// descriptors | items | entry item offsets | poses (X | Y) | eval poses | states | status word | slots | records.
struct CtBlock {
  CtDesc* descs;
  int4* items;
  int* entry_items;
  double* XY;
  double* XYe;
  CtState* st;
  unsigned* ctr;
  double* slots;
  double* out;
};
CtBlock ct_block_layout(Carver& cv, size_t P, size_t I, size_t E, bool align) {
  CtBlock b;
  b.descs = cv.take<CtDesc>(P);
  b.items = cv.take<int4>(I);
  b.entry_items = cv.take<int>(E);
  b.XY = cv.take<double>(32 * P);
  b.XYe = cv.take<double>(32 * P);
  b.st = align ? cv.take<CtState>(P) : nullptr;
  b.ctr = cv.take<unsigned>(2);
  b.slots = cv.take<double>((size_t)GB_ACC_STRIDE * I);
  b.out = cv.take<double>((size_t)GB_OUT_DOUBLES * P);
  return b;
}

gb_status ct_check_factor(const gb_factor* f, const gb_ctx* ctx) {
  GB_REQUIRE(f, "null factor");
  GB_REQUIRE(f->kind == GB_FACTOR_CT, "not a CT factor: the gb_ct_* entry points take factors of gb_ct_gicp_factor_create only");
  GB_REQUIRE(f->ctx->device == ctx->device, "factor lives on another device");
  GB_REQUIRE(f->source->num_entries > 0, "the source has no times (gb_cloud_add_times)");
  return GB_OK;
}

bool finite16(const double* T) {
  for (int k = 0; k < 16; k++)
    if (!isfinite(T[k])) return false;
  return true;
}

// A prepared call: the work items and descriptors of P CT factors staged in pinned memory, the device block carved.
struct CtCall {
  gb_ctx* ctx = nullptr;
  size_t P = 0, I = 0;
  CtBlock h{}, d{};
  int grid = 1;
};
gb_status ct_prepare(gb_ctx* ctx, size_t P, gb_factor* const* factors, bool align, CtCall& c) {
  c.ctx = ctx;
  c.P = P;
  size_t I = 0, E = 0;
  for (size_t p = 0; p < P; p++) {
    const gb_cloud* src = factors[p]->source;
    for (int b = 0; b < src->num_entries; b++) I += (size_t)((src->h_starts[b + 1] - src->h_starts[b] + kCtChunk - 1) / kCtChunk);
    E += (size_t)src->num_entries + 1;
  }
  GB_REQUIRE(I < ((size_t)1 << 30), "too many work items");
  c.I = I;
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) { c.h = ct_block_layout(cv, P, I, E, align); }));
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) { c.d = ct_block_layout(cv, P, I, E, align); }));
  size_t it = 0, e = 0;
  for (size_t p = 0; p < P; p++) {
    const gb_factor* fa = factors[p];
    const gb_cloud* src = fa->source;
    CtDesc& C = c.h.descs[p];
    memset(&C, 0, sizeof(C));
    C.D.p0 = src->p0; C.D.p1 = src->p1; C.D.p2 = src->p2;
    C.D.n = (int)src->n;
    desc_target_gicp(C.D, C.G, fa);
    C.inv_perm = src->inv_perm;
    C.tau = src->t_tau;
    C.entry_items = c.d.entry_items + e;
    C.num_entries = src->num_entries;
    size_t local = 0;
    for (int b = 0; b < src->num_entries; b++) {
      c.h.entry_items[e++] = (int)(it + local);
      for (int j = src->h_starts[b]; j < src->h_starts[b + 1]; j += kCtChunk, local++)
        c.h.items[it + local] = make_int4((int)p, b, j, std::min(kCtChunk, src->h_starts[b + 1] - j));
    }
    c.h.entry_items[e++] = (int)(it + local);
    it += local;
  }
  c.grid = (int)std::max<size_t>(1, std::min<size_t>((I + kWarps - 1) / kWarps, (size_t)ctx->num_sms * 2));
  return GB_OK;
}
// the staged prefix (descriptors .. status word) to the device
gb_status ct_upload(CtCall& c) {
  GB_CUDA(cudaMemcpyAsync(c.d.descs, c.h.descs, (char*)c.h.ctr - (char*)c.h.descs, cudaMemcpyHostToDevice, c.ctx->stream));
  return GB_OK;
}
gb_status ct_launch_sweep(CtCall& c, int mode) {
  if (c.I == 0) return GB_OK;
  const bool lin = mode == GB_MODE_LINEARIZE;
  return gb_launch(c.ctx, "k_ct_sweep", lin ? k_ct_sweep<GB_MODE_LINEARIZE> : k_ct_sweep<GB_MODE_ERROR>, c.grid, kThreads, 0, c.d.descs, c.d.items, (int)c.I, c.d.XY,
                   c.d.XYe, c.d.slots);
}

// linearize (mode LINEARIZE, out: P records) or error (mode ERROR, errors: P) of P CT factors
gb_status ct_evaluate(gb_ctx* ctx, size_t P, gb_factor* const* factors, const double* X, const double* Y, const double* Xe, const double* Ye, int mode, gb_linearized6* out, double* errors) {
  CtCall c;
  GB_CHECK(ct_prepare(ctx, P, factors, false, c));
  for (size_t p = 0; p < P; p++) {
    memcpy(c.h.XY + 32 * p, X + 16 * p, sizeof(double) * 16);
    memcpy(c.h.XY + 32 * p + 16, Y + 16 * p, sizeof(double) * 16);
    if (mode == GB_MODE_ERROR) {
      memcpy(c.h.XYe + 32 * p, Xe + 16 * p, sizeof(double) * 16);
      memcpy(c.h.XYe + 32 * p + 16, Ye + 16 * p, sizeof(double) * 16);
    }
  }
  GB_CHECK(ct_upload(c));
  GB_CHECK(ct_launch_sweep(c, mode));
  // error(): the residual blocks are not formed, so the record's poses do not matter; its error is that of the eval poses
  const bool lin = mode == GB_MODE_LINEARIZE;
  GB_CHECK(gb_launch(ctx, "k_ct_record", lin ? k_ct_record<GB_MODE_LINEARIZE> : k_ct_record<GB_MODE_ERROR>, (int)P, kCtThreads, 0, c.d.descs, c.d.XY, c.d.slots, c.d.out));
  GB_CUDA(cudaMemcpyAsync(c.h.out, c.d.out, sizeof(double) * GB_OUT_DOUBLES * P, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  for (size_t p = 0; p < P; p++) {
    if (out) memcpy(&out[p], c.h.out + GB_OUT_DOUBLES * p, sizeof(gb_linearized6));
    if (errors) errors[p] = c.h.out[GB_OUT_DOUBLES * p + 120];
  }
  return GB_OK;
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// entry points
// ---------------------------------------------------------------------------------------------
extern "C" gb_status gb_cloud_add_times(gb_ctx* ctx, gb_cloud* cloud, size_t n, const double* times) {
  GB_REQUIRE(ctx && cloud && times, "null argument");
  GB_REQUIRE(cloud->device == ctx->device, "the cloud lives on another device");
  GB_REQUIRE(n == cloud->n, "the number of times differs from the cloud's size");
  GB_REQUIRE(n >= 1, "an empty cloud has no time table");
  for (size_t i = 0; i < n; i++) {
    GB_REQUIRE(isfinite(times[i]), "times must be finite");
    GB_REQUIRE(i == 0 || times[i] >= times[i - 1], "times must be non-decreasing (as the preprocess leaves them)");
  }
  GB_ENTER(ctx);
  std::vector<int> starts(n + 1);
  std::vector<double> tau(n);
  const int B = ct_time_table(times, (int)n, starts.data(), tau.data());
  starts.resize((size_t)B + 1);
  tau.resize((size_t)B);
  // stage in pinned memory, then one device block of the pool that replaces the old table once the upload has succeeded
  CtTable h;
  size_t bytes = 0;
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) {
    h = ct_table_layout(cv, B);
    bytes = cv.off;
  }));
  memcpy(h.starts, starts.data(), sizeof(int) * starts.size());
  memcpy(h.tau, tau.data(), sizeof(double) * tau.size());
  gb_dev_block block(ctx->device);
  CtTable d;
  GB_CHECK(gb_dev_carve(ctx, block, [&](Carver& cv) { d = ct_table_layout(cv, B); }));
  const cudaError_t e1 = cudaMemcpyAsync(d.starts, h.starts, bytes, cudaMemcpyHostToDevice, ctx->stream);
  const cudaError_t e2 = e1 == cudaSuccess ? cudaStreamSynchronize(ctx->stream) : e1;
  if (e2 != cudaSuccess) {
    gb_set_error("time table upload failed: %s", cudaGetErrorString(e2));
    return GB_ERR_CUDA;
  }
  block.hand_over(cloud->t_base);  // the old table goes back to the pool on return
  cloud->t_starts = d.starts;
  cloud->t_tau = d.tau;
  cloud->num_entries = B;
  cloud->t_first = times[0];
  cloud->t_last = times[starts[(size_t)B - 1]];
  cloud->h_starts.swap(starts);
  cloud->h_tau.swap(tau);
  return GB_OK;
}

extern "C" gb_status gb_cloud_time_table(const gb_cloud* cloud, int* num_entries, int32_t* starts, double* tau, double* t_first, double* t_last) {
  GB_REQUIRE(cloud, "null cloud");
  if (num_entries) *num_entries = cloud->num_entries;
  if (starts && cloud->num_entries) memcpy(starts, cloud->h_starts.data(), sizeof(int) * cloud->h_starts.size());
  if (tau && cloud->num_entries) memcpy(tau, cloud->h_tau.data(), sizeof(double) * cloud->h_tau.size());
  if (t_first) *t_first = cloud->t_first;
  if (t_last) *t_last = cloud->t_last;
  return GB_OK;
}

extern "C" gb_status gb_ct_gicp_factor_create(gb_ctx* ctx, const gb_ivox* target, const gb_cloud* source, double max_correspondence_distance, gb_factor** out) {
  GB_REQUIRE(ctx && target && source && out, "null argument");
  *out = nullptr;
  GB_REQUIRE(std::isfinite(max_correspondence_distance) && max_correspondence_distance > 0.0, "max_correspondence_distance must be positive and finite");
  const gb_voxelmap* m = ivox_map(target);
  GB_REQUIRE(m->kind == GB_MAP_IVOX, "the target is not an iVox");
  GB_REQUIRE(m->device == ctx->device && source->device == ctx->device, "cloud / iVox live on another device");
  GB_REQUIRE(source->num_entries > 0, "the source has no times (gb_cloud_add_times)");
  GB_ENTER(ctx);
  gb_factor* f = factor_new(ctx, GB_FACTOR_CT, m, source);
  if (!f) return GB_ERR_INTERNAL;
  f->max_corr2 = (float)(max_correspondence_distance * max_correspondence_distance);
  *out = f;
  return GB_OK;
}

extern "C" gb_status gb_ct_gicp_linearize(gb_factor* f, const double X[16], const double Y[16], gb_linearized6* out) {
  GB_REQUIRE(f && X && Y && out, "null argument");
  GB_CHECK(ct_check_factor(f, f->ctx));
  GB_REQUIRE(finite16(X) && finite16(Y), "X and Y must be finite");
  GB_ENTER(f->ctx);
  return ct_evaluate(f->ctx, 1, &f, X, Y, nullptr, nullptr, GB_MODE_LINEARIZE, out, nullptr);
}

extern "C" gb_status gb_ct_gicp_error(gb_factor* f, const double X_lin[16], const double Y_lin[16], const double X_eval[16], const double Y_eval[16], double* error) {
  GB_REQUIRE(f && X_lin && Y_lin && X_eval && Y_eval && error, "null argument");
  GB_CHECK(ct_check_factor(f, f->ctx));
  GB_REQUIRE(finite16(X_lin) && finite16(Y_lin) && finite16(X_eval) && finite16(Y_eval), "poses must be finite");
  GB_ENTER(f->ctx);
  return ct_evaluate(f->ctx, 1, &f, X_lin, Y_lin, X_eval, Y_eval, GB_MODE_ERROR, nullptr, error);
}

extern "C" gb_status gb_ct_default_params(gb_ct_params* p) {
  GB_REQUIRE(p, "null params");
  GB_CHECK(gb_align_default_params(&p->lm));
  p->lm.max_iterations = 8;       // lm_max_iterations (config_odometry_ct.json)
  p->lm.lambda_initial = 1e-10;   // odometry_estimation_ct.cpp:171-182
  p->lm.absolute_error_tol = 1e-2;
  p->lm.step_translation_tol = 0.0;  // GLIM's CT loop has no step test
  p->lm.step_rotation_tol = 0.0;
  p->location_consistency_inf_scale = 1e-3;  // config_odometry_ct.json:25
  p->constant_velocity_inf_scale = 1e3;      // config_odometry_ct.json:26 (the code default is 1e-3)
  return GB_OK;
}

extern "C" gb_status gb_ct_gicp_align(gb_ctx* ctx, size_t P, gb_factor* const* factors, const double* X_init, const double* Y_init, const double* X_prior, const gb_ct_params* prm,
                                      gb_ct_result* results) {
  GB_REQUIRE(ctx, "null ctx");
  if (P == 0) return GB_OK;
  GB_REQUIRE(factors && X_init && Y_init && X_prior && prm && results, "null argument");
  GB_REQUIRE(P < ((size_t)1 << 20), "too many problems");
  for (size_t p = 0; p < P; p++) GB_CHECK(ct_check_factor(factors[p], ctx));
  for (size_t p = 0; p < P; p++)
    GB_REQUIRE(finite16(X_init + 16 * p) && finite16(Y_init + 16 * p) && finite16(X_prior + 16 * p), "X_init, Y_init and X_prior must be finite");
  GB_CHECK(gb_align_params_check(&prm->lm));
  GB_REQUIRE(isfinite(prm->location_consistency_inf_scale) && prm->location_consistency_inf_scale >= 0.0, "location_consistency_inf_scale must be finite and >= 0");
  GB_REQUIRE(isfinite(prm->constant_velocity_inf_scale) && prm->constant_velocity_inf_scale >= 0.0, "constant_velocity_inf_scale must be finite and >= 0");
  GB_ENTER(ctx);
  CtCall c;
  GB_CHECK(ct_prepare(ctx, P, factors, true, c));
  for (size_t p = 0; p < P; p++) {
    ct_init(c.h.st[p], X_init + 16 * p, Y_init + 16 * p, X_prior + 16 * p, prm->lm.lambda_initial);
    memcpy(c.h.XY + 32 * p, X_init + 16 * p, sizeof(double) * 16);
    memcpy(c.h.XY + 32 * p + 16, Y_init + 16 * p, sizeof(double) * 16);
    memcpy(c.h.XYe + 32 * p, c.h.XY + 32 * p, sizeof(double) * 32);
  }
  GB_CHECK(ct_upload(c));
  cudaStream_t stream = ctx->stream;
  GB_CUDA(cudaStreamSynchronize(stream));
  const double wl = prm->location_consistency_inf_scale, wc = prm->constant_velocity_inf_scale;
  GB_CHECK(gb_align_rounds(ctx, c.d.ctr, c.h.ctr, [&](bool need_lin) -> gb_status {
    if (need_lin) GB_CHECK(ct_launch_sweep(c, GB_MODE_LINEARIZE));
    GB_CHECK(gb_launch(ctx, "k_ct_step", k_ct_step, (int)P, kCtThreads, 0, c.d.st, c.d.descs, c.d.slots, c.d.XYe, wl, wc, c.d.ctr));
    GB_CHECK(ct_launch_sweep(c, GB_MODE_ERROR));
    return gb_launch(ctx, "k_ct_accept", k_ct_accept, (int)P, kCtThreads, 0, c.d.st, c.d.descs, c.d.slots, c.d.XY, prm->lm, wl, wc, c.d.ctr);
  }));
  GB_CUDA(cudaMemcpyAsync(c.h.st, c.d.st, sizeof(CtState) * P, cudaMemcpyDeviceToHost, stream));
  GB_CUDA(cudaStreamSynchronize(stream));
  for (size_t p = 0; p < P; p++) {
    memcpy(results[p].X, c.h.st[p].a.T, sizeof(double) * 16);
    memcpy(results[p].Y, c.h.st[p].Y, sizeof(double) * 16);
    align_result(c.h.st[p].a, results[p]);
  }
  return GB_OK;
}

extern "C" gb_status gb_ct_deskew(gb_ctx* ctx, const gb_cloud* source, const double X[16], const double Y[16], const int32_t* neighbors, int kc, int k, double* out_xyzw,
                                  double* out_cov4x4, double* out_normals4, gb_cloud** out_cloud) {
  GB_REQUIRE(ctx && source && X && Y && neighbors, "null argument");
  if (out_cloud) *out_cloud = nullptr;
  GB_REQUIRE(source->device == ctx->device, "the cloud lives on another device");
  GB_REQUIRE(source->num_entries > 0, "the source has no times (gb_cloud_add_times)");
  GB_REQUIRE(finite16(X) && finite16(Y), "X and Y must be finite");
  GB_REQUIRE(k >= 1 && k <= kc, "need 1 <= k_neighbors <= k_correspondences");
  const size_t n = source->n;
  for (size_t i = 0; i < n; i++)
    for (int j = 0; j < k; j++) {
      const int32_t v = neighbors[i * (size_t)kc + j];
      GB_REQUIRE(v >= 0 && (size_t)v < n, "neighbour index out of range");
    }
  GB_ENTER(ctx);
  gb_owned<gb_cloud> c(out_cloud ? new (std::nothrow) gb_cloud() : nullptr, cloud_free);
  if (out_cloud && !c) return GB_ERR_INTERNAL;
  if (c) { c->device = ctx->device; c->covs = true; }
  const size_t cub_b = gb_cub_temp_bytes(n);
  gb_planes staged;
  gb_sort_tmp t;
  double4 *d_pts, *d_nrm;
  double *d_cov, *d_XY;
  int *d_nb, *d_cnt;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    staged = gb_cloud_planes(cv, n, true);
    t = gb_take_sort_tmp(cv, n, cv.take<char>(cub_b), cub_b);
    d_pts = cv.take<double4>(n);
    d_nrm = cv.take<double4>(n);
    d_cov = cv.take<double>(16 * n);
    d_XY = cv.take<double>(32);
    d_nb = cv.take<int>(n * (size_t)kc);
    d_cnt = cv.take<int>(1);
  }));
  GB_CHECK(gb_upload(ctx, {{d_XY, X, sizeof(double) * 16}, {d_XY + 16, Y, sizeof(double) * 16}, {d_nb, neighbors, sizeof(int) * n * (size_t)kc}}));
  const int M = (int)n;
  GB_CHECK(gb_launch(ctx, "k_ct_deskew", k_ct_deskew, (M + 255) / 256, 256, 0, M, source->p0, source->perm, source->t_starts, source->t_tau, source->num_entries, d_XY, d_pts, d_cnt));
  GB_CHECK(gb_covariance_cloud(ctx, M, d_cnt, d_pts, d_nb, kc, k, d_nrm, d_cov, staged, t, c.get()));
  GB_CHECK(gb_download(ctx, {{out_xyzw, d_pts, sizeof(double4) * n}, {out_cov4x4, d_cov, sizeof(double) * 16 * n}, {out_normals4, d_nrm, sizeof(double4) * n}}));
  if (out_cloud) *out_cloud = c.release();
  return GB_OK;
}
