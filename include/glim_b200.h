/*
 * glim_b200.h -- C-ABI of libglim_b200.so: the H100-native (sm_90a) VGICP scan-matching hot path
 * of koide3/glim, behind the surface GLIM's modules use from gtsam_points.
 *
 * Every entry point cites the reference interface it replaces (paths relative to the GLIM tree,
 * v1.2.2).  The arithmetic of those interfaces lives in the un-vendored dependency
 * koide3/gtsam_points (CMakeLists.txt:28); the citations are GLIM's own call sites.
 *
 * Rules of the boundary
 *   - plain C: opaque handles, pointers and sizes only; no exceptions, no C++ or torch types.
 *   - every function returns gb_status (0 = OK); gb_status_string() / gb_last_error() explain.
 *   - handles are created / destroyed by the caller with the matching _create / _destroy.
 *     A gb_factor BORROWS its cloud and voxel map (the C++ shim keeps shared_ptrs alive, as the
 *     reference factor does); destroying a cloud or map that a live factor uses is a caller bug.
 *     Likewise a gb_sweep BORROWS its factors, and a sweep with a peer slab attached borrows the slab.
 *   - a gb_ctx owns one CUDA stream; all work issued through it is ordered on that stream.  The natural
 *     use is one gb_ctx per module thread (the reference drives each module from exactly one executor
 *     thread: src/glim/odometry/async_odometry_estimation.cpp:15), but a ctx may be called from several
 *     host threads (every entry point takes the ctx's mutex), and clouds / voxel maps uploaded through
 *     one ctx may be used by factors and sweeps of another ctx of the same device: frames migrate from
 *     the odometry thread to sub-mapping to global mapping (async_sub_mapping.cpp:8,
 *     async_global_mapping.cpp:24).  Every upload / build call returns after its stream has drained.
 *     Any thread may destroy a cloud, map, factor or sweep, whichever context made it.  A context destroyed while its
 *     factors or sweeps are alive lives on until the last of them is destroyed; they keep working meanwhile.
 *     A factor destroyed while sweeps cached by other contexts name it leaves those sweeps stale: each context drops its
 *     own on its next factor-set call; a caller-owned gb_sweep that names it is refused from then on.
 *   - a freed cloud / map block is recycled only after the stream of every live context of the device has drained (what
 *     cudaFree would wait for).  A stream with a capture in progress is skipped, not synchronised: that would invalidate the
 *     capture.  A free never fails and never leaves a CUDA error in the calling thread's last-error slot.
 *   - caller-owned streams (gb_ctx_create_on_stream): the library orders its work on the stream and may synchronise it.
 *     A caller that captures on such a stream (e.g. a torch CUDA graph, best in thread-local mode) must begin the capture on
 *     a drained stream, must make no call through that context while capturing, and must not destroy library objects that
 *     work still in flight on the stream reads.  Frees made by other threads during the capture do not touch the stream.
 *     On the legacy default stream (0) no graph capture can begin: small sweeps run as plain launches, with the same
 *     results.  Device results (gb_sweep_results_device) may be read on the same stream right after gb_sweep_launch.
 *   - gb_last_error() is per thread: a failure in one thread does not change another thread's message.
 *   - 4x4 poses are 16 doubles, COLUMN-MAJOR (Eigen::Isometry3d::data()).
 *   - 6x6 blocks are column-major, tangent order [rotation(3); translation(3)] (gtsam::Pose3).
 *   - there is NO CPU fallback: without a CUDA device every call fails with GB_ERR_NO_DEVICE.
 */
#ifndef GLIM_B200_H
#define GLIM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GB_API __attribute__((visibility("default")))

typedef int gb_status;
enum {
  GB_OK = 0,
  GB_ERR_INVALID_ARGUMENT = 1,
  GB_ERR_CUDA = 2,
  GB_ERR_OUT_OF_MEMORY = 3,
  GB_ERR_NO_DEVICE = 4,
  GB_ERR_INTERNAL = 5
};

typedef struct gb_ctx gb_ctx;           /* CUDAStream + StreamTempBufferRoundRobin (odometry_estimation_gpu.cpp:76-77) */
typedef struct gb_cloud gb_cloud;       /* gtsam_points::PointCloudGPU                                              */
typedef struct gb_voxelmap gb_voxelmap; /* gtsam_points::GaussianVoxelMapGPU                                        */
typedef struct gb_factor gb_factor;     /* gtsam_points::IntegratedVGICPFactorGPU                                   */
typedef struct gb_sweep gb_sweep;       /* gtsam_points::NonlinearFactorSetGPU (a prepared batch of factors)        */
typedef struct gb_ivox gb_ivox;         /* gtsam_points::iVox (odometry_estimation_cpu.cpp:57-61), kept on the device */
typedef struct gb_point_grid gb_point_grid; /* a whole frame's points on the device: the KdTree target of IntegratedGICPFactor  */
#define GB_SLAB_STRIDE 96               /* floats per row of the per-pair Hessian slab (layout below, at gb_sweep_create) */

/* LinearizedSystem6 of the reference GPU factor, widened to fp64 (SURVEY.md 8(a) a4, A.3).
 * To GTSAM: HessianFactor(k_t, k_s, H_tt, H_ts, -b_t, H_ss, -b_s, error); unary: (k_s, H_ss, -b_s, error).
 * error = sum r^T M r (no 1/2).  122 doubles. */
typedef struct gb_linearized6 {
  double H_tt[36];
  double H_ss[36];
  double H_ts[36]; /* rows: target tangent, cols: source tangent */
  double b_t[6];
  double b_s[6];
  double error;
  double num_inliers;
} gb_linearized6;

/* factor flags */
#define GB_FACTOR_DEFAULT 0
/* set_enable_surface_validation(true) (odometry_estimation_gpu.cpp:145,162).  The reference rule lives in the
 * un-vendored gtsam_points and is not recoverable here (SURVEY A.6, unpinned ledger); implemented is the documented
 * orientation-consistency gate of DESIGN.md section 7: with n = R n_source, a correspondence is kept iff
 * 3 n^T C_voxel n <= tr(C_voxel).  The source cloud must carry normals (gb_vgicp_factor_create fails otherwise). */
#define GB_FACTOR_SURFACE_VALIDATION 1

GB_API const char* gb_status_string(gb_status s);
GB_API const char* gb_last_error(void); /* thread-local detail of the last failure */
GB_API int gb_device_count(void);       /* cuda_device_names / cuda_mem_get_info: src/glim/util/debug.cpp:84 */
GB_API gb_status gb_mem_info(int device, size_t* free_bytes, size_t* total_bytes); /* src/glim/viewer/memory_monitor.cpp:39 */

/* ---- context: replaces gtsam_points::CUDAStream + StreamTempBufferRoundRobin
 *      (odometry_estimation_gpu.cpp:76-77, sub_mapping.cpp:86-87, global_mapping.cpp:110) ---- */
GB_API gb_status gb_ctx_create(int device, gb_ctx** out);
/* same, but enqueue on a caller-owned cudaStream_t (e.g. the stream NCCL collectives run on) */
GB_API gb_status gb_ctx_create_on_stream(int device, void* cuda_stream, gb_ctx** out);
GB_API gb_status gb_ctx_destroy(gb_ctx* ctx);
GB_API gb_status gb_ctx_synchronize(gb_ctx* ctx);
GB_API void* gb_ctx_stream(gb_ctx* ctx); /* the cudaStream_t */
/* launches made through ctx so far: one per kernel launch and one per cub device-wide call (a sort or scan of several
 * kernels) of this library, one per launch of a captured sweep graph; memsets and copies are not counted */
GB_API uint64_t gb_ctx_kernel_launches(gb_ctx* ctx);

/* ---- PointCloudGPU::clone(frame[, stream]) (odometry_estimation_gpu.cpp:96; sub_mapping.cpp:168,393;
 *      global_mapping.cpp:253,260,743).  Host layout as the reference's PointCloudCPU:
 *      xyzw = N x Vector4d (w = 1), cov4x4 = N x Matrix4d column-major (last row/col 0) or NULL,
 *      normals4 = N x Vector4d or NULL (standard_viewer_mem.cpp:34-41).  Device layout is fp32
 *      (standard_viewer_mem.cpp:49-58), covariance kept as its 6 unique entries. ---- */
GB_API gb_status gb_cloud_upload(gb_ctx* ctx, size_t n, const double* xyzw, const double* cov4x4, const double* normals4, gb_cloud** out);
GB_API gb_status gb_cloud_size(const gb_cloud* cloud, size_t* n);
/* device -> host copy of the fp32 device data: xyz N x 3, cov6 N x 6 (c00 c01 c02 c11 c12 c22); either may be NULL */
GB_API gb_status gb_cloud_download(const gb_cloud* cloud, float* xyz, float* cov6);
/* device pointers of the planes (points_gpu / covs_gpu / normals_gpu of the reference's PointCloud: GLIM only tests them for
 * null, sub_mapping.cpp:165, global_mapping.cpp:252, :330).  p0 = N x float4 {x y z c00}, p1 = N x float4 {c01 c02 c11 c12},
 * p2 = N x float c22, normals = N x float4 or NULL; stored in the cloud's internal (Morton) order.  Any output may be NULL. */
GB_API gb_status gb_cloud_device_ptrs(const gb_cloud* cloud, void** p0, void** p1, void** p2, void** normals);
GB_API gb_status gb_cloud_destroy(gb_cloud* cloud);

/* ---- GaussianVoxelMapGPU(resolution, init_num_buckets = 8192*2, max_bucket_scan_count = 10,
 *      target_points_drop_rate = 1e-3, stream)::insert(cloud)   (odometry_estimation_gpu.cpp:103-104;
 *      sub_mapping.cpp:398-399; global_mapping.cpp:265-266, 747-748) ---- */
GB_API gb_status gb_voxelmap_build(gb_ctx* ctx, const gb_cloud* cloud, float resolution, int init_num_buckets, int max_bucket_scan_count, double target_points_drop_rate, gb_voxelmap** out);
/* voxel_resolution(), voxelmap_info.{num_voxels,num_buckets} (standard_viewer_callbacks.cpp:117; standard_viewer_mem.cpp:76-77) */
GB_API gb_status gb_voxelmap_info(const gb_voxelmap* map, int* num_voxels, int* num_buckets, float* resolution);
/* device -> host: buckets NB x 4 int32 (x y z index, index -1 = empty), per voxel num_points, mean (V x 3),
 * cov6 (V x 6); any pointer may be NULL.  GB_ERR_INVALID_ARGUMENT for an iVox (gb_ivox_download). */
GB_API gb_status gb_voxelmap_download(const gb_voxelmap* map, int32_t* buckets, int32_t* num_points, float* means, float* cov6);
GB_API gb_status gb_voxelmap_destroy(gb_voxelmap* map);

/* ---- Incremental device map: the scan-to-map target of GLIM's odometry (odometry_estimation_cpu.cpp:177-191, update_target:
 *      random_sampling(10 %) from frame 5 on, transform, GaussianVoxelMapCPU::insert on every level; set_lru_horizon(lru_thresh
 *      = 100) at :67), kept on the device.  The result is an ordinary gb_voxelmap: info, download, destroy, factors, sweeps,
 *      gb_vgicp_align and gb_overlap take it unchanged, and sweeps created before an insert follow it (their descriptors
 *      are re-written before the next launch).
 *
 *      The rule.  Per voxel the map keeps its packed key, n, fp64 sums Sigma q (3) and Sigma C (6 unique entries) and
 *      stamp; per map the insert counter c, h = lru_horizon and k = lru_clear_cycle.  One insert:
 *        1. sample: sampling_rate = 1 keeps every point; otherwise m = (size_t)(n * rate) points are kept (random_sampling's
 *           count): those with the smallest rg_hash(seed, original index) ([EXT]: the reference draws with std::mt19937).
 *        2. transform the kept points with finite x, y, z: q = R a + t, C' = R C R^T, un-contracted fp64 (gb_merge_frames'
 *           association order).
 *        3. key: floor(q * (1.0 / (double)resolution)) in fp64, as GaussianVoxelMapCPU; points outside the 21-bit key range
 *           (+-2^20 voxels) are skipped.
 *        4. accumulate: each touched voxel starts from its stored sums (new voxels from zero) and adds its new points one at
 *           a time in original index order; then n += count, stamp = c.
 *        5. evict: c += 1; if h > 0 and c % k == 0, the voxels with stamp + h < c are dropped.  An insert that keeps no
 *           points still advances c.
 *        6. finalize: record = (float)(Sigma / n) component-wise, with n, in ascending packed-key order (the build's voxel
 *           numbering); the table is rebuilt with the build's sizing rule (init_num_buckets doubled until >= 8 V, then while
 *           more than target_points_drop_rate * Sigma n points are dropped).
 *      Voxel coordinates come from fp64 keys, while every lookup (sweeps, overlap) uses the fp32 rule of the build: a point
 *      exactly on a voxel face may resolve to a neighbouring voxel at lookup time.
 *
 *      Threading: do not insert into a map while another thread uses it (linearizes a factor on it, builds a sweep over it,
 *      ...) -- the same caller bug as destroying a map a live factor borrows.  Device work already in flight on another
 *      context stays safe: the replaced device blocks are recycled only after every stream of the device has drained.
 *      Like the build, an insert returns after its stream has drained: two host synchronisations per insert. ---- */
/* An empty map that accepts any number of inserts.  lru_horizon <= 0: no eviction; lru_clear_cycle >= 1 (gtsam_points: 10). */
GB_API gb_status gb_voxelmap_create_incremental(gb_ctx* ctx, float resolution, int init_num_buckets, int max_bucket_scan_count,
                                                double target_points_drop_rate, int lru_horizon, int lru_clear_cycle, gb_voxelmap** out);
/* Insert `cloud` at T_map_cloud (NULL = identity), keeping a sampling_rate share of its points (1 = all).  Every input is
 * validated before any launch: GB_ERR_INVALID_ARGUMENT for a map that is not incremental (from gb_voxelmap_build, which
 * keeps no sums, or an iVox), a non-finite T, sampling_rate outside (0, 1], or a cloud / map on another device than ctx. */
GB_API gb_status gb_voxelmap_insert(gb_ctx* ctx, gb_voxelmap* map, const gb_cloud* cloud, const double* T_map_cloud /* 16, col-major */,
                                    double sampling_rate, uint64_t seed);

/* ---- iVox: the scan-to-map target of GLIM's odometry with registration_type "GICP" (odometry_estimation_cpu.cpp:57-61:
 *      gtsam_points::iVox(ivox_resolution = 1.0), set_min_dist_in_cell(ivox_min_dist = 0.1), set_lru_horizon(lru_thresh = 100),
 *      set_neighbor_voxel_mode(1); update_target :177-191 inserts 10 % of each frame from frame 5 on), kept on the device.
 *      Each voxel holds a few actual points with their covariances.
 *
 *      The insert rule.  Per voxel the map keeps its packed key, its points in slot order and its stamp; per map the insert
 *      counter c, h = lru_horizon and k = lru_clear_cycle.  One insert:
 *        1-3. sample, transform and key exactly as gb_voxelmap_insert steps 1-3, with the key floor(q * (1.0 / resolution)) in
 *           fp64 (resolution is a double here).
 *        4. per touched voxel, sequentially: the stored points keep their slots; the new points are offered in original index
 *           order, and a point is admitted iff the voxel holds fewer than max_points_in_cell points and its squared distance to
 *           every point the voxel holds is >= min_dist_in_cell^2.  Stored values are the fp32 roundings of q and C'; the
 *           admission distance is computed in fp64 from the fp32-rounded positions, d2 = (dx^2 + dy^2) + dz^2, uncontracted.
 *           Every touched voxel gets stamp = c, also one whose new points were all refused.
 *        5. evict as gb_voxelmap_insert step 5: c += 1; if h > 0 and c % k == 0, the voxels with stamp + h < c are dropped; an
 *           insert that keeps no points still advances c.
 *        6. voxels in ascending packed-key order; the table is the build's (16384 buckets doubled until >= 8 V, 10 probes)
 *           with drop rate 0: every voxel is found.
 *      [EXT] gtsam_points is not vendored: the cell capacity 10 (max_points_in_cell default, recalled), the admission test of
 *      step 4 and the neighbour offsets below are this library's statement of it.
 *      Threading and lifetime as for incremental voxel maps: two host synchronisations per insert (one more per extra table
 *      attempt), sweeps created before an insert follow it, do not insert while another thread uses the map. ---- */
/* An iVox handle, a point-grid handle and a voxel-map handle are not interchangeable.  gb_ivox_insert, gb_ivox_info, gb_ivox_download and
 * gb_gicp_factor_create take an iVox only; gb_vgicp_factor_create and gb_voxelmap_download refuse one, and gb_voxelmap_insert
 * takes an incremental map only.  Each refuses another kind with GB_ERR_INVALID_ARGUMENT before any launch.  These
 * refusals are the only change of behaviour from earlier builds, which read a handle of the wrong kind as the other kind.
 * gb_overlap takes voxel maps and iVoxes: it tests occupancy only (point grids: see gb_point_grid_build).
 * neighbor_voxel_mode: 1 (centre), 7 (+ the faces), 19 (+ the edges), 27 (+ the corners).  lru_horizon <= 0: no eviction.
 * GB_ERR_INVALID_ARGUMENT for a non-finite or non-positive resolution, min_dist_in_cell < 0, max_points_in_cell outside
 * [1, 64], another mode or lru_clear_cycle < 1. */
GB_API gb_status gb_ivox_create(gb_ctx* ctx, double resolution, double min_dist_in_cell, int max_points_in_cell, int neighbor_voxel_mode,
                                int lru_horizon, int lru_clear_cycle, gb_ivox** out);
/* validated before any launch: T finite, sampling_rate in (0, 1], an iVox, cloud and map on ctx's device */
GB_API gb_status gb_ivox_insert(gb_ctx* ctx, gb_ivox* map, const gb_cloud* cloud, const double* T_map_cloud /* 16 col-major, NULL = I */,
                                double sampling_rate, uint64_t seed);
GB_API gb_status gb_ivox_info(const gb_ivox* map, int* num_voxels, size_t* num_points, double* resolution);
/* voxels in ascending packed-key order; points voxel-major, in slot order; any pointer may be NULL */
GB_API gb_status gb_ivox_download(const gb_ivox* map, int32_t* voxel_coords /* V x 3 */, int32_t* voxel_counts /* V */,
                                  float* xyz /* P x 3 */, float* cov6 /* P x 6 */);
GB_API gb_status gb_ivox_destroy(gb_ivox* map);
/* ---- The submap of GLIM's passthrough sub-mapping (SubMappingPassthrough::create_submap, src/glim/mapping/
 *      sub_mapping_passthrough.cpp:146-153): voxel_data() of the module's IncrementalVoxelMap<FlatContainer> (this iVox),
 *      transform(merged, T_world_origin^-1) and random_sampling down to submap_target_num_points, as one device call.
 *
 *      The rule.
 *        1. Points: the P = num_points stored points in map order (gb_ivox_download's: voxels by ascending packed key, each
 *           voxel's slots in order); a point's index i is its position in that order.
 *        2. Transform: from the stored fp32 record, q = R a + t and C' = R C R^T in the un-contracted fp64 of gb_merge_frames'
 *           transform (the same association order, the same per-point code); each value is stored once as fp32.
 *        3. Thinning iff target_num_points > 0 and P > target_num_points: m = (size_t)((double)P * ((double)target_num_points /
 *           (double)P)) points stay (the count of random_sampling at the module's rate, :151: not always the target, e.g. P =
 *           65692 with target 50000 keeps 49999), those with the smallest rg_hash(seed, i) (gb_thin's rule), in map order.
 *           [EXT] the reference draws with std::mt19937 over voxel_data()'s insertion order: only which points stay differs.
 *        4. Output: a new cloud with positions and covariances, and no normals, time table or FPFH features (the iVox keeps
 *           none).  It is stored as every cloud (gb_cloud_build's Morton order) and is bit-identical, planes, perm and inv_perm,
 *           to gb_cloud_upload of the rule's fp64 q and C' in output order.  An empty map, or m = 0, gives a valid empty cloud.
 *      target_num_points is an int, as in gb_merge_frames and as GLIM's submap_target_num_points is (the module passes it
 *      unchanged); callers holding a wider count clamp it to INT_MAX, which keeps the same points of any map this call accepts.
 *      The call never writes the map.  Launches: 4 (k_ivox_extract, gb_cloud_build's 3), 8 when thinning (gb_thin's 3 and the
 *      scan of its flags ahead of them), whatever P and the voxel count.  The one exception is an empty result (an empty map,
 *      or m = 0): no launch at all.  No transfer: P and m are known on the host.  One stream synchronisation, before it returns.
 *      GB_ERR_INVALID_ARGUMENT before any launch for a null ctx, map or out, a handle that is not an iVox (a voxel map or a
 *      point grid), a map on another device than ctx, a non-finite T_out_map or a map of 2^30 points or more. ---- */
GB_API gb_status gb_ivox_extract(gb_ctx* ctx, const gb_ivox* map, const double* T_out_map /* 16 col-major, NULL = I */,
                                 int target_num_points /* <= 0: keep all */, uint64_t seed, gb_cloud** out);

/* ---- IntegratedVGICPFactorGPU(target_key | fixed_target_pose, source_key, voxelmap, source, stream, buffer)
 *      (odometry_estimation_gpu.cpp:144,161; sub_mapping.cpp:307; global_mapping.cpp:335,466,860).
 *      Keys and the binary/unary distinction stay on the host side of the boundary: the device only
 *      ever sees delta = T_target^-1 * T_source (SURVEY A.1). ---- */
GB_API gb_status gb_vgicp_factor_create(gb_ctx* ctx, const gb_voxelmap* target, const gb_cloud* source, int flags, gb_factor** out);
GB_API gb_status gb_vgicp_factor_destroy(gb_factor* factor);
/* linearize(values): one fused kernel (lookup + residual + Jacobians + 6x6 reduction) */
GB_API gb_status gb_vgicp_linearize(gb_factor* factor, const double T_target_source[16], gb_linearized6* out);
/* error(values): inlier set found at T_lin, evaluated at T_eval (SURVEY A.2 / A.5) */
GB_API gb_status gb_vgicp_error(gb_factor* factor, const double T_lin[16], const double T_eval[16], double* error);
/* num_inliers() / inlier_fraction() come back in gb_linearized6::num_inliers */

/* ---- IntegratedGICPFactor_<iVox, PointCloud>(Pose3(), X(current), ivox, frame, ivox) + set_max_correspondence_distance
 *      (odometry_estimation_cpu.cpp:95-104, max_correspondence_distance = 2 * ivox_resolution).  The source must carry
 *      covariances, as for VGICP.  The result is an ordinary gb_factor: gb_vgicp_linearize / _error / _factor_destroy,
 *      gb_factor_set_*, gb_sweep_* and gb_vgicp_align take it.  The factors of one sweep or call must all be VGICP or all GICP
 *      (GB_ERR_INVALID_ARGUMENT before any launch); GICP sweeps take no pair_index, slab or peer slab; gb_overlap takes
 *      maps, not factors.
 *
 *      The correspondence rule.  q = the source point transformed with the sweep's fp32 pose (the lookup transform of every
 *      sweep), keyed with the fp32 rule (float)(1 / resolution) of every lookup (a point on a voxel face may key to its
 *      neighbour).  The voxels (cx, cy, cz) + o are searched for o in the mode's offset list, in order: the centre; the faces
 *      -x +x -y +y -z +z; the edges (zero axis x, y, z; the other two signs --, -+, +-, ++); the corners ((dx, dy, dz) in
 *      {-1, 1}^3, lexicographic).  The fp32 squared distance d2 = (dx^2 + dy^2) + dz^2 (d = p - q, uncontracted) to every
 *      stored point is formed; the nearest point with d2 < (float)(max_correspondence_distance^2) is the correspondence, ties
 *      to the earlier offset, then the earlier slot.  The per-point arithmetic is the VGICP factor's with the matched point's
 *      position and covariance in place of the voxel's mean and covariance: r = p - q, M = (C_p + R C_a R^T)^-1,
 *      error = sum r^T M r (no 1/2), and error() takes its correspondences at T_lin and evaluates at T_eval.
 *      [EXT] "nearest stored point within the maximum distance" and this error convention are this library's statement of the
 *      un-vendored gtsam_points factor.
 *      gb_sweep_stats of a GICP sweep: 48 B per source point, 48 B per stored target point, 16 B per bucket of the smallest
 *      power-of-two table >= 16384 holding the voxels, plus pose and record. ---- */
GB_API gb_status gb_gicp_factor_create(gb_ctx* ctx, const gb_ivox* target, const gb_cloud* source, double max_correspondence_distance, gb_factor** out);

/* ---- IntegratedGICPFactor(target_key, source_key, target_frame, source_frame) with the target's KdTree: GICP between two whole
 *      point clouds, the nearest target point of each source point its correspondence (sub_mapping.cpp:189-211 between factors,
 *      global_mapping.cpp:379-428 submap between factors, global_mapping_pose_graph.cpp:391-405 loop candidates), on the device.
 *      An exact KdTree returns the brute-force nearest neighbour; here a uniform grid over the target's points finds the same
 *      point by a bounded cell search.
 *
 *      The point grid.  gb_point_grid_build copies every point of a device cloud (position and covariance) into a map of its
 *      own kind; a cloud without covariances is accepted, and its records then hold zero covariances (the ICP factor below
 *      reads positions only).  Each point with finite x, y, z is keyed with the fp32 lookup rule k = floor((float)(p * (float)(1 / cell_size)))
 *      per axis (as every sweep keys its queries); points that are not finite, or whose key is outside the 21-bit range
 *      (+-2^20 cells), are stored but never match.  Cells are in ascending packed-key order, and the points of a cell in
 *      ascending original index (the cloud's caller order); a cell is {first point, count}.  Records have the iVox's layout
 *      {x y z c00} {c01 c02 c11 c12} {c22, 1, ., .}.  The table is the build's (16384 buckets doubled until >= 8 cells, 10
 *      probes) with drop rate 0: every cell is found.  The grid is built once (no insert) and owns its memory, so the cloud
 *      may be destroyed after the build.  An empty cloud gives an empty grid.  GB_ERR_INVALID_ARGUMENT before any launch for
 *      a non-finite or non-positive cell_size or a cloud on another device than ctx.
 *
 *      The correspondence.  q = the source point transformed with the sweep's fp32 pose, c = its cell.  The cells c + o are
 *      searched for o in [-m, m]^3, where m is the smallest integer that provably holds every stored point with
 *      d2 < (float)(r^2) given the fp32 rounding of 1 / cell_size, of q * inv and of r^2 (the proof is at grid_half_width,
 *      gb_grid_math.cuh; m depends on r / cell_size and, by a few ulps, on the grid's extent; gb_gicp_grid_factor_half_width
 *      reports it).  The match is the stored point with the smallest fp32 d2 = (dx^2 + dy^2) + dz^2 (d = p - q, uncontracted)
 *      subject to d2 < (float)(r^2), ties to the smaller original index: the brute-force argmin over all target points,
 *      whatever the search order (unlike the iVox rule, whose ties follow the offset order).  A query whose key saturates
 *      finds nothing.  Per point the factor is the iVox GICP factor's: r = p - q, M = (C_p + R C_a R^T)^-1, error = sum
 *      r^T M r (no 1/2); error() takes its correspondences at T_lin and evaluates at T_eval.  [EXT] the un-vendored
 *      IntegratedGICPFactor's KdTree search and error convention are this library's statement of them.
 *
 *      A grid factor is an ordinary pose gb_factor: gb_vgicp_linearize / _error / _factor_destroy, gb_factor_set_*, gb_sweep_*
 *      and gb_vgicp_align take it.  A sweep or call holds one target class -- voxel maps, iVoxes or point grids -- and a mix is
 *      GB_ERR_INVALID_ARGUMENT before any launch (ICP factors, gb_icp_grid_factor_create, are a class of their own); grid sweeps
 *      take no pair_index, slab or peer slab.  gb_sweep_stats of a grid
 *      sweep: 48 B per source point, 48 B per stored target point, 16 B per bucket of the smallest power-of-two table >= 16384
 *      holding the cells, plus pose and record.
 *      A grid is not a voxel map and not an iVox: gb_vgicp_factor_create, gb_gicp_factor_create, gb_ct_gicp_factor_create,
 *      gb_voxelmap_insert, gb_voxelmap_download, the gb_ivox_* calls and gb_overlap refuse it with GB_ERR_INVALID_ARGUMENT
 *      before any launch, and gb_point_grid_info / _download / gb_gicp_grid_factor_create refuse every other kind.  These are
 *      refusals of the new kind only: no call valid before changes. ---- */
GB_API gb_status gb_point_grid_build(gb_ctx* ctx, const gb_cloud* cloud, double cell_size, gb_point_grid** out);
GB_API gb_status gb_point_grid_info(const gb_point_grid* grid, int* num_cells, size_t* num_points, double* cell_size);
/* cells in ascending packed-key order: cell_coords (C x 3), cell_counts (C); points in record order (the keyed ones cell-major,
 * then those that never match): original indices (P), xyz (P x 3), cov6 (P x 6); any pointer may be NULL */
GB_API gb_status gb_point_grid_download(const gb_point_grid* grid, int32_t* cell_coords, int32_t* cell_counts, int32_t* indices, float* xyz, float* cov6);
GB_API gb_status gb_point_grid_destroy(gb_point_grid* grid);
/* A GICP factor on a point grid.  GB_ERR_INVALID_ARGUMENT before any launch, creating nothing, for a non-finite or
 * non-positive max_correspondence_distance, a target that is not a point grid, a source without covariances, a grid or
 * source on another device than ctx, or a search half-width m above 8 (r more than about 8 cell sizes). */
GB_API gb_status gb_gicp_grid_factor_create(gb_ctx* ctx, const gb_point_grid* target, const gb_cloud* source, double max_correspondence_distance, gb_factor** out);
/* the factor's search half-width m (0 for a factor of another kind) */
GB_API gb_status gb_gicp_grid_factor_half_width(const gb_factor* factor, int* m);

/* ---- IntegratedICPFactor(target_key, source_key, target, source) + set_max_correspondence_distance
 *      (manual_loop_close_modal.cpp:485-487), the target's KdTree being a point grid: the modal's fine registration of clouds
 *      without covariances (GICP falls back to it, with 200 LM iterations instead of 20, :479-492).  Neither cloud needs
 *      covariances: gb_point_grid_build takes a cloud without them (its records then hold zero covariances).
 *
 *      The rule.  The correspondence is exactly gb_gicp_grid_factor_create's: the same search half-width m (the same refusal
 *      above m = 8) and the same brute-force argmin of the fp32 d2 < (float)(r^2), ties to the smaller original index.  Per
 *      matched point the residual is the GICP grid factor's r = p - q with M = I: error = sum r^T r (no 1/2), and H and b are
 *      that factor's blocks with M = I.  error() takes its correspondences at T_lin and evaluates at T_eval.  [EXT] the
 *      un-vendored IntegratedICPFactor's error convention is this library's statement of it.
 *
 *      An ICP factor is an ordinary pose gb_factor: gb_vgicp_linearize / _error / _factor_destroy, gb_factor_set_*,
 *      gb_sweep_*, gb_vgicp_align and gb_gicp_grid_factor_half_width take it.  A sweep or call holds ICP factors only or none:
 *      a mix with VGICP or GICP factors of any target class is GB_ERR_INVALID_ARGUMENT before any launch.  ICP sweeps take no
 *      pair_index, slab or peer slab, and the gb_ct_* entry points refuse the factor.  gb_sweep_stats of an ICP sweep: 16 B per
 *      source point, 16 B per stored target point, 16 B per bucket of the smallest power-of-two table >= 16384 holding the
 *      cells, plus pose and record. ---- */
/* GB_ERR_INVALID_ARGUMENT before any launch, creating nothing, for a non-finite or non-positive max_correspondence_distance, a
 * target that is not a point grid, a grid or source on another device than ctx, or a search half-width m above 8. */
GB_API gb_status gb_icp_grid_factor_create(gb_ctx* ctx, const gb_point_grid* target, const gb_cloud* source, double max_correspondence_distance,
                                           gb_factor** out);

/* ---- Global registration: T_target_source between two clouds with no initial guess, as GLIM's manual loop closure runs it
 *      (ManualLoopCloseModal::align_global, src/glim/viewer/interactive/manual_loop_close_modal.cpp:370-468): FPFH features of
 *      both clouds (gtsam_points::estimate_fpfh, :382-397, :415), exact nearest-feature matching (the target's KdTreeX, :402)
 *      and RANSAC (gtsam_points::estimate_pose_ransac, :435-443).  Refine the result with a GICP factor on a point grid and
 *      gb_vgicp_align, the modal's fine registration (:470-520).  [EXT] gtsam_points is not vendored: the feature (PCL /
 *      Open3D's FPFH), the sample draw, the estimators and the selection rule below are this library's statement of it.
 *
 *      FPFH.  The neighbours of point i are every other point j with fp32 d2 = (dx^2 + dy^2) + dz^2 (uncontracted) <
 *      (float)(r^2): the brute-force set (no neighbour cap), found in a point grid of cell 1.05 r with the half-width
 *      grid_half_width proves.  Pair features in fp64 from the stored fp32 positions and normals, with d = p_j - p_i:
 *      |d| = 0 gives (0, 0, 0); the roles swap (n_s = n_j, n_t = n_i, d = -d, f3 = -n_j.d/|d|) when |n_i.d| < |n_j.d| (PCL's
 *      acos test on the cosines), else n_s = n_i, n_t = n_j, f3 = n_i.d/|d|; v = d x n_s (|v| = 0 gives (0, 0, 0)), v /= |v|,
 *      w = n_s x v, f2 = v.n_t, f1 = atan2(w.n_t, n_s.n_t).  Bins (Open3D): floor(11 (f1 + pi) / 2 pi), floor(11 (f2 + 1) / 2),
 *      floor(11 (f3 + 1) / 2), clamped to [0, 10] (NaN to 0), at offsets 0, 11, 22.  SPFH_i = (pairs of i in the bin) x
 *      (100 / K_i) for the K_i neighbours of i.  FPFH_i = A_b x 100 / (sum of A over b's 11-bin block) + SPFH_i,b with
 *      A_b = sum_j SPFH_j,b / d2_ij, d2_ij = d.d in fp64, neighbours at d2_ij = 0 skipped and a zero block sum scaling by 0
 *      (PCL and Open3D weight by the squared distance their radius search returns).  So every 11-bin block of a point with
 *      neighbours sums to 200 (100 if every neighbour coincides with it), and a point with no neighbours (a NaN point) is zero.
 *      fp64 throughout, stored once as fp32.  The SPFH counts do not depend on the visiting order; the fp64 sum A visits
 *      cells in offset order and a cell's points in ascending original index, so it may differ from an ascending-index sum in
 *      the last bits of fp64.
 *
 *      Matching.  nearest[i] = the target feature with the smallest fp32 d2 = (...((a_0 - b_0)^2 + (a_1 - b_1)^2) + ...) +
 *      (a_32 - b_32)^2, summed sequentially and uncontracted; ties to the smaller target index (the brute-force argmin of an exact
 *      KdTree); -1 when no distance is a number.  No ||a||^2 + ||b||^2 - 2 a.b shortcut: it would not give the exact argmin.
 *
 *      RANSAC, per hypothesis h = 0, 1, ...: s_j = rg_hash(seed, 3 h + j) mod N_s (j = 0, 1, 2; the hash of the random-grid
 *      pick), each paired with its match.  Invalid (counts -1) when two s_j coincide or a match is -1, or when the doubled area
 *      |(x_1 - x_0) x (x_2 - x_0)| of the source or the target triangle is below 1e-3 m^2 or not finite.  Pose in fp64 from the
 *      fp32 positions: dof 6 is Horn's quaternion (the eigenvector of the largest eigenvalue of his 4x4, from 8 cyclic Jacobi
 *      sweeps); dof 4 is yaw = atan2(sum a'_x b'_y - a'_y b'_x, sum a'_x b'_x + a'_y b'_y) over the centred points, R = Rz(yaw);
 *      both t = centroid_b - R centroid_a.  A source point is an inlier iff q = R a + t under the fp32 cast of the pose
 *      (((r0 a_x + r1 a_y) + r2 a_z) + t, uncontracted) is finite and keys (gb_coord at (float)(1 / inlier_voxel_resolution))
 *      into a cell of a point grid of the target at that resolution; inlier_rate = inliers / N_s.  The result is the lowest h
 *      with inlier_rate >= early_stop_inlier_rate (EARLY_STOP); else the h with the most inliers, ties to the lowest h (FOUND);
 *      DEGENERATE, T = I, best_hypothesis = -1 when no hypothesis has an inlier.  This is what a sequential loop with early stop
 *      returns, whatever the batching.  The device scores waves of 512 hypotheses and stops after the wave that holds the
 *      early stop: `evaluated` = the hypotheses scored (a multiple of 512, or max_iterations).
 *
 *      Launches: gb_cloud_estimate_fpfh, the point grid build's (gb_point_grid_build) + 2; gb_fpfh_match, 1 (0 for an empty
 *      source); gb_ransac_align, 1 (the match) + the target grid's build + 2 per wave, with one copy of the wave's counts and one
 *      stream synchronisation per wave. ---- */
/* ---- gtsam_points::estimate_normals(points, covs, n) (manual_loop_close_modal.cpp:391,410; map_editor.cpp:186): the normals of a
 *      cloud that has covariances but no normals (a merged submap, gb_merge_frames), before FPFH.
 *
 *      The rule.  Per point, from the stored fp32 position p and fp32 covariance (6 entries), both widened to fp64: n = the unit
 *      eigenvector of the smallest eigenvalue as eigen_sym3_direct computes it (the solver of the covariance estimation, so n
 *      agrees with gb_preprocess's normal on the same covariance); if (px nx + py ny) + pz nz > 0 (fp64, uncontracted) then
 *      n = -n (cloud_covariance_estimation.cpp:98-100); n is stored once as fp32.  A point whose position or covariance is not
 *      finite gets (0, 0, 0).  A finite covariance that is exactly zero or has a repeated smallest eigenvalue gets what the
 *      solver returns (for zero: the axis (1, 0, 0), sign-ruled).  [EXT] gtsam_points is not vendored: this is this library's
 *      statement of estimate_normals.
 *
 *      The normals go into the cloud's normals plane, in its stored order, so every consumer of normals reads them unchanged
 *      (gb_cloud_estimate_fpfh, GB_FACTOR_SURFACE_VALIDATION, gb_cloud_device_ptrs).  A cloud uploaded with normals has them
 *      overwritten in place; a cloud without gets a block of its own, which gb_cloud_destroy releases.  FPFH features computed
 *      earlier are discarded (gb_cloud_fpfh and the matchers refuse the cloud until they are estimated again).
 *      GB_ERR_INVALID_ARGUMENT before any launch for a cloud without covariances or on another device than ctx.  An empty
 *      cloud makes no launch; any other makes one launch and one stream synchronisation.  Threading as for gb_cloud_add_times:
 *      do not call it while another thread uses the cloud. ---- */
GB_API gb_status gb_cloud_estimate_normals(gb_ctx* ctx, gb_cloud* cloud);
/* host copy of the normals, N x 3 in the caller's point order; GB_ERR_INVALID_ARGUMENT for a non-empty cloud without normals */
GB_API gb_status gb_cloud_normals(const gb_cloud* cloud, float* out);
/* ---- Covariances and normals of a device cloud from its own k nearest neighbours: gtsam_points::estimate_covariances(points, n)
 *      of SubMap::load (sub_map.cpp:192-196, k = 10), the KdTree k-NN + CloudCovarianceEstimation::estimate of
 *      ManualLoopCloseModal::preprocess_maps (manual_loop_close_modal.cpp:338-356, k = 10, both outputs) and
 *      estimate_normals(points, n, k) of PointsSelector::select_points_segmentation (points_selector.cpp:785-787, k = 20).
 *
 *      The rule.  Points: the cloud's stored fp32 positions widened to fp64 (w = 1), in the caller's (original) order.
 *      Neighbours: gb_find_neighbors' rule at its 0.25 m finest cell (fp64 un-contracted d2, ties to the smaller index, the
 *      query included; the row of a non-finite point, or of a point whose cell leaves the 21-bit range, is itself k times).
 *      The k-NN is exact, so the cell size affects time only.  Covariance and normal: gb_covariances with k_correspondences =
 *      k_neighbors = k, i.e. CloudCovarianceEstimation::estimate with PLANE regularization and the sign rule of
 *      cloud_covariance_estimation.cpp:98-100.  Each value is stored once as fp32, exactly as gb_cloud_upload stores it.
 *      Postcondition: the cloud's planes, perm and inv_perm are bit-identical to a gb_cloud_upload of the widened positions,
 *      the computed covariances if GB_CLOUD_COVARIANCES is set (else the cloud's own) and the computed normals if
 *      GB_CLOUD_NORMALS is set (else the cloud's own).  Positions are never written, so the Morton order does not change.
 *      [EXT] gtsam_points is not vendored: estimate_covariances(points, n) is this rule with k = 10, and
 *      estimate_normals(points, n, k) is this rule's normal.
 *
 *      Side effects.  GB_CLOUD_COVARIANCES makes the cloud one with covariances: gb_gicp_grid_factor_create then accepts it as
 *      a source and gb_cloud_estimate_normals accepts it, and the factors that read a source's covariance planes
 *      (gb_vgicp_factor_create, gb_gicp_factor_create) read the estimated ones.  Covariances alone keep the normals and the
 *      FPFH features.  GB_CLOUD_NORMALS gives a cloud without normals a block of its own, as gb_cloud_estimate_normals does,
 *      and discards FPFH features.  Threading as for gb_cloud_estimate_normals: do not call it while another thread uses the
 *      cloud.
 *      GB_ERR_INVALID_ARGUMENT before any launch, changing nothing, for a null ctx or cloud, a cloud on another device than
 *      ctx, a k_neighbors that is not an instantiated k-NN count (1-10, 12, 15, 16, 20, 24, 32), outputs outside {1, 2, 3},
 *      or N * k_neighbors >= 2^30.
 *
 *      Launches: none for an empty cloud; any other makes 8 whatever N (k_cloud_gather_points: the stored planes into
 *      caller-order fp64 and the device count; the k-NN's 6; k_cloud_covariances: one pass that writes straight into the
 *      stored slots through inv_perm), then one stream synchronisation and no host transfer.  Scratch: per point 32 B of
 *      positions and 4 k B of neighbour rows, plus the k-NN's temporaries. ---- */
#define GB_CLOUD_COVARIANCES 1   /* sub_map.cpp:195 */
#define GB_CLOUD_NORMALS     2   /* points_selector.cpp:787; both = manual_loop_close_modal.cpp:351-353 */
GB_API gb_status gb_cloud_estimate_covariances(gb_ctx* ctx, gb_cloud* cloud, int k_neighbors, int outputs);
/* The FPFH features of `cloud` with search radius r, kept on the device with the cloud (cloud_destroy releases them); a second
 * call replaces them.  GB_ERR_INVALID_ARGUMENT before any launch for a cloud without normals, a non-finite or non-positive r,
 * or a cloud on another device than ctx. */
GB_API gb_status gb_cloud_estimate_fpfh(gb_ctx* ctx, gb_cloud* cloud, double search_radius);
/* host copy of the features, N x 33 in the caller's point order; GB_ERR_INVALID_ARGUMENT for a cloud without features */
GB_API gb_status gb_cloud_fpfh(const gb_cloud* cloud, float* out);
/* nearest[i] (N_s, the source's caller order) = the target index of source feature i's nearest target feature.  Both clouds
 * must carry features and live on ctx's device (GB_ERR_INVALID_ARGUMENT before any launch). */
GB_API gb_status gb_fpfh_match(gb_ctx* ctx, const gb_cloud* target, const gb_cloud* source, int32_t* nearest);
#define GB_RANSAC_FOUND 0
#define GB_RANSAC_EARLY_STOP 1
#define GB_RANSAC_DEGENERATE 2
typedef struct gb_ransac_params {
  int max_iterations;              /* 5000 (manual_loop_close_modal.cpp:47), in [1, 2^28] */
  double early_stop_inlier_rate;   /* 0.9 (:48); > 0, above 1 never stops early */
  double inlier_voxel_resolution;  /* 1.0 m (:49), > 0 */
  int dof;                         /* 4 (:50, global_registration_4dof) or 6 */
  uint64_t seed;                   /* 53123 (:42; the modal adds 4322 before each run) */
} gb_ransac_params;
typedef struct gb_ransac_result {
  double T_target_source[16];      /* column-major */
  double inlier_rate;
  int inliers, best_hypothesis, evaluated, status; /* GB_RANSAC_* */
} gb_ransac_result;
GB_API gb_status gb_ransac_default_params(gb_ransac_params* params);
/* hypothesis_inliers (max_iterations, or NULL): the inlier count of every evaluated hypothesis, -1 for an invalid sample, -2
 * for one not evaluated.  Validated before any launch: both clouds with features and at least one point, on ctx's device; the
 * parameter bounds above. */
GB_API gb_status gb_ransac_align(gb_ctx* ctx, const gb_cloud* target, const gb_cloud* source, const gb_ransac_params* params, gb_ransac_result* result,
                                 int32_t* hypothesis_inliers);

/* ---- GNC: the modal's other global method (gtsam_points::estimate_pose_gnc, manual_loop_close_modal.cpp:446-458), with its
 *      settings fixed as the modal fixes them (reciprocal_check = true, tuple_check = false).  [EXT] the rule below is this
 *      library's statement of it.
 *
 *      1. Samples, m = min(N_s, max_init_samples): every source index when N_s <= max_init_samples, else the m indices with the
 *      smallest rg_hash(seed, i) (the hash thinning of the random-grid pick; reference: an std::mt19937 shuffle), in ascending i.
 *      2. j(i) = the target feature nearest to sample i by gb_fpfh_match's rule.  3. Sample i keeps the pair (i, j(i)) iff j(i)
 *      >= 0, the source feature nearest to target feature j(i) over all N_s source features (same rule) is i, and both fp32
 *      positions are finite; pairs in ascending i, K of them.  K < 3: DEGENERATE, T = I, 0 iterations.
 *      4. Weighted closed form, fp64 from the fp32 positions (a source, b target), every operation rounded separately: once
 *      per call the shifts a_s = sum a / K, b_s = sum b / K; for weights w, W = sum w, p = sum w (a - a_s), q = sum w (b - b_s),
 *      M = sum w (a - a_s)(b - b_s)^T; c_a = a_s + p / W, c_b = b_s + q / W, S = M - p q^T / W; dof 6 Horn's rotation of S (as
 *      RANSAC's: 8 cyclic Jacobi sweeps), dof 4 R = Rz(atan2(S01 - S10, S00 + S11)); t = c_b - R c_a.
 *      5. Graduated non-convexity, Geman-McClure: r_k^2 = (e_x^2 + e_y^2) + e_z^2, e = b_k - (R a_k + t) (R a row by row as
 *      ((R0 a_x + R1 a_y) + R2 a_z)); T = pose(w = 1); mu = min(max(max_k r_k^2(T), 1 m^2), 1e3 m^2); then repeat: w_k =
 *      (mu / (mu + r_k^2(T)))^2, T = pose(w), iterations += 1, stop if mu == 1 m^2, else mu = max(mu / 1.4, 1 m^2).  At most 22
 *      iterations.  The reported weights are the last iteration's.
 *      6. inliers: RANSAC's inlier test of all N_s source points under T against a point grid of the target at 1.0 m (RANSAC's
 *      default inlier_voxel_resolution), inlier_rate = inliers / N_s, also for a DEGENERATE result (T = I).
 *
 *      Launches: the target grid's build (gb_point_grid_build at 1.0 m) + 7 (two matches, the gather of the matched target
 *      rows, the pair flags, the pair compaction, the solve, the score), + 5 when N_s > max_init_samples (the hash thinning's 3,
 *      the sample compaction, the gather of the sampled source rows).  One stream synchronisation, at the end. ---- */
#define GB_GNC_FOUND 0
#define GB_GNC_DEGENERATE 1
typedef struct gb_gnc_params {
  int max_init_samples;  /* 10000 (manual_loop_close_modal.cpp:52, gnc_max_samples), in [1, 2^28] */
  int dof;               /* 4 (:50, global_registration_4dof) or 6 */
  uint64_t seed;         /* 53123 (:42; the modal adds 4322 before each run) */
} gb_gnc_params;
typedef struct gb_gnc_result {
  double T_target_source[16];  /* column-major */
  double inlier_rate;
  int inliers, samples, correspondences, iterations, status; /* samples = m, correspondences = K; GB_GNC_* */
} gb_gnc_result;
GB_API gb_status gb_gnc_default_params(gb_gnc_params* params);
/* pairs (K x 2: source index, target index) and weights (K) may be NULL; their capacity is m = min(N_s, max_init_samples) rows,
 * of which the first K are written (a DEGENERATE result's weights are 0).  Validated before any launch: both clouds with
 * features and at least one point, on ctx's device; the parameter bounds above. */
GB_API gb_status gb_gnc_align(gb_ctx* ctx, const gb_cloud* target, const gb_cloud* source, const gb_gnc_params* params, gb_gnc_result* result, int32_t* pairs,
                              double* weights);

/* ---- NonlinearFactorSetGPU::add(graph) / ::linearize(values) (odometry_estimation_gpu.cpp:383-386;
 *      hook at src/glim/viewer/offline_viewer.cpp:29): F x 64 B of poses down, one launch over all
 *      factors, F records up. ---- */
GB_API gb_status gb_factor_set_linearize(gb_ctx* ctx, size_t num_factors, gb_factor* const* factors, const double* T_target_source /* F x 16 */, gb_linearized6* out /* F */);
GB_API gb_status gb_factor_set_error(gb_ctx* ctx, size_t num_factors, gb_factor* const* factors, const double* T_lin /* F x 16 */, const double* T_eval /* F x 16 */, double* errors /* F */);

/* ---- Scan registration: Levenberg-Marquardt on VGICP factors, many problems in one call
 *      (odometry_estimation_cpu.cpp:105-150: one unary IntegratedVGICPFactor(Pose3(), X(current), voxelmap, frame) per level,
 *      LevenbergMarquardtOptimizerExt; global_mapping_pose_graph.cpp:405-417: loop candidates, 10 iterations each).
 *      A problem is the set of factors (levels) that share one unknown T_target_source, the target pose fixed to identity;
 *      the factors of problem p are factors[factor_offsets[p] .. factor_offsets[p+1]).  Factors keep their flags.  The factors
 *      may be VGICP (gb_vgicp_factor_create), GICP on iVoxes (gb_gicp_factor_create) or GICP on point grids
 *      (gb_gicp_grid_factor_create) factors, or ICP factors on point grids (gb_icp_grid_factor_create), all of one class per call.
 *
 *      The rule (gtsam_points' LevenbergMarquardtOptimizerExt is not vendored: GTSAM's documented LM defaults plus GLIM's
 *      termination callback, DESIGN.md section 7 [EXT]).  Per problem, T = T_init, lambda = lambda_initial, need_lin = 1;
 *      while the problem is active:
 *        1. if need_lin: linearize every factor at T; H = sum H_ss, b = sum b_s, e = sum error, n = sum num_inliers
 *           (record order, fp64); iterations += 1.  n == 0 on the first linearization: stop, DEGENERATE, T = T_init.
 *        2. solve (H + lambda I) delta = -b by a 6x6 fp64 Cholesky (tangent [rot; trans]); a failed factorization is a
 *           rejected trial.  T' = T Exp(delta); trials += 1.
 *        3. e' = sum error(T_lin = T, T_eval = T') (inliers of T, residuals at T').
 *        4. e' < e: accept: T = T', lambda /= lambda_factor, need_lin = 1, then the first that holds:
 *             CONVERGED if |t(Exp(delta))| < step_translation_tol and |w| < step_rotation_tol, unless both are < 1e-10;
 *             CONVERGED if e - e' <= absolute_error_tol or (e - e') / e <= relative_error_tol;
 *             MAX_ITERATIONS if iterations >= max_iterations;
 *           and in every case e = e'.
 *        5. otherwise reject: lambda *= lambda_factor, need_lin = 0; LAMBDA_EXCEEDED if lambda > lambda_upper_bound.
 *      Each round is at most four launches for the whole batch (linearize sweep if any problem needs it, solve, error
 *      sweep, accept) and one small device-to-host copy; finished problems are swept until the whole batch has finished. ---- */
#define GB_ALIGN_CONVERGED 0
#define GB_ALIGN_MAX_ITERATIONS 1
#define GB_ALIGN_LAMBDA_EXCEEDED 2
#define GB_ALIGN_DEGENERATE 3
typedef struct gb_align_params {
  int max_iterations;          /* linearizations per problem (8: config_odometry_cpu.json:23; 10: global_mapping_pose_graph.cpp:412) */
  double lambda_initial;       /* 1e-5 (> 0) */
  double lambda_factor;        /* 10 (> 1) */
  double lambda_upper_bound;   /* 1e5 (finite) */
  double relative_error_tol;   /* 1e-5 */
  double absolute_error_tol;   /* 0.1 (odometry_estimation_cpu.cpp:118) */
  double step_translation_tol; /* 1e-3 m (odometry_estimation_cpu.cpp:135); <= 0 turns the step test off */
  double step_rotation_tol;    /* 1e-3 deg in rad (same line); <= 0 turns the step test off */
} gb_align_params;
typedef struct gb_align_result {
  double T_target_source[16];  /* column-major */
  double error;                /* error of the returned pose with the inliers of its last linearization (what LM holds) */
  double num_inliers;          /* of the last linearization (inlier_fraction = num_inliers / source size) */
  double lambda;
  int iterations, trials, status; /* GB_ALIGN_* */
} gb_align_result;
GB_API gb_status gb_align_default_params(gb_align_params* params); /* the odometry_estimation_cpu values above */
/* Every input is validated before any launch: offsets must start at 0 and increase strictly (no empty problem), no factor
 * may be NULL, T_init must be finite, and the parameters must satisfy the bounds above (and lambda_initial must not
 * underflow to 0 within max_iterations accepted steps). */
GB_API gb_status gb_vgicp_align(gb_ctx* ctx, size_t num_problems, const size_t* factor_offsets /* P + 1 */, gb_factor* const* factors,
                                const double* T_init /* P x 16 */, const gb_align_params* params, gb_align_result* results /* P */);

/* ---- Pose graphs: Levenberg-Marquardt over several world poses per problem, many problems in one call (sub_mapping.cpp:428-452:
 *      the submap optimization, a 1e8 prior on X(0) and VGICP factors between every pair of keyframes; global_mapping.cpp:393-426:
 *      a 1e6 prior on X(0) and a GICP factor; manual_loop_close_modal.cpp:476-517: a 1e6 prior on key 0 and GICP or ICP).
 *      Problem p has K_p = key_offsets[p+1] - key_offsets[p] keys (2 <= K_p <= GB_GRAPH_MAX_KEYS), their poses T_world_key in
 *      rows key_offsets[p] .. of T_init, the binary factors factors[factor_offsets[p] ..] on the problem-local keys
 *      factor_keys[2f] (target) and factor_keys[2f + 1] (source), and the priors prior_offsets[p] .. on the problem-local keys
 *      prior_keys[q] with poses Z_q (prior_poses, 16 each) and isotropic precisions w_q (prior_precisions).
 *
 *      The rule is gb_vgicp_align's above at 6K dof, with these differences:
 *        1. each factor is linearized at T_t^-1 T_s and its record is assembled into the 6K x 6K system in fp64: H_tt to block
 *           (t, t), H_ss to (s, s), H_ts to (t, s) and its transpose to (s, t), b_t to t and b_s to s; e and n sum the errors and
 *           inlier counts.  Every entry sums its contributions in record order.  Then each prior in prior order:
 *           r = Log(Z^-1 T_k), J = J_r^-1(r), H += w J^T J, b += w J^T r, e += w r^T r (no 1/2: priors weigh as
 *           gb_ct_gicp_align's).  DEGENERATE when the first linearization has no inlier.
 *        2. (H + lambda I) delta = -b by a 6K x 6K fp64 Cholesky (lambda on the whole diagonal); T_k' = T_k Exp(delta_k).  A key
 *           no factor or prior touches has delta_k = 0.
 *        3. e' = sum error(T_lin = T, T_eval = T') over the factors in record order, then each prior's term at T'.
 *        4. the step tests read the largest translation step and the largest rotation step over the keys.
 *      Each round is at most four launches for the whole batch (linearize sweep if any problem needs it, step, error sweep,
 *      accept) and one 8-byte device-to-host copy, whatever the number of problems.
 *      Validated before any launch: 2 <= K_p <= GB_GRAPH_MAX_KEYS; offsets that start at 0, factor offsets increasing strictly
 *      (a factor per problem), key and prior offsets not decreasing; factor keys in range with target != source; no NULL factor,
 *      all factors of one class of those gb_vgicp_align takes (CT and plane factors are refused) on ctx's device; finite
 *      poses; finite precisions >= 0; prior keys in range; the bounds of gb_align_params. ---- */
#define GB_GRAPH_MAX_KEYS 32
typedef struct gb_graph_result {
  double error;                /* of the returned poses, with the inliers of their last linearization, priors included */
  double num_inliers;          /* of the last linearization, summed over the factors */
  double lambda;
  int iterations, trials, status; /* GB_ALIGN_* */
} gb_graph_result;
GB_API gb_status gb_graph_optimize(gb_ctx* ctx, size_t num_problems, const size_t* key_offsets /* P + 1 */, const double* T_init /* (sum K) x 16 */,
                                   const size_t* factor_offsets /* P + 1 */, gb_factor* const* factors, const int32_t* factor_keys /* F x 2 */,
                                   const size_t* prior_offsets /* P + 1 */, const int32_t* prior_keys, const double* prior_poses /* x 16 */,
                                   const double* prior_precisions, const gb_align_params* params, double* T_out /* (sum K) x 16 */,
                                   gb_graph_result* results /* P */);

/* ---- Global maps: Levenberg-Marquardt over one graph of up to GB_POSE_GRAPH_MAX_KEYS poses (global_mapping.cpp:360-377 optimize,
 *      :285-351 find_overlapping_submaps, :546 save: the X(0) anchor, matching-cost factors between overlapping submaps and
 *      between factors; global_mapping_pose_graph.cpp: the X(0) anchor, odometry between factors and Huber loop factors).
 *      num_keys = K poses T_world_key in T_init; the binary factors on keys factor_keys[2f] (target), factor_keys[2f + 1]
 *      (source); the priors on prior_keys[q] with poses Z_q and isotropic precisions w_q; the between terms betweens[m].
 *
 *      The rule is gb_graph_optimize's above for one problem at 6K dof, with these additions:
 *        1. a between term on keys (i, j) with measurement Z, information L and Huber width k: r = Log(Z^-1 T_i^-1 T_j),
 *           J_j = J_r^-1(r), J_i = -J_r^-1(r) Ad((T_i^-1 T_j)^-1) (GTSAM's BetweenFactor<Pose3>); m = sqrt(r^T L r); the weight
 *           w = 1 if k == 0 or m <= k, else k / m (GTSAM's IRLS linearization, taken at the linearization poses).  It adds
 *           w J^T L J to blocks (i, i), (j, j), (i, j), (j, i) and w J^T L r to b; its error is 2 rho(m), rho Huber's loss
 *           (m^2 / 2 if m <= k, k m - k^2 / 2 otherwise), which is r^T L r without Huber: no 1/2, as the priors.  At trial poses
 *           the error is recomputed from r(T'), not with a frozen weight.
 *        2. every entry of H and b, and e, sums the factor records in record order, then the between terms in term order,
 *           then the priors in prior order.
 *        3. DEGENERATE only when F > 0 and the first linearization has no inlier; F = 0 with a between term is a pose graph.
 *           A key that nothing touches keeps delta_k = 0.
 *        4. (H + lambda I) delta = -b is solved densely: the system is padded to a multiple of 64 rows with unit diagonal and
 *           factored by a right-looking tiled Cholesky (64 x 64 fp64 tiles) without atomics, so two identical calls give
 *           bit-identical results.  A non-positive or non-finite pivot is a rejected trial.
 *      Each round is at most four launches whatever K, F or the number of between terms (linearize sweep when a linearization
 *      is needed and F > 0, step, error sweep when F > 0, accept) and one 8-byte device-to-host copy.  The context's scratch
 *      holds two (6K) x (6K) fp64 matrices: 302 MB each at K = 1024.
 *      Validated before any launch: 2 <= K <= GB_POSE_GRAPH_MAX_KEYS; F + num_betweens >= 1; factor, prior and between keys in
 *      range, factor and between keys with target != source; gb_graph_optimize's factor rules (no NULL factor, one class,
 *      no CT or plane factors, on ctx's device); finite poses and measurements; finite precisions >= 0; each information
 *      finite and exactly symmetric; huber_width finite and >= 0; the bounds of gb_align_params. ---- */
#define GB_POSE_GRAPH_MAX_KEYS 1024
typedef struct gb_between_term {
  int32_t key_i, key_j;   /* keys in [0, K), key_i != key_j */
  double Z[16];           /* the measured T_i^-1 T_j, column-major */
  double information[36]; /* L, symmetric, column-major */
  double huber_width;     /* k > 0: GTSAM's Huber on the whitened norm; 0: none */
} gb_between_term;
GB_API gb_status gb_pose_graph_optimize(gb_ctx* ctx, size_t num_keys, const double* T_init /* K x 16 */, size_t num_factors, gb_factor* const* factors,
                                        const int32_t* factor_keys /* F x 2 */, size_t num_priors, const int32_t* prior_keys, const double* prior_poses /* x 16 */,
                                        const double* prior_precisions, size_t num_betweens, const gb_between_term* betweens, const gb_align_params* params,
                                        double* T_out /* K x 16 */, gb_graph_result* result);

/* ---- IMU preintegration (imu_integration.cpp IMUIntegration::integrate_imu over GTSAM's PreintegratedImuMeasurements, tangent
 *      variant), many intervals in one call.  [EXT] GTSAM is not vendored: the tangent-space preintegration
 *      (TangentPreintegration::update / UpdatePreintegrated) and its exact theta-theta derivative are restated here.
 *
 *      Samples are rows (t, ax, ay, az, wx, wy, wz) with non-decreasing t.  Interval i has a start time, an end time and a bias
 *      b_hat = [acc; gyro]; its record starts from zero state, zero Jacobians and zero covariance, then:
 *        window: every sample with start < t <= end, in array order up to the first with t > end: dt = t - last (last starts at
 *          start); a sample with dt <= 0 is skipped, every other one is integrated and counted in num_integrated and last = t.
 *          Then, if end - last > 0, one more step of dt = end - last with the first sample after end, or the last sample when
 *          there is none.  An empty sample array integrates nothing.
 *        one step (a = a_meas - b_hat_a, w = w_meas - b_hat_g, [theta; p; v] the preintegrated vector, R = Exp(theta)):
 *          theta += J_r(theta)^-1 w dt, p += v dt + R a dt^2 / 2, v += R a dt (p with the old v), delta_t += dt;
 *          A = I_9 + [d(J_r(theta)^-1 w dt)/d theta in the theta-theta block, R [-a]x J_r(theta) dt^2 / 2 in p-theta,
 *              R [-a]x J_r(theta) dt in v-theta, I dt in p-v];  B = [0; R dt^2 / 2; R dt];  C = [J_r(theta)^-1 dt; 0; 0];
 *          H_bias_acc = A H_bias_acc - B, H_bias_omega = A H_bias_omega - C;
 *          covariance = A S A^T + B (acc_noise^2 I / dt) B^T + C (gyro_noise^2 I / dt) C^T, then its p-p block += int_noise^2 I dt
 *          (each entry computed once for its lower triangle and mirrored: the record is exactly symmetric).
 *      No Coriolis term and no body_P_sensor, as GLIM uses it.  One launch per call, one thread per interval, fp64.
 *      Validated before any launch: finite samples with non-decreasing times; finite intervals with start <= end; finite
 *      biases; finite noises >= 0 and a finite gravity. ---- */
typedef struct gb_imu_params {
  double acc_noise;  /* accelerometer noise density: 0.05 (config_sensors.json) */
  double gyro_noise; /* 0.02 */
  double int_noise;  /* integration noise: 0.001 */
  double gravity[3]; /* (0, 0, -9.81): PreintegrationParams::MakeSharedU */
} gb_imu_params;
typedef struct gb_imu_preintegrated {
  double delta_t;
  double preintegrated[9]; /* [theta; p; v] */
  double H_bias_acc[27];   /* 9 x 3, row-major */
  double H_bias_omega[27]; /* 9 x 3, row-major */
  double covariance[81];   /* preintMeasCov, 9 x 9, row-major, symmetric */
  double bias_hat[6];      /* [acc; gyro] */
  double gravity[3];
  int32_t num_integrated;
  int32_t pad;
} gb_imu_preintegrated;
GB_API gb_status gb_imu_default_params(gb_imu_params* params);
GB_API gb_status gb_imu_preintegrate(gb_ctx* ctx, size_t num_samples, const double* samples /* S x 7 */, size_t num_intervals,
                                     const double* intervals /* I x 2: start, end */, const double* biases /* I x 6 */, const gb_imu_params* params,
                                     gb_imu_preintegrated* out /* I */);

/* ---- Navigation graphs: gb_pose_graph_optimize with velocities, IMU biases and IMU factors (global_mapping.cpp:166-218 with
 *      enable_imu: the X / E / V / B variables of every submap; sub_mapping.cpp:218-243: X / V / B per odometry frame).
 *      K_X poses T_world_key (T_init), K_V velocities (v_init, 3 each) and K_B biases [acc; gyro] (b_init, 6 each); keys are
 *      per kind, from 0.  The factors, priors and between terms are gb_pose_graph_optimize's, on pose keys.
 *
 *      An IMU term (GTSAM's ImuFactor, PreintegrationBase::computeError) on (pose_i, vel_i, pose_j, vel_j, bias_i) and a
 *      preintegrated record p: delta = p.preintegrated + H_bias_acc (b_a - p.bias_hat_a) + H_bias_omega (b_g - p.bias_hat_g);
 *      R^_j = R_i Exp(delta_theta), p^_j = p_i + v_i dt + g dt^2 / 2 + R_i delta_p, v^_j = v_i + g dt + R_i delta_v (dt, g the
 *      record's delta_t and gravity); r = [Log(R_j^T R^_j); R_j^T (p^_j - p_j); R_j^T (v^_j - v_j)]; error r^T S^-1 r with S
 *      the record's covariance (no 1/2, as every term here).
 *      A vector term with isotropic precision w and error w r^T r:
 *        GB_VECTOR_VELOCITY_PRIOR (key_a a velocity) r = v - z;  GB_VECTOR_BIAS_PRIOR (key_a a bias) r = b - z;
 *        GB_VECTOR_VELOCITY_BETWEEN / GB_VECTOR_BIAS_BETWEEN (key_a != key_b of that kind) r = (x_b - x_a) - z;
 *        GB_VECTOR_ROTATE_VELOCITY (key_a a pose, key_b a velocity) r = R_a z - v_b.  [EXT] gtsam_points' RotateVector3Factor is
 *        not vendored; under an isotropic precision its error equals that of the other sign convention.
 *      z holds 3 (velocities, rotate) or 6 (biases, [acc; gyro]) entries.
 *
 *      The rule is gb_pose_graph_optimize's, with these differences:
 *        1. every variable fills a 6-dof slot, poses first, then velocities, then biases; a velocity uses the first three dofs
 *           of its slot, the other three are pinned as the padding is (unit diagonal, zero right-hand side, step 0).
 *        2. Jacobians are taken in the solver's charts and the retraction is T' = T Exp(delta), v' = v + delta, b' = b + delta;
 *           the step tests read the pose slots only.
 *        3. every entry of H and b, and e, sums the factor records in record order, then the between terms, then the IMU terms,
 *           then the vector terms (each in term order), then the priors: a call without velocities, biases, IMU and vector terms
 *           sums exactly as gb_pose_graph_optimize.
 *      Each round is at most four launches, as gb_pose_graph_optimize's.  The context's scratch holds two (6 slots)^2 fp64
 *      matrices: 1.21 GB each at GB_NAV_GRAPH_MAX_SLOTS.
 *      Validated before any launch: K_X >= 1, 2 <= K_X + K_V + K_B <= GB_NAV_GRAPH_MAX_SLOTS; F + betweens + IMU + vector terms
 *      >= 1; every key of its kind and in range, the two poses and the two velocities of an IMU term distinct, the two keys of a
 *      between vector term distinct, a known vector kind; finite inputs; each record's delta_t > 0 and its covariance exactly
 *      symmetric and positive definite under an fp64 Cholesky; finite precisions >= 0; everything gb_pose_graph_optimize
 *      validates. ---- */
#define GB_NAV_GRAPH_MAX_SLOTS 2048
typedef struct gb_imu_term {
  int32_t pose_i, vel_i, pose_j, vel_j, bias_i, pad;
  gb_imu_preintegrated pim;
} gb_imu_term;
#define GB_VECTOR_VELOCITY_PRIOR 0
#define GB_VECTOR_BIAS_PRIOR 1
#define GB_VECTOR_VELOCITY_BETWEEN 2
#define GB_VECTOR_BIAS_BETWEEN 3
#define GB_VECTOR_ROTATE_VELOCITY 4
typedef struct gb_vector_term {
  int32_t kind;         /* GB_VECTOR_* */
  int32_t key_a, key_b; /* key_b unused by a prior */
  int32_t pad;
  double z[6];
  double precision;     /* w >= 0 */
} gb_vector_term;
GB_API gb_status gb_nav_graph_optimize(gb_ctx* ctx, size_t num_poses, const double* T_init /* K_X x 16 */, size_t num_velocities,
                                       const double* v_init /* K_V x 3 */, size_t num_biases, const double* b_init /* K_B x 6 */, size_t num_factors,
                                       gb_factor* const* factors, const int32_t* factor_keys /* F x 2 */, size_t num_priors, const int32_t* prior_keys,
                                       const double* prior_poses /* x 16 */, const double* prior_precisions, size_t num_betweens,
                                       const gb_between_term* betweens, size_t num_imu_terms, const gb_imu_term* imu_terms, size_t num_vector_terms,
                                       const gb_vector_term* vector_terms, const gb_align_params* params, double* T_out /* K_X x 16 */,
                                       double* v_out /* K_V x 3 */, double* b_out /* K_B x 6 */, gb_graph_result* result);

/* ---- Continuous-time GICP: GLIM's LiDAR-only odometry (OdometryEstimationCT, src/glim/odometry/odometry_estimation_ct.cpp,
 *      config/config_odometry_ct.json) on the device: the time table of a frame (:101), IntegratedCT_GICPFactor_<iVox,
 *      PointCloud>(X, Y, ivox, frame, ivox) with max_correspondence_distance (:159-163) and the Levenberg-Marquardt solve with
 *      the two motion priors (:166-182).  X is the pose at the scan's first time-table entry, Y at its last.
 *      [EXT] gtsam_points is not vendored: the time table, the interpolation, the error convention and the weighting of the
 *      objective below are this library's statement of the un-vendored factor, written from GLIM's call site.
 *
 *      The time table (PointCloud::add_times).  The points are walked in their original order; a point opens a new entry iff
 *      its time exceeds the current entry's time by more than time_eps = 1e-3 s; an entry's time t_b is the time of its first
 *      point and every point takes the time of its entry.  tau_b = (t_b - t_0) / (t_{B-1} - t_0), or 0 when B == 1.  So Y is
 *      the pose at the LAST ENTRY's time, which may precede the last point's time by up to time_eps.
 *
 *      The factor.  With xi = Log(X^-1 Y), the pose of entry b is T_b = X Exp(tau_b xi) (Pose3 Expmap chart, tangent
 *      [rot; trans], perturbations on the right).  Each point is matched exactly as by gb_gicp_factor_create, with the fp32
 *      cast of its entry's pose as the lookup transform; residual, M and error as there: r = q - T_b p,
 *      M = (C_q + R_b C_p R_b^T)^-1, error = sum r^T M r (no 1/2); error() takes the correspondences at (X_lin, Y_lin) and
 *      evaluates at (X_eval, Y_eval).  Per entry, (H_b, b_b) are the blocks the GICP factor's record holds as H_ss / b_s at the
 *      pose T_b; they are chained to (X, Y) in fp64, entry by entry, by
 *        D0_b = Ad(Exp(-tau_b xi)) - tau_b J_r(tau_b xi) J_r^-1(xi) Ad(Y^-1 X),   D1_b = tau_b J_r(tau_b xi) J_r^-1(xi),
 *        H = sum_b [D0_b D1_b]^T H_b [D0_b D1_b],   b = sum_b [D0_b D1_b]^T b_b
 *      (J_r the SE(3) right Jacobian; exact, the pose being constant within an entry).  The 12x12 system goes into a
 *      gb_linearized6 with X IN THE TARGET SLOT and Y IN THE SOURCE SLOT: H_tt = H_XX, H_ss = H_YY, H_ts = H_XY (rows X),
 *      b_t = b_X, b_s = b_Y; so gb_hessian_blocks yields HessianFactor(X, Y, ...) unchanged.
 *
 *      A CT factor is a gb_factor of its own kind, destroyed by gb_vgicp_factor_destroy.  gb_vgicp_linearize, gb_vgicp_error,
 *      gb_factor_set_*, gb_sweep_create and gb_vgicp_align refuse it, and the gb_ct_* entry points refuse every other factor,
 *      with GB_ERR_INVALID_ARGUMENT before any launch; these refusals are the only change of behaviour of earlier entry points.
 *      A CT factor reads its source's time table at every call: do not set times while another thread uses the factor. ---- */
/* The time table of `cloud` from its n times (the cloud's original point order), built on the host and stored with the cloud
 * on the device (entry starts and tau_b; t_0 and t_{B-1} on the host as well); setting times again replaces it.  Validated
 * before any launch: times finite and non-decreasing, n equal to the cloud's size (>= 1), the cloud on ctx's device.
 * Every consumer of clouds other than the CT factor ignores the table. */
GB_API gb_status gb_cloud_add_times(gb_ctx* ctx, gb_cloud* cloud, size_t n, const double* times);
/* host copy of a cloud's time table: B, starts (B + 1, original indices), tau (B), t_0, t_{B-1}; any pointer may be NULL.
 * B = 0 for a cloud without times. */
GB_API gb_status gb_cloud_time_table(const gb_cloud* cloud, int* num_entries, int32_t* starts, double* tau, double* t_first, double* t_last);
/* The source must carry times (and covariances, as for GICP); the target must be an iVox. */
GB_API gb_status gb_ct_gicp_factor_create(gb_ctx* ctx, const gb_ivox* target, const gb_cloud* source, double max_correspondence_distance, gb_factor** out);
/* Two launches: the sweep over the work items and the per-problem chain rule. */
GB_API gb_status gb_ct_gicp_linearize(gb_factor* factor, const double X[16], const double Y[16], gb_linearized6* out);
GB_API gb_status gb_ct_gicp_error(gb_factor* factor, const double X_lin[16], const double Y_lin[16], const double X_eval[16], const double Y_eval[16], double* error);

/* The per-frame solve (odometry_estimation_ct.cpp:159-182), many problems in one call.  Problem p has one CT factor and the
 *      objective  E(X, Y) = e_ct(X, Y) + l |Log(X_prior^-1 X)|^2 + c |Log(X^-1 Y)|^2
 *      (l = location_consistency_inf_scale, c = constant_velocity_inf_scale; PriorFactor(X, last_T_world_lidar_end) and
 *      BetweenFactor(X, Y, identity) with isotropic precisions).  The small terms carry no 1/2 because the CT error carries
 *      none: the relative weight GTSAM gives HessianFactor(H, -b, e) next to a NoiseModelFactor.  Their Jacobians are
 *      J_r^-1(e), and -J_r^-1(e) Ad(Y^-1 X) for X in the between term.  The CT error takes the inliers of the linearization
 *      poses.
 *      The iteration rule is gb_vgicp_align's at 12 dof: (H + lambda I) delta = -b by a 12x12 fp64 Cholesky, trial poses
 *      X Exp(delta_X), Y Exp(delta_Y), the same accept, reject and termination steps (the step tests read the larger of the
 *      two poses' steps), DEGENERATE when the first linearization has no inliers.
 *      Each round is at most four launches for the whole batch (linearize sweep if any problem needs it, step, error sweep,
 *      accept) and one 8-byte device-to-host copy, whatever the number of problems. */
typedef struct gb_ct_params {
  gb_align_params lm;                     /* max_iterations 8 (lm_max_iterations), lambda_initial 1e-10, absolute_error_tol 1e-2,
                                             relative_error_tol 1e-5, lambda_factor 10, lambda_upper_bound 1e5, step tests off (<= 0) */
  double location_consistency_inf_scale;  /* 1e-3 (config_odometry_ct.json:25) */
  double constant_velocity_inf_scale;     /* 1e3  (config_odometry_ct.json:26; the code default at :44 is 1e-3) */
} gb_ct_params;
typedef struct gb_ct_result {
  double X[16], Y[16];                    /* column-major */
  double error, num_inliers, lambda;      /* as gb_align_result; error = the objective E */
  int iterations, trials, status;         /* GB_ALIGN_* */
} gb_ct_result;
GB_API gb_status gb_ct_default_params(gb_ct_params* params);
/* Validated before any launch: CT factors on ctx's device, finite poses, the bounds of gb_vgicp_align's parameters, finite
 * non-negative precisions. */
GB_API gb_status gb_ct_gicp_align(gb_ctx* ctx, size_t num_problems, gb_factor* const* factors /* P CT factors */, const double* X_init /* P x 16 */,
                                  const double* Y_init /* P x 16 */, const double* X_prior /* P x 16: last_T_world_lidar_end */,
                                  const gb_ct_params* params, gb_ct_result* results /* P */);
/* The deskewed frame (factor->deskewed_source_points(values, true) and the covariance re-estimation of
 * odometry_estimation_ct.cpp:199-204): every point becomes Exp(tau_b xi) p (= X^-1 T_b p) in fp64, computed from the cloud's fp32
 * position; covariances and normals are then re-estimated from the deskewed points with the caller's neighbour indices by
 * gb_preprocess's covariance stage (plane_covariance).  Outputs, each n x ... in the original point order, or NULL: points
 * (n x 4, w = 1), covariances (n x 16, column-major) and normals (n x 4); out_cloud: a new device cloud of the deskewed frame
 * with its covariances and normals, ready for gb_ivox_insert(ivox, cloud, X, 1, seed); it carries no times.
 * Validated before any launch as gb_covariances: 1 <= k_neighbors <= k_correspondences, the first k_neighbors indices of every
 * row in [0, n); X and Y finite; a source with times on ctx's device. */
GB_API gb_status gb_ct_deskew(gb_ctx* ctx, const gb_cloud* source, const double X[16], const double Y[16],
                              const int32_t* neighbors /* n x k_correspondences, original order, as gb_preprocess returns them */,
                              int k_correspondences, int k_neighbors, double* out_xyzw, double* out_cov4x4, double* out_normals4, gb_cloud** out_cloud);

/* ---- Solver hand-off (SURVEY A.3; global_mapping.cpp:492-501 feeds these to isam2->update): the blocks of
 *      gtsam::HessianFactor(k_t, k_s, G11 = H_tt, G12 = H_ts, g1 = -b_t, G22 = H_ss, g2 = -b_s, f = error_scale * error),
 *      6x6 blocks column-major, from one factor record or from one fp32 row of the pair slab (levels pre-summed on the
 *      device).  Host-only helpers (no device needed); for a unary factor use G22 / g2 / f. ---- */
GB_API gb_status gb_hessian_blocks(const gb_linearized6* lin, double error_scale, double* G11 /*36*/, double* G12 /*36*/, double* g1 /*6*/, double* G22 /*36*/, double* g2 /*6*/, double* f);
GB_API gb_status gb_slab_row_hessian_blocks(const float* slab_row /* GB_SLAB_STRIDE */, double error_scale, double* G11, double* G12, double* g1, double* G22, double* g2, double* f, double* num_inliers);

/* Prepared batch: the same sweep with its descriptor table resident on the device, split into
 * upload / launch / fetch so that callers (the bench, the multi-GPU sweep) can keep everything in HBM.
 *   pair_index (may be NULL): factor -> row of a caller-owned fp32 slab [num_pairs][GB_SLAB_STRIDE];
 *   when a slab is attached the kernel epilogue ADDS each factor's blocks to its pair row
 *   (levels of the same pair sum there), which is the buffer the multi-GPU sweep all-reduces
 *   over NCCL (SURVEY 8(e)).  Slab row: H_tt upper(21) H_ts(36, column-major) H_ss upper(21) b_t(6) b_s(6)
 *   error num_inliers, padded to GB_SLAB_STRIDE floats. */
GB_API gb_status gb_sweep_create(gb_ctx* ctx, size_t num_factors, gb_factor* const* factors, const int32_t* pair_index, gb_sweep** out);
GB_API gb_status gb_sweep_destroy(gb_sweep* sweep);
GB_API gb_status gb_sweep_attach_slab(gb_sweep* sweep, void* device_slab_f32, size_t num_pairs);
GB_API gb_status gb_sweep_set_poses(gb_sweep* sweep, const double* T_target_source /* F x 16, host */); /* async H2D */
GB_API gb_status gb_sweep_launch(gb_sweep* sweep);                                /* async: the fused kernel */
GB_API gb_status gb_sweep_fetch(gb_sweep* sweep, gb_linearized6* out /* F */);     /* D2H + stream sync */
/* set_poses + launch + fetch in one call; small sweeps run it as one CUDA-graph launch (poses H2D -> kernel -> records D2H) */
GB_API gb_status gb_sweep_linearize(gb_sweep* sweep, const double* T_target_source /* F x 16 */, gb_linearized6* out /* F */);
GB_API gb_status gb_sweep_results_device(gb_sweep* sweep, void** device_ptr);     /* F x 122 doubles in HBM */
/* bookkeeping for the roofline: sum of N_source, and algorithmic bytes B_sweep of SURVEY 8(d) */
GB_API gb_status gb_sweep_stats(const gb_sweep* sweep, uint64_t* point_factors, uint64_t* algorithmic_bytes, uint32_t* num_tiles, uint32_t* grid_size);

/* ---- Multi-GPU result exchange (SURVEY 8(e); no reference counterpart: GLIM is single-GPU).
 *      A gb_peer_slab is a pair of fp32 buffers [num_pairs][GB_SLAB_STRIDE] (ping-pong by step parity) plus completion
 *      flags, allocated with cudaMalloc and shared with the other ranks of the box through CUDA IPC.  When one is attached
 *      to a sweep (ONE sweep per slab), the epilogue of the LAST factor of every pair sums the pair's factor records in fp64
 *      and stores the finished row -- up to 4 ranks straight into EVERY rank's buffer over NVLink (fused push), above 4 ranks
 *      into this rank's buffer only (deferred push: stores to peer memory from the busy SMs slow the sweep down at 8
 *      ranks, DESIGN.md section 8).  gb_peer_slab_signal_wait() launches the kernel that (deferred push only: four CTAs per
 *      peer) copies the rank's rows into that peer's buffer, publishes this rank's completion flag and waits for the peers'.
 *      Each pair is owned by exactly one rank, so the "all-reduce" is an all-gather done by the producers.  No NCCL call, no
 *      memset, no float atomics (rows are deterministic).  With world == 1 it is simply the deterministic way to get the
 *      pair slab.  GB_PEER_PUSH=fused|deferred in the environment forces one variant. ---- */
#define GB_IPC_HANDLE_BYTES 64
typedef struct gb_peer_slab gb_peer_slab;
GB_API gb_status gb_peer_slab_create(gb_ctx* ctx, size_t num_pairs, int world, int rank, gb_peer_slab** out);
GB_API gb_status gb_peer_slab_export(gb_peer_slab* slab, void* handle /* GB_IPC_HANDLE_BYTES */);
GB_API gb_status gb_peer_slab_connect(gb_peer_slab* slab, const void* handles /* world x GB_IPC_HANDLE_BYTES, rank order */);
GB_API gb_status gb_peer_slab_destroy(gb_peer_slab* slab);
GB_API gb_status gb_sweep_attach_peer_slab(gb_sweep* sweep, gb_peer_slab* slab);
/* after gb_sweep_launch: publish completion of this step to every peer, wait (on the stream) until every peer has published */
GB_API gb_status gb_peer_slab_signal_wait(gb_peer_slab* slab);
/* the buffer completed by the last gb_peer_slab_signal_wait: device pointer / copy to host (D2H + stream sync) */
GB_API gb_status gb_peer_slab_device_ptr(gb_peer_slab* slab, void** device_ptr);
GB_API gb_status gb_peer_slab_fetch(gb_peer_slab* slab, float* host /* num_pairs x GB_SLAB_STRIDE */);
/* same copy into the slab's own pinned host buffer, WITHOUT synchronizing: valid after the next synchronization of the
 * context's stream (e.g. gb_sweep_fetch); *host_ptr receives the pinned buffer */
GB_API gb_status gb_peer_slab_fetch_async(gb_peer_slab* slab, const float** host_ptr);

/* ---- overlap_gpu(voxelmap, source, delta, stream) / overlap_gpu(voxelmaps, source, deltas, stream) /
 *      overlap_auto (odometry_estimation_gpu.cpp:231,248,265,279; sub_mapping.cpp:252; global_mapping.cpp:322,448):
 *      fraction of source points that fall in an occupied voxel of any target ---- */
GB_API gb_status gb_overlap(gb_ctx* ctx, size_t num_targets, const gb_voxelmap* const* targets, const gb_cloud* source, const double* deltas /* T x 16 */, double* overlap);

/* ---- GlobalMapping::find_overlapping_submaps (src/glim/mapping/global_mapping.cpp:285-351) and the overlap test of
 *      GlobalMapping::create_matching_cost_factors (:441-453): every candidate pair of S submaps gated, counted and
 *      thresholded in one call.  maps[k] is submap k's coarsest level (voxelmaps.back()), sources[k] the cloud its overlap is
 *      measured for (subsampled_submaps[k]), T_world_submap S x 16 column-major.
 *   - Candidates: the pairs (i, j) with i < j and j >= first_source that are not in `existing` (E x 2 (i, j) pairs that
 *     already have a factor).  The lookup is ordered, as the reference's set lookup is: an entry (j, i) does not exclude
 *     (i, j).  first_source 0 is find_overlapping_submaps; S - 1 is create_matching_cost_factors for the newest submap.
 *   - Delta: delta = T_i^-1 T_j in fp64, R = R_i^T R_j and t = R_i^T t_j + (-(R_i^T t_i)), as Eigen's Isometry3d::inverse() * T;
 *     every dot product is summed in index order ((a0 b0 + a1 b1) + a2 b2) with no FMA contraction.
 *   - Distance gate: a candidate is kept iff (t0 t0 + t1 t1) + t2 t2 <= max_distance * max_distance.
 *   - Overlap: count / n_j, exactly as gb_overlap(ctx, 1, &maps[i], sources[j], delta, &overlap) computes it (the same fp32
 *     cast of delta, NaN skip and lookup; 0 for an empty source), and so bit-identical to that call.
 *   - Output: every candidate with overlap >= min_overlap, in lexicographic (i, j) order (the order of both reference loops);
 *     min_overlap = 0 returns every gated pair.  The first min(found, capacity) results go to pairs (capacity x 2: i, j) and
 *     overlaps; *num_found is the full count, as with snprintf.  capacity = 0 with NULL arrays is allowed.
 *   - GB_ERR_INVALID_ARGUMENT before any launch unless ctx, num_found, maps, sources and T_world_submap are non-NULL,
 *     1 <= S <= GB_OVERLAP_SEARCH_MAX_SUBMAPS, first_source < S, the poses are finite, max_distance is finite and >= 0,
 *     min_overlap is finite, existing is non-NULL when E > 0 and its keys are in [0, S), pairs and overlaps are non-NULL
 *     when capacity > 0, and every map and source is non-NULL, on ctx's device and no map is a point grid.
 *   - Cost: 8 launches (4 kernels around k_overlap, gb_overlap's kernel, and 3 cub calls), whatever S and the number of
 *     candidates; none for S = 1, which has no pair.  One upload (descriptors, poses and the S x S exclusion bitmap) and at
 *     most two downloads: the count, then the pairs and overlaps.
 *   - Size: any cloud gb_cloud_upload accepts, at any distance bound.  The work (one item per pair and 256 source points)
 *     is counted in 64 bits, so a search whose pairs probe more than 2^31 x 256 points is not refused and is not cut short.
 *   - Scratch: N = S (S - 1) / 2 - first_source (first_source - 1) / 2 candidate slots (8.4 M at S = 4096), 68 bytes each
 *     (570 MB at S = 4096, 36 MB at S = 1024), plus S x 208 bytes and S^2 / 8 bytes of bitmap (2 MB at S = 4096).  The
 *     context's scratch keeps that size until it is destroyed. ---- */
#define GB_OVERLAP_SEARCH_MAX_SUBMAPS 4096
GB_API gb_status gb_find_overlapping_submaps(gb_ctx* ctx, size_t num_submaps, const gb_voxelmap* const* maps, const gb_cloud* const* sources,
                                             const double* T_world_submap /* S x 16 */, size_t first_source, size_t num_existing,
                                             const int32_t* existing /* E x 2 */, double max_distance, double min_overlap, size_t capacity,
                                             size_t* num_found, int32_t* pairs /* capacity x 2 */, double* overlaps /* capacity */);

/* ---- CloudCovarianceEstimation::estimate(points, neighbors, k, normals, covs) with PLANE regularization
 *      (src/glim/common/cloud_covariance_estimation.cpp:43-122, :181-196).  GB_ERR_INVALID_ARGUMENT, before any launch,
 *      unless 1 <= k_neighbors <= k_correspondences and the first k_neighbors indices of every row are in [0, n) ---- */
GB_API gb_status gb_covariances(gb_ctx* ctx, size_t n, const double* xyzw, const int32_t* neighbors, int k_correspondences, int k_neighbors, double* normals4, double* cov4x4);

/* ---- CloudPreprocessor::find_neighbors (src/glim/preprocess/cloud_preprocessor.cpp:190-221): exact k-NN,
 *      query included, row-major neighbors[i*k + j].  k in {1-10, 12, 15, 16, 20, 24, 32}, else GB_ERR_INVALID_ARGUMENT
 *      before any launch (the same set for k_correspondences and outlier_removal_k of gb_preprocess).  The search is
 *      gb_preprocess's grid pyramid with knn_cell_size 0.25 m: a point that is not finite, or whose 0.25 m cell lies outside
 *      the 21-bit range (a coordinate outside [-262144, 262144) m), gets a row of its own index and is no point's neighbour,
 *      at every cloud size ---- */
GB_API gb_status gb_find_neighbors(gb_ctx* ctx, size_t n, const double* xyzw, int k, int32_t* neighbors);

/* ---- gtsam_points::voxelgrid_sampling (cloud_preprocessor.cpp:108): one point per voxel = mean of
 *      points / times / intensities, ascending packed-key order.  out arrays sized n; *num_out = count ---- */
GB_API gb_status gb_voxelgrid_sampling(gb_ctx* ctx, size_t n, const double* xyzw, const double* times, const double* intensities, double resolution, double* out_xyzw, double* out_times, double* out_intensities, size_t* num_out);

/* ---- The whole per-frame preprocess in one call, kept on the device (SURVEY 8(b) gb_preprocess):
 *      glim::CloudPreprocessor::preprocess_impl (src/glim/preprocess/cloud_preprocessor.cpp:92-188: voxel-grid :108 or
 *      random-grid :104-106 downsampling, finite + range gate :116-128, time order :135-136, global shutter :138-140,
 *      crop box :143-162, k-NN :182-183) fused with glim::CloudCovarianceEstimation::estimate
 *      (src/glim/common/cloud_covariance_estimation.cpp:43-122, called at src/glim/odometry/odometry_estimation_imu.cpp:322-328)
 *      and PointCloudGPU::clone (odometry_estimation_gpu.cpp:96): one H2D of the raw scan, no host round trip between the
 *      stages, the fp32 planes of the resulting gb_cloud written by the covariance kernel.  Host products (the
 *      PreprocessedFrame fields, fp64 covariances / normals) are copied back only for the pointers that are not NULL.
 *      Statistical outlier removal (:165-167; gtsam_points::remove_outliers [EXT]): d_i = mean distance to the k nearest
 *      neighbours (query included); keep i iff d_i < mean(d) + std_mul * stddev(d) (population variance).
 *      Random grid: which points of a voxel survive is a draw from std::mt19937 in the reference (not reproducible); here it
 *      is the ceil(rate N / V) points with the smallest hash(seed, index) -- same count per voxel, a fixed pseudo-random pick. ---- */
typedef struct gb_preprocess_params {
  double distance_near_thresh, distance_far_thresh; /* config_preprocess.json:20-21 */
  int use_random_grid_downsampling;                 /* config_preprocess.json:22 */
  double downsample_resolution;                     /* <= 0: no downsampling */
  int downsample_target;                            /* > 0: rate = target / N (cloud_preprocessor.cpp:105) */
  double downsample_rate;
  uint64_t seed;                                    /* random grid */
  int global_shutter;
  int crop_bbox_frame;                              /* 0 = off, 1 = "lidar", 2 = "imu" */
  double crop_bbox_min[3], crop_bbox_max[3];
  double T_imu_lidar[16];                           /* column-major; used by crop_bbox_frame == 2 */
  int enable_outlier_removal;                       /* config_preprocess.json:26 */
  int outlier_removal_k;                            /* 10 */
  double outlier_std_mul_factor;                    /* code default 2.0 (cloud_preprocessor.cpp:36), shipped config 1.0 */
  int k_correspondences;                            /* k of the k-NN (10) */
  int estimate_covariances;                         /* fuse CloudCovarianceEstimation + the device cloud */
  int k_neighbors_cov;                              /* neighbours used by the covariance (<= k_correspondences; 0 = all) */
  double knn_cell_size;                             /* finest cell of the k-NN grid pyramid, metres (0 = 0.25) */
} gb_preprocess_params;
typedef struct gb_preprocessed {
  size_t num_points;     /* out */
  double last_time;      /* out: times.back() (scan_end_time = stamp + last_time, cloud_preprocessor.cpp:174) */
  double* times;         /* caller-allocated for n_raw entries, or NULL */
  double* xyzw;          /* n_raw x 4 */
  double* intensities;   /* n_raw */
  int32_t* neighbors;    /* n_raw x k */
  double* normals4;      /* n_raw x 4  (estimate_covariances) */
  double* cov4x4;        /* n_raw x 16 (estimate_covariances) */
  gb_cloud* cloud;       /* out: the frame as a device cloud (points + covariances + normals), or NULL; destroy with gb_cloud_destroy */
} gb_preprocessed;
GB_API gb_status gb_preprocess_default_params(gb_preprocess_params* params); /* config/config_preprocess.json + CloudPreprocessorParams defaults */
GB_API gb_status gb_preprocess(gb_ctx* ctx, size_t n_raw, const double* xyzw, const double* times, const double* intensities, const gb_preprocess_params* params, gb_preprocessed* out);

/* ---- gtsam_points::merge_frames(poses, frames, downsample_resolution, target_num_points) as SubMapping::create_submap calls
 *      it (src/glim/mapping/sub_mapping.cpp:481-497; `merge_frames_gpu` is what the reference wanted at :491): transform the
 *      keyframes' DEVICE clouds by T_origin_keyframe (points and covariances R C R^T), voxel-grid average points and
 *      covariances, thin to target_num_points (<= 0: no thinning).  Outputs: the merged submap as a device cloud and / or as
 *      host arrays (N x Vector4d, N x Matrix4d column-major, capacity = sum of the frames' sizes).  fp64 sums in
 *      (frame, original point index) order. ---- */
GB_API gb_status gb_merge_frames(gb_ctx* ctx, size_t num_frames, const gb_cloud* const* frames, const double* poses /* K x 16 */, double downsample_resolution, int target_num_points, uint64_t seed,
                                 double* out_xyzw, double* out_cov4x4, size_t* num_out, gb_cloud** out_cloud);

/* ---- The map editor's world-frame cloud (PointsSelector::update_cells / collect_neighbor_point_ids / collect_submap_points,
 *      src/glim/viewer/editor/points_selector.cpp:85-177) and GlobalMapping::export_points (global_mapping.cpp:638-680): the
 *      submaps' DEVICE clouds transformed by T_world_submap and concatenated into one device cloud, optionally only the points
 *      whose cell lies in a window.
 *
 *      The rule.  Per point a of frame k with covariance C and normal n, at pose (R, t): q = R a + t and C' = R C R^T exactly
 *      as gb_merge_frames transforms them (un-contracted fp64, the same association order, the same kernel), n' = R n with
 *      row r as (R_r0 nx + R_r1 ny) + R_r2 nz (fp64, not renormalised); each value is stored once as fp32.  The result carries
 *      covariances iff every frame does (else they are zero) and normals iff every frame does (the editor assumes all submaps
 *      alike, :118-122); zero frames give neither.  With a window, a point is kept iff k = floor(q * (1.0 / cell_size)) (fp64,
 *      per axis, on the fp64 q before it is stored) satisfies lo <= k <= hi on every axis; a non-finite q is never kept.  The
 *      editor keys its fp64 submap points; here q comes from the frames' stored fp32 positions widened to fp64, so a point
 *      within an ulp of a cell face may land in the neighbouring cell.  Without a window every point is kept, NaN included.
 *      Output order: frame-major, then ascending original index; ids[i] = (frame << 32) | original index, the editor's point id
 *      (:84, :139-140).  Zero frames, or nothing kept, give an empty cloud.
 *
 *      GB_ERR_INVALID_ARGUMENT before any launch for a non-finite pose entry, a frame on another device than ctx, a non-finite
 *      or non-positive cell_size, lo > hi on any axis, a frame of 2^32 points or more, or 2^30 points or more in all.
 *      Launches: 4 (the shared frame transform, the window flags, their scan, the emit) + 3 (gb_cloud_build's Morton reorder)
 *      = 7; 4 when nothing is kept; none when the frames hold no point.  Two stream synchronisations (the kept count, the end).
 *      ---- */
typedef struct gb_cell_window {
  double cell_size;    /* m, > 0 (the editor's map_cell_resolution) */
  int32_t lo[3], hi[3]; /* inclusive cell bounds per axis (the editor: centre -/+ cell_selection_window) */
} gb_cell_window;
/* poses: K x 16 column-major T_world_frame; window NULL = every point; ids: capacity the sum of the frames' sizes, or NULL */
GB_API gb_status gb_concat_frames(gb_ctx* ctx, size_t num_frames, const gb_cloud* const* frames, const double* poses, const gb_cell_window* window,
                                  gb_cloud** out_cloud, uint64_t* ids, size_t* num_out);

/* ---- gtsam_points::region_growing_init / region_growing_update (points_selector.cpp:798-810; docs/edit.md "Plane selection
 *      and removal"): the connected surface through a picked point of a cloud with normals, and its dilation.  [EXT]
 *      gtsam_points is not vendored: the rule below is this library's statement of region growing.
 *
 *      The rule.  Distances are the fp32 point_d2 = (dx^2 + dy^2) + dz^2 (d = p_j - p_i, uncontracted) of the stored
 *      positions.  Points i != j are joined iff both are finite, point_d2 < (float)(distance_threshold^2) and
 *      (nx_i nx_j + ny_i ny_j) + nz_i nz_j >= cos(angle_threshold) (the dot in fp64 from the fp32 normals, each operation
 *      rounded; cos in fp64; signed; a NaN dot never joins).  The joins are found in a point grid of the cloud at cell
 *      1.05 distance_threshold with the half-width grid_half_width proves, as FPFH's neighbours are; a point whose key at a
 *      grid's cell leaves the 21-bit range takes part in no search of that grid.  labels[i] = the smallest original index of
 *      i's connected component for a finite point, -1 for a non-finite one; num_components = the number of distinct labels
 *      >= 0.  The seed is the finite point with the smallest point_d2 to (float)seed_point, ties to the smaller original index
 *      (region_growing_init's nearest-point query); without one, status NO_SEED, seed -1 and nothing selected (labels are
 *      still written).  The region R = {i : labels[i] == labels[seed]}.  With dilation_radius > 0, the dilation adds every
 *      finite j outside R for which some i in R has point_d2(i, j) < (float)(dilation_radius^2): the brute-force set, found in
 *      a point grid of the cloud at cell 1.05 dilation_radius (with the same key-range rule).  selected = R plus the added
 *      points in ascending original index; num_region = |R|, num_selected = |selected|.  The result is a set: it does not
 *      depend on the order the device visits points in.
 *
 *      GB_ERR_INVALID_ARGUMENT before any launch for a non-empty cloud without normals, a cloud on another device than ctx, a
 *      non-finite seed_point, or parameters outside the bounds below.  An empty cloud makes no launch.  Launches: the point
 *      grid builds (gb_point_grid_build at 1.05 distance_threshold, and at 1.05 dilation_radius when it is > 0) + 4 (the
 *      parents and the seed, the hooks, the labels and the region, the compaction of the selection) + 1 with dilation: the
 *      same for every size and shape of the graph.  Then one copy and one stream synchronisation. ---- */
#define GB_REGION_FOUND 0
#define GB_REGION_NO_SEED 1
typedef struct gb_region_growing_params {
  double distance_threshold; /* m, finite, > 0 (editor UI: 0.01-1 m) */
  double angle_threshold;    /* rad, in [0, pi] (UI: 0.01-180 deg) */
  double dilation_radius;    /* m, finite, >= 0; 0 = no dilation (UI: 0.01-100 m) */
} gb_region_growing_params;
typedef struct gb_region_growing_result {
  int32_t seed;   /* original index, -1 for none */
  int32_t status; /* GB_REGION_* */
  size_t num_region, num_selected, num_components; /* before / after dilation; components over finite points */
} gb_region_growing_result;
/* this library's defaults, chosen for a LiDAR map at about 0.1-0.5 m spacing (not gtsam_points' values): 0.5 m, 10 deg, 0 */
GB_API gb_status gb_region_growing_default_params(gb_region_growing_params* params);
/* selected: capacity N, ascending original index (the first num_selected written), or NULL; labels: N in the caller's point
 * order, or NULL */
GB_API gb_status gb_region_growing(gb_ctx* ctx, const gb_cloud* cloud, const double seed_point[3], const gb_region_growing_params* params,
                                   gb_region_growing_result* result, int32_t* selected, int32_t* labels);

/* ---- gtsam_points::min_cut (points_selector.cpp:774-796, the editor's default segmentation; docs/edit.md "Object selection
 *      and removal"): the object around a picked point of a cloud with normals, cut from its surroundings by a minimum s-t
 *      cut.  [EXT] gtsam_points is not vendored: the rule below is this library's statement of min-cut segmentation.
 *
 *      The rule.  Positions and normals are the cloud's stored fp32 values; c = picked_point; fp64 d2 = (dx^2 + dy^2) + dz^2,
 *      each operation rounded.
 *      1. Participants: the finite points with d2(p, c) < (background_mask_radius + 1)^2 (the editor's filter, :777-783),
 *         numbered as nodes in ascending original index.  Other points take no part, not even as neighbours.
 *      2. Seed: the participant with the smallest fp32 point_d2 to (float)c, ties to the smaller index (gb_region_growing's
 *         seed rule).  With no participant: status NO_SEED, seed -1, nothing selected, no solve.
 *      3. Roles of the other participants: foreground if d2(p, c) < foreground_mask_radius^2, background if
 *         d2(p, c) > background_mask_radius^2, free otherwise.
 *      4. Edges: N(i) is participant i's row of the k_neighbors nearest participants by gb_find_neighbors' rule (fp64 d2,
 *         ties to the smaller index, the query included), with i itself dropped; a participant whose 0.25 m cell leaves the
 *         21-bit range has an empty row and is in no row.  {i, j} is an edge iff j in N(i) or i in N(j), of weight
 *         w = exp(-d2 / (2 distance_sigma^2)) * exp(-theta^2 / (2 angle_sigma^2)), theta = acos(min(|n_i . n_j|, 1)) with the
 *         dot (x + y) + z in fp64 from the fp32 normals (blind to a normal's sign); a NaN dot or a zero normal gives w = 0.
 *         Capacity q = (int32)floor(w * 65536), the same both ways.
 *      5. Network: source s = the seed, sink t = every background participant contracted (both hard); each edge is a pair of
 *         arcs of capacity q; each foreground participant has an arc s -> i of capacity floor(foreground_weight * 65536);
 *         free participants have no terminal arc.
 *      6. Cut: selected = the seed plus every participant reachable from s in the residual graph of a maximum s-t flow: the
 *         intersection of the source sides of all minimum cuts, unique whatever algorithm finds the flow, so ties between
 *         equal cuts resolve to the smallest object.  cut_value = the flow value, in units of 2^-16.  Background points are
 *         never selected; a point joined to the seed only by zero-capacity edges is not selected unless its foreground arc
 *         is not saturated.
 *      The flow is found by synchronous push-relabel with the roles swapped (the background is the source and the seed the
 *      sink), with a global relabel every 16 rounds; its rounds are bit-deterministic.  Beyond 65536 rounds the status is
 *      NOT_CONVERGED, with nothing selected and cut_value 0.  The transcendental weights may differ from another libm's by
 *      an ulp, and so a capacity by 1; edges and capacities (may be NULL) return the graph the cut was taken on: num_edges
 *      rows {i, j} of original indices, i < j, ascending, and their capacities.
 *
 *      GB_ERR_INVALID_ARGUMENT before any launch for null arguments, a cloud on another device than ctx, a non-empty cloud
 *      without normals, a non-finite picked_point, parameters outside the bounds below, or N * k_neighbors >= 2^30.  An empty
 *      cloud makes no launch.  Launches: 3 (participant flags and the seed, their scan, the nodes and their roles) + 6 (the
 *      k-NN) + 6 (the arcs, their sort, the unique flags, their scan, the CSR, the reverse arcs and capacities) + 1 (the
 *      cooperative solve) + 1 (the compaction of the selection) = 17, for every size and shape, NO_SEED included (its kernels
 *      find no node and return).  Then one copy and one stream synchronisation.  The work and scratch scale with the cloud's
 *      N (2 N k_neighbors arc slots), not with the participants: pass a window of the map, as the editor does. ---- */
#define GB_MINCUT_FOUND 0
#define GB_MINCUT_NO_SEED 1
#define GB_MINCUT_NOT_CONVERGED 2
typedef struct gb_min_cut_params {
  double distance_sigma;         /* m, finite, > 0: 0.25 (this library's) */
  double angle_sigma;            /* rad, in (0, pi]: 10 deg (this library's) */
  double foreground_mask_radius; /* m, finite, > 0: 0.5 (points_selector.cpp:43) */
  double background_mask_radius; /* m, finite, > foreground_mask_radius: 5.0 (:44) */
  double foreground_weight;      /* in [0, 1000]: 10 (:42) */
  int k_neighbors;               /* an instantiated k-NN count (1-10, 12, 15, 16, 20, 24, 32): 20 (this library's) */
} gb_min_cut_params;
typedef struct gb_min_cut_result {
  int32_t seed, status; /* original index (-1 for none); GB_MINCUT_* */
  size_t num_points, num_foreground, num_background, num_edges, num_selected; /* participants, their roles, undirected edges */
  int64_t cut_value;    /* the maximum flow, in units of 2^-16 */
  int32_t rounds;       /* push-relabel rounds (diagnostic; deterministic) */
} gb_min_cut_result;
/* 0.25 m, 10 deg, 0.5 m, 5.0 m, 10, 20 */
GB_API gb_status gb_min_cut_default_params(gb_min_cut_params* params);
/* selected: capacity N, ascending original index, or NULL.  edges (capacity N * k_neighbors rows of 2 original indices i < j,
 * ascending) and capacities (same rows) may be NULL: the graph the cut was taken on. */
GB_API gb_status gb_min_cut(gb_ctx* ctx, const gb_cloud* cloud, const double picked_point[3], const gb_min_cut_params* params,
                            gb_min_cut_result* result, int32_t* selected, int32_t* edges, int32_t* capacities);

/* ---- The map editor's gizmo tool over the whole map (PointsSelector::select_points_tool, points_selector.cpp:623-674): the
 *      points of K device clouds (submaps in their local frames, poses T_world_submap K x 16 column-major) inside the gizmo's
 *      box or sphere.
 *
 *      The rule.  T_local_world (16 doubles, column-major) is the inverse of the gizmo's model matrix, which the caller
 *      computes (:630).  Per frame, on the host in fp64: M_k = T_local_world T_world_submap_k, entry (r, c) for c < 3 as
 *      (A_r0 B_0c + A_r1 B_1c) + A_r2 B_2c and the translation as ((A_r0 B_03 + A_r1 B_13) + A_r2 B_23) + A_r3, each
 *      operation rounded (A = T_local_world, B = the pose, whose bottom row is taken as (0, 0, 0, 1) as in every posed frame
 *      list).  A stored fp32 point a, widened to fp64, becomes q = M_k a by gb_merge_frames' transform (row r as
 *      ((M_r0 a_x + M_r1 a_y) + M_r2 a_z) + M_r3, un-contracted).  GB_GIZMO_BOX selects it iff -0.5 < q_r < 0.5 on every axis
 *      (strict); GB_GIZMO_SPHERE iff (q_x^2 + q_y^2) + q_z^2 < 1, each operation rounded.  A NaN is never selected.  For an
 *      affine model matrix the editor's 0 < w < 2 test always holds.  The editor transforms its fp64 host points, this
 *      library the stored fp32 ones: a point within about 1e-7 relative of a face may fall on the other side.
 *      ids: (k << 32) | original index, frame-major and ascending (gb_concat_frames' editor ids), capacity the sum of the
 *      frames' sizes, or NULL; num_selected the count.
 *
 *      GB_ERR_INVALID_ARGUMENT before any launch for null arguments, a frame on another device than ctx, a non-finite pose,
 *      a non-finite T_local_world entry, a T_local_world whose bottom row is not exactly (0, 0, 0, 1), an unknown shape, a
 *      frame of 2^32 points or more, or 2^30 points or more in all.  Launches: 4 (the shared frame transform, the inside
 *      flags, their scan, the emit: gb_plane_patch's selection); none when the frames hold no point.  One stream
 *      synchronisation (the count), and a second one when ids are asked for and some point is selected. ---- */
#define GB_GIZMO_BOX 0
#define GB_GIZMO_SPHERE 1
GB_API gb_status gb_select_gizmo(gb_ctx* ctx, size_t num_frames, const gb_cloud* const* frames, const double* poses, const double T_local_world[16],
                                 int32_t shape, uint64_t* ids, size_t* num_selected);

/* ---- The map editor's two radius tools (PointsSelector::select_points_radius and select_outlier_points_radius,
 *      points_selector.cpp:677-759) on a device cloud, typically the window gb_concat_frames returns, as gb_min_cut takes it;
 *      callers map the selection to editor ids with ids[selected].
 *
 *      The rule.  c = center; d2 = (dx^2 + dy^2) + dz^2 in fp64 of the stored fp32 position widened to fp64 and c, each
 *      operation rounded (gb_min_cut's d2).  The editor measures its fp64 host points: a point within about 1e-7 relative of
 *      a radius may fall on the other side.
 *      INSIDE: the finite points with d2 < radius^2, in ascending original index.
 *      OUTLIERS ([EXT] gtsam_points::find_inlier_points is not vendored: this is the editor's call as this library states it):
 *      1. Participants: the finite points with d2 < (radius + radius_offset)^2, in ascending original index.
 *      2. Fewer than k participants: status NOT_ENOUGH_POINTS, nothing selected (the editor returns, :730-733).
 *      3. Each participant's k nearest participants by gb_find_neighbors' rule (fp64 d2, ties to the smaller index, the query
 *         included; a participant whose 0.25 m cell leaves the 21-bit range has itself k times in its row and is in no row).
 *      4. d_i = (sum of the k fp64 distances sqrt(d2) in row order, nearest first) / k: gb_preprocess's outlier-removal rule.
 *      5. threshold = mean + stddev_thresh * sqrt(max(var, 0)) with mean = S / m, var = S2 / m - mean^2 (population), each
 *         operation rounded, over the m participants' sums S = sum d_i and S2 = sum d_i^2.  The sums are cub's DeviceReduce
 *         over the cloud's N slots (0 beyond the participants), whose order depends on N and the device only: the same inputs
 *         give the same bits.  An inlier has d_i < threshold.
 *      6. Selected: the participants with d2 < radius^2 that are not inliers (:746-752), in ascending original index.
 *      k must be an instantiated k-NN count (1-10, 12, 15, 16, 20, 24, 32); the editor's UI allows up to 100.
 *
 *      GB_ERR_INVALID_ARGUMENT before any launch for null arguments, a cloud on another device than ctx, a non-finite center,
 *      parameters outside the bounds below, or, for OUTLIERS, N * k >= 2^30.  An empty cloud makes no launch.  Launches:
 *      INSIDE 2 (the flags, the compaction) and one stream synchronisation; OUTLIERS 3 (the flags, their scan, the nodes),
 *      one stream synchronisation (the participant count), then, with at least k participants, 6 (the k-NN) + 1 (the mean
 *      distances) + 2 (the sums) + 1 (the outlier flags) + 1 (the compaction) and a second synchronisation.  selected:
 *      capacity N, or NULL; its first num_selected entries are the selection, the others are unspecified. ---- */
#define GB_RADIUS_INSIDE 0
#define GB_RADIUS_OUTLIERS 1
#define GB_RADIUS_OK 0
#define GB_RADIUS_NOT_ENOUGH_POINTS 1
typedef struct gb_select_radius_params {
  double radius;          /* m, finite, > 0: 2.0 (points_selector.cpp:34) */
  double radius_offset;   /* m, finite, >= 0: 1.0 (:35), OUTLIERS only */
  double stddev_thresh;   /* finite: 2.0 (:37), OUTLIERS only */
  int32_t mode;           /* GB_RADIUS_INSIDE (default) or GB_RADIUS_OUTLIERS */
  int32_t k;              /* an instantiated k-NN count: 10 (:36), OUTLIERS only */
} gb_select_radius_params;
typedef struct gb_select_radius_result {
  int32_t status;           /* GB_RADIUS_* */
  size_t num_participants;  /* OUTLIERS: the participants; INSIDE: 0 */
  size_t num_selected;
  double threshold;         /* OUTLIERS with enough participants: the inlier threshold; NaN otherwise */
} gb_select_radius_result;
/* 2.0 m, 1.0 m, 2.0, INSIDE, 10 */
GB_API gb_status gb_select_radius_default_params(gb_select_radius_params* params);
GB_API gb_status gb_select_radius(gb_ctx* ctx, const gb_cloud* cloud, const double center[3], const gb_select_radius_params* params,
                                  gb_select_radius_result* result, int32_t* selected);

/* ---- Remove selected points (PointsSelector::remove_selected_points, points_selector.cpp:513-620) from K device clouds:
 *      ids are editor ids (frame << 32) | original index, the frame being the position in this list (gb_concat_frames'
 *      ids), in any order, duplicates allowed.
 *
 *      The rule.  An id whose frame is >= K or whose index is >= that frame's size is ignored and counted (the editor warns
 *      and skips it; its check at :549 misses index == size, this one does not).  Every frame that loses at least one point
 *      gets a NEW cloud in out_clouds[k]: its survivors in their original relative order, renumbered 0..n'-1
 *      (gtsam_points::sample with ascending indices, :544-561); a frame that loses nothing gets NULL and the caller keeps its
 *      handle.  The input clouds are never modified: factors, voxel maps and grids built from them stay valid.  A new cloud
 *      carries the stored fp32 positions, covariances iff the frame has them, and normals iff the frame has them (uploaded or
 *      from gb_cloud_estimate_normals; the new cloud keeps them in its own block), each value copied bit for bit.  It does
 *      NOT carry the frame's time table or FPFH features, which depend on the removed points: recompute them with
 *      gb_cloud_add_times and gb_cloud_estimate_fpfh.  A frame that loses every point becomes an empty cloud.
 *      A cloud's storage order is a stable sort on the Morton key of each stored fp32 position with the original index as
 *      the tie-break, so the survivors, taken in stored order, are already in the order gb_cloud_upload of the survivors
 *      would store them: the removal is a compaction in stored order with no re-sort, and a new cloud is bit-identical, planes,
 *      perm and inv_perm, to an upload of its survivors' downloaded values.
 *      result: num_removed = distinct points removed, num_ignored, num_changed = frames given a new cloud.  sizes (K, or NULL):
 *      every frame's size after the removal.
 *
 *      GB_ERR_INVALID_ARGUMENT before any launch for null arguments, a frame on another device than ctx, a frame of 2^32
 *      points or more, or touched frames of 2^30 points or more in all.  No launch when no id is valid.  Otherwise the work
 *      and scratch scale with the touched frames, not the map, and the launches are 5 whatever K and num_ids: the marks of
 *      the removed points, their scan in original order, the marks in stored order (through inv_perm) with each frame's
 *      removed count, their scan, and one emit over every touched frame into the new clouds' blocks (one pool block per
 *      non-empty new cloud, laid out as gb_cloud_upload's).  Two uploads (the ids and the touched frames' table, then the new
 *      clouds' table), one stream synchronisation for the removed counts and one at the end: the new clouds are complete
 *      when the call returns. ---- */
typedef struct gb_remove_points_result {
  size_t num_removed, num_ignored, num_changed;
} gb_remove_points_result;
/* out_clouds: K entries, each a new cloud or NULL */
GB_API gb_status gb_remove_points(gb_ctx* ctx, size_t num_frames, const gb_cloud* const* frames, size_t num_ids, const uint64_t* ids, gb_cloud** out_clouds,
                                  gb_remove_points_result* result, size_t* sizes);

/* ---- The interactive viewer's plane bundle adjustment (src/glim/viewer/interactive/bundle_adjustment_modal.cpp:37-60,
 *      :137-245; interactive_viewer.cpp:393, :412-418): the submap points around a right-clicked point, their covariance's
 *      eigenvalues (Update), the modal's radius search (Auto Radius), and the gtsam_points::PlaneEVMFactor made of them
 *      (Create Factor), which global mapping's iSAM2 then relinearizes.
 *
 *      Inputs of the three patch calls: K device clouds (submaps, in their local frame), poses T_k = (R_k, t_k) (K x 16
 *      doubles, column-major, T_world_submap) and the parameters below, whose `center` c is the picked point (fp64).
 *
 *      Selection (set_frames, extract_points).
 *      1. Frame k takes part iff sqrt((u_x^2 + u_y^2) + u_z^2) <= max_frame_distance for u = t_k - c (the modal skips a submap
 *         whose norm is > 25).
 *      2. A stored fp32 point a of a participating frame is widened to fp64 and transformed as q = R_k a + u, row r as
 *         ((R_r0 a_x + R_r1 a_y) + R_r2 a_z) + u_r, un-contracted: gb_merge_frames' transform at the pose [R_k | t_k - c], the
 *         modal's Translation(-center) * pose.
 *      3. The point is selected iff (q_x^2 + q_y^2) + q_z^2 < radius * radius, both sides fp64; a NaN never is.
 *      4. Selected ids are (k << 32) | original index, frame-major and ascending: gb_concat_frames' editor ids.
 *      5. The modal keys its fp64 host points, this library the stored fp32 ones: a point within about 1e-7 relative of the
 *         sphere may fall on the other side (the caveat of gb_concat_frames).
 *
 *      Patch statistics (calc_eigenvalues).  Over the n selected points in fp64: s = sum q, S = sum q q^T, mean = s / n,
 *      Cov(r, c) = (S(r, c) - mean_r s_c) / n for r <= c, mirrored; the eigenvalues, ascending, from eigen_sym3_direct (the
 *      modal's computeDirect, the solver of the covariance estimation).  n == 0 gives NaN eigenvalues (the modal's 0 / 0).  The
 *      sums are taken in a fixed order that depends on the candidates only: the same inputs give the same bits.
 *
 *      Auto radius (exactly the modal's loop, :186-227):
 *          r = radius; (n, ev) = stats(r)                      no size check on this first extraction
 *          for i in 0..9:
 *              trial = ev[0] / ev[2] > plane_eps ? r * 0.8 : r * 1.1        a NaN ratio grows
 *              if trial < min_radius or trial > max_radius: break
 *              (n', ev') = stats(trial)                        recorded as trial i: (trial, n')
 *              if n' < 10: break
 *              if trial > radius and ev'[0] / ev'[2] > plane_eps: break     `radius` is the starting radius
 *              r, n, ev = trial, n', ev'
 *          result: r, n, ev (what update_indicator then shows) and the trials.
 *
 *      The factor (Create Factor, :229-245).  The selection at `radius` gives the keys: the participating frames with at least
 *      one selected point, in the caller's frame order.  Per key, from its selected stored local points a widened to fp64:
 *      N_k, the mean m_k and the scatter S_k = sum (a - m_k)(a - m_k)^T (two passes, fixed order).  The factor keeps the
 *      offset o = c, which keeps world coordinates far from the origin out of the fp64 sums (the error does not depend on it).
 *      [EXT] gtsam_points is not vendored: the error e = lambda_0 (not N lambda_0), the exact Hessian and the record convention
 *      below are this library's statement of PlaneEVMFactor.
 *        Error at the key poses X_k: p_i = X_k a_i - o, pbar = mean p, C = (1/N) sum (p_i - pbar)(p_i - pbar)^T with ascending
 *        eigenpairs (lambda_m, u_m), e = lambda_0.  It is evaluated from the moments,
 *        C = (1/N) sum_k [R_k S_k R_k^T + N_k (q_k - pbar)(q_k - pbar)^T], q_k = R_k m_k + t_k - o, which is algebraically the
 *        definition, so a linearization costs O(K^2) whatever the point count.  C is decomposed by eigen_sym3_direct.
 *        Linearization along the chart X_k Exp(xi_k), xi_k = [omega; nu] (GTSAM Pose3 Expmap): b = (1/2) de/dxi (6K) and
 *        H = (1/2) d2e/dxi2 (6K x 6K, dense, column-major), the exact Hessian at xi = 0, including the term of the second-order
 *        expansion of Exp.  So e(xi) ~ e + 2 b^T xi + xi^T H xi, the relation of every gb_linearized6 record:
 *        HessianFactor(keys, G = H, g = -b, f = e) hands it to GTSAM as gb_hessian_blocks does for the other factors.
 *        Status DEGENERATE iff !(lambda_1 - lambda_0 > 0): then H = 0, b = 0 and e = lambda_0 (a repeated lambda_1 = lambda_2
 *        is fine).
 *
 *      Every input is validated before any launch (GB_ERR_INVALID_ARGUMENT, nothing created): null arguments, a non-finite
 *      pose or centre, a frame on another device than ctx, a frame of 2^32 points or more or 2^30 in all, and parameters
 *      outside the bounds below.  Launches (none when the participating frames hold no point):
 *        gb_plane_patch:             4 (the shared frame transform, the sphere flags, their scan, the emit) + 1 (the reduction);
 *                                    one stream synchronisation, and a second one when ids are asked for and n > 0.
 *        gb_plane_auto_radius:       4 (the selection at max(radius, max_radius)) + 1 per evaluated radius (1 + num_trials);
 *                                    one stream synchronisation per evaluated radius.
 *        gb_plane_evm_factor_create: 4 (the selection at radius, with the local points) + 1 (the per-key moments); one stream
 *                                    synchronisation.  Fewer than 3 selected points is GB_ERR_INVALID_ARGUMENT after these
 *                                    launches, and creates nothing (the modal would build a factor whose error is NaN).
 *      ---- */
#define GB_PLANE_MAX_TRIALS 10
#define GB_PLANE_EVM_OK 0
#define GB_PLANE_EVM_DEGENERATE 1
typedef struct gb_plane_patch_params {
  double center[3];          /* the picked point; finite */
  double radius;             /* m, finite, > 0: 1.0 (the modal's) */
  double max_frame_distance; /* m, >= 0, +inf allowed: 25.0 */
  double min_radius;         /* m, finite, 0 < min_radius <= max_radius: 0.1 */
  double max_radius;         /* m, finite: 5.0 */
  double plane_eps;          /* finite, >= 0: 0.01 */
} gb_plane_patch_params;
typedef struct gb_plane_patch_result {
  double radius;                                  /* the radius the statistics are taken at */
  size_t num_points;                              /* n */
  double eigenvalues[3];                          /* ascending; NaN for n == 0 */
  int32_t num_trials;                             /* gb_plane_auto_radius: evaluated trials (<= 10); 0 otherwise */
  double trial_radius[GB_PLANE_MAX_TRIALS];       /* in evaluation order */
  size_t trial_points[GB_PLANE_MAX_TRIALS];
} gb_plane_patch_result;
/* the modal's defaults: centre 0, 1.0, 25.0, 0.1, 5.0, 0.01 */
GB_API gb_status gb_plane_patch_default_params(gb_plane_patch_params* params);
/* Update: n and the eigenvalues at params->radius; ids (capacity the sum of the frames' sizes, or NULL) the selected ids */
GB_API gb_status gb_plane_patch(gb_ctx* ctx, size_t num_frames, const gb_cloud* const* frames, const double* poses, const gb_plane_patch_params* params,
                                gb_plane_patch_result* result, uint64_t* ids);
/* Auto Radius: the returned radius with n and the eigenvalues there, and the trial path */
GB_API gb_status gb_plane_auto_radius(gb_ctx* ctx, size_t num_frames, const gb_cloud* const* frames, const double* poses, const gb_plane_patch_params* params,
                                      gb_plane_patch_result* result);
/* Create Factor: uses center, radius and max_frame_distance.  The factor keeps K x 10 doubles on the host: it borrows no
 * cloud (its frames may be destroyed afterwards) and owns no device memory; gb_vgicp_factor_destroy frees it.  Every other
 * factor entry point (gb_vgicp_linearize, gb_vgicp_error, gb_factor_set_*, gb_sweep_create, gb_vgicp_align, gb_ct_*) refuses
 * it with GB_ERR_INVALID_ARGUMENT before any launch, and the gb_plane_evm_* calls refuse every other kind. */
GB_API gb_status gb_plane_evm_factor_create(gb_ctx* ctx, size_t num_frames, const gb_cloud* const* frames, const double* poses, const gb_plane_patch_params* params,
                                            gb_factor** out);
/* num_keys, num_points; frame_indices and key_points (capacity num_keys each, or NULL): each key's frame index in the
 * creating call's list and its point count.  No launch. */
GB_API gb_status gb_plane_evm_factor_info(const gb_factor* factor, size_t* num_keys, size_t* num_points, int32_t* frame_indices, uint64_t* key_points);
/* F plane factors at once: poses (sum K_f x 16, each factor's keys in key order), H (sum (6 K_f)^2, each column-major),
 * b (sum 6 K_f), errors (F), status (F, GB_PLANE_EVM_*, or NULL).  One upload, one launch (one CTA per factor), one download
 * and its stream synchronisation; none for F == 0.  The factors' context does not matter: they own no device memory. */
GB_API gb_status gb_plane_evm_linearize(gb_ctx* ctx, size_t num_factors, gb_factor* const* factors, const double* poses, double* H, double* b, double* errors,
                                        int32_t* status);
/* the errors only: the same transfers and one launch */
GB_API gb_status gb_plane_evm_error(gb_ctx* ctx, size_t num_factors, gb_factor* const* factors, const double* poses, double* errors);

/* ---- glim::CloudDeskewing::deskew (src/glim/common/cloud_deskewing.cpp:11-55 constant velocity, :57-133 predicted IMU poses;
 *      called at src/glim/odometry/odometry_estimation_imu.cpp:313).  n_imu > 0: imu_times / imu_poses (n_imu x 16, T_world_imu)
 *      and `stamp` select the IMU-pose overload; n_imu == 0: linear_vel / angular_vel (either may be NULL = zero) select the
 *      constant-velocity overload.  T_post (or NULL) is applied to every deskewed point as a second transform -- the
 *      `pt = T_imu_lidar * pt` loop of odometry_estimation_imu.cpp:314-316 fused in.  Times must be ascending, as the
 *      preprocessor leaves them (cloud_preprocessor.cpp:135-136).
 *      gb_deskew_pose_table is the host half (time table + one pose per 0.1 ms slot); it needs no device. ---- */
GB_API gb_status gb_deskew_pose_table(const double T_imu_lidar[16], const double* linear_vel, const double* angular_vel, size_t n_imu, const double* imu_times,
                                      const double* imu_poses, double stamp, size_t n, const double* times, int32_t* time_indices /* n */, double* table_poses /* <= n x 16 */, size_t* table_size);
GB_API gb_status gb_deskew(gb_ctx* ctx, const double T_imu_lidar[16], const double* linear_vel, const double* angular_vel, size_t n_imu, const double* imu_times, const double* imu_poses,
                           double stamp, size_t n, const double* times, const double* xyzw, const double* T_post, double* out_xyzw);

#ifdef __cplusplus
}
#endif
#endif /* GLIM_B200_H */
