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
 *      own kind.  Each point with finite x, y, z is keyed with the fp32 lookup rule k = floor((float)(p * (float)(1 / cell_size)))
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
 *      GB_ERR_INVALID_ARGUMENT before any launch; grid sweeps take no pair_index, slab or peer slab.  gb_sweep_stats of a grid
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
 *      (gb_gicp_grid_factor_create) factors, all of one target class per call.
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
