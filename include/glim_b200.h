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
GB_API uint64_t gb_ctx_kernel_launches(gb_ctx* ctx); /* kernels of this library launched so far */

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
 * cov6 (V x 6); any pointer may be NULL */
GB_API gb_status gb_voxelmap_download(const gb_voxelmap* map, int32_t* buckets, int32_t* num_points, float* means, float* cov6);
GB_API gb_status gb_voxelmap_destroy(gb_voxelmap* map);

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

/* ---- NonlinearFactorSetGPU::add(graph) / ::linearize(values) (odometry_estimation_gpu.cpp:383-386;
 *      hook at src/glim/viewer/offline_viewer.cpp:29): F x 64 B of poses down, one launch over all
 *      factors, F records up. ---- */
GB_API gb_status gb_factor_set_linearize(gb_ctx* ctx, size_t num_factors, gb_factor* const* factors, const double* T_target_source /* F x 16 */, gb_linearized6* out /* F */);
GB_API gb_status gb_factor_set_error(gb_ctx* ctx, size_t num_factors, gb_factor* const* factors, const double* T_lin /* F x 16 */, const double* T_eval /* F x 16 */, double* errors /* F */);

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
 *      (src/glim/common/cloud_covariance_estimation.cpp:43-122, :181-196) ---- */
GB_API gb_status gb_covariances(gb_ctx* ctx, size_t n, const double* xyzw, const int32_t* neighbors, int k_correspondences, int k_neighbors, double* normals4, double* cov4x4);

/* ---- CloudPreprocessor::find_neighbors (src/glim/preprocess/cloud_preprocessor.cpp:190-221): exact k-NN,
 *      query included, row-major neighbors[i*k + j] ---- */
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
