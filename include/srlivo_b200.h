/*
 * srlivo_b200.h — C ABI of the H100-native (sm_90a) LIO scan-matching hot path of SR-LIVO.
 *
 * The reference (ZikangYuan/sr_livo) has no plugin/FFI layer: the path is a set of member
 * functions of `class lioOptimization` (include/lioOptimization.h:334-353) operating on
 * `voxelHashMap` (include/cloudMap.h:171).  This header is the seam a maintainer binds to
 * (see INTEGRATION.md): each entry point names the reference code it replaces.
 *
 * Conventions
 *   - plain C types only; no Eigen, no exceptions, no torch types.
 *   - quaternions are (x, y, z, w) = Eigen::Quaterniond::coeffs() order; 3x3 matrices row-major.
 *   - the library owns all device memory behind opaque handles; the caller owns every host
 *     pointer it passes; nothing is retained past a call except inside srl_map / srl_sweep.
 *   - one srl_ctx per host thread / GPU; calls on a ctx are serialised by the caller
 *     (the reference hot path is single-threaded: src/lioOptimization.cpp:1596-1604).
 *   - every function returns an srl_status; srl_last_error(ctx) gives the text.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point returns
 *     SRL_CUDA_ERROR.
 */
#ifndef SRLIVO_B200_H
#define SRLIVO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SRL_ABI_VERSION 1

typedef enum srl_status {
    SRL_OK = 0,
    SRL_TOO_FEW_RESIDUALS = 1, /* optimizeSummary.success=false (src/optimize.cpp:110-123); num_residuals still filled */
    SRL_NAN_PLANARITY = 2,     /* the reference throws std::runtime_error("error") (src/optimize.cpp:348-350) */
    SRL_CUDA_ERROR = 3,
    SRL_BAD_ARG = 4,
    SRL_MAP_FULL = 5,          /* more voxels than srl_map_create's max_voxels */
    SRL_SINGULAR = 6,          /* a 17x17 inverse failed (src/optimize.cpp:234,237) */
    SRL_COMM_ERROR = 7
} srl_status;

typedef struct srl_ctx srl_ctx;     /* device + stream + scratch */
typedef struct srl_map srl_map;     /* HBM-resident voxelHashMap (include/cloudMap.h:171) */
typedef struct srl_sweep srl_sweep; /* device-resident keypoints of one reconstructed sweep */

/* icpOptions fields read by the path (include/parameters.h:8-56, config/r3live.yaml:57-69),
 * plus lioOptimization::laser_point_cov (src/lioOptimization.cpp:364) and the frame id that
 * selects init-mode behaviour (src/optimize.cpp:21-23,135). */
typedef struct srl_icp_params {
    double size_voxel_map;
    double power_planarity;
    double max_dist_to_plane_icp;
    double weight_alpha;
    double weight_neighborhood;
    double threshold_orientation_norm; /* degrees */
    double threshold_translation_norm; /* metres */
    double laser_point_cov;
    int32_t voxel_neighborhood;        /* 1 or 2 */
    int32_t min_number_neighbors;      /* <= max_number_neighbors */
    int32_t max_number_neighbors;      /* <= 32 */
    int32_t threshold_voxel_occupancy;
    int32_t max_num_residuals;         /* cap, keypoint order (src/optimize.cpp:107) */
    int32_t num_iters_icp;
    int32_t init_num_frames;
    int32_t frame_id;
} srl_icp_params;

void srl_icp_params_r3live(srl_icp_params* p); /* config/r3live.yaml values, frame_id = 100 */

/* eskfEstimator state (src/eskfEstimator.cpp:3-21) */
typedef struct srl_eskf_state {
    double p[3];
    double q[4];
    double v[3];
    double ba[3];
    double bg[3];
    double g[3];
    double cov[17 * 17];
} srl_eskf_state;

/* the per-pass pose inputs of buildPlaneResiduals (src/optimize.cpp:25-28,38,49,83) */
typedef struct srl_frame {
    double q_cur[4];  /* p_frame->p_state->rotation */
    double t_cur[3];  /* p_frame->p_state->translation */
    double t_last[3]; /* all_cloud_frame[id-1]->p_state->translation */
    double R_il[9];   /* R_imu_lidar */
    double t_il[3];   /* t_imu_lidar */
} srl_frame;

/* What one pass reduces to (src/optimize.cpp:160-170,235,239) */
typedef struct srl_normal_eq {
    double HTH[36]; /* H_x^T H_x, row-major 6x6 */
    double HTh[6];  /* H_x^T h, h = distance*weight */
    double loss_sum;
    int64_t num_residuals;
    int64_t num_full_neighborhoods; /* keypoints that passed src/optimize.cpp:78 */
    int64_t num_candidates_scanned; /* map points whose distance the GPU evaluated (<= reference's sum C_k) */
    int64_t num_keypoints;          /* keypoints processed by this rank in this pass */
    int32_t nan_planarity;
    int32_t reserved;
} srl_normal_eq;

/* optional per-keypoint outputs (host pointers, any may be NULL); layouts match oracle/srl_oracle.h */
typedef struct srl_debug_out {
    double* world_xyz;  /* n*3 */
    int32_t* status;    /* n : -1 not visited (cap), 0 <K neighbours, 1 gated out, 2 accepted */
    int16_t* nbr;       /* n*K*4 : voxel key x,y,z + index in block, ascending distance */
    double* nbr_dist;   /* n*K */
    double* plane;      /* n*16 : raw_point3 norm_vector3 jacobians6 norm_offset distance weight a2D */
} srl_debug_out;

typedef struct srl_iekf_summary {
    int32_t success;            /* optimizeSummary.success */
    int32_t passes_run;
    int32_t num_residuals_used; /* optimizeSummary.num_residuals_used */
    int32_t converged;
    double trace[32][24];       /* per pass: d_x[17], frame_t[3], frame_q[4] */
} srl_iekf_summary;

/* ---- context ------------------------------------------------------------------------------- */
int srl_abi_version(void);
const char* srl_build_info(void);
/* stream == NULL: the library creates its own non-blocking stream; otherwise a cudaStream_t to run on
 * (pass cudaStreamLegacy = (void*)1 for the legacy default stream, whose handle is NULL) */
int srl_ctx_create(int device, void* cuda_stream, srl_ctx** out);
void srl_ctx_destroy(srl_ctx* ctx);
const char* srl_last_error(const srl_ctx* ctx);
int srl_ctx_synchronize(srl_ctx* ctx);
/* number of this library's kernels launched on the ctx since creation (bench.py "gpu_launches") */
int64_t srl_ctx_kernel_launches(const srl_ctx* ctx);
/* CUDA-event timing of the scan-matching kernel (k1_assoc) on the ctx stream: enable, then read the summed device
 * time and launch count of the passes since the last reset (bench.py "roofline"). Reading synchronises the stream. */
int srl_ctx_set_timing(srl_ctx* ctx, int enable);
/* tuning / test knobs (the kernel-variant selectors "split_lanes_per_keypoint", "fast_lanes_per_keypoint", "k1_min_blocks" and
 * "fast_min_blocks" choose among compiled template instances and are process-wide, everything else is per ctx):
 * "force_exact_selection" (0|1: every keypoint takes k1_assoc's exact FP64 selection),
 * "k1_variant" (0 auto; 1: k1_fast, 3: k1_scan + k1_fit, both with the exact fallback where applicable; 2: k1_assoc
 * only), "split_lanes_per_keypoint" (2|4: lanes per keypoint in k1_scan), "k1_min_blocks" (2|3|4) and
 * "fast_min_blocks" (4|5|6|8): resident-blocks-per-SM variants of the two kernels, "fast_lanes_per_keypoint" (1|2|4:
 * lanes that share one keypoint's candidate scan in k1_fast), "mapped_result" (1 default: a pass's sums
 * reach the host through a mapped pinned buffer + sequence flag; 0: cudaMemcpyAsync + stream synchronize),
 * "exchange_in_fit" (1 default: on several GPUs k1_fit's last block runs the NVLink exchange itself when the rank
 * flagged nothing, 0: always in the fallback launch), "fast_force_ambiguous_mod" (N > 0:
 * k1_fast hands every N-th keypoint to k1_assoc, to test the hand-over), "device_loop" (1 default: srl_update_iekf[_dist]
 * keep the whole iterated update on the GPU — a persistent block runs the ESIKF algebra between the passes, all passes are
 * enqueued at once, one host wait; 0: the host-driven loop, which is also used under kernel-serialising tools and for the
 * residual cap), "pdl" (1 default: programmatic dependent launch of the pass kernels in the device loop), "eager_order"
 * (1 default: a sweep is Morton-ordered right behind its upload instead of at its first pass).  Counters: "exact_fallbacks"
 * (keypoints whose FP32 selection in k1_assoc was ambiguous and were redone exactly), "fast_ambiguous" (keypoints
 * k1_fast handed to k1_assoc), "kernel_launches", "device_loop_active" (1 when the device-resident loop is in use on this
 * ctx), "iekf_step_cycles_avg" (SM clock ticks of one ESIKF step, sums seen -> pose published; resets on read). */
int srl_ctx_set_option(srl_ctx* ctx, const char* name, int64_t value);
int srl_ctx_get_counter(srl_ctx* ctx, const char* name, int64_t* value);
int srl_ctx_pass_time(srl_ctx* ctx, double* total_ms, int64_t* launches, int reset);

/* ---- map: voxelHashMap + addPointsToMap (include/cloudMap.h:124-184, src/lioOptimization.cpp:400-446,520-554)
 * max_num_points_in_voxel <= 20 (block layout), max_voxels <= 2^25 (32-bit point indices in the kernels) */
int srl_map_create(srl_ctx* ctx, double voxel_size, int32_t max_num_points_in_voxel, size_t max_voxels,
                   srl_map** out);
void srl_map_destroy(srl_map* map);
int srl_map_clear(srl_map* map);
int srl_map_stats(srl_map* map, int64_t* n_voxels, int64_t* n_points); /* mapSize (src/lioOptimization.cpp:574-581) */
/* removePointsFarFromLocation (src/lioOptimization.cpp:556-572; the call at :1032 is commented out in the reference, the
 * function is what bounds the map of a long run): erases every voxel whose FIRST point is farther than `distance` from
 * `location`; the block pool is compacted and the slot table rebuilt. */
int srl_map_remove_far(srl_map* map, const double location[3], double distance, int64_t* n_removed);
/* mirror of a host voxelHashMap: keys n*3, counts n, xyz n*cap*3 (block order = voxelBlock::points order) */
int srl_map_upload(srl_map* map, const int16_t* keys, const int32_t* counts, const float* xyz, size_t n_voxels);
int srl_map_download(srl_map* map, int16_t* keys, int32_t* counts, float* xyz, size_t max_voxels, int64_t* n_voxels);
/* addPointsToMap, sweep order preserved per voxel. xyz_world: host (or device if *_device) n*3 doubles */
int srl_map_insert(srl_map* map, const double* xyz_world, size_t n, double min_distance_points,
                   int32_t min_num_points, int64_t* n_added);
int srl_map_insert_device(srl_map* map, const double* d_xyz_world, size_t n, double min_distance_points,
                          int32_t min_num_points, int64_t* n_added);

/* stateEstimation's map update without leaving the device (src/lioOptimization.cpp:1027 after src/optimize.cpp:441-445):
 * transformPoint over the resident sweep with pose (q,t), then addPointsToMap of the registered points, sweep order */
int srl_map_insert_sweep(srl_map* map, srl_sweep* sweep, const double q[4], const double t[3], const double R_il[9],
                         const double t_il[3], double min_distance_points, int32_t min_num_points, int64_t* n_added);

/* ---- sweep: the keypoints vector of optimize() (src/optimize.cpp:430) ------------------------ */
int srl_sweep_create(srl_ctx* ctx, size_t capacity, srl_sweep** out);
void srl_sweep_destroy(srl_sweep* sweep);
/* host -> HBM.  Pageable memory is staged through a pinned buffer (the call returns when the staging buffer is free
 * again); pinned memory goes straight to the DMA engine and is read asynchronously: keep it unchanged until the next
 * synchronising call on the ctx (any pass / update / srl_ctx_synchronize). */
int srl_sweep_upload(srl_sweep* sweep, const double* raw_xyz, size_t n);
int srl_sweep_set_device(srl_sweep* sweep, const double* d_raw_xyz, size_t n);  /* device -> device copy */
/* keypoints [begin, end) are this rank's shard (point-index sharding, SURVEY.md §8(e)); default whole sweep */
int srl_sweep_set_shard(srl_sweep* sweep, size_t begin, size_t end);

/* ---- one ESIKF pass: buildPlaneResiduals + H_x/h + HTH/HTh (src/optimize.cpp:18-131,160-170,235,239) */
int srl_build_plane_residuals(srl_ctx* ctx, srl_map* map, srl_sweep* sweep, const srl_frame* frame,
                              const srl_icp_params* prm, srl_normal_eq* out, srl_debug_out* dbg);
/* asynchronous form: enqueue the pass on the ctx stream; the 32-double result block
 * [HTH upper triangle 21 | HTh 6 | loss | num_residuals | num_full | candidates | flags] lands in d_out32
 * (device memory owned by the caller, e.g. the buffer handed to an all-reduce). No cap support. */
int srl_build_plane_residuals_async(srl_ctx* ctx, srl_map* map, srl_sweep* sweep, const srl_frame* frame,
                                    const srl_icp_params* prm, double* d_out32);
/* unpack an (all-reduced) 32-double block */
int srl_normal_eq_unpack(const double* h_out32, srl_normal_eq* out);

/* ---- the iterated update: updateIEKF (src/optimize.cpp:133-314) incl. eskfEstimator::observe -- */
/* one pass of the host algebra (src/optimize.cpp:172-310) given the reduced normal equations;
 * *done = 1 when the loop would `break` (:309); `diverged` mirrors the `continue` at :248-251 */
typedef struct srl_iekf_iter {
    srl_eskf_state predict; /* snapshot at src/optimize.cpp:138-143 */
    int32_t pass_index;     /* i in [-1, max_num_iter) */
    int32_t max_num_iter;
} srl_iekf_iter;
int srl_iekf_begin(const srl_eskf_state* eskf, const srl_icp_params* prm, srl_iekf_iter* it);
int srl_iekf_step(srl_iekf_iter* it, const srl_normal_eq* ne, const srl_icp_params* prm, srl_eskf_state* eskf,
                  double frame_q[4], double frame_t[3], double d_x_out[17], int32_t* done, int32_t* diverged);
/* ---- multi-GPU: one process and ctx per GPU, map replicated, keypoints sharded (srl_sweep_set_shard).  The exchange of
 * the 32 sums is fused into the pass's last kernel: its final block writes them into every peer's mailbox over NVLink
 * peer memory (CUDA IPC mapping) and adds the peers' sums in rank order, so every rank ends a pass with the same
 * totals and runs the same host update.  Setup: create, export the 64-byte handle, exchange handles with any host
 * transport (rank order), connect.  All ranks must run the same sequence of passes, and the same form of the loop: the
 * device-resident and the host-driven form agree to rounding, not bit for bit — after connecting, read the counter
 * "device_loop_active" on every rank and set option "device_loop" to 0 everywhere if any rank reports 0
 * (sr_livo_b200/dist.py does). */
typedef struct srl_comm srl_comm;
int srl_comm_create(srl_ctx* ctx, int rank, int world, srl_comm** out);
void srl_comm_destroy(srl_comm* comm);
int srl_comm_export(srl_comm* comm, void* handle64);
int srl_comm_connect(srl_comm* comm, const void* handles /* world x 64 bytes, rank order */);
int srl_update_iekf_dist(srl_ctx* ctx, srl_comm* comm, srl_map* map, srl_sweep* sweep, srl_eskf_state* eskf, double frame_q[4],
                         double frame_t[3], const double t_last[3], const double R_il[9], const double t_il[3],
                         const srl_icp_params* prm, srl_iekf_summary* summary);

/* the contiguous keypoint range [begin, end) of `rank` among `world` ranks (boundaries on multiples of 32) */
void srl_shard_range(size_t n, int rank, int world, size_t* begin, size_t* end);
/* optimize() on several GPUs with HOST buffers (config 3 end to end): every rank passes the whole sweep's host array; the
 * rank uploads only its own range of keypoints (srl_shard_range), registers it with the per-pass exchange of
 * srl_update_iekf_dist (all ranks end with the same state) and writes the re-transformed points of its range
 * (src/optimize.cpp:441-445) into world_xyz_out[begin*3 .. end*3).  Pinned host memory is copied without staging. */
int srl_optimize_host_dist(srl_ctx* ctx, srl_comm* comm, srl_map* map, srl_sweep* sweep, const double* raw_xyz, size_t n,
                           srl_eskf_state* eskf, double frame_q[4], double frame_t[3], const double t_last[3],
                           const double R_il[9], const double t_il[3], const srl_icp_params* prm, srl_iekf_summary* summary,
                           double* world_xyz_out, size_t* shard_begin, size_t* shard_end);

/* full loop on one GPU (sweep already resident).  Default: device-resident (see "device_loop" above); the results of both
 * forms agree to rounding (the device forms the gain with one 6x6 inverse via the Woodbury identity, the host form with the
 * reference's two 17x17 inverses). */
int srl_update_iekf(srl_ctx* ctx, srl_map* map, srl_sweep* sweep, srl_eskf_state* eskf, double frame_q[4],
                    double frame_t[3], const double t_last[3], const double R_il[9], const double t_il[3],
                    const srl_icp_params* prm, srl_iekf_summary* summary);
/* optimize() minus gridSampling (src/optimize.cpp:428-448): host keypoints in, updateIEKF, then the
 * final re-transform of the frame (:441-445) written to world_xyz_out (host, n*3, may be NULL).
 * This is the end-to-end entry point with HOST buffers (H2D + D2H inside). */
int srl_optimize_host(srl_ctx* ctx, srl_map* map, srl_sweep* sweep, const double* raw_xyz, size_t n,
                      srl_eskf_state* eskf, double frame_q[4], double frame_t[3], const double t_last[3],
                      const double R_il[9], const double t_il[3], const srl_icp_params* prm,
                      srl_iekf_summary* summary, double* world_xyz_out);
/* transformPoint over the sweep (src/utility.cpp:314-318) into a device buffer (e.g. for srl_map_insert_device) */
int srl_sweep_transform_device(srl_ctx* ctx, srl_sweep* sweep, const double q[4], const double t[3],
                               const double R_il[9], const double t_il[3], double* d_world_xyz);

/* ---- keypoint selection (SURVEY.md §8(f) row N2): gridSampling / subSampleFrame (src/utility.cpp:167-201), called at
 * src/optimize.cpp:431.  One point per cell of size_voxel_subsampling (the first in frame order), emitted in the
 * reference's order, i.e. the iteration order of its std::tr1::unordered_map<voxel, ...> grid.  The dedupe over the n
 * points runs on the GPU; the order is produced by replaying the unique cells through the same libstdc++ container.
 * xyz_world: n*3 doubles (point3D::point) in host memory or already in HBM (detected per pointer; a device frame is not
 * copied, only the coordinates of the kept points come back for the replay); keypoint_index_out: host, capacity n. */
int srl_grid_sampling(srl_ctx* ctx, const double* xyz_world, size_t n, double size_voxel_subsampling,
                      uint32_t* keypoint_index_out, size_t* n_keypoints);

/* ---- row N3: per-sweep point transforms / undistortion (src/utility.cpp:203-332) -----------------------------------
 * One thread per point.  Every point buffer may be a host or a device pointer (detected per pointer), so a sweep can
 * stay in HBM from undistortion through registration to map insertion.  relative_time is point3D::relative_time (ms).
 * srl_imu_state carries the imuState fields these functions read (include/utility.h: timestamp, quat, trans, vel,
 * un_acc, un_gyr); states[] is host memory. */
typedef struct srl_imu_state {
    double timestamp;
    double quat[4];   /* x, y, z, w */
    double trans[3];
    double vel[3];
    double un_acc[3];
    double un_gyr[3];
} srl_imu_state;
/* distortFrameByConstant (src/utility.cpp:203-236): imu_point of every point from the pose interpolated (slerp / lerp)
 * between states[0] and states[n_states-1] */
int srl_distort_frame_by_constant(srl_ctx* ctx, const double* raw_xyz, const double* relative_time_ms, size_t n,
                                  const srl_imu_state* states, size_t n_states, double time_frame_begin,
                                  const double R_imu_lidar[9], const double t_imu_lidar[3], double* imu_xyz);
/* distortFrameByImu (src/utility.cpp:238-312, "distortion method 1").  The reference walks points and IMU intervals
 * with one iterator: points are consumed in order, the first point that fits no remaining interval stops the walk.
 * imu_xyz is in/out (points never reached keep their value); *n_written = number of leading points written.
 * timestamps must be non-decreasing (SRL_BAD_ARG otherwise). */
int srl_distort_frame_by_imu(srl_ctx* ctx, const double* raw_xyz, const double* relative_time_ms, size_t n,
                             const srl_imu_state* states, size_t n_states, double time_frame_begin,
                             const double R_imu_lidar[9], const double t_imu_lidar[3], double* imu_xyz, int64_t* n_written);
/* transformAllImuPoint (src/utility.cpp:320-332): raw_point = R_il^T (R(q_end)^-1 imu_point - R(q_end)^-1 t_end) - R_il^T t_il */
int srl_transform_all_imu_point(srl_ctx* ctx, const double* imu_xyz, size_t n, const srl_imu_state* last_state,
                                const double R_imu_lidar[9], const double t_imu_lidar[3], double* raw_xyz_out);

/* ---- row N4: the colour map fed by the map update (src/lioOptimization.cpp:448-551, colour branch) and the renderer that
 * colours its points from a camera frame (src/rgbMapTracker.cpp:181-237 with rgbPoint::updateRgb, src/cloudMap.cpp:59-101).
 * A colour map = a voxel map (same HBM layout as srl_map; srl_color_map_voxels exposes it for download / stats) whose
 * points carry (rgb, N_rgb, cov_rgb, observe_distance, last_observe_time), the fine occupancy set hashmap_3d_points
 * (cells of min_distance_points) that decides which stored points enter rgb_points_vec, and the list of voxels
 * visited for the first time by the sweeps since the last rendering (voxels_recent_visited). */
typedef struct srl_color_map srl_color_map;
typedef struct srl_camera {      /* the state fields cloudFrame::project3dTo2d / if2dPointsAvailable read (include/state.h) */
    double q_camera_world[4];    /* x, y, z, w */
    double t_camera_world[3];
    double t_world_camera[3];
    double fx, fy, cx, cy;
    double fov_margin;
    int32_t cols, rows;          /* image_cols, image_rows */
} srl_camera;
int srl_color_map_create(srl_ctx* ctx, double voxel_size, int32_t max_num_points_in_voxel, size_t max_voxels,
                         double min_distance_points, srl_color_map** out);
void srl_color_map_destroy(srl_color_map* cm);
srl_map* srl_color_map_voxels(srl_color_map* cm);
int srl_color_map_stats(srl_color_map* cm, int64_t* n_voxels, int64_t* n_points, int64_t* n_rgb_points, int64_t* n_recent,
                        int64_t* n_new_recent);
/* the loop of addPointsToMap over the registered frame (:533-542): every add_point_step-th point, sweep order, through
 * addPointToColorMap (min_num_points = 0).  xyz_world: host or device, n*3 doubles.  to_rendering mirrors the flag of
 * addPointsToMap (clears voxels_recent_visited_temp first, publishes it to the renderer afterwards). */
int srl_color_map_add_points(srl_color_map* cm, const double* xyz_world, size_t n, int32_t add_point_step, double time_sweep_end,
                             double time_last_process, int32_t to_rendering, int64_t* n_stored);
/* renderPointsInRecentVoxel: every point of every recently visited voxel is projected into the frame (pinhole, scale 1),
 * tested against the FoV margin, coloured by bilinear interpolation of the BGR8 image (host or device, rows*cols*3,
 * OpenCV's saturating Vec3b arithmetic) and fused with rgbPoint::updateRgb; *n_rendered = render_point_count. */
int srl_color_map_render_recent(srl_color_map* cm, const srl_camera* cam, const uint8_t* image_bgr, double obs_time, int64_t* n_rendered);
/* colour state in the voxel order of srl_map_download(srl_color_map_voxels(cm)): rgb nv*cap*3, n_rgb nv*cap, cov nv*cap*3,
 * obs_dist nv*cap, last_obs nv*cap, last_visited nv */
int srl_color_map_download_state(srl_color_map* cm, size_t max_voxels, int16_t* rgb, int16_t* n_rgb, float* cov, double* obs_dist,
                                 double* last_obs, double* last_visited);
/* rgb_points_vec as (voxel key x,y,z, index in block) per entry, voxels_recent_visited as voxel keys */
int srl_color_map_download_lists(srl_color_map* cm, int16_t* rgb_points, int16_t* recent);

/* eskfEstimator::observe (src/eskfEstimator.cpp:219-230) — host math, exported for parity tests */
int srl_eskf_observe(srl_eskf_state* eskf, const double d_x[17]);

/* host-side unit hooks for the per-keypoint math of the kernel (same source compiled for the host);
 * used by CPU tests only — they do not run the path. */
int srl_host_plane_fit(const double* nbr_xyz /*K*3*/, int32_t K, double normal[3], double* a2D, double evals[3]);

#ifdef __cplusplus
}
#endif
#endif /* SRLIVO_B200_H */
