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
 *   - "host or device, detected per pointer": device and managed (cudaMallocManaged) memory
 *     is used in place; page-locked and pageable host memory is staged through device scratch.
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
    SRL_MAP_FULL = 5,          /* more voxels than the map's max_voxels */
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
/* Every handle created on a ctx records the ctx's device and may be destroyed before or after the ctx: no srl_*_destroy
 * reads the ctx.  A handle outliving its ctx can only be destroyed; every other call on it needs the ctx. */
void srl_ctx_destroy(srl_ctx* ctx);
const char* srl_last_error(const srl_ctx* ctx);
int srl_ctx_synchronize(srl_ctx* ctx);
/* number of this library's kernels launched on the ctx since creation (bench.py "gpu_launches") */
int64_t srl_ctx_kernel_launches(const srl_ctx* ctx);
/* CUDA-event timing of the scan-matching kernel (k1_assoc) on the ctx stream: enable, then read the summed device
 * time and launch count of the passes since the last reset (bench.py "roofline"). Reading synchronises the stream. */
int srl_ctx_set_timing(srl_ctx* ctx, int enable);
/* tuning / test knobs, all of them per ctx.  The kernel-variant selectors choose among compiled template instances; each
 * also has an environment variable that srl_ctx_create reads (a value outside the allowed set leaves the default):
 * "force_exact_selection" (0|1: every keypoint takes k1_assoc's exact FP64 selection),
 * "k1_variant" (0 auto; 1: k1_fast, 3: k1_scan + k1_fit, both with the exact fallback where applicable; 2: k1_assoc
 * only), "split_lanes_per_keypoint" (2|4, default 4, SRL_SPLIT_LPK: lanes per keypoint in k1_scan), "scan_min_blocks"
 * (6|8, default 8, SRL_SCAN_MINB), "fit_min_blocks" (4|5|6, default 6, SRL_FIT_MINB), "k1_min_blocks" (2|3|4, default 3,
 * SRL_K1_MINB) and "fast_min_blocks" (4|5|6|8, default 5, SRL_FAST_MINB): resident-blocks-per-SM variants of k1_scan,
 * k1_fit, k1_assoc and k1_fast, "fast_lanes_per_keypoint" (1|2|4, default 1, SRL_FAST_LPK: lanes that share one
 * keypoint's candidate scan in k1_fast), "cluster_order" (0|1|2|3, default 1, SRL_CLUSTER_ORDER: the sweep's Morton order
 * by CUB's radix sort (0) or by the one-launch cluster sort (1; 2 and 3 its earlier versions), which the ctx's first four
 * uses after the option is set check against CUB's order; setting it starts those checks again),
 * "fast_force_ambiguous_mod" (N > 0:
 * k1_fast hands every N-th keypoint to k1_assoc, to test the hand-over), "device_loop" (1 default: srl_update_iekf[_dist]
 * keep the whole iterated update on the GPU — a persistent block runs the ESIKF algebra between the passes, all passes are
 * enqueued at once, one host wait, with or without the max_num_residuals cap; 0: the host-driven loop, which is also used
 * under kernel-serialising tools).  Counters: "exact_fallbacks"
 * (keypoints whose FP32 selection in k1_assoc was ambiguous and were redone exactly), "fast_ambiguous" (keypoints
 * k1_fast handed to k1_assoc), "kernel_launches", "device_loop_active" (1 when the device-resident loop is in use on this
 * ctx), "iekf_step_cycles_avg" (SM clock ticks of one ESIKF step, sums seen -> pose published; resets on read),
 * "cap_chunks_run" (keypoint chunks of the capped pass whose kernels did work: summed over the passes of the last
 * srl_update_iekf, or those of the last srl_build_plane_residuals call, whichever came last; 0 without the cap; reading
 * it after the device-resident loop synchronises the ctx stream), "cluster_order_active" (the ctx's sweep-order sort: -1
 * the cluster sort while its checks run, 1 the cluster sort checked, 0 CUB's).  The name of each integer option above
 * ("k1_variant", "shuffle_rule", the kernel-variant selectors and "cluster_order") also reads back its current value. */
int srl_ctx_set_option(srl_ctx* ctx, const char* name, int64_t value);
int srl_ctx_get_counter(srl_ctx* ctx, const char* name, int64_t* value);
int srl_ctx_pass_time(srl_ctx* ctx, double* total_ms, int64_t* launches, int reset);

/* ---- map: voxelHashMap + addPointsToMap (include/cloudMap.h:124-184, src/lioOptimization.cpp:400-446,520-554)
 * max_num_points_in_voxel <= 20 (block layout), max_voxels <= 2^25 (32-bit point indices in the kernels).
 * max_voxels is the hard limit: an insert or upload past it returns SRL_MAP_FULL.  Memory is committed for initial_voxels
 * at creation and grows on demand inside srl_map_insert*, srl_map_upload (and srl_color_map_add_points for a colour map's
 * voxels): the committed voxel count doubles (or jumps to what the call needs), capped at max_voxels.  The block pool sits
 * on address space reserved for max_voxels, so growing copies no point; the slot table is rebuilt at the next power of two
 * that keeps load <= 0.5.  Nothing shrinks (srl_map_remove_far and srl_map_clear keep what is committed).  A growth that
 * fails (SRL_CUDA_ERROR when the device is out of memory) leaves the map's contents unchanged and usable.
 * 1 <= initial_voxels <= max_voxels, else SRL_BAD_ARG.  srl_map_create is initial_voxels = max_voxels: everything committed
 * up front, no growth. */
int srl_map_create(srl_ctx* ctx, double voxel_size, int32_t max_num_points_in_voxel, size_t max_voxels,
                   srl_map** out);
int srl_map_create_growable(srl_ctx* ctx, double voxel_size, int32_t max_num_points_in_voxel, size_t initial_voxels,
                            size_t max_voxels, srl_map** out);
/* what is committed now: voxels backed by blocks, slots of the slot table, device bytes of both */
int srl_map_capacity(srl_map* map, size_t* committed_voxels, size_t* slot_capacity, size_t* committed_bytes);
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
/* addPointsToMap, sweep order preserved per voxel. xyz_world: n*3 doubles, host or device, detected per pointer (both
 * names run the same code) */
int srl_map_insert(srl_map* map, const double* xyz_world, size_t n, double min_distance_points,
                   int32_t min_num_points, int64_t* n_added);
int srl_map_insert_device(srl_map* map, const double* d_xyz_world, size_t n, double min_distance_points,
                          int32_t min_num_points, int64_t* n_added);

/* stateEstimation's map update without leaving the device (src/lioOptimization.cpp:1027 after src/optimize.cpp:441-445):
 * transformPoint over the resident sweep with pose (q,t), then addPointsToMap of the registered points, sweep order */
int srl_map_insert_sweep(srl_map* map, srl_sweep* sweep, const double q[4], const double t[3], const double R_il[9],
                         const double t_il[3], double min_distance_points, int32_t min_num_points, int64_t* n_added);

/* addPointsToMap + the cloud it publishes (publishCLoudWorld, src/lioOptimization.cpp:552; addPointToPcl :432, :1346-1355).
 * The map is updated exactly as by srl_map_insert / srl_map_insert_sweep.  The cloud holds, in sweep order, the points that
 * were appended to a voxel map.find found: one present before the call (an uploaded voxel with count 0 included) or created
 * by an earlier point of the same call.  A point that creates its voxel is stored but not published.  Each point is 4 floats:
 * x, y, z as stored, intensity = (float)(50 * ((double)z - translation_z)) evaluated in FP64 and rounded once;
 * srl_map_insert_sweep_published uses translation_z = t[2].  xyz_world and xyzi_out are host or device memory (detected per
 * pointer; a pageable host output is staged through pinned memory).  max_out >= n always suffices; max_out < n returns
 * SRL_BAD_ARG before the map is touched. */
int srl_map_insert_published(srl_map* map, const double* xyz_world, size_t n, double min_distance_points,
                             int32_t min_num_points, double translation_z, float* xyzi_out, size_t max_out,
                             int64_t* n_added, int64_t* n_published);
int srl_map_insert_sweep_published(srl_map* map, srl_sweep* sweep, const double q[4], const double t[3],
                                   const double R_il[9], const double t_il[3], double min_distance_points,
                                   int32_t min_num_points, float* xyzi_out, size_t max_out, int64_t* n_added,
                                   int64_t* n_published);

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
/* the sweep's Morton order as the passes read it (order[s] = the keypoint at sorted position s), copied to host memory
 * after a synchronise of the ctx stream; an order already computed is copied as it is.  *n_out = the sweep's keypoints;
 * order == NULL only counts; SRL_BAD_ARG when max_n < n. */
int srl_sweep_download_order(srl_sweep* sweep, uint32_t* order, size_t max_n, int64_t* n_out);

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

/* full loop on one GPU (sweep already resident).  Default: device-resident (see "device_loop" above).  The device forms the
 * gain with one 6x6 inverse via the Woodbury identity, the host form with the reference's two 17x17 inverses; both are
 * exact in exact arithmetic and differ by rounding errors that grow with the conditioning: on a diagonal prior both are
 * within 1e-13 of a 50-digit evaluation, at cond(P) = 1e12 the device's d_x within 5e-12 and the host's within 5e-7
 * (relative; DESIGN §4 "Algebra").  An exactly singular covariance makes the host form return SRL_SINGULAR and the device
 * form a finite update (DESIGN §5). */
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

/* ---- buildFrame (src/lioOptimization.cpp:786-893): from a cut sweep to the frame stateEstimation receives ---------------
 * In the reference's order: makePointTimestamp (point time enabled: every point kept, alpha > 1 clamped to 1 - 1e-5; else the
 * points outside [begin, end] are erased, order kept, no clamp), undistortion (motion_compensation 0 = IMU: distortFrameByImu,
 * 1 = CONSTANT_VELOCITY: distortFrameByConstant, anything else SRL_BAD_ARG), std::shuffle with a default-seeded
 * std::mt19937_64 (boost::mt19937_64), subSampleFrame only when voxel_size > 0 at (index_frame < init_num_frames ?
 * init_voxel_size : voxel_size) over point = the raw LiDAR coordinate, a second shuffle with the same engine, transformAllImuPoint,
 * then alpha_time = 1 and the identity pose for index_frame <= 2, the predicted pose after.  imu_point starts at 0: points an
 * IMU walk never reaches keep 0 (the reference keeps whatever the cut sweep held).  The shuffles' draws follow context option
 * "shuffle_rule" (0 default: Lemire's method, libstdc++ built with __int128; 1: the division downscale of libstdc++ without
 * __int128 and of libstdc++ <= 10).  raw_xyz (n*3) and timestamp (n) are host or device memory (detected per pointer); states[]
 * is host memory, n_states >= 1.  The frame stays in HBM; its buffers chain into srl_grid_sampling / srl_map_insert_device
 * (point) and srl_sweep_set_device (raw_point, after the caller's gather of keypoints). */
typedef struct srl_cloud_frame srl_cloud_frame;
typedef struct srl_build_frame_params {
    double timestamp_begin, timestamp_offset;
    int32_t point_time_enable;     /* cloudProcessing::isPointTimeEnable() (given_offset_time) */
    int32_t motion_compensation;   /* 0 IMU, 1 CONSTANT_VELOCITY (include/utility.h:82-86) */
    int32_t index_frame, init_num_frames;
    double init_voxel_size, voxel_size;
    double R_il[9], t_il[3];       /* R_imu_lidar, t_imu_lidar */
    double q_pred[4], t_pred[3];   /* cur_state->rotation (x, y, z, w), cur_state->translation */
    double prev_time_sweep_end;    /* all_cloud_frame.back()->time_sweep_end, read when index_frame > 1 (dt_offset) */
} srl_build_frame_params;
typedef struct srl_build_frame_info {   /* the cloudFrame scalars (:880-889) and what each stage did */
    double time_sweep_begin, time_sweep_end, time_frame_begin, time_frame_end, offset_begin, offset_end, dt_offset;
    double sample_size;            /* subSampleFrame's cell (unused when voxel_size <= 0) */
    int32_t frame_id;              /* index_frame */
    int32_t reserved;
    int64_t n_input, n_timestamped, n_imu_written, n_points;   /* n_imu_written: leading points the undistortion wrote */
    int64_t engine_words;          /* mt19937_64 outputs the shuffles consumed */
    int64_t shuffle_rejections;    /* draws that had to take another word */
    double stage_ms[6];            /* host clock: timestamps, undistortion, shuffle 1, subsample, shuffle 2, transforms */
} srl_build_frame_info;
typedef struct srl_cloud_frame_ptrs {   /* device buffers, final frame order, valid until the next srl_build_frame on the frame */
    double* raw_point;      /* n*3, after transformAllImuPoint */
    double* point;          /* n*3, world under the predicted (or identity) pose */
    double* imu_point;      /* n*3 */
    double* relative_time;  /* n, ms */
    double* alpha_time;     /* n */
    double* timestamp;      /* n */
    int32_t* source_index;  /* n, the point's index in the cut sweep */
} srl_cloud_frame_ptrs;
/* capacity: points reserved up front; a larger sweep grows the frame inside srl_build_frame */
int srl_cloud_frame_create(srl_ctx* ctx, size_t capacity, srl_cloud_frame** out);
void srl_cloud_frame_destroy(srl_cloud_frame* frame);
size_t srl_cloud_frame_size(const srl_cloud_frame* frame);
int srl_cloud_frame_device(srl_cloud_frame* frame, srl_cloud_frame_ptrs* ptrs);
/* host copies; any pointer may be NULL */
int srl_cloud_frame_download(srl_cloud_frame* frame, double* raw_point, double* point, double* imu_point, double* relative_time,
                             double* alpha_time, double* timestamp, int32_t* source_index);
int srl_build_frame(srl_ctx* ctx, const double* raw_xyz, const double* timestamp, size_t n, const srl_imu_state* states,
                    size_t n_states, const srl_build_frame_params* params, srl_cloud_frame* frame, srl_build_frame_info* info);
/* the device shuffle alone, for tests: std::shuffle's permutation of n elements (perm_out[p] = element that ends at p) drawn
 * from `words` (host, n_words engine outputs) or, with words == NULL, from a default-seeded mt19937_64; *words_used and
 * *next_word (the engine's next output) may be NULL.  rule as option "shuffle_rule". */
int srl_shuffle_replay(srl_ctx* ctx, const uint64_t* words, size_t n_words, size_t n, int32_t rule, uint32_t* perm_out,
                       size_t* words_used, uint64_t* next_word);

/* ---- row N4: the colour map fed by the map update (src/lioOptimization.cpp:448-551, colour branch) and the renderer that
 * colours its points from a camera frame (src/rgbMapTracker.cpp:181-237 with rgbPoint::updateRgb, src/cloudMap.cpp:59-101).
 * A colour map = a voxel map (same HBM layout as srl_map; srl_color_map_voxels exposes it for download / stats) whose
 * points carry (rgb, N_rgb, cov_rgb, observe_distance, last_observe_time), the fine occupancy set hashmap_3d_points
 * (cells of min_distance_points) that decides which stored points enter rgb_points_vec, and the list of voxels
 * the last rendering sweep visited for the first time (voxels_recent_visited). */
typedef struct srl_color_map srl_color_map;
typedef struct srl_camera {      /* the state fields cloudFrame::project3dTo2d / if2dPointsAvailable read (include/state.h) */
    double q_camera_world[4];    /* x, y, z, w */
    double t_camera_world[3];
    double t_world_camera[3];
    double fx, fy, cx, cy;
    double fov_margin;
    int32_t cols, rows;          /* image_cols, image_rows */
} srl_camera;
/* 1 <= max_num_points_in_voxel <= 128 (the shipped map_options use 50 and 100) and max_voxels * max(cap, 20) < 2^32 (32-bit
 * point ids), else SRL_BAD_ARG.  Up to 20 points the voxel map keeps the LIO block layout (20 points per block; it also works
 * with the LIO entry points); above 20 a block holds cap points and the LIO entry points (srl_map_insert*, srl_map_upload,
 * srl_map_remove_far, srl_build_plane_residuals*, srl_update_iekf*, srl_optimize_host*) reject the map with SRL_BAD_ARG.
 * HBM per committed point slot (committed voxels * max(cap, 20) slots): 16 B position + 40 B colour state; per committed
 * rgb point 4 B rgb id + 32-64 B fine-cell slot.  srl_color_map_create commits everything for max_voxels up front (about
 * 10.6 GB for 2^20 voxels at cap 100); srl_color_map_create_growable commits initial_voxels (and initial_voxels * max(cap,
 * 20) rgb points) and grows like srl_map_create_growable: the voxel arrays with the voxels, the rgb list and the fine set
 * with the rgb points, the two recent-voxel lists with their length, each doubling up to its limit (max_voxels, max_voxels
 * * max(cap, 20) rgb points, max_voxels recent entries).  Growth happens inside srl_color_map_add_points and,
 * for cap <= 20, inside srl_map_insert / srl_map_upload on srl_color_map_voxels(cm); never inside the renderer.
 * 1 <= initial_voxels <= max_voxels, else SRL_BAD_ARG.
 * Keys (voxel and fine cell) are static_cast<short>(x / size) as the reference compiles on x86-64: the low 16 bits of the
 * int32 truncation, so they wrap past |x / size| = 32767 like the reference's; NaN, +-inf and |x / size| >= 2^31 drop the point. */
int srl_color_map_create(srl_ctx* ctx, double voxel_size, int32_t max_num_points_in_voxel, size_t max_voxels,
                         double min_distance_points, srl_color_map** out);
int srl_color_map_create_growable(srl_ctx* ctx, double voxel_size, int32_t max_num_points_in_voxel, size_t initial_voxels,
                                  size_t max_voxels, double min_distance_points, srl_color_map** out);
/* what is committed now: voxels, fine-set slots, rgb points, and the device bytes of the whole colour map */
int srl_color_map_capacity(srl_color_map* cm, size_t* committed_voxels, size_t* fine_capacity, size_t* committed_rgb_points,
                           size_t* committed_bytes);
void srl_color_map_destroy(srl_color_map* cm);
srl_map* srl_color_map_voxels(srl_color_map* cm);
int srl_color_map_stats(srl_color_map* cm, int64_t* n_voxels, int64_t* n_points, int64_t* n_rgb_points, int64_t* n_recent,
                        int64_t* n_new_recent);
/* the loop of addPointsToMap over the registered frame (:533-542): every add_point_step-th point, sweep order, through
 * addPointToColorMap (min_num_points = 0).  xyz_world: host or device, n*3 doubles.  to_rendering mirrors the flag of
 * addPointsToMap (clears voxels_recent_visited_temp first, publishes it to the renderer afterwards).  A call without
 * rendering updates the voxels' last-visited times but lists no voxel: the reference clears what such a call appends
 * before it publishes anything.  So the recent list holds at most one entry per voxel. */
int srl_color_map_add_points(srl_color_map* cm, const double* xyz_world, size_t n, int32_t add_point_step, double time_sweep_end,
                             double time_last_process, int32_t to_rendering, int64_t* n_stored);
/* renderPointsInRecentVoxel: every point of every recently visited voxel is projected into the frame (pinhole, scale 1),
 * tested against the FoV margin, coloured by bilinear interpolation of the BGR8 image (host or device, rows*cols*3,
 * OpenCV's saturating Vec3b arithmetic) and fused with rgbPoint::updateRgb; *n_rendered = render_point_count.
 * cam->fov_margin must be >= 0, else SRL_BAD_ARG before anything is staged or launched (NaN included): a negative margin
 * would read outside the image with non-zero weights, which the reference leaves undefined (DESIGN.md section 5).  Reads
 * stay inside the rows*cols*3 image. */
int srl_color_map_render_recent(srl_color_map* cm, const srl_camera* cam, const uint8_t* image_bgr, double obs_time, int64_t* n_rendered);
/* colour state in the voxel order of srl_map_download(srl_color_map_voxels(cm)): rgb nv*cap*3, n_rgb nv*cap, cov nv*cap*3,
 * obs_dist nv*cap, last_obs nv*cap, last_visited nv */
int srl_color_map_download_state(srl_color_map* cm, size_t max_voxels, int16_t* rgb, int16_t* n_rgb, float* cov, double* obs_dist,
                                 double* last_obs, double* last_visited);
/* rgb_points_vec as (voxel key x,y,z, index in block) per entry, voxels_recent_visited as voxel keys */
int srl_color_map_download_lists(srl_color_map* cm, int16_t* rgb_points, int16_t* recent);
/* the coloured map as the reference publishes and saves it: the rgb_points_vec entries with N_rgb >= min_views (a short
 * against an int, so min_views <= 0 keeps points never rendered), each as x, y, z (the stored floats) and r, g, b = rgb[2],
 * rgb[1], rgb[0] (the BGR state swapped; short -> double -> uint8_t as g++ compiles it on x86-64: the low 8 bits).
 * order 0: pubColorPoints (src/lioOptimization.cpp:1210-1241; also one round of threadPubColorPoints' topics, concatenated),
 * index 0 upward.  order 1: saveColorPoints (:1386-1426), index n-1 down to 1: index 0 is never saved.
 * xyz (n*3 floats) and rgb (n*3 bytes) are host or device memory (detected per pointer; host output is staged through
 * pinned memory in chunks); both NULL counts only.  *n_out = the number of points; with outputs, max_points smaller than
 * that returns SRL_BAD_ARG and writes nothing. */
int srl_color_map_export(srl_color_map* cm, int32_t min_views, int32_t order, float* xyz, uint8_t* rgb, size_t max_points,
                         int64_t* n_out);

/* rgbMapTracker::selectPointsForProjection (src/rgbMapTracker.cpp:45-152), the points the optical-flow tracker is seeded and
 * refreshed with.  The reference's calls:
 *   first image (src/imageProcessing.cpp:131):  minimum_dis = track_windows_size / image_scale_factor, skip_step 1, recent
 *   refreshPointsForProjection (:159, src/rgbMapTracker.cpp:26-43): minimum_dis 10, skip_step 1, recent, from the camera that
 *     updatePoseForProjection(p_frame, -0.4) set up, i.e. fov_margin -0.4 (points up to 40 % outside the image).  Its early
 *     returns (image_cols == 0, the same frame_id as the last refresh) are the caller's state.
 * Candidates, in point_index order 0, skip_step, 2 skip_step, ...: the last point of every entry of the recent-voxel list the
 * renderer reads, in stored order (a voxel listed twice is two candidates), or rgb_points_vec when use_all_points is set or the
 * recent list is empty.  A candidate is skipped when depth = |p - t_world_camera| (the stored float widened) is > maximum_depth
 * or < minimum_depth, or when the renderer's projection (scale 1, the camera's own fov_margin, negative values included) refuses
 * it.  Its cell is u = (int)(std::round(u_f / minimum_dis) * minimum_dis), the same for v; a cell goes to its first candidate,
 * then to every later one whose depth is below the float the cell stores ((float)depth of its holder).  The winners come out in
 * point_index order: point_ids (block * block_pts + index, the ids of rgb_points_vec), xyz (the stored floats, 3 per point),
 * uv (the raw projection as floats, cv::Point2f(u_f, v_f), 2 per point).  Any output may be NULL, all NULL counts only; each is
 * host or device memory (detected per pointer; host output is staged through pinned memory).  *n_out = the number of points;
 * with outputs, max_points smaller than that returns SRL_BAD_ARG and writes nothing.  The map and both lists are not changed.
 * SRL_BAD_ARG also for minimum_dis not finite or <= 0, skip_step < 1, cols or rows < 2 (what the renderer refuses), and a
 * fov_margin whose window's cell coordinates do not fit an int.
 * Point ids stay valid while the map grows (blocks never move); srl_map_remove_far refuses a colour map's voxel map. */
typedef struct srl_projection_params {
    double minimum_dis;                    /* cell size in pixels: 5 (default), 10 (refreshPointsForProjection),
                                              track_windows_size / image_scale_factor (first image) */
    int32_t skip_step;                     /* >= 1 */
    int32_t use_all_points;
    double minimum_depth, maximum_depth;   /* minimum/maximum_depth_for_projection: 0.1 and 200 in the reference */
} srl_projection_params;
int srl_color_map_select_for_projection(srl_color_map* cm, const srl_camera* cam, const srl_projection_params* prm,
                                        uint32_t* point_ids, float* xyz, float* uv, size_t max_points, int64_t* n_out);
/* the per-point state the tracker reads, by point id (opticalFlowTracker.cpp:25,75,226,280 read positions;
 * imageProcessing.cpp:465-478 colour, N_rgb and covariance): xyz n*3 floats, rgb n*3 shorts (the BGR state as stored),
 * n_rgb n shorts, cov n*3 floats (0 while N_rgb == 0; a wrapped, negative N_rgb reports it), key_index n*4 shorts (voxel key x, y, z, index in block).
 * point_ids and every output are host or device memory; any output may be NULL.  An id that names no stored point returns
 * SRL_BAD_ARG and writes nothing. */
int srl_color_map_gather_points(srl_color_map* cm, const uint32_t* point_ids, size_t n, float* xyz, int16_t* rgb,
                                int16_t* n_rgb, float* cov, int16_t* key_index);

/* ---- the optical-flow tracker's pyramidal Lucas-Kanade (DESIGN.md row N6): LKOpticalFlowKernel (include/lkpyramid.h:65-131),
 * trackImage (src/lkpyramid.cpp:755-795), called by opticalFlowTracker::init and ::trackImage (src/opticalFlowTracker.cpp:134,196).
 * Bit for bit the reference: points, status, return value and every pyramid level. */
typedef struct srl_lk srl_lk;
#define SRL_LK_COUNT 1                  /* cv::TermCriteria::COUNT */
#define SRL_LK_EPS 2                    /* cv::TermCriteria::EPS */
typedef struct srl_lk_params {
    int32_t win_w, win_h;               /* lk_win_size, 3..31 each */
    int32_t max_level;                  /* 0..8; the first image's pyramid build lowers it for good (:609-619) */
    int32_t criteria_type;              /* SRL_LK_COUNT | SRL_LK_EPS */
    int32_t max_count;                  /* normalised as setTerminationCriteria (:670-682): 30 without COUNT, else clamped to 0..100 */
    double epsilon;                     /* 0.01 without EPS, else clamped to 0..10 */
    int32_t flags;                      /* OPTFLOW_* bits; neither changes trackImage's outputs (no err output here) */
    double min_eig_threshold;
} srl_lk_params;
int srl_lk_create(srl_ctx* ctx, const srl_lk_params* params, srl_lk** out);
void srl_lk_destroy(srl_lk* lk);
/* trackImage(gray, last_pts, curr_pts, status): gray is cols x rows bytes, rows `pitch` bytes apart; last_pts and curr_pts are n
 * (x, y) float pairs, status n bytes; *n_tracked = the sum of status.  The first image only builds its pyramid: curr_pts =
 * last_pts, status untouched, *n_tracked = 0.  n = 0 still consumes the image.  Every buffer is host or device memory.
 * SRL_BAD_ARG for an image not larger than the window, or of another size than the first image. */
int srl_lk_track_image(srl_lk* lk, const uint8_t* gray, int cols, int rows, size_t pitch, const float* last_pts, size_t n,
                       float* curr_pts, uint8_t* status, int64_t* n_tracked);
/* getMaxLevel() and the first image's size (0 x 0 before it) */
int srl_lk_info(srl_lk* lk, int32_t* max_level, int32_t* cols, int32_t* rows);
/* test hook: level `level` of the last image's pyramid (which 0) or of the image before it (which 1), padding included:
 * img (level rows + 2 win_h) x (level cols + 2 win_w) bytes, deriv the same count of (Ix, Iy) int16 pairs (either may be NULL;
 * host or device).  Level l is ((cols + 1) / 2 applied l times) wide, likewise high. */
int srl_lk_download_level(srl_lk* lk, int which, int level, uint8_t* img, int16_t* deriv);
/* device time of the last srl_lk_track_image: image upload + pyramid + derivatives, then the point tracking (CUDA events) */
int srl_lk_last_times(srl_lk* lk, double* pyramid_ms, double* track_ms);

/* ---- the camera image preparation (DESIGN.md row N7): imageProcessing::process (src/imageProcessing.cpp:91-125,166-200) turns
 * each BGR8 camera image into rgb_image (undistorted, Y-equalised in YCrCb, BGR8) and gray_image (undistorted, COLOR_RGB2GRAY,
 * CLAHE clip 3), bit for bit OpenCV's initUndistortRectifyMap(CV_16SC2) / remap(INTER_LINEAR) / cvtColor / CLAHE. */
typedef struct srl_image srl_image;
typedef struct srl_image_params {
    int32_t image_width, image_height;  /* camera_parameter.image_width / image_height of the yaml */
    double camera_intrinsic[9];         /* K, row-major */
    double camera_dist_coeffs[5];       /* k1, k2, p1, p2, k3 */
} srl_image_params;
/* the first-image step (:93-104) for inputs of cols x rows: image_scale_factor = image_width / cols, fx, cx, fy, cy divided by
 * it, the output (image_width / s, image_height / s) truncated, the CLAHE grid t = (int)max(out_cols * 32 / 640, 4) in both
 * dimensions, and the undistortion map.  SRL_BAD_ARG for a non-positive size, a side over 32767, an output under 16 x 16,
 * non-finite parameters or an intrinsic matrix without a finite inverse. */
int srl_image_create(srl_ctx* ctx, const srl_image_params* params, int cols, int rows, srl_image** out);
void srl_image_destroy(srl_image* img);
/* process:120-125 for one image: bgr is cols x rows BGR8, rows `pitch` bytes apart (pitch >= cols * 3); rgb_out receives
 * out_cols * out_rows * 3 bytes (BGR8, rgb_image), gray_out out_cols * out_rows bytes (gray_image), both contiguous.  Every
 * buffer is host or device memory.  SRL_BAD_ARG for another size than the one given at creation, a short pitch or a NULL
 * buffer; the object stays usable. */
int srl_image_process(srl_image* img, const uint8_t* bgr, int cols, int rows, size_t pitch, uint8_t* rgb_out, uint8_t* gray_out);
/* the output size, the CLAHE grid, image_scale_factor and the scaled intrinsics (row-major): the ones srl_camera and the
 * vision updates must use.  Any output may be NULL. */
int srl_image_info(srl_image* img, int32_t* out_cols, int32_t* out_rows, int32_t* tiles, double* scale_factor, double intrinsic[9]);
/* test hook: the undistortion map as OpenCV's CV_16SC2 + CV_16UC1 pair: map1 out_cols * out_rows (x, y) int16 pairs, map2
 * out_cols * out_rows uint16 (either may be NULL; host or device) */
int srl_image_download_maps(srl_image* img, int16_t* map1, uint16_t* map2);
/* device time of the last srl_image_process: the input upload (0 for a device image), remap + colour planes, both CLAHEs
 * (CUDA events) */
int srl_image_last_times(srl_image* img, double* upload_ms, double* remap_ms, double* clahe_ms);

/* ---- the two camera updates of process (DESIGN.md row N8): imageProcessing::vioEsikf (src/imageProcessing.cpp:220-380) and
 * vioPhotometric (:402-552) with the reference's constants (2 iterations, intrinsics and extrinsics estimated, at least 10
 * points, Huber threshold 1), over the colour map's points.  The handle keeps imageProcessing::covariance (11 x 11, row-major,
 * setInitialCov at creation); vioPhotometric reads and writes its block (1..6, 1..6). */
typedef struct srl_vio_state {   /* the p_state fields the two updates read and write (include/state.h) */
    double rotation[4];          /* x, y, z, w: the IMU's orientation in the world */
    double translation[3];
    double R_imu_camera[9];      /* row-major */
    double t_imu_camera[3];
    double fx, fy, cx, cy, time_td;
    double q_world_camera[4];    /* x, y, z, w */
    double t_world_camera[3];
    double q_camera_world[4];    /* iteration 0 projects with these two, as given */
    double t_camera_world[3];
} srl_vio_state;
/* vioEsikf over the tracked set in the caller's order: ids (n colour-map point ids), uv (n matched (u, v) float pairs) and
 * velocity (n image_velocity (du, dv) double pairs).  The positions come from the colour map as stored floats.  n_new_visited
 * is map_tracker->number_of_new_visited_voxel: cam_measurement_weight = max(0.001, min(5.0 / n_new_visited, 0.01)).  *result
 * is the reference's return value; state and covariance are updated in place when it is 1.  n < 10: *result = 0 and nothing
 * changes.  ids, uv and velocity are host or device memory.  SRL_BAD_ARG (nothing written) for an id that names no stored
 * point; SRL_SINGULAR (nothing written) for a zero or NaN pivot of the update's 11 x 11 system, which includes any NaN or
 * +-inf component of uv or velocity (the reference writes a NaN state and covariance and returns 1 there). */
int srl_image_vio_esikf(srl_image* img, srl_color_map* cm, srl_vio_state* state, const uint32_t* ids, const float* uv,
                        const double* velocity, size_t n, int32_t n_new_visited, int32_t* result);
/* vioPhotometric on the prepared rgb_image `bgr` (BGR8, cols x rows, rows `pitch` bytes apart, host or device): each point with
 * N_rgb >= 3 compares its colour state with the image's at its projection.  The image must have the handle's output size
 * (srl_image_info), else SRL_BAD_ARG.  Image reads are clamped to the nearest row and column.  Otherwise as
 * srl_image_vio_esikf (6 x 6 system); with fewer than 10 points of N_rgb >= 3 it returns *result = 1 and changes nothing. */
int srl_image_vio_photometric(srl_image* img, srl_color_map* cm, srl_vio_state* state, const uint32_t* ids, const double* velocity,
                              size_t n, int32_t n_new_visited, const uint8_t* bgr, int cols, int rows, size_t pitch, int32_t* result);
/* imageProcessing::covariance: `set` (121 doubles, row-major) replaces it, then `get` receives it; either may be NULL */
int srl_image_covariance(srl_image* img, const double* set, double* get);
/* what the last call of each update did: iterations run (0 when it returned before iterating), points used in its last
 * iteration, its last acc_residual as the reference's convergence tests read it; which = 0 vioEsikf, 1 vioPhotometric.  Any
 * output may be NULL; SRL_BAD_ARG before the first launch of that update. */
int srl_image_vio_last_summary(srl_image* img, int32_t which, int32_t* iterations, int32_t* points_used, double* acc_residual);
/* device time of the last launch of each update (CUDA events around the kernel; inputs and the result copy excluded) */
int srl_image_vio_last_times(srl_image* img, double* esikf_ms, double* photometric_ms);

/* ---- row N9: the optical-flow tracker's bookkeeping around its Lucas-Kanade (DESIGN.md row N9): opticalFlowTracker's init /
 * setTrackPoints (src/opticalFlowTracker.cpp:188-211), trackImage (:111-186, distance -20), removeOutlierUsingRansacPnp (:267-323,
 * if_remove_ourlier 1) and updateAndAppendTrackPoints (:13-102).  The tracker keeps three point sets on the device, each sorted
 * by colour-map point id (the reference's std::maps are ordered by rgbPoint*; DESIGN.md section 5):
 *   last  = map_rgb_points_in_last_image_pose: ids + uv (float pairs)
 *   match = what trackImage's Lucas-Kanade tracked (status set), in last order: ids, last uv, new uv; the list
 *           findFundamentalMat is given, so a caller's fundamental-matrix RANSAC runs on it
 *   cur   = map_rgb_points_in_cur_image_pose: ids, uv, image_velocity (double pairs)
 * The two RANSACs stay with the caller: srl_flow_tracker_reject_matches takes findFundamentalMat's mask and
 * srl_flow_tracker_remove_outliers solvePnPRansac's inliers.  rgbPoint::is_out_lier_count is kept in the colour map's per-point
 * state (zero for a new point).  cm and lk must be created on ctx; the tracker calls lk for every image it tracks. */
typedef struct srl_flow_tracker srl_flow_tracker;
typedef struct srl_flow_tracker_sets_out {   /* device pointers, valid until the next call on the tracker */
    int64_t n_match, n_cur, n_last;
    const uint32_t* match_ids;
    const float* match_last_uv;              /* n_match (x, y) pairs: the points findFundamentalMat's first argument holds */
    const float* match_uv;                   /* n_match (x, y) pairs: its second */
    const uint32_t* cur_ids;                 /* the ids, uv and velocity srl_image_vio_esikf / _photometric take */
    const float* cur_uv;
    const double* cur_velocity;
    const uint32_t* last_ids;                /* the ids srl_color_map_gather_points takes */
    const float* last_uv;
    double last_image_time;
} srl_flow_tracker_sets_out;
/* maximum_tracked_points >= 1 (300 in the reference) */
int srl_flow_tracker_create(srl_ctx* ctx, srl_color_map* cm, srl_lk* lk, int32_t maximum_tracked_points, srl_flow_tracker** out);
void srl_flow_tracker_destroy(srl_flow_tracker* t);
/* init: last = {ids[i] -> uv[i]} (a later duplicate id overwrites an earlier one), both image times = image_time, then the
 * Lucas-Kanade call on gray (cols x rows, rows `pitch` bytes apart), which on lk's first image builds its pyramid only.  ids (n)
 * and uv (n float pairs) are host or device memory.  An id that names no stored point, or an image lk refuses: SRL_BAD_ARG,
 * and the tracker is not changed. */
int srl_flow_tracker_init(srl_flow_tracker* t, const uint8_t* gray, int cols, int rows, size_t pitch, double image_time,
                          const uint32_t* ids, const float* uv, size_t n);
/* trackImage: cur and the match list are cleared; with fewer than 30 points in last only last_image_time = image_time (lk is not
 * called, *lk_called = 0).  Otherwise Lucas-Kanade over last's uv, the matches in last order, and cur = the matches with
 * if2dPointsAvailable(x, y, 1.0, 0.05) on a cols x rows image, with velocity (1e-3, 1e-3) when image_time - last_image_time <
 * 1e-5, else (new - old) / dt in cv::Point2f arithmetic.  last is not changed.  lk_called may be NULL. */
int srl_flow_tracker_track_image(srl_flow_tracker* t, const uint8_t* gray, int cols, int rows, size_t pitch, double image_time,
                                 int32_t* lk_called);
/* findFundamentalMat's status: one byte per match (n == n_match, host or device), non-zero = inlier; cur is rebuilt as the
 * matches inside the margin whose byte is set.  mask NULL: every match is an inlier.  A length mismatch: SRL_BAD_ARG. */
int srl_flow_tracker_reject_matches(srl_flow_tracker* t, const uint8_t* mask, size_t n);
/* removeOutlierUsingRansacPnp: with fewer than 10 points in cur, *result = 0 and nothing changes.  Otherwise last and cur both
 * become the entries of cur at the n indices `inliers` (host or device, in any order, repeats allowed), with cur's uv; inliers
 * NULL: all of cur.  *result = 1.  An index outside [0, n_cur): SRL_BAD_ARG, nothing changed.  When the caller's
 * solvePnPRansac fails or throws, the reference returns before this point: do not call it. */
int srl_flow_tracker_remove_outliers(srl_flow_tracker* t, const int32_t* inliers, size_t n, int32_t* result);
/* updateAndAppendTrackPoints(p_frame, map_tracker, mini_distance): cam is the image frame's camera after the updates (fov_margin
 * as its state holds it, 0.005 in the reference); the reprojection threshold is 2 * cam->cols / 320.  Every entry of last is
 * projected; one whose error exceeds the threshold twice in a row, or twice the threshold once, is erased (its count reset);
 * the others keep their place and mark their pixel cell.  Then the candidates (n ids, host or device, the selection's order;
 * refreshPointsForProjection's points_rgb_vec_for_projection) not in last whose projection succeeds and whose cell is free
 * enter last with the projection as uv, until last holds maximum_tracked_points (one more can enter when it already did).
 * SRL_BAD_ARG (nothing changed) for an id that names no stored point, mini_distance not finite or <= 0, cols or rows < 2, a
 * fov_margin whose cell coordinates do not fit an int. */
int srl_flow_tracker_update_and_append(srl_flow_tracker* t, const srl_camera* cam, double mini_distance, const uint32_t* candidates,
                                       size_t n);
/* the three sets' counts and device pointers */
int srl_flow_tracker_sets(srl_flow_tracker* t, srl_flow_tracker_sets_out* out);
/* test hook: is_out_lier_count of n point ids (host or device) into counts (n int16, host or device) */
int srl_flow_tracker_outlier_counts(srl_flow_tracker* t, const uint32_t* ids, size_t n, int16_t* counts);

/* ---- row N10: cloudProcessing (src/cloudProcessing.cpp) and the point pops of getMeasurements (src/lioOptimization.cpp:719-723,
 * 759-763).  The handlers decode a sensor message as it comes off the wire, order its points as libstdc++'s std::sort does
 * (the order of equal keys included), filter them as the reference does and append them to a device-resident point_buffer:
 * raw xyz (3 doubles), relative_time (ms) and timestamp (s) per point.  srl_lidar_cut pops the queue's front while its
 * timestamp is below t and hands out device pointers that srl_build_frame takes as they are.  Message buffers are host or
 * device memory (detected per pointer).  Each handler call and each cut reads back once.  Where the reference is undefined:
 * a Livox message with no point left appends nothing and keeps last_end_time; a ring >= n_scans on the yaw path, or a NaN
 * sort key (a NaN time field, NaN xyz on the yaw path), is SRL_BAD_ARG with nothing appended and no state changed. */
typedef struct srl_lidar srl_lidar;
typedef struct srl_lidar_params {   /* lioOptimization::readParameters' lidar_parameter / common values */
    int32_t lidar_type;             /* 1 LIVOX, 2 VELO, 3 OUST, 4 ROBO (include/cloudProcessing.h LID_TYPE) */
    int32_t n_scans;                /* N_SCANS */
    int32_t scan_rate;              /* SCAN_RATE (Hz) */
    int32_t time_unit;              /* 0 SEC, 1 MS, 2 US, 3 NS */
    double blind;                   /* m */
    int32_t point_filter_num;       /* >= 1 */
    int32_t reserved;
} srl_lidar_params;
typedef struct srl_cloud2_layout {  /* PointCloud2: point_step and the byte offsets msg->fields gives (pcl::fromROSMsg by name) */
    uint32_t point_step;
    int32_t off_x, off_y, off_z;    /* float32 */
    int32_t off_time;               /* VELO "time" float32, OUST "t" uint32, ROBO "timestamp" float64 */
    int32_t off_ring;               /* "ring": OUST uint8, VELO / ROBO uint16; < 0: absent (ring 0, as a robosense point's default) */
    uint32_t width;                 /* msg->width: points per row */
    uint32_t row_step;              /* msg->row_step: bytes from one row to the next; 0: rows packed (width * point_step) */
} srl_cloud2_layout;
typedef struct srl_lidar_info {
    double last_end_time;           /* -1 before the first message */
    int32_t given_offset_time;      /* isPointTimeEnable(): set by the PointCloud2 handlers, false at creation */
    int32_t sweep_id;               /* process() calls that decoded a message */
    double sweep_interval;          /* getSweepInterval() = 1 / scan_rate */
    int64_t size;                   /* points queued */
    double front_timestamp, back_timestamp;   /* NaN when the queue is empty */
    int64_t capacity;               /* points the queue holds before it grows */
} srl_lidar_info;
/* initial_capacity: points reserved up front; the queue grows on demand */
int srl_lidar_create(srl_ctx* ctx, const srl_lidar_params* params, size_t initial_capacity, srl_lidar** out);
void srl_lidar_destroy(srl_lidar* l);
/* livoxHandler: n CustomPoint records `stride` (>= 19) bytes apart, packed as the ROS message (offset_time u32 @0, x y z f32 @4,
 * @8, @12, reflectivity @16, tag @17, line @18; no alignment needed).  *appended may be NULL. */
int srl_lidar_livox(srl_lidar* l, const uint8_t* records, size_t n, size_t stride, double stamp, int64_t* appended);
/* process: the handler of params->lidar_type (VELO, OUST, ROBO; SRL_BAD_ARG for LIVOX) over n = width * height points of
 * layout->point_step bytes, row r at data + r * row_step (row_step 0: rows packed).  SRL_BAD_ARG for a field outside point_step,
 * row_step below width * point_step, or n not a multiple of width (width 0 takes one row of n points). */
int srl_lidar_process(srl_lidar* l, const uint8_t* data, size_t n, const srl_cloud2_layout* layout, double stamp, int64_t* appended);
/* pop while the queue is not empty and front().timestamp < t.  *raw_xyz / *timestamp: the popped points in the queue's device
 * memory (count x 3 and count doubles), valid until the next handler call on l (which may move the queue); either may be NULL.
 * A handle is not thread-safe: calls on one srl_lidar (and the srl_build_frame that reads a cut's pointers) must not overlap. */
int srl_lidar_cut(srl_lidar* l, double t, int64_t* count, const double** raw_xyz, const double** timestamp);
int srl_lidar_info_get(srl_lidar* l, srl_lidar_info* info);
/* host copies of the whole queue, front first; any pointer may be NULL */
int srl_lidar_download(srl_lidar* l, double* raw_xyz, double* relative_time, double* timestamp);
/* the device std::sort alone, for tests: perm_out[p] = the index of the key that ends at p (host, n); keys host or device;
 * *heapsorts = segments the depth limit handed to the heapsort fallback (may be NULL).  NaN keys: SRL_BAD_ARG. */
int srl_lidar_sort_replay(srl_ctx* ctx, const double* keys, size_t n, int32_t* perm_out, int32_t* heapsorts);

/* eskfEstimator::observe (src/eskfEstimator.cpp:219-230) — host math, exported for parity tests */
int srl_eskf_observe(srl_eskf_state* eskf, const double d_x[17]);

/* host-side unit hooks for the per-keypoint math of the kernel (same source compiled for the host);
 * used by CPU tests only — they do not run the path. */
int srl_host_plane_fit(const double* nbr_xyz /*K*3*/, int32_t K, double normal[3], double* a2D, double evals[3]);
/* the device-resident updateIEKF loop (the same kernel srl_update_iekf runs) fed with given sums instead of passes:
 * block p of `sums` (n_blocks x 32 doubles, the layout of srl_build_plane_residuals_async) is what pass p hands to the
 * loop, from a one-warp kernel that waits for the pass's pose like a pass kernel.  n_blocks >= the loop's passes
 * (max_num_iter + 1, see srl_iekf_begin), <= 40.  first_delay_cycles > 0: pass 0's sums arrive that many SM clock ticks
 * late (<= 2^32), so the loop's warm-up step runs first; < 0: they are there before the loop starts, so it is skipped.
 * Outputs as srl_update_iekf.  SRL_CUDA_ERROR when the device-resident loop is not in use on the ctx (option
 * "device_loop" = 0, kernel-serialising tools).  Used by tests. */
int srl_iekf_replay(srl_ctx* ctx, srl_eskf_state* eskf, double frame_q[4], double frame_t[3], const srl_icp_params* prm,
                    const double* sums, int32_t n_blocks, int64_t first_delay_cycles, srl_iekf_summary* summary);

#ifdef __cplusplus
}
#endif
#endif /* SRLIVO_B200_H */
