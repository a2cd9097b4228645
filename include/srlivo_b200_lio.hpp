// srlivo_b200_lio.hpp — C++ host mirror of the reference's scan-matching interface over the C ABI.
//
// The reference is C++ (class lioOptimization, include/lioOptimization.h:192-385); a maintainer who wants the GPU
// path swaps the bodies of four member functions for the calls below (INTEGRATION.md shows the diff).  Header-only,
// Eigen-free by default; define SRL_HAVE_EIGEN before including to get overloads on the reference's own types
// (point3D / icpOptions / Eigen::Quaterniond), which cannot be compiled in this repository's container.
//
//   reference                                                   this header
//   lioOptimization::addPointsToMap   src/lioOptimization.cpp:520   srl::LioBackend::addPointsToMap
//   lioOptimization::mapSize          src/lioOptimization.cpp:574   srl::LioBackend::mapSize
//   lioOptimization::buildPlaneResiduals  src/optimize.cpp:18       srl::LioBackend::buildPlaneResiduals
//   lioOptimization::updateIEKF       src/optimize.cpp:133          srl::LioBackend::updateIEKF
//   lioOptimization::optimize         src/optimize.cpp:428          srl::LioBackend::optimize (keypoints given)
//   lioOptimization::removePointsFarFromLocation  src/lioOptimization.cpp:556   srl::LioBackend::removePointsFarFromLocation
//   gridSampling                      src/utility.cpp:188           srl::LioBackend::gridSampling (keypoint indices)
//   distortFrameByConstant / ByImu    src/utility.cpp:203,238       srl::LioBackend::distortFrameByConstant / distortFrameByImu
//   buildFrame (+ makePointTimestamp) src/lioOptimization.cpp:786,821 srl::LioBackend::buildFrame (frame stays in HBM: frame())
//   transformAllImuPoint              src/utility.cpp:320           srl::LioBackend::transformAllImuPoint
//   addPointToColorMap (loop :533-551) src/lioOptimization.cpp:448  srl::LioBackend::addPointsToColorMap
//   rgbMapTracker::renderPointsInRecentVoxel  src/rgbMapTracker.cpp:216  srl::LioBackend::renderPointsInRecentVoxel
//   addPointToPcl + publishCLoudWorld src/lioOptimization.cpp:432,552 srl::LioBackend::addPointsToMapPublished
//   pubColorPoints / saveColorPoints  src/lioOptimization.cpp:1210,1386 srl::LioBackend::pubColorPoints / saveColorPoints
//   rgbMapTracker::selectPointsForProjection src/rgbMapTracker.cpp:45 srl::LioBackend::selectPointsForProjection / gatherColorPoints
//   LKOpticalFlowKernel::trackImage   src/lkpyramid.cpp:755         srl::LKOpticalFlowKernel::trackImage (on LioBackend::context())
//   imageProcessing::process :91-125  src/imageProcessing.cpp:91    srl::ImageProcessing (undistortion, grey, CLAHE; on LioBackend::context())
#pragma once

#include <array>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "srlivo_b200.h"

namespace srl {

struct optimizeSummary {   // include/lioOptimization.h (same fields the path fills)
    bool success = false;
    int num_residuals_used = 0;
    std::string error_log;
    int passes_run = 0;
    bool converged = false;
};

class LioBackend {
public:
    // device: CUDA ordinal; stream: cudaStream_t or nullptr; max_voxels: the map's limit; sweep_capacity sizes the sweep
    // buffers; initial_voxels: voxels committed at creation, the map grows from there up to max_voxels (0 = max_voxels)
    LioBackend(int device, void* stream, size_t max_voxels, size_t sweep_capacity, double size_voxel_map = 1.0,
               int max_num_points_in_voxel = 20, size_t initial_voxels = 0) {
        check(srl_ctx_create(device, stream, &ctx_), "srl_ctx_create (no CPU fallback: a CUDA device is required)");
        check(srl_map_create_growable(ctx_, size_voxel_map, max_num_points_in_voxel, initial_voxels ? initial_voxels : max_voxels,
                                      max_voxels, &map_), "srl_map_create_growable");
        check(srl_sweep_create(ctx_, sweep_capacity, &sweep_), "srl_sweep_create");
        const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        std::memcpy(R_imu_lidar, I, sizeof(I));
        std::memset(t_imu_lidar, 0, sizeof(t_imu_lidar));
    }
    ~LioBackend() {
        if (frame_) srl_cloud_frame_destroy(frame_);
        if (color_) srl_color_map_destroy(color_);
        if (sweep_) srl_sweep_destroy(sweep_);
        if (map_) srl_map_destroy(map_);
        if (ctx_) srl_ctx_destroy(ctx_);
    }
    LioBackend(const LioBackend&) = delete;
    LioBackend& operator=(const LioBackend&) = delete;

    double R_imu_lidar[9];   // include/lioOptimization.h:227-228
    double t_imu_lidar[3];
    srl_eskf_state eskf{};   // eskf_pro's state (src/eskfEstimator.cpp:3-21)

    // src/lioOptimization.cpp:520-554: registered frame (world points, sweep order) into the voxel map
    long long addPointsToMap(const double* xyz_world, size_t n, double min_distance_points, int min_num_points = 0) {
        int64_t added = 0;
        check(srl_map_insert(map_, xyz_world, n, min_distance_points, min_num_points, &added), "srl_map_insert");
        return added;
    }
    // the same insert + the cloud publishCLoudWorld sends (src/lioOptimization.cpp:432,552, addPointToPcl :1346-1355): xyzi gets
    // x, y, z, intensity of each published point, sweep order; translation_z = p_frame->p_state->translation.z()
    long long addPointsToMapPublished(const double* xyz_world, size_t n, double min_distance_points, int min_num_points,
                                      double translation_z, std::vector<float>& xyzi) {
        xyzi.resize(n * 4);
        int64_t added = 0, n_pub = 0;
        check(srl_map_insert_published(map_, xyz_world, n, min_distance_points, min_num_points, translation_z, xyzi.data(), n, &added,
                                       &n_pub), "srl_map_insert_published");
        xyzi.resize((size_t)n_pub * 4);
        return added;
    }
    // src/lioOptimization.cpp:574-581
    long long mapSize() {
        int64_t nv = 0, np = 0;
        check(srl_map_stats(map_, &nv, &np), "srl_map_stats");
        return np;
    }
    // the keypoints vector of optimize() (raw_point members), uploaded once per sweep
    void setKeypoints(const double* raw_xyz, size_t n) { check(srl_sweep_upload(sweep_, raw_xyz, n), "srl_sweep_upload"); }

    // src/optimize.cpp:18-131 + :160-170,:235,:239 — one pass; returns the normal equations instead of plane_residuals
    optimizeSummary buildPlaneResiduals(const srl_icp_params& cur_icp_options, const double q_cur[4], const double t_cur[3],
                                        const double t_last[3], srl_normal_eq& ne, srl_debug_out* dbg = nullptr) {
        srl_frame fr;
        std::memcpy(fr.q_cur, q_cur, sizeof(fr.q_cur));
        std::memcpy(fr.t_cur, t_cur, sizeof(fr.t_cur));
        std::memcpy(fr.t_last, t_last, sizeof(fr.t_last));
        std::memcpy(fr.R_il, R_imu_lidar, sizeof(fr.R_il));
        std::memcpy(fr.t_il, t_imu_lidar, sizeof(fr.t_il));
        const int rc = srl_build_plane_residuals(ctx_, map_, sweep_, &fr, &cur_icp_options, &ne, dbg);
        optimizeSummary s;
        s.num_residuals_used = (int)ne.num_residuals;
        if (rc == SRL_NAN_PLANARITY) throw std::runtime_error("error");   // src/optimize.cpp:348-350
        if (rc == SRL_TOO_FEW_RESIDUALS) { s.success = false; s.error_log = srl_last_error(ctx_); return s; }   // :110-123
        check(rc, "srl_build_plane_residuals");
        s.success = true;
        return s;
    }

    // src/optimize.cpp:133-314 — frame_q/frame_t = p_frame->p_state rotation/translation (in/out)
    optimizeSummary updateIEKF(const srl_icp_params& cur_icp_options, double frame_q[4], double frame_t[3], const double t_last[3]) {
        srl_iekf_summary sm;
        const int rc = srl_update_iekf(ctx_, map_, sweep_, &eskf, frame_q, frame_t, t_last, R_imu_lidar, t_imu_lidar,
                                       &cur_icp_options, &sm);
        return summarise(rc, sm);
    }

    // src/optimize.cpp:428-448 with the keypoints already selected; world_xyz_out (n*3, may be null) receives the
    // re-transformed frame (:441-445)
    optimizeSummary optimize(const double* raw_xyz, size_t n, const srl_icp_params& cur_icp_options, double frame_q[4],
                             double frame_t[3], const double t_last[3], double* world_xyz_out) {
        srl_iekf_summary sm;
        const int rc = srl_optimize_host(ctx_, map_, sweep_, raw_xyz, n, &eskf, frame_q, frame_t, t_last, R_imu_lidar,
                                         t_imu_lidar, &cur_icp_options, &sm, world_xyz_out);
        return summarise(rc, sm);
    }

    // src/lioOptimization.cpp:556-572 — voxels whose first point is farther than `distance` from `location` go
    long long removePointsFarFromLocation(const double location[3], double distance) {
        int64_t removed = 0;
        check(srl_map_remove_far(map_, location, distance, &removed), "srl_map_remove_far");
        return removed;
    }
    // src/utility.cpp:188-201 — indices (into the frame) of the keypoints, in the reference's order
    std::vector<uint32_t> gridSampling(const double* xyz_world, size_t n, double size_voxel_subsampling) {
        std::vector<uint32_t> keep(n);
        size_t m = 0;
        check(srl_grid_sampling(ctx_, xyz_world, n, size_voxel_subsampling, keep.data(), &m), "srl_grid_sampling");
        keep.resize(m);
        return keep;
    }
    // src/utility.cpp:203-236, :238-312, :320-332 — point buffers may be host or device pointers
    void distortFrameByConstant(const double* raw_xyz, const double* relative_time_ms, size_t n, const std::vector<srl_imu_state>& imu_states,
                                double time_frame_begin, double* imu_xyz) {
        check(srl_distort_frame_by_constant(ctx_, raw_xyz, relative_time_ms, n, imu_states.data(), imu_states.size(), time_frame_begin,
                                            R_imu_lidar, t_imu_lidar, imu_xyz), "srl_distort_frame_by_constant");
    }
    long long distortFrameByImu(const double* raw_xyz, const double* relative_time_ms, size_t n, const std::vector<srl_imu_state>& imu_states,
                                double time_frame_begin, double* imu_xyz) {
        int64_t written = 0;
        check(srl_distort_frame_by_imu(ctx_, raw_xyz, relative_time_ms, n, imu_states.data(), imu_states.size(), time_frame_begin,
                                       R_imu_lidar, t_imu_lidar, imu_xyz, &written), "srl_distort_frame_by_imu");
        return written;
    }
    void transformAllImuPoint(const double* imu_xyz, size_t n, const srl_imu_state& last_state, double* raw_xyz_out) {
        check(srl_transform_all_imu_point(ctx_, imu_xyz, n, &last_state, R_imu_lidar, t_imu_lidar, raw_xyz_out), "srl_transform_all_imu_point");
    }
    // src/lioOptimization.cpp:786-893 — the cut sweep (raw_xyz n*3, timestamp n; host or device) becomes the device-resident frame
    // (created on first use, reused after: its device pointers change only when a larger sweep grows it).  params.R_il / t_il
    // are taken from this backend's extrinsics.  Returns the cloudFrame scalars.
    srl_build_frame_info buildFrame(const double* raw_xyz, const double* timestamp, size_t n, const std::vector<srl_imu_state>& imu_states,
                                    srl_build_frame_params params) {
        if (!frame_) check(srl_cloud_frame_create(ctx_, n, &frame_), "srl_cloud_frame_create");
        for (int i = 0; i < 9; ++i) params.R_il[i] = R_imu_lidar[i];
        for (int i = 0; i < 3; ++i) params.t_il[i] = t_imu_lidar[i];
        srl_build_frame_info info;
        check(srl_build_frame(ctx_, raw_xyz, timestamp, n, imu_states.data(), imu_states.size(), &params, frame_, &info), "srl_build_frame");
        return info;
    }
    srl_cloud_frame* frame() { return frame_; }

#ifdef SRL_HAVE_EIGEN
    // overloads on the reference's types (cloudMap.h / parameters.h must be included first)
    static srl_icp_params fromIcpOptions(const icpOptions& o, int frame_id, double laser_point_cov) {
        srl_icp_params p;
        p.size_voxel_map = o.size_voxel_map; p.power_planarity = o.power_planarity; p.max_dist_to_plane_icp = o.max_dist_to_plane_icp;
        p.weight_alpha = o.weight_alpha; p.weight_neighborhood = o.weight_neighborhood;
        p.threshold_orientation_norm = o.threshold_orientation_norm; p.threshold_translation_norm = o.threshold_translation_norm;
        p.laser_point_cov = laser_point_cov; p.voxel_neighborhood = o.voxel_neighborhood; p.min_number_neighbors = o.min_number_neighbors;
        p.max_number_neighbors = o.max_number_neighbors; p.threshold_voxel_occupancy = o.threshold_voxel_occupancy;
        p.max_num_residuals = o.max_num_residuals; p.num_iters_icp = o.num_iters_icp; p.init_num_frames = o.init_num_frames;
        p.frame_id = frame_id;
        return p;
    }
    void setKeypoints(const std::vector<point3D>& keypoints) {
        std::vector<double> raw(keypoints.size() * 3);
        for (size_t i = 0; i < keypoints.size(); ++i) for (int a = 0; a < 3; ++a) raw[3 * i + a] = keypoints[i].raw_point[a];
        setKeypoints(raw.data(), keypoints.size());
    }
#endif

    srl_ctx* ctx() { return ctx_; }
    srl_map* map() { return map_; }
    srl_sweep* sweep() { return sweep_; }

    // ---- row N4: color_voxel_map + hashmap_3d_points + rgb_points_vec + voxels_recent_visited (include/lioOptimization.h:275-291)
    // created on first use with the LiDAR map's voxel size and cap (src/lioOptimization.cpp:539 passes map_options' values)
    // (initial_voxels as in the constructor: 0 = commit max_voxels up front)
    void enableColorMap(double size_voxel_map, int max_num_points_in_voxel, size_t max_voxels, double min_distance_points,
                        size_t initial_voxels = 0) {
        if (!color_) check(srl_color_map_create_growable(ctx_, size_voxel_map, max_num_points_in_voxel, initial_voxels ? initial_voxels : max_voxels,
                                                         max_voxels, min_distance_points, &color_), "srl_color_map_create_growable");
    }
    // the colour branch of addPointsToMap (src/lioOptimization.cpp:533-551): every add_point_step-th point of the registered frame
    long long addPointsToColorMap(const double* xyz_world, size_t n, int add_point_step, double time_sweep_end, double time_last_process,
                                  bool to_rendering) {
        int64_t stored = 0;
        check(srl_color_map_add_points(color_, xyz_world, n, add_point_step, time_sweep_end, time_last_process, to_rendering ? 1 : 0, &stored),
              "srl_color_map_add_points");
        return stored;
    }
    // rgbMapTracker::renderPointsInRecentVoxel (src/rgbMapTracker.cpp:216-237); returns render_point_count
    long long renderPointsInRecentVoxel(const srl_camera& cam, const uint8_t* image_bgr, double obs_time) {
        int64_t rendered = 0;
        check(srl_color_map_render_recent(color_, &cam, image_bgr, obs_time, &rendered), "srl_color_map_render_recent");
        return rendered;
    }
    // pubColorPoints (src/lioOptimization.cpp:1210-1241) / saveColorPoints (:1386-1426): the rgb_points_vec entries with
    // N_rgb >= min_views (map_options.pub_point_minimum_views: 1 in config/r3live.yaml, 3 in r3live_compressed.yaml), as xyz
    // (3 floats per point) and r, g, b bytes; publish order from index 0 up, save order from the last index down to 1
    struct ColorPoints { std::vector<float> xyz; std::vector<uint8_t> rgb; };
    ColorPoints pubColorPoints(int min_views) { return exportColorPoints(min_views, 0); }
    ColorPoints saveColorPoints(int min_views) { return exportColorPoints(min_views, 1); }
    // rgbMapTracker::selectPointsForProjection (src/rgbMapTracker.cpp:45-152): ids (point ids, block * block_pts + index) and uv
    // (u_f, v_f per point) of the selected points in point_index order; returns their number.  refreshPointsForProjection is
    // {10, 1, 0, 0.1, 200} from a camera with fov_margin -0.4; the first image uses minimum_dis = track_windows_size /
    // image_scale_factor.  Refresh's early returns (image_cols == 0, the same frame_id) stay with the caller.
    long long selectPointsForProjection(const srl_camera& cam, const srl_projection_params& prm, std::vector<uint32_t>& ids,
                                        std::vector<float>& uv) {
        int64_t nv = 0, np = 0, nrgb = 0, nrec = 0, nnew = 0;
        check(srl_color_map_stats(color_, &nv, &np, &nrgb, &nrec, &nnew), "srl_color_map_stats");
        const int64_t total = (prm.use_all_points || nrec == 0) ? nrgb : nrec;
        const int64_t step = prm.skip_step > 0 ? prm.skip_step : 1;
        const size_t bound = (size_t)((total + step - 1) / step);   // at most one point per candidate
        ids.resize(bound);
        uv.resize(bound * 2);
        int64_t n = 0;
        check(srl_color_map_select_for_projection(color_, &cam, &prm, ids.data(), nullptr, uv.data(), bound, &n),
              "srl_color_map_select_for_projection");
        ids.resize((size_t)n);
        uv.resize((size_t)n * 2);
        return n;
    }
    // the tracked points' state by id (positions: opticalFlowTracker.cpp:25,75,226,280; colour, N_rgb, covariance after each
    // rendering: imageProcessing.cpp:465-478); any output may be nullptr, each holds n * (3, 3, 1, 3) values
    void gatherColorPoints(const std::vector<uint32_t>& ids, float* xyz, int16_t* rgb, int16_t* n_rgb, float* cov) {
        check(srl_color_map_gather_points(color_, ids.data(), ids.size(), xyz, rgb, n_rgb, cov, nullptr), "srl_color_map_gather_points");
    }
    srl_color_map* colorMap() { return color_; }
    srl_ctx* context() { return ctx_; }

private:
    srl_ctx* ctx_ = nullptr;
    srl_map* map_ = nullptr;
    srl_sweep* sweep_ = nullptr;
    srl_color_map* color_ = nullptr;
    srl_cloud_frame* frame_ = nullptr;

    ColorPoints exportColorPoints(int min_views, int order) {
        ColorPoints out;
        int64_t n = 0;
        check(srl_color_map_export(color_, min_views, order, nullptr, nullptr, 0, &n), "srl_color_map_export");
        out.xyz.resize((size_t)n * 3);
        out.rgb.resize((size_t)n * 3);
        if (n) check(srl_color_map_export(color_, min_views, order, out.xyz.data(), out.rgb.data(), (size_t)n, &n), "srl_color_map_export");
        return out;
    }
    void check(int rc, const char* what) {
        if (rc != SRL_OK) throw std::runtime_error(std::string(what) + ": " + (ctx_ ? srl_last_error(ctx_) : "no context"));
    }
    optimizeSummary summarise(int rc, const srl_iekf_summary& sm) {
        optimizeSummary s;
        s.num_residuals_used = sm.num_residuals_used; s.passes_run = sm.passes_run; s.converged = sm.converged != 0;
        if (rc == SRL_NAN_PLANARITY) throw std::runtime_error("error");
        if (rc == SRL_TOO_FEW_RESIDUALS) { s.success = false; s.error_log = srl_last_error(ctx_); return s; }
        check(rc, "srl_update_iekf");
        s.success = sm.success != 0;
        return s;
    }
};

// LKOpticalFlowKernel (include/lkpyramid.h:65-131) on the GPU, bit for bit: the constructor takes the reference's arguments
// and defaults (criteria = (type, max_count, epsilon) of cv::TermCriteria, SRL_LK_COUNT | SRL_LK_EPS), trackImage mirrors
// src/lkpyramid.cpp:755.  Points are (x, y) float pairs, the layout of std::vector<cv::Point2f>; every pointer overload takes
// host or device memory.  It may be destroyed before or after its context.
class LKOpticalFlowKernel {
public:
    LKOpticalFlowKernel(srl_ctx* ctx, int win_w = 21, int win_h = 21, int maxLevel = 3, int criteria_type = SRL_LK_COUNT | SRL_LK_EPS,
                        int max_count = 30, double epsilon = 0.01, int flags = 0, double minEigThreshold = 1e-4)
        : ctx_(ctx) {
        const srl_lk_params p{win_w, win_h, maxLevel, criteria_type, max_count, epsilon, flags, minEigThreshold};
        check(srl_lk_create(ctx, &p, &lk_), "srl_lk_create");
    }
    ~LKOpticalFlowKernel() { if (lk_) srl_lk_destroy(lk_); }
    LKOpticalFlowKernel(const LKOpticalFlowKernel&) = delete;
    LKOpticalFlowKernel& operator=(const LKOpticalFlowKernel&) = delete;

    // trackImage(curr_img, last_tracked_pts, curr_tracked_pts, status): curr_pts is resized to n, status to n except on the
    // first image (which only builds the pyramid and returns 0, as the reference does); returns the number of tracked points
    int trackImage(const uint8_t* gray, int cols, int rows, size_t pitch, const std::vector<float>& last_xy, std::vector<float>& curr_xy,
                   std::vector<uint8_t>& status) {
        const size_t n = last_xy.size() / 2;
        curr_xy.resize(n * 2);
        int32_t ml = 0, c0 = 0, r0 = 0;
        check(srl_lk_info(lk_, &ml, &c0, &r0), "srl_lk_info");
        std::vector<uint8_t> untouched;     // the first image leaves the caller's status as it is
        if (c0 != 0) status.assign(n, 1);   // later images: status is resized, every entry starts at 1
        else untouched.assign(n, 1);
        int64_t k = 0;
        check(srl_lk_track_image(lk_, gray, cols, rows, pitch, last_xy.data(), n, curr_xy.data(), c0 != 0 ? status.data() : untouched.data(), &k),
              "srl_lk_track_image");
        return (int)k;
    }
    // device (or host) buffers of n points, e.g. the selection's device uv straight in
    int trackImage(const uint8_t* gray, int cols, int rows, size_t pitch, const float* last_xy, size_t n, float* curr_xy, uint8_t* status) {
        int64_t k = 0;
        check(srl_lk_track_image(lk_, gray, cols, rows, pitch, last_xy, n, curr_xy, status, &k), "srl_lk_track_image");
        return (int)k;
    }
    int getMaxLevel() {
        int32_t ml = 0;
        check(srl_lk_info(lk_, &ml, nullptr, nullptr), "srl_lk_info");
        return ml;
    }

    srl_lk* handle() { return lk_; }

private:
    srl_ctx* ctx_ = nullptr;
    srl_lk* lk_ = nullptr;
    void check(int rc, const char* what) {
        if (rc != SRL_OK) throw std::runtime_error(std::string(what) + ": " + (ctx_ ? srl_last_error(ctx_) : "no context"));
    }
};

// opticalFlowTracker's bookkeeping (src/opticalFlowTracker.cpp) on the GPU: last, the match list and cur kept on the device in
// point-id order from one image to the next.  The caller's RANSACs plug in between: findFundamentalMat on matches() ->
// rejectMatches(mask); solvePnPRansac on current() -> removeOutlierUsingRansacPnp(inliers).  Pointers are host or device
// memory; the sets' pointers are device memory, valid until the next call.  Destroy before the map, the kernel and the context.
class OpticalFlowTracker {
public:
    OpticalFlowTracker(srl_ctx* ctx, srl_color_map* cm, LKOpticalFlowKernel& lk, int maximum_tracked_points = 300) : ctx_(ctx) {
        check(srl_flow_tracker_create(ctx, cm, lk.handle(), maximum_tracked_points, &t_), "srl_flow_tracker_create");
    }
    ~OpticalFlowTracker() { if (t_) srl_flow_tracker_destroy(t_); }
    OpticalFlowTracker(const OpticalFlowTracker&) = delete;
    OpticalFlowTracker& operator=(const OpticalFlowTracker&) = delete;

    void init(const uint8_t* gray, int cols, int rows, size_t pitch, double time, const uint32_t* ids, const float* uv, size_t n) {
        check(srl_flow_tracker_init(t_, gray, cols, rows, pitch, time, ids, uv, n), "srl_flow_tracker_init");
    }
    // returns whether Lucas-Kanade ran (30 points or more in last)
    bool trackImage(const uint8_t* gray, int cols, int rows, size_t pitch, double time) {
        int32_t called = 0;
        check(srl_flow_tracker_track_image(t_, gray, cols, rows, pitch, time, &called), "srl_flow_tracker_track_image");
        return called != 0;
    }
    void rejectMatches(const uint8_t* mask, size_t n) { check(srl_flow_tracker_reject_matches(t_, mask, n), "srl_flow_tracker_reject_matches"); }
    bool removeOutlierUsingRansacPnp(const int32_t* inliers, size_t n) {
        int32_t r = 0;
        check(srl_flow_tracker_remove_outliers(t_, inliers, n, &r), "srl_flow_tracker_remove_outliers");
        return r != 0;
    }
    void updateAndAppendTrackPoints(const srl_camera& cam, double mini_distance, const uint32_t* candidates, size_t n) {
        check(srl_flow_tracker_update_and_append(t_, &cam, mini_distance, candidates, n), "srl_flow_tracker_update_and_append");
    }
    srl_flow_tracker_sets_out sets() {
        srl_flow_tracker_sets_out s{};
        check(srl_flow_tracker_sets(t_, &s), "srl_flow_tracker_sets");
        return s;
    }

private:
    srl_ctx* ctx_ = nullptr;
    srl_flow_tracker* t_ = nullptr;
    void check(int rc, const char* what) {
        if (rc != SRL_OK) throw std::runtime_error(std::string(what) + ": " + (ctx_ ? srl_last_error(ctx_) : "no context"));
    }
};

// The image preparation of imageProcessing::process (src/imageProcessing.cpp:91-125) on the GPU, bit for bit OpenCV's: the
// constructor is the first-image step for inputs of cols x rows, process() turns one BGR8 image into rgb_image (BGR8) and
// gray_image.  Every pointer takes host or device memory; outputs are contiguous, outputSize() in pixels.  The object may be
// destroyed before or after its context.
class ImageProcessing {
public:
    ImageProcessing(srl_ctx* ctx, int image_width, int image_height, const std::array<double, 9>& camera_intrinsic,
                    const std::array<double, 5>& camera_dist_coeffs, int cols, int rows)
        : ctx_(ctx) {
        srl_image_params p{};
        p.image_width = image_width;
        p.image_height = image_height;
        std::memcpy(p.camera_intrinsic, camera_intrinsic.data(), sizeof(p.camera_intrinsic));
        std::memcpy(p.camera_dist_coeffs, camera_dist_coeffs.data(), sizeof(p.camera_dist_coeffs));
        check(srl_image_create(ctx, &p, cols, rows, &img_), "srl_image_create");
    }
    ~ImageProcessing() { if (img_) srl_image_destroy(img_); }
    ImageProcessing(const ImageProcessing&) = delete;
    ImageProcessing& operator=(const ImageProcessing&) = delete;

    // process:120-125: bgr rows are `pitch` bytes apart (a cv::Mat's step, a ROS image's step)
    void process(const uint8_t* bgr, int cols, int rows, size_t pitch, uint8_t* rgb_out, uint8_t* gray_out) {
        check(srl_image_process(img_, bgr, cols, rows, pitch, rgb_out, gray_out), "srl_image_process");
    }
    // (out_cols, out_rows): the size of rgb_image and gray_image
    std::array<int, 2> outputSize() {
        int32_t c = 0, r = 0;
        check(srl_image_info(img_, &c, &r, nullptr, nullptr, nullptr), "srl_image_info");
        return {c, r};
    }
    // the intrinsics divided by image_scale_factor (row-major), as camera_intrinsic holds them after the first image
    std::array<double, 9> cameraIntrinsic() {
        std::array<double, 9> k{};
        check(srl_image_info(img_, nullptr, nullptr, nullptr, nullptr, k.data()), "srl_image_info");
        return k;
    }
    // imageProcessing::vioEsikf over the tracked set in the caller's order (ids, matched uv float pairs, image_velocity double
    // pairs; host or device); `state` is updated in place, the covariance inside the handle
    bool vioEsikf(srl_color_map* cm, srl_vio_state& state, const uint32_t* ids, const float* uv, const double* velocity, size_t n,
                  int n_new_visited) {
        int32_t r = 0;
        check(srl_image_vio_esikf(img_, cm, &state, ids, uv, velocity, n, n_new_visited, &r), "srl_image_vio_esikf");
        return r != 0;
    }
    // imageProcessing::vioPhotometric on the prepared rgb_image (outputSize(), rows `pitch` bytes apart; host or device)
    bool vioPhotometric(srl_color_map* cm, srl_vio_state& state, const uint32_t* ids, const double* velocity, size_t n, int n_new_visited,
                        const uint8_t* bgr, int cols, int rows, size_t pitch) {
        int32_t r = 0;
        check(srl_image_vio_photometric(img_, cm, &state, ids, velocity, n, n_new_visited, bgr, cols, rows, pitch, &r),
              "srl_image_vio_photometric");
        return r != 0;
    }
    // imageProcessing::covariance, 11 x 11 row-major
    std::array<double, 121> covariance() {
        std::array<double, 121> c{};
        check(srl_image_covariance(img_, nullptr, c.data()), "srl_image_covariance");
        return c;
    }
    void setCovariance(const std::array<double, 121>& c) { check(srl_image_covariance(img_, c.data(), nullptr), "srl_image_covariance"); }

private:
    srl_ctx* ctx_ = nullptr;
    srl_image* img_ = nullptr;
    void check(int rc, const char* what) {
        if (rc != SRL_OK) throw std::runtime_error(std::string(what) + ": " + (ctx_ ? srl_last_error(ctx_) : "no context"));
    }
};

// cloudProcessing (include/cloudProcessing.h, src/cloudProcessing.cpp) on the GPU with its point_buffer kept on the device: the
// constructor takes what lioOptimization::readParameters sets (setLidarType, setNumScans, setScanRate, setTimeUnit, setBlind,
// setPointFilterNum); livoxHandler / process mirror the reference's handlers over the message as it comes off the wire (Livox
// CustomPoint records, PointCloud2 data with the layout msg->fields gives); cut() is getMeasurements' pop loop (front timestamp
// below t) and hands out device pointers that LioBackend::buildFrame / srl_build_frame take as they are, valid until the next
// handler call.  Message pointers take host or device memory.  Not thread-safe: serialise handler calls against cut() and the
// buildFrame that reads its pointers.  It may be destroyed before or after its context.
class cloudProcessing {
public:
    cloudProcessing(srl_ctx* ctx, int lidar_type, int N_SCANS, int SCAN_RATE, int time_unit, double blind, int point_filter_num,
                    size_t initial_capacity = size_t(1) << 18)
        : ctx_(ctx) {
        const srl_lidar_params p{lidar_type, N_SCANS, SCAN_RATE, time_unit, blind, point_filter_num, 0};
        check(srl_lidar_create(ctx, &p, initial_capacity, &l_), "srl_lidar_create");
        lidar_type_ = lidar_type;
    }
    ~cloudProcessing() { if (l_) srl_lidar_destroy(l_); }
    cloudProcessing(const cloudProcessing&) = delete;
    cloudProcessing& operator=(const cloudProcessing&) = delete;

    // livoxHandler(msg, point_buffer): msg->points as n records `stride` bytes apart (19: the packed ROS layout); returns the
    // points appended
    int64_t livoxHandler(const uint8_t* records, size_t n, double stamp, size_t stride = 19) {
        int64_t k = 0;
        check(srl_lidar_livox(l_, records, n, stride, stamp, &k), "srl_lidar_livox");
        return k;
    }
    // process(msg, point_buffer): msg->data of n = width * height points
    int64_t process(const uint8_t* data, size_t n, const srl_cloud2_layout& layout, double stamp) {
        int64_t k = 0;
        check(srl_lidar_process(l_, data, n, &layout, stamp, &k), "srl_lidar_process");
        return k;
    }
    int getLidarType() const { return lidar_type_; }
    double getSweepInterval() { return info().sweep_interval; }
    bool isPointTimeEnable() { return info().given_offset_time != 0; }

    // getMeasurements' pops: while the queue is not empty and front().timestamp < t; returns the count, *raw_xyz / *timestamp
    // point at the popped points on the device (either may be null)
    int64_t cut(double t, const double** raw_xyz = nullptr, const double** timestamp = nullptr) {
        int64_t k = 0;
        check(srl_lidar_cut(l_, t, &k, raw_xyz, timestamp), "srl_lidar_cut");
        return k;
    }
    // what the branches of getMeasurements read of point_buffer (host copies, no device access)
    size_t size() { return (size_t)info().size; }
    bool empty() { return size() == 0; }
    double frontTimestamp() { return info().front_timestamp; }
    double backTimestamp() { return info().back_timestamp; }
    // host copies of the whole queue, front first
    void download(std::vector<double>& raw_xyz, std::vector<double>& relative_time, std::vector<double>& timestamp) {
        const size_t n = size();
        raw_xyz.resize(3 * n);
        relative_time.resize(n);
        timestamp.resize(n);
        check(srl_lidar_download(l_, raw_xyz.data(), relative_time.data(), timestamp.data()), "srl_lidar_download");
    }
    srl_lidar_info info() {
        srl_lidar_info i{};
        check(srl_lidar_info_get(l_, &i), "srl_lidar_info_get");
        return i;
    }

private:
    srl_ctx* ctx_ = nullptr;
    srl_lidar* l_ = nullptr;
    int lidar_type_ = 0;
    void check(int rc, const char* what) {
        if (rc != SRL_OK) throw std::runtime_error(std::string(what) + ": " + (ctx_ ? srl_last_error(ctx_) : "no context"));
    }
};

}  // namespace srl
