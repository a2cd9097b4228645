// TEST INFRASTRUCTURE (oracle/) — NOT product code.  The optical-flow tracker's bookkeeping observed through the reference's own
// code: opticalFlowTracker::init, trackImage, removeOutlierUsingRansacPnp and updateAndAppendTrackPoints
// (src/opticalFlowTracker.cpp), compiled unmodified by oracle/flow_tracker.mk into oracle/_ref/libsrl_flow_tracker_ref.so.
// Only tests/ and scripts/ load it (tests/flow_tracker_ref.py).
//
// The rgbPoints live in one array indexed by point id, so std::map<void*, ...> iterates in id order.  Stand-ins:
//   * LKOpticalFlowKernel::trackImage calls the test's function with the points it is given (Lucas-Kanade itself is pinned by
//     row N6); the constructor's setTerminationCriteria does nothing.
//   * cv::findFundamentalMat fills its status from the test's mask function (all ones without one).
//   * cv::solvePnPRansac returns the test's inliers, or throws cv::Exception.
//   * cv::cvtColor does nothing.
#include <chrono>

#include "lioOptimization.h"
#include "opticalFlowTracker.h"
#include "rgbMapTracker.h"

extern "C" {
typedef void (*ft_lk_fn)(int n, const float* last_xy, float* cur_xy, uint8_t* status);
typedef void (*ft_mask_fn)(int n, uint8_t* mask);
}

namespace {
ft_lk_fn g_lk = nullptr;
ft_mask_fn g_mask = nullptr;
std::vector<int> g_inliers;
bool g_throw = false;
long g_lk_calls = 0;

struct FtRef {
    std::vector<rgbPoint> pts;
    opticalFlowTracker tr;
    rgbMapTracker mt;
    state st;
    std::vector<point3D> none;
    std::vector<rgbPoint*> proj;
    double time = 0.0;
};

void frame_setup(FtRef* h, cloudFrame& f, double time, int cols, int rows) {
    f.rgb_image.create(1, 1, 3);       // trackImage returns early on an empty image
    f.gray_image.create(1, 1, 1);
    f.time_sweep_end = time;
    f.image_cols = cols;
    f.image_rows = rows;
}
}  // namespace

void LKOpticalFlowKernel::setTerminationCriteria(cv::TermCriteria&) {}
int LKOpticalFlowKernel::trackImage(const cv::Mat&, const std::vector<cv::Point2f>& last, std::vector<cv::Point2f>& cur,
                                    std::vector<uchar>& status, int) {
    ++g_lk_calls;
    const int n = (int)last.size();
    cur = last;
    status.assign((size_t)n, 1);
    if (g_lk && n) g_lk(n, reinterpret_cast<const float*>(last.data()), reinterpret_cast<float*>(cur.data()), status.data());
    int k = 0;
    for (uchar s : status) k += s;
    return k;
}
namespace cv {
void cvtColor(const Mat&, Mat&, int) {}
Mat findFundamentalMat(const std::vector<Point2f>& p1, const std::vector<Point2f>&, int, double, double, std::vector<uchar>& mask) {
    mask.assign(p1.size(), 1);
    if (g_mask && !p1.empty()) g_mask((int)p1.size(), mask.data());
    return Mat();
}
bool solvePnPRansac(const std::vector<Point3f>&, const std::vector<Point2f>&, const Mat&, const Mat&, Mat&, Mat&, bool, int, float, double,
                    std::vector<int>& inliers) {
    if (g_throw) throw Exception("solvePnPRansac stand-in: the test's RANSAC failed");
    inliers = g_inliers;
    return true;
}
}  // namespace cv

extern "C" {

void ft_ref_set_callbacks(ft_lk_fn lk, ft_mask_fn mask) { g_lk = lk; g_mask = mask; }
long ft_ref_lk_calls() { return g_lk_calls; }

// n_points rgbPoints at xyz (stored floats), point id = index; maximum_tracked_points as given
void* ft_ref_create(int max_points, int n_points, const float* xyz) {
    FtRef* h = new FtRef();
    h->pts.reserve((size_t)n_points);
    for (int i = 0; i < n_points; ++i) h->pts.emplace_back(Eigen::Vector3d(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]));
    h->tr.maximum_tracked_points = (unsigned)max_points;
    return h;
}
void ft_ref_destroy(void* p) { delete static_cast<FtRef*>(p); }

void ft_ref_set_counts(void* p, const uint32_t* ids, int n, const int16_t* c) {
    FtRef* h = static_cast<FtRef*>(p);
    for (int i = 0; i < n; ++i) h->pts[ids[i]].is_out_lier_count = c[i];
}
void ft_ref_get_counts(void* p, const uint32_t* ids, int n, int16_t* c) {
    FtRef* h = static_cast<FtRef*>(p);
    for (int i = 0; i < n; ++i) c[i] = h->pts[ids[i]].is_out_lier_count;
}

// init(p_frame, rgb_points_vec, points_2d_vec) (:188-197); returns its wall time in ns
int64_t ft_ref_init(void* p, double time, const uint32_t* ids, const float* uv, int n) {
    FtRef* h = static_cast<FtRef*>(p);
    std::vector<rgbPoint*> v;
    std::vector<cv::Point2f> uv2;
    for (int i = 0; i < n; ++i) { v.push_back(&h->pts[ids[i]]); uv2.push_back(cv::Point2f(uv[2 * i], uv[2 * i + 1])); }
    cloudFrame f(h->none, &h->st);
    frame_setup(h, f, time, 1, 1);
    const auto t0 = std::chrono::steady_clock::now();
    h->tr.init(&f, v, uv2);
    return (int64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
}
// trackImage(p_frame, -20) on a cols x rows frame at `time` (:111-186)
int64_t ft_ref_track(void* p, double time, int cols, int rows) {
    FtRef* h = static_cast<FtRef*>(p);
    cloudFrame f(h->none, &h->st);
    frame_setup(h, f, time, cols, rows);
    const auto t0 = std::chrono::steady_clock::now();
    h->tr.trackImage(&f, -20);
    return (int64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
}
// removeOutlierUsingRansacPnp(p_frame, 1) (:267-323): inliers (n indices into cur's order; NULL = all of cur), or a throwing
// RANSAC; *result = its return value
int64_t ft_ref_remove_outliers(void* p, const int32_t* inliers, int n, int throws, int32_t* result) {
    FtRef* h = static_cast<FtRef*>(p);
    g_inliers.clear();
    if (inliers) g_inliers.assign(inliers, inliers + n);
    else for (int i = 0; i < (int)h->tr.map_rgb_points_in_cur_image_pose.size(); ++i) g_inliers.push_back(i);
    g_throw = throws != 0;
    cloudFrame f(h->none, &h->st);
    frame_setup(h, f, h->time, 1, 1);
    const auto t0 = std::chrono::steady_clock::now();
    *result = h->tr.removeOutlierUsingRansacPnp(&f, 1) ? 1 : 0;
    const int64_t ns = (int64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
    g_throw = false;
    return ns;
}
// updateAndAppendTrackPoints(p_frame, map_tracker, mini_distance) (:13-102).  cam15: q_camera_world (x, y, z, w),
// t_camera_world, t_world_camera, fx, fy, cx, cy, fov_margin; candidates = points_rgb_vec_for_projection
int64_t ft_ref_update(void* p, const double* c, int cols, int rows, double mini_distance, const uint32_t* cand, int n) {
    FtRef* h = static_cast<FtRef*>(p);
    h->st.q_camera_world = Eigen::Quaterniond(c[3], c[0], c[1], c[2]);
    h->st.t_camera_world = Eigen::Vector3d(c[4], c[5], c[6]);
    h->st.t_world_camera = Eigen::Vector3d(c[7], c[8], c[9]);
    h->st.fx = c[10]; h->st.fy = c[11]; h->st.cx = c[12]; h->st.cy = c[13]; h->st.fov_margin = c[14];
    h->proj.clear();
    for (int i = 0; i < n; ++i) h->proj.push_back(&h->pts[cand[i]]);
    h->mt.points_rgb_vec_for_projection = &h->proj;
    cloudFrame f(h->none, &h->st);
    frame_setup(h, f, h->time, cols, rows);
    const auto t0 = std::chrono::steady_clock::now();
    h->tr.updateAndAppendTrackPoints(&f, &h->mt, mini_distance);
    return (int64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
}
// which 0: last, 1: cur (with each point's image_velocity); returns the set's size, fills the outputs when they are not NULL
int ft_ref_get(void* p, int which, uint32_t* ids, float* uv, double* vel) {
    FtRef* h = static_cast<FtRef*>(p);
    const auto& m = which ? h->tr.map_rgb_points_in_cur_image_pose : h->tr.map_rgb_points_in_last_image_pose;
    int k = 0;
    for (const auto& e : m) {
        const rgbPoint* rp = static_cast<const rgbPoint*>(e.first);
        if (ids) ids[k] = (uint32_t)(rp - h->pts.data());
        if (uv) { uv[2 * k] = e.second.x; uv[2 * k + 1] = e.second.y; }
        if (vel) { vel[2 * k] = rp->image_velocity(0); vel[2 * k + 1] = rp->image_velocity(1); }
        ++k;
    }
    return k;
}

}  // extern "C"
