// TEST INFRASTRUCTURE (oracle/) — NOT product code.  The two camera updates of imageProcessing::process observed through the
// reference's own code: imageProcessing::vioEsikf (src/imageProcessing.cpp:220-380) and vioPhotometric (:402-552), compiled
// unmodified by oracle/vio.mk and linked with the reference objects of the main recipe into oracle/_ref/libsrl_vio_ref.so.
// Only tests/ and scripts/ load it (tests/vio_ref.py, scripts/bench_vio.py).
//
// The tracked set reaches the updates as op_tracker's two std::map<void*, cv::Point2f> (which removeOutlierUsingRansacPnp
// leaves equal whenever process goes on to the updates).  The rgbPoints live in one contiguous array in the caller's order, so
// the maps iterate in that order.
#include <chrono>

#include "lioOptimization.h"
#include "imageProcessing.h"
#include "opticalFlowTracker.h"
#include "rgbMapTracker.h"

// the tracker's own members are not under test: imageProcessing.o needs only its constructor
opticalFlowTracker::opticalFlowTracker() {}

namespace {

// srl_vio_state's layout: rotation (x,y,z,w), translation, R_imu_camera (row-major), t_imu_camera, fx, fy, cx, cy, time_td,
// q_world_camera, t_world_camera, q_camera_world, t_camera_world: 38 doubles
constexpr int kStateDoubles = 38;

Eigen::Quaterniond q4(const double* q) { return Eigen::Quaterniond(q[3], q[0], q[1], q[2]); }
void put_q(const Eigen::Quaterniond& q, double* o) { o[0] = q.x(); o[1] = q.y(); o[2] = q.z(); o[3] = q.w(); }

void load(const double* s, state& st) {
    st.rotation = q4(s);
    st.translation = Eigen::Vector3d(s[4], s[5], s[6]);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) st.R_imu_camera(r, c) = s[7 + 3 * r + c];
    st.t_imu_camera = Eigen::Vector3d(s[16], s[17], s[18]);
    st.fx = s[19]; st.fy = s[20]; st.cx = s[21]; st.cy = s[22]; st.time_td = s[23];
    st.q_world_camera = q4(s + 24);
    st.t_world_camera = Eigen::Vector3d(s[28], s[29], s[30]);
    st.q_camera_world = q4(s + 31);
    st.t_camera_world = Eigen::Vector3d(s[35], s[36], s[37]);
}

void store(const state& st, double* s) {
    put_q(st.rotation, s);
    for (int k = 0; k < 3; ++k) s[4 + k] = st.translation(k);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) s[7 + 3 * r + c] = st.R_imu_camera(r, c);
    for (int k = 0; k < 3; ++k) s[16 + k] = st.t_imu_camera(k);
    s[19] = st.fx; s[20] = st.fy; s[21] = st.cx; s[22] = st.cy; s[23] = st.time_td;
    put_q(st.q_world_camera, s + 24);
    for (int k = 0; k < 3; ++k) s[28 + k] = st.t_world_camera(k);
    put_q(st.q_camera_world, s + 31);
    for (int k = 0; k < 3; ++k) s[35 + k] = st.t_camera_world(k);
}

}  // namespace

extern "C" {

int vio_ref_state_doubles() { return kStateDoubles; }

// which: 0 vioEsikf, 1 vioPhotometric, 2 both in process's order (:147-153).  state (38 doubles) and cov (11 x 11 row-major)
// are read and written.  Points: xyz (stored floats), uv (matched, floats), vel (doubles), rgb (BGR shorts), cov_rgb (floats),
// n_rgb.  img: rows x cols BGR8 (may be NULL for which 0).  result[0..1]: the return values (-1 where not run).  Returns the
// wall time of the update calls in ns.
int64_t vio_ref_update(int which, double* st_io, double* cov_io, int n, const float* xyz, const float* uv, const double* vel,
                       const int16_t* rgb, const float* cov_rgb, const int16_t* n_rgb, int n_new_visited, const uint8_t* img, int cols,
                       int rows, int32_t* result) {
    static imageProcessing* ip = new imageProcessing();   // one object: its constructor allocates the two trackers
    for (int r = 0; r < 11; ++r)
        for (int c = 0; c < 11; ++c) ip->covariance(r, c) = cov_io[r * 11 + c];
    ip->map_tracker->number_of_new_visited_voxel = n_new_visited;
    std::vector<rgbPoint> pts;
    pts.reserve((size_t)n);
    ip->op_tracker->map_rgb_points_in_last_image_pose.clear();
    ip->op_tracker->map_rgb_points_in_cur_image_pose.clear();
    for (int i = 0; i < n; ++i) {
        pts.emplace_back(Eigen::Vector3d(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]));
        rgbPoint& p = pts.back();
        for (int c = 0; c < 3; ++c) { p.rgb[c] = rgb ? rgb[3 * i + c] : 0; p.cov_rgb(c) = cov_rgb ? cov_rgb[3 * i + c] : 0.f; }
        p.N_rgb = n_rgb ? n_rgb[i] : 0;
        p.image_velocity = Eigen::Vector2d(vel[2 * i], vel[2 * i + 1]);
    }
    for (int i = 0; i < n; ++i) {
        const cv::Point2f m = uv ? cv::Point2f(uv[2 * i], uv[2 * i + 1]) : cv::Point2f(0.f, 0.f);
        ip->op_tracker->map_rgb_points_in_last_image_pose[(void*)&pts[(size_t)i]] = m;
        ip->op_tracker->map_rgb_points_in_cur_image_pose[(void*)&pts[(size_t)i]] = m;
    }
    state st;
    load(st_io, st);
    std::vector<point3D> none;
    cloudFrame frame(none, &st);
    if (img) {
        frame.rgb_image.create(rows, cols, 3);
        std::memcpy(frame.rgb_image.data, img, (size_t)rows * cols * 3);
        frame.image_rows = rows; frame.image_cols = cols;
    }
    result[0] = result[1] = -1;
    const auto t0 = std::chrono::steady_clock::now();
    if (which == 0 || which == 2) result[0] = ip->vioEsikf(&frame) ? 1 : 0;
    if (which == 1 || which == 2) result[1] = ip->vioPhotometric(&frame) ? 1 : 0;
    const auto t1 = std::chrono::steady_clock::now();
    store(st, st_io);
    for (int r = 0; r < 11; ++r)
        for (int c = 0; c < 11; ++c) cov_io[r * 11 + c] = ip->covariance(r, c);
    return (int64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - t0).count();
}

// cloudFrame::getRgb(u, v, 0, &dx, &dy) (src/lioOptimization.cpp:100-140) on a rows x cols BGR8 image: out = value, dx, dy (9)
void vio_ref_get_rgb(const uint8_t* img, int cols, int rows, double u, double v, double* out) {
    state st;
    std::vector<point3D> none;
    cloudFrame frame(none, &st);
    frame.rgb_image.create(rows, cols, 3);
    std::memcpy(frame.rgb_image.data, img, (size_t)rows * cols * 3);
    Eigen::Vector3d dx, dy;
    const Eigen::Vector3d c = frame.getRgb(u, v, 0, &dx, &dy);
    for (int k = 0; k < 3; ++k) { out[k] = c(k); out[3 + k] = dx(k); out[6 + k] = dy(k); }
}

}  // extern "C"
