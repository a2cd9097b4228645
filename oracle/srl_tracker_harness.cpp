// TEST INFRASTRUCTURE (oracle/) — NOT product code.  The map tracker's projection selection observed through the reference's
// own code: rgbMapTracker::selectPointsForProjection (src/rgbMapTracker.cpp:45-152) and refreshPointsForProjection (:26-43)
// after updatePoseForProjection (:154-174), over a colour map filled by the reference's addPointsToMap (src/lioOptimization.cpp
// :520-554) and coloured by renderPointsInRecentVoxel.  oracle/tracker.mk links it with the unmodified reference objects the main
// recipe compiled into _ref/obj/ and srl_reference_harness.cpp (the members of the classes the LIO sources link against) into
// oracle/_ref/libsrl_tracker_ref.so.  Every entry point takes a handle of trk_create.  Only tests/ and scripts/ load it
// (tests/tracker_ref.py).
#include "lioOptimization.h"
#include "imageProcessing.h"
#include "rgbMapTracker.h"

extern std::atomic<long> render_point_count;   // src/rgbMapTracker.cpp:179

namespace {

Eigen::Vector3d v3(const double* p) { return Eigen::Vector3d(p[0], p[1], p[2]); }
Eigen::Quaterniond q4(const double* q) { return Eigen::Quaterniond(q[3], q[0], q[1], q[2]); }   // (x,y,z,w) -> ctor (w,x,y,z)

// a point of color_voxel_map as (voxel key, index in block), the way ref_color_lists names rgb_points_vec's pointers
void key_index_of(lioOptimization* L, rgbPoint* p, int16_t* out) {
    const voxel key = voxel::coordinates(*p, L->map_options.size_voxel_map);   // include/cloudMap.h:138-142
    voxelBlock& block = L->color_voxel_map[key];
    out[0] = key.x; out[1] = key.y; out[2] = key.z;
    out[3] = (int16_t)(p - &block.points[0]);
}

}  // namespace

extern "C" {

void* trk_create(void) { return new lioOptimization(); }   // the reference's constructor over the stub NodeHandle
void trk_destroy(void* lio) { delete static_cast<lioOptimization*>(lio); }

// addPointsToMap (LIO map and colour map, as the reference does it); returns the points stored in the colour map's rgb list
int64_t trk_add_points_to_map(void* lio, const double* world_xyz, int64_t n, double color_voxel_size, int32_t color_max_points,
                              double color_min_distance, int32_t add_point_step, double time_sweep_end, double time_last_process,
                              int32_t to_rendering) {
    lioOptimization* L = static_cast<lioOptimization*>(lio);
    L->map_options.size_voxel_map = color_voxel_size;
    L->map_options.max_num_points_in_voxel = color_max_points;
    L->map_options.min_distance_points = color_min_distance;
    L->map_options.add_point_step = add_point_step;
    L->img_pro->time_last_process = time_last_process;
    std::vector<point3D> pts((size_t)n);
    for (int64_t i = 0; i < n; ++i) pts[(size_t)i].point = v3(world_xyz + 3 * i);
    state st;
    cloudFrame frame(pts, &st);
    frame.time_sweep_end = time_sweep_end;
    L->addPointsToMap(L->voxel_map, &frame, 1.0, 20, 0.15, 0, to_rendering != 0);
    frame.p_state = nullptr;
    return (int64_t)L->img_pro->map_tracker->rgb_points_vec.size();
}

// renderPointsInRecentVoxel over map_tracker->voxels_recent_visited (the twin of ref_color_render).
// cam: q_camera_world (x,y,z,w), t_camera_world, t_world_camera, fx, fy, cx, cy, fov_margin (15 doubles); image BGR u8
int64_t trk_color_render(void* lio, const double* cam, const uint8_t* image_bgr, int32_t rows, int32_t cols, double obs_time) {
    lioOptimization* L = static_cast<lioOptimization*>(lio);
    rgbMapTracker* T = L->img_pro->map_tracker;
    state st;
    st.q_camera_world = q4(cam);
    st.t_camera_world = v3(cam + 4);
    st.t_world_camera = v3(cam + 7);
    st.fx = cam[10]; st.fy = cam[11]; st.cx = cam[12]; st.cy = cam[13]; st.fov_margin = cam[14];
    std::vector<point3D> none;
    cloudFrame frame(none, &st);
    frame.image_rows = rows; frame.image_cols = cols;
    // zero rows below the image: getSubPixel reads row `rows` (with weight 0) for a point at v == rows - 1 exactly, and at
    // u == cols - 1 too the pixel after that row
    frame.rgb_image.create(rows + 2, cols, 3);
    frame.rgb_image.rows = rows;
    std::memcpy(frame.rgb_image.data, image_bgr, (size_t)rows * cols * 3);
    std::vector<voxelId> voxels = T->voxels_recent_visited;
    T->renderPointsInRecentVoxel(L->color_voxel_map, &frame, &voxels, obs_time);
    frame.p_state = nullptr;
    return (int64_t)render_point_count.load();
}

int64_t trk_color_num_recent(void* lio) { return (int64_t) static_cast<lioOptimization*>(lio)->img_pro->map_tracker->voxels_recent_visited.size(); }
int64_t trk_color_num_rgb_points(void* lio) { return (int64_t) static_cast<lioOptimization*>(lio)->img_pro->map_tracker->rgb_points_vec.size(); }

// the reference's own selectPointsForProjection(color_voxel_map, frame, &pc_out_vec, &pc_2d_out_vec, minimum_dis, skip_step,
// use_all_points) with the tracker's depth bounds set to minimum_depth / maximum_depth for the call.  cam as trk_color_render.
// Returns the number of points; when it is <= max_n, key_index (n*4: voxel key, index in block) and uv (n*2) receive them.
int64_t ref_color_select(void* lio, const double* cam, int32_t rows, int32_t cols, double minimum_dis, int32_t skip_step,
                         int32_t use_all_points, double minimum_depth, double maximum_depth, int16_t* key_index, float* uv, int64_t max_n) {
    lioOptimization* L = static_cast<lioOptimization*>(lio);
    rgbMapTracker* T = L->img_pro->map_tracker;
    state st;
    st.q_camera_world = q4(cam);
    st.t_camera_world = v3(cam + 4);
    st.t_world_camera = v3(cam + 7);
    st.fx = cam[10]; st.fy = cam[11]; st.cx = cam[12]; st.cy = cam[13]; st.fov_margin = cam[14];
    std::vector<point3D> none;
    cloudFrame frame(none, &st);
    frame.image_rows = rows; frame.image_cols = cols;
    const double keep_min = T->minimum_depth_for_projection, keep_max = T->maximum_depth_for_projection;
    T->minimum_depth_for_projection = minimum_depth;
    T->maximum_depth_for_projection = maximum_depth;
    std::vector<rgbPoint*> pc_out_vec;
    std::vector<cv::Point2f> pc_2d_out_vec;
    T->selectPointsForProjection(L->color_voxel_map, &frame, &pc_out_vec, &pc_2d_out_vec, minimum_dis, skip_step, use_all_points != 0);
    T->minimum_depth_for_projection = keep_min;
    T->maximum_depth_for_projection = keep_max;
    frame.p_state = nullptr;
    const int64_t n = (int64_t)pc_out_vec.size();
    if (n > max_n || (int64_t)pc_2d_out_vec.size() != n) return n;
    for (int64_t i = 0; i < n; ++i) {
        if (key_index) key_index_of(L, pc_out_vec[(size_t)i], key_index + 4 * i);
        if (uv) { uv[2 * i] = pc_2d_out_vec[(size_t)i].x; uv[2 * i + 1] = pc_2d_out_vec[(size_t)i].y; }
    }
    return n;
}

// what the image thread does before each optical-flow update (src/imageProcessing.cpp:159): updatePoseForProjection(frame, -0.4)
// then refreshPointsForProjection.  The frame has q_world_camera (x,y,z,w), t_world_camera, fx, fy, cx, cy, a rows x cols
// image and frame_id (a frame_id equal to the last refresh's returns early, as in the reference).  q_cw_out (x,y,z,w) and
// t_cw_out receive the q_camera_world / t_camera_world the tracker derived (refreshPoseForProjection).  Returns the size of
// points_rgb_vec_for_projection (-1 when there is none yet); when it is <= max_n, key_index (n*4) receives its points.
int64_t ref_color_refresh(void* lio, const double q_world_camera[4], const double t_world_camera[3], double fx, double fy, double cx, double cy,
                          int32_t rows, int32_t cols, int32_t frame_id, int16_t* key_index, int64_t max_n, double q_cw_out[4], double t_cw_out[3]) {
    lioOptimization* L = static_cast<lioOptimization*>(lio);
    rgbMapTracker* T = L->img_pro->map_tracker;
    state st;
    st.q_world_camera = q4(q_world_camera);
    st.t_world_camera = v3(t_world_camera);
    st.fx = fx; st.fy = fy; st.cx = cx; st.cy = cy;
    std::vector<point3D> none;
    cloudFrame frame(none, &st);
    frame.image_rows = rows; frame.image_cols = cols;
    frame.frame_id = frame_id;
    T->updatePoseForProjection(&frame, -0.4);
    T->refreshPointsForProjection(L->color_voxel_map);
    frame.p_state = nullptr;
    const Eigen::Quaterniond& q = T->p_cloud_frame->p_state->q_camera_world;
    q_cw_out[0] = q.x(); q_cw_out[1] = q.y(); q_cw_out[2] = q.z(); q_cw_out[3] = q.w();
    const Eigen::Vector3d& t = T->p_cloud_frame->p_state->t_camera_world;
    t_cw_out[0] = t(0); t_cw_out[1] = t(1); t_cw_out[2] = t(2);
    if (!T->points_rgb_vec_for_projection) return -1;
    const std::vector<rgbPoint*>& v = *T->points_rgb_vec_for_projection;
    const int64_t n = (int64_t)v.size();
    if (n > max_n) return n;
    if (key_index) for (int64_t i = 0; i < n; ++i) key_index_of(L, v[(size_t)i], key_index + 4 * i);
    return n;
}

}  // extern "C"
