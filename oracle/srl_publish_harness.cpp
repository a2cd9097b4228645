// TEST INFRASTRUCTURE (oracle/) — NOT product code.  The clouds the reference publishes and saves, observed through its own
// code: lioOptimization::addPointsToMap (src/lioOptimization.cpp:520-554, the registered cloud publishCLoudWorld sends at
// :552 before :553 clears it), pubColorPoints (:1210-1241) and saveColorPoints (:1386-1426).  oracle/publish.mk compiles
// lioOptimization.cpp unmodified with oracle/srl_publish_capture.h force-included, so its calls of the stand-ins of
// pcl::toROSMsg and pcl::io::savePCDFileBinary (oracle/shim/srl_shim_ext.h) reach the specializations defined below, and
// links it with the other unmodified reference objects, srl_reference_harness.cpp (the members of the classes the LIO
// sources link against) and this file into oracle/_ref/libsrl_publish_ref.so.  Only tests/ load it (tests/publish_ref.py).
#include "lioOptimization.h"
#include "imageProcessing.h"
#include "rgbMapTracker.h"

extern std::atomic<long> render_point_count;   // src/rgbMapTracker.cpp:179

namespace {
std::vector<pcl::PointXYZI> g_cloud_xyzi;      // the last cloud of each kind, and how many were handed over
std::vector<pcl::PointXYZRGB> g_cloud_rgb, g_pcd;
long g_n_xyzi = 0, g_n_rgb = 0, g_n_pcd = 0;

Eigen::Vector3d v3(const double* p) { return Eigen::Vector3d(p[0], p[1], p[2]); }
Eigen::Quaterniond q4(const double* q) { return Eigen::Quaterniond(q[3], q[0], q[1], q[2]); }   // (x,y,z,w) -> ctor (w,x,y,z)

int64_t copy_rgb(const std::vector<pcl::PointXYZRGB>& c, float* xyz, uint8_t* rgb) {
    if (xyz)
        for (size_t i = 0; i < c.size(); ++i) {
            xyz[3 * i] = c[i].x; xyz[3 * i + 1] = c[i].y; xyz[3 * i + 2] = c[i].z;
            rgb[3 * i] = c[i].r; rgb[3 * i + 1] = c[i].g; rgb[3 * i + 2] = c[i].b;
        }
    return (int64_t)c.size();
}
}  // namespace

// the specializations oracle/srl_publish_capture.h declares: each keeps the cloud it is handed and counts the hand-over
namespace pcl {
template <> void toROSMsg<PointCloud<PointXYZI>>(const PointCloud<PointXYZI>& cloud, sensor_msgs::PointCloud2&) {
    g_cloud_xyzi = cloud.points; ++g_n_xyzi;
}
template <> void toROSMsg<PointCloud<PointXYZRGB>>(const PointCloud<PointXYZRGB>& cloud, sensor_msgs::PointCloud2&) {
    g_cloud_rgb = cloud.points; ++g_n_rgb;
}
namespace io {
template <> int savePCDFileBinary<PointCloud<PointXYZRGB>>(const std::string&, const PointCloud<PointXYZRGB>& cloud) {
    g_pcd = cloud.points; ++g_n_pcd;
    return 0;
}
}  // namespace io
}  // namespace pcl

extern "C" {

void* pub_create(void) { return new lioOptimization(); }   // the reference's constructor over the stub NodeHandle
void pub_destroy(void* lio) { delete static_cast<lioOptimization*>(lio); }

// addPointsToMap (LIO map and colour map, as the reference does it) on a frame whose state has translation (0, 0, translation_z);
// xyzi_out (capacity n*4) receives the cloud publishCLoudWorld sent.  Returns the points stored in the LIO map, -1 when the
// call did not publish exactly one cloud.
int64_t pub_add_points_to_map(void* lio, const double* world_xyz, int64_t n, double voxel_size, int32_t max_num_points_in_voxel,
                              double min_distance_points, int32_t min_num_points, double translation_z, double color_voxel_size,
                              int32_t color_max_points, double color_min_distance, int32_t add_point_step, double time_sweep_end,
                              double time_last_process, int32_t to_rendering, float* xyzi_out, int64_t* n_published) {
    lioOptimization* L = static_cast<lioOptimization*>(lio);
    L->map_options.size_voxel_map = color_voxel_size;
    L->map_options.max_num_points_in_voxel = color_max_points;
    L->map_options.min_distance_points = color_min_distance;
    L->map_options.add_point_step = add_point_step;
    L->img_pro->time_last_process = time_last_process;
    std::vector<point3D> pts((size_t)n);
    for (int64_t i = 0; i < n; ++i) pts[(size_t)i].point = v3(world_xyz + 3 * i);
    state st;
    st.translation = Eigen::Vector3d(0.0, 0.0, translation_z);
    cloudFrame frame(pts, &st);
    frame.time_sweep_end = time_sweep_end;
    const int64_t before = (int64_t)L->mapSize(L->voxel_map);
    const long calls = g_n_xyzi;
    L->addPointsToMap(L->voxel_map, &frame, voxel_size, max_num_points_in_voxel, min_distance_points, min_num_points, to_rendering != 0);
    frame.p_state = nullptr;
    if (g_n_xyzi != calls + 1) return -1;
    for (size_t i = 0; i < g_cloud_xyzi.size(); ++i) {
        const pcl::PointXYZI& p = g_cloud_xyzi[i];
        xyzi_out[4 * i] = p.x; xyzi_out[4 * i + 1] = p.y; xyzi_out[4 * i + 2] = p.z; xyzi_out[4 * i + 3] = p.intensity;
    }
    *n_published = (int64_t)g_cloud_xyzi.size();
    return (int64_t)L->mapSize(L->voxel_map) - before;
}

// rgbMapTracker::renderPointsInRecentVoxel over map_tracker->voxels_recent_visited (the twin of ref_color_render).
// cam: q_camera_world (x,y,z,w), t_camera_world, t_world_camera, fx, fy, cx, cy, fov_margin (15 doubles); image BGR u8
int64_t pub_color_render(void* lio, const double* cam, const uint8_t* image_bgr, int32_t rows, int32_t cols, double obs_time) {
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
    frame.rgb_image.create(rows, cols, 3);
    std::memcpy(frame.rgb_image.data, image_bgr, (size_t)rows * cols * 3);
    std::vector<voxelId> voxels = T->voxels_recent_visited;
    T->renderPointsInRecentVoxel(L->color_voxel_map, &frame, &voxels, obs_time);
    frame.p_state = nullptr;
    return (int64_t)render_point_count.load();
}

int64_t pub_color_num_rgb_points(void* lio) { return (int64_t) static_cast<lioOptimization*>(lio)->img_pro->map_tracker->rgb_points_vec.size(); }

// order 0: pubColorPoints, order 1: saveColorPoints, with map_options.pub_point_minimum_views = min_views.  xyz / rgb (r, g, b;
// may be NULL) receive the captured cloud; returns its size, -1 when the call did not hand over exactly one cloud.
int64_t pub_color_export(void* lio, int32_t min_views, int32_t order, float* xyz, uint8_t* rgb) {
    lioOptimization* L = static_cast<lioOptimization*>(lio);
    L->map_options.pub_point_minimum_views = min_views;
    if (order == 0) {
        const long calls = g_n_rgb;
        state st;
        std::vector<point3D> none;
        cloudFrame frame(none, &st);
        ros::Publisher pub;
        L->pubColorPoints(pub, &frame);
        frame.p_state = nullptr;
        return g_n_rgb == calls + 1 ? copy_rgb(g_cloud_rgb, xyz, rgb) : -1;
    }
    const long calls = g_n_pcd;
    L->saveColorPoints();
    return g_n_pcd == calls + 1 ? copy_rgb(g_pcd, xyz, rgb) : -1;
}

}  // extern "C"
