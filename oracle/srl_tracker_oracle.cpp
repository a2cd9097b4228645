// TEST INFRASTRUCTURE (oracle/) — NOT product code.  The oracle of the map tracker's projection selection: the whole oracle
// restatement (srl_oracle.cpp, included as it is, so its colour map and renderer are the very code the other oracle tests
// pin) plus two entry points that restate rgbMapTracker::selectPointsForProjection (src/rgbMapTracker.cpp:45-152) and the
// per-point reads of the tracker.  Built by oracle/tracker.mk into oracle/_build/libsrl_tracker_oracle.so; bound by
// oracle/tracker_oracle.py.  Nothing under sr_livo_b200/ may include, link or call it.
#include <map>

#include "srl_oracle.cpp"

/* selectPointsForProjection: cam = q_camera_world (x,y,z,w), t_camera_world, t_world_camera, fx, fy, cx, cy, fov_margin (15
 * doubles) of a rows x cols image.  Returns the number of selected points; when it is <= max_n, key_index (n*4: voxel key,
 * index in block) and uv (n*2 floats) receive them in point_index order (either may be NULL). */
extern "C" int64_t orc_color_select(void* cm, const double* cam, int32_t rows, int32_t cols, double minimum_dis, int32_t skip_step,
                                    int32_t use_all_points, double minimum_depth, double maximum_depth, int16_t* key_index, float* uv,
                                    int64_t max_n);
/* the state of the points named by key_index (n*4): xyz n*3, rgb n*3 (BGR as stored), n_rgb n, cov n*3 (0 before the first
 * observation).  Returns 0, or -1 (nothing written) when an entry names no stored point. */
extern "C" int32_t orc_color_gather(void* cm, const int16_t* key_index, int64_t n, float* xyz, int16_t* rgb, int16_t* n_rgb, float* cov);

// ======================================================================================
// rgbMapTracker::selectPointsForProjection (src/rgbMapTracker.cpp:45-152), sequential, with the reference's containers:
//   candidates: map[key].points.back() of every voxels_recent_visited entry in list order (a repeated voxel is one candidate
//     per repetition), or rgb_points_vec when use_all_points is set or the list is empty (:72-89)
//   depth = (point_world - t_world_camera).norm() against the tracker's depth bounds (:97-107), then
//   project3dPointInThisImage with scale 1 (:109, src/lioOptimization.cpp:142-198: the renderer's projection)
//   cell u = std::round(u_f / minimum_dis) * minimum_dis as int (:116-117); Hash_map_2d mask_index / mask_depth (nested
//     std::unordered_map, include/utility.h:143-168), the depth stored as float, compared against the double depth (:119)
//   the winners by point_index in a std::map (:61-62, :129-151)
// ======================================================================================
namespace {

struct Hash2d {   // Hash_map_2d<int, T>::if_exist (include/utility.h:155-168)
    template <class M> static bool exist(M& m, int x, int y) {
        auto a = m.find(x);
        if (a == m.end()) return false;
        return a->second.find(y) != a->second.end();
    }
};

const rgbPoint* find_point(ColorMap& cm, const int16_t* e) {
    auto it = cm.map.find(voxel(e[0], e[1], e[2]));
    if (it == cm.map.end()) return nullptr;
    const voxelBlock& b = MAP_VALUE(it);
    if (e[3] < 0 || e[3] >= b.NumPoints()) return nullptr;
    return &b.points[(size_t)e[3]];
}

}  // namespace

extern "C" {

int64_t orc_color_select(void* cm_, const double* cam, int32_t rows, int32_t cols, double minimum_dis, int32_t skip_step,
                         int32_t use_all_points, double minimum_depth, double maximum_depth, int16_t* key_index, float* uv,
                         int64_t max_n) {
    ColorMap& cm = *static_cast<ColorMap*>(cm_);
    const Mat3 R = quat_to_rot({cam[0], cam[1], cam[2], cam[3]});
    const Vec3 t_cw = {{cam[4], cam[5], cam[6]}}, t_wc = {{cam[7], cam[8], cam[9]}};
    const double fx = cam[10], fy = cam[11], cx = cam[12], cy = cam[13], fov_margin = cam[14];

    std::unordered_map<int, std::unordered_map<int, int>> mask_index;
    std::unordered_map<int, std::unordered_map<int, float>> mask_depth;
    std::map<int, std::array<float, 2>> map_idx_draw_center_raw_pose;

    // points_for_projection as (voxel key, index in block); a listed key without a voxel never occurs (the reference's
    // map[] would insert an empty voxel there, which NumPoints() > 0 then skips)
    std::vector<std::array<short, 4>> points_for_projection;
    if (!use_all_points && !cm.recent.empty()) {
        for (const voxelId& id : cm.recent) {
            auto it = cm.map.find(voxel((short)id.kx, (short)id.ky, (short)id.kz));
            if (it != cm.map.end() && MAP_VALUE(it).NumPoints() > 0)
                points_for_projection.push_back({{(short)id.kx, (short)id.ky, (short)id.kz, (short)(MAP_VALUE(it).NumPoints() - 1)}});
        }
    } else {
        points_for_projection = cm.rgb_points;
    }

    const int point_size = (int)points_for_projection.size();
    for (int point_index = 0; point_index < point_size; point_index += skip_step) {
        const std::array<short, 4>& e = points_for_projection[(size_t)point_index];
        const rgbPoint& point = MAP_VALUE(cm.map.find(voxel(e[0], e[1], e[2]))).points[(size_t)e[3]];
        const Vec3 point_world = point.getPosition();
        const double depth = norm3(vsub(point_world, t_wc));
        if (depth > maximum_depth) continue;
        if (depth < minimum_depth) continue;
        // project3dTo2d (src/lioOptimization.cpp:142-161), scale 1
        const Vec3 pc = vadd(matvec(R, point_world), t_cw);
        if (pc[2] < 0.001) continue;
        const double u_f = (pc[0] * fx / pc[2] + cx) * 1.0;
        const double v_f = (pc[1] * fy / pc[2] + cy) * 1.0;
        // if2dPointsAvailable (:48-60) with fov_mar = -1: the frame's own fov_margin
        if (!((u_f / 1.0 >= (fov_margin * cols + 1)) && (std::ceil(u_f / 1.0) < ((1 - fov_margin) * cols)) &&
              (v_f / 1.0 >= (fov_margin * rows + 1)) && (std::ceil(v_f / 1.0) < ((1 - fov_margin) * rows)))) continue;
        const int u = std::round(u_f / minimum_dis) * minimum_dis;
        const int v = std::round(v_f / minimum_dis) * minimum_dis;
        if ((!Hash2d::exist(mask_depth, u, v)) || mask_depth[u][v] > depth) {
            if (Hash2d::exist(mask_index, u, v)) {
                const int old_idx = mask_index[u][v];
                map_idx_draw_center_raw_pose.erase(map_idx_draw_center_raw_pose.find(old_idx));
            }
            mask_index[u][v] = point_index;
            mask_depth[u][v] = (float)depth;
            map_idx_draw_center_raw_pose[point_index] = {{(float)u_f, (float)v_f}};
        }
    }

    const int64_t n = (int64_t)map_idx_draw_center_raw_pose.size();
    if (n > max_n) return n;
    int64_t k = 0;
    for (const auto& kv : map_idx_draw_center_raw_pose) {
        if (key_index) for (int a = 0; a < 4; ++a) key_index[4 * k + a] = points_for_projection[(size_t)kv.first][(size_t)a];
        if (uv) { uv[2 * k] = kv.second[0]; uv[2 * k + 1] = kv.second[1]; }
        ++k;
    }
    return n;
}

int32_t orc_color_gather(void* cm_, const int16_t* key_index, int64_t n, float* xyz, int16_t* rgb, int16_t* n_rgb, float* cov) {
    ColorMap& cm = *static_cast<ColorMap*>(cm_);
    for (int64_t i = 0; i < n; ++i)
        if (!find_point(cm, key_index + 4 * i)) return -1;
    for (int64_t i = 0; i < n; ++i) {
        const rgbPoint& p = *find_point(cm, key_index + 4 * i);
        for (int a = 0; a < 3; ++a) {
            xyz[3 * i + a] = p.position[a];
            rgb[3 * i + a] = p.rgb[a];
            cov[3 * i + a] = p.N_rgb != 0 ? p.cov_rgb[a] : 0.f;   // cov_rgb is uninitialised before the first view; a wrapped (negative) N_rgb has one
        }
        n_rgb[i] = p.N_rgb;
    }
    return 0;
}

}  // extern "C"
