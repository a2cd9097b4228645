// TEST INFRASTRUCTURE (oracle/) — NOT product code.  The oracle of the published maps: the whole oracle restatement
// (srl_oracle.cpp, included as it is, so its voxel map, colour map and renderer are the very code the other oracle tests
// pin) plus two entry points that restate what the reference publishes and saves.  Built by oracle/publish.mk into
// oracle/_build/libsrl_publish_oracle.so (std::unordered_map container: the published clouds do not depend on the map's
// iteration order); bound by oracle/publish_oracle.py.  Nothing under sr_livo_b200/ may include, link or call it.
#include "srl_oracle.cpp"

/* addPointsToMap + its published cloud (src/lioOptimization.cpp:409-434, addPointToPcl :1346-1355): returns the points stored;
 * xyzi_out (capacity n*4 floats) receives x, y, z, intensity of each published point in sweep order */
extern "C" int64_t orc_map_add_points_published(void* map, const double* xyz, int64_t n, double voxel_size, int32_t max_num_points_in_voxel,
                                                double min_distance_points, int32_t min_num_points, double translation_z, float* xyzi_out,
                                                int64_t* n_published);
/* pubColorPoints (order 0, :1217-1233) / saveColorPoints (order 1, :1393-1419): xyz n*3, rgb n*3 (r,g,b), both NULL = count */
extern "C" int64_t orc_color_export(void* cm, int32_t min_views, int32_t order, float* xyz, uint8_t* rgb);

// ======================================================================================
// The published maps (row A7 / N4 publication):
//   addPointToMap's accept branch (src/lioOptimization.cpp:409-434) with addPointToPcl (:432, :1346-1355): a point is
//     published when it is appended to a voxel that map.find found (a created voxel, :437-444, is not published);
//     intensity = 50 * (float z - translation.z()) evaluated in double, stored as float
//   pubColorPoints (:1217-1233) and saveColorPoints (:1393-1419) over rgb_points_vec: N_rgb >= pub_point_minimum_views,
//     r, g, b = getRgb()[2], [1], [0] (double -> uint8_t: g++ on x86-64 truncates to int32 and keeps the low byte)
// ======================================================================================
namespace {

int addPointToMapPublished(voxelHashMap& map, rgbPoint& point, double voxel_size, int max_num_points_in_voxel, double min_distance_points,
                           int min_num_points, double translation_z, std::vector<float>& points_world) {
    short kx = static_cast<short>(point.getPosition()[0] / voxel_size);
    short ky = static_cast<short>(point.getPosition()[1] / voxel_size);
    short kz = static_cast<short>(point.getPosition()[2] / voxel_size);
    auto search = map.find(voxel(kx, ky, kz));
    if (search != map.end()) {
        voxelBlock& voxel_block = MAP_VALUE(search);
        if (!voxel_block.IsFull()) {
            double sq_dist_min_to_points = 10 * voxel_size * voxel_size;
            for (int i = 0; i < voxel_block.NumPoints(); ++i) {
                double sq_dist = sqnorm3(vsub(voxel_block.points[i].getPosition(), point.getPosition()));
                if (sq_dist < sq_dist_min_to_points) sq_dist_min_to_points = sq_dist;
            }
            if (sq_dist_min_to_points > (min_distance_points * min_distance_points)) {
                if (min_num_points <= 0 || voxel_block.NumPoints() >= min_num_points) {
                    voxel_block.AddPoint(point);
                    const float z = (float)point.getPosition()[2];                      // addPointToPcl: cloudTemp.z
                    points_world.push_back((float)point.getPosition()[0]);
                    points_world.push_back((float)point.getPosition()[1]);
                    points_world.push_back(z);
                    points_world.push_back((float)(50 * ((double)z - translation_z)));   // cloudTemp.intensity
                    return 1;
                }
            }
        }
    } else if (min_num_points <= 0) {
        voxelBlock voxel_block(max_num_points_in_voxel);
        voxel_block.AddPoint(point);
        map[voxel(kx, ky, kz)] = std::move(voxel_block);
        return 1;
    }
    return 0;
}

}  // namespace

extern "C" {

int64_t orc_map_add_points_published(void* map, const double* xyz, int64_t n, double voxel_size, int32_t max_num_points_in_voxel,
                                     double min_distance_points, int32_t min_num_points, double translation_z, float* xyzi_out,
                                     int64_t* n_published) {
    voxelHashMap& m = *static_cast<voxelHashMap*>(map);
    std::vector<float> points_world;   // lioOptimization::points_world
    int64_t added = 0;
    for (int64_t i = 0; i < n; ++i) {
        rgbPoint rgb_point({{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]}});
        added += addPointToMapPublished(m, rgb_point, voxel_size, max_num_points_in_voxel, min_distance_points, min_num_points, translation_z,
                                        points_world);
    }
    if (!points_world.empty()) std::memcpy(xyzi_out, points_world.data(), points_world.size() * sizeof(float));
    *n_published = (int64_t)(points_world.size() / 4);
    return added;
}

int64_t orc_color_export(void* cm_, int32_t min_views, int32_t order, float* xyz, uint8_t* rgb) {
    ColorMap& cm = *static_cast<ColorMap*>(cm_);
    const long point_size = (long)cm.rgb_points.size();
    int64_t count = 0;
    auto emit = [&](long i) {
        const std::array<short, 4>& e = cm.rgb_points[(size_t)i];
        const rgbPoint& p = MAP_VALUE(cm.map.find(voxel(e[0], e[1], e[2]))).points[(size_t)e[3]];
        if (p.N_rgb < min_views) return;
        if (xyz) {
            for (int a = 0; a < 3; ++a) xyz[3 * count + a] = (float)p.getPosition()[a];
            rgb[3 * count] = (uint8_t)(int32_t)(double)p.rgb[2];
            rgb[3 * count + 1] = (uint8_t)(int32_t)(double)p.rgb[1];
            rgb[3 * count + 2] = (uint8_t)(int32_t)(double)p.rgb[0];
        }
        ++count;
    };
    if (order == 0) for (long i = 0; i < point_size; i++) emit(i);    // pubColorPoints (:1217)
    else for (long i = point_size - 1; i > 0; i--) emit(i);           // saveColorPoints (:1398)
    return count;
}

}  // extern "C"
