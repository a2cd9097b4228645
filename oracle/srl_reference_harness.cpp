// TEST INFRASTRUCTURE (oracle/) — NOT product code.  C entry points around the REFERENCE's own LIO sources, compiled
// unmodified from where they lie (/root/reference/src/{optimize,utility,eskfEstimator,cloudMap,state,lioOptimization,
// rgbMapTracker,parameters}.cpp) into oracle/_ref/libsrl_reference.so by oracle/Makefile (target `reference`).
//
// The reference cannot be built with its own toolchain here (no Eigen, PCL, OpenCV, ROS, Ceres in the image, no network);
// the headers under oracle/shim/ stand in for them: declaration-only stubs for ROS / PCL / tf / Ceres, a minimal cv::Mat /
// cv::Vec3b, and a small Eigen look-alike (oracle/shim/Eigen/Core).  So what runs here is the reference's OWN code — its
// loops, casts, containers (tsl::robin_map, std::tr1::unordered_map, std::priority_queue), member functions and quirks —
// on top of a restated Eigen / OpenCV arithmetic.  tests/test_reference_pin.py checks the oracle restatement
// (oracle/srl_oracle.cpp) against it; the arithmetic INSIDE Eigen / OpenCV calls stays unpinned (DESIGN.md §2).
//
// Nothing here is reachable from sr_livo_b200/ (the product); only tests/ and bench.py's reference arm load this library.
#include "lioOptimization.h"
#include "imageProcessing.h"
#include "rgbMapTracker.h"
#include "cloudProcessing.h"
#include "srl_oracle.h"   // the plain-C structs shared with the oracle's interface (orc_icp_params, orc_eskf_state, ...)

extern std::atomic<long> render_point_count;   // src/rgbMapTracker.cpp:179

// ---- members of the reference's sensor-decoding / vision classes that lioOptimization.cpp links against but the LIO
//      scan-matching path never runs (src/cloudProcessing.cpp, src/imageProcessing.cpp are NOT compiled: they need the
//      real PCL / OpenCV).  Constructors keep the reference's initial values that the compiled code reads.
cloudProcessing::cloudProcessing() { lidar_type = LIVOX; }
void cloudProcessing::setLidarType(int para) { lidar_type = para; }
void cloudProcessing::setNumScans(int para) { N_SCANS = para; }
void cloudProcessing::setScanRate(int para) { SCAN_RATE = para; }
void cloudProcessing::setTimeUnit(int para) { time_unit = para; }
void cloudProcessing::setBlind(double para) { blind = para; }
void cloudProcessing::setExtrinR(Eigen::Matrix3d& R) { R_imu_lidar = R; }
void cloudProcessing::setExtrinT(Eigen::Vector3d& t) { t_imu_lidar = t; }
void cloudProcessing::setPointFilterNum(int para) { point_filter_num = para; }
void cloudProcessing::process(const sensor_msgs::PointCloud2::ConstPtr&, std::queue<point3D>&) { throw std::logic_error("cloudProcessing::process: not part of the harness"); }
void cloudProcessing::livoxHandler(const livox_ros_driver::CustomMsg::ConstPtr&, std::queue<point3D>&) { throw std::logic_error("cloudProcessing::livoxHandler: not part of the harness"); }
imageProcessing::imageProcessing() {
    time_last_process = -1e5;          // src/imageProcessing.cpp:7
    op_tracker = nullptr;              // the optical-flow tracker is outside the scope (vision module)
    map_tracker = new rgbMapTracker(); // src/imageProcessing.cpp:10 (src/rgbMapTracker.cpp IS compiled)
}
void imageProcessing::setImageWidth(int& para) { image_width = para; }
void imageProcessing::setImageHeight(int& para) { image_height = para; }
void imageProcessing::setCameraIntrinsic(std::vector<double>&) {}
void imageProcessing::setCameraDistCoeffs(std::vector<double>&) {}
void imageProcessing::setExtrinR(Eigen::Matrix3d& R) { R_imu_camera = R; }
void imageProcessing::setExtrinT(Eigen::Vector3d& t) { t_imu_camera = t; }
Eigen::Matrix3d imageProcessing::getCameraIntrinsic() { return camera_intrinsic; }
void imageProcessing::printParameter() {}
void imageProcessing::process(voxelHashMap&, cloudFrame*) { throw std::logic_error("imageProcessing::process: not part of the harness"); }

namespace {

struct RefCtx {
    lioOptimization* lio = nullptr;
    std::vector<RefCtx*> workers;        // owned: one lioOptimization per host thread for ref_update_iekf_many
    std::vector<state*> states;          // owned
    std::vector<cloudFrame*> frames;     // owned
    ~RefCtx() {
        for (cloudFrame* f : frames) delete f;
        for (state* s : states) delete s;
        for (RefCtx* w : workers) delete w;
        // lioOptimization has no destructor for its helpers; leak-free enough for a test process
        delete lio;
    }
};

Eigen::Vector3d v3(const double* p) { return Eigen::Vector3d(p[0], p[1], p[2]); }
Eigen::Quaterniond q4(const double* q) { return Eigen::Quaterniond(q[3], q[0], q[1], q[2]); }   // (x,y,z,w) -> ctor (w,x,y,z)
Eigen::Matrix3d m33(const double* p) {
    Eigen::Matrix3d M;
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) M(r, c) = p[r * 3 + c];
    return M;
}
void put3(double* o, const Eigen::Vector3d& v) { o[0] = v(0); o[1] = v(1); o[2] = v(2); }
void putq(double* o, const Eigen::Quaterniond& q) { o[0] = q.x(); o[1] = q.y(); o[2] = q.z(); o[3] = q.w(); }

icpOptions make_options(const orc_icp_params* p) {
    icpOptions o;                                  // include/parameters.h:8-56 defaults, then the fields the path reads
    o.threshold_voxel_occupancy = p->threshold_voxel_occupancy;
    o.init_num_frames = p->init_num_frames;
    o.size_voxel_map = p->size_voxel_map;
    o.num_iters_icp = p->num_iters_icp;
    o.min_number_neighbors = p->min_number_neighbors;
    o.voxel_neighborhood = p->voxel_neighborhood;
    o.power_planarity = p->power_planarity;
    o.estimate_normal_from_neighborhood = true;
    o.max_number_neighbors = p->max_number_neighbors;
    o.max_dist_to_plane_icp = p->max_dist_to_plane_icp;
    o.threshold_orientation_norm = p->threshold_orientation_norm;
    o.threshold_translation_norm = p->threshold_translation_norm;
    o.max_num_residuals = p->max_num_residuals;
    o.weight_alpha = p->weight_alpha;
    o.weight_neighborhood = p->weight_neighborhood;
    o.debug_print = false;
    return o;
}

// two frames as lioOptimization keeps them: all_cloud_frame[id - 1] is the previous sweep (only its translation is read,
// src/optimize.cpp:25,49), the current one carries the pose being optimised
cloudFrame* make_frames(RefCtx* c, const double q_cur[4], const double t_cur[3], const double t_last[3], int frame_id,
                        std::vector<point3D>& points) {
    for (cloudFrame* f : c->frames) delete f;
    for (state* s : c->states) delete s;
    c->frames.clear(); c->states.clear();
    state* s_last = new state();
    s_last->translation = v3(t_last);
    state* s_cur = new state();
    s_cur->rotation = q4(q_cur);
    s_cur->translation = v3(t_cur);
    c->states = {s_last, s_cur};
    std::vector<point3D> none;
    cloudFrame* f_last = new cloudFrame(none, s_last);
    f_last->id = 0; f_last->frame_id = frame_id - 1;
    cloudFrame* f_cur = new cloudFrame(points, s_cur);
    f_cur->id = 1; f_cur->frame_id = frame_id;
    c->frames = {f_last, f_cur};
    c->lio->all_cloud_frame.clear();
    c->lio->all_cloud_frame.push_back(f_last);
    c->lio->all_cloud_frame.push_back(f_cur);
    return f_cur;
}

void set_extrinsics(RefCtx* c, const double R_il[9], const double t_il[3]) {
    c->lio->R_imu_lidar = m33(R_il);
    c->lio->t_imu_lidar = v3(t_il);
}

void eskf_from_c(eskfEstimator* e, const orc_eskf_state* s) {
    e->setTranslation(v3(s->p));
    e->setRotation(q4(s->q));
    e->setVelocity(v3(s->v));
    e->setBa(v3(s->ba));
    e->setBg(v3(s->bg));
    e->setGravity(v3(s->g));
    Eigen::Matrix<double, 17, 17> P;
    for (int r = 0; r < 17; ++r) for (int k = 0; k < 17; ++k) P(r, k) = s->cov[r * 17 + k];
    e->setCovariance(P);
}
void eskf_to_c(eskfEstimator* e, orc_eskf_state* s) {
    put3(s->p, e->getTranslation());
    putq(s->q, e->getRotation());
    put3(s->v, e->getVelocity());
    put3(s->ba, e->getBa());
    put3(s->bg, e->getBg());
    put3(s->g, e->getGravity());
    Eigen::Matrix<double, 17, 17> P = e->getCovariance();
    for (int r = 0; r < 17; ++r) for (int k = 0; k < 17; ++k) s->cov[r * 17 + k] = P(r, k);
}

std::vector<imuState> imu_states_from_c(const orc_imu_state* st, int64_t n) {
    std::vector<imuState> v((size_t)n);
    for (int64_t i = 0; i < n; ++i) {
        v[(size_t)i].timestamp = st[i].timestamp;
        v[(size_t)i].quat = q4(st[i].quat);
        v[(size_t)i].trans = v3(st[i].trans);
        v[(size_t)i].vel = v3(st[i].vel);
        v[(size_t)i].un_acc = v3(st[i].un_acc);
        v[(size_t)i].un_gyr = v3(st[i].un_gyr);
    }
    return v;
}

voxelHashMap& pick_map(RefCtx* c, int which) { return which ? c->lio->color_voxel_map : c->lio->voxel_map; }

}  // namespace

extern "C" {

const char* ref_build_info(void) {
    return "reference sources compiled where they lie (optimize, utility, eskfEstimator, cloudMap, state, lioOptimization, "
           "rgbMapTracker, parameters .cpp) over oracle/shim (Eigen / OpenCV / ROS / PCL stand-ins), tsl::robin_map vendored";
}

void* ref_create(void) {
    RefCtx* c = new RefCtx();
    c->lio = new lioOptimization();   // the reference's constructor (src/lioOptimization.cpp:215-249) over the stub NodeHandle
    return c;
}
void ref_destroy(void* ctx) { delete static_cast<RefCtx*>(ctx); }

uint64_t ref_voxel_hash(int16_t x, int16_t y, int16_t z) { return (uint64_t)std::hash<voxel>()(voxel(x, y, z)); }   // include/cloudMap.h:173-184
double ref_laser_point_cov(void* ctx) { return static_cast<RefCtx*>(ctx)->lio->laser_point_cov; }                 // src/lioOptimization.cpp:364

// ---- maps ------------------------------------------------------------------------------------------------------
int64_t ref_map_num_voxels(void* ctx, int32_t which) { return (int64_t)pick_map(static_cast<RefCtx*>(ctx), which).size(); }
int64_t ref_map_num_points(void* ctx, int32_t which) { RefCtx* c = static_cast<RefCtx*>(ctx); return (int64_t)c->lio->mapSize(pick_map(c, which)); }
void ref_map_clear(void* ctx, int32_t which) { pick_map(static_cast<RefCtx*>(ctx), which).clear(); }

// test shortcut, the twin of orc_map_load: blocks keep the given point order
void ref_map_load(void* ctx, const int16_t* keys, const int32_t* counts, const float* xyz, int64_t n_voxels, int32_t cap) {
    voxelHashMap& map = static_cast<RefCtx*>(ctx)->lio->voxel_map;
    for (int64_t v = 0; v < n_voxels; ++v) {
        voxelBlock block(cap);
        for (int i = 0; i < counts[v]; ++i) {
            const float* p = xyz + ((size_t)v * cap + i) * 3;
            rgbPoint pt(Eigen::Vector3d(0, 0, 0));
            pt.position = Eigen::Vector3f(p[0], p[1], p[2]);   // exact FP32 content
            block.AddPoint(pt);
        }
        map[voxel(keys[3 * v], keys[3 * v + 1], keys[3 * v + 2])] = std::move(block);
    }
}

// lioOptimization::addPointsToMap (src/lioOptimization.cpp:520-554): LIO map AND colour map, as the reference does it.
// add_point_step / colour sizes are the mapOptions members; time_* feed the recent-voxel rule of addPointToColorMap
int64_t ref_add_points_to_map(void* ctx, const double* world_xyz, int64_t n, double voxel_size, int32_t max_num_points_in_voxel,
                              double min_distance_points, int32_t min_num_points, double color_voxel_size, int32_t color_max_points,
                              double color_min_distance, int32_t add_point_step, double time_sweep_end, double time_last_process,
                              int32_t to_rendering) {
    RefCtx* c = static_cast<RefCtx*>(ctx);
    lioOptimization* L = c->lio;
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
    const int64_t before = (int64_t)L->mapSize(L->voxel_map);
    L->addPointsToMap(L->voxel_map, &frame, voxel_size, max_num_points_in_voxel, min_distance_points, min_num_points, to_rendering != 0);
    frame.p_state = nullptr;
    return (int64_t)L->mapSize(L->voxel_map) - before;
}

int64_t ref_map_remove_far(void* ctx, const double location[3], double distance) {
    RefCtx* c = static_cast<RefCtx*>(ctx);
    const int64_t before = (int64_t)c->lio->voxel_map.size();
    c->lio->removePointsFarFromLocation(c->lio->voxel_map, v3(location), distance);
    return before - (int64_t)c->lio->voxel_map.size();
}

// container order; xyz n_voxels*cap*3 floats.  Colour fields (may be NULL): rgb, n_rgb, cov, obs_dist, last_obs per point, last_visited per voxel
int64_t ref_map_snapshot(void* ctx, int32_t which, int32_t cap, int16_t* keys, int32_t* counts, float* xyz, int16_t* rgb, int16_t* n_rgb,
                         float* cov, double* obs_dist, double* last_obs, double* last_visited) {
    voxelHashMap& map = pick_map(static_cast<RefCtx*>(ctx), which);
    int64_t v = 0;
    for (auto it = map.begin(); it != map.end(); ++it) {
        const voxel& key = it->first;
        voxelBlock& block = it.value();
        keys[3 * v] = key.x; keys[3 * v + 1] = key.y; keys[3 * v + 2] = key.z;
        const int cnt = std::min<int>(block.NumPoints(), cap);
        counts[v] = cnt;
        if (last_visited) last_visited[v] = block.last_visited_time;
        for (int i = 0; i < cap; ++i) {
            const size_t e = (size_t)v * cap + i;
            rgbPoint* p = i < cnt ? &block.points[(size_t)i] : nullptr;
            for (int a = 0; a < 3; ++a) {
                xyz[e * 3 + a] = p ? p->position(a) : 0.f;
                if (rgb) rgb[e * 3 + a] = p ? p->rgb[a] : (short)0;
                if (cov) cov[e * 3 + a] = (p && p->N_rgb != 0) ? p->cov_rgb(a) : 0.f;
            }
            if (n_rgb) n_rgb[e] = p ? p->N_rgb : (short)0;
            if (obs_dist) obs_dist[e] = p ? p->observe_distance : 0.0;
            if (last_obs) last_obs[e] = p ? p->last_observe_time : 0.0;
        }
        ++v;
    }
    return v;
}

// ---- the scan-matching path -------------------------------------------------------------------------------------
// lioOptimization::searchNeighbors (src/optimize.cpp:365-426): neighbours (FP64 positions) nearest first + their voxels
int32_t ref_search_neighbors(void* ctx, const double point[3], int32_t nb_voxels_visited, double size_voxel_map, int32_t max_num_neighbors,
                             int32_t threshold_voxel_capacity, double* nbr_xyz, int16_t* nbr_voxel) {
    RefCtx* c = static_cast<RefCtx*>(ctx);
    std::vector<voxel> voxels;
    auto nbrs = c->lio->searchNeighbors(c->lio->voxel_map, v3(point), nb_voxels_visited, size_voxel_map, max_num_neighbors, threshold_voxel_capacity, &voxels);
    for (size_t i = 0; i < nbrs.size(); ++i) {
        put3(nbr_xyz + 3 * i, nbrs[i]);
        nbr_voxel[3 * i] = voxels[i].x; nbr_voxel[3 * i + 1] = voxels[i].y; nbr_voxel[3 * i + 2] = voxels[i].z;
    }
    return (int32_t)nbrs.size();
}

// lioOptimization::computeNeighborhoodDistribution (src/optimize.cpp:316-353): out = center3, normal3, covariance9 (row-major), a2D
int32_t ref_neighborhood(void* ctx, const double* pts, int32_t n, double out[16]) {
    RefCtx* c = static_cast<RefCtx*>(ctx);
    std::vector<Eigen::Vector3d, Eigen::aligned_allocator<Eigen::Vector3d>> v((size_t)n);
    for (int i = 0; i < n; ++i) v[(size_t)i] = v3(pts + 3 * i);
    try {
        Neighborhood nh = c->lio->computeNeighborhoodDistribution(v);
        put3(out, nh.center); put3(out + 3, nh.normal);
        for (int r = 0; r < 3; ++r) for (int k = 0; k < 3; ++k) out[6 + r * 3 + k] = nh.covariance(r, k);
        out[15] = nh.a2D;
    } catch (const std::runtime_error&) { return 1; }   // :348-350
    return 0;
}

// lioOptimization::buildPlaneResiduals (src/optimize.cpp:18-131), one pass.  rows: per accepted residual, in order,
// raw_point3, norm_vector3, jacobians6, norm_offset, distance, weight (15 doubles; capacity n).  world_xyz: keypoint.point
// after transformKeypoints (n*3).  Returns -1 when computeNeighborhoodDistribution threw (NaN planarity).
int32_t ref_build_plane_residuals(void* ctx, const double* raw_xyz, int64_t n, const double q_cur[4], const double t_cur[3],
                                  const double t_last[3], const double R_il[9], const double t_il[3], const orc_icp_params* prm,
                                  int32_t* success, int32_t* num_residuals_used, double* loss_sum, double* rows, double* world_xyz) {
    RefCtx* c = static_cast<RefCtx*>(ctx);
    set_extrinsics(c, R_il, t_il);
    std::vector<point3D> keypoints((size_t)n);
    for (int64_t i = 0; i < n; ++i) keypoints[(size_t)i].raw_point = v3(raw_xyz + 3 * i);
    std::vector<point3D> none;
    cloudFrame* frame = make_frames(c, q_cur, t_cur, t_last, prm->frame_id, none);
    const icpOptions opt = make_options(prm);
    std::vector<planeParam> plane_residuals;
    double loss = 0.0;
    optimizeSummary summary;
    try {
        summary = c->lio->buildPlaneResiduals(opt, c->lio->voxel_map, keypoints, plane_residuals, frame, loss);
    } catch (const std::runtime_error&) { return -1; }
    *success = summary.success ? 1 : 0;
    *num_residuals_used = summary.num_residuals_used;
    *loss_sum = loss;
    for (size_t i = 0; i < plane_residuals.size(); ++i) {
        const planeParam& p = plane_residuals[i];
        double* o = rows + 15 * i;
        put3(o, p.raw_point); put3(o + 3, p.norm_vector);
        for (int k = 0; k < 6; ++k) o[6 + k] = p.jacobians(0, k);
        o[12] = p.norm_offset; o[13] = p.distance; o[14] = p.weight;
    }
    if (world_xyz) for (int64_t i = 0; i < n; ++i) put3(world_xyz + 3 * i, keypoints[(size_t)i].point);
    return (int32_t)plane_residuals.size();
}

// lioOptimization::updateIEKF (src/optimize.cpp:133-314) incl. eskfEstimator::observe.  Returns 0, or -1 on the NaN throw
int32_t ref_update_iekf(void* ctx, const double* raw_xyz, int64_t n, orc_eskf_state* eskf, double frame_q[4], double frame_t[3],
                        const double t_last[3], const double R_il[9], const double t_il[3], const orc_icp_params* prm,
                        int32_t* success, int32_t* num_residuals_used) {
    RefCtx* c = static_cast<RefCtx*>(ctx);
    set_extrinsics(c, R_il, t_il);
    c->lio->laser_point_cov = prm->laser_point_cov;
    eskf_from_c(c->lio->eskf_pro, eskf);
    std::vector<point3D> keypoints((size_t)n);
    for (int64_t i = 0; i < n; ++i) keypoints[(size_t)i].raw_point = v3(raw_xyz + 3 * i);
    std::vector<point3D> none;
    cloudFrame* frame = make_frames(c, frame_q, frame_t, t_last, prm->frame_id, none);
    const icpOptions opt = make_options(prm);
    optimizeSummary summary;
    try {
        summary = c->lio->updateIEKF(opt, c->lio->voxel_map, keypoints, frame);
    } catch (const std::runtime_error&) { return -1; }
    *success = summary.success ? 1 : 0;
    *num_residuals_used = summary.num_residuals_used;
    eskf_to_c(c->lio->eskf_pro, eskf);
    putq(frame_q, frame->p_state->rotation);
    put3(frame_t, frame->p_state->translation);
    return 0;
}

// lioOptimization::optimize (src/optimize.cpp:428-447): gridSampling of the frame (cells of point_frame[i].point) ->
// updateIEKF on the keypoints' raw points -> transformPoint of every frame point with the final pose.
// frame_world / frame_raw: n*3 in, frame_world rewritten with the re-transformed points; num_keypoints out.
int32_t ref_optimize(void* ctx, double* frame_world, const double* frame_raw, int64_t n, double sample_voxel_size, orc_eskf_state* eskf,
                     double frame_q[4], double frame_t[3], const double t_last[3], const double R_il[9], const double t_il[3],
                     const orc_icp_params* prm, int32_t* success, int32_t* num_residuals_used) {
    RefCtx* c = static_cast<RefCtx*>(ctx);
    set_extrinsics(c, R_il, t_il);
    c->lio->laser_point_cov = prm->laser_point_cov;
    eskf_from_c(c->lio->eskf_pro, eskf);
    std::vector<point3D> pts((size_t)n);
    for (int64_t i = 0; i < n; ++i) { pts[(size_t)i].point = v3(frame_world + 3 * i); pts[(size_t)i].raw_point = v3(frame_raw + 3 * i); }
    cloudFrame* frame = make_frames(c, frame_q, frame_t, t_last, prm->frame_id, pts);
    const icpOptions opt = make_options(prm);
    optimizeSummary summary;
    try {
        summary = c->lio->optimize(frame, opt, sample_voxel_size);
    } catch (const std::runtime_error&) { return -1; }
    *success = summary.success ? 1 : 0;
    *num_residuals_used = summary.num_residuals_used;
    eskf_to_c(c->lio->eskf_pro, eskf);
    putq(frame_q, frame->p_state->rotation);
    put3(frame_t, frame->p_state->translation);
    for (int64_t i = 0; i < n; ++i) put3(frame_world + 3 * i, frame->point_frame[(size_t)i].point);
    return 0;
}

// Throughput form for the CPU arm of bench.py: `n_sweeps` independent sweeps (n keypoints each, their own prior state and
// pose) registered against THIS context's voxel_map by `n_threads` host threads, each thread driving its own
// lioOptimization object through the reference's single-threaded updateIEKF (the map is passed by reference and only read:
// tsl::robin_map::find).  The reference has no threading of its own on this path; independent sweeps are the one way it
// can use more than one core.  Returns the number of sweeps whose update succeeded.
int32_t ref_update_iekf_many(void* ctx, const double* raw_xyz, int64_t n, int32_t n_sweeps, orc_eskf_state* eskf, double* frame_q,
                             double* frame_t, const double* t_last, const double R_il[9], const double t_il[3], const orc_icp_params* prm,
                             int32_t n_threads) {
    RefCtx* c = static_cast<RefCtx*>(ctx);
    if (n_threads < 1) n_threads = 1;
    if (n_threads > n_sweeps) n_threads = n_sweeps;
    while ((int)c->workers.size() < n_threads) { RefCtx* w = new RefCtx(); w->lio = new lioOptimization(); c->workers.push_back(w); }
    std::atomic<int> next(0), ok(0);
    auto run = [&](int tid) {
        RefCtx* w = c->workers[(size_t)tid];
        set_extrinsics(w, R_il, t_il);
        w->lio->laser_point_cov = prm->laser_point_cov;
        const icpOptions opt = make_options(prm);
        for (;;) {
            const int s = next.fetch_add(1);
            if (s >= n_sweeps) break;
            eskf_from_c(w->lio->eskf_pro, eskf + s);
            std::vector<point3D> keypoints((size_t)n);
            const double* raw = raw_xyz + (size_t)s * n * 3;
            for (int64_t i = 0; i < n; ++i) keypoints[(size_t)i].raw_point = v3(raw + 3 * i);
            std::vector<point3D> none;
            cloudFrame* frame = make_frames(w, frame_q + 4 * s, frame_t + 3 * s, t_last + 3 * s, prm->frame_id, none);
            try {
                optimizeSummary summary = w->lio->updateIEKF(opt, c->lio->voxel_map, keypoints, frame);
                if (summary.success) ok.fetch_add(1);
            } catch (const std::runtime_error&) {}
            eskf_to_c(w->lio->eskf_pro, eskf + s);
            putq(frame_q + 4 * s, frame->p_state->rotation);
            put3(frame_t + 3 * s, frame->p_state->translation);
        }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < n_threads; ++t) th.emplace_back(run, t);
    run(0);
    for (auto& t : th) t.join();
    return ok.load();
}

// ---- the caller of the path: lioOptimization::stateEstimation (src/lioOptimization.cpp:983-1035) over a stream of sweeps ----------
// ref_stream_reset forgets the frames pushed so far (all_cloud_frame) and empties both maps.
void ref_stream_reset(void* ctx) {
    RefCtx* c = static_cast<RefCtx*>(ctx);
    for (cloudFrame* f : c->frames) delete f;
    for (state* s : c->states) delete s;
    c->frames.clear(); c->states.clear();
    c->lio->all_cloud_frame.clear();
    c->lio->voxel_map.clear();
    c->lio->color_voxel_map.clear();
}
// One sweep through stateEstimation.  The frame is built the way buildFrame (src/lioOptimization.cpp:800-893) leaves it for the
// estimator: point = the raw point under the predicted pose (identity for the first two frames, :866-878), id = position in
// all_cloud_frame, frame_id = index_frame.  odo: init_voxel_size, init_sample_voxel_size, voxel_size, sample_voxel_size,
// min_distance_points (doubles) ; init_num_frames, max_num_points_in_voxel (ints).  prm carries the icpOptions; its frame_id is ignored.
// Outputs: the frame's pose, the filter, the re-transformed points (world_out, n*3).  Returns 0, or -1 on the NaN throw.
int32_t ref_stream_push(void* ctx, const double* raw_xyz, int64_t n, int32_t index_frame, const double q_pred[4], const double t_pred[3],
                        orc_eskf_state* eskf, const double R_il[9], const double t_il[3], const orc_icp_params* prm, const double odo_d[5],
                        const int32_t odo_i[2], int32_t* success, int32_t* num_residuals_used, double frame_q[4], double frame_t[3], double* world_out) {
    RefCtx* c = static_cast<RefCtx*>(ctx);
    lioOptimization* L = c->lio;
    set_extrinsics(c, R_il, t_il);
    L->laser_point_cov = prm->laser_point_cov;
    L->odometry_options.init_voxel_size = odo_d[0];
    L->odometry_options.init_sample_voxel_size = odo_d[1];
    L->odometry_options.voxel_size = odo_d[2];
    L->odometry_options.sample_voxel_size = odo_d[3];
    L->odometry_options.min_distance_points = odo_d[4];
    L->odometry_options.init_num_frames = odo_i[0];
    L->odometry_options.max_num_points_in_voxel = odo_i[1];
    L->odometry_options.optimize_options = make_options(prm);
    L->odometry_options.optimize_options.init_num_frames = odo_i[0];       // initialValue(), src/lioOptimization.cpp:391
    L->map_options.add_point_step = 1 << 30;                               // the colour map is not part of this check
    eskf_from_c(L->eskf_pro, eskf);
    state* st = new state();
    st->rotation = q4(q_pred);
    st->translation = v3(t_pred);
    std::vector<point3D> pts((size_t)n);
    Eigen::Quaterniond qp = index_frame > 2 ? q4(q_pred) : Eigen::Quaterniond::Identity();
    Eigen::Vector3d tp = index_frame > 2 ? v3(t_pred) : Eigen::Vector3d(Eigen::Vector3d::Zero());
    for (int64_t i = 0; i < n; ++i) {
        pts[(size_t)i].raw_point = v3(raw_xyz + 3 * i);
        transformPoint(pts[(size_t)i], qp, tp, L->R_imu_lidar, L->t_imu_lidar);
    }
    cloudFrame* frame = new cloudFrame(pts, st);
    frame->id = (int)L->all_cloud_frame.size();
    frame->sub_id = 0;
    frame->frame_id = index_frame;
    frame->time_sweep_end = 0.1 * index_frame;
    L->index_frame = index_frame;
    L->all_cloud_frame.push_back(frame);
    c->frames.push_back(frame); c->states.push_back(st);
    optimizeSummary summary;
    try {
        summary = L->stateEstimation(frame, false);
    } catch (const std::runtime_error&) { return -1; }
    *success = (index_frame > 1) ? (summary.success ? 1 : 0) : 1;           // frame 1 runs no optimisation: the default-constructed summary says false
    *num_residuals_used = summary.num_residuals_used;
    eskf_to_c(L->eskf_pro, eskf);
    putq(frame_q, frame->p_state->rotation);
    put3(frame_t, frame->p_state->translation);
    for (int64_t i = 0; i < n; ++i) put3(world_out + 3 * i, frame->point_frame[(size_t)i].point);
    return 0;
}

void ref_eskf_observe(orc_eskf_state* s, const double dx[17]) {   // eskfEstimator::observe (src/eskfEstimator.cpp:219-230)
    eskfEstimator e;
    eskf_from_c(&e, s);
    Eigen::Matrix<double, 17, 1> d;
    for (int i = 0; i < 17; ++i) d(i) = dx[i];
    e.observe(d);
    eskf_to_c(&e, s);
}

// ---- rows N2 / N3 ----------------------------------------------------------------------------------------------
// gridSampling (src/utility.cpp:187-201): indices of the kept points, in the reference's order
int64_t ref_grid_sampling(const double* xyz, int64_t n, double size_voxel_subsampling, int32_t* out) {
    std::vector<point3D> frame((size_t)n), keypoints;
    for (int64_t i = 0; i < n; ++i) { frame[(size_t)i].point = v3(xyz + 3 * i); frame[(size_t)i].index_frame = (int)i; }
    gridSampling(frame, keypoints, size_voxel_subsampling);
    for (size_t i = 0; i < keypoints.size(); ++i) out[i] = keypoints[i].index_frame;
    return (int64_t)keypoints.size();
}
void ref_distort_frame_by_constant(const double* raw_xyz, const double* relative_time, int64_t n, const orc_imu_state* st, int64_t n_states,
                                   double time_frame_begin, const double R_il[9], const double t_il[3], double* imu_xyz) {
    std::vector<point3D> pts((size_t)n);
    for (int64_t i = 0; i < n; ++i) { pts[(size_t)i].raw_point = v3(raw_xyz + 3 * i); pts[(size_t)i].relative_time = relative_time[i]; pts[(size_t)i].imu_point = v3(imu_xyz + 3 * i); }
    std::vector<imuState> states = imu_states_from_c(st, n_states);
    Eigen::Matrix3d R = m33(R_il); Eigen::Vector3d t = v3(t_il);
    distortFrameByConstant(pts, states, time_frame_begin, R, t);
    for (int64_t i = 0; i < n; ++i) put3(imu_xyz + 3 * i, pts[(size_t)i].imu_point);
}
void ref_distort_frame_by_imu(const double* raw_xyz, const double* relative_time, int64_t n, const orc_imu_state* st, int64_t n_states,
                              double time_frame_begin, const double R_il[9], const double t_il[3], double* imu_xyz) {
    std::vector<point3D> pts((size_t)n);
    for (int64_t i = 0; i < n; ++i) { pts[(size_t)i].raw_point = v3(raw_xyz + 3 * i); pts[(size_t)i].relative_time = relative_time[i]; pts[(size_t)i].imu_point = v3(imu_xyz + 3 * i); }
    std::vector<imuState> states = imu_states_from_c(st, n_states);
    Eigen::Matrix3d R = m33(R_il); Eigen::Vector3d t = v3(t_il);
    distortFrameByImu(pts, states, time_frame_begin, R, t);
    for (int64_t i = 0; i < n; ++i) put3(imu_xyz + 3 * i, pts[(size_t)i].imu_point);
}
void ref_transform_all_imu_point(const double* imu_xyz, int64_t n, const orc_imu_state* last, const double R_il[9], const double t_il[3], double* raw_out) {
    std::vector<point3D> pts((size_t)n);
    for (int64_t i = 0; i < n; ++i) pts[(size_t)i].imu_point = v3(imu_xyz + 3 * i);
    std::vector<imuState> states = imu_states_from_c(last, 1);
    Eigen::Matrix3d R = m33(R_il); Eigen::Vector3d t = v3(t_il);
    transformAllImuPoint(pts, states, R, t);
    for (int64_t i = 0; i < n; ++i) put3(raw_out + 3 * i, pts[(size_t)i].raw_point);
}
void ref_transform_point(const double* raw_xyz, int64_t n, const double q_end[4], const double t_end[3], const double R_il[9], const double t_il[3], double* world_out) {
    Eigen::Quaterniond q = q4(q_end); Eigen::Vector3d te = v3(t_end);
    Eigen::Matrix3d R = m33(R_il); Eigen::Vector3d t = v3(t_il);
    for (int64_t i = 0; i < n; ++i) {
        point3D p; p.raw_point = v3(raw_xyz + 3 * i);
        transformPoint(p, q, te, R, t);
        put3(world_out + 3 * i, p.point);
    }
}

// ---- row N4: colour map lists and renderer -----------------------------------------------------------------------
int64_t ref_color_num_rgb_points(void* ctx) { return (int64_t) static_cast<RefCtx*>(ctx)->lio->img_pro->map_tracker->rgb_points_vec.size(); }
int64_t ref_color_num_recent(void* ctx) { return (int64_t) static_cast<RefCtx*>(ctx)->lio->img_pro->map_tracker->voxels_recent_visited.size(); }
int64_t ref_color_num_new_recent(void* ctx) { return (int64_t) static_cast<RefCtx*>(ctx)->lio->img_pro->map_tracker->number_of_new_visited_voxel; }
// rgb_points_vec as (voxel key, index in block) — the pointers are resolved through the colour map; recent voxels as keys
void ref_color_lists(void* ctx, int16_t* rgb_points /* n*4 */, int32_t* recent /* m*3 */) {
    RefCtx* c = static_cast<RefCtx*>(ctx);
    lioOptimization* L = c->lio;
    rgbMapTracker* T = L->img_pro->map_tracker;
    const double size = L->map_options.size_voxel_map;
    for (size_t i = 0; i < T->rgb_points_vec.size(); ++i) {
        rgbPoint* p = T->rgb_points_vec[i];
        const voxel key = voxel::coordinates(*p, size);   // include/cloudMap.h:138-142: the same truncating division as addPointToColorMap
        voxelBlock& block = L->color_voxel_map[key];
        rgb_points[4 * i] = key.x; rgb_points[4 * i + 1] = key.y; rgb_points[4 * i + 2] = key.z;
        rgb_points[4 * i + 3] = (int16_t)(p - &block.points[0]);
    }
    for (size_t i = 0; i < T->voxels_recent_visited.size(); ++i) {
        recent[3 * i] = T->voxels_recent_visited[i].kx; recent[3 * i + 1] = T->voxels_recent_visited[i].ky; recent[3 * i + 2] = T->voxels_recent_visited[i].kz;
    }
}
// rgbMapTracker::renderPointsInRecentVoxel (src/rgbMapTracker.cpp:213-237) over map_tracker->voxels_recent_visited.
// cam: q_camera_world (x,y,z,w), t_camera_world, t_world_camera, fx, fy, cx, cy, fov_margin (15 doubles); image BGR u8
int64_t ref_color_render(void* ctx, const double* cam, const uint8_t* image_bgr, int32_t rows, int32_t cols, double obs_time) {
    RefCtx* c = static_cast<RefCtx*>(ctx);
    lioOptimization* L = c->lio;
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

}  // extern "C"
