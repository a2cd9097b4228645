// TEST INFRASTRUCTURE (oracle/) — NOT product code.  lioOptimization::buildFrame (src/lioOptimization.cpp:786-893), the
// reference's own, behind a C entry point.  Linked by oracle/build_frame.mk with the same unmodified reference objects and
// srl_reference_harness.cpp (which supplies the members of the classes the LIO sources link against but never run) into
// oracle/_ref/libsrl_build_frame_ref.so.  Only tests/ and scripts/bench_build_frame.py load it.
#include "lioOptimization.h"
#include "cloudProcessing.h"
#include "srl_oracle.h"   // orc_imu_state

namespace {

Eigen::Vector3d v3(const double* p) { return Eigen::Vector3d(p[0], p[1], p[2]); }
Eigen::Quaterniond q4(const double* q) { return Eigen::Quaterniond(q[3], q[0], q[1], q[2]); }   // (x,y,z,w) -> ctor (w,x,y,z)
void put3(double* o, const Eigen::Vector3d& v) { o[0] = v(0); o[1] = v(1); o[2] = v(2); }

}  // namespace

extern "C" {

void* ref_bf_create(void) { return new lioOptimization(); }   // the reference's constructor over the stub NodeHandle
void ref_bf_destroy(void* lio) { delete static_cast<lioOptimization*>(lio); }

// buildFrame over a cut sweep whose imu_point starts at 0.  prm: timestamp_begin, timestamp_offset, init_voxel_size,
// voxel_size, prev_time_sweep_end (doubles); cfg: point_time_enable, motion_compensation, index_frame, init_num_frames (ints).
// The cut sweep's index travels in point3D::index_frame.  Outputs (capacity n) in frame order; scalars: time_sweep_begin,
// time_sweep_end, time_frame_begin, time_frame_end, offset_begin, offset_end, dt_offset.  Returns the frame's size.  The frame
// is not kept: all_cloud_frame is as before the call.
int64_t ref_build_frame(void* lio, const double* raw_xyz, const double* timestamp, int64_t n, const orc_imu_state* st, int64_t n_states,
                        const double R_il[9], const double t_il[3], const double q_pred[4], const double t_pred[3], const double prm[5],
                        const int32_t cfg[4], double* raw_out, double* point_out, double* imu_out, double* rel_out, double* alpha_out,
                        double* ts_out, int32_t* src_out, double scalars[7]) {
    lioOptimization* L = static_cast<lioOptimization*>(lio);
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) L->R_imu_lidar(r, c) = R_il[r * 3 + c];
    L->t_imu_lidar = v3(t_il);
    if (!L->cloud_pro) L->cloud_pro = new cloudProcessing();
    L->cloud_pro->given_offset_time = cfg[0] != 0;
    L->odometry_options.motion_compensation = (MotionCompensation)cfg[1];
    L->index_frame = cfg[2];
    L->odometry_options.init_num_frames = cfg[3];
    L->odometry_options.init_voxel_size = prm[2];
    L->odometry_options.voxel_size = prm[3];
    L->imu_states.assign((size_t)n_states, imuState());
    for (int64_t i = 0; i < n_states; ++i) {
        imuState& s = L->imu_states[(size_t)i];
        s.timestamp = st[i].timestamp;
        s.quat = q4(st[i].quat);
        s.trans = v3(st[i].trans);
        s.vel = v3(st[i].vel);
        s.un_acc = v3(st[i].un_acc);
        s.un_gyr = v3(st[i].un_gyr);
    }
    std::vector<point3D> sweep((size_t)n);
    for (int64_t i = 0; i < n; ++i) {   // as the point handlers leave a point (src/cloudProcessing.cpp:141-147)
        point3D& p = sweep[(size_t)i];
        p.raw_point = v3(raw_xyz + 3 * i);
        p.point = p.raw_point;
        p.imu_point = Eigen::Vector3d(0.0, 0.0, 0.0);
        p.timestamp = timestamp[i];
        p.index_frame = (int)i;
    }
    state* s_pred = new state();
    s_pred->rotation = q4(q_pred);
    s_pred->translation = v3(t_pred);
    std::vector<cloudFrame*> saved = L->all_cloud_frame;
    L->all_cloud_frame.clear();
    std::vector<point3D> none;
    cloudFrame* prev = new cloudFrame(none, s_pred);
    prev->time_sweep_end = prm[4];
    if (cfg[2] > 1) L->all_cloud_frame.push_back(prev);   // read for dt_offset
    cloudFrame* f = L->buildFrame(sweep, s_pred, prm[0], prm[1]);
    const size_t m = f->point_frame.size();
    for (size_t k = 0; k < m; ++k) {
        const point3D& p = f->point_frame[k];
        put3(raw_out + 3 * k, p.raw_point); put3(point_out + 3 * k, p.point); put3(imu_out + 3 * k, p.imu_point);
        rel_out[k] = p.relative_time; alpha_out[k] = p.alpha_time; ts_out[k] = p.timestamp; src_out[k] = p.index_frame;
    }
    scalars[0] = f->time_sweep_begin; scalars[1] = f->time_sweep_end; scalars[2] = f->time_frame_begin; scalars[3] = f->time_frame_end;
    scalars[4] = f->offset_begin; scalars[5] = f->offset_end; scalars[6] = f->dt_offset;
    L->all_cloud_frame = saved;
    delete f; delete prev; delete s_pred;   // cloudFrame does not own its state
    return (int64_t)m;
}

}  // extern "C"
