// TEST INFRASTRUCTURE (oracle/) — NOT product code.  C entry points around the reference's own cloudProcessing
// (src/cloudProcessing.cpp, compiled unmodified by oracle/cloud_processing.mk): configure it as lioOptimization::readParameters
// does, feed it Livox CustomMsg records or PointCloud2 data, and drain the point_buffer it fills.  tests/cloud_processing_ref.py
// loads the library; tests/golden/make_cloud_processing_golden.py records its outputs.
#include "cloudProcessing.h"

#include <cstdint>
#include <cstring>
#include <queue>

namespace {
struct Handle {
    cloudProcessing cp;
    std::queue<point3D> buffer;
};
}  // namespace

extern "C" {

void* srl_cp_create(int lidar_type, int n_scans, int scan_rate, int time_unit, double blind, int point_filter_num) {
    Handle* h = new Handle();   // value-initialised: given_offset_time, which the constructor leaves unset, starts false
    h->cp.setLidarType(lidar_type);
    h->cp.setNumScans(n_scans);
    h->cp.setScanRate(scan_rate);
    h->cp.setTimeUnit(time_unit);
    h->cp.setBlind(blind);
    h->cp.setPointFilterNum(point_filter_num);
    return h;
}

void srl_cp_destroy(void* p) { delete static_cast<Handle*>(p); }

// n records `stride` bytes apart: offset_time u32 @0, x y z f32 @4 @8 @12, reflectivity @16, tag @17, line @18 (unaligned allowed)
void srl_cp_livox(void* p, const uint8_t* rec, int64_t n, int64_t stride, double stamp) {
    Handle* h = static_cast<Handle*>(p);
    auto msg = std::make_shared<livox_ros_driver::CustomMsg>();
    msg->header.stamp.fromSec(stamp);
    msg->point_num = static_cast<unsigned>(n);
    msg->points.resize(n);
    for (int64_t i = 0; i < n; ++i) {
        const uint8_t* r = rec + i * stride;
        livox_ros_driver::CustomPoint& q = msg->points[i];
        std::memcpy(&q.offset_time, r, 4);
        std::memcpy(&q.x, r + 4, 4);
        std::memcpy(&q.y, r + 8, 4);
        std::memcpy(&q.z, r + 12, 4);
        q.reflectivity = r[16];
        q.tag = r[17];
        q.line = r[18];
    }
    h->cp.livoxHandler(msg, h->buffer);
}

// n points of point_step bytes; offsets[0..4] = byte offsets of x, y, z, the time field (velodyne "time", ouster "t", robosense
// "timestamp", by lidar type) and "ring"; a negative offset leaves that field out of the message
void srl_cp_process(void* p, const uint8_t* data, int64_t n, int64_t point_step, const int32_t* offsets, double stamp) {
    Handle* h = static_cast<Handle*>(p);
    auto msg = std::make_shared<sensor_msgs::PointCloud2>();
    msg->header.stamp.fromSec(stamp);
    msg->width = static_cast<unsigned>(n);
    msg->height = 1;
    const int type = h->cp.getLidarType();
    const char* time_name = type == VELO ? "time" : type == OUST ? "t" : "timestamp";
    const char* names[5] = {"x", "y", "z", time_name, "ring"};
    for (int k = 0; k < 5; ++k) {
        if (offsets[k] < 0) continue;
        sensor_msgs::PointField f;
        f.name = names[k];
        f.offset = static_cast<unsigned>(offsets[k]);
        f.count = 1;
        msg->fields.push_back(f);
    }
    msg->data.assign(data, data + n * point_step);
    h->cp.process(msg, h->buffer);
}

int64_t srl_cp_queue_size(void* p) { return static_cast<int64_t>(static_cast<Handle*>(p)->buffer.size()); }

// pops the whole point_buffer: raw_point (3 per point), relative_time, timestamp
int64_t srl_cp_drain(void* p, double* xyz, double* rel, double* ts) {
    Handle* h = static_cast<Handle*>(p);
    int64_t i = 0;
    while (!h->buffer.empty()) {
        const point3D& q = h->buffer.front();
        for (int k = 0; k < 3; ++k) xyz[3 * i + k] = q.raw_point[k];
        rel[i] = q.relative_time;
        ts[i] = q.timestamp;
        h->buffer.pop();
        ++i;
    }
    return i;
}

void srl_cp_state(void* p, double* last_end_time, int32_t* given_offset_time, int32_t* sweep_id, double* sweep_interval) {
    Handle* h = static_cast<Handle*>(p);
    *last_end_time = h->cp.last_end_time;
    *given_offset_time = h->cp.isPointTimeEnable() ? 1 : 0;
    *sweep_id = h->cp.sweep_id;
    *sweep_interval = h->cp.getSweepInterval();
}
}
