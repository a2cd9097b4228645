// TEST INFRASTRUCTURE (oracle/): force-included after shim/srl_prelude.h in front of the reference's src/cloudProcessing.cpp only
// (oracle/cloud_processing.mk).  The shared stand-ins declare pcl::fromROSMsg nowhere and register no point fields; the handlers
// need both:
//   * POINT_CLOUD_REGISTER_POINT_STRUCT(name, (type, field, tag)...) becomes a field list pcl::srl_point_fields<name>::each that
//     visits every registered member with its name.
//   * pcl::fromROSMsg maps the message's fields into those members by name, as PCL's createMapping does: width x height points,
//     point_step = data.size() / (width x height) (the stand-in PointCloud2 carries no point_step; the harness packs the data
//     densely), every member copied from its field's byte offset.  A registered member the message lacks keeps the point's
//     default.  Field datatypes are not checked: the harness writes each field as the member's type.
#pragma once
#include <cstring>

namespace pcl {
template <class P> struct srl_point_fields;
template <class P> inline void fromROSMsg(const sensor_msgs::PointCloud2& msg, PointCloud<P>& cloud) {
    const size_t n = size_t(msg.width) * msg.height;
    const size_t step = n ? msg.data.size() / n : 0;
    cloud.points.assign(n, P());
    cloud.width = msg.width;
    cloud.height = msg.height;
    for (size_t i = 0; i < n; ++i)
        srl_point_fields<P>::each(cloud.points[i], [&](const char* name, auto& member) {
            for (const auto& f : msg.fields)
                if (f.name == name) {
                    std::memcpy(&member, msg.data.data() + i * step + f.offset, sizeof(member));
                    break;
                }
        });
}
}  // namespace pcl

// the field sequence (t, n, tag)(t, n, tag)... walked by two macros that name each other, closed by pasting _END
#define SRL_PF_A(t, n, tag) f(#n, p.n); SRL_PF_B
#define SRL_PF_B(t, n, tag) f(#n, p.n); SRL_PF_A
#define SRL_PF_A_END
#define SRL_PF_B_END
#define SRL_PF_CAT(a, b) SRL_PF_CAT_(a, b)
#define SRL_PF_CAT_(a, b) a##b
#undef POINT_CLOUD_REGISTER_POINT_STRUCT
#define POINT_CLOUD_REGISTER_POINT_STRUCT(name, seq)                                     \
    namespace pcl {                                                                     \
    template <> struct srl_point_fields<name> {                                         \
        template <class F> static void each(name& p, F f) { SRL_PF_CAT(SRL_PF_A seq, _END) } \
    };                                                                                  \
    }
