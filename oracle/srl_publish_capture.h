// TEST INFRASTRUCTURE (oracle/): force-included (-include, after shim/srl_prelude.h) by oracle/publish.mk when it compiles the
// reference's src/lioOptimization.cpp for oracle/_ref/libsrl_publish_ref.so.  The stand-ins of pcl::toROSMsg and
// pcl::io::savePCDFileBinary (shim/srl_shim_ext.h) are empty templates; this header declares explicit specializations of them
// for the two cloud types the reference publishes and saves, and oracle/srl_publish_harness.cpp defines them, so every cloud
// the compiled reference hands over (publishCLoudWorld, pubColorPoints, saveColorPoints) reaches the harness.  No other
// reference translation unit calls either function, and the other builds of the reference never see this header.
#pragma once
#include "srl_shim_ext.h"

namespace pcl {
template <> void toROSMsg<PointCloud<PointXYZI>>(const PointCloud<PointXYZI>& cloud, sensor_msgs::PointCloud2& msg);
template <> void toROSMsg<PointCloud<PointXYZRGB>>(const PointCloud<PointXYZRGB>& cloud, sensor_msgs::PointCloud2& msg);
namespace io {
template <> int savePCDFileBinary<PointCloud<PointXYZRGB>>(const std::string& path, const PointCloud<PointXYZRGB>& cloud);
}  // namespace io
}  // namespace pcl
