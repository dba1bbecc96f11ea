// Harness of the reference's LiLi-OM/src/FormatConvert.cpp: livoxLidarHandler on a CustomMsg, read back through the
// recorded publish.
#include "harness.h"
#include "FormatConvert.cpp"

// recs: n records of `stride` bytes in the driver's CustomPoint wire layout (offset_time u32, x, y, z f32, reflectivity, tag,
// line u8).  out: n PointXYZINormal.  Returns the published point count, or -1 for an empty message (the node reads
// points.back()).
REF_API int ref_fc_convert(const unsigned char* recs, int n, int stride, double stamp, void* out, int cap) {
    if (n <= 0) return -1;
    ref::reset_world();
    ros::NodeHandle nh;
    const std::string topic = "/livox_ros_points";
    pub_ros_points = nh.advertise<sensor_msgs::PointCloud2>(topic, 100);
    auto msg = std::make_shared<livox_ros_driver::CustomMsg>();
    msg->header.stamp = ros::Time(stamp);
    msg->point_num = (uint32_t)n;
    msg->points.resize(n);
    for (int i = 0; i < n; ++i) {
        const unsigned char* r = recs + (size_t)i * stride;
        livox_ros_driver::CustomPoint& p = msg->points[i];
        std::memcpy(&p.offset_time, r, 4);
        std::memcpy(&p.x, r + 4, 4); std::memcpy(&p.y, r + 8, 4); std::memcpy(&p.z, r + 12, 4);
        p.reflectivity = r[16]; p.tag = r[17]; p.line = r[18];
    }
    livoxLidarHandler(msg);
    return ref::take_published(topic, out, cap, 48);
}
