// Harness of the reference's Horizon front end, LiLi-OM/src/Preprocessing.cpp, driven through its ROS interface: imuHandler
// messages, then cloudHandler.  The node resets q_iMU to the identity after publishing (:403), so the publish hook captures it.
// Callers keep the node's IMU buffer at no more than 600 messages (it releases older entries, :176-177, and processIMU would
// then dereference them).
#include "harness.h"
#define private public
#include "Preprocessing.cpp"
#undef private

namespace {
Preprocessing* g_node = nullptr;
int g_publishes = 0;
double g_q_pub[4] = {1, 0, 0, 0};
}

REF_API void ref_hz_create(double surf_thres, double edge_thres) {
    delete g_node;
    ref::reset_world();
    ros::param::set("/preprocessing/surf_thres", surf_thres);
    ros::param::set("/preprocessing/edge_thres", edge_thres);
    g_node = new Preprocessing();
    g_publishes = 0;
    ros::publish_hook() = [](const std::string& topic) {
        if (topic != "/surf_features") return;   // the first of the node's three publishes
        ++g_publishes;
        g_q_pub[0] = g_node->q_iMU.w(); g_q_pub[1] = g_node->q_iMU.x(); g_q_pub[2] = g_node->q_iMU.y(); g_q_pub[3] = g_node->q_iMU.z();
    };
}

REF_API void ref_hz_imu(double stamp, const double gyro[3]) {
    auto m = std::make_shared<sensor_msgs::Imu>();
    m->header.stamp = ros::Time(stamp);
    m->angular_velocity.x = gyro[0]; m->angular_velocity.y = gyro[1]; m->angular_velocity.z = gyro[2];
    g_node->imuHandler(m);
}

// pts: n PointXYZINormal as the driver (FormatConvert) publishes them; is_dense is the message's flag (removeNaNFromPointCloud
// copies a dense cloud as it is).  Returns the number of clouds the node has published so far.
REF_API int ref_hz_cloud(double stamp, const void* pts, int n, int is_dense) {
    auto c = ref::cloud_of<pcl::PointXYZINormal>(pts, n);
    c->is_dense = is_dense != 0;
    auto m = std::make_shared<sensor_msgs::PointCloud2>();
    pcl::toROSMsg(*c, *m);
    m->header.stamp = ros::Time(stamp);
    g_node->cloudHandler(m);
    return g_publishes;
}

REF_API void ref_hz_set_q(const double q[4]) { g_node->q_iMU = Eigen::Quaterniond(q[0], q[1], q[2], q[3]); }
REF_API void ref_hz_q_published(double q[4]) { for (int k = 0; k < 4; ++k) q[k] = g_q_pub[k]; }

// which: 0 surf, 1 edge, 2 cutted cloud of the last publish
REF_API int ref_hz_take(int which, void* out, int cap) {
    static const char* const topic[3] = {"/surf_features", "/edge_features", "/lidar_cloud_cutted"};
    return ref::take_published(topic[which], out, cap, 48);
}
