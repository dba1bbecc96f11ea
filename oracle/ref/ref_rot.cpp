// Harness of the reference's spinning-LiDAR front end, LiLi-OM-ROT/src/Preprocessing.cpp, driven through its ROS interface:
// imuHandler messages, then cloudHandler on a typed cloud or on a driver's PointCloud2.  The node resets qIMU after publishing
// (:529), so the publish hook captures it.  Callers keep the IMU buffer at no more than 600 messages and hand the node clouds
// with at least one point left after the 3 m cut (it reads points[0], :285).
#include "harness.h"
#define private public
#include "Preprocessing.cpp"
#undef private

namespace {
Preprocessing* g_node = nullptr;
int g_publishes = 0;
double g_q_pub[4] = {1, 0, 0, 0};

int publish_count(double stamp, const std::shared_ptr<sensor_msgs::PointCloud2>& m) {
    m->header.stamp = ros::Time(stamp);
    g_node->cloudHandler(m);
    return g_publishes;
}
}

REF_API void ref_rot_create(int line_num, int ds_rate, const double q_lb[4]) {
    delete g_node;
    ref::reset_world();
    ros::param::set("/preprocessing/line_num", line_num);
    ros::param::set("/preprocessing/ds_rate", ds_rate);
    ros::param::set("/backend_fusion/ql2b_w", q_lb[0]);
    ros::param::set("/backend_fusion/ql2b_x", q_lb[1]);
    ros::param::set("/backend_fusion/ql2b_y", q_lb[2]);
    ros::param::set("/backend_fusion/ql2b_z", q_lb[3]);
    g_node = new Preprocessing();   // 6.4 MB of per-point arrays: never on the stack
    g_publishes = 0;
    ros::publish_hook() = [](const std::string& topic) {
        if (topic != "/lidar_cloud_cutted") return;   // the first of the node's three publishes
        ++g_publishes;
        g_q_pub[0] = g_node->qIMU.w(); g_q_pub[1] = g_node->qIMU.x(); g_q_pub[2] = g_node->qIMU.y(); g_q_pub[3] = g_node->qIMU.z();
    };
}

REF_API void ref_rot_imu(double stamp, const double gyro[3]) {
    auto m = std::make_shared<sensor_msgs::Imu>();
    m->header.stamp = ros::Time(stamp);
    m->angular_velocity.x = gyro[0]; m->angular_velocity.y = gyro[1]; m->angular_velocity.z = gyro[2];
    g_node->imuHandler(m);
}

// pts: n PointXYZI.  Returns the number of clouds the node has published so far.
REF_API int ref_rot_cloud(double stamp, const void* pts, int n, int is_dense) {
    auto c = ref::cloud_of<pcl::PointXYZI>(pts, n);
    c->is_dense = is_dense != 0;
    auto m = std::make_shared<sensor_msgs::PointCloud2>();
    pcl::toROSMsg(*c, *m);
    return publish_count(stamp, m);
}

// the driver's PointCloud2: payload, geometry and fields (name[16], offset, datatype, count), decoded by pcl::fromROSMsg
REF_API int ref_rot_cloud_pc2(double stamp, const unsigned char* data, unsigned height, unsigned width, unsigned point_step,
                              unsigned row_step, const RefPc2Field* fields, int n_fields, int is_dense) {
    auto m = std::make_shared<sensor_msgs::PointCloud2>();
    m->height = height; m->width = width; m->point_step = point_step; m->row_step = row_step;
    m->data.assign(data, data + (size_t)row_step * height);
    m->is_dense = is_dense != 0;
    for (int k = 0; k < n_fields; ++k) {
        sensor_msgs::PointField f;
        char name[17];
        std::memcpy(name, fields[k].name, 16); name[16] = '\0';
        f.name = name; f.offset = fields[k].offset; f.datatype = fields[k].datatype; f.count = fields[k].count;
        m->fields.push_back(f);
    }
    return publish_count(stamp, m);
}

REF_API void ref_rot_set_q(const double q[4]) { g_node->qIMU = Eigen::Quaterniond(q[0], q[1], q[2], q[3]); }
REF_API void ref_rot_q_published(double q[4]) { for (int k = 0; k < 4; ++k) q[k] = g_q_pub[k]; }

// which: 0 surf (less flat), 1 edge (less sharp), 2 the ring-ordered cloud of the last publish
REF_API int ref_rot_take(int which, void* out, int cap) {
    static const char* const topic[3] = {"/surf_features", "/edge_features", "/lidar_cloud_cutted"};
    return ref::take_published(topic[which], out, cap, 32);
}
