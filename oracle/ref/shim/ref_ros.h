// Compile-time stand-in for the part of roscpp and its message types the reference's front end and odometry use.  Nothing is
// serialised and nothing is spun: a harness calls the node's handlers itself, ros::param is a map the harness fills, and
// Publisher::publish records the message under its topic and then calls the harness's hook, if one is set.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#define ROS_INFO(...) ((void)0)
#define ROS_WARN(...) ((void)0)
#define ROS_ERROR(...) ((void)0)
#define ROS_DEBUG(...) ((void)0)
#define ROS_BREAK() std::abort()

namespace boost { using std::shared_ptr; }

namespace ros {
struct Time {
    double t = 0;
    Time() {}
    explicit Time(double s) : t(s) {}
    double toSec() const { return t; }
    static Time now() { return Time(); }
};
}  // namespace ros

namespace std_msgs {
struct Header { uint32_t seq = 0; ros::Time stamp; std::string frame_id; };
}

namespace geometry_msgs {
struct Point { double x = 0, y = 0, z = 0; };
struct Vector3 { double x = 0, y = 0, z = 0; };
struct Quaternion { double x = 0, y = 0, z = 0, w = 1; };
struct Pose { Point position; Quaternion orientation; };
struct PoseWithCovariance { Pose pose; double covariance[36] = {}; };
struct Twist { Vector3 linear, angular; };
struct TwistWithCovariance { Twist twist; double covariance[36] = {}; };
struct PoseStamped { std_msgs::Header header; Pose pose; };
struct Vector3Stamped { std_msgs::Header header; Vector3 vector; };
struct QuaternionStamped { std_msgs::Header header; Quaternion quaternion; };
}

namespace nav_msgs {
struct Odometry { std_msgs::Header header; std::string child_frame_id; geometry_msgs::PoseWithCovariance pose; geometry_msgs::TwistWithCovariance twist; };
struct Path { std_msgs::Header header; std::vector<geometry_msgs::PoseStamped> poses; };
}

namespace visualization_msgs { struct Marker { std_msgs::Header header; }; }

namespace sensor_msgs {
struct Imu {
    std_msgs::Header header;
    geometry_msgs::Quaternion orientation;
    geometry_msgs::Vector3 angular_velocity, linear_acceleration;
};
typedef std::shared_ptr<const Imu> ImuConstPtr;
struct NavSatFix { std_msgs::Header header; };

struct PointField {
    enum { INT8 = 1, UINT8 = 2, INT16 = 3, UINT16 = 4, INT32 = 5, UINT32 = 6, FLOAT32 = 7, FLOAT64 = 8 };
    std::string name; uint32_t offset = 0; uint8_t datatype = 0; uint32_t count = 0;
};
// pcl::toROSMsg does not serialise: `data` holds the published pcl::PointCloud's points as they are in memory and
// `pcl_point_size` is sizeof the point type (0 for a message that came from a driver, decoded through `fields`).
struct PointCloud2 {
    std_msgs::Header header;
    uint32_t height = 0, width = 0;
    std::vector<PointField> fields;
    bool is_bigendian = false;
    uint32_t point_step = 0, row_step = 0;
    std::vector<uint8_t> data;
    bool is_dense = false;
    uint32_t pcl_point_size = 0;
};
typedef std::shared_ptr<const PointCloud2> PointCloud2ConstPtr;
}  // namespace sensor_msgs

namespace livox_ros_driver {
struct CustomPoint { uint32_t offset_time = 0; float x = 0, y = 0, z = 0; uint8_t reflectivity = 0, tag = 0, line = 0; };
struct CustomMsg {
    std_msgs::Header header;
    uint64_t timebase = 0;
    uint32_t point_num = 0;
    uint8_t lidar_id = 0;
    uint8_t rsvd[3] = {0, 0, 0};
    std::vector<CustomPoint> points;
};
typedef std::shared_ptr<const CustomMsg> CustomMsgConstPtr;
}  // namespace livox_ros_driver

namespace ros {

// what the node published, by topic, and a hook called after every publish (the topic is its argument)
inline std::map<std::string, sensor_msgs::PointCloud2>& published_clouds() {
    static std::map<std::string, sensor_msgs::PointCloud2> m;
    return m;
}
inline std::function<void(const std::string&)>& publish_hook() {
    static std::function<void(const std::string&)> h;
    return h;
}
inline void record(const std::string& topic, const sensor_msgs::PointCloud2& msg) { published_clouds()[topic] = msg; }
template <class M> inline void record(const std::string&, const M&) {}

struct Publisher {
    std::string topic;
    template <class M> void publish(const M& msg) const {
        record(topic, msg);
        if (publish_hook()) publish_hook()(topic);
    }
};
struct Subscriber {};

struct NodeHandle {
    NodeHandle() {}
    explicit NodeHandle(const std::string&) {}
    template <class M, class C>
    Subscriber subscribe(const std::string&, uint32_t, void (C::*)(const std::shared_ptr<const M>&), C*) { return Subscriber(); }
    template <class M>
    Subscriber subscribe(const std::string&, uint32_t, void (*)(const std::shared_ptr<const M>&)) { return Subscriber(); }
    template <class M> Publisher advertise(const std::string& topic, uint32_t) { return Publisher{topic}; }
};

struct Rate { explicit Rate(double) {} void sleep() {} };
inline void init(int&, char**, const std::string&) {}
inline bool ok() { return false; }
inline void spin() {}
inline void spinOnce() {}

namespace this_node { inline std::string getName() { return "/reference_harness"; } }

// ros::param: a settable map; a name that was never set is missing, so the node falls back to its default
namespace param {
inline std::map<std::string, double>& numbers() { static std::map<std::string, double> m; return m; }
inline std::map<std::string, std::string>& strings() { static std::map<std::string, std::string> m; return m; }
inline bool search(const std::string& name, std::string& key) { key = name; return true; }
inline bool has(const std::string& key) { return numbers().count(key) || strings().count(key); }
inline bool get(const std::string& key, std::string& v) {
    auto it = strings().find(key); if (it == strings().end()) return false; v = it->second; return true;
}
inline bool get(const std::string& key, double& v) {
    auto it = numbers().find(key); if (it == numbers().end()) return false; v = it->second; return true;
}
inline bool get(const std::string& key, int& v) {
    auto it = numbers().find(key); if (it == numbers().end()) return false; v = (int)it->second; return true;
}
inline bool get(const std::string& key, bool& v) {
    auto it = numbers().find(key); if (it == numbers().end()) return false; v = it->second != 0; return true;
}
inline void set(const std::string& key, double v) { numbers()[key] = v; }
inline void clear() { numbers().clear(); strings().clear(); }
}  // namespace param

}  // namespace ros

// roscpp brings boost::bind's placeholders into the global namespace; the ROT node's std::sort comparator names them
#include <functional>
using std::placeholders::_1;
using std::placeholders::_2;
