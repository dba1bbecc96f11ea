// Shared prologue of the reference harnesses (ref_*.cpp).  Each harness includes one of the reference's translation units by
// name, unmodified, against the shim headers in shim/, and exports a small C API (REF_API) for tests/ref_lib.py.  Every standard
// and shim header is included here first, so that `private` can be read as `public` for the reference's class alone: the
// harnesses call the nodes' members directly.
#pragma once
#include <algorithm>
#include <array>
#include <cassert>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <ctime>
#include <deque>
#include <fstream>
#include <functional>
#include <iostream>
#include <map>
#include <memory>
#include <mutex>
#include <queue>
#include <string>
#include <thread>
#include <vector>
#include <assert.h>
#include <stdio.h>

#include "ref_eigen.h"
#include "ref_ros.h"
#include "ref_pcl.h"
#include "ref_ceres.h"

#define REF_API extern "C" __attribute__((visibility("default")))

namespace ref {

template <class P> inline std::shared_ptr<pcl::PointCloud<P>> cloud_of(const void* pts, int n) {
    auto c = std::make_shared<pcl::PointCloud<P>>();
    c->points.resize(n > 0 ? n : 0);
    if (n > 0) std::memcpy(c->points.data(), pts, sizeof(P) * (size_t)n);
    c->width = (uint32_t)(n > 0 ? n : 0); c->height = 1;
    return c;
}

template <class P> inline int copy_out(const std::vector<P>& pts, void* out, int cap) {
    const int n = (int)pts.size();
    if (out && n > 0) std::memcpy(out, pts.data(), sizeof(P) * (size_t)std::min(n, cap));
    return n;
}

// the points of the cloud the node last published on `topic` (-1: nothing published there)
inline int take_published(const std::string& topic, void* out, int cap, int point_size) {
    auto& m = ros::published_clouds();
    auto it = m.find(topic);
    if (it == m.end()) return -1;
    const sensor_msgs::PointCloud2& msg = it->second;
    if ((int)msg.pcl_point_size != point_size) std::abort();
    const int n = (int)msg.width * (int)msg.height;
    if (out && n > 0) std::memcpy(out, msg.data.data(), (size_t)point_size * (size_t)std::min(n, cap));
    return n;
}

inline void reset_world() {
    ros::published_clouds().clear();
    ros::publish_hook() = nullptr;
    ros::param::clear();
}

}  // namespace ref
