// Compile-time stand-in for the part of PCL (and pcl_conversions) the reference's front end and odometry use.  The two point
// types have PCL's 48- and 32-byte layouts; their default constructor writes what the oracle writes (x = y = z = 0, data[3] = 1,
// every other float 0).  VoxelGrid forwards to orc_voxelgrid and KdTreeFLANN to the oracle's kd-tree (orc_kdtree_build /
// orc::knn5_one); fromROSMsg of a driver's message forwards to the PointCloud2 restatement of tests/pc2_oracle.cpp.
#pragma once
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <memory>
#include <vector>
#include "ref_ros.h"
#include "oracle_api.h"

namespace orc { void knn5_one(const void* tree, const float q[3], int idx[5], float sqd[5]); }

struct RefPc2Field { char name[16]; unsigned int offset; unsigned char datatype; unsigned int count; };
extern "C" int orc_pc2_to_pt32(const unsigned char* data, unsigned int height, unsigned int width, unsigned int point_step,
                               unsigned int row_step, const RefPc2Field* fields, int n_fields, float* out);

#define PCL_ADD_POINT4D
#define POINT_CLOUD_REGISTER_POINT_STRUCT(name, fseq)

namespace pcl {

struct PCLHeader { uint32_t seq = 0; uint64_t stamp = 0; std::string frame_id; };

struct alignas(16) PointXYZI {
    union { float data[4]; struct { float x, y, z; }; };
    union { struct { float intensity; }; float data_c[4]; };
    PointXYZI() { std::memset(this, 0, sizeof(*this)); data[3] = 1.0f; }
    // the fields pcl::fromROSMsg maps (POINT_CLOUD_REGISTER_POINT_STRUCT of PointXYZI)
    void copy_fields(const PointXYZI& o) { x = o.x; y = o.y; z = o.z; intensity = o.intensity; }
};

struct alignas(16) PointXYZINormal {
    union { float data[4]; struct { float x, y, z; }; };
    union { float data_n[4]; float normal[3]; struct { float normal_x, normal_y, normal_z; }; };
    union { struct { float intensity; float curvature; }; float data_c[4]; };
    PointXYZINormal() { std::memset(this, 0, sizeof(*this)); data[3] = 1.0f; }
    void copy_fields(const PointXYZINormal& o) {
        x = o.x; y = o.y; z = o.z; intensity = o.intensity;
        normal_x = o.normal_x; normal_y = o.normal_y; normal_z = o.normal_z; curvature = o.curvature;
    }
};
static_assert(sizeof(PointXYZI) == 32 && sizeof(PointXYZINormal) == 48, "PCL point layouts");

template <class P> struct PointCloud {
    typedef std::shared_ptr<PointCloud> Ptr;
    typedef std::shared_ptr<const PointCloud> ConstPtr;
    PCLHeader header;
    std::vector<P> points;
    uint32_t width = 0, height = 0;
    bool is_dense = true;
    size_t size() const { return points.size(); }
    bool empty() const { return points.empty(); }
    void clear() { points.clear(); width = 0; height = 0; }
    void resize(size_t n) { points.resize(n); width = (uint32_t)n; height = 1; }
    void push_back(const P& p) { points.push_back(p); width = (uint32_t)points.size(); height = 1; }
    P& back() { return points.back(); }
    PointCloud& operator+=(const PointCloud& o) {
        points.insert(points.end(), o.points.begin(), o.points.end());
        width = (uint32_t)points.size(); height = 1;
        is_dense = is_dense && o.is_dense;
        return *this;
    }
};

template <class P> void copyPointCloud(const PointCloud<P>& in, PointCloud<P>& out) { out = in; }

// pcl::removeNaNFromPointCloud: a cloud that declares itself dense is copied as it is; otherwise the points with a non-finite
// x, y or z are dropped
template <class P> void removeNaNFromPointCloud(const PointCloud<P>& in, PointCloud<P>& out, std::vector<int>& index) {
    if (in.is_dense) {
        if (&in != &out) out = in;
        index.resize(out.points.size());
        for (size_t j = 0; j < index.size(); ++j) index[j] = (int)j;
        return;
    }
    std::vector<P> kept;
    index.clear();
    for (size_t i = 0; i < in.points.size(); ++i) {
        const P& p = in.points[i];
        if (!std::isfinite(p.x) || !std::isfinite(p.y) || !std::isfinite(p.z)) continue;
        kept.push_back(p);
        index.push_back((int)i);
    }
    out.header = in.header;
    out.points.swap(kept);
    out.height = 1; out.width = (uint32_t)out.points.size();
    out.is_dense = true;
}

template <class P> void toROSMsg(const PointCloud<P>& cloud, sensor_msgs::PointCloud2& msg) {
    msg.height = 1;
    msg.width = (uint32_t)cloud.points.size();
    msg.point_step = sizeof(P);
    msg.row_step = msg.point_step * msg.width;
    msg.fields.clear();
    msg.is_dense = cloud.is_dense;
    msg.pcl_point_size = sizeof(P);
    msg.data.resize((size_t)msg.row_step);
    if (msg.width) std::memcpy(msg.data.data(), cloud.points.data(), msg.data.size());
}

template <class P> void fromROSMsg(const sensor_msgs::PointCloud2& msg, PointCloud<P>& cloud) {
    const size_t n = (size_t)msg.width * msg.height;
    cloud.points.assign(n, P());
    if (msg.pcl_point_size == sizeof(P)) {
        const P* src = reinterpret_cast<const P*>(msg.data.data());
        for (size_t i = 0; i < n; ++i) cloud.points[i].copy_fields(src[i]);
    } else if (msg.pcl_point_size == 0 && sizeof(P) == sizeof(PointXYZI)) {
        std::vector<RefPc2Field> f(msg.fields.size());
        for (size_t k = 0; k < f.size(); ++k) {
            std::memset(f[k].name, 0, 16);
            std::strncpy(f[k].name, msg.fields[k].name.c_str(), 15);
            f[k].offset = msg.fields[k].offset; f[k].datatype = msg.fields[k].datatype; f[k].count = msg.fields[k].count;
        }
        if (orc_pc2_to_pt32(msg.data.data(), msg.height, msg.width, msg.point_step, msg.row_step, f.data(), (int)f.size(),
                            reinterpret_cast<float*>(cloud.points.data())) != (int)n)
            std::abort();
    } else {
        std::abort();
    }
    cloud.width = msg.width; cloud.height = msg.height;
    cloud.is_dense = msg.is_dense;
}

// pcl::VoxelGrid: orc_voxelgrid
template <class P> struct VoxelGrid {
    std::shared_ptr<const PointCloud<P>> input;
    float leaf = 0;
    void setLeafSize(float lx, float, float) { leaf = lx; }
    void setInputCloud(const std::shared_ptr<PointCloud<P>>& c) { input = c; }
    void filter(PointCloud<P>& out) {
        const PointCloud<P> in = *input;   // the input may be the output
        std::vector<P> buf(in.points.size());
        int m = orc_voxelgrid(in.points.data(), (int)in.points.size(), (int)sizeof(P), leaf, buf.data(), (int)buf.size());
        if (m < 0 || m > (int)buf.size()) std::abort();
        out.header = in.header;
        out.points.assign(buf.begin(), buf.begin() + m);
        out.width = (uint32_t)m; out.height = 1; out.is_dense = true;
    }
};

// pcl::KdTreeFLANN: the oracle's exact 5-NN (ascending squared distance, ties by index)
template <class P> struct KdTreeFLANN {
    typedef std::shared_ptr<KdTreeFLANN> Ptr;
    void* tree = nullptr;
    KdTreeFLANN() {}
    KdTreeFLANN(const KdTreeFLANN&) = delete;
    ~KdTreeFLANN() { if (tree) orc_kdtree_free(tree); }
    void setInputCloud(const std::shared_ptr<PointCloud<P>>& c) {
        std::vector<float> xyzw(4 * c->points.size());
        for (size_t i = 0; i < c->points.size(); ++i) {
            xyzw[4 * i] = c->points[i].x; xyzw[4 * i + 1] = c->points[i].y; xyzw[4 * i + 2] = c->points[i].z; xyzw[4 * i + 3] = 1.0f;
        }
        if (tree) orc_kdtree_free(tree);
        tree = orc_kdtree_build(xyzw.data(), (int)c->points.size());
        size_ = (int)c->points.size();
    }
    int nearestKSearch(const P& q, int k, std::vector<int>& idx, std::vector<float>& sqd) const {
        if (k != 5 || size_ < 5) std::abort();   // the odometry asks for 5 and reads all 5
        const float qv[3] = {q.x, q.y, q.z};
        idx.resize(5); sqd.resize(5);
        orc::knn5_one(tree, qv, idx.data(), sqd.data());
        return 5;
    }
    int size_ = 0;
};

template <class P> struct IterativeClosestPoint {};
class RangeImage {};

}  // namespace pcl
