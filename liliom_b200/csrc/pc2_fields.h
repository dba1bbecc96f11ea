// PCL's field tables of the library's two point types and the field matching of pcl::fromROSMsg, for the publishing side
// (liliom_pc2_layout) and the PointCloud2 ingest (liliom_convert_pc2 / liliom_extract_rot_pc2, liliom_pre_cloud_pc2).
// Host-only and free of CUDA types, so that the CPU tests compile it as it is (tests/pc2_host.cpp).
#pragma once
#include <climits>
#include <cstring>
#include "../../include/liliom.h"

namespace lili {

constexpr unsigned char kPc2Float32 = 7;       // sensor_msgs::PointField::FLOAT32

// from-knowledge: POINT_CLOUD_REGISTER_POINT_STRUCT of pcl::PointXYZINormal / pcl::PointXYZI (PCL 1.8-1.10), in the order
// pcl::toROSMsg lists the fields; every field is FLOAT32 with count 1
struct Pc2Name { const char* name; unsigned int offset; };
constexpr Pc2Name kPc2Fields48[] = {{"x", 0}, {"y", 4}, {"z", 8}, {"normal_x", 16}, {"normal_y", 20}, {"normal_z", 24},
                                    {"intensity", 32}, {"curvature", 36}};
constexpr Pc2Name kPc2Fields32[] = {{"x", 0}, {"y", 4}, {"z", 8}, {"intensity", 16}};
constexpr int kPc2Fields32N = 4;

// Where each field of pcl::PointXYZI comes from in one message: src[k] = byte offset inside a point of the message field
// mapped to kPc2Fields32[k] (x, y, z, intensity), or -1 when no field matches (the point keeps PCL's default value 0).
struct Pc2Map {
    int src[kPc2Fields32N];
    int n;                          // width * height
};

// name equality on the 16-byte, NUL-terminated liliom_pc2_field::name (a name without a NUL in 16 bytes matches nothing)
inline bool pc2_name_is(const char (&name)[16], const char* want) {
    const size_t len = strlen(want);
    return len < sizeof(name) && memcmp(name, want, len) == 0 && name[len] == '\0';
}

// from-knowledge: pcl::createMapping / pcl::detail::FieldMatches (PCL 1.8-1.10) — a point field is mapped to the FIRST message
// field whose name is equal, whose datatype is the point field's (FLOAT32) and whose count is 1 or 0.  A field that does not
// match is simply unmapped.  The message itself is input from outside the program: LILIOM_E_ARG for a null msg / data (a
// non-empty payload) / fields (n_fields > 0), n_fields < 0, point_step 0, row_step < width * point_step, width * height > INT_MAX,
// a mapped field that does not fit in point_step, or a big-endian payload.
inline int pc2_match(const liliom_pc2_msg* msg, Pc2Map* out) {
    if (!msg || !out || msg->n_fields < 0 || (msg->n_fields > 0 && !msg->fields)) return LILIOM_E_ARG;
    if (msg->point_step == 0 || msg->is_bigendian != 0) return LILIOM_E_ARG;
    if ((unsigned long long)msg->row_step < (unsigned long long)msg->width * msg->point_step) return LILIOM_E_ARG;
    const unsigned long long n = (unsigned long long)msg->width * msg->height;
    if (n > (unsigned long long)INT_MAX) return LILIOM_E_ARG;
    if (!msg->data && (unsigned long long)msg->height * msg->row_step > 0) return LILIOM_E_ARG;
    Pc2Map m;
    m.n = (int)n;
    for (int k = 0; k < kPc2Fields32N; ++k) {
        m.src[k] = -1;
        for (int f = 0; f < msg->n_fields; ++f) {
            const liliom_pc2_field& F = msg->fields[f];
            if (!pc2_name_is(F.name, kPc2Fields32[k].name) || F.datatype != kPc2Float32 || (F.count != 1 && F.count != 0)) continue;
            if ((unsigned long long)F.offset + 4 > msg->point_step) return LILIOM_E_ARG;
            m.src[k] = (int)F.offset;
            break;
        }
    }
    *out = m;
    return LILIOM_OK;
}

}  // namespace lili
