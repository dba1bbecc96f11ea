// PCL's field tables of the library's two point types and the field matching of pcl::fromROSMsg, for the publishing side
// (liliom_pc2_layout) and the PointCloud2 ingest (liliom_convert_pc2 / liliom_extract_rot_pc2, liliom_pre_cloud_pc2), the
// match and read of the driver's per-point `ring` field (LILIOM_RING_FIELD) and of its per-point time field (LILIOM_TIME_FIELD).
// Free of CUDA types, so that the CPU tests compile it as it is (tests/pc2_host.cpp); the functions the kernels share with the
// host (pc2_ring_value, pc2_time_value, pc2_rel_time) are __host__ __device__ under nvcc.
#pragma once
#include <climits>
#include <cstring>
#include "../../include/liliom.h"

namespace lili {

#if defined(__CUDACC__)
#define PC2_HD __host__ __device__ __forceinline__
#else
#define PC2_HD inline
#endif

constexpr unsigned char kPc2Float32 = 7;       // sensor_msgs::PointField::FLOAT32
constexpr unsigned char kPc2Uint8 = 2;         // sensor_msgs::PointField::UINT8
constexpr unsigned char kPc2Uint16 = 4;        // sensor_msgs::PointField::UINT16
constexpr unsigned char kPc2Uint32 = 6;        // sensor_msgs::PointField::UINT32
constexpr unsigned char kPc2Float64 = 8;       // sensor_msgs::PointField::FLOAT64

// from-knowledge: POINT_CLOUD_REGISTER_POINT_STRUCT of pcl::PointXYZINormal / pcl::PointXYZI (PCL 1.8-1.10), in the order
// pcl::toROSMsg lists the fields; every field is FLOAT32 with count 1
struct Pc2Name { const char* name; unsigned int offset; };
constexpr Pc2Name kPc2Fields48[] = {{"x", 0}, {"y", 4}, {"z", 8}, {"normal_x", 16}, {"normal_y", 20}, {"normal_z", 24},
                                    {"intensity", 32}, {"curvature", 36}};
constexpr Pc2Name kPc2Fields32[] = {{"x", 0}, {"y", 4}, {"z", 8}, {"intensity", 16}};
constexpr int kPc2Fields32N = 4;

// Where each field of pcl::PointXYZI comes from in one message: src[k] = byte offset inside a point of the message field
// mapped to kPc2Fields32[k] (x, y, z, intensity), or -1 when no field matches (the point keeps PCL's default value 0).
// ring_src / ring_bytes: the `ring` field (offset, 1 for UINT8 or 2 for UINT16), matched only when the caller asks for it;
// -1 / 0 otherwise.
// time_src / time_type: the per-point time field (offset, datatype FLOAT32 / FLOAT64 / UINT32), matched only when the caller
// names it; -1 / 0 otherwise.
struct Pc2Map {
    int src[kPc2Fields32N];
    int n;                          // width * height
    int ring_src = -1;
    int ring_bytes = 0;
    int time_src = -1;
    int time_type = 0;
};

// name equality on the 16-byte, NUL-terminated liliom_pc2_field::name (a name without a NUL in 16 bytes matches nothing)
inline bool pc2_name_is(const char (&name)[16], const char* want) {
    const size_t len = strlen(want);
    return len < sizeof(name) && memcmp(name, want, len) == 0 && name[len] == '\0';
}

constexpr unsigned pc2_type_bit(unsigned char datatype) { return datatype < 32 ? 1u << datatype : 0u; }

// The one field rule of pc2_match: the FIRST field whose name is `name`, whose datatype is one of `types` (pc2_type_bit mask) and
// whose count is 1 or 0.  *off / *type = its offset and datatype, or -1 / 0 when there is none.  LILIOM_E_ARG when that field
// does not fit in point_step at its datatype's width; a field of another datatype is skipped, so it is never read.
inline int pc2_find(const liliom_pc2_msg* msg, const char* name, unsigned types, int* off, int* type) {
    *off = -1;
    *type = 0;
    for (int f = 0; f < msg->n_fields; ++f) {
        const liliom_pc2_field& F = msg->fields[f];
        if (!pc2_name_is(F.name, name) || !(types & pc2_type_bit(F.datatype)) || (F.count != 1 && F.count != 0)) continue;
        const int bytes = F.datatype == kPc2Float64 ? 8 : F.datatype == kPc2Uint16 ? 2 : F.datatype == kPc2Uint8 ? 1 : 4;
        if ((unsigned long long)F.offset + bytes > msg->point_step) return LILIOM_E_ARG;
        *off = (int)F.offset;
        *type = F.datatype;
        break;
    }
    return LILIOM_OK;
}

// from-knowledge: pcl::createMapping / pcl::detail::FieldMatches (PCL 1.8-1.10) — a point field is mapped to the FIRST message
// field whose name is equal, whose datatype is the point field's (FLOAT32) and whose count is 1 or 0.  A field that does not
// match is simply unmapped.  The message itself is input from outside the program: LILIOM_E_ARG for a null msg / data (a
// non-empty payload) / fields (n_fields > 0), n_fields < 0, point_step 0, row_step < width * point_step, width * height > INT_MAX,
// a mapped field that does not fit in point_step, or a big-endian payload.
// want_ring (LILIOM_RING_FIELD): the ring source is the FIRST field named `ring` with datatype UINT8 or UINT16 and count 1 or 0
// (what Velodyne, Ouster, Hesai and Robosense drivers publish; any other datatype is skipped).  LILIOM_E_ARG, too, when there
// is no such field or it does not fit in point_step.  Without want_ring the `ring` field is not looked at.
// time_name (LILIOM_TIME_FIELD): the time source is the FIRST field with that name, datatype FLOAT32, FLOAT64 or UINT32 and
// count 1 or 0 (Velodyne `time`, Ouster `t`, Hesai / Robosense `timestamp`; any other datatype is skipped).  LILIOM_E_ARG
// when there is no such field or it does not fit in point_step.  Without time_name no time field is looked at.
inline int pc2_match(const liliom_pc2_msg* msg, Pc2Map* out, bool want_ring = false, const char* time_name = nullptr) {
    if (!msg || !out || msg->n_fields < 0 || (msg->n_fields > 0 && !msg->fields)) return LILIOM_E_ARG;
    if (msg->point_step == 0 || msg->is_bigendian != 0) return LILIOM_E_ARG;
    if ((unsigned long long)msg->row_step < (unsigned long long)msg->width * msg->point_step) return LILIOM_E_ARG;
    const unsigned long long n = (unsigned long long)msg->width * msg->height;
    if (n > (unsigned long long)INT_MAX) return LILIOM_E_ARG;
    if (!msg->data && (unsigned long long)msg->height * msg->row_step > 0) return LILIOM_E_ARG;
    Pc2Map m;
    m.n = (int)n;
    int type;
    for (int k = 0; k < kPc2Fields32N; ++k)
        if (pc2_find(msg, kPc2Fields32[k].name, pc2_type_bit(kPc2Float32), &m.src[k], &type) != LILIOM_OK) return LILIOM_E_ARG;
    if (want_ring) {
        if (pc2_find(msg, "ring", pc2_type_bit(kPc2Uint8) | pc2_type_bit(kPc2Uint16), &m.ring_src, &type) != LILIOM_OK || m.ring_src < 0)
            return LILIOM_E_ARG;
        m.ring_bytes = type == kPc2Uint16 ? 2 : 1;
    }
    if (time_name) {
        const unsigned types = pc2_type_bit(kPc2Float32) | pc2_type_bit(kPc2Float64) | pc2_type_bit(kPc2Uint32);
        if (pc2_find(msg, time_name, types, &m.time_src, &m.time_type) != LILIOM_OK || m.time_src < 0) return LILIOM_E_ARG;
    }
    *out = m;
    return LILIOM_OK;
}

// The ring of one point (its bytes at `point`): the little-endian UINT8 / UINT16 at ring_src, read byte by byte (any offset).
PC2_HD unsigned pc2_ring_value(const unsigned char* point, int ring_src, int ring_bytes) {
    const unsigned char* p = point + ring_src;
    return ring_bytes == 2 ? (unsigned)p[0] | ((unsigned)p[1] << 8) : (unsigned)p[0];
}

// The time of one point: the little-endian FLOAT32 / FLOAT64 / UINT32 at time_src, read byte by byte (point i of a packed
// layout is unaligned) and converted exactly to double.
PC2_HD double pc2_time_value(const unsigned char* point, int time_src, int time_type) {
    const unsigned char* p = point + time_src;
    const int bytes = time_type == kPc2Float64 ? 8 : 4;
    unsigned long long u = 0;
    for (int b = 0; b < bytes; ++b) u |= (unsigned long long)p[b] << (8 * b);
    if (time_type == kPc2Float64) { double d; memcpy(&d, &u, 8); return d; }
    const unsigned w = (unsigned)u;
    if (time_type == kPc2Float32) { float f; memcpy(&f, &w, 4); return (double)f; }
    return (double)w;
}

// relTime of a return under LILIOM_TIME_FIELD: the reference's normalisation (:367, the first return 0 and the last 1) with the
// time in place of the azimuth; t_min / t_max over the returns that survive the NaN / 3 m removal.  A span of 0 gives 0.
PC2_HD float pc2_rel_time(double t, double t_min, double t_max) {
    const double span = t_max - t_min;
    return span > 0.0 ? (float)((t - t_min) / span) : 0.0f;
}

}  // namespace lili
