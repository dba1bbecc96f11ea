// TEST INFRASTRUCTURE: an independent CPU restatement of pcl::fromROSMsg(sensor_msgs::PointCloud2 -> pcl::PointXYZI)
// (R/src/Preprocessing.cpp:277), the reference the device decode (k_pc2_to_pt32) is compared against.  It deliberately does not
// include the library's pc2_fields.h: field matching and the copy are written out again here.
// from-knowledge (PCL 1.8-1.10, conversions.h / point_cloud.h): createMapping maps each field of the point type to the FIRST
// message field with the same name, the same datatype (FLOAT32 = 7) and count 1 (or 0); fromPCLPointCloud2 then copies each
// mapped field of point (row, col) from data + row * row_step + col * point_step into a default-constructed point
// (x = y = z = intensity = 0, data[3] = 1).  Unmapped fields keep their default.
#include <cstring>

namespace {
struct OrcField { char name[16]; unsigned int offset; unsigned char datatype; unsigned int count; };   // sensor_msgs::PointField

bool same_name(const OrcField& f, const char* want) {
    char buf[17];
    memcpy(buf, f.name, 16);
    buf[16] = '\0';
    return strcmp(buf, want) == 0 && memchr(f.name, '\0', 16) != nullptr;
}
}  // namespace

// out: width * height PointXYZI records (8 floats each).  Returns the number of points, or -1 when a mapped field does not fit
// in point_step (never read past a point).
extern "C" int orc_pc2_to_pt32(const unsigned char* data, unsigned int height, unsigned int width, unsigned int point_step,
                               unsigned int row_step, const OrcField* fields, int n_fields, float* out) {
    static const char* const kName[4] = {"x", "y", "z", "intensity"};
    static const int kDst[4] = {0, 1, 2, 4};          // float slot inside pcl::PointXYZI
    int src[4];
    for (int k = 0; k < 4; ++k) {
        src[k] = -1;
        for (int f = 0; f < n_fields; ++f) {
            if (same_name(fields[f], kName[k]) && fields[f].datatype == 7 && (fields[f].count == 1 || fields[f].count == 0)) {
                if (fields[f].offset + 4ull > point_step) return -1;
                src[k] = (int)fields[f].offset;
                break;
            }
        }
    }
    for (unsigned int r = 0; r < height; ++r) {
        for (unsigned int c = 0; c < width; ++c) {
            const unsigned char* p = data + (size_t)r * row_step + (size_t)c * point_step;
            float* o = out + 8 * ((size_t)r * width + c);
            const float init[8] = {0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 0.f};
            memcpy(o, init, sizeof(init));
            for (int k = 0; k < 4; ++k)
                if (src[k] >= 0) memcpy(o + kDst[k], p + src[k], 4);
        }
    }
    return (int)((size_t)height * width);
}
