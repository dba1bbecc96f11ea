// The per-point decode of the two driver formats the library takes, shared by the decode stages (WireStLivox, WireStPc2 in
// api.cu) and the CPU tests (tests/wire_host.cpp compiles this same file):
//   * livox_ros_driver::CustomPoint -> pcl::PointXYZINormal (FormatConvert, L/src/FormatConvert.cpp:11-24);
//   * one point of a sensor_msgs/PointCloud2 -> pcl::PointXYZI (pcl::fromROSMsg, R/src/Preprocessing.cpp:277), with the ring
//     and time side channels of LILIOM_RING_FIELD / LILIOM_TIME_FIELD (field matching: pc2_fields.h).
// Payload fields sit at any byte offset, so every word is assembled from bytes.  The float operations are spelled with
// round-to-nearest intrinsics on the device and as plain operators on the host (built with -ffp-contract=off), so both give
// the bits of the reference's x86-64 build.
#pragma once
#include <cstdint>
#include <cstring>
#include "pcl_xform.h"      // VGB_HD, vg_st4, mulx / addx
#include "pc2_fields.h"     // pc2_ring_value, pc2_time_value

namespace lili {

// little-endian 32-bit word assembled from bytes: sensor payloads carry fields at any byte offset, never read them wider
VGB_HD unsigned rd32(const unsigned char* p) {
    return (unsigned)p[0] | ((unsigned)p[1] << 8) | ((unsigned)p[2] << 16) | ((unsigned)p[3] << 24);
}

#ifdef __CUDA_ARCH__
VGB_HD float wire_bits_f32(unsigned u) { return __uint_as_float(u); }
VGB_HD float wire_u2f(unsigned u) { return __uint2float_rn(u); }
VGB_HD float wire_fdiv(float a, float b) { return __fdiv_rn(a, b); }
#else
inline float wire_bits_f32(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
inline float wire_u2f(unsigned u) { return (float)u; }
inline float wire_fdiv(float a, float b) { return a / b; }
#endif

// Point i of n CustomPoint records of `stride` bytes (19, or 20 with the trailing pad) at `in`: the PointXYZINormal at
// out + 48 i.  Nothing for i >= n.
VGB_HD void livox_point_at(const unsigned char* __restrict__ in, int n, int stride, unsigned char* __restrict__ out, int i) {
    if (i >= n) return;
    const unsigned time_end = rd32(in + (size_t)(n - 1) * stride);                       // :13 points.back().offset_time
    const unsigned char* p = in + (size_t)i * stride;
    const unsigned off = rd32(p);
    const float x = wire_bits_f32(rd32(p + 4)), y = wire_bits_f32(rd32(p + 8)), z = wire_bits_f32(rd32(p + 12));
    const unsigned refl = p[16], line = p[18];
    const float s = wire_fdiv(wire_u2f(off), wire_u2f(time_end));                        // :19 float(offset_time / (float)time_end)
    const float intensity = (float)addx((double)line, mulx((double)s, 0.1));            // :20
    const float curvature = (float)mulx(0.1, (double)refl);                             // :21
    unsigned char* o = out + (size_t)i * 48;
    vg_st4(o, x, y, z, 1.0f);                                                           // pcl::PointXYZINormal default ctor: data[3] = 1
    vg_st4(o + 16, 0.f, 0.f, 0.f, 0.f);
    vg_st4(o + 32, intensity, curvature, 0.f, 0.f);
}

// How one accepted PointCloud2 is laid out and which of its fields the decode reads (pc2_match's Pc2Map and the header):
// src = byte offsets of x, y, z, intensity inside a point (-1: unmapped -> 0); ring_src / ring_bytes and time_src / time_type
// as in Pc2Map (read only when the decode is given a ring / time output).
struct Pc2Wire {
    unsigned width, point_step, row_step;
    int src[4];
    int ring_src, ring_bytes, time_src, time_type;
};
inline Pc2Wire pc2_wire(const liliom_pc2_msg* msg, const Pc2Map& m) {
    return Pc2Wire{msg->width, msg->point_step, msg->row_step, {m.src[0], m.src[1], m.src[2], m.src[3]},
                   m.ring_src, m.ring_bytes, m.time_src, m.time_type};
}

// Point i of the n = width * height points of the payload `in`, row-major over (row, column): the PointXYZI at out + 32 i and,
// when given, its ring at ring_out[i] and its time at time_out[i].  Nothing for i >= n.
VGB_HD void pc2_point_at(const unsigned char* __restrict__ in, int n, const Pc2Wire& w, unsigned char* __restrict__ out,
                         uint16_t* __restrict__ ring_out, double* __restrict__ time_out, int i) {
    if (i >= n) return;
    const unsigned r = (unsigned)i / w.width, col = (unsigned)i - r * w.width;
    const unsigned char* p = in + (size_t)r * w.row_step + (size_t)col * w.point_step;
    auto fld = [p](int off) { return off < 0 ? 0.0f : wire_bits_f32(rd32(p + off)); };
    // the fields are read before each output address is formed, the order that keeps the decode at 32 registers
    const float x = fld(w.src[0]), y = fld(w.src[1]), z = fld(w.src[2]);
    vg_st4(out + (size_t)i * 32, x, y, z, 1.0f);                                        // pcl::PointXYZI default ctor: data[3] = 1
    const float intensity = fld(w.src[3]);
    vg_st4(out + (size_t)i * 32 + 16, intensity, 0.f, 0.f, 0.f);
    if (ring_out) ring_out[i] = (uint16_t)pc2_ring_value(p, w.ring_src, w.ring_bytes);
    if (time_out) time_out[i] = pc2_time_value(p, w.time_src, w.time_type);
}

}  // namespace lili
