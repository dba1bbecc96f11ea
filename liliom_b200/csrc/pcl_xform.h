// transformCloud of one PCL point, shared by host and device (L/src/LidarOdometry.cpp:246-278, L/src/BackendFusion.cpp:730-767;
// R/src/LidarOdometry.cpp:239-264): the fp64 quaternion rotation of Eigen and the fp32 stores of the output point.
// Every operation is spelled with round-to-nearest intrinsics on the device and as a plain operator on the host (the host
// build is compiled with -ffp-contract=off), so the kernels, tests/gmap_host.cpp and the reference's generic x86-64 build
// give the same bits (SURVEY.md Appendix C.2).
#pragma once
#include "vg_box.h"

namespace lili {

struct D3 { double x, y, z; };
struct Q4 { double w, x, y, z; };

#ifdef __CUDA_ARCH__
VGB_HD double mulx(double a, double b) { return __dmul_rn(a, b); }
VGB_HD double addx(double a, double b) { return __dadd_rn(a, b); }
VGB_HD double subx(double a, double b) { return __dsub_rn(a, b); }
#else
VGB_HD double mulx(double a, double b) { return a * b; }
VGB_HD double addx(double a, double b) { return a + b; }
VGB_HD double subx(double a, double b) { return a - b; }
#endif

VGB_HD D3 cross_x(D3 a, D3 b) {
    return {subx(mulx(a.y, b.z), mulx(a.z, b.y)), subx(mulx(a.z, b.x), mulx(a.x, b.z)), subx(mulx(a.x, b.y), mulx(a.y, b.x))};
}

// Eigen::Quaterniond * Vector3d (QuaternionBase::_transformVector), not normalising:
//   uv = q.vec x v; uv += uv; v + w*uv + q.vec x uv
// reference call sites: L/src/LidarOdometry.cpp:231, L/src/Preprocessing.cpp:118.
VGB_HD D3 qrot_x(Q4 q, D3 v) {
    D3 qv{q.x, q.y, q.z};
    D3 uv = cross_x(qv, v);
    uv = {addx(uv.x, uv.x), addx(uv.y, uv.y), addx(uv.z, uv.z)};
    D3 c = cross_x(qv, uv);
    return {addx(addx(v.x, mulx(q.w, uv.x)), c.x), addx(addx(v.y, mulx(q.w, uv.y)), c.y), addx(addx(v.z, mulx(q.w, uv.z)), c.z)};
}

// the transformed xyz of a point (fp64 rotation + translation, stored as fp32)
VGB_HD VgXyz pcl_transform_xyz(Q4 q, D3 t, float x, float y, float z) {
    const D3 r = qrot_x(q, D3{(double)x, (double)y, (double)z});
    return {(float)addx(r.x, t.x), (float)addx(r.y, t.y), (float)addx(r.z, t.z)};
}

// One point of `stride` bytes (48: PointXYZINormal, 32: PointXYZI): xyz and, for 48-byte points, the normal rotated in fp64;
// w = 1, intensity/curvature copied, padding cleared.  `out` may be `in`.
VGB_HD void pcl_transform_point(const unsigned char* in, int stride, Q4 q, D3 t, unsigned char* out) {
    const VgF4 a = vg_ld4(in);
    const VgXyz p = pcl_transform_xyz(q, t, a.x, a.y, a.z);
    vg_st4(out, p.x, p.y, p.z, 1.0f);
    if (stride == 48) {
        const VgF4 b = vg_ld4(in + 16);
        const VgF4 cc = vg_ld4(in + 32);
        D3 nr = qrot_x(q, D3{(double)b.x, (double)b.y, (double)b.z});
        vg_st4(out + 16, (float)nr.x, (float)nr.y, (float)nr.z, 0.f);
        vg_st4(out + 32, cc.x, cc.y, 0.f, 0.f);
    } else {
        const VgF4 b = vg_ld4(in + 16);
        vg_st4(out + 16, b.x, 0.f, 0.f, 0.f);
    }
}

}  // namespace lili
