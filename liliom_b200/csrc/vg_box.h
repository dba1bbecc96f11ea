// The bounding box every VoxelGrid and cell grid starts from, and PCL's VoxelGrid parameters derived from it
// (pcl::getMinMax3D + pcl::VoxelGrid::applyFilter, voxel_grid.hpp).  The box is 7 ints: min xyz and max xyz of the finite
// points in the ordered-int encoding below, so that integer atomics order floats, then the finite count.  Every kernel that
// measures a box or turns one into voxel indices (voxelgrid.cu, map_inc.cu, extract_rot.cu, grid_knn.cu) and the host code
// that reads a box back use this file, so they agree on every voxel.  Plain C++ usable from device code and from the host
// (tests/vg_box_host.cpp compiles this same file for the CPU test tier).
//
// No expression here is a contractible a*b+c: the file is compiled both with --fmad=false (voxelgrid.cu) and without it
// (grid_knn.cu) and must give the same bits either way.  Integer products that can leave int / long long are formed in
// unsigned arithmetic and converted back: the device's wrapped bits, no undefined behaviour in the host build.
#pragma once
#include <climits>
#include <cmath>
#include <cstring>

#ifdef __CUDACC__
#define VGB_HD __host__ __device__ __forceinline__
#else
#define VGB_HD inline
#endif

namespace lili {

// Parameters of one VoxelGrid pass (on the device: produced there, no host round trip).
struct VgParams {
    float inv_leaf;
    int   min_b[3];
    int   div_b[3];
    int   mul[3];
    int   overflow;    // PCL: "Leaf size is too small" -> output = input
    int   n_finite;
    int   bail;        // cooperative single-launch filter declined this input (see k_vg_coop): redo with the sort chain
};

// float <-> ordered int: integer order = float order (-0 below +0; NaNs of either sign outside every finite value)
VGB_HD int vg_f2ord(float f) {
#ifdef __CUDA_ARCH__
    const int i = __float_as_int(f);
#else
    int i;
    memcpy(&i, &f, 4);
#endif
    return i >= 0 ? i : i ^ 0x7fffffff;
}
VGB_HD float vg_ord2f(int i) {
    const int j = i >= 0 ? i : i ^ 0x7fffffff;
#ifdef __CUDA_ARCH__
    return __int_as_float(j);
#else
    float f;
    memcpy(&f, &j, 4);
    return f;
#endif
}

// Word k of a box: [0..2] min, [3..5] max, [6] finite count.  vg_box_empty(k) is the empty box's word; vg_box_join(k, a, b)
// the word of the union of two boxes holding a and b there.
constexpr int kBoxInts = 7;
VGB_HD int vg_box_empty(int k) { return k < 3 ? INT_MAX : (k < 6 ? INT_MIN : 0); }
VGB_HD int vg_box_join(int k, int a, int b) { return k < 3 ? (a < b ? a : b) : (k < 6 ? (a > b ? a : b) : a + b); }
VGB_HD void vg_box_add(int* box, float x, float y, float z) {      // a finite point
    const int e[3] = {vg_f2ord(x), vg_f2ord(y), vg_f2ord(z)};
    for (int k = 0; k < 3; ++k) { box[k] = vg_box_join(k, box[k], e[k]); box[3 + k] = vg_box_join(3 + k, box[3 + k], e[k]); }
    box[6] += 1;
}
VGB_HD void vg_box_merge(int* box, const int* other) {
    for (int k = 0; k < kBoxInts; ++k) box[k] = vg_box_join(k, box[k], other[k]);
}
#ifdef __CUDACC__
__device__ __forceinline__ void vg_box_atomic(int* dst, int k, int v) {      // word k of a box joined into *dst
    if (k < 3) atomicMin(dst, v);
    else if (k < 6) atomicMax(dst, v);
    else atomicAdd(dst, v);
}
#endif

VGB_HD long long vgb_mul64(long long a, long long b) { return (long long)((unsigned long long)a * (unsigned long long)b); }

// PCL's parameters for a box: min_b = floor(min / leaf), div_b = max_b - min_b + 1, mul = {1, dx, dx*dy}, and the
// "leaf size too small" test dx*dy*dz > INT_MAX with d = (long long)((max - min) / leaf) + 1.  An empty box gives
// min_b = 0, div_b = 1.
VGB_HD VgParams vg_params(const int* box, float leaf) {
    VgParams p;
    p.inv_leaf = 1.0f / leaf;                       // Eigen::Array4f::Ones() / leaf_size_
    p.n_finite = box[6];
    p.overflow = 0;
    p.bail = 0;
    if (p.n_finite == 0) {
        for (int k = 0; k < 3; ++k) { p.min_b[k] = 0; p.div_b[k] = 1; }
    } else {
        long long d[3];
        for (int k = 0; k < 3; ++k) {
            const float lo = vg_ord2f(box[k]), hi = vg_ord2f(box[3 + k]);
            d[k] = (long long)((unsigned long long)(long long)((hi - lo) * p.inv_leaf) + 1ull);
            p.min_b[k] = (int)floorf(lo * p.inv_leaf);
            const int max_b = (int)floorf(hi * p.inv_leaf);
            p.div_b[k] = (int)((unsigned)max_b - (unsigned)p.min_b[k] + 1u);
        }
        if (vgb_mul64(vgb_mul64(d[0], d[1]), d[2]) > (long long)INT_MAX) p.overflow = 1;
    }
    p.mul[0] = 1; p.mul[1] = p.div_b[0]; p.mul[2] = (int)((unsigned)p.div_b[0] * (unsigned)p.div_b[1]);
    return p;
}

// Width of the VoxelGrid sort chain's keys for a cloud with this box: the fewest bits (at least 8) that hold every voxel
// index with the all-ones key of that width left free for the non-finite points' sentinel; 32 when the box is empty, in
// PCL's overflow case, or when the voxel count does not fit.
VGB_HD int vg_key_bits(const int* box, float leaf) {
    const VgParams p = vg_params(box, leaf);
    if (p.n_finite <= 0 || p.overflow) return 32;
    const long long cells = vgb_mul64(vgb_mul64(p.div_b[0], p.div_b[1]), p.div_b[2]);
    if (!(cells > 0 && cells < (1LL << 31))) return 32;
    int bits = 8;
    while ((1LL << bits) <= cells) ++bits;
    return bits;
}

// Absolute voxel key of a finite point: 21 bits per coordinate floor(p / leaf) + 2^20, packed (z, y, x) from the top, so
// that key order is PCL's index order for any box.  False (key untouched) when a coordinate is outside (-2^20, 2^20).
VGB_HD bool vg_abs_key(float x, float y, float z, float inv_leaf, unsigned long long* key) {
    const float fx = floorf(x * inv_leaf), fy = floorf(y * inv_leaf), fz = floorf(z * inv_leaf);
    const float lim = 1048576.0f;
    if (!(fabsf(fx) < lim && fabsf(fy) < lim && fabsf(fz) < lim)) return false;
    *key = ((unsigned long long)((int)fz + (1 << 20)) << 42) | ((unsigned long long)((int)fy + (1 << 20)) << 21) |
           (unsigned long long)((int)fx + (1 << 20));
    return true;
}

}  // namespace lili
