// The VoxelGrid arithmetic shared by host and device (pcl::getMinMax3D + pcl::VoxelGrid::applyFilter, voxel_grid.hpp, and
// pcl::CentroidPoint, centroid.hpp):
//   * the bounding box every VoxelGrid and cell grid starts from: 7 ints, min xyz and max xyz of the finite points in the
//     ordered-int encoding below, so that integer atomics order floats, then the finite count;
//   * PCL's parameters derived from it and a point's voxel index;
//   * a voxel's centroid: the fields summed, the walk over its members in a sorted entry array, and the output point.
// The kernels that measure a box, index voxels or write centroids (the sort chain and k_vg_coop in voxelgrid.cu, the
// incremental map in map.cu, the per-ring filter in extract_rot.cu, the cell grid in grid_knn.cu, the global map's table
// filter in keyframes.cu) and the host code that
// reads a box back use this file, so they agree on every voxel and every bit of a centroid.  Plain C++ usable from device
// code and from the host (tests/vg_box_host.cpp compiles this same file for the CPU test tier).
//
// No expression here is a contractible a*b+c: the file is compiled both with --fmad=false (voxelgrid.cu) and without it
// (grid_knn.cu) and must give the same bits either way; the one sum of products (a normal's squared norm) is spelled with
// round-to-nearest intrinsics on the device.  Integer products that can leave int / long long are formed in unsigned
// arithmetic and converted back: the device's wrapped bits, no undefined behaviour in the host build.
#pragma once
#include <climits>
#include <cmath>
#include <cstring>
#include <type_traits>

#ifdef __CUDACC__
#define VGB_HD __host__ __device__ __forceinline__
#define VGB_PRAGMA(x) _Pragma(#x)      // loop pragmas of the device build
#else
#define VGB_HD inline
#define VGB_PRAGMA(x)
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
    int   bail;        // cooperative single-launch filter declined this input (see k_vg_coop), or a box bound's cell lies outside
                       // int range (vg_params: x86 then sends indices to INT_MIN, outside the box): redo with full-width sort keys
    int   wraps;       // div_b[0]*div_b[1]*div_b[2] >= 2^32 (vg_wraps): PCL's int index wraps, so two cells can share an index, the
                       // index order is not the cells' (z, y, x) order, and a finite point can take the all-ones 32-bit index
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
// Every thread of a block (blockDim.x <= 256) joins its box into the box at mm: a warp reduction, then one set of atomics per
// BLOCK.  (The seven words are single addresses, and one set per warp (9.5k warps) serialised into ~55 us at the L2 whatever
// the input size: measured on a 500k-point frame, push 25 -> 83 us.)
__device__ __forceinline__ void vg_box_commit(int* box, int* mm) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int k = 0; k < kBoxInts; ++k) box[k] = vg_box_join(k, box[k], __shfl_xor_sync(0xffffffffu, box[k], o));
    }
    __shared__ int s_box[kBoxInts][8];
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < kBoxInts; ++k) s_box[k][w] = box[k];
    }
    __syncthreads();
    if (threadIdx.x < kBoxInts) {
        const int k = threadIdx.x, nw = (blockDim.x + 31) >> 5;
        int v = vg_box_empty(k);
        for (int j = 0; j < nw; ++j) v = vg_box_join(k, v, s_box[k][j]);
        if (v != vg_box_empty(k)) vg_box_atomic(&mm[k], k, v);
    }
}
#endif

VGB_HD long long vgb_mul64(long long a, long long b) { return (long long)((unsigned long long)a * (unsigned long long)b); }

// Whether div_b[0]*div_b[1]*div_b[2] >= 2^32, each division read as the unsigned count max_b - min_b + 1 (0: 2^32 cells).  The
// overflow test multiplies d = trunc((max - min) / leaf) + 1, which can be one smaller per axis than div_b, so this can hold
// while PCL filters: its int index then wraps modulo 2^32.
VGB_HD bool vg_wraps(const int* div_b) {
    unsigned long long c = 1;
    for (int k = 0; k < 3; ++k) {
        const unsigned long long d = div_b[k] == 0 ? (1ull << 32) : (unsigned long long)(unsigned)div_b[k];
        if (d >= (1ull << 32)) return true;
        c *= d;                                     // < 2^32 * 2^32: no wrap
        if (c >= (1ull << 32)) return true;
    }
    return false;
}

// float -> int and float -> int64 as PCL's x86-64 build converts them (cvttss2si): truncation toward zero, and INT_MIN /
// INT64_MIN for NaN, +-inf and every value outside the target's range.  The device's own conversion saturates instead, and in
// C++ an out-of-range conversion is undefined, so the rule is written out: a far or huge box gives PCL's indices, not clamped ones.
VGB_HD bool vg_int_ok(float v) { return v >= -2147483648.0f && v < 2147483648.0f; }
VGB_HD int vg_f2i_x86(float v) { return vg_int_ok(v) ? (int)v : INT_MIN; }
VGB_HD long long vg_f2ll_x86(float v) { return (v >= -9223372036854775808.0f && v < 9223372036854775808.0f) ? (long long)v : LLONG_MIN; }

// PCL's parameters for a box: min_b = floor(min / leaf), div_b = max_b - min_b + 1, mul = {1, dx, dx*dy}, and the
// "leaf size too small" test dx*dy*dz > INT_MAX with d = (long long)((max - min) / leaf) + 1.  An empty box gives
// min_b = 0, div_b = 1.  Conversions follow x86's rule (vg_f2i_x86); d + 1 and the products wrap as x86's do.
VGB_HD VgParams vg_params(const int* box, float leaf) {
    VgParams p;
    p.inv_leaf = 1.0f / leaf;                       // Eigen::Array4f::Ones() / leaf_size_
    p.n_finite = box[6];
    p.overflow = 0;
    p.bail = 0;
    p.wraps = 0;
    if (p.n_finite == 0) {
        for (int k = 0; k < 3; ++k) { p.min_b[k] = 0; p.div_b[k] = 1; }
    } else {
        long long d[3];
        for (int k = 0; k < 3; ++k) {
            const float lo = vg_ord2f(box[k]), hi = vg_ord2f(box[3 + k]);
            d[k] = (long long)((unsigned long long)vg_f2ll_x86((hi - lo) * p.inv_leaf) + 1ull);
            const float flo = floorf(lo * p.inv_leaf), fhi = floorf(hi * p.inv_leaf);
            if (!vg_int_ok(flo) || !vg_int_ok(fhi)) p.bail = 1;
            p.min_b[k] = vg_f2i_x86(flo);
            const int max_b = vg_f2i_x86(fhi);
            p.div_b[k] = (int)((unsigned)max_b - (unsigned)p.min_b[k] + 1u);
        }
        if (vgb_mul64(vgb_mul64(d[0], d[1]), d[2]) > (long long)INT_MAX) p.overflow = 1;
        p.wraps = vg_wraps(p.div_b) ? 1 : 0;
    }
    p.mul[0] = 1; p.mul[1] = p.div_b[0]; p.mul[2] = (int)((unsigned)p.div_b[0] * (unsigned)p.div_b[1]);
    return p;
}

// PCL's voxel index of a finite point relative to the box: i0·mul0 + i1·mul1 + i2·mul2 with ik = floor(p_k / leaf) - min_b[k]
// (x86's conversion: an ik out of int range is INT_MIN)
VGB_HD unsigned vg_rel_index(const VgParams& p, float x, float y, float z) {
    const int i0 = vg_f2i_x86(floorf(x * p.inv_leaf) - (float)p.min_b[0]);
    const int i1 = vg_f2i_x86(floorf(y * p.inv_leaf) - (float)p.min_b[1]);
    const int i2 = vg_f2i_x86(floorf(z * p.inv_leaf) - (float)p.min_b[2]);
    return (unsigned)i0 * (unsigned)p.mul[0] + (unsigned)i1 * (unsigned)p.mul[1] + (unsigned)i2 * (unsigned)p.mul[2];
}

// Width of the VoxelGrid sort chain's keys for a cloud with this box, when they are 32-bit ones: the fewest bits (at least 8)
// that hold every voxel index with the all-ones key of that width left free for the non-finite points' sentinel; 32 when the
// box is empty, in PCL's overflow case, when the voxel count does not fit, or when a box bound's cell leaves int range (x86
// then sends the indices to INT_MIN, outside the box).  Where the index wraps, 32-bit keys do not suffice (vg_chain_key_bits).
VGB_HD int vg_key_bits(const int* box, float leaf) {
    const VgParams p = vg_params(box, leaf);
    if (p.n_finite <= 0 || p.overflow || p.bail) return 32;
    const long long cells = vgb_mul64(vgb_mul64(p.div_b[0], p.div_b[1]), p.div_b[2]);
    if (!(cells > 0 && cells < (1LL << 31))) return 32;
    int bits = 8;
    while ((1LL << bits) <= cells) ++bits;
    return bits;
}

// Sort keys wider than 32 bits: 64-bit keys, the voxel index in the low 32 bits and the non-finite points' flag at bit 32,
// sorted on 33 bits.  Needed when PCL filters a box whose index wraps (VgParams::wraps): any 32-bit value is then a finite
// point's index, and an all-ones sentinel would share a key with it.
constexpr int kVgWideKeyBits = 33;
VGB_HD bool vg_wide_keys(const VgParams& p) { return p.n_finite > 0 && !p.overflow && p.wraps; }

// The sort chain's key width for a box known in advance: kVgWideKeyBits where the index wraps, vg_key_bits otherwise.
VGB_HD int vg_chain_key_bits(const int* box, float leaf) {
    return vg_wide_keys(vg_params(box, leaf)) ? kVgWideKeyBits : vg_key_bits(box, leaf);
}

// Absolute voxel key of a finite point: 21 bits per coordinate floor(p / leaf) + 2^20, packed (z, y, x) from the top.  Key
// order is the cells' (z, y, x) order, which is PCL's index order, and distinct cells have distinct PCL indices, only while
// the index does not wrap (VgParams::wraps): the paths built on these keys decline such boxes.  False (key untouched) when a
// coordinate is outside (-2^20, 2^20).
VGB_HD bool vg_abs_key(float x, float y, float z, float inv_leaf, unsigned long long* key) {
    const float fx = floorf(x * inv_leaf), fy = floorf(y * inv_leaf), fz = floorf(z * inv_leaf);
    const float lim = 1048576.0f;
    if (!(fabsf(fx) < lim && fabsf(fy) < lim && fabsf(fz) < lim)) return false;
    *key = ((unsigned long long)((int)fz + (1 << 20)) << 42) | ((unsigned long long)((int)fy + (1 << 20)) << 21) |
           (unsigned long long)((int)fx + (1 << 20));
    return true;
}

// ---- the centroid of a voxel (pcl::CentroidPoint over a 48-byte PointXYZINormal or a 32-byte PointXYZI)
#ifdef __CUDACC__
typedef float4 VgF4;
VGB_HD VgF4 vg_ld4(const unsigned char* p) { return *reinterpret_cast<const float4*>(p); }
VGB_HD void vg_st4(unsigned char* p, float a, float b, float c, float d) { *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d); }
#else
struct VgF4 { float x, y, z, w; };
inline VgF4 vg_ld4(const unsigned char* p) { VgF4 v; memcpy(&v, p, 16); return v; }
inline void vg_st4(unsigned char* p, float a, float b, float c, float d) { const VgF4 v{a, b, c, d}; memcpy(p, &v, 16); }
#endif

// The fields of a point the centroid sums, in this order: x y z nx ny nz intensity curvature (48 bytes), x y z intensity (32).
template <int STRIDE> constexpr int kVgFields = STRIDE == 48 ? 8 : 4;
template <int STRIDE>
VGB_HD void vg_load(const unsigned char* src, float* f) {
    const VgF4 a = vg_ld4(src), b = vg_ld4(src + 16);
    f[0] = a.x; f[1] = a.y; f[2] = a.z;
    if constexpr (STRIDE == 48) {
        const VgF4 c = vg_ld4(src + 32);
        f[3] = b.x; f[4] = b.y; f[5] = b.z; f[6] = c.x; f[7] = c.y;
    } else {
        f[3] = b.x;
    }
}

// Per-field fp32 sums and the member count; points are added in member order.
template <int STRIDE>
struct VgAcc {
    float s[kVgFields<STRIDE>] = {};
    int n = 0;
    VGB_HD void add(const float* f) {
        VGB_PRAGMA(unroll)
        for (int k = 0; k < kVgFields<STRIDE>; ++k) s[k] += f[k];
        ++n;
    }
};

// Entry i of a sorted key array whose first n_valid entries are valid starts a voxel.
template <typename K>
VGB_HD bool vg_is_head(const K* keys, int i, int n_valid) { return i < n_valid && (i == 0 || keys[i] != keys[i - 1]); }

// The fields of point m through a loader: either the plain loader load(m), the address of a stored point (read with vg_load),
// or load(m, f), which writes the fields itself (a point transformed on load, kf_table.h).
template <int STRIDE, typename Load>
VGB_HD void vg_fetch(const Load& load, int m, float* f) {
    if constexpr (std::is_invocable_v<const Load&, int, float*>) load(m, f);
    else vg_load<STRIDE>(load(m), f);
}

// The sums of the voxel whose first sorted entry is `head`: entries j = head, head + 1, ... while j < n_valid and keys[j] is
// keys[head], in entry order.  member(j) is the point of entry j (an int >= 0), load the loader of its fields (vg_fetch).
// Members are fetched 8 at a time so that their loads overlap; the sums stay sequential.
template <int STRIDE, typename K, typename Member, typename Load>
VGB_HD VgAcc<STRIDE> vg_walk(const K* keys, int head, int n_valid, Member member, Load load) {
    VgAcc<STRIDE> acc;
    const K key = keys[head];
    VGB_PRAGMA(unroll 1)
    for (int k0 = head;; k0 += 8) {
        int m[8];
        VGB_PRAGMA(unroll)
        for (int u = 0; u < 8; ++u) m[u] = (k0 + u < n_valid && keys[k0 + u] == key) ? member(k0 + u) : -1;
        float f[8][kVgFields<STRIDE>];
        VGB_PRAGMA(unroll)
        for (int u = 0; u < 8; ++u)
            if (m[u] >= 0) vg_fetch<STRIDE>(load, m[u], f[u]);
        VGB_PRAGMA(unroll)
        for (int u = 0; u < 8; ++u)
            if (m[u] >= 0) acc.add(f[u]);
        if (m[7] < 0) return acc;
    }
}

// ((x·x + y·y) + z·z), never contracted
VGB_HD float vg_sqnorm(float x, float y, float z) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
#else
    return (x * x + y * y) + z * z;
#endif
}

struct VgXyz { float x, y, z; };

// Writes the output point of a voxel from its sums s and member count n, as pcl::CentroidPoint::get does: xyz, intensity and
// curvature divided by the count, the normal normalised (not divided) when its squared norm is > 0, w = 1, padding 0.
// Returns the centroid's xyz.
template <int STRIDE>
VGB_HD VgXyz vg_write(const float* s, int n, unsigned char* dst) {
    const float fc = (float)n;
    const VgXyz c{s[0] / fc, s[1] / fc, s[2] / fc};
    vg_st4(dst, c.x, c.y, c.z, 1.0f);
    if constexpr (STRIDE == 48) {
        float nx = s[3], ny = s[4], nz = s[5];
        const float n2 = vg_sqnorm(nx, ny, nz);
        if (n2 > 0.0f) { const float nn = sqrtf(n2); nx = nx / nn; ny = ny / nn; nz = nz / nn; }
        vg_st4(dst + 16, nx, ny, nz, 0.0f);
        vg_st4(dst + 32, s[6] / fc, s[7] / fc, 0.0f, 0.0f);
    } else {
        vg_st4(dst + 16, s[3] / fc, 0.0f, 0.0f, 0.0f);
    }
    return c;
}

#ifdef __CUDACC__
// flags[i] = 1 at the first entry of every voxel of a sorted key array; 0 at entries past the valid count (*d_valid, or n
// when d_valid is null) and at flags[n] (the sentinel of the exclusive scan that numbers the voxels)
template <typename K>
__device__ __forceinline__ void vg_heads_at(const K* __restrict__ keys, int n, const int* __restrict__ d_valid, int* __restrict__ flags,
                                            const int i) {
    if (i > n) return;
    flags[i] = i < n && vg_is_head(keys, i, d_valid ? *d_valid : n);
}
template <typename K>
__global__ void k_vg_heads(const K* __restrict__ keys, int n, const int* __restrict__ d_valid, int* __restrict__ flags) {
    vg_heads_at(keys, n, d_valid, flags, blockIdx.x * blockDim.x + threadIdx.x);
}
#endif

}  // namespace lili
