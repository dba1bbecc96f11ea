// TEST INFRASTRUCTURE: host build of liliom_b200/csrc/vg_box.h (the ordered-int box, PCL's VoxelGrid parameters and voxel index,
// the centroid walk and writer), so that the CPU test tier checks the SAME SOURCE the VoxelGrid, incremental-map, ROT and
// cell-grid kernels use.
#include "../liliom_b200/csrc/vg_box.h"
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <vector>

extern "C" void vb_f2ord(const float* in, int* out, int n) { for (int i = 0; i < n; ++i) out[i] = lili::vg_f2ord(in[i]); }
extern "C" void vb_ord2f(const int* in, float* out, int n) { for (int i = 0; i < n; ++i) out[i] = lili::vg_ord2f(in[i]); }

// box of the finite points among xyz[n][3]: the first half added to one box, the rest to another, then merged
extern "C" void vb_box_of(const float* xyz, int n, int* box) {
    int other[lili::kBoxInts];
    for (int k = 0; k < lili::kBoxInts; ++k) box[k] = other[k] = lili::vg_box_empty(k);
    for (int i = 0; i < n; ++i) {
        const float* p = xyz + 3 * i;
        if (std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2])) lili::vg_box_add(i < n / 2 ? box : other, p[0], p[1], p[2]);
    }
    lili::vg_box_merge(box, other);
}

// out: min_b[3], div_b[3], mul[3], overflow, n_finite, bail; *inv_leaf
extern "C" void vb_params(const int* box, float leaf, int* out, float* inv_leaf) {
    const lili::VgParams p = lili::vg_params(box, leaf);
    for (int k = 0; k < 3; ++k) { out[k] = p.min_b[k]; out[3 + k] = p.div_b[k]; out[6 + k] = p.mul[k]; }
    out[9] = p.overflow; out[10] = p.n_finite; out[11] = p.bail;
    *inv_leaf = p.inv_leaf;
}

extern "C" int vb_key_bits(const int* box, float leaf) { return lili::vg_key_bits(box, leaf); }

extern "C" int vb_abs_key(float x, float y, float z, float inv_leaf, unsigned long long* key) {
    return lili::vg_abs_key(x, y, z, inv_leaf, key) ? 1 : 0;
}

// ---- the centroid arithmetic, composed the way the device does it

// heads -> output ranks -> walk -> writer over a sorted entry array (k_vg_heads, the exclusive scan, the centroid kernels);
// xyz (optional) receives the centroids' xyz that the writer returns
template <int STRIDE, typename K>
static int vb_emit(const unsigned char* pts, const std::vector<K>& keys, const std::vector<int>& vals, int n_valid, unsigned char* out,
                   float* xyz) {
    int o = 0;
    for (int i = 0; i < (int)keys.size(); ++i) {
        if (!lili::vg_is_head(keys.data(), i, n_valid)) continue;
        const lili::VgAcc<STRIDE> a = lili::vg_walk<STRIDE>(keys.data(), i, n_valid, [&](int j) { return vals[j]; },
                                                            [&](int m) { return pts + (size_t)m * STRIDE; });
        const lili::VgXyz c = lili::vg_write<STRIDE>(a.s, a.n, out + (size_t)o * STRIDE);
        if (xyz) { xyz[3 * o] = c.x; xyz[3 * o + 1] = c.y; xyz[3 * o + 2] = c.z; }
        ++o;
    }
    return o;
}

// the entries sorted by key, equal keys in entry order (the device's stable radix sort)
template <typename K>
static void vb_stable_sort(std::vector<K>& keys, std::vector<int>& vals) {
    std::vector<int> ord(keys.size());
    std::iota(ord.begin(), ord.end(), 0);
    std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return keys[a] < keys[b]; });
    std::vector<K> k2(keys.size());
    std::vector<int> v2(keys.size());
    for (size_t i = 0; i < ord.size(); ++i) { k2[i] = keys[ord[i]]; v2[i] = vals[ord[i]]; }
    keys.swap(k2); vals.swap(v2);
}

static bool vb_finite(const lili::VgF4& v) { return std::isfinite(v.x) && std::isfinite(v.y) && std::isfinite(v.z); }

// The VoxelGrid sort chain (voxelgrid_dev): box -> vg_params -> vg_rel_index keys (all-ones for non-finite points) -> stable
// sort -> heads over the finite entries -> walk -> writer.  PCL's overflow case copies the input.  Returns the output count.
template <int STRIDE>
static int vb_sort_chain(const unsigned char* pts, int n, float leaf, unsigned char* out, float* xyz) {
    int box[lili::kBoxInts];
    for (int k = 0; k < lili::kBoxInts; ++k) box[k] = lili::vg_box_empty(k);
    for (int i = 0; i < n; ++i) {
        const lili::VgF4 v = lili::vg_ld4(pts + (size_t)i * STRIDE);
        if (vb_finite(v)) lili::vg_box_add(box, v.x, v.y, v.z);
    }
    const lili::VgParams p = lili::vg_params(box, leaf);
    if (p.overflow) { memcpy(out, pts, (size_t)n * STRIDE); return n; }
    std::vector<uint32_t> keys(n);
    std::vector<int> vals(n);
    for (int i = 0; i < n; ++i) {
        const lili::VgF4 v = lili::vg_ld4(pts + (size_t)i * STRIDE);
        keys[i] = vb_finite(v) ? lili::vg_rel_index(p, v.x, v.y, v.z) : 0xffffffffu;
        vals[i] = i;
    }
    vb_stable_sort(keys, vals);
    return vb_emit<STRIDE>(pts, keys, vals, p.n_finite, out, xyz);
}

extern "C" int vb_voxelgrid(const void* pts, int n, int stride, float leaf, void* out, float* xyz) {
    if (stride == 48) return vb_sort_chain<48>((const unsigned char*)pts, n, leaf, (unsigned char*)out, xyz);
    if (stride == 32) return vb_sort_chain<32>((const unsigned char*)pts, n, leaf, (unsigned char*)out, xyz);
    return -1;
}

// The ROT extractor's per-ring VoxelGrid of finite 32-byte points in one batch (k_rot_lf_*): a box and parameters per ring,
// 64-bit keys ring << 32 | voxel index (the entry's position in PCL's overflow case), stable sort, heads, walk, writer.
extern "C" int vb_voxelgrid_rings(const void* pts_, const int* ring, int n, float leaf, void* out, float* xyz) {
    const unsigned char* pts = (const unsigned char*)pts_;
    const int nr = n > 0 ? *std::max_element(ring, ring + n) + 1 : 0;
    std::vector<int> boxes((size_t)nr * lili::kBoxInts);
    for (size_t k = 0; k < boxes.size(); ++k) boxes[k] = lili::vg_box_empty((int)(k % lili::kBoxInts));
    for (int t = 0; t < n; ++t) {
        const lili::VgF4 v = lili::vg_ld4(pts + (size_t)t * 32);
        lili::vg_box_add(&boxes[(size_t)ring[t] * lili::kBoxInts], v.x, v.y, v.z);
    }
    std::vector<lili::VgParams> prm(nr);
    for (int r = 0; r < nr; ++r) prm[r] = lili::vg_params(&boxes[(size_t)r * lili::kBoxInts], leaf);
    std::vector<unsigned long long> keys(n);
    std::vector<int> vals(n);
    for (int t = 0; t < n; ++t) {
        const lili::VgF4 v = lili::vg_ld4(pts + (size_t)t * 32);
        const lili::VgParams& p = prm[ring[t]];
        const unsigned idx = p.overflow ? (unsigned)t : lili::vg_rel_index(p, v.x, v.y, v.z);
        keys[t] = ((unsigned long long)ring[t] << 32) | idx;
        vals[t] = t;
    }
    vb_stable_sort(keys, vals);
    return vb_emit<32>(pts, keys, vals, n, (unsigned char*)out, xyz);
}
