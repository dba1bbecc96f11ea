// TEST INFRASTRUCTURE: host build of liliom_b200/csrc/vg_box.h (the ordered-int box and PCL's VoxelGrid parameters), so that
// the CPU test tier checks the SAME SOURCE the VoxelGrid, incremental-map, ROT and cell-grid kernels use.
#include "../liliom_b200/csrc/vg_box.h"

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
