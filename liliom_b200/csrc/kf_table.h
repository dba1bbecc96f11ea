// A table of keyframe clouds transformed on load, shared by host and device (keyframes.cu; tests/gmap_host.cpp compiles this
// same file for the CPU test tier).  A row names n stored points and the pose(s) that place them at dst_off of the transformed
// concatenation, so that a kernel reads the store where it lies instead of a concatenation written first:
//   * k_kf_gather writes the concatenation (the local map, the loop-closure clouds, PCL's declined global map);
//   * the global map's VoxelGrid (liliom_global_map) measures its box and its voxel keys from kf_row_xyz and sums its centroids
//     through KfRowLoader, which finds a member's row by binary search over dst_off.
// The three transforms of a point (box, key, centroid) are the same code, so they give the same bits.
#pragma once
#include "pcl_xform.h"

namespace lili {

// n points of the arena from src_off (in points) -> dst_off of the concatenation: transformed by (pq, pt) when `pre` is set (the
// intermediate point stored in fp32, as the pcl::PointCloud in between holds it), then by (q, t).
struct KfRow { long long src_off, dst_off; Q4 q; D3 t; Q4 pq; D3 pt; int n, pre; };

// the transformed xyz of a stored point of row r
VGB_HD VgXyz kf_row_xyz(const KfRow& r, const unsigned char* src) {
    const VgF4 a = vg_ld4(src);
    VgXyz p{a.x, a.y, a.z};
    if (r.pre) p = pcl_transform_xyz(r.pq, r.pt, p.x, p.y, p.z);
    return pcl_transform_xyz(r.q, r.t, p.x, p.y, p.z);
}

// the whole transformed point (stride bytes)
VGB_HD void kf_row_point(const KfRow& r, const unsigned char* src, int stride, unsigned char* out) {
    if (r.pre) {
        alignas(16) unsigned char mid[48];
        pcl_transform_point(src, stride, r.pq, r.pt, mid);
        pcl_transform_point(mid, stride, r.q, r.t, out);
    } else {
        pcl_transform_point(src, stride, r.q, r.t, out);
    }
}

// the row holding concatenation index i: the last row with dst_off <= i (rows in ascending dst_off, none empty)
VGB_HD int kf_row_of(const KfRow* tab, int rows, long long i) {
    int lo = 0, hi = rows - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (tab[mid].dst_off <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// vg_walk's loader over the table: the fields of concatenation index m, transformed on load
template <int STRIDE>
struct KfRowLoader {
    const unsigned char* arena;
    const KfRow* tab;
    int rows;
    VGB_HD void operator()(int m, float* f) const {
        const KfRow& r = tab[kf_row_of(tab, rows, m)];
        alignas(16) unsigned char p[STRIDE];
        kf_row_point(r, arena + (size_t)(r.src_off + (m - r.dst_off)) * STRIDE, STRIDE, p);
        vg_load<STRIDE>(p, f);
    }
};

}  // namespace lili
