// A table of keyframe clouds transformed on load, shared by host and device (keyframes.cu; tests/gmap_host.cpp compiles this
// same file for the CPU test tier).  A row names n stored points and the pose(s) that place them at dst_off of the transformed
// concatenation, so that a kernel reads the store where it lies instead of a concatenation written first:
//   * k_kf_gather writes the concatenation (the local map, the loop-closure clouds, PCL's declined global map);
//   * the global map's VoxelGrid (liliom_global_map) measures its box and its voxel keys from kf_row_xyz and sums its centroids
//     through KfRowLoader, which finds a member's row by binary search over dst_off.
// The three transforms of a point (box, key, centroid) are the same code, so they give the same bits.
// Two row types: KfRow reads the one arena its kernel is given (one context's store), KfRowM carries its own arena (the calls
// over keyframes of several stores, liliom_*_multi).  kf_row_src gives either's stored point.  The host builds the local map's
// table here (kf_bmap_rows), so that tests/bmap_multi_host.cpp compiles the same builder.
#pragma once
#include "pcl_xform.h"
#include <algorithm>
#include <type_traits>
#include <vector>

namespace lili {

// n points of the arena from src_off (in points) -> dst_off of the concatenation: transformed by (pq, pt) when `pre` is set (the
// intermediate point stored in fp32, as the pcl::PointCloud in between holds it), then by (q, t).
struct KfRow { long long src_off, dst_off; Q4 q; D3 t; Q4 pq; D3 pt; int n, pre; };
// ... whose points lie in `base` (its store's arena) instead of the kernel's arena
struct KfRowM : KfRow { const unsigned char* base; };

// a row of either type: n points from src -> dst, transformed by pre7 (optional) and then by pose7; a KfRowM's points lie in
// `arena` (KfRow: not read, its kernel is given the arena)
template <class Row>
inline Row kf_row_in(const void* arena, long long src, long long dst, int n, const double* pose7, const double* pre7 = nullptr) {
    Row e{};
    e.src_off = src; e.dst_off = dst; e.n = n;
    e.q = Q4{pose7[0], pose7[1], pose7[2], pose7[3]};
    e.t = D3{pose7[4], pose7[5], pose7[6]};
    if (pre7) {
        e.pre = 1;
        e.pq = Q4{pre7[0], pre7[1], pre7[2], pre7[3]};
        e.pt = D3{pre7[4], pre7[5], pre7[6]};
    }
    if constexpr (std::is_same<Row, KfRowM>::value) e.base = (const unsigned char*)arena;
    return e;
}

// A listed keyframe's stored edge and surf clouds: the arena they lie in, where (in points) and how many
struct KfClouds { const void* arena; long long edge_off, surf_off; int n_edge, n_surf; };

// The backend local map's table (buildLocalMapWithLandMark :1479-1483): every entry's edge cloud at destinations from 0 and its
// surf cloud at destinations from E (the listed edge points), both in list order, placed by poses7[7i..]; an empty cloud has no
// row.  clouds(i): entry i's KfClouds.  n[0] = E, n[1] = S (the listed surf points); *largest = the largest listed cloud.
template <class Row, class Clouds>
inline void kf_bmap_rows(Clouds clouds, const double* poses7, int k, std::vector<Row>& tab, long long n[2], long long* largest) {
    long long E = 0, S = 0;
    *largest = 0;
    for (int i = 0; i < k; ++i) {
        const KfClouds f = clouds(i);
        E += f.n_edge; S += f.n_surf;
        *largest = std::max(*largest, (long long)std::max(f.n_edge, f.n_surf));
    }
    tab.clear();
    tab.reserve(2 * (size_t)k);
    long long de = 0, ds = E;
    for (int i = 0; i < k; ++i) {
        const KfClouds f = clouds(i);
        if (f.n_edge) tab.push_back(kf_row_in<Row>(f.arena, f.edge_off, de, f.n_edge, poses7 + 7 * (size_t)i));
        if (f.n_surf) tab.push_back(kf_row_in<Row>(f.arena, f.surf_off, ds, f.n_surf, poses7 + 7 * (size_t)i));
        de += f.n_edge; ds += f.n_surf;
    }
    n[0] = E; n[1] = S;
}

// point j (an index into its arena: r.src_off + the point's index in the row) of the arena row r reads, stride bytes each
VGB_HD const unsigned char* kf_row_src(const KfRow&, const unsigned char* arena, int stride, long long j) { return arena + (size_t)j * stride; }
VGB_HD const unsigned char* kf_row_src(const KfRowM& r, const unsigned char*, int stride, long long j) { return r.base + (size_t)j * stride; }

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
template <class Row>
VGB_HD int kf_row_of(const Row* tab, int rows, long long i) {
    int lo = 0, hi = rows - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (tab[mid].dst_off <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// vg_walk's loader over the table: the fields of concatenation index m, transformed on load (arena: KfRow's, unused by KfRowM)
template <int STRIDE, class Row = KfRow>
struct KfRowLoader {
    const unsigned char* arena;
    const Row* tab;
    int rows;
    VGB_HD void operator()(int m, float* f) const {
        const Row& r = tab[kf_row_of(tab, rows, m)];
        alignas(16) unsigned char p[STRIDE];
        // KfRow's address spelled out: through kf_row_src ptxas allocates the 32-byte kernels' registers differently
        if constexpr (std::is_same<Row, KfRow>::value) kf_row_point(r, arena + (size_t)(r.src_off + (m - r.dst_off)) * STRIDE, STRIDE, p);
        else kf_row_point(r, kf_row_src(r, arena, STRIDE, r.src_off + (m - r.dst_off)), STRIDE, p);
        vg_load<STRIDE>(p, f);
    }
};

}  // namespace lili
