// TEST INFRASTRUCTURE: host build of the backend local map's table (liliom_b200/csrc/kf_table.h's kf_bmap_rows) for both row
// types, composed the way liliom_bmap_build and liliom_bmap_build_multi compose it on the device: the gather (k_kf_gather's body:
// kf_row_point of every row's points at their destinations) into the edge-then-surf concatenation, then each layer's VoxelGrid
// (box -> vg_params -> keys -> stable sort -> heads -> walk -> writer; PCL's declined case passes the layer through).  KfRow rows
// read one arena (the merged store), KfRowM rows each the arena of their entry's store.  Compiled with -ffp-contract=off.
#include "../liliom_b200/csrc/kf_table.h"
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <numeric>
#include <vector>

using namespace lili;

static bool bm_finite(const VgXyz& p) { return std::isfinite(p.x) && std::isfinite(p.y) && std::isfinite(p.z); }

// The table of k entries (entry i: n_edge[i] edge points from edge_off[i] and n_surf[i] surf points from surf_off[i] of arenas[i]
// for KfRowM, of arenas[0] for KfRow), gathered into out (E + S points).  rows_out: dst_off, n, src_off of every row (3 per row).
// n[0] = E, n[1] = S, *largest as the device's gather grid takes it.  Returns the rows.
template <class Row>
static int bm_gather(const void* const* arenas, int stride, const long long* edge_off, const long long* surf_off, const int* n_edge,
                     const int* n_surf, int k, const double* poses7, unsigned char* out, long long* n, long long* largest, long long* rows_out) {
    constexpr bool multi = std::is_same<Row, KfRowM>::value;
    std::vector<Row> tab;
    kf_bmap_rows([&](int i) { return KfClouds{multi ? arenas[i] : nullptr, edge_off[i], surf_off[i], n_edge[i], n_surf[i]}; }, poses7, k, tab,
                 n, largest);
    const unsigned char* arena = multi ? nullptr : (const unsigned char*)arenas[0];
    for (size_t y = 0; y < tab.size(); ++y) {
        const Row& r = tab[y];
        for (int i = 0; i < r.n; ++i)
            kf_row_point(r, kf_row_src(r, arena, stride, r.src_off + i), stride, out + (size_t)(r.dst_off + i) * stride);
        rows_out[3 * y] = r.dst_off; rows_out[3 * y + 1] = r.n; rows_out[3 * y + 2] = r.src_off;
    }
    return (int)tab.size();
}

// one store: every cloud in arenas[0]
extern "C" int bm_gather_single(const void* const* arenas, int stride, const long long* edge_off, const long long* surf_off, const int* n_edge,
                                const int* n_surf, int k, const double* poses7, unsigned char* out, long long* n, long long* largest,
                                long long* rows_out) {
    return bm_gather<KfRow>(arenas, stride, edge_off, surf_off, n_edge, n_surf, k, poses7, out, n, largest, rows_out);
}

// several stores: entry i's clouds in arenas[i]
extern "C" int bm_gather_multi(const void* const* arenas, int stride, const long long* edge_off, const long long* surf_off, const int* n_edge,
                               const int* n_surf, int k, const double* poses7, unsigned char* out, long long* n, long long* largest,
                               long long* rows_out) {
    return bm_gather<KfRowM>(arenas, stride, edge_off, surf_off, n_edge, n_surf, k, poses7, out, n, largest, rows_out);
}

// A layer's VoxelGrid (voxelgrid_dev's chain on the concatenation): N points at pts -> out; returns the points written
template <int STRIDE>
static long long bm_vg(const unsigned char* pts, long long N, float leaf, unsigned char* out) {
    if (N == 0) return 0;
    auto xyz = [&](long long i) { const VgF4 a = vg_ld4(pts + (size_t)i * STRIDE); return VgXyz{a.x, a.y, a.z}; };
    int box[kBoxInts];
    for (int k = 0; k < kBoxInts; ++k) box[k] = vg_box_empty(k);
    for (long long i = 0; i < N; ++i) {
        const VgXyz p = xyz(i);
        if (bm_finite(p)) vg_box_add(box, p.x, p.y, p.z);
    }
    const VgParams p = vg_params(box, leaf);
    if (p.overflow) {                                    // PCL declines the filter and publishes its input
        memcpy(out, pts, (size_t)N * STRIDE);
        return N;
    }
    std::vector<uint32_t> keys(N);
    for (long long i = 0; i < N; ++i) {
        const VgXyz x = xyz(i);
        keys[i] = bm_finite(x) ? vg_rel_index(p, x.x, x.y, x.z) : 0xffffffffu;
    }
    std::vector<int> ord(N);                             // the stable radix sort
    std::iota(ord.begin(), ord.end(), 0);
    std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return keys[a] < keys[b]; });
    std::vector<uint32_t> k2(N);
    for (long long i = 0; i < N; ++i) k2[i] = keys[ord[i]];
    auto load = [&](int m, float* f) { vg_load<STRIDE>(pts + (size_t)m * STRIDE, f); };
    int o = 0;
    for (int i = 0; i < p.n_finite; ++i) {
        if (!vg_is_head(k2.data(), i, p.n_finite)) continue;
        const VgAcc<STRIDE> a = vg_walk<STRIDE>(k2.data(), i, p.n_finite, [&](int j) { return ord[j]; }, load);
        vg_write<STRIDE>(a.s, a.n, out + (size_t)o * STRIDE);
        ++o;
    }
    return o;
}

extern "C" long long bm_voxelgrid(const void* pts, long long N, int stride, float leaf, void* out) {
    if (stride == 48) return bm_vg<48>((const unsigned char*)pts, N, leaf, (unsigned char*)out);
    if (stride == 32) return bm_vg<32>((const unsigned char*)pts, N, leaf, (unsigned char*)out);
    return -1;
}
