// TEST INFRASTRUCTURE: host build of liliom_b200/csrc/kf_table.h (keyframe table rows, the transform on load, the row search and
// vg_walk's transforming loader) with vg_box.h and pcl_xform.h, composed the way liliom_global_map composes them on the device:
// box of the transformed rows -> vg_params -> voxel keys -> stable sort -> heads -> walk through KfRowLoader -> writer; PCL's
// declined case gathers the transformed concatenation.  The CPU test tier checks it against the oracle's
// voxelgrid(concat(transform_cloud(...))).  Compiled with -ffp-contract=off.
#include "../liliom_b200/csrc/kf_table.h"
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <vector>

using namespace lili;

static bool gm_finite(const VgXyz& p) { return std::isfinite(p.x) && std::isfinite(p.y) && std::isfinite(p.z); }

template <int STRIDE>
static long long gm_run(const unsigned char* arena, const std::vector<KfRow>& tab, long long N, float leaf, unsigned char* out, int* declined) {
    const int rows = (int)tab.size();
    int box[kBoxInts];
    for (int k = 0; k < kBoxInts; ++k) box[k] = vg_box_empty(k);
    for (const KfRow& r : tab)
        for (int i = 0; i < r.n; ++i) {
            const VgXyz p = kf_row_xyz(r, arena + (size_t)(r.src_off + i) * STRIDE);
            if (gm_finite(p)) vg_box_add(box, p.x, p.y, p.z);
        }
    const VgParams p = vg_params(box, leaf);
    *declined = p.overflow;
    if (p.overflow) {                                    // k_kf_gather
        for (const KfRow& r : tab)
            for (int i = 0; i < r.n; ++i)
                kf_row_point(r, arena + (size_t)(r.src_off + i) * STRIDE, STRIDE, out + (size_t)(r.dst_off + i) * STRIDE);
        return N;
    }
    std::vector<uint32_t> keys(N);
    std::vector<int> vals(N);
    for (const KfRow& r : tab)                           // k_kf_keys
        for (int i = 0; i < r.n; ++i) {
            const VgXyz x = kf_row_xyz(r, arena + (size_t)(r.src_off + i) * STRIDE);
            keys[r.dst_off + i] = gm_finite(x) ? vg_rel_index(p, x.x, x.y, x.z) : 0xffffffffu;
            vals[r.dst_off + i] = (int)(r.dst_off + i);
        }
    std::vector<int> ord(N);                             // the stable radix sort
    std::iota(ord.begin(), ord.end(), 0);
    std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return keys[a] < keys[b]; });
    std::vector<uint32_t> k2(N);
    std::vector<int> v2(N);
    for (long long i = 0; i < N; ++i) { k2[i] = keys[ord[i]]; v2[i] = vals[ord[i]]; }
    const KfRowLoader<STRIDE> load{arena, tab.data(), rows};
    int o = 0;                                           // k_vg_heads, the scan, k_kf_centroid
    for (int i = 0; i < p.n_finite; ++i) {
        if (!vg_is_head(k2.data(), i, p.n_finite)) continue;
        const VgAcc<STRIDE> a = vg_walk<STRIDE>(k2.data(), i, p.n_finite, [&](int j) { return v2[j]; }, load);
        vg_write<STRIDE>(a.s, a.n, out + (size_t)o * STRIDE);
        ++o;
    }
    return o;
}

// k keyframes of a store: cloud i = n[i] points of `arena` from src_off[i]; the listed order is 0..k-1.  pre7 optional.
// Returns the output count (out holds at least sum(n) points); *declined = PCL's overflow case.
extern "C" long long gm_global_map(const void* arena, int stride, const long long* src_off, const int* n, int k, const double* poses7,
                                   const double* pre7, float leaf, void* out, int* declined) {
    std::vector<KfRow> tab;
    long long N = 0;
    for (int i = 0; i < k; ++i) {                        // liliom_global_map's table: list order, empty clouds skipped
        if (n[i]) {
            KfRow r{};
            r.src_off = src_off[i]; r.dst_off = N; r.n = n[i];
            const double* q = poses7 + 7 * (size_t)i;
            r.q = Q4{q[0], q[1], q[2], q[3]}; r.t = D3{q[4], q[5], q[6]};
            if (pre7) { r.pre = 1; r.pq = Q4{pre7[0], pre7[1], pre7[2], pre7[3]}; r.pt = D3{pre7[4], pre7[5], pre7[6]}; }
            tab.push_back(r);
        }
        N += n[i];
    }
    *declined = 0;
    if (N == 0) return 0;
    if (stride == 48) return gm_run<48>((const unsigned char*)arena, tab, N, leaf, (unsigned char*)out, declined);
    if (stride == 32) return gm_run<32>((const unsigned char*)arena, tab, N, leaf, (unsigned char*)out, declined);
    return -1;
}

// the row each concatenation index falls in (kf_row_of), for rows of the given sizes (empty ones skipped as above)
extern "C" void gm_rows_of(const int* n, int k, const long long* idx, int m, int* row) {
    std::vector<KfRow> tab;
    long long N = 0;
    for (int i = 0; i < k; ++i)
        if (n[i]) { KfRow r{}; r.dst_off = N; r.n = n[i]; tab.push_back(r); N += n[i]; }
    for (int j = 0; j < m; ++j) row[j] = kf_row_of(tab.data(), (int)tab.size(), idx[j]);
}
