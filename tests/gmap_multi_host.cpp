// TEST INFRASTRUCTURE: host build of liliom_b200/csrc/kf_table.h's two row types, composed the way liliom_global_map and
// liliom_global_map_multi compose them on the device (box of the transformed rows -> vg_params -> voxel keys -> stable sort ->
// heads -> walk through KfRowLoader<STRIDE, Row> -> writer; PCL's declined case gathers): KfRow rows over one arena, KfRowM rows
// that each name an arena of their own.  The CPU test tier checks that both give the same bytes for the same clouds.
// Compiled with -ffp-contract=off.
#include "../liliom_b200/csrc/kf_table.h"
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <vector>

using namespace lili;

static bool gmm_finite(const VgXyz& p) { return std::isfinite(p.x) && std::isfinite(p.y) && std::isfinite(p.z); }

template <int STRIDE, class Row>
static long long gmm_run(const unsigned char* arena, const std::vector<Row>& tab, long long N, float leaf, unsigned char* out, int* declined) {
    const int rows = (int)tab.size();
    int box[kBoxInts];
    for (int k = 0; k < kBoxInts; ++k) box[k] = vg_box_empty(k);
    for (const Row& r : tab)                             // k_kf_box
        for (int i = 0; i < r.n; ++i) {
            const VgXyz p = kf_row_xyz(r, kf_row_src(r, arena, STRIDE, r.src_off + i));
            if (gmm_finite(p)) vg_box_add(box, p.x, p.y, p.z);
        }
    const VgParams p = vg_params(box, leaf);
    *declined = p.overflow;
    if (p.overflow) {                                    // k_kf_gather
        for (const Row& r : tab)
            for (int i = 0; i < r.n; ++i)
                kf_row_point(r, kf_row_src(r, arena, STRIDE, r.src_off + i), STRIDE, out + (size_t)(r.dst_off + i) * STRIDE);
        return N;
    }
    std::vector<uint32_t> keys(N);
    std::vector<int> vals(N);
    for (const Row& r : tab)                             // k_kf_keys
        for (int i = 0; i < r.n; ++i) {
            const VgXyz x = kf_row_xyz(r, kf_row_src(r, arena, STRIDE, r.src_off + i));
            keys[r.dst_off + i] = gmm_finite(x) ? vg_rel_index(p, x.x, x.y, x.z) : 0xffffffffu;
            vals[r.dst_off + i] = (int)(r.dst_off + i);
        }
    std::vector<int> ord(N);                             // the stable radix sort
    std::iota(ord.begin(), ord.end(), 0);
    std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return keys[a] < keys[b]; });
    std::vector<uint32_t> k2(N);
    std::vector<int> v2(N);
    for (long long i = 0; i < N; ++i) { k2[i] = keys[ord[i]]; v2[i] = vals[ord[i]]; }
    const KfRowLoader<STRIDE, Row> load{arena, tab.data(), rows};
    int o = 0;                                           // k_vg_heads, the scan, k_kf_centroid
    for (int i = 0; i < p.n_finite; ++i) {
        if (!vg_is_head(k2.data(), i, p.n_finite)) continue;
        const VgAcc<STRIDE> a = vg_walk<STRIDE>(k2.data(), i, p.n_finite, [&](int j) { return v2[j]; }, load);
        vg_write<STRIDE>(a.s, a.n, out + (size_t)o * STRIDE);
        ++o;
    }
    return o;
}

// The table of k entries in list order (empty clouds skipped): entry i = n[i] points from src_off[i] of arenas[i] (KfRowM) or
// of arenas[0] (KfRow), placed by poses7[7i..] after pre7s[7i..] (pre7s optional)
template <class Row>
static long long gmm_table(const void* const* arenas, const long long* src_off, const int* n, int k, const double* poses7,
                           const double* pre7s, std::vector<Row>& tab) {
    long long N = 0;
    for (int i = 0; i < k; ++i) {
        if (n[i]) {
            Row r{};
            r.src_off = src_off[i]; r.dst_off = N; r.n = n[i];
            const double* q = poses7 + 7 * (size_t)i;
            r.q = Q4{q[0], q[1], q[2], q[3]}; r.t = D3{q[4], q[5], q[6]};
            if (pre7s) {
                const double* e = pre7s + 7 * (size_t)i;
                r.pre = 1; r.pq = Q4{e[0], e[1], e[2], e[3]}; r.pt = D3{e[4], e[5], e[6]};
            }
            if constexpr (std::is_same<Row, KfRowM>::value) r.base = (const unsigned char*)arenas[i];
            tab.push_back(r);
        }
        N += n[i];
    }
    return N;
}

template <class Row>
static long long gmm_map(const void* const* arenas, int stride, const long long* src_off, const int* n, int k, const double* poses7,
                         const double* pre7s, float leaf, void* out, int* declined) {
    std::vector<Row> tab;
    const long long N = gmm_table(arenas, src_off, n, k, poses7, pre7s, tab);
    *declined = 0;
    if (N == 0) return 0;
    const unsigned char* arena = std::is_same<Row, KfRow>::value ? (const unsigned char*)arenas[0] : nullptr;    // KfRowM: never read
    if (stride == 48) return gmm_run<48>(arena, tab, N, leaf, (unsigned char*)out, declined);
    if (stride == 32) return gmm_run<32>(arena, tab, N, leaf, (unsigned char*)out, declined);
    return -1;
}

// one store: every cloud in the arena arenas[0]
extern "C" long long gmm_single(const void* const* arenas, int stride, const long long* src_off, const int* n, int k, const double* poses7,
                                const double* pre7s, float leaf, void* out, int* declined) {
    return gmm_map<KfRow>(arenas, stride, src_off, n, k, poses7, pre7s, leaf, out, declined);
}

// several stores: entry i's cloud in the arena arenas[i]
extern "C" long long gmm_multi(const void* const* arenas, int stride, const long long* src_off, const int* n, int k, const double* poses7,
                               const double* pre7s, float leaf, void* out, int* declined) {
    return gmm_map<KfRowM>(arenas, stride, src_off, n, k, poses7, pre7s, leaf, out, declined);
}
