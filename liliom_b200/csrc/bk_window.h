// Sliding-window bookkeeping of the backend LiDAR rows (L/src/BackendFusion.cpp:919-979, R/src/BackendFusion.cpp:832-861):
// which window keyframe a concatenated query belongs to, and the variant's factor weights.  Plain C++ usable from device code
// (backend_corr.cu) and from the host (tests/bk_window_host.cpp compiles this same file for the CPU test tier).
#pragma once

#ifdef __CUDACC__
#define BKW_HD __host__ __device__ __forceinline__
#else
#define BKW_HD inline
#endif

namespace lili {

constexpr int kWinMax = 16;      // window keyframes per liliom_backend_window_correspond call

// Keyframe of concatenated query qi: the j with start[j] <= qi < start[j + 1], start[0] = 0, start[k] = total (k + 1 entries,
// non-decreasing; an empty keyframe has start[j] == start[j + 1] and owns no query).  -1 when qi is outside [0, start[k]).
BKW_HD int bkw_find(const long long* start, int k, long long qi) {
    if (k <= 0 || qi < 0 || qi >= start[k]) return -1;
    int lo = 0, hi = k;              // invariant: start[lo] <= qi < start[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (start[mid] <= qi) lo = mid; else hi = mid;
    }
    return lo;
}

// LidarEdgeFactor weight s.  Variant 0 (L:1581): the constant travels in the float `intensity` field -> (double)(float)lidar_const.
// Variant 1 (R:843): intensity * 200 / vec_edge_res_cnt[idVec], float * int -> float, float / int -> float.
BKW_HD double bkw_edge_weight(int variant, double lidar_const, int n_edge_corr) {
    const float lc = (float)lidar_const;
    if (variant != 1) return (double)lc;
    const float a = lc * 200.0f;
    return (double)(a / (float)n_edge_corr);
}

// LidarPlaneNormFactor score.  Variant 0 (L:1676): the search's score as it is.  Variant 1 (R:861):
// vec_surf_scores[idVec][i] * 1000 / vec_surf_res_cnt[idVec], in double.
BKW_HD double bkw_surf_score(int variant, double score, int n_surf_corr) {
    if (variant != 1) return score;
    return score * 1000.0 / (double)n_surf_corr;
}

}  // namespace lili
