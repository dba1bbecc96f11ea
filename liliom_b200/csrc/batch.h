// Launches that several independent sessions share (the batched calls: scan-to-map in grid_knn.cu, extraction in extract_rot.cu
// and extract_horizon.cu, the map update in map.cu).  A launch serves up to kBatchMax sessions; session s owns blocks
// [off[s], off[s + 1]) of its grid, and the table of the sessions' entries travels as a __grid_constant__ kernel parameter.
// Plain C++ for host and device, so that the CPU tests compile it as it is (tests/batch_host.cpp).
#pragma once
#include <vector>

#ifdef __CUDACC__
#define LILI_BATCH_HD __host__ __device__
#else
#define LILI_BATCH_HD
#endif

namespace lili {

constexpr int kBatchMax = 32;                 // sessions per batched launch

// The session table of a batched launch, for up to N sessions.  A launch that needs launch-wide scalars declares them beside it
// in a derived struct.  Every table must fit the 32 764-byte kernel parameter space: batch_tables (ctx.cuh), which fills them
// all, checks it.  The stage chains launch a one-session launch with N = 1, so that it carries one entry rather than kBatchMax.
template <class Entry, int N = kBatchMax>
struct BatchTab {
    int n;                              // sessions in this launch
    int off[N + 1];                     // session s owns blocks [off[s], off[s + 1])
    Entry s[N];
};

// The session that block b of a shared grid belongs to: the last s with off[s] <= b.  A session without blocks owns none; the last
// session takes what is left.
LILI_BATCH_HD inline int batch_session_of(int n_sessions, const int* off, int b) {
    int s = 0;
    while (s + 1 < n_sessions && b >= off[s + 1]) ++s;
    return s;
}

// blocks of `threads` threads for `items` items, one thread per item (0 items: no block)
LILI_BATCH_HD inline int stage_blocks(int items, int threads) { return (items + threads - 1) / threads; }

// grid of the box pass over n points (k_vg_minmax: a grid-stride loop, capped at eight blocks per SM)
LILI_BATCH_HD inline int box_blocks(int n, int sm_count) {
    const int b = stage_blocks(n, 256);
    return b < sm_count * 8 ? b : sm_count * 8;
}

// Cooperative launches that sessions share.  Session i wants grid blocks of the kernel instantiation `kind`; a session that may
// not share (coop false) or whose grid is not co-resident alone goes to `solo`.  The others are packed first-fit, in call order,
// into launches of one kind whose summed grid is co-resident (occ[kind] blocks per SM times sm_count) and that hold at most
// max_per_launch sessions.
struct BatchItem {
    int grid, kind;
    bool coop;
};
struct BatchLaunch {
    int kind, grid;                 // instantiation, summed grid
    std::vector<int> sessions;      // indices into the items, in call order; blocks follow in this order
};
struct BatchPack {
    std::vector<BatchLaunch> launches;
    std::vector<int> solo;          // sessions that take their solo path
};
inline BatchPack batch_pack(const std::vector<BatchItem>& items, const int* occ, int sm_count, int max_per_launch = kBatchMax) {
    BatchPack out;
    for (int i = 0; i < (int)items.size(); ++i) {
        const BatchItem& it = items[i];
        const long long cap = (long long)occ[it.kind] * sm_count;
        if (!it.coop || it.grid > cap) { out.solo.push_back(i); continue; }
        BatchLaunch* fit = nullptr;
        for (BatchLaunch& l : out.launches)
            if (l.kind == it.kind && (int)l.sessions.size() < max_per_launch && l.grid + it.grid <= cap) { fit = &l; break; }
        if (!fit) { out.launches.push_back(BatchLaunch{it.kind, 0, {}}); fit = &out.launches.back(); }
        fit->grid += it.grid;
        fit->sessions.push_back(i);
    }
    return out;
}

}  // namespace lili
