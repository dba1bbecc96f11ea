// Launch plan of one scan-to-map call (s2m_run, grid_knn.cu): work shape, grid, persistent or per-pass launches, dynamic shared
// memory.  Host-only and free of CUDA types, so that the CPU tests compile it as it is (tests/s2m_plan_host.cpp).
#pragma once
#include <algorithm>
#include <cstddef>
#include <vector>
#include "../../include/liliom.h"
#include "batch.h"

namespace lili {

constexpr int kBlock = 256;
constexpr int kWarps = kBlock / 32;
constexpr int kRunCap = 8;                    // runs per thread of the one-thread-per-query search (thread_knn5, knn_core.cuh)
constexpr size_t kStageTileBytes = 3616;      // sizeof(StageTile), knn_core.cuh (checked there)

struct S2mPlanIn {
    int n, n_last;                  // query upper bound (the exact count unless dev_count); count of the previous scan (0: none)
    bool dev_count;                 // the exact count is only known on the device
    int sm_count, mode, iters;      // mode: LILIOM_MODE_GN / LILIOM_MODE_CERES
    bool want_corr;
    int nranks; bool peer;          // peer: fused exchange attached (liliom_comm_peer_attach)
    int force_lanes, force_rounds;  // LILIOM_KNN_LANES / LILIOM_KNN_ROUNDS (0: none)
    bool knn_tma;                   // LILIOM_KNN_TMA
};
struct S2mPlan {
    int n_est, lanes, rounds, per_task, grid;   // predicted query count, work shape, blocks
    bool persistent, tma;           // all iterations in one launch of k_gn_persistent; its 16-lane search with bulk-copy staging
    size_t dyn_smem;                // dynamic shared memory of the launch
};

// Work decomposition.  LANES lanes cooperate on one query; a warp finishes (32/LANES)*rounds queries per task before the fp64
// phase.  Large query sets: one thread per query (every issue slot ranks 32 candidates, neighbouring threads share cells in L1).
// Small sets (a down-sampled 24k-point sweep leaves 1-3k queries) are latency bound: split each query's 9 runs over 4 or 8
// lanes so that the whole GPU is busy and the per-warp critical path is short.
inline S2mPlan s2m_plan(const S2mPlanIn& in) {
    auto cdiv = [](long long a, long long b) { return (int)((a + b - 1) / b); };
    S2mPlan p{};
    // device-side count: predicted from the previous scan.  The first such call has none and is sized from the upper bound
    // (per-pass launches); the next ones are sized from the scan before, with a margin for a larger one.
    p.n_est = in.dev_count ? (in.n_last > 0 ? std::min(in.n_last, in.n) : in.n) : in.n;
    const int n_size = in.dev_count ? std::max(p.n_est + p.n_est / 4, 1) : in.n;
    const long long w8 = (long long)in.sm_count * 8;      // warps for ~8 per SM
    // 8..32 warps' worth of queries per SM: two lanes per query (a sweep of the lane count at 16k queries, tools/knn_sweep.py,
    // put 2 lanes ahead of 1, 4 and 8); tiny scans: one run per lane (9 of 16 lanes)
    p.lanes = p.n_est >= w8 * 32 ? 1 : p.n_est >= w8 * 8 ? 2 : (long long)p.n_est * 16 / 32 <= w8 * 2 ? 16 : 8;
    p.rounds = 1;
    if (in.force_lanes) { p.lanes = in.force_lanes; p.rounds = in.force_rounds > 0 ? in.force_rounds : 1; }
    if ((32 / p.lanes) * p.rounds > 32) p.rounds = p.lanes;   // at most 32 queries per warp task
    p.per_task = (32 / p.lanes) * p.rounds;
    p.grid = std::min(std::max(cdiv(cdiv(n_size, p.per_task), kWarps), 1), in.sm_count * 2);
    const bool gn = in.mode == LILIOM_MODE_GN;
    // A 16-lane scan that needs more than one block per SM (1.9k-3.8k queries, e.g. a down-sampled HDL-64E sweep) would
    // leave the single-launch path.  Eight lanes per query (four queries per warp, one round) keep it there, which on the
    // configs[2] workload (3.1k queries) is faster than two rounds of 16 lanes or per-iteration launches.
    if (p.lanes == 16 && p.rounds == 1 && !in.force_lanes && p.grid > in.sm_count && gn && !in.want_corr) {
        const int grid8 = std::max(cdiv(cdiv(n_size, 4), kWarps), 1);
        if (grid8 <= in.sm_count) { p.lanes = 8; p.per_task = 4; p.grid = grid8; }
    }
    p.persistent = gn && (in.nranks == 1 || in.peer) && in.iters > 0 && !in.want_corr && p.grid <= in.sm_count;
    p.tma = p.persistent && p.lanes == 16 && in.knn_tma;
    // one thread per query: per-thread run lists (int4) in dynamic shared memory (thread_knn5); static + dynamic exceed 48 KB
    p.dyn_smem = p.tma ? (size_t)kWarps * 2 * kStageTileBytes : p.lanes == 1 ? (size_t)kRunCap * kBlock * 16 : 0;
    return p;
}

// Instantiation of the persistent GN kernel a plan launches: 0..4 = 1, 2, 4, 8, 16 lanes; 5 = 16 lanes with bulk-copy staging.
constexpr int kGnKinds = 6;
inline int s2m_kind(const S2mPlan& p) {
    return p.tma ? 5 : p.lanes == 1 ? 0 : p.lanes == 2 ? 1 : p.lanes == 4 ? 2 : p.lanes == 8 ? 3 : 4;
}

// The launches of a batched scan-to-map step (s2m_batch, grid_knn.cu).  Each session keeps the plan its solo call would make:
// its grid and instantiation are packed by batch_pack against the occupancy occ[kind] of k_gn_batch<kind>; a session whose plan
// is not persistent (or whose kernel cannot be resident at all) takes s2m_run's own path.
inline BatchPack s2m_batch_pack(const std::vector<S2mPlan>& plans, const int occ[kGnKinds], int sm_count, int max_per_launch = kBatchMax) {
    std::vector<BatchItem> items;
    for (const S2mPlan& p : plans) items.push_back(BatchItem{p.grid, s2m_kind(p), p.persistent});
    return batch_pack(items, occ, sm_count, max_per_launch);
}

// A GN-mode batched step whose sessions run different iteration counts (liliom_scan_to_map_resident_batch_ex): k_gn_batch
// shares one count per launch, so the sessions are grouped by count (groups in the order of their first session) and each
// group is packed by s2m_batch_pack.  The pack's indices are into `plans`, as for one s2m_batch_pack call over all of them.
struct S2mGnGroup {
    int iters;
    BatchPack pack;
};
inline std::vector<S2mGnGroup> s2m_gn_groups(const std::vector<S2mPlan>& plans, const std::vector<int>& iters, const int occ[kGnKinds],
                                             int sm_count, int max_per_launch = kBatchMax) {
    std::vector<S2mGnGroup> out;
    std::vector<char> done(plans.size(), 0);
    for (size_t i = 0; i < plans.size(); ++i) {
        if (done[i]) continue;
        std::vector<int> members;
        std::vector<S2mPlan> sub;
        for (size_t j = i; j < plans.size(); ++j)
            if (!done[j] && iters[j] == iters[i]) { done[j] = 1; members.push_back((int)j); sub.push_back(plans[j]); }
        S2mGnGroup g{iters[i], s2m_batch_pack(sub, occ, sm_count, max_per_launch)};
        for (BatchLaunch& l : g.pack.launches)
            for (int& s : l.sessions) s = members[s];
        for (int& s : g.pack.solo) s = members[s];
        out.push_back(std::move(g));
    }
    return out;
}

// The launches of a Ceres-mode batched step (s2m_batch, grid_knn.cu).  Outer iteration `it` (a pass) serves the sessions with
// iters[j] > it: first the per-pass kNN launches (k_knn_plane_batch), each of one lane count and at most max_per_launch
// sessions, lane counts in the order of their first session; then the LM launches (k_lm_solve_batch) of the same sessions, at
// most max_per_launch each.  Sessions keep call order inside every launch.  Per-pass launches are not cooperative, so any grid
// fits; each session keeps the plan (lanes, grid) of its solo call.
struct S2mKnnLaunch {
    int lanes;
    std::vector<int> sessions;      // indices into the plans, in call order; blocks follow in this order
};
struct S2mPass {
    std::vector<S2mKnnLaunch> knn;
    std::vector<std::vector<int>> lm;
};
inline std::vector<S2mPass> s2m_pass_pack(const std::vector<S2mPlan>& plans, const std::vector<int>& iters, int max_per_launch = kBatchMax) {
    int passes = 0;
    for (int n : iters) passes = std::max(passes, n);
    std::vector<S2mPass> out(passes);
    for (int it = 0; it < passes; ++it) {
        std::vector<int> live, lanes;
        for (int j = 0; j < (int)plans.size(); ++j) {
            if (iters[j] <= it) continue;
            live.push_back(j);
            if (std::find(lanes.begin(), lanes.end(), plans[j].lanes) == lanes.end()) lanes.push_back(plans[j].lanes);
        }
        for (int ln : lanes)
            for (int j : live) {
                if (plans[j].lanes != ln) continue;
                std::vector<S2mKnnLaunch>& knn = out[it].knn;
                if (knn.empty() || knn.back().lanes != ln || (int)knn.back().sessions.size() >= max_per_launch) knn.push_back(S2mKnnLaunch{ln, {}});
                knn.back().sessions.push_back(j);
            }
        for (size_t k = 0; k < live.size(); k += (size_t)max_per_launch)
            out[it].lm.emplace_back(live.begin() + k, live.begin() + std::min(live.size(), k + (size_t)max_per_launch));
    }
    return out;
}

}  // namespace lili
