// TEST INFRASTRUCTURE: host build of s2m_batch_pack (liliom_b200/csrc/s2m_plan.h), the packing of a batched scan-to-map step's
// sessions into cooperative launches, so that the CPU test tier checks the same source s2m_batch uses.
#include "../liliom_b200/csrc/s2m_plan.h"

// plans: per session {lanes, tma, grid, persistent}.  out_kind / out_grid per launch, out_sess: the launches' sessions in order,
// out_count per launch, solo: the sessions on the solo path.  Returns the launch count; *n_solo the solo count.
extern "C" int sb_pack(int B, const int* plans, const int* occ, int sm_count, int max_per_launch, int* out_kind, int* out_grid,
                       int* out_count, int* out_sess, int* solo, int* n_solo) {
    std::vector<lili::S2mPlan> ps(B);
    for (int i = 0; i < B; ++i) {
        ps[i] = lili::S2mPlan{};
        ps[i].lanes = plans[4 * i]; ps[i].tma = plans[4 * i + 1] != 0; ps[i].grid = plans[4 * i + 2]; ps[i].persistent = plans[4 * i + 3] != 0;
    }
    const lili::BatchPack p = lili::s2m_batch_pack(ps, occ, sm_count, max_per_launch);
    int k = 0;
    for (size_t l = 0; l < p.launches.size(); ++l) {
        out_kind[l] = p.launches[l].kind; out_grid[l] = p.launches[l].grid; out_count[l] = (int)p.launches[l].sessions.size();
        for (int s : p.launches[l].sessions) out_sess[k++] = s;
    }
    for (size_t j = 0; j < p.solo.size(); ++j) solo[j] = p.solo[j];
    *n_solo = (int)p.solo.size();
    return (int)p.launches.size();
}

// the kBatchMax the library packs with
extern "C" int sb_batch_max() { return lili::kBatchMax; }
