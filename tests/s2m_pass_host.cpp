// TEST INFRASTRUCTURE: host build of s2m_pass_pack and s2m_gn_groups (liliom_b200/csrc/s2m_plan.h), the launches of a batched
// scan-to-map step with per-session iteration counts, so that the CPU test tier checks the same source s2m_batch uses.
// Both write their result as one flat int stream into out[cap] and return its length (-1: cap too small).
#include "../liliom_b200/csrc/s2m_plan.h"

namespace {
struct Out {
    int* p; int cap, n = 0;
    void put(int v) { if (n < cap) p[n] = v; ++n; }
    void list(const std::vector<int>& v) { put((int)v.size()); for (int s : v) put(s); }
    int done() const { return n <= cap ? n : -1; }
};
std::vector<lili::S2mPlan> plans_of(int B, const int* plans) {
    std::vector<lili::S2mPlan> ps(B);
    for (int i = 0; i < B; ++i) {
        ps[i] = lili::S2mPlan{};
        ps[i].lanes = plans[4 * i]; ps[i].tma = plans[4 * i + 1] != 0; ps[i].grid = plans[4 * i + 2]; ps[i].persistent = plans[4 * i + 3] != 0;
    }
    return ps;
}
}  // namespace

// plans: per session {lanes, tma, grid, persistent}.  Stream: passes, then per pass: knn launches, each {lanes, count,
// sessions...}, then LM launches, each {count, sessions...}.
extern "C" int sp_pass_pack(int B, const int* plans, const int* iters, int max_per_launch, int* out, int cap) {
    const std::vector<lili::S2mPass> ps = lili::s2m_pass_pack(plans_of(B, plans), std::vector<int>(iters, iters + B), max_per_launch);
    Out o{out, cap};
    o.put((int)ps.size());
    for (const lili::S2mPass& p : ps) {
        o.put((int)p.knn.size());
        for (const lili::S2mKnnLaunch& l : p.knn) { o.put(l.lanes); o.list(l.sessions); }
        o.put((int)p.lm.size());
        for (const std::vector<int>& l : p.lm) o.list(l);
    }
    return o.done();
}

// Stream: groups, then per group: iters, launches, each {kind, grid, count, sessions...}, then the solo list {count, sessions...}.
extern "C" int sp_gn_groups(int B, const int* plans, const int* iters, const int* occ, int sm_count, int max_per_launch, int* out, int cap) {
    const std::vector<lili::S2mGnGroup> gs = lili::s2m_gn_groups(plans_of(B, plans), std::vector<int>(iters, iters + B), occ, sm_count,
                                                                 max_per_launch);
    Out o{out, cap};
    o.put((int)gs.size());
    for (const lili::S2mGnGroup& g : gs) {
        o.put(g.iters);
        o.put((int)g.pack.launches.size());
        for (const lili::BatchLaunch& l : g.pack.launches) { o.put(l.kind); o.put(l.grid); o.list(l.sessions); }
        o.list(g.pack.solo);
    }
    return o.done();
}
