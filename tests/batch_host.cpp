// TEST INFRASTRUCTURE: host build of liliom_b200/csrc/batch.h, the geometry and the packing of the launches several sessions
// share, so that the CPU test tier checks the same source the batched kernels and calls use.
#include "../liliom_b200/csrc/batch.h"

extern "C" int bh_stage_blocks(int items, int threads) { return lili::stage_blocks(items, threads); }
extern "C" int bh_box_blocks(int n, int sm_count) { return lili::box_blocks(n, sm_count); }
// session of block b among n <= kBatchMax sessions with blocks[s] blocks each, looked up in the prefix offsets of a launch's
// table; *place: the block's place inside its session
template <class Tab>
static int session_of(int n, const int* blocks, int b, int* place) {
    Tab tab{};
    tab.n = n;
    for (int s = 0; s < n; ++s) tab.off[s + 1] = tab.off[s] + blocks[s];
    const int s = lili::batch_session_of(tab.n, tab.off, b);
    *place = b - tab.off[s];
    return s;
}
extern "C" int bh_session_of(int n, const int* blocks, int b, int* place) {
    return session_of<lili::BatchTab<int>>(n, blocks, b, place);
}
// the same in the one-entry table of a one-session launch (n == 1)
extern "C" int bh_session_of1(int n, const int* blocks, int b, int* place) {
    return session_of<lili::BatchTab<int, 1>>(n, blocks, b, place);
}
// batch_pack of B sessions {grid, kind, coop}: out_kind / out_grid / out_count per launch, out_sess the launches' sessions in
// order, solo the sessions on their solo path.  Returns the launch count; *n_solo the solo count.
extern "C" int bh_pack(int B, const int* items, const int* occ, int sm_count, int max_per_launch, int* out_kind, int* out_grid,
                       int* out_count, int* out_sess, int* solo, int* n_solo) {
    std::vector<lili::BatchItem> its;
    for (int i = 0; i < B; ++i) its.push_back(lili::BatchItem{items[3 * i], items[3 * i + 1], items[3 * i + 2] != 0});
    const lili::BatchPack p = lili::batch_pack(its, occ, sm_count, max_per_launch);
    int k = 0;
    for (size_t l = 0; l < p.launches.size(); ++l) {
        out_kind[l] = p.launches[l].kind; out_grid[l] = p.launches[l].grid; out_count[l] = (int)p.launches[l].sessions.size();
        for (int s : p.launches[l].sessions) out_sess[k++] = s;
    }
    for (size_t j = 0; j < p.solo.size(); ++j) solo[j] = p.solo[j];
    *n_solo = (int)p.solo.size();
    return (int)p.launches.size();
}
extern "C" int bh_batch_max() { return lili::kBatchMax; }
