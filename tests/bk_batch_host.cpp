// TEST INFRASTRUCTURE: host build of liliom_b200/csrc/bk_batch.h, the layout of the batched backend window calls (the sessions'
// offsets in a concatenated table, each segment's place, the launches past kBatchMax sessions), so that the CPU test tier checks
// the same source the batched calls use.
#include "../liliom_b200/csrc/bk_batch.h"

// offsets of n sessions with count[m] items each into off (n + 1 ints)
extern "C" void bb_offsets(int n, const int* count, int* off) {
    const std::vector<int> o = lili::bkb_offsets(std::vector<int>(count, count + n));
    for (int m = 0; m <= n; ++m) off[m] = o[m];
}
// the concatenated segment index of session m's keyframe i and kind, the sessions having 2 k[m] segments each
extern "C" int bb_segment(int n, const int* k, int m, int i, int kind) {
    std::vector<int> c(n);
    for (int s = 0; s < n; ++s) c[s] = 2 * k[s];
    return lili::bkb_segment(lili::bkb_offsets(c), m, i, kind);
}
// the launches over n sessions with count[m] items each: 4 ints per launch {first, n, item0, items}; returns the launch count
extern "C" int bb_launches(int n, const int* count, int* out) {
    const std::vector<lili::BkbLaunch> L = lili::bkb_launches(lili::bkb_offsets(std::vector<int>(count, count + n)));
    for (size_t l = 0; l < L.size(); ++l) {
        out[4 * l] = L[l].first; out[4 * l + 1] = L[l].n; out[4 * l + 2] = L[l].item0; out[4 * l + 3] = L[l].items;
    }
    return (int)L.size();
}
extern "C" long long bb_region(long long n, long long size) { return (long long)lili::bkb_region((size_t)n, (size_t)size); }
extern "C" int bb_cnt_ints() { return lili::kBkbCntInts; }
extern "C" int bb_batch_max() { return lili::kBatchMax; }
extern "C" int bb_win_max() { return lili::kWinMax; }
