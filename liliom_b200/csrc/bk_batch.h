// Host layout of the batched backend window calls (liliom_backend_window_correspond_batch / _blocks_batch, backend_corr.cu): where
// each session's entries sit in the tables one call uploads and the results it downloads, and which sessions each launch covers.
// Plain C++, so that the CPU tests compile it as it is (tests/bk_batch_host.cpp).
#pragma once
#include <vector>
#include "batch.h"
#include "bk_window.h"

namespace lili {

// Session m of a call (the sessions that take part, in call order) owns items [off[m], off[m + 1]) of a concatenated table,
// count[m] of them: off has count.size() + 1 entries, off[0] = 0.
inline std::vector<int> bkb_offsets(const std::vector<int>& count) {
    std::vector<int> off(count.size() + 1, 0);
    for (size_t m = 0; m < count.size(); ++m) off[m + 1] = off[m] + count[m];
    return off;
}

// The blocks of a window of k keyframes: 2 k segments, segment 2 i = the edge rows, 2 i + 1 = the surf rows of keyframe i
// (liliom_backend_window_blocks' order).  Session m's segment of keyframe i and kind in the concatenated segment table:
inline int bkb_segment(const std::vector<int>& seg_off, int m, int i, int kind) { return seg_off[m] + 2 * i + kind; }

// The launches over the sessions of a concatenated table: launch L covers sessions [first, first + n), at most kBatchMax of them,
// and their items [item0, item0 + items), in order.
struct BkbLaunch {
    int first, n, item0, items;
};
inline std::vector<BkbLaunch> bkb_launches(const std::vector<int>& off) {
    std::vector<BkbLaunch> out;
    const int S = (int)off.size() - 1;
    for (int first = 0; first < S; first += kBatchMax) {
        const int n = S - first < kBatchMax ? S - first : kBatchMax;
        out.push_back(BkbLaunch{first, n, off[first], off[first + n] - off[first]});
    }
    return out;
}

// The correspondence counts of a batched correspond call, read back at once: session m's edge count of keyframe i at
// m * kBkbCntInts + i, its surf count at m * kBkbCntInts + kWinMax + i (the layout of one context's win_cnt).
constexpr int kBkbCntInts = 2 * kWinMax;

// Bytes of a region of `n` items of `size` bytes each, rounded up to 256 so that the next region starts aligned.
inline size_t bkb_region(size_t n, size_t size) { return (n * size + 255) / 256 * 256; }

}  // namespace lili
