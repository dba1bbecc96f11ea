// Block geometry of the launches that several sessions share (k_map_stage_batch, map.cu): how many blocks a stage gives a session,
// and which session a block of the shared grid belongs to.  Plain C++ for host and device, so that the CPU tests check the source
// the kernels run (tests/map_stage_host.cpp).
#pragma once

#ifdef __CUDACC__
#define LILI_MS_HD __host__ __device__
#else
#define LILI_MS_HD
#endif

namespace lili {

// blocks of `threads` threads for `items` items, one thread per item (0 items: no block)
LILI_MS_HD inline int stage_blocks(int items, int threads) { return (items + threads - 1) / threads; }

// grid of the box pass over n points (k_vg_minmax: a grid-stride loop, capped at eight blocks per SM)
LILI_MS_HD inline int box_blocks(int n, int sm_count) {
    const int b = stage_blocks(n, 256);
    return b < sm_count * 8 ? b : sm_count * 8;
}

// The session that block b of a shared grid belongs to, when session s owns the blocks_of(s) blocks after those of sessions
// 0 .. s-1; b becomes the block's place inside its session.  A session without blocks owns none; the grid is the sum of the
// sessions' blocks, so the last session takes what is left.
template <class F>
LILI_MS_HD inline int batch_session_of(int n_sessions, int& b, F blocks_of) {
    int s = 0;
    while (s + 1 < n_sessions && b >= blocks_of(s)) { b -= blocks_of(s); ++s; }
    return s;
}

}  // namespace lili
