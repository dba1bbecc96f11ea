// TEST INFRASTRUCTURE: host build of the block geometry of the batched map update (liliom_b200/csrc/map_stage.h), so that the CPU
// test tier checks the same source k_map_stage_batch runs.
#include "../liliom_b200/csrc/map_stage.h"

extern "C" int ms_stage_blocks(int items, int threads) { return lili::stage_blocks(items, threads); }
extern "C" int ms_box_blocks(int n, int sm_count) { return lili::box_blocks(n, sm_count); }
// session of block b among n sessions with blocks[s] blocks each; *place: the block's place inside it
extern "C" int ms_session_of(int n, const int* blocks, int b, int* place) {
    const int s = lili::batch_session_of(n, b, [&](int k) { return blocks[k]; });
    *place = b;
    return s;
}
