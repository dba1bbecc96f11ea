// Host build of liliom_b200/csrc/ctx.cuh for tests/test_ctx_host.py: the ownership rules of the context's device buffers.
// cudaFree is counted (and not forwarded) so that the buffers can hold made-up addresses on a machine without a GPU.
#include <cuda_runtime.h>
#include <type_traits>
#include <utility>
#include <vector>

static int g_frees = 0;
static void* g_last_freed = nullptr;
static cudaError_t counted_cudaFree(void* p) { ++g_frees; g_last_freed = p; return cudaSuccess; }
#define cudaFree counted_cudaFree
#include "../liliom_b200/csrc/ctx.cuh"
#undef cudaFree

using lili::DevBuf;
using lili::Frame;
using lili::MapIndex;

template <class T> constexpr bool move_only() {
    return !std::is_copy_constructible<T>::value && !std::is_copy_assignable<T>::value &&
           std::is_nothrow_move_constructible<T>::value && std::is_nothrow_move_assignable<T>::value;
}
static_assert(move_only<DevBuf>(), "DevBuf owns its allocation: move-only, nothrow moves");
static_assert(move_only<MapIndex>(), "MapIndex owns its buffers: move-only, nothrow moves");
static_assert(move_only<Frame>(), "Frame owns its buffer: move-only, nothrow moves");

static DevBuf fake(unsigned long long addr, size_t cap) {
    DevBuf b;
    b.p = reinterpret_cast<void*>(addr); b.cap = cap;
    return b;
}

// Each check returns 0 when it holds; the first failing check's number otherwise.
extern "C" int ctx_host_run() {
    g_frees = 0;
    { DevBuf empty; }
    if (g_frees != 0) return 1;                                        // an empty buffer makes no CUDA call
    {
        DevBuf a = fake(0x1000, 64);
        DevBuf b(std::move(a));
        if (a.p || a.cap || b.p != reinterpret_cast<void*>(0x1000) || b.cap != 64) return 2;
        DevBuf d;
        d = std::move(b);
        if (b.p || b.cap || d.cap != 64 || g_frees != 0) return 3;      // moves free nothing
    }
    if (g_frees != 1 || g_last_freed != reinterpret_cast<void*>(0x1000)) return 4;   // the owner frees once; moved-from ones are silent
    g_frees = 0;
    {
        DevBuf x = fake(0x2000, 16), y = fake(0x3000, 32);
        x = std::move(y);                                               // the target's old allocation is freed
        if (g_frees != 1 || g_last_freed != reinterpret_cast<void*>(0x2000) || x.cap != 32 || y.p) return 5;
        x = std::move(x);                                               // self-move keeps the allocation
        if (g_frees != 1 || x.p != reinterpret_cast<void*>(0x3000)) return 6;
    }
    if (g_frees != 2) return 7;
    g_frees = 0;
    {   // the map FIFO: recycling the front frame's buffer, erasing it and pushing by move (with regrowth) free nothing
        std::vector<Frame> frames;
        for (int i = 0; i < 20; ++i) {
            Frame f;
            f.buf = fake(0x10000 + 0x100 * (unsigned long long)i, 256);
            frames.push_back(std::move(f));
        }
        for (int s = 0; s < 50; ++s) {
            Frame f;
            f.buf = std::move(frames.front().buf);
            frames.erase(frames.begin());
            frames.push_back(std::move(f));
        }
        if (g_frees != 0) return 8;
        frames.clear();
        if (g_frees != 20) return 9;
    }
    g_frees = 0;
    { MapIndex mi; mi.xyzw = fake(0x4000, 16); mi.sorted = fake(0x5000, 16); MapIndex m2(std::move(mi)); }
    if (g_frees != 2) return 10;
    return 0;
}
