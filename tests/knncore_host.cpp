// TEST INFRASTRUCTURE: host build of the pruned search of liliom_b200/csrc/knn_core.cuh (query_cell, cell_bound, row_cells, consider,
// thread_knn5 — the one-thread-per-query shape of the roofline kernel — group_knn5, the 2/4/8/16-lane shape of the small-scan
// and backend kernels, and coherence_tau, the start threshold of every GN pass after the first) so that the CPU test tier can run
// the SAME SOURCE the kernels compile against an exhaustive search: the claim under test is that thresholds, cell lower bounds, run
// trimming, the per-thread run list, the per-lane rows, the butterfly merge and the coherence bound never change the five nearest
// keys.  Round-to-nearest intrinsics become plain operators (-ffp-contract=off), the round-up ones the same operators under
// FE_UPWARD (-frounding-math keeps the compiler from folding or moving them across the mode switch), read-only loads become plain
// loads.  A lane group is LANES host threads in lock step: __shfl_xor_sync publishes the value, meets the group at a barrier, reads
// the partner's slot and meets it again (the merge calls it equally often on every lane, so this cannot deadlock).
// Only the register path of group_knn5 runs (stage == nullptr).  The bulk-copy staging branch of group_knn5<16> holds sm_90a inline
// PTX that no host assembler accepts: it is dropped as dead code because every call here passes a null `stage` into the
// always-inlined function, which needs optimisation — the fixture compiles at -O2, and an unoptimised build fails to assemble.
// Compiled with -std=c++20 -pthread (std::barrier).
#include <algorithm>
#include <barrier>
#include <cfenv>
#include <cmath>
#include <cfloat>
#include <cstring>
#include <thread>
#include <vector>
using std::min;
using std::max;
using std::isfinite;
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
// round toward +inf: the operation runs under FE_UPWARD, the previous mode is restored afterwards
struct Upward {
    int old;
    Upward() : old(fegetround()) { fesetround(FE_UPWARD); }
    ~Upward() { fesetround(old); }
};
static inline float __fadd_ru(float a, float b) { Upward u; volatile float r = a + b; return r; }
static inline float __fmul_ru(float a, float b) { Upward u; volatile float r = a * b; return r; }
static inline float __fsqrt_ru(float a) { Upward u; volatile float r = std::sqrt(a); return r; }
static inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline int __float_as_int(float f) { int u; memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
static inline float __int_as_float(int u) { float f; memcpy(&f, &u, 4); return f; }
template <class T> static inline T __ldg(const T* p) { return *p; }

// One lane group: a slot per lane and the barrier the exchanges meet at.  Every lane thread knows its group and lane.
struct LaneGroup {
    std::barrier<>* bar;
    unsigned long long slot[32];
};
static thread_local LaneGroup* tl_group = nullptr;
static thread_local int tl_lane = 0;
template <class T> static T __shfl_xor_sync(unsigned, T v, int o) {
    static_assert(sizeof(T) <= sizeof(unsigned long long), "one slot per lane");
    unsigned long long w = 0;
    memcpy(&w, &v, sizeof(T));
    tl_group->slot[tl_lane] = w;
    tl_group->bar->arrive_and_wait();          // every lane has published
    w = tl_group->slot[tl_lane ^ o];
    tl_group->bar->arrive_and_wait();          // every lane has read: the slots may be overwritten
    T r;
    memcpy(&r, &w, sizeof(T));
    return r;
}
static inline long long clock64() { return 0; }
static inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)p; }
#include <cuda_runtime.h>
#ifndef __noinline__
#define __noinline__
#endif
#include "../liliom_b200/csrc/knn_core.cuh"

using namespace lili;

static GridDesc make_grid(float inv_cell, const int org[3], const int dim[3]) {
    GridDesc g;
    g.inv_cell = inv_cell;
    for (int k = 0; k < 3; ++k) { g.org[k] = org[k]; g.dim[k] = dim[k]; }
    g.ncells = dim[0] * dim[1] * dim[2];
    return g;
}

// nq queries through one lane group of LANES threads; lane `sub` of query i leaves its merged set in lane_out[(i * LANES + sub) * 5]
template <int LANES>
static void run_group(int nq, const float* q3, const float4* map, const int* cell_start, const GridDesc& g, const float* tau0,
                      unsigned long long* lane_out, unsigned long long* cand) {
    std::barrier<> bar(LANES);
    LaneGroup grp{&bar, {}};
    const unsigned gmask = (1u << LANES) - 1u;
    std::vector<std::thread> lanes;
    for (int sub = 0; sub < LANES; ++sub) {
        lanes.emplace_back([&, sub] {
            tl_group = &grp;
            tl_lane = sub;
            for (int i = 0; i < nq; ++i) {
                Top5 top;
                top5_init(top);
                unsigned long long c = 0;
                group_knn5<LANES>(q3[3 * i], q3[3 * i + 1], q3[3 * i + 2], map, cell_start, g, sub, gmask, tau0[i], top, c);
                unsigned long long* o = lane_out + ((size_t)i * LANES + sub) * 5;
                o[0] = top.k0; o[1] = top.k1; o[2] = top.k2; o[3] = top.k3; o[4] = top.k4;
                cand[(size_t)i * LANES + sub] = c;
            }
        });
    }
    for (auto& t : lanes) t.join();
}

extern "C" {
float kc_gate_tau(double max_sqd) { return knn_gate_tau(max_sqd); }
int kc_owner_of(float x, float y, float z, int nranks, float inv_block) { return owner_of(x, y, z, nranks, inv_block); }

// map_sorted: m x {x, y, z, index bits} in cell order; returns the number of map points examined
unsigned long long kc_thread_knn5(float sx, float sy, float sz, const float* map_sorted, const int* cell_start, float inv_cell,
                                  const int org[3], const int dim[3], float tau0, unsigned long long out5[5]) {
    const GridDesc g = make_grid(inv_cell, org, dim);
    Top5 top;
    top5_init(top);
    unsigned long long cand = 0;
    int4 runs[kRunCap];
    thread_knn5<8, 4>(sx, sy, sz, reinterpret_cast<const float4*>(map_sorted), cell_start, g, tau0, runs, 1, top, cand);
    out5[0] = top.k0; out5[1] = top.k1; out5[2] = top.k2; out5[3] = top.k3; out5[4] = top.k4;
    return cand;
}

// coherence_tau for n queries: st4[4 * i ..] = {previous position, previous fifth distance}, s3[3 * i ..] = new position
void kc_coherence_tau(int n, const float* st4, const float* s3, float tau0, float* out) {
    for (int i = 0; i < n; ++i) {
        const float4 st = make_float4(st4[4 * i], st4[4 * i + 1], st4[4 * i + 2], st4[4 * i + 3]);
        out[i] = coherence_tau(st, s3[3 * i], s3[3 * i + 1], s3[3 * i + 2], tau0);
    }
}

// group_knn5<lanes> (lanes = 2, 4, 8 or 16; register path) for nq queries q3[3 * i ..] with start thresholds tau0[i].
// out5[5 * i ..]: lane 0's merged set; agree[i] = 1 when every lane of the group ended with the same set; cand[i]: map points the
// group examined.  Returns 0, or -1 for an unsupported lane count.
int kc_group_knn5(int lanes, int nq, const float* q3, const float* map_sorted, const int* cell_start, float inv_cell, const int org[3],
                  const int dim[3], const float* tau0, unsigned long long* out5, int* agree, unsigned long long* cand) {
    if (lanes != 2 && lanes != 4 && lanes != 8 && lanes != 16) return -1;
    const GridDesc g = make_grid(inv_cell, org, dim);
    const float4* map = reinterpret_cast<const float4*>(map_sorted);
    std::vector<unsigned long long> lane_out((size_t)nq * lanes * 5), lane_cand((size_t)nq * lanes);
    switch (lanes) {
        case 2: run_group<2>(nq, q3, map, cell_start, g, tau0, lane_out.data(), lane_cand.data()); break;
        case 4: run_group<4>(nq, q3, map, cell_start, g, tau0, lane_out.data(), lane_cand.data()); break;
        case 8: run_group<8>(nq, q3, map, cell_start, g, tau0, lane_out.data(), lane_cand.data()); break;
        default: run_group<16>(nq, q3, map, cell_start, g, tau0, lane_out.data(), lane_cand.data()); break;
    }
    for (int i = 0; i < nq; ++i) {
        const unsigned long long* l0 = lane_out.data() + (size_t)i * lanes * 5;
        int same = 1;
        unsigned long long c = 0;
        for (int s = 0; s < lanes; ++s) {
            if (memcmp(l0, l0 + (size_t)s * 5, 5 * sizeof(unsigned long long)) != 0) same = 0;
            c += lane_cand[(size_t)i * lanes + s];
        }
        memcpy(out5 + (size_t)i * 5, l0, 5 * sizeof(unsigned long long));
        agree[i] = same;
        cand[i] = c;
    }
    return 0;
}
}
