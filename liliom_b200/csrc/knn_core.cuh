// Exact 5-NN over the dense cell grid (shared by the scan-to-map kernel and the backend correspondence kernels).
// See grid_knn.cu for the design notes.
//
// Candidate ordering is (fp32 squared distance, map index).  Both live in one 64-bit key
//     key = (bits(d) << 32) | index             (d >= +0, so the bit pattern orders like the value)
// so a single unsigned compare implements FLANN's distance order plus our index tie-break with
// no branches and no extra loads.
//
// Pruning (without it, every query ranks all ~63 points of its 27 cells and the 64-bit ranking chain dominates the issued
// instructions).  A correspondence needs its FIFTH neighbour inside the
// gate (d5 < knn_max_sqdist, L/src/LidarOdometry.cpp:365), so a candidate at or beyond the gate can never be part of an
// accepted set, and once five candidates are held nothing beyond the current fifth distance can enter the set either:
//   * every candidate is tested against the running threshold `tau` with ONE fp32 compare before its key is built;
//   * whole cells are skipped when their lower bound exceeds `tau`.  The bound is the candidate distance expression itself,
//     ((dx*dx) + dy*dy) + dz*dz in round-to-nearest fp32, evaluated at the faces of the query's own cell: every point of the
//     skipped cell has |coordinate difference| >= the face distance per axis in exact arithmetic, fp32 subtraction,
//     multiplication and addition are monotonic, hence its computed distance is >= the bound.  The accepted sets and
//     their order are bit-identical to the exhaustive search (and to the oracle's kd-tree); a query that ends with
//     fewer than five candidates inside the gate is rejected by both.
// Loops are deliberately NOT unrolled: unrolled, this kernel grows to ~12k SASS instructions and
// stalls on instruction-cache misses.
#pragma once
#include "ctx.cuh"
#include "dev_math.cuh"
#include "s2m_plan.h"
#include <cmath>

namespace lili {

__device__ __forceinline__ int cell_coord(float v, float inv_cell) { return (int)floorf(v * inv_cell); }

// Ownership of a point for the sharded map: space is cut into cubes of 1/inv_block metres (a power of two, default 16 m)
// and the cube's hash picks the rank (SURVEY.md §8 e).  The hash is linear, h = bx + 3 by + 5 bz (mod nranks): over any
// rectangular stretch of cubes every rank gets the same share (a multiplicative hash left one of 8 ranks 20 % and another
// 7 % of a 1.2 km map in 64 m cubes) and face neighbours never share a rank.  The cubes are shifted by half an edge in z:
// a vehicle's map is a thin slab around z = 0, and a cube boundary there would put every ground point into the halo of
// two cubes (measured on 2 GPUs: 75 % of the map on each rank instead of 60 %).
__device__ __forceinline__ int owner_of(float x, float y, float z, int nranks, float inv_block) {
    const int bx = (int)floorf(x * inv_block), by = (int)floorf(y * inv_block), bz = (int)floorf(z * inv_block + 0.5f);
    const int h = (bx + 3 * by + 5 * bz) % nranks;
    return h < 0 ? h + nranks : h;
}

typedef unsigned long long u64;

// Largest float t with (double)t < max_sqd: "d <= t" is then the reference's gate "(double)d < max_sqd".
inline float knn_gate_tau(double max_sqd) {
    float f = (float)max_sqd;
    while ((double)f >= max_sqd) f = nextafterf(f, -INFINITY);
    while ((double)nextafterf(f, INFINITY) < max_sqd) f = nextafterf(f, INFINITY);
    return f;
}

// Sorted (ascending) list of the five best keys.  The low word of a key is the neighbour's index in
// the un-sorted map array (map_download order), which is also where phase B fetches its coordinates
// from, so no separate payload has to ride through the compare-exchanges.
struct Top5 { u64 k0, k1, k2, k3, k4; };

__device__ __forceinline__ void top5_init(Top5& t) { t.k0 = t.k1 = t.k2 = t.k3 = t.k4 = ~0ull; }
__device__ __forceinline__ float top5_dist(u64 k) { return __uint_as_float((unsigned)(k >> 32)); }
__device__ __forceinline__ int top5_index(u64 k) { return k == ~0ull ? -1 : (int)(unsigned)(k & 0xffffffffull); }

__device__ __forceinline__ void cswap(u64& a, u64& b) {   // afterwards a <= b
    const bool s = b < a;
    const u64 lo = s ? b : a, hi = s ? a : b;
    a = lo; b = hi;
}

__device__ __forceinline__ void top5_insert(Top5& t, u64 k) {
    if (k < t.k4) {
        t.k4 = k;
        cswap(t.k3, t.k4);
        cswap(t.k2, t.k3);
        cswap(t.k1, t.k2);
        cswap(t.k0, t.k1);
    }
}

// FLANN L2_Simple<float>: ((dx*dx) + dy*dy) + dz*dz with no contraction (exact-op intrinsics)
__device__ __forceinline__ float cand_dist(float sx, float sy, float sz, const float4& m) {
    const float dx = fsubx(sx, m.x), dy = fsubx(sy, m.y), dz = fsubx(sz, m.z);
    return faddx(faddx(fmulx(dx, dx), fmulx(dy, dy)), fmulx(dz, dz));
}
__device__ __forceinline__ u64 make_key(float d, const float4& m) {
    return ((u64)__float_as_uint(d) << 32) | (u64)(unsigned)__float_as_int(m.w);
}

// One candidate: cheap fp32 reject against the running threshold, then the ranked insert.  tau is the largest distance that
// can still enter the set: the gate until five candidates are held, then the fifth distance (ties go on to the index compare).
__device__ __forceinline__ void consider(float sx, float sy, float sz, const float4& m, Top5& top, float& tau) {
    const float d = cand_dist(sx, sy, sz, m);
    if (d <= tau) {
        top5_insert(top, make_key(d, m));
        tau = fminf(tau, top5_dist(top.k4));        // k4 == ~0 decodes to NaN: fminf keeps tau
    }
}

// Temporal coherence of the GN passes: a query whose five neighbours lay within r = sqrt(d5) at its previous position p'
// still has those five map points within r + |p - p'| of its new position p, so its new fifth distance is at most
// (r + |p - p'|)^2.  Starting the search with that bound instead of the gate skips most cells outright and leaves little to
// rank — from the second pass of a scan on the poses move by centimetres.  The bound is evaluated with upward roundings and
// a 1e-5 relative margin (the candidate distance expression carries ~3 fp32 roundings, ~2e-7), so every point of the true
// 5-NN set passes the filter: the sets found, their order and the accept decisions are exactly those of the full search.
// `st`: {p', d5} of the previous pass (d5 = +inf or NaN: no five neighbours inside the gate then).
__device__ __forceinline__ float coherence_tau(const float4& st, float sx, float sy, float sz, float tau0) {
    if (!(st.w <= tau0)) return tau0;                    // no five neighbours inside the gate last time (or NaN): nothing to exploit
    const float dx = fsubx(sx, st.x), dy = fsubx(sy, st.y), dz = fsubx(sz, st.z);
    const float mv = __fsqrt_ru(__fadd_ru(__fadd_ru(__fmul_ru(dx, dx), __fmul_ru(dy, dy)), __fmul_ru(dz, dz)));
    const float r = __fadd_ru(__fsqrt_ru(st.w), mv);
    return fminf(tau0, __fmul_ru(__fmul_ru(r, r), 1.00001f));
}

// The query's cell and the SQUARED distances to its six faces (>= 0; 0 is always a valid lower bound).
struct QCell {
    int cx, cy, cz;                     // grid-relative cell coordinates (may lie outside the grid)
    float xl, xh, yl, yh, zl, zh;       // (sx - lo_x)^2, (hi_x - sx)^2, ... each rounded once, like a candidate's dx*dx
};
__device__ __forceinline__ QCell query_cell(float sx, float sy, float sz, const GridDesc& g) {
    QCell q;
    const float cell = 1.0f / g.inv_cell;                      // power of two: all products below are exact
    const float fx = floorf(sx * g.inv_cell), fy = floorf(sy * g.inv_cell), fz = floorf(sz * g.inv_cell);
    q.cx = (int)fx - g.org[0]; q.cy = (int)fy - g.org[1]; q.cz = (int)fz - g.org[2];
    const float lx = fx * cell, ly = fy * cell, lz = fz * cell;
    const float xl = fmaxf(fsubx(sx, lx), 0.f), xh = fmaxf(fsubx(faddx(lx, cell), sx), 0.f);
    const float yl = fmaxf(fsubx(sy, ly), 0.f), yh = fmaxf(fsubx(faddx(ly, cell), sy), 0.f);
    const float zl = fmaxf(fsubx(sz, lz), 0.f), zh = fmaxf(fsubx(faddx(lz, cell), sz), 0.f);
    q.xl = fmulx(xl, xl); q.xh = fmulx(xh, xh); q.yl = fmulx(yl, yl); q.yh = fmulx(yh, yh); q.zl = fmulx(zl, zl); q.zh = fmulx(zh, zh);
    return q;
}
// lower bound of the candidate distance over a cell at offset (ox, oy, oz) in {-1,0,1}^3: the candidate expression
// ((dx*dx) + dy*dy) + dz*dz with the face distances in place of the differences, same roundings
__device__ __forceinline__ float cell_bound(const QCell& q, int ox, int oy, int oz) {
    const float bx = ox < 0 ? q.xl : ox > 0 ? q.xh : 0.f;
    const float by = oy < 0 ? q.yl : oy > 0 ? q.yh : 0.f;
    const float bz = oz < 0 ? q.zl : oz > 0 ? q.zh : 0.f;
    return faddx(faddx(bx, by), bz);
}

// Run of the cell-sorted map covering the cells of row (oy, oz) that can still hold a neighbour: the three x-adjacent
// cells are ONE contiguous run, its ends are trimmed by the bound.  Returns false when nothing is left.
__device__ __forceinline__ bool row_cells(const QCell& q, const GridDesc& g, int oy, int oz, float tau, int& idx_b, int& idx_e) {
    const int y = q.cy + oy, z = q.cz + oz;
    if (y < 0 || y >= g.dim[1] || z < 0 || z >= g.dim[2]) return false;
    if (cell_bound(q, 0, oy, oz) > tau) return false;
    int xs = q.cx - 1, xe = q.cx + 1;
    if (cell_bound(q, -1, oy, oz) > tau) xs = q.cx;
    if (cell_bound(q, +1, oy, oz) > tau) xe = q.cx;
    xs = max(xs, 0); xe = min(xe, g.dim[0] - 1);
    if (xs > xe) return false;
    const int base = (z * g.dim[1] + y) * g.dim[0];
    idx_b = base + xs; idx_e = base + xe + 1;
    return true;
}

// ---- bulk-asynchronous staging of a lane's run in shared memory (sm_90a: cp.async.bulk + mbarrier; SASS UBLKCP / SYNCS) ----
// The 16-lane search gives every (y,z) row of the 27-cell block to one lane.  Instead of pulling its run through registers in
// batches of eight 16-byte loads (a dependent L2 round trip per batch), a lane hands the whole run to the copy engine — one
// cp.async.bulk of 16 x length bytes into its slot of the warp's staging tile — and the 16 lanes of the query meet at one
// mbarrier whose transaction count is the sum of their run sizes; ranking then reads shared memory.
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, unsigned parity) {
    unsigned ok;
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
constexpr int kStageCap = 24;                 // candidates per staged run (longer runs finish through registers)
constexpr int kStageRow = kStageCap + 1;      // row pitch in float4: 25 x 16 B = 100 words -> lane k starts at bank 4k (conflict-free 16-byte reads)
struct StageTile {                            // one per lane group (query) of a warp
    float4 pts[9][kStageRow];
    unsigned long long bar;
    unsigned long long pad;
};
static_assert(sizeof(StageTile) == kStageTileBytes, "s2m_plan.h sizes the staging tiles");

// LANES (2, 4, 8 or 16) lanes — mask `gmask`, lane-in-group `sub` — search the 3x3x3 cell block around
// (sx,sy,sz); lane `sub` walks rows sub, sub+LANES, ...  Each lane pulls its run in batches of independent 16-byte
// loads (memory-level parallelism without occupancy), ranks them into a private sorted top-5, and the group merges with
// 5 min-butterflies.  On return every lane of the group holds the merged top-5.
// `cand` accumulates the number of map points this lane examined.
// `stage` (16-lane shape only, may be null): the group's staging tile; `stage_phase` its mbarrier parity, flipped per use.
template <int LANES, int BATCH = 8>
__device__ __forceinline__ void group_knn5(float sx, float sy, float sz, const float4* __restrict__ map,
                                           const int* __restrict__ cell_start, const GridDesc& g, int sub, unsigned gmask, float tau0,
                                           Top5& top, unsigned long long& cand, long long* dbg = nullptr, StageTile* stage = nullptr,
                                           unsigned* stage_phase = nullptr) {
    static_assert(LANES > 1, "one thread per query: thread_knn5");
    const QCell qc = query_cell(sx, sy, sz, g);
    float tau = tau0;
    if (LANES == 16 && stage) {
        // one row per lane (9 of the 16), the whole run staged by ONE bulk copy; all 16 lanes meet at the mbarrier
        int b = 0, e = 0, ib, ie;
        if (sub < 9 && row_cells(qc, g, (sub % 3) - 1, (sub / 3) - 1, tau, ib, ie)) { b = __ldg(cell_start + ib); e = __ldg(cell_start + ie); }
        const int n1 = min(e - b, kStageCap);
        // the tile's previous contents were read through the generic proxy: order those reads before the async-proxy write
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if (n1 > 0) {
            mbar_arrive_expect_tx(&stage->bar, (unsigned)n1 * 16u);
            bulk_g2s(&stage->pts[sub][0], map + b, (unsigned)n1 * 16u, &stage->bar);
        } else mbar_arrive(&stage->bar);
        cand += (unsigned long long)(e - b);
        const unsigned ph = *stage_phase;
        while (!mbar_try_wait(&stage->bar, ph)) { }
        *stage_phase = ph ^ 1u;
#pragma unroll 1
        for (int i = 0; i < n1; ++i) consider(sx, sy, sz, stage->pts[sub][i], top, tau);
#pragma unroll 1
        for (int p0 = b + n1; p0 < e; p0 += BATCH) {       // a run longer than the tile: the rest through registers
            float4 c[BATCH];
#pragma unroll
            for (int i = 0; i < BATCH; ++i) if (p0 + i < e) c[i] = __ldg(map + p0 + i);
#pragma unroll
            for (int i = 0; i < BATCH; ++i) if (p0 + i < e) consider(sx, sy, sz, c[i], top, tau);
        }
    } else {
    auto row_range = [&](int row, int& b, int& e) {
        b = 0; e = 0;
        int ib, ie;
        if (row < 9 && row_cells(qc, g, (row % 3) - 1, (row / 3) - 1, tau, ib, ie)) {
            b = __ldg(cell_start + ib);
            e = __ldg(cell_start + ie);
        }
    };
    int b, e;
    row_range(sub, b, e);
    if (dbg) dbg[9] = clock64() + (long long)(b & 0);
#pragma unroll 1
    for (int row = sub; row < 9; row += LANES) {
        int nb, ne;
        row_range(row + LANES, nb, ne);          // next run's bounds are in flight while this run is ranked
        cand += (unsigned long long)(e - b);
#pragma unroll 1
        for (int p0 = b; p0 < e; p0 += BATCH) {
            float4 c[BATCH];
#pragma unroll
            for (int i = 0; i < BATCH; ++i) if (p0 + i < e) c[i] = __ldg(map + p0 + i);
#pragma unroll
            for (int i = 0; i < BATCH; ++i) if (p0 + i < e) consider(sx, sy, sz, c[i], top, tau);
        }
        b = nb; e = ne;
    }
    }
    if (dbg) dbg[10] = clock64() + (long long)(top.k0 & 0);
    // merge: 5 rounds of "group-wide minimum of the list heads, winner pops".  The minimum is an xor
    // butterfly of 64-bit keys (a hardware redux on a partial lane mask is not cheaper: it only takes
    // 32-bit operands).  Keys are unique — a map point lives in exactly one lane's list — so exactly
    // one lane pops per round.
    Top5 res;
#define LILI_MERGE_ROUND(KJ)                                                              \
    {                                                                                     \
        u64 mn = top.k0;                                                                  \
        _Pragma("unroll")                                                                 \
        for (int o = 1; o < LANES; o <<= 1) { const u64 other = __shfl_xor_sync(gmask, mn, o); mn = other < mn ? other : mn; } \
        KJ = mn;                                                                          \
        if (top.k0 == mn && mn != ~0ull) { top.k0 = top.k1; top.k1 = top.k2; top.k2 = top.k3; top.k3 = top.k4; top.k4 = ~0ull; } \
    }
    LILI_MERGE_ROUND(res.k0)
    LILI_MERGE_ROUND(res.k1)
    LILI_MERGE_ROUND(res.k2)
    LILI_MERGE_ROUND(res.k3)
    LILI_MERGE_ROUND(res.k4)
#undef LILI_MERGE_ROUND
    top = res;
}

// One thread per query (large query sets: every issue slot ranks 32 candidates; consecutive queries are spatial
// neighbours, so the warp's loads hit the same cells in L1).  Three steps:
//   1. the centre row (the query's own (y,z) row, three x-adjacent cells, ~1/3 of the block's points and nearly always
//      the five nearest among them) — after it `tau` is at or near the final fifth distance;
//   2. the eight other rows are bounded against that tau; the survivors' trimmed runs go to a per-thread list in shared
//      memory, all their cell-table loads in flight together;
//   3. ONE loop over the concatenated list.  A warp's trip count is then the maximum over its lanes of the total number of
//      batches — not the sum over rows of the per-row maxima, which costs up to twice the mean.
// `runs`: this thread's slots of a [kRunCap][run_stride] int4 array in shared memory {begin, end, bound bits, -}.
template <int BATCH1 = 8, int BATCH3 = 4>
__device__ __forceinline__ void thread_knn5(float sx, float sy, float sz, const float4* __restrict__ map,
                                            const int* __restrict__ cell_start, const GridDesc& g, float tau0, int4* runs, int run_stride,
                                            Top5& top, unsigned long long& cand) {
    const QCell qc = query_cell(sx, sy, sz, g);
    float tau = tau0;
    {   // 1. centre row
        int ib, ie, b = 0, e = 0;
        if (row_cells(qc, g, 0, 0, tau, ib, ie)) { b = __ldg(cell_start + ib); e = __ldg(cell_start + ie); }
        cand += (unsigned long long)(e - b);
#pragma unroll 1
        for (int p0 = b; p0 < e; p0 += BATCH1) {
            float4 c[BATCH1];
#pragma unroll
            for (int i = 0; i < BATCH1; ++i) if (p0 + i < e) c[i] = __ldg(map + p0 + i);
#pragma unroll
            for (int i = 0; i < BATCH1; ++i) if (p0 + i < e) consider(sx, sy, sz, c[i], top, tau);
        }
    }
    // 2. surviving rows: faces first (they hold the nearer cells), then corners; four rows' cell-table loads in flight at a time
    int nruns = 0;
#pragma unroll 1
    for (int half = 0; half < 2; ++half) {
        int rb[4], re[4];
        float bnd[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            // half 0: (oy,oz) = (-1,0) (1,0) (0,-1) (0,1)    half 1: (-1,-1) (1,-1) (-1,1) (1,1)
            const int oy = half == 0 ? (k == 0 ? -1 : k == 1 ? 1 : 0) : ((k & 1) ? 1 : -1);
            const int oz = half == 0 ? (k == 2 ? -1 : k == 3 ? 1 : 0) : (k < 2 ? -1 : 1);
            int ib, ie;
            rb[k] = 0; re[k] = 0;
            bnd[k] = cell_bound(qc, 0, oy, oz);
            if (row_cells(qc, g, oy, oz, tau, ib, ie)) { rb[k] = __ldg(cell_start + ib); re[k] = __ldg(cell_start + ie); }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (re[k] > rb[k]) { runs[nruns * run_stride] = make_int4(rb[k], re[k], __float_as_int(bnd[k]), 0); ++nruns; }
        }
    }
    // 3. one flat loop over the listed runs
    int k = 0, p = 0, e = 0;
#pragma unroll 1
    while (true) {
        if (p >= e) {
            bool have = false;
            while (k < nruns) {
                const int4 r = runs[k * run_stride];
                ++k;
                if (__int_as_float(r.z) <= tau) { p = r.x; e = r.y; have = true; break; }   // tau has shrunk since step 2
            }
            if (!have) break;
        }
        float4 c[BATCH3];
#pragma unroll
        for (int i = 0; i < BATCH3; ++i) if (p + i < e) c[i] = __ldg(map + p + i);
#pragma unroll
        for (int i = 0; i < BATCH3; ++i) if (p + i < e) consider(sx, sy, sz, c[i], top, tau);
        cand += (unsigned long long)(min(e - p, BATCH3));
        p += BATCH3;
    }
}

}  // namespace lili
