// SURVEY.md §8 (f4): the loop-closure alignment of BackendFusion::performLoopClosure (L/src/BackendFusion.cpp:2552-2582) on the
// same cell grid as the scan-to-map search:
//     pcl::IterativeClosestPoint icp; setMaxCorrespondenceDistance(30); setMaximumIterations(100);
//     setTransformationEpsilon(1e-6); setEuclideanFitnessEpsilon(1e-6); setRANSACIterations(5);
//     setInputSource(latest_key_frames_ds); setInputTarget(his_key_frames_ds); align(); hasConverged(); getFitnessScore();
// from-knowledge (PCL 1.8-1.10, registration/impl/icp.hpp, default_convergence_criteria.hpp, transformation_estimation_svd.hpp):
//   per iteration: nearest target point of every (transformed) source point, kept when its squared distance is <= max^2;
//   fewer than 3 correspondences -> not converged; rigid transform by Umeyama's closed form without scale (R = U S V^T of the
//   cross-covariance, S = diag(1,1,sign det)); final = incremental * final; convergence (DefaultConvergenceCriteria, zero
//   "similar transform" iterations allowed): iteration cap -> converged; rotation cos >= 1 - eps AND |t|^2 <= eps -> converged;
//   |mse - prev| / prev < euclidean_fitness_epsilon -> converged; |mse - prev| < 1e-12 -> converged.
//   setRANSACIterations has no effect on icp.hpp's loop (no rejector is installed), so the alignment is deterministic.
//   getFitnessScore(): mean squared nearest-neighbour distance of the aligned source, no range cut.
// PCL runs this in single precision (Matrix4f, float clouds); here the transform and the sums are fp64 — parity with PCL is at
// tolerance level either way.
//
// The whole loop is ONE cooperative launch (k_icp_persistent).  The source is dealt in virtual blocks of 256 points; per
// iteration each virtual block runs one thread per point — exact 1-NN over the target's cells by expanding shells — and
// reduces the 16 sums of the closed form + the count in a fixed order into its partials slot; after a grid barrier every
// block folds the partials in virtual-block order and takes the step of icp_math.h (SVD, Umeyama, composition, convergence)
// redundantly, with the same bits, so no broadcast is needed.  The final fitness pass runs in the same launch, and the
// results go straight to the context's pinned block: one stream synchronise per alignment.
//
// The walk starts at the query's cell clamped into the grid (the 27-cell block first, then shells of Chebyshev radius r), so
// max(dim) + 1 shells reach every cell from anywhere, and the fitness pass finds a neighbour for every source point however
// far outside the target's box it lies: getFitnessScore() averages over all of them.  A point of shell r lies at least
// sqrt(out^2 + ((r-1) cell)^2) from the query, out = the query's distance to the grid's cell box (0 inside; along the shell's
// axis the point is (r-1) cells beyond the query's cell, or beyond the box face plus r - 1 cells, and along every axis at
// least `out` away).  Inside the box the fp32 value ((r-1) cell)^2 bounds every such point's fp32 distance exactly (fp32
// subtraction, multiplication and addition are monotonic); outside, the bound is shrunk by 2^-20, more than the five
// roundings of the fp32 distance can take off it.  The walk stops once the best distance is below the bound, or the bound
// is beyond the cut-off.  A correspondence is kept when (double)d <= max_corr_dist^2, PCL's test, i.e. d <= the largest float
// with that property (icp_cut_tau).
#include "ctx.cuh"
#include "dev_math.cuh"
#include "knn_core.cuh"
#include "icp_math.h"
#include <cmath>

namespace lili {

constexpr int kIcpBlock = 256;    // points per virtual block = threads per block

__device__ __forceinline__ void icp_run(const float4* __restrict__ map, int b, int e, float sx, float sy, float sz, u64& best) {
    for (int p = b; p < e; ++p) {
        const float4 m = __ldg(map + p);
        const u64 k = make_key(cand_dist(sx, sy, sz, m), m);
        best = k < best ? k : best;
    }
}

// Axis k of the query's cell, clamped into the grid (in double: no int overflow however far away v lies), and the square of v's
// distance to the grid's cell box along that axis added to out2 (0 inside)
__device__ __forceinline__ int icp_cell(float v, const GridDesc& g, float cell, int k, double& out2) {
    const double lo = (double)g.org[k] * cell, hi = ((double)g.org[k] + g.dim[k]) * cell;
    const double o = fmax(fmax(lo - v, v - hi), 0.0);
    out2 = __fma_rn(o, o, out2);
    return (int)fmin(fmax((double)floorf(v * g.inv_cell) - g.org[k], 0.0), (double)(g.dim[k] - 1));
}

// One virtual block of one pass: the 17 sums of source points vb*256 .. vb*256+255 under T (row-major 3x4), written to
// part[k * nvb + vb].  max_d2 < 0: no cut-off (fitness pass).
__device__ __forceinline__ void icp_vblock(const IcpArgs& a, int vb, const double* T, float max_d2, int rmax, double* part,
                                           double (*red)[kIcpSums]) {
    const int i = vb * kIcpBlock + threadIdx.x;
    double v[kIcpSums];
#pragma unroll
    for (int k = 0; k < kIcpSums; ++k) v[k] = 0.0;
    if (i < a.n) {
        const float4 s = a.src[i];
        // T[0] x + T[1] y + T[2] z + T[3] as the compiler contracts it (a DMUL, two DFMA, a DADD per row), spelled out so that
        // no edit of the kernel can change its rounding; tests/icp_math_host.cpp's im_transform is the same sequence
        const double px = __dadd_rn(__fma_rn(T[2], s.z, __fma_rn(T[0], s.x, __dmul_rn(T[1], s.y))), T[3]);
        const double py = __dadd_rn(__fma_rn(T[6], s.z, __fma_rn(T[4], s.x, __dmul_rn(T[5], s.y))), T[7]);
        const double pz = __dadd_rn(__fma_rn(T[10], s.z, __fma_rn(T[8], s.x, __dmul_rn(T[9], s.y))), T[11]);
        const float sx = (float)px, sy = (float)py, sz = (float)pz;
        const GridDesc& g = a.g;
        const float cell = 1.0f / g.inv_cell;
        double out2 = 0.0;
        const int cx = icp_cell(sx, g, cell, 0, out2), cy = icp_cell(sy, g, cell, 1, out2), cz = icp_cell(sz, g, cell, 2, out2);
        const bool cut = max_d2 >= 0.f;
        u64 best = ~0ull;
#pragma unroll 1
        for (int r = 1; r <= rmax; ++r) {
            // every unvisited point is at least sqrt(out2 + gap^2) away (see the header): stop when the best is strictly closer,
            // or the bound is beyond the cut-off
            const float gap = (float)(r - 1) * cell, gap2 = gap * gap;
            const float lb = out2 == 0.0 ? gap2 : __double2float_rd(__dmul_rn(__dadd_rn(out2, (double)gap2), 1.0 - 0x1p-20));
            if (cut && lb > max_d2) break;
            if (best != ~0ull && top5_dist(best) < lb) break;
            const int z0 = max(cz - r, 0), z1 = min(cz + r, g.dim[2] - 1), y0 = max(cy - r, 0), y1 = min(cy + r, g.dim[1] - 1);
            for (int z = z0; z <= z1; ++z) {
                for (int y = y0; y <= y1; ++y) {
                    const int base = (z * g.dim[1] + y) * g.dim[0];
                    if (r == 1 || abs(z - cz) == r || abs(y - cy) == r) {      // the whole x-stretch (r == 1: the 27-cell block) is one run
                        const int x0 = max(cx - r, 0), x1 = min(cx + r, g.dim[0] - 1);
                        if (x0 <= x1) icp_run(a.map, __ldg(a.cell_start + base + x0), __ldg(a.cell_start + base + x1 + 1), sx, sy, sz, best);
                    } else {                                                     // interior row of the shell: its two end cells
                        const int xa = cx - r, xb = cx + r;
                        if (xa >= 0 && xa < g.dim[0]) icp_run(a.map, __ldg(a.cell_start + base + xa), __ldg(a.cell_start + base + xa + 1), sx, sy, sz, best);
                        if (xb >= 0 && xb < g.dim[0]) icp_run(a.map, __ldg(a.cell_start + base + xb), __ldg(a.cell_start + base + xb + 1), sx, sy, sz, best);
                    }
                }
            }
        }
        if (best != ~0ull && (!cut || top5_dist(best) <= max_d2)) {
            const float4 q = __ldg(a.map_orig + top5_index(best));
            v[0] = px; v[1] = py; v[2] = pz;
            v[3] = q.x; v[4] = q.y; v[5] = q.z;
            v[6] = px * q.x; v[7] = px * q.y; v[8] = px * q.z;
            v[9] = py * q.x; v[10] = py * q.y; v[11] = py * q.z;
            v[12] = pz * q.x; v[13] = pz * q.y; v[14] = pz * q.z;
            v[15] = (double)top5_dist(best); v[16] = 1.0;
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kIcpSums; ++k) {
        double s = v[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) red[warp][k] = s;
    }
    __syncthreads();
    if (threadIdx.x < kIcpSums) {
        double s = 0.0;
        for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
        part[(size_t)threadIdx.x * a.nvb + vb] = s;
    }
    __syncthreads();      // red is reused by the block's next virtual block
}

// One pass over every virtual block under T, the grid barrier `phase`, and the fold of the partials in virtual-block order
// 0..nvb-1 into sums[] (every block).  blk: the block's place among its session's blocks (ctx.cuh).
template <class Blk>
__device__ __forceinline__ void icp_pass(const IcpArgs& a, const double* T, float max_d2, int rmax, int phase, double (*red)[kIcpSums],
                                         double* sums, const Blk blk) {
    double* part = a.partials + (size_t)(phase & 1) * kIcpSums * a.nvb;
    for (int vb = blk.bi(); vb < a.nvb; vb += blk.G()) icp_vblock(a, vb, T, max_d2, rmax, part, red);
    // grid_barrier spelled out: thread 0 computes the target after the first block barrier (as an argument of grid_barrier it
    // would be computed before it, and the kernel would take one register more)
    __syncthreads();
    if (threadIdx.x == 0) grid_arrive<kReleaseOnly>(a.bar, (unsigned int)(phase + 1) * blk.G(), true);
    __syncthreads();
    if (threadIdx.x < kIcpSums) {
        const double* p = part + (size_t)threadIdx.x * a.nvb;
        double s = 0.0;
#pragma unroll 8
        for (int b = 0; b < a.nvb; ++b) s = addx(s, __ldcg(p + b));
        sums[threadIdx.x] = s;
    }
    __syncthreads();
}

// The step of thread 0 out of line: its fp64 SVD and local arrays stay off the register budget of the search.  One copy per
// kernel (Blk): ptxas allocates the registers of a function with a single caller around that caller.
template <class Blk>
__device__ __noinline__ int icp_step_dev(IcpState& st, const double* sums, int max_iter, double trans_eps, double fit_eps) {
    return icp_step(st, sums, max_iter, trans_eps, fit_eps);
}

// The whole alignment in one cooperative launch (grid <= co-resident blocks; any grid gives the same bits).  The partials
// alternate between two buffers by barrier parity: a block can only write phase p + 2's partials after every block has
// arrived at barrier p + 1, i.e. after every block has folded phase p's.
// The kernels declare the shared arrays (k_icp_persistent keeps its shared-memory layout): red[8][kIcpSums], sums[kIcpSums],
// T[12] (rows 0..2 of F, the transform of the next pass), verdict.
template <class Blk>
__device__ __forceinline__ void icp_body(const IcpArgs& a, const Blk blk, double (*red)[kIcpSums], double* sums, double* T, int& verdict) {
    IcpState st;                            // thread 0's copy (the step is redundant across blocks)
    icp_init(st);
    if (threadIdx.x < 12) T[threadIdx.x] = st.F[threadIdx.x / 4][threadIdx.x % 4];
    __syncthreads();
    int phase = 0;
#pragma unroll 1
    while (true) {
        icp_pass(a, T, a.max_d2, a.rmax, phase++, red, sums, blk);
        if (threadIdx.x == 0) {
            verdict = icp_step_dev<Blk>(st, sums, a.max_iter, a.trans_eps, a.fit_eps);
            for (int k = 0; k < 12; ++k) T[k] = st.F[k / 4][k % 4];
        }
        __syncthreads();
        if (verdict != kIcpGo) break;
    }
    // getFitnessScore(): mean squared NN distance of every point of the aligned source, no cut-off
    icp_pass(a, T, -1.0f, a.rmax_fit, phase, red, sums, blk);
    if (blk.bi() == 0 && threadIdx.x == 0) {
        for (int k = 0; k < 16; ++k) a.out->T[k] = st.F[k / 4][k % 4];
        a.out->fitness = icp_fitness(sums);
        a.out->converged = verdict == kIcpConverged ? 1 : 0;
        a.out->iters = st.it;
        __threadfence_system();
    }
}

__global__ void __launch_bounds__(kIcpBlock) k_icp_persistent(const __grid_constant__ IcpArgs a) {
    __shared__ double red[8][kIcpSums];
    __shared__ double sums[kIcpSums];
    __shared__ double T[12];
    __shared__ int verdict;
    icp_body(a, SoloBlock{}, red, sums, T, verdict);
}

// Several sessions' alignments in one cooperative launch (liliom_loop_align_batch).  Session s owns blocks [off[s], off[s+1])
// and runs exactly the body of its solo launch, with its own barrier word, partials and results; the cooperative launch only
// guarantees that all blocks are resident.  The sessions meet no common barrier, so each ends after its own iterations.
__global__ void __launch_bounds__(kIcpBlock, 1) k_icp_batch(const __grid_constant__ BatchTab<IcpArgs> tab) {
    __shared__ double red[8][kIcpSums];
    __shared__ double sums[kIcpSums];
    __shared__ double T[12];
    __shared__ int verdict;
    const BatchSlot at = batch_slot(tab);
    icp_body(tab.s[at.s], at.blk, red, sums, T, verdict);
}

// Largest float t with (double)t <= max_sqd: "d <= t" is then PCL's correspondence test, which rejects (double)d > max_dist_sqr
// (knn_gate_tau's search with <= for <)
static float icp_cut_tau(double max_sqd) {
    float f = (float)max_sqd;
    while ((double)f > max_sqd) f = nextafterf(f, -INFINITY);
    return f;
}

int icp_begin(liliom_ctx* c, const MapIndex& tgt, const float4* d_src, int n, double max_corr_dist, int max_iter, double trans_eps,
              double fit_eps, IcpJob& j) {
    j = IcpJob{};
    j.c = c;
    if (n <= 0 || tgt.n <= 0) { j.done = true; return LILIOM_OK; }
    IcpArgs& a = j.a;
    a.src = d_src; a.n = n; a.nvb = cdiv(n, kIcpBlock);
    a.map = tgt.sorted.as<float4>(); a.map_orig = tgt.xyzw.as<float4>(); a.cell_start = tgt.cell_start.as<int>(); a.g = tgt.grid;
    const float cell = 1.0f / tgt.grid.inv_cell;
    a.max_d2 = icp_cut_tau(max_corr_dist * max_corr_dist);
    a.rmax_fit = std::max(tgt.grid.dim[0], std::max(tgt.grid.dim[1], tgt.grid.dim[2])) + 1;
    a.rmax = (int)std::min(std::ceil(max_corr_dist / cell) + 1.0, (double)a.rmax_fit);
    a.max_iter = max_iter; a.trans_eps = trans_eps; a.fit_eps = fit_eps;
    int per_sm = 0;
    LILI_CUDA(c, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_icp_persistent, kIcpBlock, 0));
    j.grid = std::max(1, std::min(a.nvb, per_sm * c->sm_count));
    LILI_CUDA(c, c->partials.ensure((size_t)2 * kIcpSums * a.nvb * sizeof(double)));
    LILI_CUDA(c, c->icp_ctl.ensure(64 + sizeof(PinIcp)));
    LILI_CUDA(c, cudaMemsetAsync(c->icp_ctl.p, 0, sizeof(unsigned int), c->stream));
    a.partials = c->partials.as<double>();
    a.bar = c->icp_ctl.as<unsigned int>();
    j.dev_out = reinterpret_cast<PinIcp*>(c->icp_ctl.as<unsigned char>() + 64);
    a.out = c->h_pin_dev ? &c->h_pin_dev->icp : j.dev_out;
    return LILIOM_OK;
}

int icp_launch(const IcpJob& j) {
    liliom_ctx* c = j.c;
    IcpArgs a = j.a;
    void* kargs[] = {&a};
    LILI_CUDA(c, cudaLaunchCooperativeKernel((const void*)k_icp_persistent, dim3(j.grid), dim3(kIcpBlock), kargs, 0, c->stream));
    return launch_check(c, "k_icp_persistent");
}

int icp_fetch(const IcpJob& j) {
    liliom_ctx* c = j.c;
    if (!c->h_pin_dev) LILI_CUDA(c, cudaMemcpyAsync(&c->h_pin->icp, j.dev_out, sizeof(PinIcp), cudaMemcpyDeviceToHost, c->stream));
    return LILIOM_OK;
}

void icp_finish(const IcpJob& j, double T16[16], double* fitness, int* converged, int* iters) {
    for (int k = 0; k < 16; ++k) T16[k] = (k % 5 == 0) ? 1.0 : 0.0;
    *fitness = 0.0; *converged = 0; *iters = 0;
    if (j.done) return;
    const PinIcp& r = j.c->h_pin->icp;
    for (int k = 0; k < 16; ++k) T16[k] = r.T[k];
    *fitness = r.fitness;
    *converged = r.converged;
    *iters = r.iters;
}

// src (device float4, n points) against the index `tgt`; T16 row-major 4x4 out
int icp_align(liliom_ctx* c, const MapIndex& tgt, const float4* d_src, int n, double max_corr_dist, int max_iter, double trans_eps,
              double fit_eps, double T16[16], double* fitness, int* converged, int* iters) {
    IcpJob j;
    j.done = true;
    icp_finish(j, T16, fitness, converged, iters);      // identity until the results are in
    LILI_TRY(icp_begin(c, tgt, d_src, n, max_corr_dist, max_iter, trans_eps, fit_eps, j));
    if (!j.done) {
        LILI_TRY(icp_launch(j));
        LILI_TRY(icp_fetch(j));
        LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    }
    icp_finish(j, T16, fitness, converged, iters);
    return LILIOM_OK;
}

int icp_batch_launch(liliom_ctx* c0, const std::vector<IcpJob*>& jobs) {
    if (jobs.empty()) return LILIOM_OK;
    int occ = 0;
    LILI_CUDA(c0, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_icp_batch, kIcpBlock, 0));
    std::vector<BatchItem> items;
    for (const IcpJob* j : jobs) {
        const int cap = j->c->test_icp_blocks;
        items.push_back(BatchItem{cap > 0 ? std::min(cap, j->grid) : j->grid, 0, true});
    }
    const BatchPack pack = batch_pack(items, &occ, c0->sm_count);
    for (const BatchLaunch& l : pack.launches)
        LILI_TRY(batch_tables<BatchTab<IcpArgs>>(l.sessions, [&](IcpArgs& e, int s) {
            e = jobs[s]->a;
            return BatchPart{jobs[s]->c, items[s].grid};
        }, [&](BatchTab<IcpArgs>& tab, int grid) -> int {
            void* kargs[] = {&tab};
            LILI_CUDA(c0, cudaLaunchCooperativeKernel((const void*)k_icp_batch, dim3(grid), dim3(kIcpBlock), kargs, 0, c0->stream));
            LILI_CUDA(c0, cudaGetLastError());
            return LILIOM_OK;
        }));
    for (int s : pack.solo) LILI_TRY(icp_launch(*jobs[s]));
    for (const IcpJob* j : jobs) LILI_TRY(icp_fetch(*j));
    return LILIOM_OK;
}

}  // namespace lili
