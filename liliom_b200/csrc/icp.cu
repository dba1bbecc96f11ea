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
// iteration each virtual block runs one thread per point — expanding-shell exact 1-NN over the target's cells (the 27-cell
// block first, then shells of Chebyshev radius r; the search stops once the best distance is below r-1 cells or the shell lies
// beyond the cut-off) — and reduces the 16 sums of the closed form + the count in a fixed order into its partials slot; after
// a grid barrier every block folds the partials in virtual-block order and takes the step of icp_math.h (SVD, Umeyama,
// composition, convergence) redundantly, with the same bits, so no broadcast is needed.  The final fitness pass runs in the
// same launch, and the results go straight to the context's pinned block: one stream synchronise per alignment.
#include "ctx.cuh"
#include "dev_math.cuh"
#include "knn_core.cuh"
#include "icp_math.h"
#include <cmath>

namespace lili {

constexpr int kIcpBlock = 256;    // points per virtual block = threads per block

struct IcpArgs {
    const float4* src; int n, nvb;                   // source points (float4 xyz*), virtual blocks cdiv(n, 256)
    const float4* map; const float4* map_orig; const int* cell_start; GridDesc g;
    float max_d2;                                    // squared correspondence cut-off
    int rmax, rmax_fit;                              // shells to visit at most: correspondence passes, the fitness pass
    int max_iter; double trans_eps, fit_eps;
    double* partials;                                // [2 parities][kIcpSums][nvb]
    unsigned int* bar; int sync_mode;                // grid barrier word (zeroed before the launch), LILIOM_GN_SYNC
    PinIcp* out;                                     // results (the pinned block, or device memory)
};

__device__ __forceinline__ void icp_run(const float4* __restrict__ map, int b, int e, float sx, float sy, float sz, u64& best) {
    for (int p = b; p < e; ++p) {
        const float4 m = __ldg(map + p);
        const u64 k = make_key(cand_dist(sx, sy, sz, m), m);
        best = k < best ? k : best;
    }
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
        const double px = T[0] * s.x + T[1] * s.y + T[2] * s.z + T[3];
        const double py = T[4] * s.x + T[5] * s.y + T[6] * s.z + T[7];
        const double pz = T[8] * s.x + T[9] * s.y + T[10] * s.z + T[11];
        const float sx = (float)px, sy = (float)py, sz = (float)pz;
        const GridDesc& g = a.g;
        const float cell = 1.0f / g.inv_cell;
        const int cx = cell_coord(sx, g.inv_cell) - g.org[0], cy = cell_coord(sy, g.inv_cell) - g.org[1], cz = cell_coord(sz, g.inv_cell) - g.org[2];
        const bool cut = max_d2 >= 0.f;
        u64 best = ~0ull;
#pragma unroll 1
        for (int r = 1; r <= rmax; ++r) {
            if (r >= 2) {
                // every unvisited point is at least (r-1) cells away: stop when the best is strictly closer, or the shell is out of range
                const float gap = (float)(r - 1) * cell, gap2 = gap * gap;
                if (cut && gap2 > max_d2) break;
                if (best != ~0ull && top5_dist(best) < gap2) break;
            }
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
// 0..nvb-1 into sums[] (every block).
__device__ __forceinline__ void icp_pass(const IcpArgs& a, const double* T, float max_d2, int rmax, int phase, double (*red)[kIcpSums],
                                         double* sums) {
    double* part = a.partials + (size_t)(phase & 1) * kIcpSums * a.nvb;
    for (int vb = blockIdx.x; vb < a.nvb; vb += gridDim.x) icp_vblock(a, vb, T, max_d2, rmax, part, red);
    if (a.sync_mode == 0) __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) grid_barrier(a.bar, (unsigned int)(phase + 1) * gridDim.x, a.sync_mode, true);
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

// The step of thread 0 out of line: its fp64 SVD and local arrays stay off the register budget of the search
__device__ __noinline__ int icp_step_dev(IcpState& st, const double* sums, int max_iter, double trans_eps, double fit_eps) {
    return icp_step(st, sums, max_iter, trans_eps, fit_eps);
}

// The whole alignment in one cooperative launch (grid <= co-resident blocks; any grid gives the same bits).  The partials
// alternate between two buffers by barrier parity: a block can only write phase p + 2's partials after every block has
// arrived at barrier p + 1, i.e. after every block has folded phase p's.
__global__ void __launch_bounds__(kIcpBlock) k_icp_persistent(const __grid_constant__ IcpArgs a) {
    __shared__ double red[8][kIcpSums];
    __shared__ double sums[kIcpSums];
    __shared__ double T[12];                // rows 0..2 of F, the transform of the next pass
    __shared__ int verdict;
    IcpState st;                            // thread 0's copy (the step is redundant across blocks)
    icp_init(st);
    if (threadIdx.x < 12) T[threadIdx.x] = st.F[threadIdx.x / 4][threadIdx.x % 4];
    __syncthreads();
    int phase = 0;
#pragma unroll 1
    while (true) {
        icp_pass(a, T, a.max_d2, a.rmax, phase++, red, sums);
        if (threadIdx.x == 0) {
            verdict = icp_step_dev(st, sums, a.max_iter, a.trans_eps, a.fit_eps);
            for (int k = 0; k < 12; ++k) T[k] = st.F[k / 4][k % 4];
        }
        __syncthreads();
        if (verdict != kIcpGo) break;
    }
    // getFitnessScore(): mean squared NN distance of the aligned source, no cut-off; the walk is bounded by the grid's extent
    icp_pass(a, T, -1.0f, a.rmax_fit, phase, red, sums);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        for (int k = 0; k < 16; ++k) a.out->T[k] = st.F[k / 4][k % 4];
        a.out->fitness = icp_fitness(sums);
        a.out->converged = verdict == kIcpConverged ? 1 : 0;
        a.out->iters = st.it;
        __threadfence_system();
    }
}

// src (device float4, n points) against the index `tgt`; T16 row-major 4x4 out
int icp_align(liliom_ctx* c, const MapIndex& tgt, const float4* d_src, int n, double max_corr_dist, int max_iter, double trans_eps,
              double fit_eps, double T16[16], double* fitness, int* converged, int* iters) {
    for (int k = 0; k < 16; ++k) T16[k] = (k % 5 == 0) ? 1.0 : 0.0;
    *fitness = 0.0; *converged = 0; *iters = 0;
    if (n <= 0 || tgt.n <= 0) return LILIOM_OK;
    IcpArgs a{};
    a.src = d_src; a.n = n; a.nvb = cdiv(n, kIcpBlock);
    a.map = tgt.sorted.as<float4>(); a.map_orig = tgt.xyzw.as<float4>(); a.cell_start = tgt.cell_start.as<int>(); a.g = tgt.grid;
    const float cell = 1.0f / tgt.grid.inv_cell;
    a.max_d2 = (float)(max_corr_dist * max_corr_dist);
    a.rmax = (int)std::ceil(max_corr_dist / cell) + 1;
    a.rmax_fit = std::max(tgt.grid.dim[0], std::max(tgt.grid.dim[1], tgt.grid.dim[2])) + 1;
    a.max_iter = max_iter; a.trans_eps = trans_eps; a.fit_eps = fit_eps;
    a.sync_mode = c->gn_sync;
    int per_sm = 0;
    LILI_CUDA(c, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_icp_persistent, kIcpBlock, 0));
    const int grid = std::max(1, std::min(a.nvb, per_sm * c->sm_count));
    LILI_CUDA(c, c->partials.ensure((size_t)2 * kIcpSums * a.nvb * sizeof(double)));
    LILI_CUDA(c, c->icp_ctl.ensure(64 + sizeof(PinIcp)));
    LILI_CUDA(c, cudaMemsetAsync(c->icp_ctl.p, 0, sizeof(unsigned int), c->stream));
    a.partials = c->partials.as<double>();
    a.bar = c->icp_ctl.as<unsigned int>();
    PinIcp* dev_out = reinterpret_cast<PinIcp*>(c->icp_ctl.as<unsigned char>() + 64);
    a.out = c->h_pin_dev ? &c->h_pin_dev->icp : dev_out;
    void* kargs[] = {&a};
    LILI_CUDA(c, cudaLaunchCooperativeKernel((const void*)k_icp_persistent, dim3(grid), dim3(kIcpBlock), kargs, 0, c->stream));
    LILI_TRY(launch_check(c, "k_icp_persistent"));
    if (!c->h_pin_dev) LILI_CUDA(c, cudaMemcpyAsync(&c->h_pin->icp, dev_out, sizeof(PinIcp), cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    const PinIcp& r = c->h_pin->icp;
    for (int k = 0; k < 16; ++k) T16[k] = r.T[k];
    *fitness = r.fitness;
    *converged = r.converged;
    *iters = r.iters;
    return LILIOM_OK;
}

}  // namespace lili
