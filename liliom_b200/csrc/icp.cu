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
// One thread per source point: expanding-shell exact 1-NN over the target's 1 m cells (the 27-cell block first, then shells of
// Chebyshev radius r; the search stops once the best distance is below r-1 cells or the shell lies beyond the cut-off), the 16
// sums of the closed form + the count reduced per block in a fixed order, the 3x3 SVD on the host (one-sided Jacobi).
#include "ctx.cuh"
#include "dev_math.cuh"
#include "knn_core.cuh"
#include <cmath>
#include <vector>

namespace lili {

constexpr int kIcpSums = 17;      // sum p (3), sum q (3), sum p q^T (9, row = p, col = q), sum d2, count

struct IcpArgs {
    const float4* src; int n;                       // source points (float4 xyz*)
    const float4* map; const float4* map_orig; const int* cell_start; GridDesc g;
    double T[12];                                    // current source -> target transform, row-major 3x4
    float max_d2;                                    // squared correspondence cut-off (<0: none, fitness pass)
    int rmax;                                        // shells to visit at most
    double* partials;                                // [kIcpSums][gridDim.x]
};

__device__ __forceinline__ void icp_run(const float4* __restrict__ map, int b, int e, float sx, float sy, float sz, u64& best) {
    for (int p = b; p < e; ++p) {
        const float4 m = __ldg(map + p);
        const u64 k = make_key(cand_dist(sx, sy, sz, m), m);
        best = k < best ? k : best;
    }
}

__global__ void __launch_bounds__(256) k_icp_pass(IcpArgs a) {
    __shared__ double red[8][kIcpSums];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    double v[kIcpSums];
#pragma unroll
    for (int k = 0; k < kIcpSums; ++k) v[k] = 0.0;
    if (i < a.n) {
        const float4 s = a.src[i];
        const double px = a.T[0] * s.x + a.T[1] * s.y + a.T[2] * s.z + a.T[3];
        const double py = a.T[4] * s.x + a.T[5] * s.y + a.T[6] * s.z + a.T[7];
        const double pz = a.T[8] * s.x + a.T[9] * s.y + a.T[10] * s.z + a.T[11];
        const float sx = (float)px, sy = (float)py, sz = (float)pz;
        const GridDesc& g = a.g;
        const float cell = 1.0f / g.inv_cell;
        const int cx = cell_coord(sx, g.inv_cell) - g.org[0], cy = cell_coord(sy, g.inv_cell) - g.org[1], cz = cell_coord(sz, g.inv_cell) - g.org[2];
        const bool cut = a.max_d2 >= 0.f;
        u64 best = ~0ull;
#pragma unroll 1
        for (int r = 1; r <= a.rmax; ++r) {
            if (r >= 2) {
                // every unvisited point is at least (r-1) cells away: stop when the best is strictly closer, or the shell is out of range
                const float gap = (float)(r - 1) * cell, gap2 = gap * gap;
                if (cut && gap2 > a.max_d2) break;
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
        if (best != ~0ull && (!cut || top5_dist(best) <= a.max_d2)) {
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
        a.partials[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = s;
    }
}

// ---- host side: 3x3 SVD by one-sided Jacobi (Hestenes), A = U diag(s) V^T
static void svd3(const double A[3][3], double U[3][3], double s[3], double V[3][3]) {
    double B[3][3];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { B[i][j] = A[i][j]; V[i][j] = i == j ? 1.0 : 0.0; }
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                double alpha = 0, beta = 0, gamma = 0;
                for (int i = 0; i < 3; ++i) { alpha += B[i][p] * B[i][p]; beta += B[i][q] * B[i][q]; gamma += B[i][p] * B[i][q]; }
                off = std::fmax(off, std::fabs(gamma) / std::sqrt(alpha * beta + 1e-300));
                if (std::fabs(gamma) < 1e-300) continue;
                const double zeta = (beta - alpha) / (2.0 * gamma);
                const double t = (zeta >= 0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / std::sqrt(1.0 + t * t), sn = c * t;
                for (int i = 0; i < 3; ++i) {
                    const double bp = B[i][p], bq = B[i][q];
                    B[i][p] = c * bp - sn * bq; B[i][q] = sn * bp + c * bq;
                    const double vp = V[i][p], vq = V[i][q];
                    V[i][p] = c * vp - sn * vq; V[i][q] = sn * vp + c * vq;
                }
            }
        if (off < 1e-15) break;
    }
    for (int j = 0; j < 3; ++j) {
        s[j] = std::sqrt(B[0][j] * B[0][j] + B[1][j] * B[1][j] + B[2][j] * B[2][j]);
        for (int i = 0; i < 3; ++i) U[i][j] = s[j] > 1e-300 ? B[i][j] / s[j] : 0.0;
    }
    // a zero singular value leaves a zero column in U: complete it to an orthonormal basis (cross product of the other two)
    for (int j = 0; j < 3; ++j) {
        if (s[j] > 1e-300) continue;
        const int a = (j + 1) % 3, b = (j + 2) % 3;
        U[0][j] = U[1][a] * U[2][b] - U[2][a] * U[1][b];
        U[1][j] = U[2][a] * U[0][b] - U[0][a] * U[2][b];
        U[2][j] = U[0][a] * U[1][b] - U[1][a] * U[0][b];
    }
}
static double det3(const double M[3][3]) {
    return M[0][0] * (M[1][1] * M[2][2] - M[1][2] * M[2][1]) - M[0][1] * (M[1][0] * M[2][2] - M[1][2] * M[2][0]) + M[0][2] * (M[1][0] * M[2][1] - M[1][1] * M[2][0]);
}

static int icp_pass(liliom_ctx* c, IcpArgs& a, int grid, double sums[kIcpSums]) {
    k_icp_pass<<<grid, 256, 0, c->stream>>>(a);
    LILI_TRY(launch_check(c, "k_icp_pass"));
    std::vector<double> h((size_t)kIcpSums * grid);
    LILI_CUDA(c, cudaMemcpyAsync(h.data(), a.partials, h.size() * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    for (int k = 0; k < kIcpSums; ++k) { double s = 0.0; for (int b = 0; b < grid; ++b) s += h[(size_t)k * grid + b]; sums[k] = s; }      // fixed order
    return LILIOM_OK;
}

// src (device float4, n points) against the map installed in c; T16 row-major 4x4 out
int icp_align(liliom_ctx* c, const float4* d_src, int n, double max_corr_dist, int max_iter, double trans_eps, double fit_eps,
              double T16[16], double* fitness, int* converged, int* iters) {
    for (int k = 0; k < 16; ++k) T16[k] = (k % 5 == 0) ? 1.0 : 0.0;
    *fitness = 0.0; *converged = 0; *iters = 0;
    if (n <= 0 || c->map.n <= 0) return LILIOM_OK;
    const int grid = cdiv(n, 256);
    LILI_CUDA(c, c->partials.ensure((size_t)kIcpSums * grid * sizeof(double)));
    IcpArgs a{};
    a.src = d_src; a.n = n; a.map = c->map.sorted.as<float4>(); a.map_orig = c->map.xyzw.as<float4>(); a.cell_start = c->map.cell_start.as<int>(); a.g = c->map.grid;
    a.partials = c->partials.as<double>();
    const float cell = 1.0f / c->map.grid.inv_cell;
    a.max_d2 = (float)(max_corr_dist * max_corr_dist);
    a.rmax = (int)std::ceil(max_corr_dist / cell) + 1;
    double F[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
    double prev_mse = std::numeric_limits<double>::max();
    int it = 0;
    bool conv = false;
    while (true) {
        for (int r = 0; r < 3; ++r) for (int k = 0; k < 4; ++k) a.T[4 * r + k] = F[r][k];
        double s[kIcpSums];
        LILI_TRY(icp_pass(c, a, grid, s));
        const double cnt = s[16];
        if (cnt < 3.0) { conv = false; break; }                       // icp.hpp: "Not enough correspondences found"
        // Umeyama without scale on the matched pairs (p = transformed source, q = target)
        const double mp[3] = {s[0] / cnt, s[1] / cnt, s[2] / cnt}, mq[3] = {s[3] / cnt, s[4] / cnt, s[5] / cnt};
        double Sg[3][3];                                              // sigma = 1/n sum (q - mq)(p - mp)^T  (dst x src^T)
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Sg[i][j] = s[6 + 3 * j + i] / cnt - mq[i] * mp[j];
        double U[3][3], sv[3], V[3][3];
        svd3(Sg, U, sv, V);
        const double sgn = det3(U) * det3(V) < 0 ? -1.0 : 1.0;
        // the reflection fix belongs to the SMALLEST singular value (Eigen sorts them descending and flips the last)
        int jmin = 0;
        for (int j = 1; j < 3; ++j) if (sv[j] < sv[jmin]) jmin = j;
        double R[3][3];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
            double acc = 0.0;
            for (int k = 0; k < 3; ++k) acc += U[i][k] * (k == jmin ? sgn : 1.0) * V[j][k];
            R[i][j] = acc;
        }
        double t[3];
        for (int i = 0; i < 3; ++i) t[i] = mq[i] - (R[i][0] * mp[0] + R[i][1] * mp[1] + R[i][2] * mp[2]);
        double N[4][4] = {{0}};                                       // final = incremental * final
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 4; ++j) N[i][j] = R[i][0] * F[0][j] + R[i][1] * F[1][j] + R[i][2] * F[2][j] + (j == 3 ? t[i] : 0.0);
        }
        N[3][3] = 1.0;
        memcpy(F, N, sizeof(F));
        ++it;
        // DefaultConvergenceCriteria::hasConverged (max_iterations_similar_transforms_ = 0)
        const double mse = s[15] / cnt;
        if (it >= max_iter) { conv = true; break; }
        const double cos_angle = 0.5 * (R[0][0] + R[1][1] + R[2][2] - 1.0);
        const double tr2 = t[0] * t[0] + t[1] * t[1] + t[2] * t[2];
        if (cos_angle >= 1.0 - trans_eps && tr2 <= trans_eps) { conv = true; break; }
        if (std::fabs(mse - prev_mse) / prev_mse < fit_eps) { conv = true; break; }
        if (std::fabs(mse - prev_mse) < 1e-12) { conv = true; break; }
        prev_mse = mse;
    }
    // getFitnessScore(): mean squared NN distance of the aligned source, no cut-off
    for (int r = 0; r < 3; ++r) for (int k = 0; k < 4; ++k) a.T[4 * r + k] = F[r][k];
    a.max_d2 = -1.0f;
    a.rmax = std::max(c->map.grid.dim[0], std::max(c->map.grid.dim[1], c->map.grid.dim[2])) + 1;
    {   // sources far outside the grid would walk many empty shells: bound the walk by the distance to the grid plus its extent
        double s[kIcpSums];
        LILI_TRY(icp_pass(c, a, grid, s));
        *fitness = s[16] > 0 ? s[15] / s[16] : std::numeric_limits<double>::max();
    }
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) T16[4 * i + j] = F[i][j];
    *converged = conv ? 1 : 0;
    *iters = it;
    return LILIOM_OK;
}

}  // namespace lili
