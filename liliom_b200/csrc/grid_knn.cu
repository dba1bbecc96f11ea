// Scan-to-map on sm_90a: dense 1 m cell grid over the down-sampled map (stand-in for the
// per-scan FLANN kd-tree, L/src/LidarOdometry.cpp:490) and the fused
//   transform -> exact 5-NN -> 5x3 QR plane -> gates -> residual + SE(3) Jacobian row ->
//   Huber -> 21+6 reduction -> 6x6 solve -> pose update
// kernel replacing findCorrespondingSurfFeatures + the Ceres problem/solve
// (L/src/LidarOdometry.cpp:352-413, 506-561; L/include/factors/LidarKeyframeFactor.h:111-139).
//
// HBM-bound integer/float gather work: no dense contraction, so no tensor cores.  Design:
//   * map points stored as float4 {x,y,z,orig_index} sorted by cell id (z,y,x order) so the
//     3 x-adjacent cells of a row are ONE contiguous run: 9 coalesced runs per query;
//   * 8 lanes ("octet") cooperate on one query: lanes stride through each run with 16-byte
//     loads, keep a private sorted top-5 in registers, then merge with 3 xor-shuffles;
//   * a warp finishes 4*R queries, parks the 5 neighbour slots in shared memory, and then every
//     lane runs the fp64 plane fit / Jacobian of a DIFFERENT query (no redundant fp64 issue);
//   * 29 fp64 partial sums per block -> fixed-order cross-block sum by the last block (ticket),
//     which also solves the 6x6 system and updates the pose in HBM: one launch per iteration,
//     the pose never visits the host inside the loop, results are run-to-run deterministic.
// Exactness: a query's cell block covers its full `cell`-metre ball and cells are aligned to
// the integer lattice (floorf(x * 2^-k) is exact), so any point outside the 27 cells is at
// fp32 distance >= cell >= sqrt(knn_max_sqdist): the accepted 5-NN sets equal the kd-tree's.
#include "ctx.cuh"
#include "dev_math.cuh"
#include "knn_core.cuh"

namespace lili {

// ------------------------------------------------------------------ small utilities
__global__ void k_repack_f4(const unsigned char* __restrict__ in, int n_max, const int* __restrict__ d_n, int stride, float4* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = d_n ? min(*d_n, n_max) : n_max;
    if (i >= n) return;
    float4 v = *reinterpret_cast<const float4*>(in + (size_t)i * stride);
    v.w = __int_as_float(i);
    out[i] = v;
}

int repack_to_f4(liliom_ctx* c, const void* d_in, int n, int stride, float4* d_out, const int* d_n) {
    if (n <= 0) return LILIOM_OK;
    k_repack_f4<<<cdiv(n, 256), 256, 0, c->stream>>>((const unsigned char*)d_in, n, d_n, stride, d_out);
    return launch_check(c, "k_repack_f4");
}

// `escaped` (optional): set when a point lies outside the grid's box — only possible when the box was handed in by the caller
// (grid_build's host_box); the key is then clamped into range for memory safety and the caller rebuilds with the exact box.
__global__ void k_cell_keys(const float4* __restrict__ p, int n, GridDesc g, uint32_t* __restrict__ keys, int* __restrict__ vals,
                            int* __restrict__ escaped) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float4 v = p[i];
    int cx = cell_coord(v.x, g.inv_cell) - g.org[0];
    int cy = cell_coord(v.y, g.inv_cell) - g.org[1];
    int cz = cell_coord(v.z, g.inv_cell) - g.org[2];
    if (escaped && ((unsigned)cx >= (unsigned)g.dim[0] || (unsigned)cy >= (unsigned)g.dim[1] || (unsigned)cz >= (unsigned)g.dim[2])) {
        *escaped = 1;
        cx = min(max(cx, 0), g.dim[0] - 1); cy = min(max(cy, 0), g.dim[1] - 1); cz = min(max(cz, 0), g.dim[2] - 1);
    }
    keys[i] = (uint32_t)((cz * g.dim[1] + cy) * g.dim[0] + cx);
    vals[i] = i;
}

__global__ void k_gather_sorted(const float4* __restrict__ p, const int* __restrict__ vals, int n, float4* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int src = vals[i];
    float4 v = p[src];
    out[i] = make_float4(v.x, v.y, v.z, __int_as_float(src));   // w = index into the un-sorted map array
}

// cell_start[c] = first sorted position whose key >= c = number of points with key < c = upper bound of cell c-1.
// Run ENDS are scattered (cell_start[key+1] = position after the run) into a zeroed table and a running maximum fills the
// empty cells: two streaming passes over the table.  (Filling every gap with one warp per sorted position is an order of
// magnitude slower on a 10 M-point map.)
__global__ void k_cell_run_ends(const uint32_t* __restrict__ keys, int n, int* __restrict__ cell_start) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= n) return;
    const uint32_t k = keys[w];
    if (w == n - 1 || keys[w + 1] != k) cell_start[(size_t)k + 1] = w + 1;
}

int grid_build(liliom_ctx* c, MapIndex& mi, float cell, int m, const int* host_box) {
    mi.ready = false;
    mi.n = m;
    if (m <= 0) {   // empty (shard of the) map: a 1-cell grid with no points, so that collective callers still run every launch
        GridDesc g{};
        g.inv_cell = 1.0f; g.dim[0] = g.dim[1] = g.dim[2] = 1; g.ncells = 1;
        mi.grid = g;
        LILI_CUDA(c, mi.cell_start.ensure(4 * sizeof(int)));
        LILI_CUDA(c, cudaMemsetAsync(mi.cell_start.p, 0, 4 * sizeof(int), c->stream));
        LILI_CUDA(c, mi.sorted.ensure(sizeof(float4)));
        LILI_CUDA(c, mi.xyzw.ensure(sizeof(float4)));
        mi.n = 0;
        mi.ready = true;
        return LILIOM_OK;
    }
    float4* pts = mi.xyzw.as<float4>();
    int h[6];
    // A box handed in by the caller contains the raw points.  A voxel centroid (a sequential fp32 mean of such points) can leave
    // it by rounding, in which case its cell may not exist: k_cell_keys reports that, and the grid is rebuilt from the exact
    // min/max below.  (One cell of padding instead would be free of the re-run but can push the cell count over a power of
    // 256 and cost every rebuild a whole extra radix pass: 2^24 -> 17.7 M cells on the 10 M-point bench map, +90 us.)
    int* escaped = nullptr;
    if (host_box) {
        for (int k = 0; k < 6; ++k) h[k] = host_box[k];
        if (c->test_shrink_box) h[3] = h[0];      // test hook: a box that is too small in x -> the escape path below must run
        LILI_CUDA(c, c->vg_minmax.ensure(8 * sizeof(int)));
        escaped = c->vg_minmax.as<int>() + 7;
        LILI_CUDA(c, cudaMemsetAsync(escaped, 0, sizeof(int), c->stream));
    } else {
        LILI_TRY(vg_minmax_dev(c, pts, m, nullptr, sizeof(float4)));
        int hb[kBoxInts];
        LILI_TRY(read_back(c, {{hb, c->vg_minmax.p, sizeof(hb)}}));
        if (hb[6] < m) { c->last_error = "non-finite map point"; return LILIOM_E_ARG; }      // the box counts finite points only
        for (int k = 0; k < 6; ++k) h[k] = hb[k];
    }
    GridDesc g;
    g.inv_cell = 1.0f / cell;
    long long nc = 1;
    for (int k = 0; k < 3; ++k) {
        float lo = vg_ord2f(h[k]), hi = vg_ord2f(h[3 + k]);
        int clo = (int)floorf(lo * g.inv_cell), chi = (int)floorf(hi * g.inv_cell);
        g.org[k] = clo;
        g.dim[k] = chi - clo + 1;
        nc *= g.dim[k];
    }
    if (nc > (1LL << 29)) { c->last_error = "map extent needs more than 2^29 cells"; return LILIOM_E_GRID; }
    g.ncells = (int)nc;
    mi.grid = g;
    LILI_CUDA(c, c->grid_keys.ensure((size_t)m * 4));
    LILI_CUDA(c, c->grid_keys2.ensure((size_t)m * 4));
    LILI_CUDA(c, c->grid_vals.ensure((size_t)m * 4));
    LILI_CUDA(c, c->grid_vals2.ensure((size_t)m * 4));
    LILI_CUDA(c, mi.sorted.ensure((size_t)m * sizeof(float4)));
    LILI_CUDA(c, mi.cell_start.ensure(((size_t)g.ncells + 2) * 4));
    k_cell_keys<<<cdiv(m, 256), 256, 0, c->stream>>>(pts, m, g, c->grid_keys.as<uint32_t>(), c->grid_vals.as<int>(), escaped);
    LILI_TRY(launch_check(c, "k_cell_keys"));
    int bits = 1;
    while ((1LL << bits) < nc) ++bits;
    LILI_TRY(sort_pairs_u32(c, c->grid_keys.as<uint32_t>(), c->grid_keys2.as<uint32_t>(), c->grid_vals.as<int>(),
                            c->grid_vals2.as<int>(), m, bits));
    k_gather_sorted<<<cdiv(m, 256), 256, 0, c->stream>>>(pts, c->grid_vals2.as<int>(), m, mi.sorted.as<float4>());
    LILI_TRY(launch_check(c, "k_gather_sorted"));
    LILI_CUDA(c, cudaMemsetAsync(mi.cell_start.p, 0, ((size_t)g.ncells + 2) * 4, c->stream));
    k_cell_run_ends<<<cdiv(m, 256), 256, 0, c->stream>>>(c->grid_keys2.as<uint32_t>(), m, mi.cell_start.as<int>());
    LILI_TRY(launch_check(c, "k_cell_run_ends"));
    LILI_TRY(inclusive_max_scan_i32(c, mi.cell_start.as<int>(), g.ncells + 1));
    if (escaped) {
        int esc = 0;
        LILI_TRY(read_back(c, {{&esc, escaped, sizeof(int)}}));
        if (esc) return grid_build(c, mi, cell, m, nullptr);
    }
    mi.ready = true;
    return LILIOM_OK;
}

// ------------------------------------------------------------------ the hot kernel
struct KnnArgs {
    const float4* feats; int n; const int* n_dev;   // n = host upper bound, n_dev = optional device-side count
    const float4* map; const float4* map_orig; const int* cell_start; GridDesc g;   // cell-sorted / download-order map
    const double* pose;                 // 7 doubles in HBM: the per-pass kernel's start pose
    double max_sqd, plane_thres, w_gate, huber_a;
    unsigned char* valid; float4* plane; int* nn_idx; float* nn_sqd;   // optional outputs
    double* partials; double* neq;
    double* pose_out;                   // where the updated pose goes (== pose for GN)
    unsigned long long* cand_total;     // instrumentation
    int rounds;                         // a warp handles (32/LANES)*rounds queries per task
    int nranks, rank;                   // multi-GPU ownership filter (16 m block hash)
    long long* dbg;                     // optional phase timestamps (LILIOM_DEBUG_TIMING)
    float tau0;                         // largest fp32 distance inside the gate (knn_gate_tau(max_sqd)): search pruning threshold
    float4* qstate;                     // per query {transformed position, fifth distance} of the previous pass of this call (see coherence_tau)
    float inv_block;                    // 1 / shard block edge (multi-GPU ownership)
    unsigned long long* queries_total;  // instrumentation: queries processed (device-side count), one add per pass
};

// What only the per-pass kernel (k_knn_plane) reads.
struct PassArgs {
    unsigned int* ticket;               // last-block ticket
    double* stats;                      // this iteration's stats row (kStatsDoubles) or null
    int update_pose;                    // 1: the last block performs the GN step
    int use_state;                      // 1: qstate holds the previous pass of this call
};

// Small scans (8 or 16 lanes per query) deal tasks to warps block-cyclically: queries arrive in voxel order (spatially sorted),
// and dealing neighbouring tasks to different blocks evens out the per-block work (dense vs sparse regions) at the grid barrier;
// large scans keep neighbours together for L1 reuse.
template <int LANES> __device__ __forceinline__ int first_task(int warp) {
    return LANES >= 8 ? warp * (int)gridDim.x + (int)blockIdx.x : (int)blockIdx.x * kWarps + warp; }

// per-thread instrumentation word: examined candidates in the low 40 bits, searched queries above (summed per block)
constexpr int kCandBits = 40;
constexpr unsigned long long kCandMask = (1ull << kCandBits) - 1ull;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Per-query scratch a warp keeps in shared memory between the phases.
struct Slot {
    int   idx[5];            // neighbour indices into map_orig; idx[0] < 0: no 5-NN inside the radius
    float sx, sy, sz;        // transformed query (fp32, as the kd-tree saw it)
    float fx, fy, fz;        // body-frame query (phase B re-derives R p from it)
    int   pad;               // 48 bytes
};
struct Row { double J[6]; double r; double half_rho; };   // robustified Jacobian row, residual, rho/2

// scalar k of the 29-vector is  sum_i row.J[kA[k]] * row.X[kB[k]]  (X = J for k<21, r for 21..26)
__constant__ unsigned char kPairA[27] = {0,0,0,0,0,0, 1,1,1,1,1, 2,2,2,2, 3,3,3, 4,4, 5, 0,1,2,3,4,5};
__constant__ unsigned char kPairB[27] = {0,1,2,3,4,5, 1,2,3,4,5, 2,3,4,5, 3,4,5, 4,5, 5, 6,6,6,6,6,6};

__device__ __forceinline__ double q_t7(const Q4& q, const D3& t, int k) {
    return k == 0 ? q.w : k == 1 ? q.x : k == 2 ? q.y : k == 3 ? q.z : k == 4 ? t.x : k == 5 ? t.y : t.z;
}

struct KnnSmem {
    Slot slots[kWarps][32];
    Row rows[kWarps][32];
    unsigned char rvalid[kWarps][32];
    double red[kWarps][kNormEq];
    double xch[kMaxPeers][kNormEq];   // fused multi-GPU exchange: every rank's 29 sums before they are added in rank order
    unsigned long long red_cand[kWarps];
    double pose[8];
    int is_last;
    int peer_lost;               // fused exchange: a peer did not publish within the wait bound -> the pose is poisoned (NaN), the host reports it
};

#define LILI_STAMP(i) do { if (a.dbg && blockIdx.x == 0 && threadIdx.x == 0) a.dbg[i] = clock64(); } while (0)
#define LILI_STAMP_LAST(i) do { if (a.dbg && threadIdx.x == 0) a.dbg[i] = clock64(); } while (0)

// One pass over this block's share of the queries at pose (q,t): phases A (search), B (fit + row), C (lane k
// accumulates scalar k).  On return lane k < 29 of every warp holds its partial of scalar k in `acc`.
template <int LANES, bool TMA = false>
__device__ __forceinline__ void knn_phases(const KnnArgs& a, const Q4& q, const D3& t, const int n_q, KnnSmem& S,
                                           double& acc, unsigned long long& cand, const bool use_state, const float4* fpre = nullptr,
                                           unsigned* stage_phase = nullptr) {
    constexpr int GROUPS = 32 / LANES;                 // queries a warp searches concurrently
    extern __shared__ __align__(16) unsigned char dyn_smem[];      // LANES == 1: [kRunCap][kBlock] int4 run lists (thread_knn5)
    int4* runs = reinterpret_cast<int4*>(dyn_smem) + threadIdx.x;
    StageTile* stage = nullptr;                                    // TMA: [kWarps][2] staging tiles (bulk-copy path of the 16-lane search)
    if constexpr (TMA) stage = reinterpret_cast<StageTile*>(dyn_smem) + (threadIdx.x >> 5) * 2 + ((threadIdx.x & 31) >> 4);
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int sub = lane & (LANES - 1);
    const int grp = lane / LANES;
    const unsigned gmask = (LANES == 32) ? 0xffffffffu : (((1u << LANES) - 1u) << (grp * LANES));
    // lane k (< 29) owns scalar k of the normal equations: no per-lane 29-vector, no final shuffle tree
    const int pa = lane < 27 ? kPairA[lane] : 0, pb = lane < 27 ? kPairB[lane] : 0;

    const int per_task = GROUPS * a.rounds;            // <= 32
    const int ntasks = (n_q + per_task - 1) / per_task;
    const int gw = first_task<LANES>(warp);
    const int nw = gridDim.x * kWarps;

#pragma unroll 1
    for (int task = gw; task < ntasks; task += nw) {
        // ---------------- phase A: cooperative exact 5-NN, one query per lane group per round
#pragma unroll 1
        for (int r = 0; r < a.rounds; ++r) {
            const int slot = r * GROUPS + grp;
            const int qi = task * per_task + slot;
            Top5 top;
            top5_init(top);
            float sx = 0.f, sy = 0.f, sz = 0.f;
            float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
            bool live = qi < n_q;
            if (live) {
                f = fpre ? *fpre : a.feats[qi];   // (persistent kernel: the query stays in registers across iterations)
                const D3 pw = qrot_x(q, D3{(double)f.x, (double)f.y, (double)f.z});             // L/src/LidarOdometry.cpp:230-231
                sx = (float)addx(pw.x, t.x); sy = (float)addx(pw.y, t.y); sz = (float)addx(pw.z, t.z);   // :236-238
                if (a.nranks > 1 && owner_of(sx, sy, sz, a.nranks, a.inv_block) != a.rank) live = false;
            }
            // `live` is uniform inside a lane group and the shuffles are masked per group
            LILI_STAMP(8);
            float tau_q = a.tau0;
            if (live && use_state) tau_q = coherence_tau(__ldcg(a.qstate + qi), sx, sy, sz, a.tau0);
            if (live) {
                if (sub == 0) cand += 1ull << kCandBits;
                if constexpr (LANES == 1) thread_knn5(sx, sy, sz, a.map, a.cell_start, a.g, tau_q, runs, kBlock, top, cand);
                else group_knn5<LANES>(sx, sy, sz, a.map, a.cell_start, a.g, sub, gmask, tau_q, top, cand, (a.dbg && blockIdx.x == 0 && threadIdx.x == 0) ? a.dbg : nullptr,
                                       stage, stage_phase);
            }
            LILI_STAMP(11);
            if (sub == 0) {
                Slot& s = S.slots[warp][slot];
                const bool ok = live && top.k4 != ~0ull && ((double)top5_dist(top.k4) < a.max_sqd);  // :365
                // this pass's position and fifth distance for the next pass (a query this rank does not own keeps no bound)
                if (qi < n_q) a.qstate[qi] = make_float4(sx, sy, sz, ok ? top5_dist(top.k4) : __int_as_float(0x7f800000));
                s.idx[0] = ok ? top5_index(top.k0) : -1; s.idx[1] = top5_index(top.k1); s.idx[2] = top5_index(top.k2);
                s.idx[3] = top5_index(top.k3); s.idx[4] = top5_index(top.k4);
                s.sx = sx; s.sy = sy; s.sz = sz;
                s.fx = f.x; s.fy = f.y; s.fz = f.z;
                s.pad = 0;
                if (live && a.nn_idx) {
                    int* o = a.nn_idx + (size_t)qi * 5;
                    const u64 kk[5] = {top.k0, top.k1, top.k2, top.k3, top.k4};
#pragma unroll
                    for (int j = 0; j < 5; ++j) { const int li = top5_index(kk[j]); o[j] = li >= 0 ? __float_as_int(a.map_orig[li].w) : -1; }
                }
                if (live && a.nn_sqd) {
                    float* o = a.nn_sqd + (size_t)qi * 5;
                    o[0] = top5_dist(top.k0); o[1] = top5_dist(top.k1); o[2] = top5_dist(top.k2); o[3] = top5_dist(top.k3); o[4] = top5_dist(top.k4);
                }
            }
        }
        __syncwarp();
        LILI_STAMP(1);
        // ---------------- phase B: one lane per query — plane fit, gates, residual, Jacobian row
        bool ok = false;
        if (lane < per_task) {
            const int qi = task * per_task + lane;
            const Slot s = S.slots[warp][lane];
            float pl0 = 0.f, pl1 = 0.f, pl2 = 0.f, pl3 = 0.f;
            if (qi < n_q && s.idx[0] >= 0) {
                float4 m[5];
#pragma unroll
                for (int j = 0; j < 5; ++j) m[j] = __ldg(a.map_orig + s.idx[j]);                                     // :369-371
                double nv[3];
                if (!plane_fit5_fast(m, nv)) plane_fit5_qr(m, nv);                                                    // :375 (see dev_math.cuh)
                const double n2 = nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2];
                const double nn = sqrt(n2);
                const double normInverse = 1.0 / nn;                                                                  // :376
                if (n2 > 0) { nv[0] /= nn; nv[1] /= nn; nv[2] /= nn; }                                                // :377
                bool planeValid = true;
#pragma unroll
                for (int j = 0; j < 5; ++j)                                                                            // :386-393
                    if (fabs(nv[0] * m[j].x + nv[1] * m[j].y + nv[2] * m[j].z + normInverse) > a.plane_thres) planeValid = false;
                if (planeValid) {
                    // :397-398 with the reference's mixed widths; exact ops keep the fp32 roundings stable
                    const float pd = (float)addx(addx(addx(mulx(nv[0], (double)s.sx), mulx(nv[1], (double)s.sy)), mulx(nv[2], (double)s.sz)), normInverse);
                    const float rng = __fsqrt_rn(__fsqrt_rn(faddx(faddx(fmulx(s.sx, s.sx), fmulx(s.sy, s.sy)), fmulx(s.sz, s.sz))));
                    const float weight = (float)subx(1.0, mulx(0.9, (double)fabsf(pd)) / (double)rng);
                    if ((double)weight > a.w_gate) {                                                                  // :400
                        pl0 = (float)mulx((double)weight, nv[0]);                                                     // :402-405
                        pl1 = (float)mulx((double)weight, nv[1]);
                        pl2 = (float)mulx((double)weight, nv[2]);
                        pl3 = (float)mulx((double)weight, normInverse);
                        ok = true;
                    }
                }
            }
            if (qi < n_q) {
                if (a.valid) a.valid[qi] = ok ? 1 : 0;
                if (a.plane) a.plane[qi] = make_float4(pl0, pl1, pl2, pl3);
            }
            if (ok) {
                // LidarPlaneNormIncreFactor (LidarKeyframeFactor.h:118-128) in closed form:
                //   r = n~ . (q*p + t) + d~ ;  row = [ 2 (R p x n~)^T , n~^T ]  (SURVEY.md Appendix A)
                const D3 rp = qrot_x(q, D3{(double)s.fx, (double)s.fy, (double)s.fz});
                const double nx = pl0, ny = pl1, nz = pl2;
                double r = nx * (rp.x + t.x) + ny * (rp.y + t.y) + nz * (rp.z + t.z) + (double)pl3;
                // ceres::HuberLoss(a) + Corrector (rho'' <= 0 branch): scale row and residual by sqrt(rho')
                const double s2 = r * r, b2 = a.huber_a * a.huber_a;
                double rho0 = s2, rho1 = 1.0;
                if (s2 > b2) { const double rt = sqrt(s2); rho0 = 2.0 * a.huber_a * rt - b2; rho1 = fmax(DBL_MIN, a.huber_a / rt); }
                const double sr = sqrt(rho1);
                Row& R = S.rows[warp][lane];
                R.J[0] = sr * 2.0 * (rp.y * nz - rp.z * ny);
                R.J[1] = sr * 2.0 * (rp.z * nx - rp.x * nz);
                R.J[2] = sr * 2.0 * (rp.x * ny - rp.y * nx);
                R.J[3] = sr * nx; R.J[4] = sr * ny; R.J[5] = sr * nz;
                R.r = sr * r;
                R.half_rho = 0.5 * rho0;
            }
            S.rvalid[warp][lane] = ok ? 1 : 0;
        }
        __syncwarp();
        LILI_STAMP(2);
        // ---------------- phase C: lane k accumulates scalar k over the task's rows (fixed slot order)
        // (four interleaved partial sums, folded in a fixed order: a 32-row task is a chain of 8 dependent fp64 adds instead of 32)
        if (lane < kNormEq) {
            double p4[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll 1
            for (int s0 = 0; s0 < per_task; s0 += 4) {
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int sl = s0 + u;
                    if (sl < per_task && S.rvalid[warp][sl]) {
                        const double* R = reinterpret_cast<const double*>(&S.rows[warp][sl]);
                        p4[u] += lane < 27 ? R[pa] * R[pb] : lane == 27 ? R[7] : 1.0;
                    }
                }
            }
            acc += (p4[0] + p4[1]) + (p4[2] + p4[3]);
        }
        __syncwarp();
    }

}

// Block partial -> partials[29][G] (scalar-major) + candidate counter.
__device__ __forceinline__ void write_block_partials(const KnnArgs& a, KnnSmem& S, double acc, unsigned long long cand) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane < kNormEq) S.red[warp][lane] = acc;
    {
        unsigned long long v = cand;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) S.red_cand[warp] = v;
    }
    __syncthreads();
    const int G = gridDim.x;
    if (threadIdx.x < kNormEq) {
        double v = 0;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) v += S.red[w][threadIdx.x];
        a.partials[(size_t)threadIdx.x * G + blockIdx.x] = v;          // scalar-major: [29][G]
    }
    if (threadIdx.x == 0 && a.cand_total) {     // instrumentation (liliom_set_kernel_timing): examined candidates | searched queries
        unsigned long long v = 0;
        for (int w = 0; w < kWarps; ++w) v += S.red_cand[w];
        if (v & kCandMask) atomicAdd(a.cand_total, v & kCandMask);
        if (v >> kCandBits) atomicAdd(a.queries_total, v >> kCandBits);
    }
}

// Fixed-order sum over the G block partials into S.red[0][0..28]: 8 lanes per scalar.  This is exposed latency, so
// every load of a lane is issued before the first add: ONE L2 round trip for up to 8*kRedLoads = 160 blocks (the
// persistent kernel never has more than one block per SM); larger grids take another trip per 160 blocks.
constexpr int kRedLoads = 20;
__device__ __forceinline__ void reduce_partials(const KnnArgs& a, KnnSmem& S) {
    const int G = gridDim.x;
    const int sc = threadIdx.x >> 3, l8 = threadIdx.x & 7;
    double v = 0.0;
    if (sc < kNormEq) {
        const double* src = a.partials + (size_t)sc * G;
#pragma unroll 1
        for (int base = l8; base < G; base += 8 * kRedLoads) {
            double w[kRedLoads];
#pragma unroll
            for (int j = 0; j < kRedLoads; ++j) w[j] = (base + 8 * j < G) ? __ldcg(src + base + 8 * j) : 0.0;
            // fixed pairwise tree (deterministic, short dependency chain)
#pragma unroll
            for (int j = 0; j < 10; ++j) w[j] += w[j + 10];
#pragma unroll
            for (int j = 0; j < 5; ++j) w[j] += w[j + 5];
            v += ((w[0] + w[1]) + (w[2] + w[3])) + w[4];
        }
    }
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    if (l8 == 0 && sc < kNormEq) S.red[0][sc] = v;
    __syncthreads();
}

// ---- fused multi-GPU exchange (persistent kernel; liliom_comm_peer_attach) -----------------------------------------------
// Every 8-byte word carries the pass's epoch in its upper half (a double travels as {epoch|lo32, epoch|hi32}): an aligned 8-byte
// store is single-copy atomic, so a reader that sees the epoch sees the data — no fence and no flag word.  Stores and loads are
// system scope (the writer is another GPU over NVLink).  Two buffers alternate by epoch parity: a rank can publish pass e+1 only
// after it has read every rank's pass e, i.e. after every block of every rank has finished reading pass e-1 (they pass their own
// grid barrier of pass e before their block 0 publishes).  Epochs grow monotonically across launches and the buffers are zeroed
// once, so a stale word never matches.  On entry S.red[0][0..28] holds this rank's sums (identical in every block); on return it
// holds the sums over all ranks, added in rank order (bit-identical on every rank).
// `writer`: the block that publishes (block 0 of the persistent kernel; the last block of the per-iteration kernel, the only caller there).
__device__ __forceinline__ void peer_exchange(const PeerArgs& pa, unsigned int epoch, KnnSmem& S, bool writer) {
    const size_t base = (size_t)(epoch & 1u) * kMaxPeers * 32;
    const bool already_lost = S.peer_lost != 0;     // block-uniform (written before the previous exchange's closing barrier): no second wait
    if (writer && threadIdx.x < kNormEq) {
        const double v = S.red[0][threadIdx.x];
        const u64 w0 = ((u64)epoch << 32) | (u64)(unsigned)__double2loint(v);
        const u64 w1 = ((u64)epoch << 32) | (u64)(unsigned)__double2hiint(v);
        for (int p = 0; p < pa.nranks; ++p) {
            ulonglong2* dst = pa.buf[p] + base + (size_t)pa.rank * 32 + threadIdx.x;
            asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"(w0), "l"(w1) : "memory");
        }
    }
    for (int t = threadIdx.x; t < pa.nranks * kNormEq; t += blockDim.x) {
        const int r = t / kNormEq, k = t - r * kNormEq;
        const ulonglong2* src = pa.buf[pa.rank] + base + (size_t)r * 32 + k;
        u64 w0 = 0, w1 = 0;
        unsigned int spins = 0;
        bool lost = already_lost;
        while (!already_lost) {
            asm volatile("ld.relaxed.sys.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(src) : "memory");
            if ((unsigned int)(w0 >> 32) == epoch && (unsigned int)(w1 >> 32) == epoch) break;
            if (++spins > (1u << 23)) { lost = true; S.peer_lost = 1; break; }      // ~6 s: a lost peer must end in a NaN pose, never in a hung GPU
            __nanosleep(20);
        }
        S.xch[r][k] = lost ? __longlong_as_double(0x7ff8000000000000ll) : __hiloint2double((int)(unsigned int)w1, (int)(unsigned int)w0);
    }
    __syncthreads();
    if (threadIdx.x < kNormEq) {
        double v = 0.0;
        for (int r = 0; r < pa.nranks; ++r) v += S.xch[r][threadIdx.x];
        S.red[0][threadIdx.x] = v;
    }
    __syncthreads();
}

// Inside one GPU only block 0 talks to the peers: it republishes the sums over all ranks (and the loss flag) for the other
// blocks, which wait on one epoch word instead of polling nranks x 29 system-scope words each (one block per SM doing that
// adds tens of microseconds per pass on 2 GPUs).
__device__ __forceinline__ void peer_local_publish(const PeerArgs& pa, unsigned int epoch, KnnSmem& S) {
    double* dst = pa.lsum + (size_t)(epoch & 1u) * 32;
    if (threadIdx.x < kNormEq) dst[threadIdx.x] = S.red[0][threadIdx.x];
    if (threadIdx.x == kNormEq) dst[kNormEq] = S.peer_lost ? 1.0 : 0.0;
    __syncthreads();
    if (threadIdx.x == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(pa.lflag + (epoch & 1u)), "r"(epoch) : "memory");
}
__device__ __forceinline__ void peer_local_wait(const PeerArgs& pa, unsigned int epoch, KnnSmem& S) {
    if (threadIdx.x == 0) {
        unsigned int v;
        do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(pa.lflag + (epoch & 1u)) : "memory"); } while (v != epoch);
    }
    __syncthreads();
    const double* src = pa.lsum + (size_t)(epoch & 1u) * 32;
    if (threadIdx.x < kNormEq) S.red[0][threadIdx.x] = __ldcg(src + threadIdx.x);
    if (threadIdx.x == kNormEq && __ldcg(src + kNormEq) != 0.0) S.peer_lost = 1;
    __syncthreads();
}

// One thread: 6x6 solve of the 29 reduced sums `sums`, Plus, sign-unify -> xn.  A lost peer poisons the pose (NaN).
__device__ __forceinline__ void gn_step(const double* sums, bool peer_lost, const Q4& q, const D3& t, double xn[7]) {
    double s[kNormEq];
#pragma unroll
    for (int k = 0; k < kNormEq; ++k) s[k] = sums[k];
    double x[7], nb[6], d[6];
#pragma unroll
    for (int k = 0; k < 7; ++k) x[k] = q_t7(q, t, k);
#pragma unroll
    for (int k = 0; k < 6; ++k) nb[k] = -s[21 + k];
    const bool solved = gn_safe_step(s, nb, d);
    if (s[28] > 0.0 && solved) pose_plus(x, d, xn);
    else {
#pragma unroll
        for (int k = 0; k < 7; ++k) xn[k] = x[k];
    }
    if (xn[0] < 0) { xn[0] = -xn[0]; xn[1] = -xn[1]; xn[2] = -xn[2]; xn[3] = -xn[3]; }   // :539-549
    if (peer_lost) {
#pragma unroll
        for (int k = 0; k < 7; ++k) xn[k] = __longlong_as_double(0x7ff8000000000000ll);
    }
}

// Part k of one row of the per-iteration stats (kStatsDoubles doubles: n_corr, lm_iters, cost, the 27 sums, pose7, pad).
// Part k < kNormEq is scalar k of the sums s; part kNormEq is the LM iteration count and the pose xn after the step.  The block
// kernels store one part per thread, the one-thread kernels every part.
__device__ __forceinline__ void write_stats(double* st, int k, const double* s, double lm_iters, const double* xn) {
    if (k < kNormEq) st[k < 27 ? 3 + k : k == 27 ? 2 : 0] = s[k];
    else {
        st[1] = lm_iters;
#pragma unroll
        for (int j = 0; j < 7; ++j) st[30 + j] = xn[j];
    }
}

__device__ __forceinline__ void write_neq_stats(const KnnArgs& a, const KnnSmem& S, double* stats) {
    if (threadIdx.x < kNormEq) {
        a.neq[threadIdx.x] = S.red[0][threadIdx.x];
        if (stats) write_stats(stats, threadIdx.x, S.red[0], 0.0, nullptr);
    }
}


// (Search and fit as two kernels — the search alone runs at 64 registers and twice the resident warps — was slower than the
// fused kernel at 128k queries, with the exhaustive and with the pruned search: what limits the one-thread-per-query shape is
// divergence between the lanes' candidate lists, not latency hiding.)
// Blocks per SM of the one-thread-per-query instance: that shape is bound by latency per issued instruction at ~4 warps per
// scheduler, so it trades registers (spills in the fp64 fit) for resident warps.
#ifndef LILI_KNN1_MINBLOCKS
#define LILI_KNN1_MINBLOCKS 2
#endif
template <int LANES>
__global__ void __launch_bounds__(kBlock, LANES == 1 ? LILI_KNN1_MINBLOCKS : 2) k_knn_plane(KnnArgs a, PassArgs p, const __grid_constant__ PeerArgs pa) {
    __shared__ __align__(16) KnnSmem S;
    if (threadIdx.x == 0) S.peer_lost = 0;
    LILI_STAMP(0);
    const Q4 q{a.pose[0], a.pose[1], a.pose[2], a.pose[3]};
    const D3 t{a.pose[4], a.pose[5], a.pose[6]};
    const int n_q = a.n_dev ? min(*a.n_dev, a.n) : a.n;
    double acc = 0.0;
    unsigned long long cand = 0;
    knn_phases<LANES>(a, q, t, n_q, S, acc, cand, p.use_state != 0);
    LILI_STAMP(3);
    write_block_partials(a, S, acc, cand);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int tk = atomicAdd(p.ticket, 1u);
        S.is_last = (tk == gridDim.x - 1);
    }
    __syncthreads();
    LILI_STAMP(4);
    if (!S.is_last) return;
    __threadfence();
    LILI_STAMP_LAST(5);
    // ---------------- last block: fixed-order sum over blocks, then the 6x6 step
    reduce_partials(a, S);
    if (pa.enabled) peer_exchange(pa, pa.epoch0, S, true);      // multi-GPU, one launch per iteration: the last block trades sums with the peers
    LILI_STAMP_LAST(6);
    if (threadIdx.x == 0) {
        *p.ticket = 0;
        if (p.update_pose) {
            double xn[7];
            gn_step(S.red[0], S.peer_lost, q, t, xn);
#pragma unroll
            for (int k = 0; k < 7; ++k) a.pose_out[k] = xn[k];
            if (pa.enabled) a.pose_out[7] = S.peer_lost ? 1.0 : 0.0;
            if (p.stats) write_stats(p.stats, kNormEq, nullptr, 1.0, xn);
        }
    }
    LILI_STAMP_LAST(7);
    write_neq_stats(a, S, p.update_pose ? p.stats : nullptr);
}

// All GN iterations in ONE cooperative launch (single GPU, GN mode): per iteration the blocks meet at one
// grid barrier after publishing their partials; then EVERY block sums the partials and solves the 6x6
// system redundantly (bit-identical), so no second barrier or broadcast is needed.  Removes the launch
// gap, the drain and the ticket round trip of the per-iteration kernel (~6 us of ~18 per iteration).
// The persistent kernel never runs more than one block per SM (grid <= sm_count), so it takes a 176-register cap instead
// of the 128 of __launch_bounds__(256, 2): the spills (200-600 B per thread in the fp64 fit) disappear, while a
// 64-register block of the Preprocessing node's cooperative kernel still fits beside it (176*256 + 64*256 <= 65536
// registers), which the two-node e2e leg relies on (A/B of the caps in one process: tools/ab_variants.py).
// (__maxnreg__ and __launch_bounds__ cannot be combined; the block size is fixed by the host code.)
#ifndef LILI_GN_MAXNREG
#define LILI_GN_MAXNREG 176
#endif
#define LILI_GN_BOUNDS __maxnreg__(LILI_GN_MAXNREG)
template <int LANES, bool TMA = false>
__global__ void LILI_GN_BOUNDS k_gn_persistent(KnnArgs a, int iters, unsigned int* bar, double* stats_base, unsigned int bar_base,
                                                             int sync_mode, const __grid_constant__ PeerArgs pa, const __grid_constant__ GnIo io) {
    __shared__ __align__(16) KnnSmem S;
    unsigned stage_phase = 0;
    if constexpr (TMA) {       // one mbarrier per lane group, 16 arrivals (every lane of the group, with or without a run to stage)
        extern __shared__ __align__(16) unsigned char dyn_smem_k[];
        StageTile* tile = reinterpret_cast<StageTile*>(dyn_smem_k) + (threadIdx.x >> 5) * 2 + ((threadIdx.x & 31) >> 4);
        if ((threadIdx.x & 15) == 0) mbar_init(&tile->bar, 16u);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    const int n_q = a.n_dev ? min(*a.n_dev, a.n) : a.n;
    if (threadIdx.x == 32) S.peer_lost = 0;
    if (threadIdx.x < 7) S.pose[threadIdx.x] = io.pose0[threadIdx.x];
    if (a.dbg && blockIdx.x == 0 && threadIdx.x == 0) a.dbg[30] = (long long)globaltimer_ns();
    __syncthreads();
    const unsigned int G = gridDim.x;
    // bar_base = arrivals of all previous launches on this context (tracked by the host, advanced by iters*G per launch)
    // one task per warp and one round per task (the small-scan shape): each lane group serves the same
    // query in every iteration, so its body-frame point is loaded once and kept in registers
    float4 f_keep = make_float4(0.f, 0.f, 0.f, 0.f);
    bool keep = false;
    {
        constexpr int GROUPS = 32 / LANES;
        const int per_task = GROUPS * a.rounds;
        const int ntasks = (n_q + per_task - 1) / per_task;
        const int gw = first_task<LANES>(threadIdx.x >> 5);
        const int nw = gridDim.x * kWarps;
        if (a.rounds == 1 && ntasks <= nw) {
            keep = true;
            const int qi = gw * per_task + ((threadIdx.x & 31) / LANES);
            if (qi < n_q) f_keep = a.feats[qi];
        }
    }
#pragma unroll 1
    for (int it = 0; it < iters; ++it) {
        const Q4 q{S.pose[0], S.pose[1], S.pose[2], S.pose[3]};
        const D3 t{S.pose[4], S.pose[5], S.pose[6]};
        double acc = 0.0;
        unsigned long long cand = 0;
        const bool stamp = a.dbg && blockIdx.x == 0 && threadIdx.x == 0 && it == 2;
        if (stamp) a.dbg[16] = clock64();
        knn_phases<LANES, TMA>(a, q, t, n_q, S, acc, cand, it > 0, keep ? &f_keep : nullptr, &stage_phase);
        if (stamp) a.dbg[17] = clock64();
        // ---- grid barrier + cross-block sum.  Mode 3 (default; measured 12.70 -> 11.99 us per pass against mode 0): one release by
        // thread 0 after the block barrier (cumulative over bar.sync, as in cooperative groups' grid.sync; SASS: MEMBAR.ALL.GPU +
        // RED, no L1 invalidate) and NO acquire fence after the relaxed poll.  An acquire would only add an L1 invalidation:
        // everything this kernel reads through L1 (map, cell table, features) is immutable for the launch, and the partials are
        // read with L2-scope loads (__ldcg) issued after the poll's control dependency and a bar.sync.  The PTX model formally
        // asks for the acquire: mode 1 polls with ld.acquire (slower per pass: tools/ab_variants.py), mode 0 fences both
        // sides; tests pin all three to the same bits (test_gpu_variants.py, test_persistent_barrier_stress_all_sync_modes).
        // Multi-GPU (fused exchange): the other blocks of this GPU arrive but do not wait here — they wait for block 0's
        // republished sums over all ranks.
        const bool follower = pa.enabled && blockIdx.x != 0;
        write_block_partials(a, S, acc, cand);
        if (sync_mode == 0) __threadfence();
        __syncthreads();
        if (stamp) a.dbg[18] = clock64();
        if (threadIdx.x == 0) grid_barrier(bar, bar_base + (unsigned int)(it + 1) * G, sync_mode, !follower);
        if (!follower) {
            __syncthreads();
            if (stamp) a.dbg[19] = clock64();
            reduce_partials(a, S);
            if (pa.enabled) {       // block 0: this rank's sums -> sums over all ranks, then on to the other blocks
                peer_exchange(pa, pa.epoch0 + (unsigned int)it, S, true);
                peer_local_publish(pa, pa.epoch0 + (unsigned int)it, S);
            }
        } else peer_local_wait(pa, pa.epoch0 + (unsigned int)it, S);
        if (stamp) a.dbg[20] = clock64();
        double* stats = stats_base ? stats_base + (size_t)it * kStatsDoubles : nullptr;
        if (threadIdx.x == 0) {
            double xn[7];
            gn_step(S.red[0], S.peer_lost, q, t, xn);
            if (stamp) a.dbg[21] = clock64();
#pragma unroll
            for (int k = 0; k < 7; ++k) S.pose[k] = xn[k];
            if (blockIdx.x == 0) {
#pragma unroll
                for (int k = 0; k < 7; ++k) a.pose_out[k] = xn[k];
                if (pa.enabled) a.pose_out[7] = S.peer_lost ? 1.0 : 0.0;      // explicit loss flag for the host (the pose is NaN as well)
                if (stats) write_stats(stats, kNormEq, nullptr, 1.0, xn);
            }
        }
        if (blockIdx.x == 0) write_neq_stats(a, S, stats);
        if (blockIdx.x == 0 && it == iters - 1 && io.host_out) {      // results straight into the host's pinned block
            if (threadIdx.x == 0) {
#pragma unroll
                for (int k = 0; k < 7; ++k) io.host_out->pose[k] = S.pose[k];
                io.host_out->pose[7] = (pa.enabled && S.peer_lost) ? 1.0 : 0.0;
                if (a.n_dev) io.host_out->n_feats = *a.n_dev;
            }
            if (io.vgp && threadIdx.x >= 32 && threadIdx.x < 32 + (int)(sizeof(VgParams) / sizeof(int))) reinterpret_cast<int*>(&io.host_out->vgp)[threadIdx.x - 32] = io.vgp[threadIdx.x - 32];
            __threadfence_system();
        }
        __syncthreads();
        // the partials of this iteration may only be overwritten after every block has summed them: the next
        // barrier is behind the next write, so alternate between two partial buffers
        a.partials = (it & 1) ? a.partials - (size_t)kNormEq * G : a.partials + (size_t)kNormEq * G;
    }
    if (a.dbg && blockIdx.x == 0 && threadIdx.x == 0) a.dbg[31] = (long long)globaltimer_ns();
}

// GN step for the multi-GPU path: runs after the all-reduce of neq[29], identically on every rank.
__global__ void k_gn_update(const double* __restrict__ neq, double* __restrict__ pose, double* __restrict__ stats) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double xn[7];
    gn_step(neq, false, Q4{pose[0], pose[1], pose[2], pose[3]}, D3{pose[4], pose[5], pose[6]}, xn);
    for (int k = 0; k < 7; ++k) pose[k] = xn[k];
    if (stats) {
#pragma unroll
        for (int k = 0; k <= kNormEq; ++k) write_stats(stats, k, neq, 1.0, xn);
    }
}

// ------------------------------------------------------------------ Ceres-faithful LM on frozen correspondences
// One block: every LM iteration is a pass over the correspondences (cost + 27 scalars at the
// candidate), a block reduction, and the trust-region bookkeeping of Ceres 2.0's
// TrustRegionMinimizer + LevenbergMarquardtStrategy on thread 0 (Jacobi scaling fixed at
// iteration 0, D = sqrt(clamp(diag)/radius), rho-based radius update), with the dense QR on
// [J; D] replaced by its normal equations (J^T J + D^2) y = J^T r in fp64 (6x6 LDL^T).
struct LmArgs {
    const float4* feats; const unsigned char* valid; const float4* plane; int n; const int* n_dev;
    double* pose;         // in/out
    double* stats;        // slot of this outer iteration
    double huber_a;
    int max_num_iter;
    const double* neq0;   // 29 scalars at the linearisation pose (from k_knn_plane)
};

constexpr int kLmBlock = 512;

__device__ void lm_eval(const LmArgs& a, const double x[7], double out[kNormEq], double (*red)[kNormEq]) {
    Q4 q{x[0], x[1], x[2], x[3]};
    double acc[kNormEq];
#pragma unroll
    for (int k = 0; k < kNormEq; ++k) acc[k] = 0.0;
    const int n_c = a.n_dev ? min(*a.n_dev, a.n) : a.n;
    for (int i = threadIdx.x; i < n_c; i += blockDim.x) {
        if (!a.valid[i]) continue;
        float4 f = a.feats[i];
        float4 pl = a.plane[i];
        D3 rp = qrot_x(q, D3{(double)f.x, (double)f.y, (double)f.z});
        double nx = pl.x, ny = pl.y, nz = pl.z;
        double r = nx * (rp.x + x[4]) + ny * (rp.y + x[5]) + nz * (rp.z + x[6]) + (double)pl.w;
        double J[6];
        J[0] = 2.0 * (rp.y * nz - rp.z * ny);
        J[1] = 2.0 * (rp.z * nx - rp.x * nz);
        J[2] = 2.0 * (rp.x * ny - rp.y * nx);
        J[3] = nx; J[4] = ny; J[5] = nz;
        double s2 = r * r, rho0, rho1;
        const double b2 = a.huber_a * a.huber_a;
        if (s2 > b2) { double rt = sqrt(s2); rho0 = 2.0 * a.huber_a * rt - b2; rho1 = fmax(DBL_MIN, a.huber_a / rt); }
        else { rho0 = s2; rho1 = 1.0; }
        double sr = sqrt(rho1);
#pragma unroll
        for (int k = 0; k < 6; ++k) J[k] *= sr;
        r *= sr;
        int k = 0;
#pragma unroll
        for (int i2 = 0; i2 < 6; ++i2)
#pragma unroll
            for (int j = i2; j < 6; ++j) acc[k++] += J[i2] * J[j];
#pragma unroll
        for (int i2 = 0; i2 < 6; ++i2) acc[21 + i2] += J[i2] * r;
        acc[27] += 0.5 * rho0;
        acc[28] += 1.0;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kNormEq; ++k) {
        double v = warp_sum(acc[k]);
        if (lane == 0) red[warp][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < kNormEq) {
        double v = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v += red[w][threadIdx.x];
        red[0][threadIdx.x] = v;
    }
    __syncthreads();
    for (int k = 0; k < kNormEq; ++k) out[k] = red[0][k];
    __syncthreads();
}

__global__ void __launch_bounds__(kLmBlock) k_lm_solve(LmArgs a) {
    __shared__ double red[kLmBlock / 32][kNormEq];
    __shared__ double sh_x[7];
    __shared__ int sh_cmd;   // 0 = stop, 1 = evaluate candidate in sh_x
    double x[7];
    for (int k = 0; k < 7; ++k) x[k] = a.pose[k];
    double S[kNormEq];
    lm_eval(a, x, S, red);          // iteration 0: cost, gradient, J^T J at x
    // --- thread-0 state (replicated arithmetic is avoided: only thread 0 decides) ---
    double radius = 1e4, decrease_factor = 2.0;
    bool reuse_diagonal = false, last_successful = false;
    double diagonal[6], scaling[6];
    double x_cost = S[27];
    int iteration = 0, invalid = 0;
    if (threadIdx.x == 0) {
        int kk = 0;
        for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) { if (i == j) scaling[i] = 1.0 / (1.0 + sqrt(S[kk])); ++kk; }
    }
    const double count0 = S[28];
    double step_keep[6];
    double model_cost_change = 0;
    for (;;) {
        if (threadIdx.x == 0) {
            int cmd = 1;
            double xc[7];
            for (;;) {   // loop over invalid steps without evaluation
                if (count0 <= 0.0) { cmd = 0; break; }
                if (iteration >= a.max_num_iter) { cmd = 0; break; }
                if (last_successful) {
                    double gmax = 0;
                    for (int k = 0; k < 6; ++k) gmax = fmax(gmax, fabs(S[21 + k]));
                    if (gmax <= 1e-10) { cmd = 0; break; }
                }
                if (radius < 1e-32) { cmd = 0; break; }
                ++iteration;
                last_successful = false;
                // scaled normal equations  Hs = S H S, gs = S g
                double Hs[21], gs[6];
                int kk = 0;
                for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) { Hs[kk] = S[kk] * scaling[i] * scaling[j]; ++kk; }
                for (int i = 0; i < 6; ++i) gs[i] = S[21 + i] * scaling[i];
                if (!reuse_diagonal) {
                    kk = 0;
                    for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) { if (i == j) diagonal[i] = fmin(fmax(Hs[kk], 1e-6), 1e32); ++kk; }
                }
                double Ha[21];
                kk = 0;
                for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) { Ha[kk] = Hs[kk] + (i == j ? diagonal[i] / radius : 0.0); ++kk; }
                double y[6];
                bool ok = solve6_ldlt(Ha, gs, y);
                reuse_diagonal = true;
                double step[6];
                model_cost_change = 0;
                if (ok) {
                    for (int k = 0; k < 6; ++k) step[k] = -y[k];
                    // -(step.gs + 1/2 step^T Hs step)
                    double Hfull[6][6];
                    kk = 0;
                    for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) { Hfull[i][j] = Hs[kk]; Hfull[j][i] = Hs[kk]; ++kk; }
                    double sg = 0, shs = 0;
                    for (int i = 0; i < 6; ++i) {
                        sg += step[i] * gs[i];
                        double hv = 0;
                        for (int j = 0; j < 6; ++j) hv += Hfull[i][j] * step[j];
                        shs += step[i] * hv;
                    }
                    model_cost_change = -(sg + 0.5 * shs);
                }
                if (!ok || !(model_cost_change > 0.0)) {
                    if (++invalid >= 5) { cmd = 0; break; }
                    radius *= 0.5; reuse_diagonal = false;
                    continue;
                }
                invalid = 0;
                for (int k = 0; k < 6; ++k) step_keep[k] = step[k] * scaling[k];
                pose_plus(x, step_keep, xc);
                for (int k = 0; k < 7; ++k) sh_x[k] = xc[k];
                cmd = 1;
                break;
            }
            sh_cmd = cmd;
        }
        __syncthreads();
        if (sh_cmd == 0) break;
        double xc[7];
        for (int k = 0; k < 7; ++k) xc[k] = sh_x[k];
        double Sc[kNormEq];
        lm_eval(a, xc, Sc, red);
        int stop = 0;
        if (threadIdx.x == 0) {
            double candidate_cost = Sc[27];
            double xn = 0, sn = 0;
            for (int k = 0; k < 7; ++k) { xn += x[k] * x[k]; sn += (x[k] - xc[k]) * (x[k] - xc[k]); }
            xn = sqrt(xn); sn = sqrt(sn);
            double cost_change = x_cost - candidate_cost;
            if (sn <= 1e-8 * (xn + 1e-8)) stop = 1;                                   // parameter tolerance
            else if (fabs(cost_change) <= 1e-6 * x_cost) stop = 1;                    // function tolerance
            else {
                double relative_decrease = cost_change / model_cost_change;
                if (relative_decrease > 1e-3) {
                    for (int k = 0; k < 7; ++k) x[k] = xc[k];
                    for (int k = 0; k < kNormEq; ++k) S[k] = Sc[k];
                    x_cost = candidate_cost;
                    last_successful = true;
                    double qd = 2.0 * relative_decrease - 1.0;
                    radius = radius / fmax(1.0 / 3.0, 1.0 - qd * qd * qd);
                    radius = fmin(1e16, radius);
                    decrease_factor = 2.0;
                    reuse_diagonal = false;
                } else {
                    radius = radius / decrease_factor;
                    decrease_factor *= 2.0;
                    reuse_diagonal = true;
                }
            }
            sh_cmd = stop ? 0 : 1;
        }
        __syncthreads();
        if (sh_cmd == 0) break;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        if (x[0] < 0) { x[0] = -x[0]; x[1] = -x[1]; x[2] = -x[2]; x[3] = -x[3]; }     // :539-549
        for (int k = 0; k < 7; ++k) a.pose[k] = x[k];
        if (a.stats) {
#pragma unroll
            for (int k = 0; k <= kNormEq; ++k) write_stats(a.stats, k, a.neq0, (double)iteration, x);
        }
    }
}

// ------------------------------------------------------------------ instrumentation: the C-bar of SURVEY.md §8(d)
// Points in the full 3x3x3 cell block of every (owned) query at pose (q,t): the candidate count the algorithmic-bytes figure
// B_q = 16 + 27*8 + 16*C-bar is defined on.  The search kernels examine fewer (pruning, knn_core.cuh) and count those
// separately (liliom_counters::knn_candidates).  out[0] += queries, out[1] += block points.
__global__ void k_block27_count(const float4* __restrict__ feats, int n, Q4 q, D3 t, const int* __restrict__ cell_start, GridDesc g,
                                int nranks, int rank, float inv_block, unsigned long long* __restrict__ out) {
    unsigned long long cnt = 0, nq = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float4 f = feats[i];
        const D3 pw = qrot_x(q, D3{(double)f.x, (double)f.y, (double)f.z});
        const float sx = (float)addx(pw.x, t.x), sy = (float)addx(pw.y, t.y), sz = (float)addx(pw.z, t.z);
        if (nranks > 1 && owner_of(sx, sy, sz, nranks, inv_block) != rank) continue;
        ++nq;
        const int cx = cell_coord(sx, g.inv_cell) - g.org[0], cy = cell_coord(sy, g.inv_cell) - g.org[1], cz = cell_coord(sz, g.inv_cell) - g.org[2];
        const int x0 = max(cx - 1, 0), x1 = min(cx + 1, g.dim[0] - 1);
        if (x0 > x1) continue;
        for (int row = 0; row < 9; ++row) {
            const int y = cy + (row % 3) - 1, z = cz + (row / 3) - 1;
            if (y < 0 || y >= g.dim[1] || z < 0 || z >= g.dim[2]) continue;
            const int base = (z * g.dim[1] + y) * g.dim[0];
            cnt += (unsigned long long)(__ldg(cell_start + base + x1 + 1) - __ldg(cell_start + base + x0));
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { cnt += __shfl_xor_sync(0xffffffffu, cnt, o); nq += __shfl_xor_sync(0xffffffffu, nq, o); }
    if ((threadIdx.x & 31) == 0) { if (nq) atomicAdd(out, nq); if (cnt) atomicAdd(out + 1, cnt); }
}

int block27_stats(liliom_ctx* c, const double pose7[7], unsigned long long out[2]) {
    out[0] = out[1] = 0;
    if (!c->map.ready) return LILIOM_E_NOMAP;
    const int n = c->n_feats_actual;
    if (n <= 0) return LILIOM_OK;
    LILI_CUDA(c, c->lm_state.ensure(64 * sizeof(long long)));
    unsigned long long* d = c->lm_state.as<unsigned long long>();
    LILI_CUDA(c, cudaMemsetAsync(d, 0, 16, c->stream));
    const Q4 q{pose7[0], pose7[1], pose7[2], pose7[3]};
    const D3 t{pose7[4], pose7[5], pose7[6]};
    k_block27_count<<<min(cdiv(n, 256), c->sm_count * 4), 256, 0, c->stream>>>(c->feats.as<float4>(), n, q, t, c->map.cell_start.as<int>(), c->map.grid,
                                                                              c->nranks, c->rank, c->shard_inv_block, d);
    LILI_TRY(launch_check(c, "k_block27_count"));
    return read_back(c, {{out, d, 16}});
}

// ------------------------------------------------------------------ host orchestration
int nccl_allreduce_sum_f64(liliom_ctx* c, double* buf, int count);   // comm.cu

// Fused exchange (liliom_comm_peer_attach): every rank's buffer as mapped here; epoch0 = epoch of the launch's first pass.
static PeerArgs peer_args(const liliom_ctx* c, unsigned int epoch0) {
    PeerArgs pa{{}, c->nranks, c->rank, epoch0, 1, c->peer_local.as<double>(), reinterpret_cast<unsigned int*>(c->peer_local.as<double>() + 64)};
    for (int p = 0; p < c->nranks; ++p) pa.buf[p] = reinterpret_cast<ulonglong2*>(c->peer_ptrs[p]);
    return pa;
}

// Kernel timing (liliom_set_kernel_timing): an event pair around `launch`, which runs `passes` passes of the kernel body.
// s2m_run folds the pairs into the counters after its synchronise.
template <class F>
static int timed_launch(liliom_ctx* c, bool timed, int passes, F&& launch) {
    if (!timed) return launch();
    const size_t ev = 2 * c->ev_passes.size();
    while (ev + 2 > c->ev_pool.size()) { cudaEvent_t e; LILI_CUDA(c, cudaEventCreate(&e)); c->ev_pool.push_back(e); }
    LILI_CUDA(c, cudaEventRecord(c->ev_pool[ev], c->stream));
    LILI_TRY(launch());
    LILI_CUDA(c, cudaEventRecord(c->ev_pool[ev + 1], c->stream));
    c->ev_passes.push_back(passes);
    return LILIOM_OK;
}

static const void* knn_kernel(int lanes) {
    return lanes == 16 ? (const void*)k_knn_plane<16> : lanes == 1 ? (const void*)k_knn_plane<1> : lanes == 2 ? (const void*)k_knn_plane<2>
         : lanes == 4 ? (const void*)k_knn_plane<4> : (const void*)k_knn_plane<8>;
}
static const void* gn_kernel(int lanes, bool tma) {
    return tma ? (const void*)k_gn_persistent<16, true> : lanes == 16 ? (const void*)k_gn_persistent<16> : lanes == 1 ? (const void*)k_gn_persistent<1>
         : lanes == 2 ? (const void*)k_gn_persistent<2> : lanes == 4 ? (const void*)k_gn_persistent<4> : (const void*)k_gn_persistent<8>;
}

// Buffers of one scan-to-map call and the arguments the search kernels share.
static int s2m_prepare(liliom_ctx* c, const S2mPlan& p, int iters, int mode, bool want_corr, bool timed, KnnArgs& a) {
    const int n = c->n_feats;
    LILI_CUDA(c, c->pose_dev.ensure(16 * sizeof(double)));
    // two buffers (the persistent kernel alternates); sized for the largest grid so that a bigger scan never reallocates mid-stream
    LILI_CUDA(c, c->partials.ensure((size_t)2 * max(p.grid, c->sm_count * 2) * kNormEq * sizeof(double)));
    LILI_CUDA(c, c->neq.ensure(32 * sizeof(double)));
    LILI_CUDA(c, c->stats_dev.ensure((size_t)(iters + 1) * kStatsDoubles * sizeof(double)));
    if (!c->counter.p) {
        LILI_CUDA(c, c->counter.ensure(64));
        LILI_CUDA(c, cudaMemsetAsync(c->counter.p, 0, 64, c->stream));
    }
    const bool need_corr = want_corr || mode == LILIOM_MODE_CERES;
    if (need_corr) {
        LILI_CUDA(c, c->corr_valid.ensure((size_t)n + 16));
        LILI_CUDA(c, c->corr_plane.ensure((size_t)n * sizeof(float4) + 16));
    }
    if (want_corr) {
        LILI_CUDA(c, c->nn_idx.ensure((size_t)n * 5 * sizeof(int) + 16));
        LILI_CUDA(c, c->nn_sqd.ensure((size_t)n * 5 * sizeof(float) + 16));
        LILI_CUDA(c, cudaMemsetAsync(c->nn_idx.p, 0xff, (size_t)n * 5 * sizeof(int), c->stream));
        LILI_CUDA(c, cudaMemsetAsync(c->nn_sqd.p, 0x7f, (size_t)n * 5 * sizeof(float), c->stream));
    }
    LILI_CUDA(c, c->qstate.ensure((size_t)(n > 0 ? n : 1) * sizeof(float4)));
    a = KnnArgs{};
    a.feats = c->feats.as<float4>(); a.n = n; a.n_dev = c->d_nfeats;
    a.map = c->map.sorted.as<float4>(); a.map_orig = c->map.xyzw.as<float4>(); a.cell_start = c->map.cell_start.as<int>(); a.g = c->map.grid;
    a.pose = c->pose_dev.as<double>(); a.pose_out = c->pose_dev.as<double>();
    a.max_sqd = c->prm.knn_max_sqdist; a.plane_thres = c->prm.plane_thres; a.w_gate = c->prm.weight_gate; a.huber_a = c->prm.huber_a;
    a.valid = need_corr ? c->corr_valid.as<unsigned char>() : nullptr; a.plane = need_corr ? c->corr_plane.as<float4>() : nullptr;
    a.nn_idx = want_corr ? c->nn_idx.as<int>() : nullptr; a.nn_sqd = want_corr ? c->nn_sqd.as<float>() : nullptr;
    a.partials = c->partials.as<double>(); a.neq = c->neq.as<double>();
    unsigned long long* counts = reinterpret_cast<unsigned long long*>(c->counter.as<unsigned char>() + 16);   // candidates, queries
    a.cand_total = timed ? counts : nullptr; a.queries_total = timed ? counts + 1 : nullptr;
    a.tau0 = knn_gate_tau(c->prm.knn_max_sqdist); a.qstate = c->qstate.as<float4>(); a.inv_block = c->shard_inv_block;
    a.rounds = p.rounds; a.nranks = c->nranks; a.rank = c->rank;
    if (c->dbg_timing) {
        LILI_CUDA(c, c->lm_state.ensure(64 * sizeof(long long)));
        LILI_CUDA(c, cudaMemsetAsync(c->lm_state.p, 0, 64 * sizeof(long long), c->stream));
        a.dbg = c->lm_state.as<long long>();
    }
    if (p.lanes == 1 && !c->knn1_smem_set) {
        LILI_CUDA(c, cudaFuncSetAttribute(knn_kernel(1), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.dyn_smem));
        LILI_CUDA(c, cudaFuncSetAttribute(gn_kernel(1, false), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.dyn_smem));
        c->knn1_smem_set = true;
    }
    if (p.tma && !c->knn_tma_smem_set) {
        LILI_CUDA(c, cudaFuncSetAttribute(gn_kernel(16, true), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.dyn_smem));
        c->knn_tma_smem_set = true;
    }
    return LILIOM_OK;
}

// LILIOM_DEBUG_TIMING: stage clocks of the two cooperative kernels that ran before this call (resident pipeline), the step's
// device timeline and the phase clocks of the GN kernel, to stderr.
static void print_debug_timing(liliom_ctx* c, const long long* dbg, bool persistent) {
    long long t[12], gt[6] = {0, 0, 0, 0, 0, 0};
    if (c->hz_ctl.p && cudaMemcpy(t, c->hz_ctl.as<unsigned char>() + 16, sizeof(t), cudaMemcpyDeviceToHost) == cudaSuccess && t[4] > t[0]) {
        gt[0] = t[10]; gt[1] = t[11];
        fprintf(stderr, "[k_hz_coop, cycles, block 0] A keep-flags+barrier %lld, B de-skew/bin+barrier %lld, C patches+barrier %lld (patch 0: window %lld, "
                        "lists %lld, centroid+scatter %lld, eigen %lld, decisions %lld), D emit %lld\n",
                t[1] - t[0], t[2] - t[1], t[3] - t[2], t[5] - t[2], t[6] - t[5], t[7] - t[6], t[8] - t[7], t[9] - t[8], t[4] - t[3]);
    }
    const long long* vs = vg_coop_stamps(c);
    if (vs && cudaMemcpy(t, vs, 7 * sizeof(long long), cudaMemcpyDeviceToHost) == cudaSuccess && t[4] > t[0]) {
        gt[2] = t[5]; gt[3] = t[6];
        fprintf(stderr, "[k_vg_coop, cycles, block 0] 1 hash insert+barrier %lld, 2 ranks+barrier %lld, 3 group+barrier %lld, 4 centroids %lld\n",
                t[1] - t[0], t[2] - t[1], t[3] - t[2], t[4] - t[3]);
    }
    if (cudaMemcpy(t, dbg + 30, 2 * sizeof(long long), cudaMemcpyDeviceToHost) == cudaSuccess) { gt[4] = t[0]; gt[5] = t[1]; }
    if (gt[0] && gt[2] && gt[4])      // the step's device timeline (block 0 of each kernel, %globaltimer)
        fprintf(stderr, "[step timeline, ns from k_hz_coop start] hz 0..%lld | gap %lld | vg %lld..%lld | gap %lld | gn %lld..%lld (%lld)\n",
                gt[1] - gt[0], gt[2] - gt[1], gt[2] - gt[0], gt[3] - gt[0], gt[4] - gt[3], gt[4] - gt[0], gt[5] - gt[0], gt[5] - gt[4]);
    long long h[24];
    cudaMemcpy(h, dbg, sizeof(h), cudaMemcpyDeviceToHost);
    if (h[16]) fprintf(stderr, "[persistent it=2, cycles] phases %lld, partials+fence %lld, barrier %lld, reduce %lld, solve %lld\n",
                       h[17] - h[16], h[18] - h[17], h[19] - h[18], h[20] - h[19], h[21] - h[20]);
    if (!persistent && h[0] && h[1] > h[0])
        fprintf(stderr, "[phase A detail] pose+feat+transform %lld, first row bounds %lld, candidates+rank %lld, merge %lld, slot %lld\n",
                h[8] - h[0], h[9] - h[8], h[10] - h[9], h[11] - h[10], h[1] - h[11]);
    if (!persistent && h[0] && h[4] > h[0])
        fprintf(stderr, "[knn phases, cycles] blk0: start->A %lld, B %lld, C %lld, loop-end %lld, block-reduce+ticket %lld | last block: reduce %lld, solve %lld (abs tail %lld after blk0 start)\n",
                h[1] - h[0], h[2] - h[1], h[3] - h[2], 0LL, h[4] - h[3], h[6] - h[5], h[7] - h[6], h[7] - h[0]);
}

int s2m_run(liliom_ctx* c, double pose7[7], int match_cnt, int max_num_iter, int mode, liliom_iter_stats* stats,
            bool want_corr, double out29[29]) {
    if (!c->map.ready) return LILIOM_E_NOMAP;
    if (c->map_n_global < 10) return LILIOM_E_FEWMAP;          // L/src/LidarOdometry.cpp:485-488
    const int n = c->n_feats, iters = match_cnt;
    if (iters < 0) return LILIOM_E_ARG;
    // the per-iteration stats come back through the pinned block: check its capacity before anything is enqueued
    if (stats && iters > 0 && offsetof(PinBlock, stats) + (size_t)iters * kStatsDoubles * sizeof(double) > c->h_pin_bytes) return LILIOM_E_CAPACITY;
    // kernel timing (liliom_set_kernel_timing): an event pair + the device-side query/candidate counts on every time_every-th call
    const bool timed = c->time_kernels && (c->time_calls++ % (unsigned)c->time_every) == 0;
    const bool peer = c->peer_ready && c->peer_ptrs[c->rank] != nullptr;       // fused exchange instead of ncclAllReduce + k_gn_update
    const S2mPlan p = s2m_plan({n, c->last_n_feats, c->d_nfeats != nullptr, c->sm_count, mode, iters, want_corr, c->nranks, peer,
                                c->force_lanes, c->force_rounds, c->knn_tma});
    KnnArgs a;
    LILI_TRY(s2m_prepare(c, p, iters, mode, want_corr, timed, a));
    // zero-copy results (GnIo): the persistent kernel leaves pose, query count and VoxelGrid parameters in the pinned block
    // itself when the device can address it; only per-iteration stats / the 29 sums still travel by copy
    const bool host_io = p.persistent && c->h_pin_dev != nullptr;
    if (p.persistent) {         // all iterations in one cooperative launch, the start pose as a kernel parameter
        int iters_arg = iters, sync_mode = c->gn_sync;
        unsigned int* bar = reinterpret_cast<unsigned int*>(c->counter.as<unsigned char>() + 32);
        double* stats_base = c->stats_dev.as<double>();
        unsigned int bar_base = c->bar_arrivals;
        PeerArgs pa{};
        if (peer) { pa = peer_args(c, c->peer_epoch + 1u); c->peer_epoch += (unsigned int)iters; }   // same calls on every rank: same epochs
        GnIo io{};
        memcpy(io.pose0, pose7, 7 * sizeof(double));
        io.host_out = host_io ? &c->h_pin_dev->s2m : nullptr;
        io.vgp = host_io && c->vg_check ? c->vg_params.as<int>() : nullptr;
        void* kargs[] = {&a, &iters_arg, &bar, &stats_base, &bar_base, &sync_mode, &pa, &io};
        LILI_TRY(timed_launch(c, timed, iters, [&] {
            LILI_CUDA(c, cudaLaunchCooperativeKernel(gn_kernel(p.lanes, p.tma), dim3(p.grid), dim3(kBlock), kargs, p.dyn_smem, c->stream));
            return launch_check(c, "k_gn_persistent");
        }));
        c->bar_arrivals += (unsigned int)iters * (unsigned int)p.grid;
    } else {                    // one launch per iteration; the start pose goes through the pinned block to pose_dev
        double* pin = c->h_pin->pose_stage;
        memcpy(pin, pose7, 7 * sizeof(double)); pin[7] = 0.0;          // + cleared peer-loss flag
        LILI_CUDA(c, cudaMemcpyAsync(c->pose_dev.p, pin, 8 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
        const bool multi = c->nranks > 1;
        // fused exchange, one launch per iteration (large scans: grid > one block per SM): the last block trades the sums with the
        // peers and performs the GN step itself — no ncclAllReduce, no update kernel
        const bool peer_iter = peer && multi && mode == LILIOM_MODE_GN && iters > 0;
        const int update_pose = (mode == LILIOM_MODE_GN && (!multi || peer_iter) && iters > 0) ? 1 : 0;
        const int launches = (iters == 0 && want_corr) ? 1 : iters;
        for (int it = 0; it < launches; ++it) {
            PassArgs pass{c->counter.as<unsigned int>(), c->stats_dev.as<double>() + (size_t)it * kStatsDoubles, update_pose, it > 0 ? 1 : 0};
            PeerArgs pit = peer_iter ? peer_args(c, ++c->peer_epoch) : PeerArgs{};
            void* kargs[] = {&a, &pass, &pit};
            LILI_TRY(timed_launch(c, timed, 1, [&] {
                LILI_CUDA(c, cudaLaunchKernel(knn_kernel(p.lanes), dim3(p.grid), dim3(kBlock), kargs, p.dyn_smem, c->stream));
                return launch_check(c, "k_knn_plane");
            }));
            if (iters == 0) break;
            if (multi && !peer_iter) LILI_TRY(nccl_allreduce_sum_f64(c, c->neq.as<double>(), kNormEq));
            if (mode == LILIOM_MODE_GN && multi && !peer_iter) {
                k_gn_update<<<1, 32, 0, c->stream>>>(c->neq.as<double>(), c->pose_dev.as<double>(), pass.stats);
                LILI_TRY(launch_check(c, "k_gn_update"));
            } else if (mode != LILIOM_MODE_GN) {
                if (multi) { c->last_error = "CERES mode is single-GPU (the LM solve is one block); use GN mode with a communicator"; return LILIOM_E_ARG; }
                LmArgs l{};
                l.feats = a.feats; l.valid = a.valid; l.plane = a.plane; l.n = n; l.n_dev = c->d_nfeats;
                l.pose = c->pose_dev.as<double>(); l.stats = pass.stats; l.huber_a = a.huber_a; l.max_num_iter = max_num_iter;
                l.neq0 = c->neq.as<double>();
                k_lm_solve<<<1, kLmBlock, 0, c->stream>>>(l);
                LILI_TRY(launch_check(c, "k_lm_solve"));
            }
        }
    }
    // ---- results: pose + stats in one pinned block
    PinResult& r = c->h_pin->s2m;
    const bool want_stats = stats && iters > 0;
    if (!host_io) LILI_CUDA(c, cudaMemcpyAsync(r.pose, c->pose_dev.p, 8 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));     // pose + peer-loss flag
    if (out29) LILI_CUDA(c, cudaMemcpyAsync(r.neq, c->neq.p, kNormEq * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (c->d_nfeats && !host_io) LILI_CUDA(c, cudaMemcpyAsync(&r.n_feats, c->d_nfeats, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    if (c->vg_check && !host_io) LILI_CUDA(c, cudaMemcpyAsync(&r.vgp, c->vg_params.p, sizeof(VgParams), cudaMemcpyDeviceToHost, c->stream));
    if (want_stats) LILI_CUDA(c, cudaMemcpyAsync(c->h_pin->stats, c->stats_dev.p, (size_t)iters * kStatsDoubles * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    c->n_feats_actual = c->d_nfeats ? min(r.n_feats, n) : n;
    c->last_n_feats = c->n_feats_actual;
    if (c->vg_check) {
        c->vg_ncells = r.vgp.overflow ? 0 : (long long)r.vgp.div_b[0] * r.vgp.div_b[1] * r.vgp.div_b[2];
        c->vg_bail = r.vgp.bail != 0;
    }
    if (iters > 0 && peer && r.pose[7] != 0.0) {
        c->last_error = "fused exchange: a peer rank did not publish its sums within the wait bound (collective call not entered on every rank?)";
        return LILIOM_E_NCCL;
    }
    if (iters > 0) for (int k = 0; k < 7; ++k) pose7[k] = r.pose[k];
    if (out29) for (int k = 0; k < kNormEq; ++k) out29[k] = r.neq[k];
    for (int it = 0; want_stats && it < iters; ++it) {
        const double* s = c->h_pin->stats + (size_t)it * kStatsDoubles;
        stats[it].n_corr = (int)s[0]; stats[it].lm_iters = (int)s[1]; stats[it].cost = s[2];
        memcpy(stats[it].jtj_jtr, s + 3, 27 * sizeof(double)); memcpy(stats[it].pose7, s + 30, 7 * sizeof(double));
    }
    if (c->dbg_timing) print_debug_timing(c, a.dbg, p.persistent);
    for (size_t k = 0; timed && k < c->ev_passes.size(); ++k) {        // fold finished kernel timings into the counters
        float ms = 0;
        if (cudaEventElapsedTime(&ms, c->ev_pool[2 * k], c->ev_pool[2 * k + 1]) == cudaSuccess) {
            // a persistent launch covers `iters` passes of the kernel body: count each pass as one "launch"
            c->cnt.knn_ms += ms; c->cnt.knn_launches += (unsigned long long)c->ev_passes[k];
        }
    }
    if (timed) c->ev_passes.clear();
    return LILIOM_OK;
}

}  // namespace lili
