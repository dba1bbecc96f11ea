// BackendFusion correspondence searches on the same kNN core (SURVEY.md §8 rows a16/a18):
//   point-to-line : L/src/BackendFusion.cpp:1531-1599 (variant 0), R/src/BackendFusion.cpp:1394-1462 (variant 1)
//   point-to-plane: R/src/BackendFusion.cpp:1464-1520 (configurable radius / plane gate / weight gate / score)
// and the LiDAR rows of the sliding window reduced to 6x6 blocks (f1).  Every kernel here works on a small TABLE of keyframes
// (SURVEY.md §8 f5): the queries of all listed keyframes are concatenated, each query finds its keyframe (bk_window.h) and that
// keyframe's pose.  The single-keyframe entry points (liliom_correspond_*, liliom_backend_*_block) are the k = 1 case of the
// window calls (liliom_backend_window_*), so a keyframe's results are the same bits through either.
// The sliding-window optimiser that consumes the blocks stays on the host.
#include "ctx.cuh"
#include "dev_math.cuh"
#include "knn_core.cuh"
#include "bk_window.h"

namespace lili {

constexpr int kLanes = 8;

struct BkArgs {
    const unsigned char* qpts; int qstride;            // queries: float4 xyz at qpts + (qoff[j] + qi - start[j]) * qstride
    int k; long long start[kWinMax + 1]; long long qoff[kWinMax]; Q4 q[kWinMax]; D3 t[kWinMax];   // per keyframe of the table
    const float4* map; const float4* map_orig; const int* cell_start; GridDesc g;
    int variant;
    double max_sqd, plane_thres, w_gate, lidar_const;
    float tau0;        // largest fp32 distance inside the gate (search pruning, knn_core.cuh)
    unsigned char* valid; float* pa; float* pb; float4* plane; double* score;   // indexed by the concatenated query
    const float* map_refl; double reflect_thres;   // Horizon backend variant (L:1617-1638; query reflectivity = 48-byte field 9), nullptr = ROT variant
};

// the query's body-frame point and its keyframe's pose
__device__ __forceinline__ const unsigned char* bk_query(const BkArgs& a, long long qi, Q4& q, D3& t) {
    const int j = bkw_find(a.start, a.k, qi);
    q = a.q[j]; t = a.t[j];
    return a.qpts + (size_t)(a.qoff[j] + (qi - a.start[j])) * a.qstride;
}

__global__ void __launch_bounds__(kBlock) k_backend_edge(const __grid_constant__ BkArgs a) {
    const int lane = threadIdx.x & 31;
    const int sub = lane & (kLanes - 1), oct = lane / kLanes;
    const unsigned omask = ((1u << kLanes) - 1u) << (oct * kLanes);
    const long long qi = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / kLanes;
    if (qi >= a.start[a.k]) return;   // uniform per octet
    Q4 q; D3 t;
    const float4 f = *reinterpret_cast<const float4*>(bk_query(a, qi, q, t));
    const VgXyz pw = pcl_transform_xyz(q, t, f.x, f.y, f.z);
    const float sx = pw.x, sy = pw.y, sz = pw.z;
    Top5 top;
    top5_init(top);
    unsigned long long cand = 0;
    group_knn5<kLanes>(sx, sy, sz, a.map, a.cell_start, a.g, sub, omask, a.tau0, top, cand);
    if (sub != 0) return;
    bool ok = false;
    float A3[3] = {0, 0, 0}, B3[3] = {0, 0, 0};
    if (top5_accepts(top, 1.0)) {                                                                    // L:1543
        int pos[5]; top5_indices(top, pos);
        double px[5], py[5], pz[5], cx = 0, cy = 0, cz = 0;
        for (int j = 0; j < 5; ++j) {
            float4 m = a.map_orig[pos[j]];
            px[j] = m.x; py[j] = m.y; pz[j] = m.z;
            cx = addx(cx, px[j]); cy = addx(cy, py[j]); cz = addx(cz, pz[j]);
        }
        cx = cx / 5.0; cy = cy / 5.0; cz = cz / 5.0;                                  // L:1555
        double a00 = 0, a10 = 0, a20 = 0, a11 = 0, a21 = 0, a22 = 0;
        for (int j = 0; j < 5; ++j) {                                                  // L:1560-1564
            double z0 = subx(px[j], cx), z1 = subx(py[j], cy), z2 = subx(pz[j], cz);
            a00 = addx(a00, mulx(z0, z0)); a10 = addx(a10, mulx(z1, z0)); a20 = addx(a20, mulx(z2, z0));
            a11 = addx(a11, mulx(z1, z1)); a21 = addx(a21, mulx(z2, z1)); a22 = addx(a22, mulx(z2, z2));
        }
        double ev[3], evec[3][3];
        eigen_sym3(a00, a10, a20, a11, a21, a22, ev, evec);                            // L:1568
        if (ev[2] > 3 * ev[1]) {                                                       // L:1575
            const double ux = evec[0][2], uy = evec[1][2], uz = evec[2][2];
            const double ax = cx + 0.1 * ux, ay = cy + 0.1 * uy, az = cz + 0.1 * uz;   // L:1579
            const double bx = cx - 0.1 * ux, by = cy - 0.1 * uy, bz = cz - 0.1 * uz;   // L:1580
            ok = true;
            if (a.variant == 1) {                                                      // R:1435-1439
                const double ux_ = sx - ax, uy_ = sy - ay, uz_ = sz - az;
                const double vx_ = sx - bx, vy_ = sy - by, vz_ = sz - bz;
                const double nx = uy_ * vz_ - uz_ * vy_, ny = uz_ * vx_ - ux_ * vz_, nz = ux_ * vy_ - uy_ * vx_;
                const double dx = ax - bx, dy = ay - by, dz = az - bz;
                const double dist = sqrt(nx * nx + ny * ny + nz * nz) / sqrt(dx * dx + dy * dy + dz * dz);
                if (!(dist < 0.1)) ok = false;
            }
            if (ok) {
                A3[0] = (float)ax; A3[1] = (float)ay; A3[2] = (float)az;
                B3[0] = (float)bx; B3[1] = (float)by; B3[2] = (float)bz;
            }
        }
    }
    a.valid[qi] = ok ? 1 : 0;
    for (int k = 0; k < 3; ++k) { a.pa[3 * (size_t)qi + k] = A3[k]; a.pb[3 * (size_t)qi + k] = B3[k]; }
}

__global__ void __launch_bounds__(kBlock) k_backend_surf(const __grid_constant__ BkArgs a) {
    const int lane = threadIdx.x & 31;
    const int sub = lane & (kLanes - 1), oct = lane / kLanes;
    const unsigned omask = ((1u << kLanes) - 1u) << (oct * kLanes);
    const long long qi = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / kLanes;
    if (qi >= a.start[a.k]) return;
    Q4 q; D3 t;
    const unsigned char* qp = bk_query(a, qi, q, t);
    const float4 f = *reinterpret_cast<const float4*>(qp);
    const VgXyz pw = pcl_transform_xyz(q, t, f.x, f.y, f.z);
    const float sx = pw.x, sy = pw.y, sz = pw.z;
    Top5 top;
    top5_init(top);
    unsigned long long cand = 0;
    group_knn5<kLanes>(sx, sy, sz, a.map, a.cell_start, a.g, sub, omask, a.tau0, top, cand);
    if (sub != 0) return;
    bool ok = false;
    float4 pl = make_float4(0, 0, 0, 0);
    double sc = 0;
    if (top5_accepts(top, a.max_sqd)) {                                                               // R:1476
        int pos[5]; top5_indices(top, pos);
        double A[5][3], B[5];
        float4 m[5];
        for (int j = 0; j < 5; ++j) { m[j] = a.map_orig[pos[j]]; A[j][0] = m[j].x; A[j][1] = m[j].y; A[j][2] = m[j].z; B[j] = -1.0; }
        double sum_w = 0.0;
        bool skip = false;
        if (a.map_refl) {                                                              // L:1617-1638: rows weighted by 1/|d reflectivity| / sum
            double vw[5];
            const float fr = reinterpret_cast<const float*>(qp)[9];
            for (int j = 0; j < 5; ++j) {
                const double tmp_w = (double)fabsf(fsubx(fr, a.map_refl[pos[j]]));
                sum_w = addx(sum_w, tmp_w);
                vw[j] = 1.0 / tmp_w;          // +inf when the reflectivities coincide, as in the reference
            }
            if (sum_w > a.reflect_thres) skip = true;                                  // L:1628
            for (int j = 0; j < 5; ++j) {
                const double w = vw[j] / sum_w;
                A[j][0] = mulx(w, (double)m[j].x); A[j][1] = mulx(w, (double)m[j].y); A[j][2] = mulx(w, (double)m[j].z);
                B[j] = mulx(B[j], w);
            }
        }
        double nv[3] = {0, 0, 0};
        if (!skip) colpiv_qr_solve_5x3(A, B, nv);                                      // R:1484 / L:1641
        float weight;
        if (plane_gate(nv, m, sx, sy, sz, a.plane_thres, a.w_gate, skip, pl, weight)) {
            sc = a.map_refl ? a.lidar_const * ((double)weight + exp(-sum_w))              // L:1676
                            : a.lidar_const * (double)weight;                                 // R:1515
            ok = true;
        }
    }
    a.valid[qi] = ok ? 1 : 0;
    a.plane[qi] = pl;
    a.score[qi] = sc;
}

// correspondences found per keyframe (vec_edge_res_cnt / vec_surf_res_cnt): blockIdx.x = keyframe, blockIdx.y = kind
struct CntArgs { const unsigned char* valid[2]; long long start[2][kWinMax + 1]; int* cnt; };   // cnt[kind * kWinMax + keyframe]
__global__ void k_win_count(const __grid_constant__ CntArgs a) {
    const int j = blockIdx.x, kind = blockIdx.y;
    int s = 0;
    for (long long i = a.start[kind][j] + threadIdx.x; i < a.start[kind][j + 1]; i += blockDim.x) s += a.valid[kind][i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    __shared__ int red[8];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        int v = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v += red[w];
        a.cnt[kind * kWinMax + j] = v;
    }
}

static int search_launch(liliom_ctx* c, bool edge, const BkArgs& a) {
    const long long n = a.start[a.k];
    if (n <= 0) return LILIOM_OK;
    if (edge) k_backend_edge<<<cdiv(n * kLanes, kBlock), kBlock, 0, c->stream>>>(a);
    else k_backend_surf<<<cdiv(n * kLanes, kBlock), kBlock, 0, c->stream>>>(a);
    return launch_check(c, edge ? "k_backend_edge" : "k_backend_surf");
}

static void bk_set_map(BkArgs& a, const MapIndex& mi) {
    a.map = mi.sorted.as<float4>(); a.map_orig = mi.xyzw.as<float4>(); a.cell_start = mi.cell_start.as<int>(); a.g = mi.grid;
}

static int backend_prepare(liliom_ctx* c, const void* feats, int n, int stride) {
    if (!c->map.ready) return LILIOM_E_NOMAP;
    if (n < 0 || (n > 0 && !feats)) return LILIOM_E_ARG;
    if (stride != 16 && stride != 32 && stride != 48) return LILIOM_E_ARG;
    c->n_feats = n;
    c->d_nfeats = nullptr;
    c->bk_kind = 0; c->bk_n = 0;
    if (n == 0) return LILIOM_OK;
    LILI_CUDA(c, c->feats.ensure((size_t)n * sizeof(float4)));
    if (stride == 16) {
        LILI_CUDA(c, cudaMemcpyAsync(c->feats.p, feats, (size_t)n * 16, cudaMemcpyHostToDevice, c->stream));
    } else {
        LILI_CUDA(c, c->raw.ensure((size_t)n * stride));
        LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, feats, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream));
        LILI_TRY(repack_to_f4(c, c->raw.p, n, stride, c->feats.as<float4>()));
    }
    return LILIOM_OK;
}


// ---------------------------------------------------------------------------------------
// SURVEY.md §8 (f1): the LiDAR residual blocks of window keyframes (L/src/BackendFusion.cpp:919-979) reduced on the
// device to 6x6 normal-equation blocks.  Rows are the closed forms of SURVEY.md Appendix A:
//   LidarEdgeFactor      (LidarKeyframeFactor.h:12-62):  r = s |u x v| / |a-b|, u = p_w-a, v = p_w-b, p_w = q p + t
//                                                        g = dr/dp_w = s ((a-b) x c^) / |a-b|
//   LidarPlaneNormFactor (LidarKeyframeFactor.h:65-108): r = score (n~ . p_w + d~), p_w = q (q_lb^-1 (p - t_lb)) + t, g = score n~
//   row = sqrt(rho') [ g^T , 2 (R p' x g)^T ]   (parameter blocks t, q -> tangent order [t, rot]),  CauchyLoss(b) (:845)
// One segment = one keyframe's rows of one kind; blockIdx.y = segment, the segment's first `nblocks` blocks split its rows.
// ---------------------------------------------------------------------------------------
struct BlkSeg {
    const unsigned char* qpts; int qstride, n;  // the keyframe's queries (float4 xyz at qpts + i * qstride)
    int nblocks, edge;                          // blocks of this segment; 1 = LidarEdgeFactor rows, 0 = LidarPlaneNormFactor rows
    const unsigned char* valid;
    const float* pa; const float* pb;           // edge
    const float4* plane; const double* score;   // surf
    Q4 q; D3 t;                                 // body pose
    int wvariant;                               // -1: s_weight / score as given; 0, 1: the window weights of bk_window.h
    const int* n_corr;                          // device-side correspondence count of this keyframe and kind (wvariant >= 0)
    double s_weight, lidar_const;
};
struct BlkCommon { Q4 qlb_inv; D3 tlb; double cauchy_b; double* partials; };   // partials: [segment][kMaxBlk][29]

constexpr int kBlkThreads = 256;
constexpr int kMaxBlk = 64;

__global__ void __launch_bounds__(kBlkThreads) k_backend_block(const BlkSeg* __restrict__ segs, BlkCommon a) {
    __shared__ double red[kBlkThreads / 32][kNormEq];
    const BlkSeg& s = segs[blockIdx.y];
    const int nblocks = s.nblocks;
    if ((int)blockIdx.x >= nblocks) return;        // uniform per block
    double acc[kNormEq];
#pragma unroll
    for (int k = 0; k < kNormEq; ++k) acc[k] = 0.0;
    const double b2 = a.cauchy_b * a.cauchy_b, c2 = 1.0 / b2;
    const bool edge = s.edge != 0;
    const Q4 q = s.q; const D3 t = s.t;
    const int wv = s.wvariant;
    const int ncorr = wv >= 0 ? *s.n_corr : 0;
    const double s_weight = wv >= 0 ? bkw_edge_weight(wv, s.lidar_const, ncorr) : s.s_weight;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < s.n; i += nblocks * blockDim.x) {
        if (!s.valid[i]) continue;
        const float4 f = *reinterpret_cast<const float4*>(s.qpts + (size_t)i * s.qstride);
        D3 pr, g;        // the point the keyframe rotation acts on, and dr/dp_w
        double r;
        if (edge) {
            pr = D3{(double)f.x, (double)f.y, (double)f.z};
            const D3 rp = qrot_x(q, pr);
            const D3 lp{rp.x + t.x, rp.y + t.y, rp.z + t.z};
            const D3 A{(double)s.pa[3 * (size_t)i], (double)s.pa[3 * (size_t)i + 1], (double)s.pa[3 * (size_t)i + 2]};
            const D3 B{(double)s.pb[3 * (size_t)i], (double)s.pb[3 * (size_t)i + 1], (double)s.pb[3 * (size_t)i + 2]};
            const D3 u{lp.x - A.x, lp.y - A.y, lp.z - A.z}, v{lp.x - B.x, lp.y - B.y, lp.z - B.z};
            const D3 nu = cross_x(u, v);
            const D3 de{A.x - B.x, A.y - B.y, A.z - B.z};
            const double nn = sqrt(nu.x * nu.x + nu.y * nu.y + nu.z * nu.z);
            const double dn = sqrt(de.x * de.x + de.y * de.y + de.z * de.z);
            r = nn / dn * s_weight;
            g = D3{0, 0, 0};
            if (nn > 0) {    // a zero cross product has no derivative (the reference's autodiff yields NaN there)
                const D3 cx = cross_x(de, nu);
                const double k = s_weight / (dn * nn);
                g = D3{k * cx.x, k * cx.y, k * cx.z};
            }
        } else {
            const D3 d{(double)f.x - a.tlb.x, (double)f.y - a.tlb.y, (double)f.z - a.tlb.z};
            pr = qrot_x(a.qlb_inv, d);
            const D3 rp = qrot_x(q, pr);
            const float4 pl = s.plane[i];
            const double sc = wv >= 0 ? bkw_surf_score(wv, s.score[i], ncorr) : s.score[i];
            r = sc * ((double)pl.x * (rp.x + t.x) + (double)pl.y * (rp.y + t.y) + (double)pl.z * (rp.z + t.z) + (double)pl.w);
            g = D3{sc * (double)pl.x, sc * (double)pl.y, sc * (double)pl.z};
        }
        const D3 rp = qrot_x(q, pr);
        Row R;
        R.J[0] = g.x; R.J[1] = g.y; R.J[2] = g.z;
        R.J[3] = 2.0 * (rp.y * g.z - rp.z * g.y);
        R.J[4] = 2.0 * (rp.z * g.x - rp.x * g.z);
        R.J[5] = 2.0 * (rp.x * g.y - rp.y * g.x);
        R.r = r;
        cauchy_correct(R, b2, c2);
        add_row29(acc, R);
    }
    const double v = block_sum29(acc, red, kBlkThreads / 32);
    if (threadIdx.x < kNormEq) a.partials[((size_t)blockIdx.y * kMaxBlk + blockIdx.x) * kNormEq + threadIdx.x] = v;
}

// fixed-order sum over each segment's block partials (run-to-run deterministic): blockIdx.x = segment
__global__ void k_backend_block_sum(const BlkSeg* __restrict__ segs, const double* __restrict__ partials, double* __restrict__ out29) {
    if (threadIdx.x >= kNormEq) return;
    const int nblocks = segs[blockIdx.x].nblocks;
    double v = 0;
    for (int b = 0; b < nblocks; ++b) v += partials[((size_t)blockIdx.x * kMaxBlk + b) * kNormEq + threadIdx.x];
    out29[(size_t)blockIdx.x * kNormEq + threadIdx.x] = v;
}

static int seg_blocks(int n) { return n > 0 ? min(cdiv(n, kBlkThreads), kMaxBlk) : 1; }

// one launch pair for all segments; out = nseg x 29 doubles
static int backend_block_run(liliom_ctx* c, const std::vector<BlkSeg>& segs, BlkCommon a, double* out) {
    const int nseg = (int)segs.size();
    int gx = 1;
    for (const BlkSeg& s : segs) gx = max(gx, s.nblocks);
    LILI_CUDA(c, c->partials.ensure((size_t)nseg * kMaxBlk * kNormEq * sizeof(double)));
    LILI_CUDA(c, c->neq.ensure((size_t)max(nseg * kNormEq, 32) * sizeof(double)));
    LILI_CUDA(c, c->win_tab.ensure((size_t)nseg * sizeof(BlkSeg)));
    LILI_CUDA(c, cudaMemcpyAsync(c->win_tab.p, segs.data(), (size_t)nseg * sizeof(BlkSeg), cudaMemcpyHostToDevice, c->stream));
    a.partials = c->partials.as<double>();
    k_backend_block<<<dim3(gx, nseg), kBlkThreads, 0, c->stream>>>(c->win_tab.as<BlkSeg>(), a);
    LILI_TRY(launch_check(c, "k_backend_block"));
    k_backend_block_sum<<<nseg, 32, 0, c->stream>>>(c->win_tab.as<BlkSeg>(), a.partials, c->neq.as<double>());
    LILI_TRY(launch_check(c, "k_backend_block_sum"));
    if (nseg == 1) return read_back(c, {{out, c->neq.p, kNormEq * sizeof(double)}});     // the 29 sums through pinned memory
    LILI_CUDA(c, cudaMemcpyAsync(out, c->neq.p, (size_t)nseg * kNormEq * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

// Eigen::Quaternion::inverse(): conjugate / squared norm (zero quaternion for a zero input)
static Q4 q_inverse(const double q[4]) {
    const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    return n2 > 0 ? Q4{q[0] / n2, -q[1] / n2, -q[2] / n2, -q[3] / n2} : Q4{0, 0, 0, 0};
}

// k = 1 table over the resident c->feats (or the 48-byte upload in c->raw when the search reads the reflectivity)
static BkArgs single_table(liliom_ctx* c, int n, const double pose7[7], bool raw48) {
    BkArgs a{};
    a.qpts = raw48 ? (const unsigned char*)c->raw.p : c->feats.as<unsigned char>(); a.qstride = raw48 ? 48 : 16;
    a.k = 1; a.start[0] = 0; a.start[1] = n; a.qoff[0] = 0;
    a.q[0] = Q4{pose7[0], pose7[1], pose7[2], pose7[3]}; a.t[0] = D3{pose7[4], pose7[5], pose7[6]};
    return a;
}

static BlkSeg single_seg(liliom_ctx* c, bool edge, const double pose7_body[7]) {
    BlkSeg s{};
    s.qpts = c->feats.as<unsigned char>(); s.qstride = 16; s.n = c->bk_n; s.nblocks = seg_blocks(c->bk_n); s.edge = edge ? 1 : 0;
    s.valid = c->corr_valid.as<unsigned char>();
    s.q = Q4{pose7_body[0], pose7_body[1], pose7_body[2], pose7_body[3]}; s.t = D3{pose7_body[4], pose7_body[5], pose7_body[6]};
    s.wvariant = -1;
    return s;
}

}  // namespace lili

using namespace lili;

extern "C" int liliom_correspond_edge(liliom_ctx* c, const void* feats, int n, int stride, const double pose7[7], int variant,
                                      unsigned char* valid, float* pa, float* pb) {
    if (!c || !pose7 || !valid || !pa || !pb || (variant != 0 && variant != 1)) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_TRY(backend_prepare(c, feats, n, stride));
    if (n == 0) { c->bk_kind = 1; return LILIOM_OK; }
    LILI_CUDA(c, c->corr_valid.ensure((size_t)n + 16));
    LILI_CUDA(c, c->corr_plane.ensure((size_t)n * 24 + 16));
    BkArgs a = single_table(c, n, pose7, false);
    bk_set_map(a, c->map);
    a.variant = variant;
    a.tau0 = knn_gate_tau(1.0);                                                   // L:1543 sqdist[4] < 1.0
    a.valid = c->corr_valid.as<unsigned char>();
    a.pa = c->corr_plane.as<float>(); a.pb = a.pa + 3 * (size_t)n;
    LILI_TRY(search_launch(c, true, a));
    c->bk_kind = 1; c->bk_n = n;
    LILI_CUDA(c, cudaMemcpyAsync(valid, a.valid, (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaMemcpyAsync(pa, a.pa, (size_t)n * 12, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaMemcpyAsync(pb, a.pb, (size_t)n * 12, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

static int correspond_surf_impl(liliom_ctx* c, const void* feats, int n, int stride, const double pose7[7], double kd_max_radius,
                                double surf_dist_thres, double w_gate, double lidar_const, bool refl, double reflect_thres,
                                unsigned char* valid, float* plane, double* score) {
    if (!c || !pose7 || !valid || !plane || !score) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    {   // the grid's cell size bounds the exact search radius
        float cell = 1.0f / c->map.grid.inv_cell;
        if (c->map.ready && c->map.n > 0 && kd_max_radius > (double)cell * (double)cell) {
            c->last_error = "kd_max_radius exceeds the cell size the map grid was built with (raise params.knn_max_sqdist)";
            return LILIOM_E_ARG;
        }
    }
    LILI_TRY(backend_prepare(c, feats, n, stride));
    if (n == 0) { c->bk_kind = 2; return LILIOM_OK; }
    LILI_CUDA(c, c->corr_valid.ensure((size_t)n + 16));
    LILI_CUDA(c, c->corr_plane.ensure((size_t)n * 16 + 16));
    LILI_CUDA(c, c->nn_sqd.ensure((size_t)n * 8 + 16));
    if (refl && (stride != 48 || !c->map.refl.p)) {
        c->last_error = "reflectivity variant needs 48-byte features and a map installed with liliom_map_set_cloud";
        return LILIOM_E_ARG;
    }
    BkArgs a = single_table(c, n, pose7, refl);
    bk_set_map(a, c->map);
    a.tau0 = knn_gate_tau(kd_max_radius);
    a.max_sqd = kd_max_radius; a.plane_thres = surf_dist_thres; a.w_gate = w_gate; a.lidar_const = lidar_const;
    if (refl) { a.map_refl = c->map.refl.as<float>(); a.reflect_thres = reflect_thres; }
    a.valid = c->corr_valid.as<unsigned char>(); a.plane = c->corr_plane.as<float4>(); a.score = c->nn_sqd.as<double>();
    LILI_TRY(search_launch(c, false, a));
    c->bk_kind = 2; c->bk_n = n;
    LILI_CUDA(c, cudaMemcpyAsync(valid, a.valid, (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaMemcpyAsync(plane, a.plane, (size_t)n * 16, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaMemcpyAsync(score, a.score, (size_t)n * 8, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

extern "C" int liliom_correspond_surf(liliom_ctx* c, const void* feats, int n, int stride, const double pose7[7], double kd_max_radius,
                                      double surf_dist_thres, double w_gate, double lidar_const, unsigned char* valid, float* plane,
                                      double* score) {
    return correspond_surf_impl(c, feats, n, stride, pose7, kd_max_radius, surf_dist_thres, w_gate, lidar_const, false, 0.0, valid, plane, score);
}

extern "C" int liliom_correspond_surf_refl(liliom_ctx* c, const void* feats48, int n, const double pose7[7], double kd_max_radius,
                                           double surf_dist_thres, double w_gate, double lidar_const, double reflect_thres,
                                           unsigned char* valid, float* plane, double* score) {
    return correspond_surf_impl(c, feats48, n, 48, pose7, kd_max_radius, surf_dist_thres, w_gate, lidar_const, true, reflect_thres, valid, plane, score);
}

extern "C" int liliom_backend_edge_block(liliom_ctx* c, const double pose7_body[7], double s_weight, double cauchy_b, double out29[29]) {
    if (!c || !pose7_body || !out29 || !(cauchy_b > 0)) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    if (c->bk_kind != 1) { c->last_error = "liliom_backend_edge_block needs the correspondences of a preceding liliom_correspond_edge call"; return LILIOM_E_ARG; }
    BlkSeg s = single_seg(c, true, pose7_body);
    s.pa = c->corr_plane.as<float>(); s.pb = s.pa + 3 * (size_t)c->bk_n;
    s.s_weight = s_weight;
    BlkCommon a{};
    a.cauchy_b = cauchy_b;
    return backend_block_run(c, {s}, a, out29);
}

extern "C" int liliom_backend_surf_block(liliom_ctx* c, const double pose7_body[7], const double q_lb_wxyz[4], const double t_lb[3],
                                         double cauchy_b, double out29[29]) {
    if (!c || !pose7_body || !q_lb_wxyz || !t_lb || !out29 || !(cauchy_b > 0)) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    if (c->bk_kind != 2) { c->last_error = "liliom_backend_surf_block needs the correspondences of a preceding liliom_correspond_surf* call"; return LILIOM_E_ARG; }
    BlkSeg s = single_seg(c, false, pose7_body);
    s.plane = c->corr_plane.as<float4>(); s.score = c->nn_sqd.as<double>();
    BlkCommon a{};
    a.qlb_inv = q_inverse(q_lb_wxyz);
    a.tlb = D3{t_lb[0], t_lb[1], t_lb[2]};
    a.cauchy_b = cauchy_b;
    return backend_block_run(c, {s}, a, out29);
}

// ===================== SURVEY §8 (f5): the window's LiDAR rows against the device-resident local map =====================
extern "C" int liliom_backend_window_correspond(liliom_ctx* c, const liliom_backend_params* bp, const int* kf_ids, const double* poses7_lidar,
                                                int k, int* n_edge_corr, int* n_surf_corr) {
    if (!c || !bp || !kf_ids || !poses7_lidar || !n_edge_corr || !n_surf_corr || k < 1 || k > kWinMax) return LILIOM_E_ARG;
    if (c->nranks > 1 || (bp->variant != 0 && bp->variant != 1) || !(bp->kd_max_radius > 0) || !(bp->cauchy_b > 0)) return LILIOM_E_ARG;
    for (int i = 0; i < k; ++i) {
        n_edge_corr[i] = n_surf_corr[i] = 0;
        if (kf_ids[i] < 0 || kf_ids[i] >= (int)c->kfs.size()) { c->last_error = "unknown keyframe id"; return LILIOM_E_ARG; }
    }
    if (bp->variant == 0 && c->prm.point_stride != 48) {
        c->last_error = "variant 0 weights the planes by reflectivity: it needs 48-byte points";
        return LILIOM_E_ARG;
    }
    LILI_CUDA(c, cudaSetDevice(c->device));
    c->win_k = 0;
    if (!c->bmap_built) return LILIOM_E_NOMAP;
    {
        const float cell = 1.0f / c->bmap[1].grid.inv_cell;
        if (c->bmap_n[1] > 0 && bp->kd_max_radius > (double)cell * (double)cell) {
            c->last_error = "kd_max_radius exceeds the cell size the surf layer was built with (liliom_bmap_build's kd_max_radius)";
            return LILIOM_E_ARG;
        }
    }
    if (!(c->bmap_n[1] > 50 && c->bmap_n[0] > 0)) return LILIOM_E_FEWMAP;        // L:933
    const int stride = c->prm.point_stride;
    BkArgs ae{}, as{};
    for (BkArgs* a : {&ae, &as}) {
        a->qpts = (const unsigned char*)c->kf_arena.p; a->qstride = stride; a->k = k; a->start[0] = 0;
    }
    for (int i = 0; i < k; ++i) {
        const KfEntry& f = c->kfs[kf_ids[i]];
        const double* p = poses7_lidar + 7 * (size_t)i;
        for (BkArgs* a : {&ae, &as}) { a->q[i] = Q4{p[0], p[1], p[2], p[3]}; a->t[i] = D3{p[4], p[5], p[6]}; }
        ae.qoff[i] = f.edge_off; ae.start[i + 1] = ae.start[i] + f.n_edge;
        as.qoff[i] = f.surf_off; as.start[i + 1] = as.start[i] + f.n_surf;
    }
    const long long Qe = ae.start[k], Qs = as.start[k];
    LILI_CUDA(c, c->win_valid[0].ensure((size_t)Qe + 16));
    LILI_CUDA(c, c->win_line.ensure((size_t)Qe * 24 + 16));
    LILI_CUDA(c, c->win_valid[1].ensure((size_t)Qs + 16));
    LILI_CUDA(c, c->win_plane.ensure((size_t)Qs * 16 + 16));
    LILI_CUDA(c, c->win_score.ensure((size_t)Qs * 8 + 16));
    LILI_CUDA(c, c->win_cnt.ensure(2 * kWinMax * sizeof(int)));
    // edge: L:1531-1599 / R:1394-1462 against edge_local_map_ds
    bk_set_map(ae, c->bmap[0]);
    ae.variant = bp->variant;
    ae.tau0 = knn_gate_tau(1.0);
    ae.valid = c->win_valid[0].as<unsigned char>(); ae.pa = c->win_line.as<float>(); ae.pb = ae.pa + 3 * (size_t)Qe;
    LILI_TRY(search_launch(c, true, ae));
    // surf: L:1601-1681 / R:1464-1520 against surf_local_map_ds
    bk_set_map(as, c->bmap[1]);
    as.variant = bp->variant;
    as.tau0 = knn_gate_tau(bp->kd_max_radius);
    as.max_sqd = bp->kd_max_radius; as.plane_thres = bp->surf_dist_thres; as.w_gate = bp->w_gate; as.lidar_const = bp->lidar_const;
    if (bp->variant == 0) { as.map_refl = c->bmap[1].refl.as<float>(); as.reflect_thres = bp->reflect_thres; }
    as.valid = c->win_valid[1].as<unsigned char>(); as.plane = c->win_plane.as<float4>(); as.score = c->win_score.as<double>();
    LILI_TRY(search_launch(c, false, as));
    CntArgs ca{};
    ca.valid[0] = ae.valid; ca.valid[1] = as.valid; ca.cnt = c->win_cnt.as<int>();
    for (int i = 0; i <= k; ++i) { ca.start[0][i] = ae.start[i]; ca.start[1][i] = as.start[i]; }
    k_win_count<<<dim3(k, 2), 256, 0, c->stream>>>(ca);
    LILI_TRY(launch_check(c, "k_win_count"));
    int cnt[2 * kWinMax];
    LILI_TRY(read_back(c, {{cnt, c->win_cnt.p, sizeof(cnt)}}));
    for (int i = 0; i < k; ++i) { n_edge_corr[i] = cnt[i]; n_surf_corr[i] = cnt[kWinMax + i]; }
    c->win_ids.assign(kf_ids, kf_ids + k);
    c->win_qoff[0].assign(ae.start, ae.start + k + 1);
    c->win_qoff[1].assign(as.start, as.start + k + 1);
    c->win_bp = *bp;
    c->win_k = k;
    return LILIOM_OK;
}

extern "C" int liliom_backend_window_blocks(liliom_ctx* c, const double* poses7_body, int k, double* out29) {
    if (!c || !poses7_body || !out29 || k < 1) return LILIOM_E_ARG;
    if (k != c->win_k) {
        c->last_error = "liliom_backend_window_blocks needs the k of the window left resident by liliom_backend_window_correspond";
        return LILIOM_E_ARG;
    }
    LILI_CUDA(c, cudaSetDevice(c->device));
    const liliom_backend_params& bp = c->win_bp;
    const int stride = c->prm.point_stride;
    const long long Qe = c->win_qoff[0][k];
    std::vector<BlkSeg> segs((size_t)2 * k);
    for (int i = 0; i < k; ++i) {
        const KfEntry& f = c->kfs[c->win_ids[i]];
        const double* p = poses7_body + 7 * (size_t)i;
        for (int kind = 0; kind < 2; ++kind) {     // segment 2i = edge rows, 2i + 1 = surf rows of keyframe i
            BlkSeg& s = segs[2 * (size_t)i + kind];
            const long long q0 = c->win_qoff[kind][i];
            s.n = (int)(c->win_qoff[kind][i + 1] - q0);
            s.nblocks = seg_blocks(s.n);
            s.edge = kind == 0;
            s.qpts = (const unsigned char*)c->kf_arena.p + (size_t)(kind == 0 ? f.edge_off : f.surf_off) * stride;
            s.qstride = stride;
            s.valid = c->win_valid[kind].as<unsigned char>() + q0;
            if (kind == 0) { s.pa = c->win_line.as<float>() + 3 * (size_t)q0; s.pb = c->win_line.as<float>() + 3 * (size_t)(Qe + q0); }
            else { s.plane = c->win_plane.as<float4>() + q0; s.score = c->win_score.as<double>() + q0; }
            s.q = Q4{p[0], p[1], p[2], p[3]}; s.t = D3{p[4], p[5], p[6]};
            s.wvariant = bp.variant;
            s.n_corr = c->win_cnt.as<int>() + kind * kWinMax + i;
            s.lidar_const = bp.lidar_const;
        }
    }
    BlkCommon a{};
    a.qlb_inv = q_inverse(bp.q_lb);
    a.tlb = D3{bp.t_lb[0], bp.t_lb[1], bp.t_lb[2]};
    a.cauchy_b = bp.cauchy_b;
    return backend_block_run(c, segs, a, out29);
}

extern "C" int liliom_backend_window_corr(liliom_ctx* c, int slot, int kind, unsigned char* valid, void* a, void* b, int cap, int* n_out) {
    if (!c || !n_out || slot < 0 || slot >= c->win_k || (kind != 0 && kind != 1)) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    const long long q0 = c->win_qoff[kind][slot];
    const int n = (int)(c->win_qoff[kind][slot + 1] - q0);
    *n_out = n;
    if (n > cap && (valid || a || b)) return LILIOM_E_CAPACITY;
    if (n == 0) return LILIOM_OK;
    if (valid) LILI_CUDA(c, cudaMemcpyAsync(valid, c->win_valid[kind].as<unsigned char>() + q0, (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    if (kind == 0) {
        const long long Qe = c->win_qoff[0][c->win_k];
        if (a) LILI_CUDA(c, cudaMemcpyAsync(a, c->win_line.as<float>() + 3 * (size_t)q0, (size_t)n * 12, cudaMemcpyDeviceToHost, c->stream));
        if (b) LILI_CUDA(c, cudaMemcpyAsync(b, c->win_line.as<float>() + 3 * (size_t)(Qe + q0), (size_t)n * 12, cudaMemcpyDeviceToHost, c->stream));
    } else {
        if (a) LILI_CUDA(c, cudaMemcpyAsync(a, c->win_plane.as<float4>() + q0, (size_t)n * 16, cudaMemcpyDeviceToHost, c->stream));
        if (b) LILI_CUDA(c, cudaMemcpyAsync(b, c->win_score.as<double>() + q0, (size_t)n * 8, cudaMemcpyDeviceToHost, c->stream));
    }
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}
