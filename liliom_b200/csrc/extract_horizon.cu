// Livox-Horizon feature extraction on sm_90a — replaces the loops of
// Preprocessing::cloudHandler, L/src/Preprocessing.cpp:225-383:
//   k_hz_flags     removeNaN (:225) + removeClosedPointCloud 0.1 m (:72-97,226) + scan_id>=0 (:253)
//   (scan)         stable compaction index = position in lidar_cloud_cutted
//   k_hz_deskew_bin  undistortion (:104-127) -> cutted cloud (:257); range/reflectivity gates
//                  (:259-261); time column (:262); first-writer-wins cell occupancy (:265-267)
//                  via atomicMin on the point index (the reference loop is sequential)
//   k_hz_patch     one warp per 6x6 patch (664 patches, :270): PCA of the valid cells (:271-298),
//                  per-line depth-Laplacian arg-max (:302-331), edge PCA + gate (:333-365),
//                  planar gate (:367-382).  Patches are independent (SURVEY.md App. C.5).
//   k_hz_offsets / k_hz_emit   patch-major ordered compaction into the published clouds.
// Compiled with --fmad=false: every fp32/fp64 expression rounds as in the reference's
// non-FMA x86-64 build, so labels and feature indices are bit-exact against the oracle.
#include "ctx.cuh"
#include "dev_math.cuh"
#include <climits>

namespace lili {

constexpr int HZ_LINES = 6;       // N_SCANS, Preprocessing.cpp:34
constexpr int HZ_COLS = 4000;     // H_SCANS, Preprocessing.cpp:35
constexpr int HZ_PATCHES = 664;   // i = 5 .. 3983 step 6
constexpr int HZ_EMPTY = INT_MAX;

struct Pt48 { float4 a, b, c; };  // {x,y,z,1} {nx,ny,nz,0} {intensity,curvature,0,0}

__device__ __forceinline__ int hz_keep(const Pt48* __restrict__ pts, int i) {
    float4 a = pts[i].a;
    float inten = pts[i].c.x;
    const float thres = 0.1f;
    bool fin = isfinite(a.x) && isfinite(a.y) && isfinite(a.z);
    bool close = (a.x * a.x + a.y * a.y + a.z * a.z) < thres * thres;
    int scan_id = (int)inten;
    return fin && !close && scan_id >= 0;
}

__global__ void k_hz_flags(const Pt48* __restrict__ pts, int n, int* __restrict__ flags) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    flags[i] = i < n ? hz_keep(pts, i) : 0;
}

__global__ void k_hz_fill(int* __restrict__ mat, int n, int v) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) mat[i] = v;
}

// one kept point: undistort, write it at position ci of the cutted cloud, claim its (line, column) cell
__device__ __forceinline__ void hz_deskew_bin_point(const Pt48* __restrict__ pts, int i, int ci, const Q4& q_imu, Pt48* __restrict__ cut,
                                                    int* __restrict__ mat) {
    const float4 a = pts[i].a;
    const float intensity = pts[i].c.x, curvature = pts[i].c.y;
    const int scan_id = (int)intensity;
    // undistortion, :104-127
    int line = (int)intensity;
    double dt_i = (double)(intensity - (float)line);
    double ratio_i = dt_i / 0.1;
    if (ratio_i >= 1.0) ratio_i = 1.0;
    Q4 q_si = qslerp_x(Q4{1, 0, 0, 0}, ratio_i, q_imu);
    D3 ps = qrot_x(q_si, D3{(double)a.x, (double)a.y, (double)a.z});
    const float ux = (float)ps.x, uy = (float)ps.y, uz = (float)ps.z;
    Pt48 o;
    o.a = make_float4(ux, uy, uz, 1.0f);
    o.b = make_float4(0.f, 0.f, 0.f, 0.f);
    o.c = make_float4(intensity, curvature, 0.f, 0.f);
    cut[ci] = o;
    double dep = (double)(ux * ux + uy * uy + uz * uz);                                          // :259
    if (dep > 40000.0 || dep < 4.0 || (double)curvature < 0.05 || (double)curvature > 25.45) return;   // :260
    const double t_interval = 0.1 / (HZ_COLS - 1);                                               // :239
    int col = (int)round((double)(intensity - (float)scan_id) / t_interval);                     // :262
    if (col >= HZ_COLS || col < 0) return;
    if (scan_id >= HZ_LINES) return;   // the reference indexes mat[] out of bounds here (UB); guarded
    atomicMin(&mat[scan_id * HZ_COLS + col], ci);                                                // :265-267 first writer wins
}

__global__ void k_hz_deskew_bin(const Pt48* __restrict__ pts, int n, const int* __restrict__ flags, const int* __restrict__ cidx,
                                Q4 q_imu, Pt48* __restrict__ cut, int* __restrict__ mat) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !flags[i]) return;
    hz_deskew_bin_point(pts, i, cidx[i], q_imu, cut, mat);
}

struct HzCell { float x, y, z, curv, inten, depth; };

constexpr int HZ_WIN = 14;   // columns i-4 .. i+9
constexpr int HZ_WARPS = 4;

// One warp per patch.  The reference's patch body is a chain of short sequential reductions; every
// reduction keeps its exact left-to-right order here (bit-exact labels), but independent reductions run
// on different lanes at the same time: the 36 depth-Laplacians, the 6 per-line arg-max scans, the two
// centroids (3+3 lanes), the two scatter matrices (6+6 lanes) and the two 3x3 eigen-solves (2 lanes).
struct HzPatchSmem {
    HzCell win[HZ_LINES * HZ_WIN];
    double g1[36];            // depth Laplacian of patch cell e = j*6+k (valid cells only)
    int    ids_y[HZ_LINES];   // arg-max column offset per line, -1 = none
    int    list_s[36];        // valid cells in (j,k) order  (indices into win)
    int    list_e[6];         // edge candidates in line order
    double cen[6];            // surf centre xyz, edge centre xyz
    double cov[12];           // surf a00,a10,a20,a11,a21,a22 ; edge likewise
    double ev[6];             // eigenvalues surf[3], edge[3]
    float  nrm[6];            // surf normal (evec col 0), edge direction (evec col 2)
    int    out_s[36], out_e[6];
    int    ns, ne, num, nedge;
    double sxyz[36 * 3], exyz[6 * 3];   // coordinates of the listed cells, widened once, in list order (centroid / scatter loops)
};

// Evaluates one patch with one warp: fills P (window, lists, normals, out_s/out_e, ns/ne).
template <bool COHERENT>
__device__ __forceinline__ void hz_patch_eval(HzPatchSmem& P, const Pt48* __restrict__ cut, const int* __restrict__ mat, int patch, int lane,
                                              double surf_thres, double edge_thres, long long* st = nullptr) {
#define HZ_ST(i) do { if (st) st[i] = clock64(); } while (0)
    const int i0 = 5 + 6 * patch;
    HzCell* W = P.win;
    for (int e = lane; e < HZ_LINES * HZ_WIN; e += 32) {
        int k = e / HZ_WIN, cc = e % HZ_WIN;
        // COHERENT: mat / cut were produced earlier in the same (cooperative) launch by other SMs -> bypass L1
        int idx = COHERENT ? __ldcg(&mat[k * HZ_COLS + (i0 - 4 + cc)]) : mat[k * HZ_COLS + (i0 - 4 + cc)];
        HzCell h{0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (idx != HZ_EMPTY) {
            float4 a = COHERENT ? __ldcg(&cut[idx].a) : cut[idx].a, c = COHERENT ? __ldcg(&cut[idx].c) : cut[idx].c;
            h.x = a.x; h.y = a.y; h.z = a.z; h.inten = c.x; h.curv = c.y;
            h.depth = sqrtf(a.x * a.x + a.y * a.y + a.z * a.z);                                   // getDepth :99-102
        }
        W[e] = h;
    }
    __syncwarp();
    HZ_ST(0);      // window loaded
    auto cell_of = [](int e) { return (e % 6) * HZ_WIN + (e / 6 + 4); };   // patch cell e = j*6+k -> window index (k, j)
    // ---- (1) validity + depth Laplacian of the 36 patch cells, :276-279 and :310-315
    for (int e = lane; e < 36; e += 32) {
        const int k = e % 6, j = e / 6;
        const HzCell* R = W + k * HZ_WIN + 4;   // R[j] = (k, i0 + j)
        double g = 0.0;
        if (R[j].curv > 0) {
            g = (double)R[j - 4].depth + (double)R[j - 3].depth + (double)R[j - 2].depth + (double)R[j - 1].depth - 8 * (double)R[j].depth +
                (double)R[j + 1].depth + (double)R[j + 2].depth + (double)R[j + 3].depth + (double)R[j + 4].depth;
            g = g / (8 * (double)R[j].depth + 1e-3);
        }
        P.g1[e] = g;
    }
    __syncwarp();
    // ---- (2) per-line arg-max g1 > 0.06, :302-331 (lanes 0..5), and the ordered list of valid cells (lane 6)
    if (lane < HZ_LINES) {
        double max_s = 0;
        int idx = -1;
        for (int j = 0; j < 6; ++j) {
            if (W[lane * HZ_WIN + j + 4].curv <= 0) continue;
            const double g1 = P.g1[j * 6 + lane];
            if (g1 > 0.06 && g1 > max_s) { max_s = g1; idx = j; }
        }
        P.ids_y[lane] = (max_s != 0) ? idx : -1;
    }
    {   // ordered list of the valid cells (e = j*6 + k ascending): two ballots + prefix popcounts instead of a 36-step serial walk
        const bool v0 = W[cell_of(lane)].curv > 0;
        const bool v1 = lane < 4 && W[cell_of(32 + lane)].curv > 0;
        const unsigned m0 = __ballot_sync(0xffffffffu, v0), m1 = __ballot_sync(0xffffffffu, v1);
        const unsigned lt = (1u << lane) - 1u;
        if (v0) P.list_s[__popc(m0 & lt)] = cell_of(lane);
        if (v1) P.list_s[__popc(m0) + __popc(m1 & lt)] = cell_of(32 + lane);
        if (lane == 0) P.num = __popc(m0) + __popc(m1);
    }
    __syncwarp();
    if (lane == 0) {
        int n = 0;
        for (int k = 0; k < HZ_LINES; ++k) if (P.ids_y[k] >= 0) P.list_e[n++] = k * HZ_WIN + P.ids_y[k] + 4;
        P.nedge = n;
        P.ns = 0; P.ne = 0;
    }
    __syncwarp();
    const int num = P.num, nedge = P.nedge;
    HZ_ST(1);      // Laplacians, arg-max, lists
    if (num >= 25) {                                                                              // :287 (else: `continue`, no edge either)
        // the listed cells' coordinates, gathered by the whole warp into list order: the sequential fp64 sums below then read
        // consecutive doubles instead of chasing list -> window -> field per step (measured: 12k cycles for the two loops)
        for (int e = lane; e < num; e += 32) {
            const HzCell& h = W[P.list_s[e]];
            P.sxyz[3 * e] = (double)h.x; P.sxyz[3 * e + 1] = (double)h.y; P.sxyz[3 * e + 2] = (double)h.z;
        }
        if (lane < nedge) {
            const HzCell& h = W[P.list_e[lane]];
            P.exyz[3 * lane] = (double)h.x; P.exyz[3 * lane + 1] = (double)h.y; P.exyz[3 * lane + 2] = (double)h.z;
        }
        __syncwarp();
        // ---- (3) centroids: lanes 0-2 surf xyz (:280-289), lanes 3-5 edge xyz (:335-342); sequential sums
        if (lane < 6) {
            const bool is_e = lane >= 3;
            const int comp = lane % 3;
            const double* arr = is_e ? P.exyz : P.sxyz;
            const int len = is_e ? nedge : num;
            double acc = 0.0;
#pragma unroll 4
            for (int t = 0; t < len; ++t) acc += arr[3 * t + comp];
            if (len > 0) acc /= len;
            P.cen[lane] = acc;
        }
        __syncwarp();
        // ---- (4) scatter matrices: lanes 0-5 surf, 6-11 edge; entries (0,0),(1,0),(2,0),(1,1),(2,1),(2,2)  (:291-296, :344-349)
        if (lane < 12) {
            const bool is_e = lane >= 6;
            const int ent = lane % 6;
            const int r = ent == 0 ? 0 : ent == 1 ? 1 : ent == 2 ? 2 : ent == 3 ? 1 : 2;
            const int c = ent <= 2 ? 0 : ent == 3 ? 1 : ent == 4 ? 1 : 2;
            const double* arr = is_e ? P.exyz : P.sxyz;
            const int len = is_e ? nedge : num;
            const double cr = P.cen[(is_e ? 3 : 0) + r], cc = P.cen[(is_e ? 3 : 0) + c];
            double acc = 0.0;
#pragma unroll 4
            for (int t = 0; t < len; ++t) {
                const double vr = arr[3 * t + r] - cr;
                const double vc = arr[3 * t + c] - cc;
                acc += vr * vc;
            }
            P.cov[lane] = acc;
        }
        __syncwarp();
        HZ_ST(2);  // centroids + scatter matrices
        // ---- (5) the two eigen-solves side by side (:298, :351)
        if (lane < 2 && (lane == 0 || nedge > 0)) {
            const double* M = P.cov + 6 * lane;
            double ev[3], evec[3][3];
            eigen_sym3(M[0], M[1], M[2], M[3], M[4], M[5], ev, evec);
            P.ev[3 * lane] = ev[0]; P.ev[3 * lane + 1] = ev[1]; P.ev[3 * lane + 2] = ev[2];
            const int col = lane == 0 ? 0 : 2;
            P.nrm[3 * lane] = (float)evec[0][col]; P.nrm[3 * lane + 1] = (float)evec[1][col]; P.nrm[3 * lane + 2] = (float)evec[2][col];
        }
        __syncwarp();
        HZ_ST(3);  // eigen-solves
        // ---- (6) decisions, :353-382: the (at most six) edge candidates on lane 0, the surf list compacted by ballots
        unsigned long long flipped = 0, flipped_hi = 0;      // bit = window index of an emitted edge point (:363 curvature *= -1)
        int surf_ok = 0;
        if (lane == 0) {
            int ne = 0;
            if (nedge > 0 && P.ev[5] > edge_thres * P.ev[4] && nedge > 3) {                      // :353
                for (int m = 0; m < nedge; ++m) {
                    const int wi = P.list_e[m];
                    const HzCell& h = W[wi];
                    if (h.curv <= 0 && h.inten <= 0) continue;                                    // :356
                    P.out_e[ne++] = wi;
                    if (wi < 64) flipped |= 1ull << wi; else flipped_hi |= 1ull << (wi - 64);
                }
            }
            P.ne = ne;
            surf_ok = (P.ev[0] < surf_thres * P.ev[1]) ? 1 : 0;                                  // :367
        }
        flipped = __shfl_sync(0xffffffffu, flipped, 0); flipped_hi = __shfl_sync(0xffffffffu, flipped_hi, 0);
        surf_ok = __shfl_sync(0xffffffffu, surf_ok, 0);
        {
            auto keep = [&](int t) {                                                             // :371 still-valid cells, list order
                if (!surf_ok || t >= num) return false;
                const int wi = P.list_s[t];
                return !(wi < 64 ? ((flipped >> wi) & 1ull) : ((flipped_hi >> (wi - 64)) & 1ull));
            };
            const bool k0 = keep(lane), k1 = lane < 4 && keep(32 + lane);
            const unsigned m0 = __ballot_sync(0xffffffffu, k0), m1 = __ballot_sync(0xffffffffu, k1);
            const unsigned lt = (1u << lane) - 1u;
            if (k0) P.out_s[__popc(m0 & lt)] = P.list_s[lane];
            if (k1) P.out_s[__popc(m0) + __popc(m1 & lt)] = P.list_s[32 + lane];
            if (lane == 0) P.ns = __popc(m0) + __popc(m1);
        }
        __syncwarp();
        HZ_ST(4);  // decisions
    }
#undef HZ_ST
}

// Writes the patch's selected cells (P.out_s / P.out_e) as published points starting at dst_s / dst_e.
__device__ __forceinline__ void hz_patch_emit(const HzPatchSmem& P, int lane, Pt48* __restrict__ dst_s, Pt48* __restrict__ dst_e) {
    const HzCell* W = P.win;
    const int ns = P.ns, ne = P.ne;
    for (int s2 = lane; s2 < ns; s2 += 32) {
        const HzCell& h = W[P.out_s[s2]];
        Pt48 o;
        o.a = make_float4(h.x, h.y, h.z, 1.0f);
        o.b = make_float4(P.nrm[0], P.nrm[1], P.nrm[2], 0.f);
        o.c = make_float4(h.inten, h.curv, 0.f, 0.f);
        dst_s[s2] = o;
    }
    if (lane < ne) {
        const HzCell& h = W[P.out_e[lane]];
        Pt48 o;
        o.a = make_float4(h.x, h.y, h.z, 1.0f);
        o.b = make_float4(P.nrm[3], P.nrm[4], P.nrm[5], 0.f);
        o.c = make_float4(h.inten, h.curv, 0.f, 0.f);
        dst_e[lane] = o;
    }
}

__global__ void __launch_bounds__(HZ_WARPS * 32) k_hz_patch(const Pt48* __restrict__ cut, const int* __restrict__ mat,
                                                           double surf_thres, double edge_thres,
                                                           Pt48* __restrict__ stage_surf, Pt48* __restrict__ stage_edge,
                                                           int* __restrict__ counts) {
    __shared__ HzPatchSmem sm[HZ_WARPS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int patch = blockIdx.x * HZ_WARPS + warp;
    if (patch >= HZ_PATCHES) return;
    HzPatchSmem& P = sm[warp];
    hz_patch_eval<false>(P, cut, mat, patch, lane, surf_thres, edge_thres);
    if (lane == 0) { counts[patch] = P.ns; counts[HZ_PATCHES + 1 + patch] = P.ne; }
    hz_patch_emit(P, lane, stage_surf + patch * 36, stage_edge + patch * 6);
}

// counts layout: [0..663] surf counts, [664] spare, [665..1328] edge counts, [1329] spare.
// offs layout  : same, exclusive prefix; totals -> totals[0] (surf), totals[1] (edge).
__global__ void __launch_bounds__(1024) k_hz_offsets(const int* __restrict__ counts, int* __restrict__ offs, int* __restrict__ totals) {
    __shared__ int wsum[32];
    for (int part = 0; part < 2; ++part) {
        const int base = part * (HZ_PATCHES + 1);
        int t = threadIdx.x;
        int v = (t < HZ_PATCHES) ? counts[base + t] : 0;
        int lane = t & 31, warp = t >> 5;
        int inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
        if (lane == 31) wsum[warp] = inc;
        __syncthreads();
        if (warp == 0) {
            int w = wsum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += u; }
            wsum[lane] = w;
        }
        __syncthreads();
        int excl = inc - v + (warp > 0 ? wsum[warp - 1] : 0);
        if (t < HZ_PATCHES) offs[base + t] = excl;
        if (t == HZ_PATCHES - 1) totals[part] = excl + v;
        __syncthreads();
    }
}

__global__ void k_hz_emit(const Pt48* __restrict__ stage_surf, const Pt48* __restrict__ stage_edge, const int* __restrict__ counts,
                          const int* __restrict__ offs, Pt48* __restrict__ surf, Pt48* __restrict__ edge) {
    const int patch = blockIdx.x;
    const int t = threadIdx.x;   // 64 threads: 0..35 surf slots, 36..41 edge slots
    if (t < 36) {
        if (t < counts[patch]) surf[offs[patch] + t] = stage_surf[patch * 36 + t];
    } else if (t < 42) {
        int e = t - 36;
        if (e < counts[HZ_PATCHES + 1 + patch]) edge[offs[HZ_PATCHES + 1 + patch] + e] = stage_edge[patch * 6 + e];
    }
}

// ---------------------------------------------------------------------------------------
// The whole extractor as ONE cooperative launch (8 launches + a CUB scan otherwise, most of their ~75 us
// launch latency): three grid barriers separate the four dependent stages.
//   A  keep-flags counted per block (block b owns the contiguous points [b*chunk, (b+1)*chunk)); mat := EMPTY
//   B  block prefix = sum of the preceding blocks' counts -> stable compaction index; de-skew, cutted cloud,
//      first-writer-wins cell claims (atomicMin), exactly as k_hz_deskew_bin
//   C  one warp per patch (hz_patch_eval, L1 bypassed for data written in B); per-patch counts published
//   D  every warp sums the counts of the patches before its own (patch-major order of the reference) and
//      writes its selected cells straight from shared memory — no staging copy
// Same device functions as the multi-launch chain, so the bits are the chain's.
// ---------------------------------------------------------------------------------------
constexpr int HZC_THREADS = 256;
constexpr int HZC_WARPS = HZC_THREADS / 32;

// (A release-only variant of this barrier — one cumulative red.release by thread 0, no acquire fence; legal here because
// every cross-block read is an L2-scope load — was measured in round 1 and changed nothing: 4586/4629 vs 4653/4563 scans/s.
// These kernels spend their time in the stages, not in the three fences.)
__device__ __forceinline__ void hz_grid_barrier(unsigned int* bar, unsigned int target) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        atomicAdd(bar, 1u);
        while ((int)(*reinterpret_cast<volatile unsigned int*>(bar) - target) < 0) { }
        __threadfence();
    }
    __syncthreads();
}

__global__ void __launch_bounds__(HZC_THREADS) k_hz_coop(const Pt48* __restrict__ pts, int n, Q4 q_imu, double surf_thres, double edge_thres,
                                                         Pt48* __restrict__ cut, int* __restrict__ mat, int* __restrict__ blockcnt,
                                                         int* __restrict__ counts, int* __restrict__ totals, int* __restrict__ ncut_out,
                                                         Pt48* __restrict__ surf, Pt48* __restrict__ edge, unsigned int* __restrict__ ctl,
                                                         unsigned int call) {
    __shared__ HzPatchSmem sm[HZC_WARPS];
    __shared__ int wsum[HZC_WARPS];
    __shared__ int s_bpre;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int G = gridDim.x, b = blockIdx.x;
    // bit 31 of `call` (LILIOM_DEBUG_TIMING): block 0 leaves clock64 stamps of the stage boundaries in the spare control words
    long long* stamp = ((call >> 31) != 0u && b == 0 && tid == 0) ? reinterpret_cast<long long*>(ctl + 4) : nullptr;
    call &= 0x7fffffffu;
    if (stamp) { stamp[0] = clock64(); stamp[10] = (long long)globaltimer_ns(); }
    unsigned int* bar = ctl + (call & 3u);
    if (b == 0 && tid == 0) ctl[(call + 1u) & 3u] = 0u;      // the next launch's barrier word
    // ---- A
    for (int e = b * HZC_THREADS + tid; e < HZ_LINES * HZ_COLS; e += G * HZC_THREADS) mat[e] = HZ_EMPTY;
    const int chunk = (n + G - 1) / G;
    const int ipt = (chunk + HZC_THREADS - 1) / HZC_THREADS;
    const int j0 = tid * ipt, j1 = min(j0 + ipt, chunk);
    int mine = 0;
    for (int j = j0; j < j1; ++j) {
        const int i = b * chunk + j;
        if (i < n) mine += hz_keep(pts, i);
    }
    int inc = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    int tpre = inc - mine;
    for (int w = 0; w < warp; ++w) tpre += wsum[w];
    if (tid == HZC_THREADS - 1) blockcnt[b] = tpre + mine;
    hz_grid_barrier(bar, (unsigned int)G);
    if (stamp) stamp[1] = clock64();
    // ---- B
    if (warp == 0) {
        int pre = 0, tot = 0;
        for (int k = lane; k < G; k += 32) { const int v = __ldcg(&blockcnt[k]); tot += v; if (k < b) pre += v; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { pre += __shfl_xor_sync(0xffffffffu, pre, o); tot += __shfl_xor_sync(0xffffffffu, tot, o); }
        if (lane == 0) { s_bpre = pre; if (b == 0) *ncut_out = tot; }
    }
    __syncthreads();
    {
        int ci = s_bpre + tpre;
        for (int j = j0; j < j1; ++j) {
            const int i = b * chunk + j;
            if (i < n && hz_keep(pts, i)) { hz_deskew_bin_point(pts, i, ci, q_imu, cut, mat); ++ci; }
        }
    }
    hz_grid_barrier(bar, 2u * (unsigned int)G);
    if (stamp) stamp[2] = clock64();
    // ---- C  (host guarantees G * HZC_WARPS >= HZ_PATCHES: one patch per warp)
    const int patch = b * HZC_WARPS + warp;
    HzPatchSmem& P = sm[warp];
    if (patch < HZ_PATCHES) {
        hz_patch_eval<true>(P, cut, mat, patch, lane, surf_thres, edge_thres, (stamp && warp == 0) ? stamp + 5 : nullptr);
        if (lane == 0) { counts[patch] = P.ns; counts[HZ_PATCHES + 1 + patch] = P.ne; }
    }
    hz_grid_barrier(bar, 3u * (unsigned int)G);
    if (stamp) stamp[3] = clock64();
    // ---- D
    if (patch < HZ_PATCHES) {
        int os = 0, oe = 0;
        for (int k = lane; k < patch; k += 32) { os += __ldcg(&counts[k]); oe += __ldcg(&counts[HZ_PATCHES + 1 + k]); }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { os += __shfl_xor_sync(0xffffffffu, os, o); oe += __shfl_xor_sync(0xffffffffu, oe, o); }
        hz_patch_emit(P, lane, surf + os, edge + oe);
        if (patch == HZ_PATCHES - 1 && lane == 0) { totals[0] = os + P.ns; totals[1] = oe + P.ne; }
    }
    if (stamp) { stamp[4] = clock64(); stamp[11] = (long long)globaltimer_ns(); }
}

// raw points must already be in c->raw (n x 48 B).  Leaves cut/surf/edge on the device and the
// three counts in pinned host memory (returned through the pointers after a stream sync).
int horizon_extract_dev(liliom_ctx* c, int n, const double q_imu[4], int* n_surf, int* n_edge, int* n_cut, bool sync_counts) {
    const size_t npts = (size_t)(n > 0 ? n : 1);
    LILI_CUDA(c, c->cut.ensure(npts * sizeof(Pt48)));
    LILI_CUDA(c, c->surf.ensure((size_t)HZ_PATCHES * 36 * sizeof(Pt48)));
    LILI_CUDA(c, c->edge.ensure((size_t)HZ_PATCHES * 6 * sizeof(Pt48)));
    LILI_CUDA(c, c->flags.ensure((npts + 2) * sizeof(int)));
    LILI_CUDA(c, c->idx_a.ensure((npts + 2) * sizeof(int)));
    LILI_CUDA(c, c->hz_mat.ensure((size_t)HZ_LINES * HZ_COLS * sizeof(int)));
    LILI_CUDA(c, c->hz_stage_surf.ensure((size_t)HZ_PATCHES * 36 * sizeof(Pt48)));
    LILI_CUDA(c, c->hz_stage_edge.ensure((size_t)HZ_PATCHES * 6 * sizeof(Pt48)));
    LILI_CUDA(c, c->hz_counts.ensure((size_t)(4 * (HZ_PATCHES + 1) + 8) * sizeof(int)));
    Q4 q{q_imu[0], q_imu[1], q_imu[2], q_imu[3]};
    if (std::isnan(q.w) || std::isnan(q.x) || std::isnan(q.y) || std::isnan(q.z)) q = Q4{1, 0, 0, 0};   // :232-234
    const Pt48* raw = c->raw_src ? reinterpret_cast<const Pt48*>(c->raw_src) : c->raw.as<Pt48>();   // read-only input
    int* flags = c->flags.as<int>();
    int* cidx = c->idx_a.as<int>();
    int* mat = c->hz_mat.as<int>();
    int* counts = c->hz_counts.as<int>();
    int* offs = counts + 2 * (HZ_PATCHES + 1);
    int* totals = counts + 4 * (HZ_PATCHES + 1);
    const bool coop = c->sm_count * HZC_WARPS >= HZ_PATCHES && n > 0;
    if (coop) {
        // one cooperative launch; scratch: per-block counts behind the patch counts, barrier words in their own buffer
        if (!c->hz_ctl.p) {
            LILI_CUDA(c, c->hz_ctl.ensure(128 + (size_t)c->sm_count * sizeof(int)));
            LILI_CUDA(c, cudaMemsetAsync(c->hz_ctl.p, 0, c->hz_ctl.cap, c->stream));
            c->hz_coop_calls = 0;
        }
        unsigned int* ctl = c->hz_ctl.as<unsigned int>();
        int* blockcnt = reinterpret_cast<int*>(c->hz_ctl.as<unsigned char>() + 128);
        int* ncut_out = cidx + n;
        const Pt48* raw_c = raw;
        Pt48* cutp = c->cut.as<Pt48>(); Pt48* surfp = c->surf.as<Pt48>(); Pt48* edgep = c->edge.as<Pt48>();
        double st = c->prm.surf_thres, et = c->prm.edge_thres;
        unsigned int call = (c->hz_coop_calls & 0x7fffffffu) | (c->dbg_timing ? 0x80000000u : 0u);
        void* kargs[] = {&raw_c, &n, &q, &st, &et, &cutp, &mat, &blockcnt, &counts, &totals, &ncut_out, &surfp, &edgep, &ctl, &call};
        LILI_CUDA(c, cudaLaunchCooperativeKernel((const void*)k_hz_coop, dim3(c->sm_count), dim3(HZC_THREADS), kargs, 0, c->stream));
        LILI_TRY(launch_check(c, "k_hz_coop"));
        c->hz_coop_calls++;
    } else {
        k_hz_flags<<<cdiv(n + 1, 256), 256, 0, c->stream>>>(raw, n, flags);
        LILI_TRY(launch_check(c, "k_hz_flags"));
        LILI_TRY(exclusive_scan_i32(c, flags, cidx, n));
        k_hz_fill<<<cdiv(HZ_LINES * HZ_COLS, 256), 256, 0, c->stream>>>(mat, HZ_LINES * HZ_COLS, HZ_EMPTY);
        LILI_TRY(launch_check(c, "k_hz_fill"));
        if (n > 0) {
            k_hz_deskew_bin<<<cdiv(n, 128), 128, 0, c->stream>>>(raw, n, flags, cidx, q, c->cut.as<Pt48>(), mat);
            LILI_TRY(launch_check(c, "k_hz_deskew_bin"));
            if (c->early_cut_dst && c->early_cut_cap >= n) {      // only when no count can overflow the caller's buffer: an error return leaves it untouched
                const size_t cnt = (size_t)min(n, c->early_cut_cap);
                LILI_CUDA(c, cudaEventRecord(c->ev_ready, c->stream));
                LILI_CUDA(c, cudaStreamWaitEvent(c->copy_stream, c->ev_ready, 0));
                LILI_CUDA(c, cudaMemcpyAsync(c->early_cut_dst, c->cut.p, cnt * sizeof(Pt48), cudaMemcpyDeviceToHost, c->copy_stream));
                LILI_CUDA(c, cudaEventRecord(c->ev_copied, c->copy_stream));
                c->early_cut_issued = true;
            }
        }
        k_hz_patch<<<cdiv(HZ_PATCHES, HZ_WARPS), HZ_WARPS * 32, 0, c->stream>>>(c->cut.as<Pt48>(), mat, c->prm.surf_thres, c->prm.edge_thres,
                                                                                c->hz_stage_surf.as<Pt48>(), c->hz_stage_edge.as<Pt48>(), counts);
        LILI_TRY(launch_check(c, "k_hz_patch"));
        k_hz_offsets<<<1, 1024, 0, c->stream>>>(counts, offs, totals);
        LILI_TRY(launch_check(c, "k_hz_offsets"));
        k_hz_emit<<<HZ_PATCHES, 64, 0, c->stream>>>(c->hz_stage_surf.as<Pt48>(), c->hz_stage_edge.as<Pt48>(), counts, offs,
                                                    c->surf.as<Pt48>(), c->edge.as<Pt48>());
        LILI_TRY(launch_check(c, "k_hz_emit"));
    }
    c->d_nsurf = totals;
    c->n_surf_max = min(n, HZ_PATCHES * 36);
    if (!sync_counts) {          // resident pipeline: the counts stay on the device, no host round trip
        c->n_surf_dev = -1;
        *n_surf = *n_edge = *n_cut = -1;
        return LILIOM_OK;
    }
    int hp[3];
    LILI_TRY(read_back(c, {{hp, totals, 2 * sizeof(int)}, {hp + 2, cidx + n, sizeof(int)}}));
    *n_surf = hp[0]; *n_edge = hp[1]; *n_cut = hp[2];
    c->n_surf_dev = hp[0];
    return LILIOM_OK;
}

}  // namespace lili
