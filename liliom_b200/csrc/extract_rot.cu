// Spinning-LiDAR (LOAM-style) feature extraction on sm_90a — replaces the loops of
// Preprocessing::cloudHandler, R/src/Preprocessing.cpp:280-509.
//
//   k_rot_pre      removeNaN + removeClosedPointCloud 3.0 m (:280-281), elevation -> scanID
//                  (:315-347) or the driver's ring id (LILIOM_RING_FIELD), raw azimuth -atan2f(y,x)
//                  (:349); first/last surviving index; with the driver's times (LILIOM_TIME_FIELD)
//                  their min / max over the surviving points instead
//   k_rot_hp       the sequential `halfPassed` latch (:350-358) as a prefix-min: the first valid
//                  index whose (un-latched) azimuth passes startOri + pi (not launched with times)
//   (stable sort)  bucket by ring preserving arrival order == laserCloudScans[scanID] (:371,378-382)
//   k_rot_build    azimuth wrap (:350-365), relTime (:367; from the time with LILIOM_TIME_FIELD), intensity (:368), de-skew with
//                  q_lb*slerp*q_lb^-1 (:153-177) -> laserCloud; ring start/end
//   k_rot_curv     11-point curvature in the literal left-to-right fp32 order (:385-394)
//   k_rot_ring     one CTA per ring: its 6 segments in order (the picked[] marks of segment j
//                  are visible to segment j+1, :401-500): shared-memory bitonic sort by
//                  (curvature, index), then warp 0 walks the sorted list 32 candidates at a time
//                  (ballot for the next unpicked one) — <=2 sharp, <=10 less-sharp, +-5 neighbour
//                  suppression, <=4 flat, less-flat flags
//   k_rot_lf_*     per-ring pcl::VoxelGrid(0.6) of the less-flat points (:502-508), all rings
//                  in one batch with 64-bit (ring, voxel) keys
//   k_rot_edge_emit  ordered compaction of the <=10 edge picks per segment (:517-521)
// atan/atan2 use lili::det_atanf/det_atan2f (bit-identical to glibc 2.39, see detmath.h).
// Compiled with --fmad=false so every fp32 expression rounds like the reference's x86-64 build.
#include "ctx.cuh"
#include "dev_math.cuh"
#include "detmath.h"
#include "pc2_fields.h"
#include <climits>
#include <cstdlib>
#include <cstdint>
#include <cstdio>
#include <algorithm>

namespace lili {

struct Pt32 { float4 a, b; };   // {x,y,z,1} {intensity,0,0,0}

// One CTA of k_rot_ring per ring, ~122 KB of shared memory each (RingSmem): one CTA per SM, so 128 rings are one wave on a
// 132-SM H100.  Ring keys stay below the 255 sentinel (8-bit ring sort, 40-bit (ring, voxel) keys).
constexpr int ROT_MAX_RINGS = 128;
constexpr int ROT_SEG_CAP = 4096;          // max points per segment (ring <= ~24k points)
constexpr int ROT_RING_CAP = 16384;        // picked[] bytes per ring in shared memory
constexpr double ROT_PI = 3.14159265358979323846;   // M_PI

// meta layout (ints): [0] first idx, [1] last idx, [2] halfPassed idx, [3] n_valid (cloudSize),
// [4] error flag, [5] n_lessflat, [6] n_edge, [M_RF..M_RF+ROT_MAX_RINGS) ring_first, [M_RE..M_RE+ROT_MAX_RINGS) ring_end,
// [M_TMIN, M_TMAX) / [M_TMAX, M_SIZE): t_min / t_max as 64-bit order keys (LILIOM_TIME_FIELD; 8-byte aligned)
constexpr int M_FIRST = 0, M_LAST = 1, M_HP = 2, M_NVALID = 3, M_ERR = 4, M_NLF = 5, M_NEDGE = 6, M_RF = 8, M_RE = M_RF + ROT_MAX_RINGS,
              M_TMIN = M_RE + ROT_MAX_RINGS, M_TMAX = M_TMIN + 2, M_SIZE = M_TMAX + 2;
static_assert(M_TMIN % 2 == 0, "the time keys are 8-byte words");

// A double as an unsigned key with the same order (finite values): sign bit flipped for >= 0, every bit for < 0.
__device__ __forceinline__ unsigned long long rot_time_key(double t) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(t);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double rot_key_time(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

bool rot_lines_ok(int line_num, bool field) {
    return field ? (line_num >= 1 && line_num <= ROT_MAX_RINGS) : (line_num == 16 || line_num == 32 || line_num == 64);
}

__global__ void k_rot_meta_init(int* meta) {
    // t_min key starts at ~0 (both words -1), t_max key at 0
    for (int t = threadIdx.x; t < M_SIZE; t += blockDim.x)
        meta[t] = (t == M_LAST || t == M_TMIN || t == M_TMIN + 1) ? -1 : (t == M_FIRST || t == M_HP) ? INT_MAX : 0;
}

__device__ __forceinline__ bool rot_keep(float4 a) {
    const float thres = 3.0f;
    if (!(isfinite(a.x) && isfinite(a.y) && isfinite(a.z))) return false;
    return !(a.x * a.x + a.y * a.y + a.z * a.z < thres * thres);
}

// scanID of a point from its elevation through the reference's tables (:315-347), -1 for a table miss
__device__ __forceinline__ int rot_table_scan_id(float4 a, int n_scans) {
    float angle = (float)((double)(det_atanf(a.z / sqrtf(a.x * a.x + a.y * a.y)) * 180.0f) / ROT_PI);        // :315
    int scanID = 0;
    bool ok = true;
    if (n_scans == 16) {
        scanID = (int)((double)((angle + 15.0f) / 2.0f) + 0.5);
        if (scanID > (n_scans - 1) || scanID < 0) ok = false;
    } else if (n_scans == 32) {
        scanID = (int)(((double)angle + 92.0 / 3.0) * 3.0 / 4.0);
        if (scanID > (n_scans - 1) || scanID < 0) ok = false;
    } else {
        if ((double)angle >= -8.83) scanID = (int)((double)(2.0f - angle) * 3.0 + 0.5);
        else scanID = n_scans / 2 + (int)((-8.83 - (double)angle) * 2.0 + 0.5);
        if (angle > 2.0f || (double)angle < -24.33 || scanID > 50 || scanID < 0) ok = false;
    }
    return ok ? scanID : -1;
}

// rings: nullptr = the elevation tables; else the driver's ring id of each point, kept iff < n_scans (LILIOM_RING_FIELD: the
// only difference between the two modes)
// kTimed (LILIOM_TIME_FIELD): times[i] is the driver's time of each point; a non-finite time drops the point with the NaN
// points, the raw azimuth is not needed, and t_min / t_max over the surviving points are reduced per block, then one atomic per
// block on the order keys.  The azimuth instantiation is the kernel as it was without a time source.
constexpr int ROT_PRE_THREADS = 256;
template <bool kTimed>
__global__ void __launch_bounds__(ROT_PRE_THREADS) k_rot_pre(const Pt32* __restrict__ pts, const uint16_t* __restrict__ rings,
                                                             const double* __restrict__ times, int n, int n_scans, uint32_t* __restrict__ keys,
                                                             int* __restrict__ vals, float* __restrict__ ori, int* __restrict__ meta) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (!kTimed && i >= n) return;
    unsigned long long kmin = ~0ull, kmax = 0ull;
    if (i < n) {
        const float4 a = pts[i].a;
        uint32_t key = 255u;
        float o = 0.f;
        const double t = kTimed ? times[i] : 0.0;
        if (rot_keep(a) && (!kTimed || isfinite(t))) {
            atomicMin(&meta[M_FIRST], i);
            atomicMax(&meta[M_LAST], i);
            const int scanID = rings ? (rings[i] < (unsigned)n_scans ? (int)rings[i] : -1) : rot_table_scan_id(a, n_scans);
            if (!kTimed) o = -det_atan2f(a.y, a.x);                                                         // :349
            if (scanID >= 0) key = (uint32_t)scanID;
            if (kTimed) kmin = kmax = rot_time_key(t);
        }
        keys[i] = key;
        vals[i] = i;
        ori[i] = o;
    }
    if (!kTimed) return;
    __shared__ unsigned long long s_min[ROT_PRE_THREADS / 32], s_max[ROT_PRE_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, o));
        kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, o));
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s_min[warp] = kmin; s_max[warp] = kmax; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < ROT_PRE_THREADS / 32; ++w) { kmin = min(kmin, s_min[w]); kmax = max(kmax, s_max[w]); }
        if (kmin != ~0ull) {          // the block kept a point
            atomicMin(reinterpret_cast<unsigned long long*>(meta + M_TMIN), kmin);
            atomicMax(reinterpret_cast<unsigned long long*>(meta + M_TMAX), kmax);
        }
    }
}

__device__ __forceinline__ void rot_start_end(const Pt32* __restrict__ pts, const int* __restrict__ meta, float& startOri, float& endOri) {
    float4 f = pts[meta[M_FIRST]].a, l = pts[meta[M_LAST]].a;
    startOri = -det_atan2f(f.y, f.x);                                                                       // :285
    endOri = (float)((double)(-det_atan2f(l.y, l.x)) + 2 * ROT_PI);                                         // :286-288
    if ((double)(endOri - startOri) > 3 * ROT_PI) endOri = (float)((double)endOri - 2 * ROT_PI);            // :290-294
    else if ((double)(endOri - startOri) < ROT_PI) endOri = (float)((double)endOri + 2 * ROT_PI);
}

// un-latched branch of :350-358 for every valid point; the latch fires at the smallest such index
__global__ void k_rot_hp(const Pt32* __restrict__ pts, int n, const uint32_t* __restrict__ keys, const float* __restrict__ ori_raw,
                         int* __restrict__ meta) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || keys[i] == 255u) return;
    if (meta[M_FIRST] == INT_MAX) return;
    float startOri, endOri;
    rot_start_end(pts, meta, startOri, endOri);
    float ori = ori_raw[i];
    if ((double)ori < (double)startOri - ROT_PI / 2) ori = (float)((double)ori + 2 * ROT_PI);
    else if ((double)ori > (double)startOri + ROT_PI * 3 / 2) ori = (float)((double)ori - 2 * ROT_PI);
    if ((double)(ori - startOri) > ROT_PI) atomicMin(&meta[M_HP], i);
}

// kTimed: relTime from the point's time over [t_min, t_max] (pc2_rel_time); else from the azimuth rule (:350-367)
template <bool kTimed>
__global__ void k_rot_build(const Pt32* __restrict__ pts, int n, const uint32_t* __restrict__ skeys, const int* __restrict__ svals,
                            const float* __restrict__ ori_raw, const double* __restrict__ times, Q4 qIMU, Q4 q_lb, Pt32* __restrict__ cloud,
                            int* __restrict__ meta) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const uint32_t key = skeys[s];
    const uint32_t prev = s > 0 ? skeys[s - 1] : 0xffffffffu;
    if (key != prev) {
        if (s > 0 && prev != 255u) meta[M_RE + prev] = s;
        if (key != 255u) meta[M_RF + key] = s;
        if (key == 255u) meta[M_NVALID] = s;
    }
    if (s == n - 1 && key != 255u) { meta[M_RE + key] = n; meta[M_NVALID] = n; }
    if (key == 255u) return;
    const int i = svals[s];
    float relTime;
    if constexpr (kTimed) {                                                                                 // LILIOM_TIME_FIELD
        const double t_min = rot_key_time(*reinterpret_cast<const unsigned long long*>(meta + M_TMIN));
        const double t_max = rot_key_time(*reinterpret_cast<const unsigned long long*>(meta + M_TMAX));
        relTime = pc2_rel_time(times[i], t_min, t_max);
    } else {
        float startOri, endOri;
        rot_start_end(pts, meta, startOri, endOri);
        float ori = ori_raw[i];
        if (i <= meta[M_HP]) {                                                                              // :350-358
            if ((double)ori < (double)startOri - ROT_PI / 2) ori = (float)((double)ori + 2 * ROT_PI);
            else if ((double)ori > (double)startOri + ROT_PI * 3 / 2) ori = (float)((double)ori - 2 * ROT_PI);
        } else {                                                                                            // :359-365
            ori = (float)((double)ori + 2 * ROT_PI);
            if ((double)ori < (double)endOri - ROT_PI * 3 / 2) ori = (float)((double)ori + 2 * ROT_PI);
            else if ((double)ori > (double)endOri + ROT_PI / 2) ori = (float)((double)ori - 2 * ROT_PI);
        }
        relTime = (ori - startOri) / (endOri - startOri);                                                   // :367
    }
    const float intensity = (float)((double)(int)key + 0.1 * (double)relTime);                              // :368
    // undistortion, :153-177
    const int line = (int)intensity;
    double dt_i = (double)(intensity - (float)line);
    double ratio_i = dt_i / 0.1;
    if (ratio_i >= 1.0) ratio_i = 1.0;
    Q4 q_si = qslerp_x(Q4{1, 0, 0, 0}, ratio_i, qIMU);
    q_si = qmul_x(qmul_x(q_lb, q_si), qinv_x(q_lb));                                                        // :168
    const float4 a = pts[i].a;
    D3 ps = qrot_x(q_si, D3{(double)a.x, (double)a.y, (double)a.z});
    Pt32 o;
    o.a = make_float4((float)ps.x, (float)ps.y, (float)ps.z, 1.0f);
    o.b = make_float4(intensity, 0.f, 0.f, 0.f);
    cloud[s] = o;
}

__global__ void k_rot_curv(const Pt32* __restrict__ cloud, const int* __restrict__ meta, float* __restrict__ curv, int* __restrict__ label,
                           int* __restrict__ lessflat, int n_alloc) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n_alloc) return;
    const int cloudSize = meta[M_NVALID];
    float c = 0.f;
    if (i >= 5 && i < cloudSize - 5) {
        const float4 m5 = cloud[i - 5].a, m4 = cloud[i - 4].a, m3 = cloud[i - 3].a, m2 = cloud[i - 2].a, m1 = cloud[i - 1].a,
                     p0 = cloud[i].a, p1 = cloud[i + 1].a, p2 = cloud[i + 2].a, p3 = cloud[i + 3].a, p4 = cloud[i + 4].a, p5 = cloud[i + 5].a;
        float dX = m5.x + m4.x + m3.x + m2.x + m1.x - 10.0f * p0.x + p1.x + p2.x + p3.x + p4.x + p5.x;
        float dY = m5.y + m4.y + m3.y + m2.y + m1.y - 10.0f * p0.y + p1.y + p2.y + p3.y + p4.y + p5.y;
        float dZ = m5.z + m4.z + m3.z + m2.z + m1.z - 10.0f * p0.z + p1.z + p2.z + p3.z + p4.z + p5.z;
        c = dX * dX + dY * dY + dZ * dZ;                                                                    // :390
    }
    if (i < n_alloc) { curv[i] = c; label[i] = 0; }
    lessflat[i] = 0;   // includes the scan sentinel at n_alloc
}

// dynamic shared memory of k_rot_ring
constexpr int ROT_FAST_CAP = 1024;         // segments up to this many points take the mask walk (one 32-rank word per lane of warp 0)
struct RingSmem {
    unsigned long long keys[ROT_SEG_CAP];      // (curvature bits << 32) | index
    float4 pts[ROT_SEG_CAP + 16];              // segment window [sp-5, ep+5]
    unsigned char picked[ROT_RING_CAP];        // cloudNeighborPicked of this ring
    // mask walk (L <= ROT_FAST_CAP): the sorted order as ranks, everything a pick needs precomputed in parallel
    unsigned short ind_of_rank[ROT_FAST_CAP];  // segment-local point index at sorted rank r
    unsigned short rank_of[ROT_FAST_CAP];      // inverse
    unsigned char cls[ROT_FAST_CAP];           // by rank: bit 0 curvature > 2.0 (sharp candidate), bit 1 curvature < 0.1 and not within 0.5 m (flat candidate)
    unsigned char ext[ROT_FAST_CAP];           // by point: neighbours a pick marks, forward | backward << 4 (each 0..5)
    unsigned char brk[ROT_FAST_CAP + 16];      // by window index i: |p_i - p_(i-1)|^2 > 0.05 (:434-451's break test, one per consecutive pair)
    unsigned int availS[32], availF[32];       // by rank: still-unpicked sharp / flat candidates
};

__global__ void __launch_bounds__(512) k_rot_ring(const Pt32* __restrict__ cloud, const float* __restrict__ curv, int* __restrict__ meta,
                                                  int ds_rate, int* __restrict__ label, int* __restrict__ lessflat,
                                                  int* __restrict__ seg_edge /* [rings*6][10] */, int* __restrict__ seg_cnt /* [rings*6] */,
                                                  long long* __restrict__ dbg /* LILIOM_DEBUG_TIMING: [rings][8] cycles */,
                                                  int fast_cap /* ROT_FAST_CAP; 0 (LILIOM_ROT_SLOW_WALK, tests): every segment takes the general path */) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    RingSmem& S = *reinterpret_cast<RingSmem*>(smem_raw);
    const int ring = blockIdx.x;
    long long t_all = 0, t_load = 0, t_sort = 0, t_walk = 0, t_flag = 0, t0 = 0;
    const bool tm = dbg != nullptr && threadIdx.x == 0;
    if (tm) { t_all = clock64(); for (int k = 0; k < 7; ++k) dbg[ring * 8 + k] = 0; dbg[ring * 8 + 7] = (long long)globaltimer_ns(); }
    const int rf = meta[M_RF + ring], re = meta[M_RE + ring];
    const int scanStart = rf + 5, scanEnd = re - 6;                                                         // :379-381
    for (int j = 0; j < 6; ++j) if (threadIdx.x == 0) seg_cnt[ring * 6 + j] = 0;
    if (re <= rf) return;                                   // empty ring
    if (scanEnd - scanStart < 6 || ring % ds_rate != 0) return;                                             // :402
    const int ring_len = re - rf;
    if (ring_len > ROT_RING_CAP) { if (threadIdx.x == 0) meta[M_ERR] = 1; return; }
    for (int k = threadIdx.x; k < ring_len; k += blockDim.x) S.picked[k] = 0;
    __syncthreads();
    for (int j = 0; j < 6; ++j) {
        const int sp = scanStart + (scanEnd - scanStart) * j / 6;                                           // :406-407
        const int ep = scanStart + (scanEnd - scanStart) * (j + 1) / 6 - 1;
        const int L = ep - sp + 1;
        if (L > ROT_SEG_CAP) { if (threadIdx.x == 0) meta[M_ERR] = 1; return; }
        int P = 1;
        while (P < L) P <<= 1;
        if (tm) t0 = clock64();
        for (int k = threadIdx.x; k < P; k += blockDim.x) {
            unsigned long long key = ~0ull;
            if (k < L) key = ((unsigned long long)__float_as_uint(curv[sp + k]) << 32) | (unsigned)(sp + k);
            S.keys[k] = key;
        }
        for (int k = threadIdx.x; k < L + 10; k += blockDim.x) S.pts[k] = cloud[sp - 5 + k].a;
        __syncthreads();
        if (tm) { const long long t = clock64(); t_load += t - t0; t0 = t; }
        if (L <= fast_cap) {
            // ---- mask walk.  The walk over the sorted candidates (:413-492) is sequential only in its PICKS (<= 14 per segment):
            // whether a candidate qualifies (curvature class, range) and which neighbours a pick marks (the break test between
            // consecutive points) are static, so all of that is computed in parallel first, the sorted order becomes a rank per
            // point (counting sort: one barrier instead of the 45 of a bitonic network), and "the next unpicked candidate" is the
            // highest / lowest set bit of a 32-word availability mask that every pick clears bits in (the sorted walk it
            // replaces was a chain of dependent single-warp instructions per candidate; LILIOM_DEBUG_TIMING shows the stages).
            for (int t = threadIdx.x; t < L; t += blockDim.x) {
                const unsigned long long mine = S.keys[t];
                int r = 0;
#pragma unroll 8
                for (int q = 0; q < L; ++q) r += (S.keys[q] < mine) ? 1 : 0;       // keys are unique (the index is part of them)
                const float cv = __uint_as_float((unsigned)(mine >> 32));
                const float4& p = S.pts[t + 5];
                const bool nearp = (double)(p.x * p.x + p.y * p.y + p.z * p.z) < 0.25;             // :463-466 `continue`
                unsigned char cl = 0;
                if ((double)cv > 2.0) cl |= 1;                                                        // :416
                if ((double)cv < 0.1 && !nearp) cl |= 2;                                              // :459
                S.ind_of_rank[r] = (unsigned short)t;
                S.cls[r] = cl;
                S.rank_of[t] = (unsigned short)r;
            }
            for (int i = threadIdx.x + 1; i < L + 10; i += blockDim.x) {
                const float4& a = S.pts[i]; const float4& b = S.pts[i - 1];
                const float dX = a.x - b.x, dY = a.y - b.y, dZ = a.z - b.z;
                S.brk[i] = ((double)(dX * dX + dY * dY + dZ * dZ) > 0.05) ? 1 : 0;
            }
            if (threadIdx.x < 32) { S.availS[threadIdx.x] = 0u; S.availF[threadIdx.x] = 0u; }
            __syncthreads();
            for (int t = threadIdx.x; t < L; t += blockDim.x) {
                const int w = t + 5;
                int nf = 0, nb = 0;
                while (nf < 5 && !S.brk[w + nf + 1]) ++nf;       // forward: pairs (w+1,w), (w+2,w+1), ...
                while (nb < 5 && !S.brk[w - nb]) ++nb;           // backward: pairs (w,w-1), (w-1,w-2), ...
                S.ext[t] = (unsigned char)(nf | (nb << 4));
            }
            for (int base = 0; base < L; base += blockDim.x) {
                const int r = base + (int)threadIdx.x;
                bool sh = false, fl = false;
                if (r < L) {
                    const unsigned char cl = S.cls[r];
                    const bool un = S.picked[sp + (int)S.ind_of_rank[r] - rf] == 0;      // marks carried over from the previous segment
                    sh = (cl & 1) && un; fl = (cl & 2) && un;
                }
                const unsigned ms = __ballot_sync(0xffffffffu, sh), mf = __ballot_sync(0xffffffffu, fl);
                if ((threadIdx.x & 31) == 0 && r < L) { S.availS[r >> 5] = ms; S.availF[r >> 5] = mf; }
            }
            __syncthreads();
            if (tm) { const long long t = clock64(); t_sort += t - t0; t0 = t; }
            if (threadIdx.x < 32) {
                const unsigned full = 0xffffffffu;
                const int lane = threadIdx.x;
                // a pick at segment-local point t: lane 0 marks t, lanes 1-5 its forward and lanes 6-10 its backward neighbours up to the
                // first break; marked points leave both availability masks
                auto mark = [&](int t) {
                    const unsigned e = S.ext[t];
                    int q = t;
                    bool on = lane == 0;
                    if (lane >= 1 && lane <= 5) { on = lane <= (int)(e & 15u); q = t + lane; }
                    else if (lane >= 6 && lane <= 10) { on = lane - 5 <= (int)(e >> 4); q = t - (lane - 5); }
                    if (on) {
                        S.picked[sp + q - rf] = 1;
                        if (q >= 0 && q < L) {
                            const int rq = S.rank_of[q];
                            atomicAnd(&S.availS[rq >> 5], ~(1u << (rq & 31)));
                            atomicAnd(&S.availF[rq >> 5], ~(1u << (rq & 31)));
                        }
                    }
                    __syncwarp();
                };
                int largest = 0, nedge = 0;
                while (true) {                                                                              // :413-453
                    const unsigned m = S.availS[lane];
                    const unsigned any = __ballot_sync(full, m != 0u);
                    if (!any) break;
                    largest++;
                    if (largest > 10) break;
                    const int lw = 31 - __clz((int)any);
                    const unsigned mw = __shfl_sync(full, m, lw);
                    const int t = S.ind_of_rank[(lw << 5) + 31 - __clz((int)mw)];
                    if (lane == 0) { label[sp + t] = largest <= 2 ? 2 : 1; seg_edge[(ring * 6 + j) * 10 + nedge] = sp + t; }
                    nedge++;
                    mark(t);
                }
                if (lane == 0) seg_cnt[ring * 6 + j] = nedge;
                int smallest = 0;
                while (true) {                                                                              // :456-492
                    const unsigned m = S.availF[lane];
                    const unsigned any = __ballot_sync(full, m != 0u);
                    if (!any) break;
                    const int lw = __ffs((int)any) - 1;
                    const unsigned mw = __shfl_sync(full, m, lw);
                    const int t = S.ind_of_rank[(lw << 5) + __ffs((int)mw) - 1];
                    if (lane == 0) label[sp + t] = -1;
                    smallest++;
                    if (smallest >= 4) break;              // the fourth pick leaves no marks (:476-478)
                    mark(t);
                }
            }
        } else {
            // bitonic sort ascending on (curvature, index): curvature >= 0 so its bit pattern orders like the value
            for (int size = 2; size <= P; size <<= 1) {
                for (int stride = size >> 1; stride > 0; stride >>= 1) {
                    for (int t = threadIdx.x; t < P / 2; t += blockDim.x) {
                        int lo = 2 * t - (t & (stride - 1));
                        int hi = lo + stride;
                        bool up = ((lo & size) == 0);
                        unsigned long long a = S.keys[lo], b = S.keys[hi];
                        if ((a > b) == up) { S.keys[lo] = b; S.keys[hi] = a; }
                    }
                    __syncthreads();
                }
            }
            if (tm) { const long long t = clock64(); t_sort += t - t0; t0 = t; }
            // The picks are sequential by definition (a pick marks its +-5 neighbours, which later candidates must see), but the
            // candidates BETWEEN picks are not: warp 0 examines 32 sorted candidates at a time, a ballot finds the first one that
            // is still unpicked (or the first that ends the walk), and only that one is acted on before the scan resumes behind it
            // with the fresh marks.  Sequential steps = picks (<= 14 per segment), not candidates; one thread walking the list
            // spends most of the segment's cycles in that walk.
            if (threadIdx.x < 32) {
                const unsigned full = 0xffffffffu;
                const int lane = threadIdx.x;
                auto PT = [&](int ind) -> const float4& { return S.pts[ind - sp + 5]; };
                auto gap2 = [&](int a, int b) {
                    float dX = PT(a).x - PT(b).x, dY = PT(a).y - PT(b).y, dZ = PT(a).z - PT(b).z;
                    return dX * dX + dY * dY + dZ * dZ;
                };
                // :434-451 — lanes 0-4: ind+1..ind+5, lanes 5-9: ind-1..ind-5; each side marks up to its first gap > 0.05
                auto suppress = [&](int ind) {
                    bool brk = false;
                    int l = 0;
                    if (lane < 5) { l = lane + 1; brk = (double)gap2(ind + l, ind + l - 1) > 0.05; }
                    else if (lane < 10) { l = -(lane - 4); brk = (double)gap2(ind + l, ind + l + 1) > 0.05; }
                    const unsigned bm = __ballot_sync(full, brk);
                    const unsigned fwd = bm & 0x1fu, bwd = (bm >> 5) & 0x1fu;
                    const int nf = fwd ? __ffs(fwd) - 1 : 5, nb = bwd ? __ffs(bwd) - 1 : 5;
                    if (lane < 5) { if (lane < nf) S.picked[ind + l - rf] = 1; }
                    else if (lane < 10) { if (lane - 5 < nb) S.picked[ind + l - rf] = 1; }
                    __syncwarp();
                };
                int largest = 0, nedge = 0;
                bool done = false;
                for (int k = L - 1; !done && k >= 0;) {                                                         // :413-453
                    const int kk = k - lane;
                    bool stop = false, avail = false;
                    int ind = 0;
                    if (kk >= 0) {
                        const unsigned long long key = S.keys[kk];
                        ind = (int)(unsigned)(key & 0xffffffffu);
                        const float cv = __uint_as_float((unsigned)(key >> 32));
                        stop = !((double)cv > 2.0);       // sorted: nothing further can be picked (no side effects skipped)
                        avail = !stop && S.picked[ind - rf] == 0;
                    }
                    const unsigned ms = __ballot_sync(full, stop), ma = __ballot_sync(full, avail);
                    const int fs = ms ? __ffs(ms) - 1 : 32, fa = ma ? __ffs(ma) - 1 : 32;
                    if (fa < fs) {
                        largest++;
                        if (largest > 10) { done = true; continue; }
                        const int pind = __shfl_sync(full, ind, fa);
                        if (lane == 0) {
                            label[pind] = largest <= 2 ? 2 : 1;
                            seg_edge[(ring * 6 + j) * 10 + nedge] = pind;
                            S.picked[pind - rf] = 1;
                        }
                        nedge++;
                        __syncwarp();
                        suppress(pind);
                        k -= fa + 1;
                    } else if (fs < 32) done = true;
                    else k -= 32;
                }
                if (lane == 0) seg_cnt[ring * 6 + j] = nedge;
                int smallest = 0;
                done = false;
                for (int k = 0; !done && k < L;) {                                                              // :456-492
                    const int kk = k + lane;
                    bool stop = false, avail = false;
                    int ind = 0;
                    if (kk < L) {
                        const unsigned long long key = S.keys[kk];
                        ind = (int)(unsigned)(key & 0xffffffffu);
                        const float cv = __uint_as_float((unsigned)(key >> 32));
                        stop = !((double)cv < 0.1);       // sorted ascending: the rest cannot qualify
                        if (!stop) {
                            const float4& p = PT(ind);
                            const bool nearp = (double)(p.x * p.x + p.y * p.y + p.z * p.z) < 0.25;             // `continue`: no side effect
                            avail = !nearp && S.picked[ind - rf] == 0;
                        }
                    }
                    const unsigned ms = __ballot_sync(full, stop), ma = __ballot_sync(full, avail);
                    const int fs = ms ? __ffs(ms) - 1 : 32, fa = ma ? __ffs(ma) - 1 : 32;
                    if (fa < fs) {
                        const int pind = __shfl_sync(full, ind, fa);
                        if (lane == 0) label[pind] = -1;
                        smallest++;
                        if (smallest >= 4) { done = true; continue; }      // the fourth pick leaves no marks (:476-478)
                        if (lane == 0) S.picked[pind - rf] = 1;
                        __syncwarp();
                        suppress(pind);
                        k += fa + 1;
                    } else if (fs < 32) done = true;
                    else k += 32;
                }
            }
        }
        if (tm) { const long long t = clock64(); t_walk += t - t0; t0 = t; }
        __syncthreads();
        for (int k = sp + (int)threadIdx.x; k <= ep; k += blockDim.x) {                                     // :494-499
            const float4& p = S.pts[k - sp + 5];
            bool far = !((double)(p.x * p.x + p.y * p.y + p.z * p.z) < 0.25);
            lessflat[k] = (far && label[k] <= 0) ? 1 : 0;
        }
        __syncthreads();
        if (tm) { const long long t = clock64(); t_flag += t - t0; dbg[ring * 8 + 5] = max(dbg[ring * 8 + 5], (long long)L); }
    }
    if (tm) {
        dbg[ring * 8 + 0] = clock64() - t_all; dbg[ring * 8 + 1] = t_load; dbg[ring * 8 + 2] = t_sort; dbg[ring * 8 + 3] = t_walk; dbg[ring * 8 + 4] = t_flag;
        dbg[ring * 8 + 6] = (long long)globaltimer_ns();
    }
}

// ---- per-ring VoxelGrid(0.6) of the less-flat points, batched over rings
// ringmm: [ring][8] a box (vg_box.h) per ring, word 7 unused
__global__ void k_rot_lf_init(int* ringmm) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ROT_MAX_RINGS * 8) return;
    ringmm[t] = vg_box_empty(t & 7);
}

__global__ void k_rot_lf_gather(const Pt32* __restrict__ cloud, const uint32_t* __restrict__ skeys, const int* __restrict__ lessflat,
                                const int* __restrict__ lfpos, int n, int n_rings, int* __restrict__ lf_src, int* __restrict__ ringmm,
                                int* __restrict__ meta) {
    // per-ring boxes: block-local in shared memory first (the cloud is ring-major, so a block meets one to three rings), then one
    // set of global atomics per ring the block saw — per-point global atomics on 64 x 7 words cost this kernel 38 us
    __shared__ int s_mm[ROT_MAX_RINGS * 8];
    for (int t = threadIdx.x; t < n_rings * 8; t += blockDim.x) s_mm[t] = vg_box_empty(t & 7);
    __syncthreads();
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k == 0) meta[M_NLF] = lfpos[n];
    if (k < n && lessflat[k]) {
        lf_src[lfpos[k]] = k;
        const int ring = (int)skeys[k];
        float4 a = cloud[k].a;
        int* mm = s_mm + ring * 8;
        atomicMin(&mm[0], vg_f2ord(a.x)); atomicMin(&mm[1], vg_f2ord(a.y)); atomicMin(&mm[2], vg_f2ord(a.z));
        atomicMax(&mm[3], vg_f2ord(a.x)); atomicMax(&mm[4], vg_f2ord(a.y)); atomicMax(&mm[5], vg_f2ord(a.z));
        atomicAdd(&mm[6], 1);
    }
    __syncthreads();
    for (int t = threadIdx.x; t < n_rings * 8; t += blockDim.x) {
        const int f = t & 7;
        if (f == 7 || s_mm[(t & ~7) + 6] == 0) continue;          // ring not seen by this block
        vg_box_atomic(&ringmm[t], f, s_mm[t]);
    }
}

__global__ void k_rot_lf_params(const int* __restrict__ ringmm, float leaf, VgParams* __restrict__ prm) {
    int ring = threadIdx.x;
    if (ring >= ROT_MAX_RINGS) return;
    prm[ring] = vg_params(ringmm + ring * 8, leaf);
}

__global__ void k_rot_lf_keys(const Pt32* __restrict__ cloud, const uint32_t* __restrict__ skeys, const int* __restrict__ lf_src,
                              const int* __restrict__ meta, const VgParams* __restrict__ prm, unsigned long long* __restrict__ keys,
                              int* __restrict__ vals, int cap) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= cap) return;
    unsigned long long key = ~0ull;
    if (t < meta[M_NLF]) {
        const int k = lf_src[t];
        const int ring = (int)skeys[k];
        const VgParams p = prm[ring];
        float4 a = cloud[k].a;
        unsigned idx;
        if (p.overflow) idx = (unsigned)t;     // PCL returns the input unchanged: every point its own voxel, input order
        else idx = vg_rel_index(p, a.x, a.y, a.z);
        key = ((unsigned long long)ring << 32) | idx;
    }
    keys[t] = key;
    vals[t] = t;
}

__global__ void k_rot_lf_centroid(const Pt32* __restrict__ cloud, const int* __restrict__ lf_src, const unsigned long long* __restrict__ keys,
                                  const int* __restrict__ vals, const int* __restrict__ flags, const int* __restrict__ rank,
                                  const int* __restrict__ meta, int cap, Pt32* __restrict__ out, int* __restrict__ n_out) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t == 0) *n_out = rank[cap];
    if (t >= cap || !flags[t]) return;
    const VgAcc<32> a = vg_walk<32>(keys, t, meta[M_NLF], [&](int j) { return lf_src[vals[j]]; },
                                    [&](int m) { return reinterpret_cast<const unsigned char*>(cloud + m); });
    vg_write<32>(a.s, a.n, reinterpret_cast<unsigned char*>(out + rank[t]));
}

// edge output: segment-major, pick order inside the segment (one block, one thread per possible segment: 128*6 = 768)
constexpr int ROT_EMIT_THREADS = ROT_MAX_RINGS * 6;
__global__ void __launch_bounds__(ROT_EMIT_THREADS) k_rot_edge_emit(const Pt32* __restrict__ cloud, const int* __restrict__ seg_edge,
                                                                    const int* __restrict__ seg_cnt, int nseg, Pt32* __restrict__ edge,
                                                                    int* __restrict__ meta) {
    constexpr int nwarps = ROT_EMIT_THREADS / 32;
    __shared__ int wsum[nwarps];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    int v = t < nseg ? seg_cnt[t] : 0;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    if (t == 0) { int acc = 0; for (int w = 0; w < nwarps; ++w) { int x = wsum[w]; wsum[w] = acc; acc += x; } meta[M_NEDGE] = acc; }
    __syncthreads();
    const int off = inc - v + wsum[warp];
    for (int e = 0; e < v; ++e) edge[off + e] = cloud[seg_edge[t * 10 + e]];
}

int rot_extract_dev(liliom_ctx* c, int n, const double q_imu[4], const double q_lb[4], int* n_surf, int* n_edge, int* n_cut,
                    const uint16_t* rings, const double* times) {
    const int n_scans = c->prm.line_num;
    if (!rot_lines_ok(n_scans, rings != nullptr)) return LILIOM_E_LINES;
    if (c->prm.ds_rate < 1) return LILIOM_E_ARG;
    *n_surf = *n_edge = *n_cut = 0;
    c->n_surf_dev = 0; c->n_rot_cloud = 0;
    if (n <= 0) return LILIOM_OK;
    const size_t N = (size_t)n;
    LILI_CUDA(c, c->rot_keys.ensure(N * 8)); LILI_CUDA(c, c->rot_keys2.ensure(N * 8));
    LILI_CUDA(c, c->rot_vals.ensure(N * 4)); LILI_CUDA(c, c->rot_vals2.ensure(N * 4));
    LILI_CUDA(c, c->rot_ring.ensure(N * 4));                 // raw azimuth
    LILI_CUDA(c, c->rot_cloud.ensure(N * sizeof(Pt32)));
    LILI_CUDA(c, c->cut.ensure(N * sizeof(Pt32)));
    LILI_CUDA(c, c->rot_curv.ensure(N * 4)); LILI_CUDA(c, c->rot_label.ensure(N * 4));
    LILI_CUDA(c, c->rot_lessflat.ensure((N + 2) * 4)); LILI_CUDA(c, c->rot_sort.ensure((N + 2) * 4));
    LILI_CUDA(c, c->rot_picked.ensure((N + 2) * 4));         // lf_src
    LILI_CUDA(c, c->rot_meta.ensure((M_SIZE + ROT_MAX_RINGS * 8) * 4 + ROT_MAX_RINGS * sizeof(VgParams) + ROT_MAX_RINGS * 8 * sizeof(long long) + 16));
    LILI_CUDA(c, c->rot_seg_edge.ensure((size_t)ROT_MAX_RINGS * 6 * 11 * 4));
    LILI_CUDA(c, c->surf.ensure(N * sizeof(Pt32)));
    LILI_CUDA(c, c->edge.ensure((size_t)ROT_MAX_RINGS * 6 * 10 * sizeof(Pt32)));
    LILI_CUDA(c, c->vg_flags.ensure((N + 2) * 4)); LILI_CUDA(c, c->vg_rank.ensure((N + 2) * 4));
    LILI_CUDA(c, c->vg_count.ensure(16));

    Q4 qI{q_imu[0], q_imu[1], q_imu[2], q_imu[3]};
    if (std::isnan(qI.w) || std::isnan(qI.x) || std::isnan(qI.y) || std::isnan(qI.z)) qI = Q4{1, 0, 0, 0};   // :299-301
    Q4 qL{q_lb[0], q_lb[1], q_lb[2], q_lb[3]};
    const Pt32* raw = c->raw_src ? reinterpret_cast<const Pt32*>(c->raw_src) : c->raw.as<Pt32>();   // read-only input
    int* meta = c->rot_meta.as<int>();
    int* ringmm = meta + M_SIZE;
    VgParams* rprm = reinterpret_cast<VgParams*>(ringmm + ROT_MAX_RINGS * 8);
    uint32_t* keys = c->rot_keys.as<uint32_t>(); uint32_t* keys2 = c->rot_keys2.as<uint32_t>();
    int* vals = c->rot_vals.as<int>(); int* vals2 = c->rot_vals2.as<int>();
    float* ori = c->rot_ring.as<float>();
    Pt32* cloud = c->rot_cloud.as<Pt32>();
    int* seg_edge = c->rot_seg_edge.as<int>();
    int* seg_cnt = seg_edge + ROT_MAX_RINGS * 6 * 10;

    k_rot_meta_init<<<1, 256, 0, c->stream>>>(meta);
    LILI_TRY(launch_check(c, "k_rot_meta_init"));
    if (times) {
        k_rot_pre<true><<<cdiv(n, ROT_PRE_THREADS), ROT_PRE_THREADS, 0, c->stream>>>(raw, rings, times, n, n_scans, keys, vals, ori, meta);
        LILI_TRY(launch_check(c, "k_rot_pre"));
    } else {
        k_rot_pre<false><<<cdiv(n, ROT_PRE_THREADS), ROT_PRE_THREADS, 0, c->stream>>>(raw, rings, nullptr, n, n_scans, keys, vals, ori, meta);
        LILI_TRY(launch_check(c, "k_rot_pre"));
        k_rot_hp<<<cdiv(n, 256), 256, 0, c->stream>>>(raw, n, keys, ori, meta);     // the halfPassed latch: azimuth rule only
        LILI_TRY(launch_check(c, "k_rot_hp"));
    }
    LILI_TRY(sort_pairs_u32(c, keys, keys2, vals, vals2, n, 8));
    if (times) k_rot_build<true><<<cdiv(n, 128), 128, 0, c->stream>>>(raw, n, keys2, vals2, ori, times, qI, qL, cloud, meta);
    else k_rot_build<false><<<cdiv(n, 128), 128, 0, c->stream>>>(raw, n, keys2, vals2, ori, nullptr, qI, qL, cloud, meta);
    LILI_TRY(launch_check(c, "k_rot_build"));
    k_rot_curv<<<cdiv(n + 1, 256), 256, 0, c->stream>>>(cloud, meta, c->rot_curv.as<float>(), c->rot_label.as<int>(),
                                                        c->rot_lessflat.as<int>(), n);
    LILI_TRY(launch_check(c, "k_rot_curv"));
    // per-device function attribute (cheap; a process may hold contexts on several GPUs)
    LILI_CUDA(c, cudaFuncSetAttribute(k_rot_ring, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(RingSmem)));
    long long* ring_dbg = c->dbg_timing ? reinterpret_cast<long long*>(reinterpret_cast<unsigned char*>(rprm + ROT_MAX_RINGS) + 8) : nullptr;
    if (ring_dbg) ring_dbg = reinterpret_cast<long long*>((reinterpret_cast<uintptr_t>(ring_dbg) + 7) & ~(uintptr_t)7);
    k_rot_ring<<<n_scans, 512, sizeof(RingSmem), c->stream>>>(cloud, c->rot_curv.as<float>(), meta, c->prm.ds_rate, c->rot_label.as<int>(),
                                                              c->rot_lessflat.as<int>(), seg_edge, seg_cnt, ring_dbg, c->rot_slow_walk ? 0 : ROT_FAST_CAP);
    LILI_TRY(launch_check(c, "k_rot_ring"));
    if (ring_dbg) {       // LILIOM_DEBUG_TIMING: per-ring stage cycles of this launch
        long long h[ROT_MAX_RINGS * 8];
        if (cudaMemcpyAsync(h, ring_dbg, sizeof(h), cudaMemcpyDeviceToHost, c->stream) == cudaSuccess && cudaStreamSynchronize(c->stream) == cudaSuccess) {
            long long mx = 0, sum = 0, t_first = LLONG_MAX, t_last = 0; int arg = -1, cnt = 0;
            for (int r = 0; r < n_scans; ++r) {
                const long long* d = h + r * 8;
                if (d[0] <= 0) continue;
                ++cnt; sum += d[0];
                if (d[0] > mx) { mx = d[0]; arg = r; }
                t_first = std::min(t_first, d[7]); t_last = std::max(t_last, d[6]);
            }
            if (arg >= 0) {
                const long long* d = h + arg * 8;
                fprintf(stderr, "[k_rot_ring, cycles] %d rings, mean %lld, slowest ring %d: %lld (loads %lld, sort %lld, walk %lld, flags %lld, longest segment %lld points); "
                                "first block start -> last block end %lld ns\n", cnt, sum / cnt, arg, d[0], d[1], d[2], d[3], d[4], d[5], t_last - t_first);
                long long late = 0; for (int r = 0; r < n_scans; ++r) if (h[r * 8] > 0) late = std::max(late, h[r * 8 + 7] - t_first);
                fprintf(stderr, "[k_rot_ring] latest block start after the first: %lld ns\n", late);
            }
        }
    }
    k_rot_edge_emit<<<1, ROT_EMIT_THREADS, 0, c->stream>>>(cloud, seg_edge, seg_cnt, n_scans * 6, c->edge.as<Pt32>(), meta);
    LILI_TRY(launch_check(c, "k_rot_edge_emit"));
    // less-flat -> per-ring VoxelGrid
    int* lfpos = c->rot_sort.as<int>();
    int* lf_src = c->rot_picked.as<int>();
    LILI_TRY(exclusive_scan_i32(c, c->rot_lessflat.as<int>(), lfpos, n));
    k_rot_lf_init<<<cdiv(ROT_MAX_RINGS * 8, 256), 256, 0, c->stream>>>(ringmm);
    LILI_TRY(launch_check(c, "k_rot_lf_init"));
    k_rot_lf_gather<<<cdiv(n, 256), 256, 0, c->stream>>>(cloud, keys2, c->rot_lessflat.as<int>(), lfpos, n, n_scans, lf_src, ringmm, meta);
    LILI_TRY(launch_check(c, "k_rot_lf_gather"));
    k_rot_lf_params<<<1, ROT_MAX_RINGS, 0, c->stream>>>(ringmm, c->prm.rot_ds_leaf, rprm);
    LILI_TRY(launch_check(c, "k_rot_lf_params"));
    unsigned long long* k64 = c->rot_keys.as<unsigned long long>();
    unsigned long long* k64b = c->rot_keys2.as<unsigned long long>();
    // keys2 (ring ids, sorted) is still needed by k_rot_lf_keys: stash it before reusing the buffers
    LILI_CUDA(c, c->idx_b.ensure(N * 4));
    LILI_CUDA(c, cudaMemcpyAsync(c->idx_b.p, keys2, N * 4, cudaMemcpyDeviceToDevice, c->stream));
    const uint32_t* ring_of = c->idx_b.as<uint32_t>();
    k_rot_lf_keys<<<cdiv(n, 256), 256, 0, c->stream>>>(cloud, ring_of, lf_src, meta, rprm, k64, vals, n);
    LILI_TRY(launch_check(c, "k_rot_lf_keys"));
    LILI_TRY(sort_pairs_u64(c, k64, k64b, vals, vals2, n, 40));
    k_vg_heads<<<cdiv(n + 1, 256), 256, 0, c->stream>>>(k64b, n, meta + M_NLF, c->vg_flags.as<int>());
    LILI_TRY(launch_check(c, "k_vg_heads"));
    LILI_TRY(exclusive_scan_i32(c, c->vg_flags.as<int>(), c->vg_rank.as<int>(), n));
    k_rot_lf_centroid<<<cdiv(n, 128), 128, 0, c->stream>>>(cloud, lf_src, k64b, vals2, c->vg_flags.as<int>(), c->vg_rank.as<int>(), meta, n,
                                                           c->surf.as<Pt32>(), c->vg_count.as<int>());
    LILI_TRY(launch_check(c, "k_rot_lf_centroid"));
    int hp[9];
    LILI_TRY(read_back(c, {{hp, meta, 8 * sizeof(int)}, {hp + 8, c->vg_count.p, sizeof(int)}}));
    if (hp[M_ERR]) { c->last_error = "ring/segment larger than the shared-memory capacity (16384 / 4096 points)"; return LILIOM_E_CAPACITY; }
    *n_cut = hp[M_NVALID]; *n_edge = hp[M_NEDGE]; *n_surf = hp[8];
    c->n_surf_dev = hp[8];
    c->d_nsurf = c->vg_count.as<int>();
    c->n_surf_max = n;
    c->n_rot_cloud = hp[M_NVALID];
    return LILIOM_OK;
}

}  // namespace lili
