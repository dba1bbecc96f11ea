// Internal context of libliliom_b200.so (not part of the ABI).
#pragma once
#include <climits>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <string>
#include <utility>
#include <vector>
#include "../../include/liliom.h"
#include "batch.h"
#include "vg_box.h"

namespace lili {

// One growable device allocation, owned: freed by the destructor, moved (never copied) between owners.  Buffers only grow;
// 80 GB of HBM3 per GPU (a 10 M-point map needs well under 1 GB) makes reallocation-on-demand a cold path (first scan),
// never a steady-state cost.
struct DevBuf {
    void*  p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
        return *this;
    }
    ~DevBuf() { release(); }
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

// One growable pinned host allocation, owned, growing as DevBuf does: the staging of a batched call's tables and results.
struct PinBuf {
    void*  p = nullptr;
    size_t cap = 0;
    PinBuf() = default;
    PinBuf(const PinBuf&) = delete;
    PinBuf& operator=(const PinBuf&) = delete;
    ~PinBuf() { release(); }
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        release();
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaHostAlloc(&p, want, cudaHostAllocDefault);
        if (e == cudaSuccess) cap = want; else p = nullptr;
        return e;
    }
    void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
    template <class T> T* as(size_t byte_off = 0) const { return reinterpret_cast<T*>(static_cast<unsigned char*>(p) + byte_off); }
};

// Dense cell grid over the down-sampled map (the kd-tree's stand-in).
struct GridDesc {
    float inv_cell;        // 1 / cell size (power of two => exact)
    int   org[3];          // cell coordinate of grid cell (0,0,0)
    int   dim[3];
    int   ncells;
};

// One searchable point set: the float4 points, their cell grid and (optionally) a reflectivity channel.  grid_build writes it.
// The odometry map (liliom_ctx::map) and the two layers of the backend local map (liliom_ctx::bmap) are each one.
struct MapIndex {
    DevBuf xyzw;                         // float4 in download order (w = index)
    DevBuf refl;                         // optional per-point reflectivity channel (liliom_map_set_cloud, backend surf layer)
    DevBuf sorted;                       // float4 sorted by cell, w = original index bits
    DevBuf cell_start;                   // ncells + 1
    GridDesc grid{};
    int  n = 0;                          // points resident on this rank (sorted grid)
    bool ready = false;
};

// Cell edge for a squared-distance gate: the smallest power of two whose square reaches it (1.0 for the reference's gates).
inline float gate_cell(double sqgate) {
    float cell = 1.0f;
    while ((double)cell * (double)cell < sqgate) cell *= 2.0f;
    return cell;
}

// Keyframe store (keyframes.cu): body-frame clouds of every keyframe in one device arena, edge then surf per keyframe; the full
// clouds (liliom_kf_add_full) in an arena of their own.  Offsets in points; n_full < 0: no full cloud attached.
struct KfEntry {
    long long edge_off, surf_off;
    int n_edge, n_surf;
    long long full_off = 0;
    int n_full = -1;
};

// Fused multi-GPU exchange (single node): pointers to every rank's exchange buffer (own entry = own buffer), see
// peer_exchange() in grid_knn.cu.  Passed to the persistent GN kernel by value.
constexpr int kMaxPeers = 16;
struct PeerArgs {
    ulonglong2* buf[kMaxPeers];
    int nranks, rank;
    unsigned int epoch0;       // epoch of iteration 0 of this launch (monotonic across launches, identical on all ranks)
    int enabled;
    double* lsum;              // [2 parities][32] the sums over all ranks, republished by block 0 for the other blocks of this GPU
    unsigned int* lflag;       // [2] epoch of the republished sums
};

constexpr int kStatsDoubles = 40;   // per outer iteration on the device: n_corr, lm_iters, cost, 27, pose7, pad
constexpr int kNormEq = 29;         // 21 + 6 + cost + count

struct PinIcp {                // ICP results (icp.cu), stored by the last block of the ICP kernel
    double T[16];              // row-major 4x4 source -> target
    double fitness;
    int    converged, iters;
};

// The context's small pinned host block (liliom_ctx::h_pin): disjoint members, each read after its user's stream synchronise.
struct PinResult {             // scan-to-map results: stored by the persistent GN kernel through GnIo::host_out, or copied
    double pose[8];            // pose (wxyz, t) + peer-loss flag
    double neq[kNormEq];       // the 29 sums of the last pass
    int    n_feats;            // device-side query count
    VgParams vgp;              // parameters of the scan's VoxelGrid (speculation check)
};
struct PinBlock {
    PinResult s2m;
    double pose_stage[8];      // scan-to-map start pose + cleared peer-loss flag, copied to the device for per-pass launches
    double map_status[4];      // multi-rank map rebuild: {owned voxels, failed} out, their sums over the ranks back
    alignas(16) unsigned char scratch[kNormEq * sizeof(double)];   // read_back(); its largest user: the backend's 29 sums
    PinIcp icp;                // ICP: the results of k_icp_persistent
    double stats[];         // kStatsDoubles per GN iteration, up to the end of the block (h_pin_bytes)
};

// Scan-to-map results written straight into the context's pinned host block by the persistent GN kernel (zero-copy: the
// stream then ends with the kernel and the host reads the block after its stream synchronise), and the start pose as a
// kernel parameter: per scan this removes one host-to-device and three device-to-host copy operations from the stream,
// each of which costs a few microseconds of dependent latency on a ~200 us step.
struct GnIo {
    double pose0[8];           // start pose (wxyz, t) + cleared peer-loss flag
    PinResult* host_out;       // device-visible address of the pinned block's results, nullptr: results stay on the device
    const int* vgp;            // VgParams of the scan's VoxelGrid (speculation check) to forward to host_out->vgp, or nullptr
};

#ifdef __CUDACC__
// Where a block sits in its session: blk.bi() of blk.G() blocks.  A solo launch reads blockIdx.x / gridDim.x at each use
// (the kernels keep the code and registers they had before the batched launch existed); a batched launch (k_gn_batch,
// k_hz_batch, k_icp_batch) passes the block's place inside its session's range.
struct SoloBlock {
    __device__ __forceinline__ int bi() const { return (int)blockIdx.x; }
    __device__ __forceinline__ unsigned int G() const { return gridDim.x; }
};
struct SessionBlock {
    int b; unsigned int g;
    __device__ __forceinline__ int bi() const { return b; }
    __device__ __forceinline__ unsigned int G() const { return g; }
};

// The session of this block in a batched launch (batch.h) and the block's place in that session's range.
struct BatchSlot {
    int s;
    SessionBlock blk;
};
template <class Entry, int N>
__device__ __forceinline__ BatchSlot batch_slot(const BatchTab<Entry, N>& tab) {
    const int s = batch_session_of(tab.n, tab.off, (int)blockIdx.x);
    return BatchSlot{s, SessionBlock{(int)blockIdx.x - tab.off[s], (unsigned int)(tab.off[s + 1] - tab.off[s])}};
}

// One stage of a batched chain (the ROT extraction in extract_rot.cu, the map update in map.cu): its Entry, its block size, its
// blocks for a session (host side: the table's off[] carries them to the device) and its body run(entry, bx) for block bx of the
// session, each as the solo launch has them.  The macro's run copies the entry by value, as the solo kernels' parameters are, and
// gives CALL `e`, `bx` and the thread's place `i` in its session's launch.
#define LILI_STAGE(NAME, ENTRY, THREADS, BLOCKS, CALL)                                                \
    struct NAME {                                                                                     \
        typedef ENTRY Entry;                                                                          \
        static constexpr int kThreads = THREADS;                                                      \
        static int blocks(const Entry& e) { return BLOCKS; }                                          \
        __device__ static void run(const Entry& te, int bx) {                                         \
            const Entry e = te;                                                                       \
            const int i = bx * THREADS + (int)threadIdx.x;                                            \
            (void)i;                                                                                  \
            CALL;                                                                                     \
        }                                                                                             \
    };
template <class St, int N>
__global__ void __launch_bounds__(St::kThreads) k_stage_batch(const __grid_constant__ BatchTab<typename St::Entry, N> tab) {
    const BatchSlot at = batch_slot(tab);
    St::run(tab.s[at.s], at.blk.bi());
}

// Bodies of the box and cell-grid kernels (voxelgrid.cu, grid_knn.cu), `i` = the thread's place in its session's launch: the solo
// kernels pass blockIdx.x * blockDim.x + threadIdx.x, the batched map update (k_stage_batch, map.cu) the same place counted
// from its session's first block.
__device__ __forceinline__ void vg_box_init(int* __restrict__ mm) {
    if (threadIdx.x < kBoxInts) mm[threadIdx.x] = vg_box_empty(threadIdx.x);
}
template <class Blk>
__device__ __forceinline__ void vg_minmax_body(const unsigned char* __restrict__ pts, int n_max, const int* __restrict__ d_n, int stride,
                                               int* __restrict__ mm, const Blk blk) {
    const int n = d_n ? min(*d_n, n_max) : n_max;
    int box[kBoxInts];
#pragma unroll
    for (int k = 0; k < kBoxInts; ++k) box[k] = vg_box_empty(k);
    for (int i = blk.bi() * blockDim.x + threadIdx.x; i < n; i += blk.G() * blockDim.x) {
        float4 v = *reinterpret_cast<const float4*>(pts + (size_t)i * stride);
        if (!(isfinite(v.x) && isfinite(v.y) && isfinite(v.z))) continue;
        vg_box_add(box, v.x, v.y, v.z);
    }
    vg_box_commit(box, mm);
}

// Bodies of the VoxelGrid chain's parameter, key and centroid kernels (voxelgrid.cu), `i` as above; the batched loop closure
// (keyframes.cu) runs them too.
__device__ __forceinline__ void vg_params_at(const int* __restrict__ mm, float leaf, VgParams* __restrict__ out) {
    if (threadIdx.x == 0) *out = vg_params(mm, leaf);
}

// K = uint32_t: non-finite points take the all-ones key; K = unsigned long long (wide keys, vg_wide_keys): the flag at bit 32
template <typename K>
__device__ __forceinline__ void vg_keys_at(const unsigned char* __restrict__ pts, int n_max, const int* __restrict__ d_n, int stride,
                                           const VgParams* __restrict__ pp, K* __restrict__ keys, int* __restrict__ vals, const int i) {
    if (i >= n_max) return;
    const int n = d_n ? min(*d_n, n_max) : n_max;
    const VgParams p = *pp;
    float4 v = make_float4(NAN, 0.f, 0.f, 0.f);
    if (i < n) v = *reinterpret_cast<const float4*>(pts + (size_t)i * stride);
    K key = sizeof(K) == 4 ? (K)0xffffffffu : (K)(1ull << 32);
    if (isfinite(v.x) && isfinite(v.y) && isfinite(v.z)) key = vg_rel_index(p, v.x, v.y, v.z);
    keys[i] = key;
    vals[i] = i;
}

template <int STRIDE, typename K>
__device__ __forceinline__ void vg_centroid_at(const unsigned char* __restrict__ pts, const K* __restrict__ keys, const int* __restrict__ vals,
                                               const int* __restrict__ flags, const int* __restrict__ rank, int n_max, const int* __restrict__ d_n,
                                               const VgParams* __restrict__ pp, unsigned char* __restrict__ out, int* __restrict__ count_out,
                                               float4* __restrict__ feats_out, const int i) {
    const VgParams p = *pp;
    const int n = d_n ? min(*d_n, n_max) : n_max;
    if (i == 0) *count_out = p.overflow ? n : rank[n_max];
    if (p.overflow) {   // PCL: output = *input_ (not the centroids of one-point voxels: the normal and the padding would differ)
        if (i < n) {
            const float4* src = reinterpret_cast<const float4*>(pts + (size_t)i * STRIDE);
            float4* dst = reinterpret_cast<float4*>(out + (size_t)i * STRIDE);
#pragma unroll
            for (int k = 0; k < STRIDE / 16; ++k) dst[k] = src[k];
            if (feats_out) feats_out[i] = make_float4(src[0].x, src[0].y, src[0].z, __int_as_float(i));
        }
        return;
    }
    if (i >= n || !flags[i]) return;
    const int o = rank[i];
    const VgAcc<STRIDE> a = vg_walk<STRIDE>(keys, i, p.n_finite, [&](int j) { return vals[j]; },
                                            [&](int m) { return pts + (size_t)m * STRIDE; });
    const VgXyz c = vg_write<STRIDE>(a.s, a.n, out + (size_t)o * STRIDE);
    if (feats_out) feats_out[o] = make_float4(c.x, c.y, c.z, __int_as_float(o));
}

__device__ __forceinline__ void repack_f4_at(const unsigned char* __restrict__ in, int n_max, const int* __restrict__ d_n, int stride,
                                             float4* __restrict__ out, const int i) {
    const int n = d_n ? min(*d_n, n_max) : n_max;
    if (i >= n) return;
    float4 v = *reinterpret_cast<const float4*>(in + (size_t)i * stride);
    v.w = __int_as_float(i);
    out[i] = v;
}

__device__ __forceinline__ int cell_coord(float v, float inv_cell) { return (int)floorf(v * inv_cell); }

// `escaped` (optional): set when a point lies outside the grid's box — only possible when the box was handed in by the caller
// (grid_build's host_box); the key is then clamped into range for memory safety and the caller rebuilds with the exact box.
__device__ __forceinline__ void cell_keys_at(const float4* __restrict__ p, int n, const GridDesc& g, uint32_t* __restrict__ keys,
                                             int* __restrict__ vals, int* __restrict__ escaped, const int i) {
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

__device__ __forceinline__ void gather_sorted_at(const float4* __restrict__ p, const int* __restrict__ vals, int n, float4* __restrict__ out,
                                                 const int i) {
    if (i >= n) return;
    int src = vals[i];
    float4 v = p[src];
    out[i] = make_float4(v.x, v.y, v.z, __int_as_float(src));   // w = index into the un-sorted map array
}

// cell_start[c] = first sorted position whose key >= c = number of points with key < c = upper bound of cell c-1.
// Run ENDS are scattered (cell_start[key+1] = position after the run) into a zeroed table and a running maximum fills the
// empty cells: two streaming passes over the table.  (Filling every gap with one warp per sorted position is an order of
// magnitude slower on a 10 M-point map.)
__device__ __forceinline__ void cell_run_ends_at(const uint32_t* __restrict__ keys, int n, int* __restrict__ cell_start, const int w) {
    if (w >= n) return;
    const uint32_t k = keys[w];
    if (w == n - 1 || keys[w + 1] != k) cell_start[(size_t)k + 1] = w + 1;
}

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// The grid barrier of every cooperative kernel.  grid_barrier is called by all threads of a block: the block's writes are
// ordered before one arrival of thread 0 on `bar`, thread 0 polls until the arrivals reach `target`, and the block meets again.
// grid_arrive is thread 0's part, for a caller that places the block barriers itself: the GN step, whose multi-GPU followers
// arrive without waiting (wait = false), and the ICP pass.  The flavour is fixed per kernel:
//   kReleaseOnly (GN, ICP): one release by thread 0 after the block barrier (cumulative over bar.sync, as in cooperative
//     groups' grid.sync; SASS: MEMBAR.ALL.GPU + RED, no L1 invalidate) and NO acquire fence after the relaxed poll.  An acquire
//     would only add an L1 invalidation: everything these kernels read through L1 (map, cell table, features, source points) is
//     immutable for the launch, and the partials are read with L2-scope loads (__ldcg) issued after the poll's control
//     dependency and a bar.sync.  (The PTX model formally asks for the acquire; an acquire poll and the fenced flavour give the
//     same bits and are slower per pass: 12.70 us fenced against 11.99 us release-only for the headline GN pass.)
//   kFenced (Horizon extractor, cooperative VoxelGrid): __threadfence on both sides of an atomicAdd arrival and a volatile poll.
//     The release-only flavour is legal there too (every cross-block read is an L2-scope load) and was measured to change
//     nothing: 4586/4629 vs 4653/4563 scans/s.  Those kernels spend their time in the stages, not in the three fences.
enum GridBarrierFlavour { kReleaseOnly, kFenced };
template <GridBarrierFlavour F>
__device__ __forceinline__ void grid_arrive(unsigned int* bar, unsigned int target, bool wait) {
    if constexpr (F == kFenced) {
        atomicAdd(bar, 1u);
        if (wait) { while ((int)(*reinterpret_cast<volatile unsigned int*>(bar) - target) < 0) { } __threadfence(); }
    } else {
        asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(bar), "r"(1u) : "memory");
        unsigned int v;
        if (wait) { do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory"); } while ((int)(v - target) < 0); }
    }
}
template <GridBarrierFlavour F>
__device__ __forceinline__ void grid_barrier(unsigned int* bar, unsigned int target) {
    if constexpr (F == kFenced) __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) grid_arrive<F>(bar, target, true);
    __syncthreads();
}
#endif

struct Frame {        // one entry of recent_surf_frames (world frame, point_stride bytes per point)
    DevBuf buf;
    int n = 0;
    // incremental map (map.cu): slot id carried by the frame's entries, unrepresentable key seen
    int slot = 0;
    bool bad = false;
    // box of the stored points (vg_box.h; mm[6] = finite points), taken when the frame was pushed: the rebuild's VoxelGrid, the
    // cell grid and the incremental map get their bounding boxes from the union over the frames instead of passes over the map
    int mm[kBoxInts] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN, 0};
};

// The per-point side channels decoded with one PointCloud2 sweep: the `ring` field (LILIOM_RING_FIELD) and the time field
// (LILIOM_TIME_FIELD), and whether each buffer holds them for that sweep.
struct Pc2Side {
    DevBuf ring;               // u16 ring id per point
    DevBuf time;               // double time per point
    bool has_ring = false;
    bool has_time = false;
    void clear() { has_ring = has_time = false; }
    const uint16_t* rings() const { return has_ring ? ring.as<uint16_t>() : nullptr; }
    const double* times() const { return has_time ? time.as<double>() : nullptr; }
};

}  // namespace lili

struct liliom_ctx {
    liliom_params prm;
    int device = 0;
    cudaStream_t stream = nullptr;       // stream all work is issued on (own_stream unless liliom_set_stream)
    cudaStream_t own_stream = nullptr;
    cudaStream_t copy_stream = nullptr;  // D2H of a finished output while later kernels of the same call still run
    cudaEvent_t  ev_ready = nullptr, ev_copied = nullptr;
    cudaEvent_t  ev_batch = nullptr;     // orders this context's stream around a batched step (liliom_scan_to_map_resident_batch)
    void*  early_cut_dst = nullptr;      // host destination for the cutted cloud (set per call by the API layer)
    int    early_cut_cap = 0;
    bool   early_cut_issued = false;
    std::string last_error;
    int sm_count = 132;                  // H100 SXM; replaced by the device's multiProcessorCount at create

    // ---- staging (pinned host) ----
    lili::PinBlock* h_pin = nullptr;      // small pinned block: counts, pose, stats
    lili::PinBlock* h_pin_dev = nullptr;  // the same block as the device sees it (mapped); nullptr: not mappable, results are copied
    size_t h_pin_bytes = 0;

    // ---- extraction ----
    lili::DevBuf raw, cut, surf, edge, flags, scan_tmp, idx_a, idx_b;
    lili::DevBuf hz_mat, hz_stage_surf, hz_stage_edge, hz_counts;
    lili::DevBuf rot_keys, rot_keys2, rot_vals, rot_vals2, rot_cloud, rot_curv, rot_label, rot_picked, rot_sort, rot_ring, rot_meta, rot_lessflat, rot_seg_edge;
    int n_surf_dev = 0;          // surf features resident after the last extract call (-1: only known on the device)
    const int* d_nsurf = nullptr; // device-side count of the resident surf features
    int n_surf_max = 0;          // host upper bound for it
    const int* d_nfeats = nullptr; // device-side query count for scan-to-map (nullptr: n_feats is exact)
    int last_n_feats = 0;        // query count of the previous scan (kernel-shape predictor)
    int n_feats_actual = 0;      // query count read back with the pose
    int n_ds_resident = -1;      // >= 0: vg_out holds surf_last_ds of the last odometry call, that many points
                                 // (liliom_map_update_resident): set by odo_finish, -1 from every other writer of vg_out.  A count
                                 // of its own: n_feats_actual moves with every scan-to-map call, which leaves vg_out alone
    bool vg_check = false;       // s2m_run also reads vg_params back (speculative key width of the scan VoxelGrid)
    bool vg_used24 = false;      // ... the sort chain ran with 24-bit keys
    bool vg_bail = false;        // ... the cooperative filter declined (valid after the sync)
    bool vg_wide = false;        // ... ran on keys of <= 32 bits where the index wraps: redo with wide keys (valid after the sync)
    unsigned int vg_coop_calls = 0;   // launches of k_vg_coop so far (selects the rotating control slot)
    lili::DevBuf vg_coop;        // hash table + scratch of the cooperative filter
    lili::DevBuf hz_ctl;         // barrier words + per-block counts of the cooperative Horizon extractor
    unsigned int hz_coop_calls = 0;
    long long vg_ncells = 0;     // voxel-box cell count of that VoxelGrid, valid after the sync
    lili::DevBuf raw_scan;       // resident raw sweep (liliom_upload_scan / liliom_convert_livox / liliom_convert_pc2)
    lili::DevBuf wire_in;        // staged sensor payload: livox CustomPoint records (19/20 bytes each) or PointCloud2 data
    int n_raw_scan = 0;
    const void* raw_src = nullptr; // when set, the extractors read the sweep from here instead of c->raw (resident pipeline: no copy)
    int ring_source = LILIOM_RING_ELEVATION;   // liliom_set_ring_source
    int time_source = LILIOM_TIME_AZIMUTH;     // liliom_set_time_source
    char time_name[16] = {};     // LILIOM_TIME_FIELD: the name of the per-point time field
    lili::Pc2Side raw_side;      // side channels of c->raw (liliom_extract_rot_pc2)
    lili::Pc2Side raw_scan_side; // ... of the resident sweep (liliom_convert_pc2)
    int n_rot_cloud = 0;
    // the clouds the last extraction left resident (surf, edge and cut / laserCloud; liliom_features_download)
    bool feat_ready = false;
    int feat_counts[3] = {0, 0, 0};      // their sizes; -1: only on the device (resident Horizon extraction)
    int feat_max[3] = {0, 0, 0};         // Horizon: host upper bounds of those sizes (the extractor sizes the buffers from them)
    int* feat_dcounts = nullptr;         // Horizon: the surf and edge counts on the device, a spare word behind them
    const int* feat_dcut = nullptr;      // Horizon: the cut count on the device (idx_a[n], or feat_dcounts[2] once idx_a is reused)

    // ---- voxel grid scratch ----
    lili::DevBuf vg_keys, vg_keys2, vg_vals, vg_vals2, vg_flags, vg_rank, vg_params, vg_out, vg_minmax, vg_count;
    lili::DevBuf cub_tmp;

    // ---- map (map.cu) ----
    std::vector<lili::Frame> frames;     // FIFO, oldest first
    // incremental map (liliom_map_update): entries {voxel key, slot<<24|index} sorted by (key, frame age, index), double-buffered
    lili::DevBuf inc_key[2], inc_ref[2], inc_newkey[2], inc_newref[2], inc_removed, inc_rpos, inc_flags, inc_rank, inc_bad;
    int inc_cur = 0, inc_E = 0;
    bool inc_valid = false;
    lili::DevBuf map_raw;                // concatenated frames (stride bytes)
    lili::DevBuf map_ds;                 // VoxelGrid output (stride bytes); scratch of the sharded install
    int map_ds_n = 0;                    // records of the filtered cloud in map_ds; -1: an installed map has none behind it
    lili::MapIndex map;                  // the odometry map's search index (scan-to-map, backend single-keyframe calls, ICP target)
    lili::DevBuf grid_keys, grid_keys2, grid_vals, grid_vals2;   // grid_build scratch, shared by every index
    int map_n_global = 0;                // map size over all ranks: the "< 10 map points" guard

    // ---- backend (keyframes.cu, backend_corr.cu): keyframe store, local map layers, window correspondences ----
    lili::DevBuf kf_arena;               // body-frame clouds of every keyframe (point_stride bytes per point)
    long long kf_used = 0;               // points in use
    lili::DevBuf kf_full;                // full clouds of the keyframes (liliom_kf_add_full), point_stride bytes per point
    long long kf_full_used = 0;          // points in use
    std::vector<lili::KfEntry> kfs;      // per keyframe: offsets and counts (host)
    lili::DevBuf kf_tab;                 // per-call keyframe table (kf_table.h: k_kf_gather, the global map's kernels)
    lili::DevBuf kf_img, kf_img_seg, kf_img_sum;   // liliom_kf_export's staged points, the image calls' segments and checksum word
    lili::MapIndex bmap[2];              // backend local map: [0] edge layer, [1] surf layer
    lili::DevBuf bmap_raw, bmap_ds[2];   // concatenation of the transformed keyframes; the filtered layers (all fields)
    int bmap_n[2] = {0, 0};
    bool bmap_built = false;
    int win_k = 0;                       // window correspondences resident (liliom_backend_window_correspond)
    liliom_backend_params win_bp{};      // ... and the parameters they were found with (weights, extrinsics, loss of the blocks)
    std::vector<int> win_ids;
    std::vector<long long> win_qoff[2];  // per kind: query prefix offsets (k + 1)
    lili::DevBuf win_valid[2], win_line, win_plane, win_score, win_cnt, win_tab;
    // a batched backend window call whose shared launches run on this context (ctxs[0]): every session's keyframe tables or
    // block segments, the block partials and the results on the device, and the pinned staging of the one upload and the one
    // read-back (backend_corr.cu)
    lili::DevBuf bk_batch_dev;
    lili::PinBuf bk_batch_pin;
    lili::MapIndex loop;                 // loop-closure target (liliom_loop_align): its own index, so the odometry map stays
    lili::DevBuf loop_src;               // ... and its float4 source

    // ---- scan-to-map ----
    lili::DevBuf feats;                  // float4 body-frame queries
    int n_feats = 0;
    lili::DevBuf corr_valid, corr_plane, nn_idx, nn_sqd;
    lili::DevBuf qstate;                 // float4 per query: transformed position + fifth distance of the previous GN pass
    lili::DevBuf pose_dev;               // 7 doubles (current) + 7 (candidate)
    lili::DevBuf partials;               // grid x 29 doubles
    lili::DevBuf neq;                    // 29 doubles (reduced)
    lili::DevBuf stats_dev;              // iterations x kStatsDoubles
    lili::DevBuf counter;                // last-block ticket + scratch ints
    lili::DevBuf lm_state;
    lili::DevBuf lm_coll;                // the collective LM's state and round sums (grid_knn.cu: LmColl)
    lili::DevBuf icp_ctl;                // ICP kernel: barrier word, and its results when the pinned block is not mappable
    int bk_kind = 0, bk_n = 0;           // backend correspondences resident from the last liliom_correspond_* call (1 edge, 2 surf)
    unsigned int bar_arrivals = 0;       // total grid-barrier arrivals issued so far (persistent GN kernel)

    // ---- multi-GPU ----
    void* nccl_comm = nullptr;
    int nranks = 1, rank = 0;
    float shard_inv_block = 0.0625f;     // 1 / shard block edge (LILIOM_SHARD_BLOCK, metres, power of two; must agree on all ranks)
    bool comm_ceres = false;             // liliom_comm_set_ceres: Ceres mode with a communicator runs the collective LM
    lili::DevBuf peer_local;             // block 0 -> other blocks of this GPU: [2][32] doubles + 2 epoch words (fused exchange)
    lili::DevBuf peer_buf;               // this rank's exchange buffer: [2 parities][kMaxPeers][32] {epoch|lo32, epoch|hi32}
    void* peer_ptrs[lili::kMaxPeers] = {};   // every rank's buffer as mapped into this process (cudaIpcOpenMemHandle)
    bool peer_ready = false;
    unsigned int peer_epoch = 0;         // last epoch issued
    // LILIOM_TEST_LOOPBACK=<group>:<rank>/<nranks> (test hook): this context is rank `rank` of `nranks` contexts in one process,
    // and its all-reduce meets the group's other ranks on the host (comm.cu) instead of in NCCL.  LILIOM_TEST_LOOPBACK_MS bounds
    // the wait.  Empty group: not a loopback member.
    std::string loopback_group;
    int loopback_ms = 30000;

    // ---- instrumentation ----
    liliom_counters cnt{};
    bool time_kernels = false;
    int  time_every = 1;          // liliom_set_kernel_timing(c, N): time every N-th scan-to-map call
    unsigned time_calls = 0;
    // run-time switches: read by liliom_create and nowhere else (DESIGN.md §6)
    int force_lanes = 0, force_rounds = 0;   // tuning override (LILIOM_KNN_LANES / LILIOM_KNN_ROUNDS)
    bool dbg_timing = false;             // LILIOM_DEBUG_TIMING: stage clocks of the cooperative kernels, printed by s2m_run
    bool rot_slow_walk = false;          // LILIOM_ROT_SLOW_WALK (test hook): the general walk of k_rot_ring for every segment
    bool hz_chain = false;               // LILIOM_HZ_CHAIN=1 (test hook): the Horizon extractor's multi-launch chain, not k_hz_coop
    bool test_shrink_box = false;        // LILIOM_TEST_SHRINK_BOX (test hook): grid_build takes a box too small in x
    int test_icp_blocks = 0;             // LILIOM_TEST_ICP_BLOCKS=N (test hook): the batched ICP gives this context's session at most
                                         // N blocks instead of its solo grid (the bits must not move)
    bool knn_tma = false, knn_tma_smem_set = false;   // LILIOM_KNN_TMA=1: bulk-copy (cp.async.bulk + mbarrier) staging of the runs in the 16-lane search
    bool knn1_smem_set = false;          // dynamic shared memory limit raised for the one-thread-per-query kernels on this device
    std::vector<cudaEvent_t> ev_pool;
    std::vector<int> ev_passes;          // kernel-body passes covered by each pending event pair k (ev_pool[2k], ev_pool[2k + 1])
};

namespace lili {

inline int fail_cuda(liliom_ctx* c, cudaError_t e, const char* where) {
    char buf[256];
    snprintf(buf, sizeof(buf), "%s: %s", where, cudaGetErrorString(e));
    if (c) c->last_error = buf;
    return LILIOM_E_CUDA;
}

#define LILI_CUDA(c, expr)                                                      \
    do {                                                                        \
        cudaError_t _e = (expr);                                                \
        if (_e != cudaSuccess) return lili::fail_cuda((c), _e, #expr);          \
    } while (0)

#define LILI_TRY(expr)                    \
    do {                                  \
        int _r = (expr);                  \
        if (_r != LILIOM_OK) return _r;   \
    } while (0)

inline int launch_check(liliom_ctx* c, const char* name) {
    cudaError_t e = cudaGetLastError();
    c->cnt.launches++;
    if (e != cudaSuccess) return fail_cuda(c, e, name);
    return LILIOM_OK;
}

inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// One read-back of a few device words: every range is copied into the pinned block's scratch region, the stream is synchronised
// once, and the bytes land in the range's host destination.  The scratch region is never read after the call returns.
struct ReadBack { void* dst; const void* src; size_t bytes; };
inline int read_back(liliom_ctx* c, std::initializer_list<ReadBack> parts) {
    unsigned char* s = c->h_pin->scratch;
    size_t off = 0;
    for (const ReadBack& r : parts) {
        if (off + r.bytes > sizeof(PinBlock::scratch)) { c->last_error = "read_back: larger than the pinned scratch region"; return LILIOM_E_ARG; }
        LILI_CUDA(c, cudaMemcpyAsync(s + off, r.src, r.bytes, cudaMemcpyDeviceToHost, c->stream));
        off += r.bytes;
    }
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    off = 0;
    for (const ReadBack& r : parts) { memcpy(r.dst, s + off, r.bytes); off += r.bytes; }
    return LILIOM_OK;
}

// The caller-buffer contract of the download entry points: *n_out = m; out == NULL is a size query; m > cap gives
// LILIOM_E_CAPACITY and leaves out untouched; otherwise fill() runs (the work that produces the m items, if any is left) and
// m * elem bytes of src are copied and the stream synchronised.
struct NoFill { int operator()() const { return LILIOM_OK; } };
template <class Fill = NoFill>
int download_sized(liliom_ctx* c, const DevBuf& src, int m, size_t elem, void* out, int cap, int* n_out, Fill fill = {}) {
    *n_out = m;
    if (!out) return LILIOM_OK;
    if (m > cap) return LILIOM_E_CAPACITY;
    LILI_TRY(fill());
    if (m) LILI_CUDA(c, cudaMemcpyAsync(out, src.p, (size_t)m * elem, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

// Before idx_a is reused as scratch: the cut count of a resident Horizon extraction, which sits in it, moves to the spare word
// behind the surf / edge counts (liliom_features_download reads it there).
inline int feat_keep_cut(liliom_ctx* c) {
    if (!c->feat_ready || c->feat_counts[2] >= 0 || c->feat_dcut == c->feat_dcounts + 2) return LILIOM_OK;
    LILI_CUDA(c, cudaMemcpyAsync(c->feat_dcounts + 2, c->feat_dcut, sizeof(int), cudaMemcpyDeviceToDevice, c->stream));
    c->feat_dcut = c->feat_dcounts + 2;
    return LILIOM_OK;
}

// The clouds the last extraction left resident, in the order surf, edge, cut (ROT: laserCloud): the buffer each lies in and its
// size, known on the host (n >= 0, n_max = n, d_n = nullptr) or only on the device after a resident Horizon extraction (n = -1,
// n_max a host upper bound, d_n the size on the device).  LILIOM_E_ARG when nothing is resident.
struct FeatCloud {
    DevBuf* buf;
    int n, n_max;
    const int* d_n;
};
inline int feat_clouds(liliom_ctx* c, FeatCloud f[3]) {
    if (!c->feat_ready) return LILIOM_E_ARG;
    DevBuf* buf[3] = {&c->surf, &c->edge, c->prm.point_stride == 48 ? &c->cut : &c->rot_cloud};
    const int* d_n[3] = {c->feat_dcounts, c->feat_dcounts + 1, c->feat_dcut};
    for (int k = 0; k < 3; ++k) {
        const int n = c->feat_counts[k];
        f[k] = n >= 0 ? FeatCloud{buf[k], n, n, nullptr} : FeatCloud{buf[k], n, c->feat_max[k], d_n[k]};
    }
    return LILIOM_OK;
}
// Their sizes on the host: one read-back of all three when they are only on the device.
inline int feat_sizes(liliom_ctx* c, const FeatCloud f[3], int m[3]) {
    for (int k = 0; k < 3; ++k) m[k] = f[k].n;
    if (f[0].d_n) LILI_TRY(read_back(c, {{m, f[0].d_n, sizeof(int)}, {m + 1, f[1].d_n, sizeof(int)}, {m + 2, f[2].d_n, sizeof(int)}}));
    return LILIOM_OK;
}

// ---- modules (implemented in the .cu files) ----
int sort_pairs_u32(liliom_ctx* c, const uint32_t* kin, uint32_t* kout, const int* vin, int* vout, int n, int end_bit);
int sort_pairs_u64(liliom_ctx* c, const unsigned long long* kin, unsigned long long* kout, const int* vin, int* vout, int n, int end_bit);
int exclusive_scan_i32(liliom_ctx* c, const int* in, int* out, int n);   // out has n+1 entries (total at out[n])
int inclusive_max_scan_i32(liliom_ctx* c, int* data, int n);            // in-place running maximum

// VoxelGrid on device buffers; d_count receives the output count (int, device).  n_max = host upper bound, d_n = optional
// device-side count (<= n_max); d_feats (optional) also receives float4{x,y,z,index}.  key_bits, host_mm: see voxelgrid.cu.
int voxelgrid_dev(liliom_ctx* c, const void* d_in, int n_max, const int* d_n, int stride, float leaf, void* d_out, int* d_count,
                  float4* d_feats = nullptr, int key_bits = 32, const int* host_mm = nullptr);
int voxelgrid_dev_sync(liliom_ctx* c, const void* d_in, int n, int stride, float leaf, void* d_out, int* d_count, float4* d_feats, int* m,
                       int key_bits = 32);
int vg_minmax_dev(liliom_ctx* c, const void* d_in, int n_max, const int* d_n, int stride);
int vg_chain_ensure(liliom_ctx* c, long long n, size_t kb);     // the buffers of voxelgrid_dev's chain over n points, kb-byte keys
int voxelgrid_coop(liliom_ctx* c, const void* d_in, int n_max, const int* d_n, int stride, float leaf, void* d_out, int* d_count, float4* d_feats,
                   bool* used);
__global__ void k_kf_refl(const unsigned char* __restrict__ pts, int n, float* __restrict__ out);      // keyframes.cu: reflectivity of 48-byte points

// grid build of index `mi` from float4 points already on the device (mi.xyzw[0..m)), cells of `cell` metres (gate_cell).
// host_box (optional): 6 ordered ints, a box known to contain the points up to rounding of a mean (the union of the frames'
// boxes): no min/max pass and no host round trip.
int grid_build(liliom_ctx* c, MapIndex& mi, float cell, int m, const int* host_box = nullptr);
inline int grid_build(liliom_ctx* c, int m, const int* host_box = nullptr) {      // the odometry map
    return grid_build(c, c->map, gate_cell(c->prm.knn_max_sqdist), m, host_box);
}

// grid_build in parts, for callers that share its launches between several indexes (the batched map update, map.cu):
// grid_begin (host: the grid's box and dimensions, the buffers; done = an empty index, already complete), then k_cell_keys,
// grid_sort, k_gather_sorted, grid_clear, k_cell_run_ends, grid_scan, and grid_finish with the escape flag read back from
// `escaped` (0 when escaped is null), which re-builds from the exact box when a point escaped.
struct GridJob {
    liliom_ctx* c = nullptr;
    MapIndex* mi = nullptr;
    float cell = 0.0f;
    int m = 0;
    bool done = false;
    int bits = 0;                        // key width of the cell sort
    int* escaped = nullptr;              // device flag of k_cell_keys (a host_box was given)
};
int grid_begin(liliom_ctx* c, MapIndex& mi, float cell, int m, const int* host_box, GridJob& j);
// grid_begin of m > 0 points without a host_box, its box pass (k_vg_init, k_vg_minmax over mi.xyzw) already run and its box
// (kBoxInts ints) read back by the caller (the batched loop closure reads every session's with one wait)
int grid_begin_exact(liliom_ctx* c, MapIndex& mi, float cell, int m, const int* hb, GridJob& j);
int grid_sort(const GridJob& j);
int grid_clear(const GridJob& j);
int grid_scan(const GridJob& j);
int grid_finish(const GridJob& j, int esc);

const long long* vg_coop_stamps(liliom_ctx* c);   // voxelgrid.cu

int s2m_run(liliom_ctx* c, double pose7[7], int match_cnt, int max_num_iter, int mode, liliom_iter_stats* stats,
            bool want_corr, double out29[29]);
// Scan-to-map step of B distinct single-GPU contexts (grid_knn.cu): sessions with status[i] == LILIOM_OK run, status[i] = their
// result; the others are skipped.  Session i: pose at poses7 + 7 i, match_cnt[i] iterations, max_num_iter[i] (Ceres mode; may be
// null in GN mode), stats (optional) at stats[i].  Returns a whole-call CUDA error.
int s2m_batch(liliom_ctx* const* cs, int B, double* poses7, const int* match_cnt, const int* max_num_iter, int mode,
              liliom_iter_stats* const* stats, int* status);

// A batched call's shared launches run on ctxs[0]'s stream (c0): the stream of every other session in cs (its work so far) is
// ordered before them ...
inline int batch_join_in(liliom_ctx* c0, const std::vector<liliom_ctx*>& cs) {
    for (liliom_ctx* c : cs) {
        if (c->stream == c0->stream) continue;
        LILI_CUDA(c, cudaEventRecord(c->ev_batch, c->stream));
        LILI_CUDA(c0, cudaStreamWaitEvent(c0->stream, c->ev_batch, 0));
    }
    return LILIOM_OK;
}
// ... and after them: c0->ev_batch is recorded behind the last shared launch, and the others' streams wait for it (no event when
// every session is on c0's stream)
inline int batch_join_out(liliom_ctx* c0, const std::vector<liliom_ctx*>& cs) {
    bool recorded = false;
    for (liliom_ctx* c : cs) {
        if (c->stream == c0->stream) continue;
        if (!recorded) LILI_CUDA(c0, cudaEventRecord(c0->ev_batch, c0->stream));
        recorded = true;
        LILI_CUDA(c, cudaStreamWaitEvent(c->stream, c0->ev_batch, 0));
    }
    return LILIOM_OK;
}

// One session's part of a batched launch: the context whose launch count the launch advances, and the session's blocks.
struct BatchPart {
    liliom_ctx* c;
    int blocks;
};
// The launches of type Tab (a BatchTab, batch.h) over the sessions `ids`, in order, at most kBatchMax sessions each (one launch
// for a packer's launch, which holds no more); a launch of one session fills a Tab1 instead (the one-entry table of the stage
// chains).  part = fill(tab.s[m], ids[m]) writes session m's entry and gives its context and blocks, off[] follows the blocks,
// every session's launch count advances by one, then launch(tab, grid) queues the launch.
template <class Tab, class Tab1 = Tab, class Fill, class Launch>
int batch_tables(const std::vector<int>& ids, Fill fill, Launch launch) {
    static_assert(sizeof(Tab) <= 32764 && sizeof(Tab1) <= 32764, "a batched launch's session table must fit in the kernel parameter space");
    auto queue = [&](auto& tab, size_t first, int n) -> int {
        tab.n = n;
        for (int m = 0; m < n; ++m) {
            const BatchPart p = fill(tab.s[m], ids[first + m]);
            tab.off[m + 1] = tab.off[m] + p.blocks;
            p.c->cnt.launches++;
        }
        return launch(tab, tab.off[n]);
    };
    for (size_t first = 0; first < ids.size(); first += kBatchMax) {
        const int n = (int)(ids.size() - first < (size_t)kBatchMax ? ids.size() - first : (size_t)kBatchMax);
        if (n == 1) { Tab1 tab{}; LILI_TRY(queue(tab, first, n)); }
        else { Tab tab{}; LILI_TRY(queue(tab, first, n)); }
    }
    return LILIOM_OK;
}

#ifdef __CUDACC__
// One stage (LILI_STAGE) for the sessions `which` on c0's stream: fill(entry, id) writes session id's entry and returns its context.
template <class St, class Fill>
int stage_batch(liliom_ctx* c0, const std::vector<int>& which, Fill fill) {
    typedef typename St::Entry Entry;
    return batch_tables<BatchTab<Entry>, BatchTab<Entry, 1>>(
        which, [&](Entry& e, int id) { liliom_ctx* c = fill(e, id); return BatchPart{c, St::blocks(e)}; },
        [&](const auto& tab, int grid) -> int {
            k_stage_batch<St><<<grid, St::kThreads, 0, c0->stream>>>(tab);
            LILI_CUDA(c0, cudaGetLastError());
            return LILIOM_OK;
        });
}
#endif

// Points each session's work at one stream while a batch queues it (the library sorts and scans, the clears and the read-backs
// take the context's stream), and gives every session its own stream back when it ends.
struct BatchStreams {
    std::vector<std::pair<liliom_ctx*, cudaStream_t>> saved;
    BatchStreams(const std::vector<liliom_ctx*>& cs, cudaStream_t s) {
        for (liliom_ctx* c : cs) { saved.emplace_back(c, c->stream); c->stream = s; }
    }
    BatchStreams(const BatchStreams&) = delete;
    BatchStreams& operator=(const BatchStreams&) = delete;
    ~BatchStreams() { for (auto& p : saved) p.first->stream = p.second; }
};

int horizon_extract_dev(liliom_ctx* c, int n, const double q_imu[4], int* n_surf, int* n_edge, int* n_cut, bool sync_counts = true);
// One Horizon session of liliom_extract_resident_batch (n points of the resident sweep): horizon_batch_queue queues every session
// (status: its error, or LILIOM_OK; counts -1, as the solo resident call) and returns a whole-call CUDA error.
struct HzBatchSession {
    liliom_ctx* c;
    int n;
    const double* q_imu;
    int* n_surf; int* n_edge; int* n_cut;
    int status;
};
int horizon_batch_queue(liliom_ctx* c0, std::vector<HzBatchSession>& ss);
// rings: nullptr = scanID from the elevation tables (line_num 16/32/64), else the u16 ring id of every input point (line_num 1..128)
// times: nullptr = relTime from the azimuth rule, else the time of every input point (LILIOM_TIME_FIELD)
int rot_extract_dev(liliom_ctx* c, int n, const double q_imu[4], const double q_lb[4], int* n_surf, int* n_edge, int* n_cut,
                    const uint16_t* rings = nullptr, const double* times = nullptr);
bool rot_lines_ok(int line_num, bool field);
// One ROT session of liliom_extract_resident_batch: what its solo rot_extract_dev call takes (n points of the resident sweep).
// rot_batch_queue queues every session (status: its error, or LILIOM_OK; pending: read-back words queued on its stream); after
// one synchronise of every session's stream, rot_batch_finish completes each pending session as its solo call would.
struct RotBatchSession {
    liliom_ctx* c;
    int n;
    const double* q_imu;
    const double* q_lb;
    const uint16_t* rings;
    const double* times;
    int* n_surf; int* n_edge; int* n_cut;
    int status;
    bool pending;
};
int rot_batch_queue(liliom_ctx* c0, std::vector<RotBatchSession>& ss);   // returns a whole-call CUDA error
int rot_batch_finish(RotBatchSession& s);

int icp_align(liliom_ctx* c, const MapIndex& tgt, const float4* d_src, int n, double max_corr_dist, int max_iter, double trans_eps,
              double fit_eps, double T16[16], double* fitness, int* converged, int* iters);     // icp.cu

// icp_align in parts (icp.cu), for the batched loop closure (keyframes.cu), which shares the launches of several sessions:
// icp_begin (host: the launch's arguments and grid, the buffers, the zeroed barrier word; done = an empty source or target,
// nothing to launch), icp_launch (the solo cooperative launch), icp_fetch (the results to the pinned block when it is not
// mapped), and, after a synchronise of the stream, icp_finish (the results out of the pinned block; identity when done).
struct IcpArgs {
    const float4* src; int n, nvb;                   // source points (float4 xyz*), virtual blocks cdiv(n, 256)
    const float4* map; const float4* map_orig; const int* cell_start; GridDesc g;
    float max_d2;                                    // squared correspondence cut-off
    int rmax, rmax_fit;                              // shells to visit at most: correspondence passes, the fitness pass
    int max_iter; double trans_eps, fit_eps;
    double* partials;                                // [2 parities][kIcpSums][nvb]
    unsigned int* bar;                               // grid barrier word (zeroed before the launch)
    PinIcp* out;                                     // results (the pinned block, or device memory)
};
struct IcpJob {
    liliom_ctx* c = nullptr;
    IcpArgs a{};
    int grid = 0;                        // the solo launch's blocks: min(nvb, co-resident k_icp_persistent blocks)
    bool done = false;
    PinIcp* dev_out = nullptr;           // the results in device memory when the pinned block is not mapped
};
int icp_begin(liliom_ctx* c, const MapIndex& tgt, const float4* d_src, int n, double max_corr_dist, int max_iter, double trans_eps,
              double fit_eps, IcpJob& j);
int icp_launch(const IcpJob& j);
int icp_fetch(const IcpJob& j);
void icp_finish(const IcpJob& j, double T16[16], double* fitness, int* converged, int* iters);
// The ICP launches of the jobs `jobs` (none done) on c0's stream, every session's stream pointing at it (BatchStreams): sessions
// share cooperative k_icp_batch launches, each with its solo grid; a session whose grid is not co-resident in k_icp_batch takes
// icp_launch.  Then icp_fetch of every job.  Returns a whole-call CUDA error.
int icp_batch_launch(liliom_ctx* c0, const std::vector<IcpJob*>& jobs);
int map_install_host(liliom_ctx* c, const void* pts, int m, int stride, bool keep_refl);     // map.cu
// liliom_map_update_resident of B distinct single-GPU contexts on one device (map.cu): status[i] = session i's result, n_map
// (optional) its voxel count.  Returns a whole-call CUDA error.
int map_update_batch(liliom_ctx* const* cs, int B, const double* poses7, int* n_map, int* status);
bool batch_ctxs_ok(liliom_ctx* const* ctxs, int B);      // api.cu: the contexts of a batched call are distinct, single-GPU, on one device

int block27_stats(liliom_ctx* c, const double pose7[7], unsigned long long out[2]);   // grid_knn.cu

int repack_to_f4(liliom_ctx* c, const void* d_in, int n, int stride, float4* d_out, const int* d_n = nullptr);

}  // namespace lili
