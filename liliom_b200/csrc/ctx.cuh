// Internal context of libliliom_b200.so (not part of the ABI).
#pragma once
#include <climits>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <string>
#include <vector>
#include "../../include/liliom.h"
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
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Grid barrier of the persistent kernels (k_gn_persistent, k_icp_persistent), run by thread 0 of each block after the block's
// __syncthreads: one arrival on `bar`, then, when `wait`, a poll until the arrivals reach `target`.  sync_mode (LILIOM_GN_SYNC,
// see liliom_ctx::gn_sync): 3 = release-only arrival and a relaxed poll, 1 = acquire poll, 0 = full fences on both sides.
__device__ __forceinline__ void grid_barrier(unsigned int* bar, unsigned int target, int sync_mode, bool wait) {
    unsigned int v;
    if (sync_mode == 0) {
        atomicAdd(bar, 1u);
        if (wait) { while ((int)(*reinterpret_cast<volatile unsigned int*>(bar) - target) < 0) { } __threadfence(); }
    } else {
        asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(bar), "r"(1u) : "memory");
        if (wait) {
            if (sync_mode == 1) { do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory"); } while ((int)(v - target) < 0); }
            else { do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory"); } while ((int)(v - target) < 0); }
        }
    }
}
#endif

struct Frame {        // one entry of recent_surf_frames (world frame, point_stride bytes per point)
    DevBuf buf;
    int n = 0;
    // incremental map (map_inc.cu): slot id carried by the frame's entries, unrepresentable key seen
    int slot = 0;
    bool bad = false;
    // box of the stored points (vg_box.h; mm[6] = finite points), taken when the frame was pushed: the rebuild's VoxelGrid, the
    // cell grid and the incremental map get their bounding boxes from the union over the frames instead of passes over the map
    int mm[kBoxInts] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN, 0};
};

}  // namespace lili

struct liliom_ctx {
    liliom_params prm;
    int device = 0;
    cudaStream_t stream = nullptr;       // stream all work is issued on (own_stream unless liliom_set_stream)
    cudaStream_t own_stream = nullptr;
    cudaStream_t copy_stream = nullptr;  // D2H of a finished output while later kernels of the same call still run
    cudaEvent_t  ev_ready = nullptr, ev_copied = nullptr;
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
    bool vg_check = false;       // s2m_run also reads vg_params back (speculative key width of the scan VoxelGrid)
    bool vg_used24 = false;      // ... the sort chain ran with 24-bit keys
    bool vg_bail = false;        // ... the cooperative filter declined (valid after the sync)
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
    lili::DevBuf raw_ring;       // LILIOM_RING_FIELD: u16 ring id per point of c->raw (liliom_extract_rot_pc2)
    lili::DevBuf raw_scan_ring;  // ... of the resident sweep (liliom_convert_pc2)
    bool raw_scan_rings = false; // raw_scan_ring holds the ring ids of the resident sweep
    int time_source = LILIOM_TIME_AZIMUTH;     // liliom_set_time_source
    char time_name[16] = {};     // LILIOM_TIME_FIELD: the name of the per-point time field
    lili::DevBuf raw_time;       // LILIOM_TIME_FIELD: double time per point of c->raw (liliom_extract_rot_pc2)
    lili::DevBuf raw_scan_time;  // ... of the resident sweep (liliom_convert_pc2)
    bool raw_scan_times = false; // raw_scan_time holds the times of the resident sweep
    int n_rot_cloud = 0;

    // ---- voxel grid scratch ----
    lili::DevBuf vg_keys, vg_keys2, vg_vals, vg_vals2, vg_flags, vg_rank, vg_params, vg_out, vg_minmax, vg_count;
    lili::DevBuf cub_tmp;

    // ---- map ----
    std::vector<lili::Frame> frames;     // FIFO, oldest first
    // incremental map (liliom_map_update, map_inc.cu): entries {voxel key, slot<<24|index} sorted by (key, frame age, index), double-buffered
    lili::DevBuf inc_key[2], inc_ref[2], inc_newkey[2], inc_newref[2], inc_removed, inc_rpos, inc_flags, inc_rank, inc_bad;
    int inc_cur = 0, inc_E = 0;
    bool inc_valid = false;
    lili::DevBuf map_raw;                // concatenated frames (stride bytes)
    lili::DevBuf map_ds;                 // VoxelGrid output (stride bytes) or installed float4
    lili::MapIndex map;                  // the odometry map's search index (scan-to-map, backend single-keyframe calls, ICP target)
    lili::DevBuf grid_keys, grid_keys2, grid_vals, grid_vals2;   // grid_build scratch, shared by every index
    int map_n_global = 0;

    // ---- backend (keyframes.cu, backend_corr.cu): keyframe store, local map layers, window correspondences ----
    lili::DevBuf kf_arena;               // body-frame clouds of every keyframe (point_stride bytes per point)
    long long kf_used = 0;               // points in use
    lili::DevBuf kf_full;                // full clouds of the keyframes (liliom_kf_add_full), point_stride bytes per point
    long long kf_full_used = 0;          // points in use
    std::vector<lili::KfEntry> kfs;      // per keyframe: offsets and counts (host)
    lili::DevBuf kf_tab;                 // per-call keyframe table (kf_table.h: k_kf_gather, the global map's kernels)
    lili::MapIndex bmap[2];              // backend local map: [0] edge layer, [1] surf layer
    lili::DevBuf bmap_raw, bmap_ds[2];   // concatenation of the transformed keyframes; the filtered layers (all fields)
    int bmap_n[2] = {0, 0};
    bool bmap_built = false;
    int win_k = 0;                       // window correspondences resident (liliom_backend_window_correspond)
    liliom_backend_params win_bp{};      // ... and the parameters they were found with (weights, extrinsics, loss of the blocks)
    std::vector<int> win_ids;
    std::vector<long long> win_qoff[2];  // per kind: query prefix offsets (k + 1)
    lili::DevBuf win_valid[2], win_line, win_plane, win_score, win_cnt, win_tab;
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
    lili::DevBuf icp_ctl;                // ICP kernel: barrier word, and its results when the pinned block is not mappable
    int bk_kind = 0, bk_n = 0;           // backend correspondences resident from the last liliom_correspond_* call (1 edge, 2 surf)
    unsigned int bar_arrivals = 0;       // total grid-barrier arrivals issued so far (persistent GN kernel)

    // ---- multi-GPU ----
    void* nccl_comm = nullptr;
    int nranks = 1, rank = 0;
    float shard_inv_block = 0.0625f;     // 1 / shard block edge (LILIOM_SHARD_BLOCK, metres, power of two; must agree on all ranks)
    lili::DevBuf peer_local;             // block 0 -> other blocks of this GPU: [2][32] doubles + 2 epoch words (fused exchange)
    lili::DevBuf peer_buf;               // this rank's exchange buffer: [2 parities][kMaxPeers][32] {epoch|lo32, epoch|hi32}
    void* peer_ptrs[lili::kMaxPeers] = {};   // every rank's buffer as mapped into this process (cudaIpcOpenMemHandle)
    bool peer_ready = false;
    unsigned int peer_epoch = 0;         // last epoch issued

    // ---- instrumentation ----
    liliom_counters cnt{};
    bool time_kernels = false;
    int  time_every = 1;          // liliom_set_kernel_timing(c, N): time every N-th scan-to-map call
    unsigned time_calls = 0;
    // run-time switches: read by liliom_create and nowhere else (DESIGN.md §6)
    int force_lanes = 0, force_rounds = 0;   // tuning override (LILIOM_KNN_LANES / LILIOM_KNN_ROUNDS)
    int gn_sync = 3;                     // persistent kernels' grid barrier (LILIOM_GN_SYNC): 3 = release-only arrival, no acquire fence (default),
                                         // 1 = acquire poll, 0 = full fences on both sides
    bool dbg_timing = false;             // LILIOM_DEBUG_TIMING: stage clocks of the cooperative kernels, printed by s2m_run
    bool rot_slow_walk = false;          // LILIOM_ROT_SLOW_WALK (test hook): the general walk of k_rot_ring for every segment
    bool test_shrink_box = false;        // LILIOM_TEST_SHRINK_BOX (test hook): grid_build takes a box too small in x
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

// ---- modules (implemented in the .cu files) ----
int sort_pairs_u32(liliom_ctx* c, const uint32_t* kin, uint32_t* kout, const int* vin, int* vout, int n, int end_bit);
int sort_pairs_u64(liliom_ctx* c, const unsigned long long* kin, unsigned long long* kout, const int* vin, int* vout, int n, int end_bit);
int exclusive_scan_i32(liliom_ctx* c, const int* in, int* out, int n);   // out has n+1 entries (total at out[n])
int inclusive_max_scan_i32(liliom_ctx* c, int* data, int n);            // in-place running maximum

// VoxelGrid on device buffers; d_count receives the output count (int, device).  n_max = host upper bound, d_n = optional
// device-side count (<= n_max); d_feats (optional) also receives float4{x,y,z,index}.  key_bits, host_mm: see voxelgrid.cu.
int voxelgrid_dev(liliom_ctx* c, const void* d_in, int n_max, const int* d_n, int stride, float leaf, void* d_out, int* d_count,
                  float4* d_feats = nullptr, int key_bits = 32, const int* host_mm = nullptr);
int vg_minmax_dev(liliom_ctx* c, const void* d_in, int n_max, const int* d_n, int stride);
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

const long long* vg_coop_stamps(liliom_ctx* c);   // voxelgrid.cu

int s2m_run(liliom_ctx* c, double pose7[7], int match_cnt, int max_num_iter, int mode, liliom_iter_stats* stats,
            bool want_corr, double out29[29]);

int horizon_extract_dev(liliom_ctx* c, int n, const double q_imu[4], int* n_surf, int* n_edge, int* n_cut, bool sync_counts = true);
// rings: nullptr = scanID from the elevation tables (line_num 16/32/64), else the u16 ring id of every input point (line_num 1..128)
// times: nullptr = relTime from the azimuth rule, else the time of every input point (LILIOM_TIME_FIELD)
int rot_extract_dev(liliom_ctx* c, int n, const double q_imu[4], const double q_lb[4], int* n_surf, int* n_edge, int* n_cut,
                    const uint16_t* rings = nullptr, const double* times = nullptr);
bool rot_lines_ok(int line_num, bool field);

int icp_align(liliom_ctx* c, const MapIndex& tgt, const float4* d_src, int n, double max_corr_dist, int max_iter, double trans_eps,
              double fit_eps, double T16[16], double* fitness, int* converged, int* iters);     // icp.cu
int map_inc_update(liliom_ctx* c, int popped_slot, int popped_nfin, int* m_out);     // map_inc.cu
int map_finish_from_ds(liliom_ctx* c, int m);                                        // api.cu
void frames_box(const liliom_ctx* c, int mm[7]);                                     // api.cu: union of the frames' boxes

int block27_stats(liliom_ctx* c, const double pose7[7], unsigned long long out[2]);   // grid_knn.cu

int repack_to_f4(liliom_ctx* c, const void* d_in, int n, int stride, float4* d_out, const int* d_n = nullptr);

}  // namespace lili
