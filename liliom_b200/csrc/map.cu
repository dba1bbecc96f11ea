// The odometry local map (L/src/LidarOdometry.cpp:246-323, 490): the FIFO of the last max_map_frames transformed frames, its
// VoxelGrid (the rebuild, or the incremental update below) and cell grid, the installed maps, the shard filter of multi-GPU
// contexts, and every liliom_map_* entry point.  Compiled with --fmad=false: the transform and the centroid sums are bit-exact
// with the reference's arithmetic.
//
// SURVEY.md §8 (f2): device-resident INCREMENTAL local map — liliom_map_update = liliom_map_push_frame + liliom_map_rebuild,
// bit for bit, without re-sorting the 20-frame concatenation every scan
// (replaces L/src/LidarOdometry.cpp:280-303 buildLocalMap, :316-317 downSampleCloud(map), per scan).
//
// pcl::VoxelGrid's output is (a) the occupied voxels in ascending index idx = i + j*dx + k*dx*dy, which is the lexicographic
// (k, j, i) order of the ABSOLUTE voxel coordinates floor(p / leaf) whatever the bounding box (i, j, k differ from them by the
// box minimum only), and (b) per voxel the centroid of its members summed in input order, here: frames oldest first, points
// in frame order (the stable order voxelgrid.cu and the oracle define).  So the filter's state can live across scans as ONE
// array of entries {voxel key, (frame slot, point index)} sorted by (key, frame age, index):
//   * the newest frame's entries are sorted on their own (n_f log n_f) and MERGED in by rank arithmetic — an old entry moves
//     down by the number of new entries with a smaller key (one binary search in the new frame's keys), a new entry lands
//     behind every old entry with key <= its own (one binary search in the old keys): equal keys keep "older frame first";
//   * the entries of the frame that leaves the FIFO are dropped in the same pass (flag + exclusive scan);
//   * voxel heads, output ranks and centroids are then recomputed from the merged array exactly as the sort chain does it
//     (same sequential fp32 sums: compiled with --fmad=false like voxelgrid.cu).
// Per scan this is a handful of streaming passes over the entry array instead of 4 radix passes over 8-byte pairs + the concat;
// the cell grid for the search is rebuilt from the filtered cloud as before (grid_build).
// Inputs the absolute-key scheme cannot represent (|voxel coordinate| >= 2^20, PCL's int32 index overflow) and sharded contexts
// take the ordinary push + rebuild path; the result is the same by construction.
#include "ctx.cuh"
#include "dev_math.cuh"
#include "knn_core.cuh"
#include <algorithm>
#include <climits>
#include <vector>
#include <ctime>

namespace lili {
int nccl_allreduce_sum_f64(liliom_ctx* c, double* buf, int count);   // comm.cu

// ---- map sharding (multi-GPU): flags[i] = shard_keep() of record i (stride bytes, x y z first); flags[n] = 0 (scan sentinel)
__global__ void k_shard_flags(const unsigned char* __restrict__ p, int n, int stride, float halo, float inv_block, int nranks, int rank,
                              int* __restrict__ flags) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    int f = 0;
    if (i < n) {
        const float4 v = *reinterpret_cast<const float4*>(p + (size_t)i * stride);
        f = shard_keep(v.x, v.y, v.z, halo, nranks, rank, inv_block);
    }
    flags[i] = f;
}
__global__ void k_compact_strided(const unsigned char* __restrict__ in, const int* __restrict__ flags, const int* __restrict__ pos, int n, int stride,
                                  unsigned char* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !flags[i]) return;
    const float4* src = reinterpret_cast<const float4*>(in + (size_t)i * stride);
    float4* dst = reinterpret_cast<float4*>(out + (size_t)pos[i] * stride);
    for (int k = 0; k < stride / 16; ++k) dst[k] = src[k];
}
// the shard filter and the repack to float4 {x,y,z,index} in one pass (on float4 input whose w is already the index, as every
// installed map's is, it writes the kept records unchanged)
__global__ void k_compact_repack(const unsigned char* __restrict__ in, const int* __restrict__ flags, const int* __restrict__ pos, int n, int stride,
                                 float4* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !flags[i]) return;
    float4 v = *reinterpret_cast<const float4*>(in + (size_t)i * stride);
    v.w = __int_as_float(i);
    out[pos[i]] = v;
}

// *count += the points of p[0..n) that this rank owns (owner_of): over all ranks, every voxel of a sharded map counted once
__global__ void k_count_owned(const float4* __restrict__ p, int n, float inv_block, int nranks, int rank, int* __restrict__ count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    bool own = false;
    if (i < n) { const float4 v = p[i]; own = owner_of(v.x, v.y, v.z, nranks, inv_block) == rank; }
    const unsigned b = __ballot_sync(0xffffffffu, own);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(count, __popc(b));
}

// transformCloud (L/src/LidarOdometry.cpp:246-278; R/src/LidarOdometry.cpp:239-264).  Every kernel of the map update has its body in
// a function of `i`, the thread's place in its session's launch: the solo kernel passes blockIdx.x * blockDim.x + threadIdx.x,
// the batched update (k_stage_batch, ctx.cuh) the same place counted from its session's first block.
__device__ __forceinline__ void transform_cloud_at(const unsigned char* __restrict__ in, int n, int stride, const Q4& q, const D3& t,
                                                   unsigned char* __restrict__ out, const int i) {
    if (i >= n) return;
    pcl_transform_point(in + (size_t)i * stride, stride, q, t, out + (size_t)i * stride);
}
__global__ void k_transform_cloud(const unsigned char* __restrict__ in, int n, int stride, Q4 q, D3 t, unsigned char* __restrict__ out) {
    transform_cloud_at(in, n, stride, q, t, out, blockIdx.x * blockDim.x + threadIdx.x);
}

// Concatenation of the FIFO frames (L/src/LidarOdometry.cpp:301-302), up to kConcatMax frames per launch: blockIdx.y = frame,
// the blocks of a row stream that frame's 16-byte words to its offset in the concatenated cloud.  (20 cudaMemcpyAsync calls
// cost a fixed latency per copy whatever the size, which a single launch does not.)
constexpr int kConcatMax = 64;
struct ConcatTab { const float4* src[kConcatMax]; long long off[kConcatMax + 1]; };      // offsets in 16-byte words
__global__ void k_concat_frames(const __grid_constant__ ConcatTab tab, float4* __restrict__ out) {
    const int f = blockIdx.y;
    const long long n16 = tab.off[f + 1] - tab.off[f];
    const float4* __restrict__ src = tab.src[f];
    float4* __restrict__ dst = out + tab.off[f];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i];
}

typedef unsigned long long u64;
constexpr int kIncSlots = 64;                 // frame slots (refs carry the slot in their top 6 bits... 8 bits reserved)
constexpr unsigned kIncIdxMask = (1u << 24) - 1u;
struct FrameTab { const unsigned char* base[kIncSlots]; };

// keys of one frame's points (world frame, already transformed), refs = slot << 24 | index; *bad |= 1 when a voxel coordinate
// does not fit 21 bits (the frame's box and finite count were measured at its push: Frame::mm)
__device__ __forceinline__ void inc_keys_at(const unsigned char* __restrict__ pts, int n, int stride, float inv_leaf, unsigned slot,
                                            u64* __restrict__ keys, unsigned* __restrict__ refs, int* __restrict__ bad, const int i) {
    bool miss = false;
    if (i < n) {
        const float4 v = *reinterpret_cast<const float4*>(pts + (size_t)i * stride);
        u64 key = ~0ull;
        if (isfinite(v.x) && isfinite(v.y) && isfinite(v.z)) miss = !vg_abs_key(v.x, v.y, v.z, inv_leaf, &key);
        keys[i] = key;
        refs[i] = (slot << 24) | (unsigned)i;
    }
    if (__any_sync(0xffffffffu, miss) && (threadIdx.x & 31) == 0) atomicOr(bad, 1);
}
__global__ void k_inc_keys(const unsigned char* __restrict__ pts, int n, int stride, float inv_leaf, unsigned slot, u64* __restrict__ keys,
                           unsigned* __restrict__ refs, int* __restrict__ bad) {
    inc_keys_at(pts, n, stride, inv_leaf, slot, keys, refs, bad, blockIdx.x * blockDim.x + threadIdx.x);
}

__device__ __forceinline__ int lower_bound_u64(const u64* __restrict__ a, int n, u64 k) {      // first i with a[i] >= k
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (__ldg(a + mid) < k) lo = mid + 1; else hi = mid; }
    return lo;
}
__device__ __forceinline__ int upper_bound_u64(const u64* __restrict__ a, int n, u64 k) {      // first i with a[i] > k
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (__ldg(a + mid) <= k) lo = mid + 1; else hi = mid; }
    return lo;
}

// removed[i] = 1 for the entries of the frame slot that leaves the FIFO; removed[E] = 0 (scan sentinel)
__device__ __forceinline__ void inc_mark_at(const unsigned* __restrict__ refs, int E, int popped, int* __restrict__ removed, const int i) {
    if (i > E) return;
    removed[i] = (i < E && popped >= 0 && (int)(refs[i] >> 24) == popped) ? 1 : 0;
}
__global__ void k_inc_mark(const unsigned* __restrict__ refs, int E, int popped, int* __restrict__ removed) {
    inc_mark_at(refs, E, popped, removed, blockIdx.x * blockDim.x + threadIdx.x);
}
// surviving old entries: down by the removed entries before them, up by the new entries with a smaller key.  The entries of a
// warp are consecutive in a sorted array, so their lower bounds in the new keys are nested between those of lanes 0 and 31:
// two full binary searches per warp, then every lane searches only the (short) range between them.
__device__ __forceinline__ void inc_merge_old_at(const u64* __restrict__ keys, const unsigned* __restrict__ refs, const int* __restrict__ removed,
                                                 const int* __restrict__ rpos, int E, const u64* __restrict__ newkeys, int nnew,
                                                 u64* __restrict__ keys2, unsigned* __restrict__ refs2, const int i) {
    const int lane = threadIdx.x & 31;
    const int ic = min(i, E - 1);
    const u64 k = keys[ic];
    int lb = 0;
    if (lane == 0 || lane == 31) lb = lower_bound_u64(newkeys, nnew, k);
    const int lo = __shfl_sync(0xffffffffu, lb, 0), hi = __shfl_sync(0xffffffffu, lb, 31);
    if (lane != 0 && lane != 31) lb = lo + lower_bound_u64(newkeys + lo, hi - lo, k);
    if (i >= E || removed[i]) return;
    const int pos = i - rpos[i] + lb;
    keys2[pos] = k; refs2[pos] = refs[i];
}
__global__ void k_inc_merge_old(const u64* __restrict__ keys, const unsigned* __restrict__ refs, const int* __restrict__ removed,
                                const int* __restrict__ rpos, int E, const u64* __restrict__ newkeys, int nnew, u64* __restrict__ keys2,
                                unsigned* __restrict__ refs2) {
    inc_merge_old_at(keys, refs, removed, rpos, E, newkeys, nnew, keys2, refs2, blockIdx.x * blockDim.x + threadIdx.x);
}
// new entries (sorted by key, then index): behind every surviving old entry with key <= their own
__device__ __forceinline__ void inc_merge_new_at(const u64* __restrict__ newkeys, const unsigned* __restrict__ newrefs, int nnew,
                                                 const u64* __restrict__ keys, const int* __restrict__ rpos, int E, u64* __restrict__ keys2,
                                                 unsigned* __restrict__ refs2, const int j) {
    if (j >= nnew) return;
    const u64 k = newkeys[j];
    const int ub = upper_bound_u64(keys, E, k);
    const int pos = j + (ub - rpos[ub]);
    keys2[pos] = k; refs2[pos] = newrefs[j];
}
__global__ void k_inc_merge_new(const u64* __restrict__ newkeys, const unsigned* __restrict__ newrefs, int nnew, const u64* __restrict__ keys,
                                const int* __restrict__ rpos, int E, u64* __restrict__ keys2, unsigned* __restrict__ refs2) {
    inc_merge_new_at(newkeys, newrefs, nnew, keys, rpos, E, keys2, refs2, blockIdx.x * blockDim.x + threadIdx.x);
}
// centroid of every voxel, members in entry order (vg_box.h), the points fetched through the frame table
template <int STRIDE>
__device__ __forceinline__ void inc_centroid_at(const FrameTab& tab, const u64* __restrict__ keys, const unsigned* __restrict__ refs,
                                                const int* __restrict__ flags, const int* __restrict__ rank, int E,
                                                unsigned char* __restrict__ out, int* __restrict__ count_out, const int i) {
    if (i == 0) *count_out = rank[E];
    if (i >= E || !flags[i]) return;
    const VgAcc<STRIDE> a = vg_walk<STRIDE>(keys, i, E, [&](int j) { return (int)refs[j]; },       // (slot < 64: a ref is below 2^30)
                                            [&](int r) { return tab.base[r >> 24] + (size_t)(r & kIncIdxMask) * STRIDE; });
    vg_write<STRIDE>(a.s, a.n, out + (size_t)rank[i] * STRIDE);
}
template <int STRIDE>
__global__ void k_inc_centroid(const __grid_constant__ FrameTab tab, const u64* __restrict__ keys, const unsigned* __restrict__ refs,
                               const int* __restrict__ flags, const int* __restrict__ rank, int E, unsigned char* __restrict__ out,
                               int* __restrict__ count_out) {
    inc_centroid_at<STRIDE>(tab, keys, refs, flags, rank, E, out, count_out, blockIdx.x * blockDim.x + threadIdx.x);
}

// ---- the map update of several sessions (liliom_map_update_batch): one launch per stage for up to kBatchMax sessions.
// Everything one session's stages read or write, on its own buffers; the host parts of the update fill it as they go (MapJob).
struct MapEntry {
    // the new frame: transform, box, keys
    const unsigned char* src; unsigned char* fbuf; int n, stride; Q4 q; D3 t; int* mm; int mm_blocks;
    float inv_leaf; unsigned slot; u64* newkey; unsigned* newref; int* bad;
    // merge into the entry array
    const u64* keys; const unsigned* refs; int E, popped; int* removed; int* rpos; const u64* snewkey; const unsigned* snewref; int nnew;
    u64* keys2; unsigned* refs2;
    // voxel heads and centroids of the entry array (ekeys / erefs, E2 entries)
    const u64* ekeys; const unsigned* erefs; int E2; int* flags; int* rank; unsigned char* ds; int* count;
    // search index of the m filtered points
    int m; float4* xyzw; GridDesc g; uint32_t* gkeys; int* gvals; int* escaped; const uint32_t* gkeys2; const int* gvals2; float4* sorted;
    int* cell_start;
};
// The centroid stage also needs each session's frame pointers
struct MapCentroidEntry {
    FrameTab tab;
    const u64* ekeys; const unsigned* erefs; int E2, stride; const int* flags; const int* rank; unsigned char* ds; int* count;
};

// The stages of the update (k_stage_batch, ctx.cuh), each with the block size, the blocks and the body of its solo launch
LILI_STAGE(MapStTransform, MapEntry, 256, stage_blocks(e.n, 256), transform_cloud_at(e.src, e.n, e.stride, e.q, e.t, e.fbuf, i))
LILI_STAGE(MapStBoxInit, MapEntry, 32, 1, vg_box_init(e.mm))
LILI_STAGE(MapStBox, MapEntry, 256, e.mm_blocks, vg_minmax_body(e.fbuf, e.n, nullptr, e.stride, e.mm, SessionBlock{bx, (unsigned)e.mm_blocks}))
LILI_STAGE(MapStKeys, MapEntry, 256, stage_blocks(e.n, 256), inc_keys_at(e.fbuf, e.n, e.stride, e.inv_leaf, e.slot, e.newkey, e.newref, e.bad, i))
LILI_STAGE(MapStMark, MapEntry, 256, stage_blocks(e.E + 1, 256), inc_mark_at(e.refs, e.E, e.popped, e.removed, i))
LILI_STAGE(MapStMergeOld, MapEntry, 256, stage_blocks(e.E, 256),
           inc_merge_old_at(e.keys, e.refs, e.removed, e.rpos, e.E, e.snewkey, e.nnew, e.keys2, e.refs2, i))
LILI_STAGE(MapStMergeNew, MapEntry, 256, stage_blocks(e.nnew, 256),
           inc_merge_new_at(e.snewkey, e.snewref, e.nnew, e.keys, e.rpos, e.E, e.keys2, e.refs2, i))
LILI_STAGE(MapStHeads, MapEntry, 256, stage_blocks(e.E2 + 1, 256), vg_heads_at(e.ekeys, e.E2, (const int*)nullptr, e.flags, i))
LILI_STAGE(MapStRepack, MapEntry, 256, stage_blocks(e.m, 256), repack_f4_at(e.ds, e.m, nullptr, e.stride, e.xyzw, i))
LILI_STAGE(MapStCellKeys, MapEntry, 256, stage_blocks(e.m, 256), cell_keys_at(e.xyzw, e.m, e.g, e.gkeys, e.gvals, e.escaped, i))
LILI_STAGE(MapStGather, MapEntry, 256, stage_blocks(e.m, 256), gather_sorted_at(e.xyzw, e.gvals2, e.m, e.sorted, i))
LILI_STAGE(MapStRunEnds, MapEntry, 256, stage_blocks(e.m, 256), cell_run_ends_at(e.gkeys2, e.m, e.cell_start, i))
// The centroids: the scalars by value, the 512-byte frame table read in place from the parameter space (as k_inc_centroid reads its own)
template <int STRIDE>
struct MapStCentroid {
    typedef MapCentroidEntry Entry;
    static constexpr int kThreads = 128;
    static int blocks(const MapCentroidEntry& e) { return stage_blocks(e.E2, 128); }
    __device__ static void run(const MapCentroidEntry& te, int bx) {
        const u64* ekeys = te.ekeys; const unsigned* erefs = te.erefs; const int* flags = te.flags; const int* rank = te.rank;
        inc_centroid_at<STRIDE>(te.tab, ekeys, erefs, flags, rank, te.E2, te.ds, te.count, bx * 128 + (int)threadIdx.x);
    }
};

// ---- host side

// Shard filter (multi-GPU): the n records of `in` (stride bytes each) that shard_keep() gives this rank, in their order, into
// `out` (repack: as float4 {x, y, z, index in `in`}; otherwise whole records); *kept = their count.  box (optional): the box of
// the kept records (vg_box.h), read back with the count.
static int shard_filter(liliom_ctx* c, const void* in, int n, int stride, float halo, void* out, bool repack, int* kept,
                        int* box = nullptr) {
    LILI_CUDA(c, c->flags.ensure(((size_t)n + 2) * 4));
    LILI_TRY(feat_keep_cut(c));
    LILI_CUDA(c, c->idx_a.ensure(((size_t)n + 2) * 4));
    const unsigned char* p = (const unsigned char*)in;
    int* flags = c->flags.as<int>();
    int* pos = c->idx_a.as<int>();
    k_shard_flags<<<cdiv(n + 1, 256), 256, 0, c->stream>>>(p, n, stride, halo, c->shard_inv_block, c->nranks, c->rank, flags);
    LILI_TRY(launch_check(c, "k_shard_flags"));
    LILI_TRY(exclusive_scan_i32(c, flags, pos, n));
    if (repack) {
        k_compact_repack<<<cdiv(n, 256), 256, 0, c->stream>>>(p, flags, pos, n, stride, (float4*)out);
        LILI_TRY(launch_check(c, "k_compact_repack"));
    } else {
        k_compact_strided<<<cdiv(n, 256), 256, 0, c->stream>>>(p, flags, pos, n, stride, (unsigned char*)out);
        LILI_TRY(launch_check(c, "k_compact_strided"));
    }
    if (!box) return read_back(c, {{kept, pos + n, sizeof(int)}});
    LILI_TRY(vg_minmax_dev(c, out, n, pos + n, stride));
    return read_back(c, {{kept, pos + n, sizeof(int)}, {box, c->vg_minmax.p, kBoxInts * sizeof(int)}});
}

// No search index and no filtered cloud: what the map is between a reset and the end of the rebuild or update that follows.
static void map_reset(liliom_ctx* c) {
    c->map.ready = false; c->map.n = 0; c->map_n_global = 0; c->map_ds_n = 0;
}

// Installs m host points (stride 16: float4, w ignored; 32 / 48: PCL layout) as the odometry map, sharded when a communicator
// is attached.  keep_refl: with the reflectivity channel (the curvature field of 48-byte points, zeros otherwise).  An installed
// map has no filtered cloud behind it (liliom_map_download_cloud).
int map_install_host(liliom_ctx* c, const void* pts, int m, int stride, bool keep_refl) {
    const size_t cap = (size_t)(m > 0 ? m : 1);
    if (!keep_refl) c->map.refl.release();
    c->map.ready = false;
    LILI_CUDA(c, c->map.xyzw.ensure(cap * sizeof(float4)));
    if (keep_refl) LILI_CUDA(c, c->map.refl.ensure(cap * sizeof(float)));
    LILI_CUDA(c, c->raw.ensure(cap * stride));
    if (m > 0) {
        LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, pts, (size_t)m * stride, cudaMemcpyHostToDevice, c->stream));
        LILI_TRY(repack_to_f4(c, c->raw.p, m, stride, c->map.xyzw.as<float4>()));
        if (keep_refl && stride == 48) {
            k_kf_refl<<<cdiv(m, 256), 256, 0, c->stream>>>((const unsigned char*)c->raw.p, m, c->map.refl.as<float>());
            LILI_TRY(launch_check(c, "k_kf_refl"));
        } else if (keep_refl) LILI_CUDA(c, cudaMemsetAsync(c->map.refl.p, 0, (size_t)m * sizeof(float), c->stream));
    }
    c->map_n_global = m;
    c->map_ds_n = -1;
    if (c->nranks > 1 && m > 0) {
        LILI_CUDA(c, c->map_ds.ensure((size_t)m * sizeof(float4)));
        LILI_TRY(shard_filter(c, c->map.xyzw.p, m, 16, gate_cell(c->prm.knn_max_sqdist), c->map_ds.p, true, &m));
        LILI_CUDA(c, cudaMemcpyAsync(c->map.xyzw.p, c->map_ds.p, (size_t)m * sizeof(float4), cudaMemcpyDeviceToDevice, c->stream));
    }
    return grid_build(c, m);
}

// The frame that left the FIFO in a push: its slot and finite count (slot -1, count 0: none left).
struct Popped { int slot = -1, nfin = 0; };

// One map update in flight.  The update is written in parts so that the solo call and the batched one (map_update_batch) run
// the same host code: each *_begin part takes the host's decisions (FIFO, buffer sizes, fall-backs) from the words read back so
// far and fills the kernel arguments in `e`; the launches between the parts are the solo kernels here and the shared stage
// launches there.
struct MapJob {
    liliom_ctx* c = nullptr;
    Frame f;                            // the frame being pushed, until push_end moves it into the FIFO
    Popped popped;
    MapEntry e{};
    FrameTab ft{};
    GridJob g;
    int m = 0;                          // voxels of the filtered cloud
};

// Push, part 1: the FIFO makes room (L/src/LidarOdometry.cpp:293-296 pop_front) and the new frame gets its buffer.
static int push_begin(liliom_ctx* c, const void* d_src, int n, const double pose7[7], bool keep_inc, MapJob& j) {
    const int stride = c->prm.point_stride;
    j.c = c;
    if (!keep_inc) c->inc_valid = false;        // the entry array of liliom_map_update no longer describes the FIFO
    Frame& f = j.f;
    f.slot = (int)c->frames.size();
    if ((int)c->frames.size() >= c->prm.max_map_frames && !c->frames.empty()) {
        Frame& old = c->frames.front();
        j.popped = Popped{old.slot, old.mm[6]};
        f.buf = std::move(old.buf);             // the popped frame's allocation is recycled: cudaFree + cudaMalloc per scan cost
        f.slot = old.slot;                      // more than the whole map maintenance of a 10 M-point map (cudaFree synchronises)
        c->frames.erase(c->frames.begin());
    }
    f.n = n;
    if (n > 0) {
        LILI_CUDA(c, f.buf.ensure((size_t)n * stride));
        LILI_CUDA(c, c->vg_minmax.ensure(8 * sizeof(int)));
    }
    MapEntry& e = j.e;
    e.src = (const unsigned char*)d_src; e.fbuf = (unsigned char*)f.buf.p; e.n = n; e.stride = stride;
    e.q = Q4{pose7[0], pose7[1], pose7[2], pose7[3]};
    e.t = D3{pose7[4], pose7[5], pose7[6]};
    e.mm = c->vg_minmax.as<int>();
    e.mm_blocks = box_blocks(n, c->sm_count);     // vg_minmax_dev's grid
    return LILIOM_OK;
}
// Push, part 2: the frame's box as read back (nullptr: an empty frame keeps the empty box) and its place in the FIFO.
static void push_end(MapJob& j, const int* mm) {
    if (mm) memcpy(j.f.mm, mm, kBoxInts * sizeof(int));
    j.c->frames.push_back(std::move(j.f));
}

// Shared body of the push entry points: d_src = n body-frame points of point_stride bytes ON THE DEVICE.
static int push_frame_from_device(liliom_ctx* c, const void* d_src, int n, const double pose7[7], bool keep_inc = false,
                                  Popped* popped = nullptr) {
    MapJob j;
    LILI_TRY(push_begin(c, d_src, n, pose7, keep_inc, j));
    if (popped) *popped = j.popped;
    const MapEntry& e = j.e;
    Frame& f = j.f;
    if (n > 0) {
        if (c->nranks == 1) {
            k_transform_cloud<<<cdiv(n, 256), 256, 0, c->stream>>>(e.src, n, e.stride, e.q, e.t, e.fbuf);
            LILI_TRY(launch_check(c, "k_transform_cloud"));
            LILI_TRY(vg_minmax_dev(c, f.buf.p, n, nullptr, e.stride));                 // the frame's box, for the rebuilds it takes part in
            LILI_TRY(read_back(c, {{f.mm, c->vg_minmax.p, kBoxInts * sizeof(int)}}));
        } else {
            // sharded map maintenance: every rank receives the frame, keeps the points within (search radius + one voxel
            // diagonal) of a block it owns — every voxel that can reach an owned query's 1 m ball is then complete locally —
            // and voxel-filters / indexes only its shard.  No inter-rank traffic.
            LILI_CUDA(c, c->map_ds.ensure((size_t)n * e.stride));
            k_transform_cloud<<<cdiv(n, 256), 256, 0, c->stream>>>(e.src, n, e.stride, e.q, e.t, (unsigned char*)c->map_ds.p);
            LILI_TRY(launch_check(c, "k_transform_cloud"));
            // The frame's extent is that of the WHOLE transformed frame, as one GPU measures it: PCL's declined case and its
            // wrapping index depend on the box, and every rank must decide them as one GPU does.  The finite count is that of the
            // points this rank keeps, the points its VoxelGrid filters.
            int whole[kBoxInts];
            LILI_TRY(vg_minmax_dev(c, c->map_ds.p, n, nullptr, e.stride));
            LILI_TRY(read_back(c, {{whole, c->vg_minmax.p, kBoxInts * sizeof(int)}}));
            const float halo = gate_cell(c->prm.knn_max_sqdist) + 1.7320508f * c->prm.leaf_map + 0.05f;
            LILI_TRY(shard_filter(c, c->map_ds.p, n, e.stride, halo, f.buf.p, false, &f.n, f.mm));
            for (int k = 0; k < 6; ++k) f.mm[k] = whole[k];
        }
    }
    push_end(j, nullptr);
    return LILIOM_OK;
}

// union of the frames' boxes: the box and finite count of their concatenation
static void frames_box(const liliom_ctx* c, int mm[kBoxInts]) {
    for (int k = 0; k < kBoxInts; ++k) mm[k] = vg_box_empty(k);
    for (const auto& f : c->frames) vg_box_merge(mm, f.mm);
}

// Tail of the incremental update (single GPU), part 1: c->map_ds holds m filtered points; sizes the float4 map for the repack.
static int finish_begin(liliom_ctx* c, int m, MapEntry& e) {
    LILI_CUDA(c, c->map.xyzw.ensure((size_t)(m > 0 ? m : 1) * sizeof(float4)));
    c->map_n_global = m;
    c->map_ds_n = m;
    e.ds = (unsigned char*)c->map_ds.p; e.m = m; e.stride = c->prm.point_stride; e.xyzw = c->map.xyzw.as<float4>();
    return LILIOM_OK;
}

static int map_finish_from_ds(liliom_ctx* c, int m) {
    MapEntry e{};
    LILI_TRY(finish_begin(c, m, e));
    LILI_TRY(repack_to_f4(c, e.ds, m, e.stride, e.xyzw));
    int mm[kBoxInts];
    frames_box(c, mm);
    LILI_TRY(grid_build(c, m, mm[6] > 0 ? mm : nullptr));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

// keys + refs of frame `f` (points already in f.buf) go to keys / refs and its key flag to c->inc_bad: the flag cleared, the
// arguments of k_inc_keys in `e`
static int inc_keys_begin(liliom_ctx* c, const Frame& f, u64* keys, unsigned* refs, MapEntry& e) {
    LILI_CUDA(c, c->inc_bad.ensure(sizeof(int)));
    e.fbuf = (unsigned char*)f.buf.p; e.n = f.n; e.stride = c->prm.point_stride;
    e.inv_leaf = 1.0f / c->prm.leaf_map; e.slot = (unsigned)f.slot; e.newkey = keys; e.newref = refs; e.bad = c->inc_bad.as<int>();
    LILI_CUDA(c, cudaMemsetAsync(e.bad, 0, sizeof(int), c->stream));
    return LILIOM_OK;
}

// keys + refs of frame `f`, written at keys/refs, and its key flag; one sync
static int inc_frame_keys(liliom_ctx* c, Frame& f, u64* keys, unsigned* refs) {
    MapEntry e{};
    LILI_TRY(inc_keys_begin(c, f, keys, refs, e));
    if (f.n > 0) {
        k_inc_keys<<<cdiv(f.n, 256), 256, 0, c->stream>>>(e.fbuf, e.n, e.stride, e.inv_leaf, e.slot, e.newkey, e.newref, e.bad);
        LILI_TRY(launch_check(c, "k_inc_keys"));
    }
    int flag = 0;
    LILI_TRY(read_back(c, {{&flag, e.bad, sizeof(int)}}));
    f.bad = flag != 0;
    return LILIOM_OK;
}

// the representability of the absolute keys, PCL's "leaf size too small" test on the union box of the live frames, and that
// box's index not wrapping (absolute-key order is PCL's index order only then)
static bool inc_representable(liliom_ctx* c) {
    for (auto& f : c->frames)
        if (f.bad) return false;
    int box[kBoxInts];
    frames_box(c, box);
    const VgParams p = vg_params(box, c->prm.leaf_map);
    return !p.overflow && !p.wraps;
}

// entry array from scratch (first call, or after liliom_map_push_frame / liliom_map_clear touched the FIFO)
static int inc_build_all(liliom_ctx* c) {
    size_t total = 0;
    for (auto& f : c->frames) total += (size_t)f.n;
    const size_t cap = total > 0 ? total : 1;
    for (int b = 0; b < 2; ++b) {
        LILI_CUDA(c, c->inc_key[b].ensure(cap * sizeof(u64) + 64));
        LILI_CUDA(c, c->inc_ref[b].ensure(cap * sizeof(unsigned) + 64));
    }
    size_t off = 0;
    long long nfin = 0;
    for (auto& f : c->frames) {
        LILI_TRY(inc_frame_keys(c, f, c->inc_key[1].as<u64>() + off, c->inc_ref[1].as<unsigned>() + off));
        off += (size_t)f.n; nfin += f.mm[6];
    }
    if (total > 0)      // stable: equal keys stay in concatenation order (frames oldest first, points in frame order); ~0 keys last
        LILI_TRY(sort_pairs_u64(c, c->inc_key[1].as<u64>(), c->inc_key[0].as<u64>(), c->inc_ref[1].as<int>(), c->inc_ref[0].as<int>(), (int)total, 64));
    c->inc_cur = 0;
    c->inc_E = (int)nfin;
    return LILIOM_OK;
}

// Emit, part 1: heads -> ranks -> centroids of the current entry array go into c->map_ds.  e.E2 = 0: nothing to launch.
static int inc_emit_begin(liliom_ctx* c, MapEntry& e, FrameTab& ft) {
    const int stride = c->prm.point_stride;
    const int E = c->inc_E;
    e.E2 = 0;
    LILI_CUDA(c, c->map_ds.ensure((size_t)(E > 0 ? E : 1) * stride));
    LILI_CUDA(c, c->vg_count.ensure(16));
    if (E == 0) return LILIOM_OK;
    LILI_CUDA(c, c->inc_flags.ensure(((size_t)E + 2) * 4));
    LILI_CUDA(c, c->inc_rank.ensure(((size_t)E + 2) * 4));
    e.ekeys = c->inc_key[c->inc_cur].as<u64>(); e.erefs = c->inc_ref[c->inc_cur].as<unsigned>(); e.E2 = E; e.stride = stride;
    e.flags = c->inc_flags.as<int>(); e.rank = c->inc_rank.as<int>(); e.ds = (unsigned char*)c->map_ds.p; e.count = c->vg_count.as<int>();
    ft = FrameTab{};
    for (auto& f : c->frames) ft.base[f.slot] = (const unsigned char*)f.buf.p;
    return LILIOM_OK;
}

// heads -> ranks -> centroids of the current entry array into c->map_ds; m = number of voxels
static int inc_emit(liliom_ctx* c, int* m_out) {
    MapEntry e{};
    FrameTab tab;
    *m_out = 0;
    LILI_TRY(inc_emit_begin(c, e, tab));
    const int E = e.E2;
    if (E == 0) return LILIOM_OK;
    k_vg_heads<<<cdiv(E + 1, 256), 256, 0, c->stream>>>(e.ekeys, E, nullptr, e.flags);
    LILI_TRY(launch_check(c, "k_vg_heads"));
    LILI_TRY(exclusive_scan_i32(c, e.flags, e.rank, E));
    if (e.stride == 48)
        k_inc_centroid<48><<<cdiv(E, 128), 128, 0, c->stream>>>(tab, e.ekeys, e.erefs, e.flags, e.rank, E, e.ds, e.count);
    else
        k_inc_centroid<32><<<cdiv(E, 128), 128, 0, c->stream>>>(tab, e.ekeys, e.erefs, e.flags, e.rank, E, e.ds, e.count);
    LILI_TRY(launch_check(c, "k_inc_centroid"));
    return read_back(c, {{m_out, e.count, sizeof(int)}});
}

// New frame (at the back of c->frames), part 1: where its keys and refs go, unsorted
static int inc_new_begin(liliom_ctx* c, MapEntry& e) {
    Frame& fn = c->frames.back();
    const size_t ncap = (size_t)(fn.n > 0 ? fn.n : 1);
    for (int b = 0; b < 2; ++b) {
        LILI_CUDA(c, c->inc_newkey[b].ensure(ncap * sizeof(u64) + 64));
        LILI_CUDA(c, c->inc_newref[b].ensure(ncap * sizeof(unsigned) + 64));
    }
    return inc_keys_begin(c, fn, c->inc_newkey[0].as<u64>(), c->inc_newref[0].as<unsigned>(), e);
}

// Merge, part 1 (the keys are representable): the new frame's entries sorted on their own, the next entry array sized
static int inc_merge_begin(liliom_ctx* c, const Popped& popped, MapEntry& e) {
    Frame& fn = c->frames.back();
    const int E = c->inc_E, nnew = fn.mm[6];
    if (fn.n > 0)
        LILI_TRY(sort_pairs_u64(c, c->inc_newkey[0].as<u64>(), c->inc_newkey[1].as<u64>(), c->inc_newref[0].as<int>(), c->inc_newref[1].as<int>(), fn.n, 64));
    const int E2 = E - popped.nfin + nnew;
    const int cur = c->inc_cur, nxt = cur ^ 1;
    LILI_CUDA(c, c->inc_key[nxt].ensure((size_t)(E2 > 0 ? E2 : 1) * sizeof(u64) + 64));
    LILI_CUDA(c, c->inc_ref[nxt].ensure((size_t)(E2 > 0 ? E2 : 1) * sizeof(unsigned) + 64));
    LILI_CUDA(c, c->inc_removed.ensure(((size_t)E + 2) * 4));
    LILI_CUDA(c, c->inc_rpos.ensure(((size_t)E + 2) * 4));
    e.keys = c->inc_key[cur].as<u64>(); e.refs = c->inc_ref[cur].as<unsigned>(); e.E = E; e.popped = popped.slot;
    e.removed = c->inc_removed.as<int>(); e.rpos = c->inc_rpos.as<int>();
    e.snewkey = c->inc_newkey[1].as<u64>(); e.snewref = c->inc_newref[1].as<unsigned>(); e.nnew = nnew;
    e.keys2 = c->inc_key[nxt].as<u64>(); e.refs2 = c->inc_ref[nxt].as<unsigned>(); e.E2 = E2;
    return LILIOM_OK;
}
// Merge, part 2 (the merge kernels are queued): the merged array is the current one
static void inc_merge_end(liliom_ctx* c, const MapEntry& e) {
    c->inc_cur ^= 1;
    c->inc_E = e.E2;
}

// The frame at the back of c->frames has just been pushed (points in its buffer, slot assigned); `popped` is the frame that
// left the FIFO in the same push.  Brings the entry array up to date and emits the filtered cloud.
static int map_inc_update(liliom_ctx* c, const Popped& popped, int* m_out) {
    Frame& fn = c->frames.back();
    if (!c->inc_valid) {
        LILI_TRY(inc_build_all(c));
        if (!inc_representable(c)) return LILIOM_E_GRID;                              // caller falls back to the sort chain
        c->inc_valid = true;
        return inc_emit(c, m_out);
    }
    MapEntry e{};
    {   // new frame: keys, refs, key flag; sorted on its own below
        LILI_TRY(inc_new_begin(c, e));
        if (fn.n > 0) {
            k_inc_keys<<<cdiv(fn.n, 256), 256, 0, c->stream>>>(e.fbuf, e.n, e.stride, e.inv_leaf, e.slot, e.newkey, e.newref, e.bad);
            LILI_TRY(launch_check(c, "k_inc_keys"));
        }
        int flag = 0;
        LILI_TRY(read_back(c, {{&flag, e.bad, sizeof(int)}}));
        fn.bad = flag != 0;
    }
    if (!inc_representable(c)) { c->inc_valid = false; return LILIOM_E_GRID; }
    LILI_TRY(inc_merge_begin(c, popped, e));
    const int E = e.E, nnew = e.nnew;
    k_inc_mark<<<cdiv(E + 1, 256), 256, 0, c->stream>>>(e.refs, E, e.popped, e.removed);
    LILI_TRY(launch_check(c, "k_inc_mark"));
    LILI_TRY(exclusive_scan_i32(c, e.removed, e.rpos, E));
    if (E > 0) {
        k_inc_merge_old<<<cdiv(E, 256), 256, 0, c->stream>>>(e.keys, e.refs, e.removed, e.rpos, E, e.snewkey, nnew, e.keys2, e.refs2);
        LILI_TRY(launch_check(c, "k_inc_merge_old"));
    }
    if (nnew > 0) {
        k_inc_merge_new<<<cdiv(nnew, 256), 256, 0, c->stream>>>(e.snewkey, e.snewref, nnew, e.keys, e.rpos, E, e.keys2, e.refs2);
        LILI_TRY(launch_check(c, "k_inc_merge_new"));
    }
    inc_merge_end(c, e);
    return inc_emit(c, m_out);
}

}  // namespace lili

using namespace lili;

extern "C" int liliom_map_clear(liliom_ctx* c) {
    if (!c) return LILIOM_E_ARG;
    c->frames.clear();
    c->inc_valid = false;
    map_reset(c);
    return LILIOM_OK;
}

extern "C" int liliom_map_push_frame(liliom_ctx* c, const void* surf_ds_body, int n, const double pose7[7]) {
    if (!c || n < 0 || (n > 0 && !surf_ds_body) || !pose7) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    if (n > 0) {
        LILI_CUDA(c, c->raw.ensure((size_t)n * stride));
        LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, surf_ds_body, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream));
    }
    return push_frame_from_device(c, c->raw.p, n, pose7);
}

extern "C" int liliom_map_push_frame_device(liliom_ctx* c, const void* d_surf_ds_body, int n, const double pose7[7]) {
    if (!c || n < 0 || (n > 0 && !d_surf_ds_body) || !pose7) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    return push_frame_from_device(c, d_surf_ds_body, n, pose7);
}

extern "C" int liliom_map_rebuild(liliom_ctx* c, int* n_map_out) {
    if (!c) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    // LILIOM_DEBUG_TIMING: wall clock of the phases (each closed by a stream sync), printed by rank 0
    double tph[8] = {0};
    int nph = 0;
    auto mark = [&]() {
        if (c->dbg_timing && nph < 8) { cudaStreamSynchronize(c->stream); timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); tph[nph++] = ts.tv_sec * 1e6 + ts.tv_nsec * 1e-3; }
    };
    mark();
    size_t total = 0;
    for (auto& f : c->frames) total += (size_t)f.n;
    map_reset(c);
    if (n_map_out) *n_map_out = 0;
    if (total == 0 && c->nranks == 1) { c->map.ready = true; return LILIOM_OK; }
    LILI_CUDA(c, c->map_raw.ensure((total > 0 ? total : 1) * stride));
    LILI_CUDA(c, c->map_ds.ensure((total > 0 ? total : 1) * stride));
    LILI_CUDA(c, c->vg_count.ensure(16));
    // bounding box and finite count of the concatenation = union over the frames (each measured once, at its push)
    int box[kBoxInts];
    frames_box(c, box);
    // single GPU: the centroid kernel writes the float4 map itself (no repack pass); at most `total` voxels
    if (c->nranks == 1) LILI_CUDA(c, c->map.xyzw.ensure((total > 0 ? total : 1) * sizeof(float4)));
    size_t off = 0;                                                                 // :301-302 concatenation, oldest first
    for (size_t g = 0; g < c->frames.size(); g += kConcatMax) {
        const int nf = (int)std::min(c->frames.size() - g, (size_t)kConcatMax);
        ConcatTab tab{};
        size_t largest = 0;
        for (int k = 0; k < nf; ++k) {
            const Frame& f = c->frames[g + k];
            tab.src[k] = (const float4*)f.buf.p; tab.off[k] = (long long)(off * (stride / 16));
            off += (size_t)f.n; largest = f.n > (int)largest ? (size_t)f.n : largest;
        }
        for (int k = nf; k <= kConcatMax; ++k) tab.off[k] = (long long)(off * (stride / 16));
        if (largest == 0) continue;
        const int bx = max(1, min(cdiv((long long)largest * (stride / 16), 256 * 4), c->sm_count * 4));
        k_concat_frames<<<dim3(bx, (unsigned)nf), 256, 0, c->stream>>>(tab, (float4*)c->map_raw.p);
        LILI_TRY(launch_check(c, "k_concat_frames"));
    }
    mark();      // [1] concatenation
    int m = 0;
    if (total > 0) {
        // (The single-launch cooperative filter of the scan VoxelGrid was tried here for maps of <= 32k points: within the noise
        // of the real-size streamed lifecycle — not kept.)
        LILI_TRY(voxelgrid_dev(c, c->map_raw.p, (int)total, nullptr, stride, c->prm.leaf_map, c->map_ds.p, c->vg_count.as<int>(),   // :316-317
                               c->nranks == 1 ? c->map.xyzw.as<float4>() : nullptr, 32, box));
        LILI_TRY(read_back(c, {{&m, c->vg_count.p, sizeof(int)}}));
    }
    mark();      // [2] VoxelGrid
    LILI_CUDA(c, c->map.xyzw.ensure((size_t)(m > 0 ? m : 1) * sizeof(float4)));
    c->map_n_global = m;
    c->map_ds_n = m;
    if (c->nranks > 1) {
        // Every rank ENTERS the all-reduce whatever happened locally (a rank that returned early would leave its peers waiting
        // in the collective): the local status travels as a second scalar and all ranks fail together.
        // Shard filter: drops the (possibly incomplete) voxels beyond the 1-cell halo, fused with the repack to float4.
        // owned: the voxels whose centroid this rank owns.  The rank holds each of them complete, and every voxel has one owner.
        int owned = 0;
        auto shard_and_index = [&]() -> int {
            int local = 0;
            if (m > 0) LILI_TRY(shard_filter(c, c->map_ds.p, m, stride, gate_cell(c->prm.knn_max_sqdist), c->map.xyzw.p, true, &local));
            LILI_TRY(grid_build(c, local, box[6] > 0 ? box : nullptr));
            int* d_owned = c->vg_count.as<int>() + 1;
            LILI_CUDA(c, cudaMemsetAsync(d_owned, 0, sizeof(int), c->stream));
            if (local > 0) {
                k_count_owned<<<cdiv(local, 256), 256, 0, c->stream>>>(c->map.xyzw.as<float4>(), local, c->shard_inv_block, c->nranks, c->rank, d_owned);
                LILI_TRY(launch_check(c, "k_count_owned"));
            }
            return read_back(c, {{&owned, d_owned, sizeof(int)}});
        };
        const int rc_local = shard_and_index();
        mark();  // [3] shard filter + cell grid
        // the "< 10 map points" guard (L/src/LidarOdometry.cpp:485-488) is about the whole map: sum the owned-voxel counts
        LILI_CUDA(c, c->neq.ensure(32 * sizeof(double)));
        double* pin = c->h_pin->map_status;
        pin[0] = rc_local == LILIOM_OK ? (double)owned : 0.0;
        pin[1] = rc_local == LILIOM_OK ? 0.0 : 1.0;
        LILI_CUDA(c, cudaMemcpyAsync(c->neq.p, pin, 2 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
        LILI_TRY(nccl_allreduce_sum_f64(c, c->neq.as<double>(), 2));
        LILI_CUDA(c, cudaMemcpyAsync(pin + 2, c->neq.p, 2 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        LILI_CUDA(c, cudaStreamSynchronize(c->stream));
        if (rc_local != LILIOM_OK) return rc_local;
        if (pin[3] != 0.0) { c->map.ready = false; c->last_error = "liliom_map_rebuild failed on another rank"; return LILIOM_E_NCCL; }
        c->map_n_global = (int)pin[2];                  // each voxel counted on its owner only: the size one GPU's map has
    } else {
        LILI_TRY(grid_build(c, m, box[6] > 0 ? box : nullptr));     // map_xyzw was written by the VoxelGrid's centroid kernel
    }
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    mark();      // [3 or 4] cell grid (single GPU) / map-size all-reduce (sharded)
    if (c->dbg_timing && c->rank == 0 && nph >= 4) {
        fprintf(stderr, "[liliom_map_rebuild, us] %zu raw points, %d voxels: concat %.0f, VoxelGrid %.0f, %s %.0f", total, m, tph[1] - tph[0], tph[2] - tph[1],
                c->nranks > 1 ? "shard filter + grid" : "grid", tph[3] - tph[2]);
        if (nph >= 5) fprintf(stderr, ", all-reduce %.0f", tph[4] - tph[3]);
        fprintf(stderr, "\n");
    }
    if (n_map_out) *n_map_out = m;
    return LILIOM_OK;
}

// Whether an update of n points takes the incremental path (otherwise: push + the sort chain)
static bool map_incremental(const liliom_ctx* c, int n) { return c->nranks == 1 && c->prm.max_map_frames <= kIncSlots && n < (1 << 24); }

// The incremental update behind its push (`popped` left the FIFO in it); falls back to the sort chain where the entry array cannot
// describe the FIFO
static int map_update_tail(liliom_ctx* c, const Popped& popped, int* n_map_out) {
    map_reset(c);
    int m = 0;
    const int rc = map_inc_update(c, popped, &m);
    if (rc == LILIOM_OK) {
        LILI_TRY(map_finish_from_ds(c, m));
        if (n_map_out) *n_map_out = m;
        return LILIOM_OK;
    }
    c->inc_valid = false;
    if (rc != LILIOM_E_GRID) return rc;       // E_GRID: keys not representable / PCL's overflow case -> the sort chain decides
    return liliom_map_rebuild(c, n_map_out);
}

// SURVEY §8 (f2): push + incremental refresh; same result as liliom_map_push_frame + liliom_map_rebuild
static int map_update_from_device(liliom_ctx* c, const void* d_src, int n, const double pose7[7], int* n_map_out) {
    if (n_map_out) *n_map_out = 0;
    const bool incremental = map_incremental(c, n);
    Popped popped;
    LILI_TRY(push_frame_from_device(c, d_src, n, pose7, incremental, &popped));
    if (incremental) return map_update_tail(c, popped, n_map_out);
    return liliom_map_rebuild(c, n_map_out);
}

extern "C" int liliom_map_update(liliom_ctx* c, const void* surf_ds_body, int n, const double pose7[7], int* n_map_out) {
    if (!c || n < 0 || (n > 0 && !surf_ds_body) || !pose7) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    if (n > 0) {
        LILI_CUDA(c, c->raw.ensure((size_t)n * stride));
        LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, surf_ds_body, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream));
    }
    return map_update_from_device(c, c->raw.p, n, pose7, n_map_out);
}

extern "C" int liliom_map_update_device(liliom_ctx* c, const void* d_surf_ds_body, int n, const double pose7[7], int* n_map_out) {
    if (!c || n < 0 || (n > 0 && !d_surf_ds_body) || !pose7) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    return map_update_from_device(c, d_surf_ds_body, n, pose7, n_map_out);
}

// The frame of liliom_map_update_resident: surf_last_ds of the context's last odometry call, still in vg_out
static bool resident_frame_ok(liliom_ctx* c) {
    if (c->n_ds_resident >= 0) return true;
    c->last_error = "liliom_map_update_resident: no down-sampled scan is resident (an odometry call leaves one; liliom_voxelgrid, "
                    "liliom_kf_add, liliom_kf_cloud, liliom_loop_align and liliom_global_map overwrite it)";
    return false;
}

// The update reads vg_out and never writes it (its VoxelGrid output is map_ds), so the frame stays resident across the call.
extern "C" int liliom_map_update_resident(liliom_ctx* c, const double pose7[7], int* n_map_out) {
    if (!c || !pose7) return LILIOM_E_ARG;
    if (!resident_frame_ok(c)) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    return map_update_from_device(c, c->vg_out.p, c->n_ds_resident, pose7, n_map_out);
}

namespace lili {
namespace {

// One stage for the sessions `which` (indices into J); each session's launch count advances as its solo call's does.
template <class St>
int map_stage(liliom_ctx* c0, std::vector<MapJob>& J, const std::vector<int>& which) {
    return stage_batch<St>(c0, which, [&](MapEntry& e, int i) { e = J[i].e; return J[i].c; });
}
template <int STRIDE>
int map_centroid_stage(liliom_ctx* c0, std::vector<MapJob>& J, const std::vector<int>& which) {
    return stage_batch<MapStCentroid<STRIDE>>(c0, which, [&](MapCentroidEntry& t, int i) {
        const MapJob& j = J[i];
        const MapEntry& e = j.e;
        t = MapCentroidEntry{j.ft, e.ekeys, e.erefs, e.E2, e.stride, e.flags, e.rank, e.ds, e.count};
        return j.c;
    });
}

// Where a session of the batch stands: on the shared path, finished (its status set), or off the shared path, to be finished
// by the solo code it would have run: the whole update, the update behind the push, or the sort chain.
enum MapWhere { kMapLive, kMapDone, kMapSoloAll, kMapSoloTail, kMapSoloRebuild };

// The shared phases of map_update_batch, every session's stream pointing at c0's.  Each phase: the solo call's host part per
// session, the stage launches for all of them, every session's read-back words into its own pinned block, ONE synchronise.
int map_batch_run(liliom_ctx* c0, std::vector<MapJob>& J, std::vector<MapWhere>& where, const double* poses7, int* nm, int* status) {
    const int B = (int)J.size();
    auto fail = [&](int i, int rc, bool inc) {
        status[i] = rc; where[i] = kMapDone;
        if (inc) J[i].c->inc_valid = false;
    };
    auto live = [&](auto pred) {
        std::vector<int> v;
        for (int i = 0; i < B; ++i) if (where[i] == kMapLive && pred(J[i])) v.push_back(i);
        return v;
    };
    auto any = [](const MapJob&) { return true; };
    // `bytes` at src(job) of every session in `which` into its pinned scratch, then the phase's one wait
    auto wait_words = [&](const std::vector<int>& which, auto src, size_t bytes) -> int {
        for (int i : which)
            if (cudaError_t err = cudaMemcpyAsync(J[i].c->h_pin->scratch, src(J[i]), bytes, cudaMemcpyDeviceToHost, c0->stream); err != cudaSuccess)
                fail(i, fail_cuda(J[i].c, err, "map update batch: read-back"), true);
        LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
        return LILIOM_OK;
    };
    auto word = [&](int i) { int w; memcpy(&w, J[i].c->h_pin->scratch, sizeof(int)); return w; };

    // 1. transform + box of the new frame -> every session's Frame::mm
    for (int i : live(any)) {
        liliom_ctx* c = J[i].c;
        const int n = c->n_ds_resident;
        if (!map_incremental(c, n)) { where[i] = kMapSoloAll; continue; }
        if (const int rc = push_begin(c, c->vg_out.p, n, poses7 + 7 * i, true, J[i]); rc != LILIOM_OK) fail(i, rc, false);
    }
    {
        const std::vector<int> w = live([](const MapJob& j) { return j.e.n > 0; });
        LILI_TRY(map_stage<MapStTransform>(c0, J, w));
        LILI_TRY(map_stage<MapStBoxInit>(c0, J, w));
        LILI_TRY(map_stage<MapStBox>(c0, J, w));
        LILI_TRY(wait_words(w, [](const MapJob& j) { return j.e.mm; }, kBoxInts * sizeof(int)));
    }
    for (int i : live(any)) {
        push_end(J[i], J[i].e.n > 0 ? reinterpret_cast<const int*>(J[i].c->h_pin->scratch) : nullptr);
        map_reset(J[i].c);
    }
    // 2. keys of the new frame + key flag -> inc_representable per session
    for (int i : live(any)) {
        liliom_ctx* c = J[i].c;
        if (!c->inc_valid) { where[i] = kMapSoloTail; continue; }       // first update, or the FIFO was touched: inc_build_all
        if (const int rc = inc_new_begin(c, J[i].e); rc != LILIOM_OK) fail(i, rc, true);
    }
    LILI_TRY(map_stage<MapStKeys>(c0, J, live([](const MapJob& j) { return j.e.n > 0; })));
    LILI_TRY(wait_words(live(any), [](const MapJob& j) { return j.e.bad; }, sizeof(int)));
    for (int i : live(any)) J[i].c->frames.back().bad = word(i) != 0;
    // 3. merge into the entry array, heads, centroids -> every session's voxel count
    for (int i : live(any)) {
        liliom_ctx* c = J[i].c;
        if (!inc_representable(c)) { c->inc_valid = false; where[i] = kMapSoloRebuild; continue; }
        if (const int rc = inc_merge_begin(c, J[i].popped, J[i].e); rc != LILIOM_OK) fail(i, rc, true);
    }
    LILI_TRY(map_stage<MapStMark>(c0, J, live(any)));
    for (int i : live(any))
        if (const int rc = exclusive_scan_i32(J[i].c, J[i].e.removed, J[i].e.rpos, J[i].e.E); rc != LILIOM_OK) fail(i, rc, true);
    LILI_TRY(map_stage<MapStMergeOld>(c0, J, live([](const MapJob& j) { return j.e.E > 0; })));
    LILI_TRY(map_stage<MapStMergeNew>(c0, J, live([](const MapJob& j) { return j.e.nnew > 0; })));
    for (int i : live(any)) {
        inc_merge_end(J[i].c, J[i].e);
        if (const int rc = inc_emit_begin(J[i].c, J[i].e, J[i].ft); rc != LILIOM_OK) fail(i, rc, true);
    }
    {
        const std::vector<int> w = live([](const MapJob& j) { return j.e.E2 > 0; });
        LILI_TRY(map_stage<MapStHeads>(c0, J, w));
        for (int i : w)
            if (const int rc = exclusive_scan_i32(J[i].c, J[i].e.flags, J[i].e.rank, J[i].e.E2); rc != LILIOM_OK) fail(i, rc, true);
        LILI_TRY(map_centroid_stage<48>(c0, J, live([](const MapJob& j) { return j.e.E2 > 0 && j.e.stride == 48; })));
        LILI_TRY(map_centroid_stage<32>(c0, J, live([](const MapJob& j) { return j.e.E2 > 0 && j.e.stride != 48; })));
        const std::vector<int> counted = live([](const MapJob& j) { return j.e.E2 > 0; });
        LILI_TRY(wait_words(counted, [](const MapJob& j) { return j.e.count; }, sizeof(int)));
        for (int i : counted) if (where[i] == kMapLive) J[i].m = word(i);
    }
    // 4. repack, cell grid -> escape flags
    for (int i : live(any))
        if (const int rc = finish_begin(J[i].c, J[i].m, J[i].e); rc != LILIOM_OK) fail(i, rc, false);
    LILI_TRY(map_stage<MapStRepack>(c0, J, live([](const MapJob& j) { return j.m > 0; })));
    for (int i : live(any)) {
        MapJob& j = J[i];
        liliom_ctx* c = j.c;
        int mm[kBoxInts];
        frames_box(c, mm);
        if (const int rc = grid_begin(c, c->map, gate_cell(c->prm.knn_max_sqdist), j.m, mm[6] > 0 ? mm : nullptr, j.g); rc != LILIOM_OK) {
            fail(i, rc, false);
            continue;
        }
        if (j.g.done) { nm[i] = j.m; where[i] = kMapDone; continue; }        // an empty map: nothing to index
        MapEntry& e = j.e;
        e.g = c->map.grid; e.gkeys = c->grid_keys.as<uint32_t>(); e.gvals = c->grid_vals.as<int>(); e.escaped = j.g.escaped;
        e.gkeys2 = c->grid_keys2.as<uint32_t>(); e.gvals2 = c->grid_vals2.as<int>(); e.sorted = c->map.sorted.as<float4>();
        e.cell_start = c->map.cell_start.as<int>();
    }
    LILI_TRY(map_stage<MapStCellKeys>(c0, J, live(any)));
    for (int i : live(any)) if (const int rc = grid_sort(J[i].g); rc != LILIOM_OK) fail(i, rc, false);
    LILI_TRY(map_stage<MapStGather>(c0, J, live(any)));
    for (int i : live(any)) if (const int rc = grid_clear(J[i].g); rc != LILIOM_OK) fail(i, rc, false);
    LILI_TRY(map_stage<MapStRunEnds>(c0, J, live(any)));
    for (int i : live(any)) if (const int rc = grid_scan(J[i].g); rc != LILIOM_OK) fail(i, rc, false);
    LILI_TRY(wait_words(live([](const MapJob& j) { return j.g.escaped != nullptr; }), [](const MapJob& j) { return j.g.escaped; }, sizeof(int)));
    bool rebuilt = false;
    for (int i : live(any)) {
        const int esc = J[i].g.escaped ? word(i) : 0;
        status[i] = grid_finish(J[i].g, esc);      // an escaped box: the exact re-build, as in the solo call
        rebuilt = rebuilt || esc != 0;
        if (status[i] == LILIOM_OK) nm[i] = J[i].m;
        where[i] = kMapDone;
    }
    // the re-build's kernels are still queued: the call returns with every index complete, as the solo call does
    if (rebuilt) LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
    // 5. sessions that left the shared path finish on their solo path
    for (int i = 0; i < B; ++i) {
        liliom_ctx* c = J[i].c;
        if (where[i] == kMapSoloAll) status[i] = map_update_from_device(c, c->vg_out.p, c->n_ds_resident, poses7 + 7 * i, &nm[i]);
        else if (where[i] == kMapSoloTail) status[i] = map_update_tail(c, J[i].popped, &nm[i]);
        else if (where[i] == kMapSoloRebuild) status[i] = liliom_map_rebuild(c, &nm[i]);
    }
    return LILIOM_OK;
}

}  // namespace

// liliom_map_update_resident of several sessions.  Shared launches and waits on cs[0]'s stream (the other sessions' streams
// joined before and after with events); every buffer, library sort and scan, FIFO and host decision stays the session's own,
// made by the solo call's code from the session's own read-back words.
int map_update_batch(liliom_ctx* const* cs, int B, const double* poses7, int* n_map, int* status) {
    liliom_ctx* c0 = cs[0];
    std::vector<MapJob> J(B);
    std::vector<MapWhere> where(B, kMapLive);
    std::vector<int> nm(B, 0);
    const std::vector<liliom_ctx*> all(cs, cs + B);
    for (int i = 0; i < B; ++i) {
        J[i].c = cs[i];
        status[i] = LILIOM_OK;
        if (!resident_frame_ok(cs[i])) { status[i] = LILIOM_E_ARG; where[i] = kMapDone; }
    }
    LILI_TRY(batch_join_in(c0, all));
    int rc;
    {
        const BatchStreams on_c0(all, c0->stream);
        rc = map_batch_run(c0, J, where, poses7, nm.data(), status);
    }
    LILI_TRY(batch_join_out(c0, all));
    for (int i = 0; n_map && i < B; ++i) n_map[i] = nm[i];
    return rc;
}

}  // namespace lili

extern "C" int liliom_map_update_batch(liliom_ctx* const* ctxs, int B, const double* poses7, int* n_map, int* status) {
    if (!batch_ctxs_ok(ctxs, B) || !poses7 || !status) return LILIOM_E_ARG;
    LILI_CUDA(ctxs[0], cudaSetDevice(ctxs[0]->device));
    return map_update_batch(ctxs, B, poses7, n_map, status);
}

// surf_from_map_ds as a point cloud (all fields), in liliom_map_download order
extern "C" int liliom_map_download_cloud(liliom_ctx* c, void* out, int cap, int* m_out) {
    if (!c || !m_out) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    if (c->nranks > 1) { c->last_error = "liliom_map_download_cloud is single-GPU"; return LILIOM_E_ARG; }
    if (c->map_ds_n < 0) {
        *m_out = 0;
        c->last_error = "liliom_map_download_cloud: the map was installed, not filtered from frames (rebuild or update it first)";
        return LILIOM_E_NOMAP;
    }
    return download_sized(c, c->map_ds, c->map_ds_n, c->prm.point_stride, out, cap, m_out);
}

extern "C" int liliom_map_set_points(liliom_ctx* c, const liliom_f4* xyzw, int m) {
    if (!c || m < 0 || (m > 0 && !xyzw)) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_TRY(map_install_host(c, xyzw, m, 16, false));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

// Install a PCL-layout cloud as the map, keeping its reflectivity channel for the Horizon backend variant.
extern "C" int liliom_map_set_cloud(liliom_ctx* c, const void* pts, int m, int stride) {
    if (!c || m < 0 || (m > 0 && !pts) || (stride != 48 && stride != 32)) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    if (c->nranks > 1) { c->last_error = "liliom_map_set_cloud is single-GPU"; return LILIOM_E_ARG; }
    LILI_TRY(map_install_host(c, pts, m, stride, true));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

extern "C" int liliom_map_size(const liliom_ctx* c) { return c ? c->map.n : 0; }

extern "C" int liliom_map_download(liliom_ctx* c, liliom_f4* out, int cap, int* m_out) {
    if (!c || !m_out) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    return download_sized(c, c->map.xyzw, c->map.n, sizeof(float4), out, cap, m_out);
}
