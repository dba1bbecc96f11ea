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
#include <climits>

namespace lili {

typedef unsigned long long u64;
constexpr int kIncSlots = 64;                 // frame slots (refs carry the slot in their top 6 bits... 8 bits reserved)
constexpr unsigned kIncIdxMask = (1u << 24) - 1u;
struct FrameTab { const unsigned char* base[kIncSlots]; };

// keys of one frame's points (world frame, already transformed), refs = slot << 24 | index; *bad |= 1 when a voxel coordinate
// does not fit 21 bits (the frame's box and finite count were measured at its push: Frame::mm)
__global__ void k_inc_keys(const unsigned char* __restrict__ pts, int n, int stride, float inv_leaf, unsigned slot, u64* __restrict__ keys,
                           unsigned* __restrict__ refs, int* __restrict__ bad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
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
__global__ void k_inc_mark(const unsigned* __restrict__ refs, int E, int popped, int* __restrict__ removed) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > E) return;
    removed[i] = (i < E && popped >= 0 && (int)(refs[i] >> 24) == popped) ? 1 : 0;
}
// surviving old entries: down by the removed entries before them, up by the new entries with a smaller key.  The entries of a
// warp are consecutive in a sorted array, so their lower bounds in the new keys are nested between those of lanes 0 and 31:
// two full binary searches per warp, then every lane searches only the (short) range between them.
__global__ void k_inc_merge_old(const u64* __restrict__ keys, const unsigned* __restrict__ refs, const int* __restrict__ removed,
                                const int* __restrict__ rpos, int E, const u64* __restrict__ newkeys, int nnew, u64* __restrict__ keys2,
                                unsigned* __restrict__ refs2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
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
// new entries (sorted by key, then index): behind every surviving old entry with key <= their own
__global__ void k_inc_merge_new(const u64* __restrict__ newkeys, const unsigned* __restrict__ newrefs, int nnew, const u64* __restrict__ keys,
                                const int* __restrict__ rpos, int E, u64* __restrict__ keys2, unsigned* __restrict__ refs2) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nnew) return;
    const u64 k = newkeys[j];
    const int ub = upper_bound_u64(keys, E, k);
    const int pos = j + (ub - rpos[ub]);
    keys2[pos] = k; refs2[pos] = newrefs[j];
}
// centroid of every voxel, members in entry order (vg_box.h), the points fetched through the frame table
template <int STRIDE>
__global__ void k_inc_centroid(const __grid_constant__ FrameTab tab, const u64* __restrict__ keys, const unsigned* __restrict__ refs,
                               const int* __restrict__ flags, const int* __restrict__ rank, int E, unsigned char* __restrict__ out,
                               int* __restrict__ count_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) *count_out = rank[E];
    if (i >= E || !flags[i]) return;
    const VgAcc<STRIDE> a = vg_walk<STRIDE>(keys, i, E, [&](int j) { return (int)refs[j]; },       // (slot < 64: a ref is below 2^30)
                                            [&](int r) { return tab.base[r >> 24] + (size_t)(r & kIncIdxMask) * STRIDE; });
    vg_write<STRIDE>(a.s, a.n, out + (size_t)rank[i] * STRIDE);
}

// keys + refs of frame `f` (points already in f.buf), written at keys/refs, and its key flag; one sync
static int inc_frame_keys(liliom_ctx* c, Frame& f, u64* keys, unsigned* refs) {
    const int stride = c->prm.point_stride;
    LILI_CUDA(c, c->inc_bad.ensure(sizeof(int)));
    int* bad = c->inc_bad.as<int>();
    LILI_CUDA(c, cudaMemsetAsync(bad, 0, sizeof(int), c->stream));
    if (f.n > 0) {
        k_inc_keys<<<cdiv(f.n, 256), 256, 0, c->stream>>>((const unsigned char*)f.buf.p, f.n, stride, 1.0f / c->prm.leaf_map, (unsigned)f.slot, keys, refs, bad);
        LILI_TRY(launch_check(c, "k_inc_keys"));
    }
    int flag = 0;
    LILI_TRY(read_back(c, {{&flag, bad, sizeof(int)}}));
    f.bad = flag != 0;
    return LILIOM_OK;
}

// the representability of the absolute keys, and PCL's "leaf size too small" test on the union box of the live frames
static bool inc_representable(liliom_ctx* c) {
    for (auto& f : c->frames)
        if (f.bad) return false;
    int box[kBoxInts];
    frames_box(c, box);
    return !vg_params(box, c->prm.leaf_map).overflow;
}

int map_finish_from_ds(liliom_ctx* c, int m);      // api.cu: repack + cell grid of the filtered cloud in c->map_ds

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

// heads -> ranks -> centroids of the current entry array into c->map_ds; m = number of voxels
static int inc_emit(liliom_ctx* c, int* m_out) {
    const int stride = c->prm.point_stride;
    const int E = c->inc_E;
    *m_out = 0;
    LILI_CUDA(c, c->map_ds.ensure((size_t)(E > 0 ? E : 1) * stride));
    LILI_CUDA(c, c->vg_count.ensure(16));
    if (E == 0) return LILIOM_OK;
    LILI_CUDA(c, c->inc_flags.ensure(((size_t)E + 2) * 4));
    LILI_CUDA(c, c->inc_rank.ensure(((size_t)E + 2) * 4));
    const u64* keys = c->inc_key[c->inc_cur].as<u64>();
    const unsigned* refs = c->inc_ref[c->inc_cur].as<unsigned>();
    k_vg_heads<<<cdiv(E + 1, 256), 256, 0, c->stream>>>(keys, E, nullptr, c->inc_flags.as<int>());
    LILI_TRY(launch_check(c, "k_vg_heads"));
    LILI_TRY(exclusive_scan_i32(c, c->inc_flags.as<int>(), c->inc_rank.as<int>(), E));
    FrameTab tab{};
    for (auto& f : c->frames) tab.base[f.slot] = (const unsigned char*)f.buf.p;
    if (stride == 48)
        k_inc_centroid<48><<<cdiv(E, 128), 128, 0, c->stream>>>(tab, keys, refs, c->inc_flags.as<int>(), c->inc_rank.as<int>(), E, (unsigned char*)c->map_ds.p, c->vg_count.as<int>());
    else
        k_inc_centroid<32><<<cdiv(E, 128), 128, 0, c->stream>>>(tab, keys, refs, c->inc_flags.as<int>(), c->inc_rank.as<int>(), E, (unsigned char*)c->map_ds.p, c->vg_count.as<int>());
    LILI_TRY(launch_check(c, "k_inc_centroid"));
    return read_back(c, {{m_out, c->vg_count.p, sizeof(int)}});
}

// The frame at the back of c->frames has just been pushed (points in its buffer, slot assigned); `popped` is the slot of the
// frame that left the FIFO in the same call (-1: none).  Brings the entry array up to date and emits the filtered cloud.
int map_inc_update(liliom_ctx* c, int popped_slot, int popped_nfin, int* m_out) {
    Frame& fn = c->frames.back();
    if (!c->inc_valid) {
        LILI_TRY(inc_build_all(c));
        if (!inc_representable(c)) return LILIOM_E_GRID;                              // caller falls back to the sort chain
        c->inc_valid = true;
        return inc_emit(c, m_out);
    }
    {   // new frame: keys, refs, key flag; sorted on its own below
        const size_t ncap = (size_t)(fn.n > 0 ? fn.n : 1);
        for (int b = 0; b < 2; ++b) {
            LILI_CUDA(c, c->inc_newkey[b].ensure(ncap * sizeof(u64) + 64));
            LILI_CUDA(c, c->inc_newref[b].ensure(ncap * sizeof(unsigned) + 64));
        }
        LILI_TRY(inc_frame_keys(c, fn, c->inc_newkey[0].as<u64>(), c->inc_newref[0].as<unsigned>()));
    }
    if (!inc_representable(c)) { c->inc_valid = false; return LILIOM_E_GRID; }
    const int E = c->inc_E, nnew = fn.mm[6];
    if (fn.n > 0)
        LILI_TRY(sort_pairs_u64(c, c->inc_newkey[0].as<u64>(), c->inc_newkey[1].as<u64>(), c->inc_newref[0].as<int>(), c->inc_newref[1].as<int>(), fn.n, 64));
    const int E2 = E - (popped_slot >= 0 ? popped_nfin : 0) + nnew;
    const int cur = c->inc_cur, nxt = cur ^ 1;
    LILI_CUDA(c, c->inc_key[nxt].ensure((size_t)(E2 > 0 ? E2 : 1) * sizeof(u64) + 64));
    LILI_CUDA(c, c->inc_ref[nxt].ensure((size_t)(E2 > 0 ? E2 : 1) * sizeof(unsigned) + 64));
    LILI_CUDA(c, c->inc_removed.ensure(((size_t)E + 2) * 4));
    LILI_CUDA(c, c->inc_rpos.ensure(((size_t)E + 2) * 4));
    k_inc_mark<<<cdiv(E + 1, 256), 256, 0, c->stream>>>(c->inc_ref[cur].as<unsigned>(), E, popped_slot, c->inc_removed.as<int>());
    LILI_TRY(launch_check(c, "k_inc_mark"));
    LILI_TRY(exclusive_scan_i32(c, c->inc_removed.as<int>(), c->inc_rpos.as<int>(), E));
    if (E > 0) {
        k_inc_merge_old<<<cdiv(E, 256), 256, 0, c->stream>>>(c->inc_key[cur].as<u64>(), c->inc_ref[cur].as<unsigned>(), c->inc_removed.as<int>(), c->inc_rpos.as<int>(), E,
                                                            c->inc_newkey[1].as<u64>(), nnew, c->inc_key[nxt].as<u64>(), c->inc_ref[nxt].as<unsigned>());
        LILI_TRY(launch_check(c, "k_inc_merge_old"));
    }
    if (nnew > 0) {
        k_inc_merge_new<<<cdiv(nnew, 256), 256, 0, c->stream>>>(c->inc_newkey[1].as<u64>(), c->inc_newref[1].as<unsigned>(), nnew, c->inc_key[cur].as<u64>(),
                                                               c->inc_rpos.as<int>(), E, c->inc_key[nxt].as<u64>(), c->inc_ref[nxt].as<unsigned>());
        LILI_TRY(launch_check(c, "k_inc_merge_new"));
    }
    c->inc_cur = nxt;
    c->inc_E = E2;
    return inc_emit(c, m_out);
}

}  // namespace lili
