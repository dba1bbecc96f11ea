// SURVEY.md §8 (f5): the backend's keyframe clouds and local map on the device.
//   keyframe store   BackendFusion::downSampleCloud, scan half (L/src/BackendFusion.cpp:1502-1514) + the clouds of
//                    saveKeyFramesAndFactors (:1688-1695): VoxelGrid of the received body-frame clouds, appended to one arena
//   local map        buildLocalMapWithLandMark (:1387-1484) + downSampleCloud, map half (:1486-1492): transform + concatenate
//                    the listed keyframes in ONE launch, VoxelGrid per layer, a cell grid per layer (MapIndex)
//   loop closure     detectLoopClosure's clouds (:2473-2547): edge then surf per keyframe, transformed, VoxelGrid; with
//                    performLoopClosure's ICP (:2552-2582) on them in the same call (liliom_loop_align); several sessions' in one call
//                    (liliom_loop_align_batch)
//   full clouds      downSampleCloud, full-cloud half (:1494-1500; R:1373-1376): the /full_point_cloud of a keyframe, stored
//   global map       publishCompleteMap (:2644-2685) and save_pcd's map (:2703-2718): listed keyframes transformed, concatenated,
//                    VoxelGrid, in a VoxelGrid that reads the store through the keyframe table (kf_table.h): no concatenation
// The deque policy of the local map (:1407-1477) stays with the caller: every call lists the keyframes and the poses to use.
// Compiled with --fmad=false (the VoxelGrid centroids and the transform are bit-exact with the reference's arithmetic).
#include "ctx.cuh"
#include "dev_math.cuh"
#include "kf_table.h"
#include <algorithm>
#include <tuple>
#include <type_traits>

namespace lili {

// The table kernels: blockIdx.y walks the rows (grid-strided past 65535 rows), the blocks of a row stream through its points.
// The table lives in device memory, so one launch serves any number of keyframes (the odometry map's ConcatTab holds 64).
static dim3 kf_row_grid(size_t rows, long long largest, int bx_max, int by_max = 65535) {
    return dim3(std::max(1, std::min(cdiv(largest, 256), bx_max)), (unsigned)std::min<size_t>(rows, by_max));
}

// the transformed concatenation of the rows, block `blk` of its grid: the solo launch's own 2-D grid (KfGridSolo), or the flattened
// one of a session in the batched loop closure (KfGridAt)
struct KfGridSolo {
    __device__ __forceinline__ unsigned int bx() const { return blockIdx.x; }
    __device__ __forceinline__ unsigned int by() const { return blockIdx.y; }
    __device__ __forceinline__ unsigned int gx() const { return gridDim.x; }
    __device__ __forceinline__ unsigned int gy() const { return gridDim.y; }
};
struct KfGridAt {
    unsigned int x, y, w, h;
    __device__ __forceinline__ unsigned int bx() const { return x; }
    __device__ __forceinline__ unsigned int by() const { return y; }
    __device__ __forceinline__ unsigned int gx() const { return w; }
    __device__ __forceinline__ unsigned int gy() const { return h; }
};
template <class Row, class Grid>
__device__ __forceinline__ void kf_gather_at(const unsigned char* __restrict__ arena, const Row* __restrict__ tab, int rows, int stride,
                                             unsigned char* __restrict__ out, const Grid blk) {
    for (int y = blk.by(); y < rows; y += blk.gy()) {
        const Row& r = tab[y];
        for (int i = blk.bx() * blockDim.x + threadIdx.x; i < r.n; i += blk.gx() * blockDim.x)
            kf_row_point(r, kf_row_src(r, arena, stride, r.src_off + i), stride, out + (size_t)(r.dst_off + i) * stride);
    }
}

// box (vg_box.h) of the finite transformed points of the rows, joined into mm
template <class Row>
__device__ __forceinline__ void kf_box_at(const unsigned char* __restrict__ arena, const Row* __restrict__ tab, int rows, int stride,
                                          int* __restrict__ mm) {
    int box[kBoxInts];
#pragma unroll
    for (int k = 0; k < kBoxInts; ++k) box[k] = vg_box_empty(k);
    for (int y = blockIdx.y; y < rows; y += gridDim.y) {
        const Row& r = tab[y];
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < r.n; i += gridDim.x * blockDim.x) {
            const VgXyz p = kf_row_xyz(r, kf_row_src(r, arena, stride, r.src_off + i));
            if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) vg_box_add(box, p.x, p.y, p.z);
        }
    }
    vg_box_commit(box, mm);
}

// PCL's relative voxel index of every transformed point (not finite: all-ones, or bit 32 of a wide key), value = its index in
// the concatenation
template <typename K, class Row>
__device__ __forceinline__ void kf_keys_at(const unsigned char* __restrict__ arena, const Row* __restrict__ tab, int rows, int stride,
                                           const VgParams p, K* __restrict__ keys, int* __restrict__ vals) {
    const K sentinel = sizeof(K) == 4 ? (K)0xffffffffu : (K)(1ull << 32);
    for (int y = blockIdx.y; y < rows; y += gridDim.y) {
        const Row& r = tab[y];
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < r.n; i += gridDim.x * blockDim.x) {
            const VgXyz x = kf_row_xyz(r, kf_row_src(r, arena, stride, r.src_off + i));
            const long long d = r.dst_off + i;
            keys[d] = (isfinite(x.x) && isfinite(x.y) && isfinite(x.z)) ? (K)vg_rel_index(p, x.x, x.y, x.z) : sentinel;
            vals[d] = (int)d;
        }
    }
}

// centroid of every voxel of the sorted keys (the first n_fin entries are the finite points), members transformed on load
template <int STRIDE, typename K, class Row>
__device__ __forceinline__ void kf_centroid_at(const unsigned char* arena, const Row* tab, int rows,
                                               const K* keys, const int* vals, const int* flags,
                                               const int* rank, int n_fin, unsigned char* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_fin || !flags[i]) return;
    const VgAcc<STRIDE> a = vg_walk<STRIDE>(keys, i, n_fin, [&](int j) { return vals[j]; }, KfRowLoader<STRIDE, Row>{arena, tab, rows});
    vg_write<STRIDE>(a.s, a.n, out + (size_t)rank[i] * STRIDE);
}

// The table kernels over one store's arena (KfRow) ...
__global__ void k_kf_gather(const unsigned char* __restrict__ arena, const KfRow* __restrict__ tab, int rows, int stride,
                            unsigned char* __restrict__ out) {
    kf_gather_at(arena, tab, rows, stride, out, KfGridSolo{});
}
__global__ void k_kf_box(const unsigned char* __restrict__ arena, const KfRow* __restrict__ tab, int rows, int stride, int* __restrict__ mm) {
    kf_box_at(arena, tab, rows, stride, mm);
}
template <typename K>
__global__ void k_kf_keys(const unsigned char* __restrict__ arena, const KfRow* __restrict__ tab, int rows, int stride, const VgParams p,
                          K* __restrict__ keys, int* __restrict__ vals) {
    kf_keys_at(arena, tab, rows, stride, p, keys, vals);
}
template <int STRIDE, typename K>
__global__ void k_kf_centroid(const unsigned char* __restrict__ arena, const KfRow* __restrict__ tab, int rows, const K* __restrict__ keys,
                              const int* __restrict__ vals, const int* __restrict__ flags, const int* __restrict__ rank, int n_fin,
                              unsigned char* __restrict__ out) {
    kf_centroid_at<STRIDE>(arena, tab, rows, keys, vals, flags, rank, n_fin, out);
}
// ... and over rows of several stores (KfRowM: each row names its arena; `arena` is not read)
__global__ void k_kf_gather_m(const unsigned char* __restrict__ arena, const KfRowM* __restrict__ tab, int rows, int stride,
                              unsigned char* __restrict__ out) {
    kf_gather_at(arena, tab, rows, stride, out, KfGridSolo{});
}
__global__ void k_kf_box_m(const unsigned char* __restrict__ arena, const KfRowM* __restrict__ tab, int rows, int stride, int* __restrict__ mm) {
    kf_box_at(arena, tab, rows, stride, mm);
}
template <typename K>
__global__ void k_kf_keys_m(const unsigned char* __restrict__ arena, const KfRowM* __restrict__ tab, int rows, int stride, const VgParams p,
                            K* __restrict__ keys, int* __restrict__ vals) {
    kf_keys_at(arena, tab, rows, stride, p, keys, vals);
}
template <int STRIDE, typename K>
__global__ void k_kf_centroid_m(const unsigned char* __restrict__ arena, const KfRowM* __restrict__ tab, int rows, const K* __restrict__ keys,
                                const int* __restrict__ vals, const int* __restrict__ flags, const int* __restrict__ rank, int n_fin,
                                unsigned char* __restrict__ out) {
    kf_centroid_at<STRIDE>(arena, tab, rows, keys, vals, flags, rank, n_fin, out);
}

// Each row type's kernels, for the host code written once over both (kf_gather, gmap_run, loop_cloud)
template <class Row> struct KfKern;
template <> struct KfKern<KfRow> {
    static constexpr auto gather = k_kf_gather;
    static constexpr auto box = k_kf_box;
    template <typename K> static constexpr auto keys = k_kf_keys<K>;
    template <int S, typename K> static constexpr auto centroid = k_kf_centroid<S, K>;
};
template <> struct KfKern<KfRowM> {
    static constexpr auto gather = k_kf_gather_m;
    static constexpr auto box = k_kf_box_m;
    template <typename K> static constexpr auto keys = k_kf_keys_m<K>;
    template <int S, typename K> static constexpr auto centroid = k_kf_centroid_m<S, K>;
};

// reflectivity (curvature = 0.1 * reflectivity, L/src/FormatConvert.cpp:21) of 48-byte points; `i` as in the other bodies
__device__ __forceinline__ void kf_refl_at(const unsigned char* __restrict__ pts, int n, float* __restrict__ out, const int i) {
    if (i < n) out[i] = reinterpret_cast<const float*>(pts + (size_t)i * 48)[9];
}
__global__ void k_kf_refl(const unsigned char* __restrict__ pts, int n, float* __restrict__ out) {
    kf_refl_at(pts, n, out, blockIdx.x * blockDim.x + threadIdx.x);
}

// Room for `pts` points in `arena`, of which the first `used` are stored.  Grows geometrically and COPIES the stored points
// (DevBuf::ensure would discard them); the cudaFree of the old block synchronises, which only happens on growth.
// The store has two arenas: kf_arena (the down-sampled edge/surf clouds, ~2k points per keyframe) and kf_full (the full clouds,
// ~20k points per keyframe, GBs over a long run).  One arena would recopy every full cloud each time the small clouds grow it.
static int kf_reserve(liliom_ctx* c, DevBuf& arena, long long used, long long pts) {
    const size_t stride = (size_t)c->prm.point_stride;
    const size_t need = (size_t)pts * stride;
    if (need <= arena.cap) return LILIOM_OK;
    const size_t want = std::max(need + need / 2, std::max(arena.cap * 2, (size_t)1 << 20));
    DevBuf grown;
    LILI_CUDA(c, cudaMalloc(&grown.p, want));
    grown.cap = want;
    if (used > 0) {
        LILI_CUDA(c, cudaMemcpyAsync(grown.p, arena.p, (size_t)used * stride, cudaMemcpyDeviceToDevice, c->stream));
        LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    }
    arena = std::move(grown);
    return LILIOM_OK;
}

static bool kf_ids_ok(liliom_ctx* c, const int* ids, int k) {
    for (int i = 0; i < k; ++i)
        if (ids[i] < 0 || ids[i] >= (int)c->kfs.size()) {
            char buf[96];
            snprintf(buf, sizeof(buf), "unknown keyframe id %d (%d stored)", ids[i], (int)c->kfs.size());
            c->last_error = buf;
            return false;
        }
    return true;
}

template <class Row>
static int kf_upload_table(liliom_ctx* c, const std::vector<Row>& tab) {
    LILI_CUDA(c, c->kf_tab.ensure(tab.size() * sizeof(Row)));
    LILI_CUDA(c, cudaMemcpyAsync(c->kf_tab.p, tab.data(), tab.size() * sizeof(Row), cudaMemcpyHostToDevice, c->stream));
    return LILIOM_OK;
}

// Transform + concatenate rows (of `arena`, or each of its own: KfRowM) into `out` (one launch).
template <class Row>
static int kf_gather(liliom_ctx* c, const void* arena, const std::vector<Row>& tab, long long largest, void* out) {
    if (tab.empty() || largest <= 0) return LILIOM_OK;
    LILI_TRY(kf_upload_table(c, tab));
    KfKern<Row>::gather<<<kf_row_grid(tab.size(), largest, c->sm_count * 4), 256, 0, c->stream>>>(
        (const unsigned char*)arena, c->kf_tab.as<Row>(), (int)tab.size(), c->prm.point_stride, (unsigned char*)out);
    return launch_check(c, "k_kf_gather");
}

// The store of each list entry: c for every entry (the single-store calls) or stores[i] (liliom_*_multi)
struct KfStores {
    liliom_ctx* c;
    liliom_ctx* const* per = nullptr;
    liliom_ctx* operator[](int i) const { return per ? per[i] : c; }
};

// The multi-store calls' lists: every store there, on c's device, of c's point layout and without a communicator, every id known
// to its store.  Nothing changes on an error.
static bool kf_stores_ok(liliom_ctx* c, liliom_ctx* const* stores, const int* kf_ids, int k) {
    for (int i = 0; i < k; ++i) {
        const liliom_ctx* st = stores[i];
        const char* why = !st ? "is NULL"
                        : st->device != c->device ? "is on another device"
                        : st->prm.point_stride != c->prm.point_stride ? "has another point_stride"
                        : st->nranks > 1 ? "has a communicator: the backend keyframe store is single-GPU" : nullptr;
        if (why) { c->last_error = "store of entry " + std::to_string(i) + " " + why; return false; }
        if (kf_ids[i] < 0 || kf_ids[i] >= (int)st->kfs.size()) {
            c->last_error = "unknown keyframe id " + std::to_string(kf_ids[i]) + " in the store of entry " + std::to_string(i) + " (" +
                            std::to_string(st->kfs.size()) + " stored)";
            return false;
        }
    }
    return true;
}

// The ids of a list: known to c's own store (KfRow) or each to its entry's store (KfRowM, kf_stores_ok).  Nothing changes on an error.
template <class Row>
static bool kf_list_ok(liliom_ctx* c, liliom_ctx* const* stores, const int* kf_ids, int k) {
    if constexpr (std::is_same<Row, KfRowM>::value) return kf_stores_ok(c, stores, kf_ids, k);
    else return kf_ids_ok(c, kf_ids, k);
}

// The distinct stores of the lists, in order of first appearance, appended to v (each once)
static void kf_add_stores(std::vector<liliom_ctx*>& v, liliom_ctx* const* stores, int k) {
    for (int i = 0; i < k; ++i)
        if (std::find(v.begin(), v.end(), stores[i]) == v.end()) v.push_back(stores[i]);
}

// The stores' work so far before c's reads of their arenas (as liliom_kf_add_resident joins its source): each distinct stream once
static int kf_join_stores(liliom_ctx* c, std::initializer_list<std::pair<liliom_ctx* const*, int>> lists) {
    std::vector<liliom_ctx*> v;
    for (const auto& l : lists) kf_add_stores(v, l.first, l.second);
    return batch_join_in(c, v);
}

// The sort chain's values and PCL's indices are ints
static int kf_points_ok(liliom_ctx* c, long long N) {
    if (N < (1LL << 31)) return LILIOM_OK;
    c->last_error = "the listed keyframes hold " + std::to_string(N) + " points (at most 2^31 - 1)";
    return LILIOM_E_CAPACITY;
}

// detectLoopClosure's cloud of the listed keyframes (:2476-2497, :2502-2547): edge then surf of each, transformed by its pose,
// concatenated into bmap_raw (one launch), VoxelGrid(leaf) into vg_out with its count at d_count (device) and *m (host).
// *n_in: the points read (0: nothing was launched, d_count is not written and *m = 0).
// The rows of such a cloud appended to tab (destinations from 0); returns its points, *largest = the largest keyframe cloud.
template <class Row>
static long long kf_cloud_rows(KfStores s, const int* kf_ids, const double* poses7, int k, std::vector<Row>& tab, long long* largest) {
    long long off = 0;
    *largest = 0;
    for (int i = 0; i < k; ++i) {                                 // :2492-2493 / :2519-2520: *edge_frames[i] then *surf_frames[i]
        const KfEntry& f = s[i]->kfs[kf_ids[i]];
        const void* arena = s[i]->kf_arena.p;
        if (f.n_edge) tab.push_back(kf_row_in<Row>(arena, f.edge_off, off, f.n_edge, poses7 + 7 * (size_t)i));
        off += f.n_edge;
        if (f.n_surf) tab.push_back(kf_row_in<Row>(arena, f.surf_off, off, f.n_surf, poses7 + 7 * (size_t)i));
        off += f.n_surf;
        *largest = std::max(*largest, (long long)std::max(f.n_edge, f.n_surf));
    }
    return off;
}

static int kf_cloud_dev(liliom_ctx* c, const int* kf_ids, const double* poses7, int k, float leaf, int* d_count, long long* n_in, int* m) {
    const int stride = c->prm.point_stride;
    std::vector<KfRow> tab;
    long long largest = 0;
    const long long off = kf_cloud_rows(KfStores{c}, kf_ids, poses7, k, tab, &largest);
    *n_in = off;
    *m = 0;
    if (off == 0) return LILIOM_OK;
    LILI_CUDA(c, c->bmap_raw.ensure((size_t)off * stride));      // scratch: the local map's layers live in bmap_ds / bmap
    c->n_ds_resident = -1;      // vg_out is rewritten: no scan for liliom_map_update_resident
    LILI_CUDA(c, c->vg_out.ensure((size_t)off * stride));
    LILI_TRY(kf_gather(c, c->kf_arena.p, tab, largest, c->bmap_raw.p));
    return voxelgrid_dev_sync(c, c->bmap_raw.p, (int)off, stride, leaf, c->vg_out.p, d_count, nullptr, m);
}

static int backend_check(liliom_ctx* c, const liliom_backend_params* bp) {
    if (c->nranks > 1) { c->last_error = "the backend keyframe store is single-GPU"; return LILIOM_E_ARG; }
    if (bp && (!(bp->edge_leaf > 0) || !(bp->surf_leaf > 0) || !(bp->kd_max_radius > 0) || (bp->variant != 0 && bp->variant != 1)))
        return LILIOM_E_ARG;
    return LILIOM_OK;
}

// the scan half's surf output (ms points in vg_out) behind its me edge points, at the tail of kf_arena
static int kf_surf_behind(liliom_ctx* c, int me, int ms) {
    const size_t stride = (size_t)c->prm.point_stride;
    unsigned char* tail = (unsigned char*)c->kf_arena.p + (size_t)c->kf_used * stride;
    if (ms) LILI_CUDA(c, cudaMemcpyAsync(tail + (size_t)me * stride, c->vg_out.p, (size_t)ms * stride, cudaMemcpyDeviceToDevice, c->stream));
    return LILIOM_OK;
}

// The keyframe store's writes, from clouds already on the device (the host calls upload them first; liliom_kf_add_resident
// reads them where an extraction left them).  The caller has reserved room behind the stored points (kf_reserve) and records
// the keyframe (KfEntry) once everything it stores is written.
// The scan half (:1502-1514): VoxelGrid(edge_leaf) of edge and VoxelGrid(surf_leaf) of surf behind the stored points of
// kf_arena, edge first; the surf output also stays in vg_out.
static int kf_scan_dev(liliom_ctx* c, const liliom_backend_params* bp, const void* edge, int n_edge, const void* surf, int n_surf,
                       int* me, int* ms) {
    const int stride = c->prm.point_stride;
    c->n_ds_resident = -1;      // vg_out is rewritten: no scan for liliom_map_update_resident
    LILI_CUDA(c, c->vg_out.ensure((size_t)(n_surf > 0 ? n_surf : 1) * stride));
    LILI_CUDA(c, c->vg_count.ensure(16));
    unsigned char* tail = (unsigned char*)c->kf_arena.p + (size_t)c->kf_used * stride;
    int* cnt = c->vg_count.as<int>();
    LILI_TRY(voxelgrid_dev_sync(c, edge, n_edge, stride, bp->edge_leaf, tail, cnt, nullptr, me));                 // :1502-1507
    LILI_TRY(voxelgrid_dev_sync(c, surf, n_surf, stride, bp->surf_leaf, c->vg_out.p, cnt + 1, nullptr, ms));      // :1509-1514
    return kf_surf_behind(c, *me, *ms);
}

// The full-cloud half (L:1494-1500 / R:1373-1376) behind the stored points of kf_full: variant 0 the n points as received (one
// copy from wherever they lie, host or device), variant 1 VoxelGrid(surf_leaf) of them (on the device).  *m: the points written.
static int kf_full_dev(liliom_ctx* c, const liliom_backend_params* bp, const void* full, int n, int* m) {
    const int stride = c->prm.point_stride;
    unsigned char* tail = (unsigned char*)c->kf_full.p + (size_t)c->kf_full_used * stride;
    *m = n;
    if (n > 0 && bp->variant == 0) {                              // L:1498-1500 full_clouds: the cloud as received
        LILI_CUDA(c, cudaMemcpyAsync(tail, full, (size_t)n * stride, cudaMemcpyDefault, c->stream));
    } else if (n > 0) {                                           // R:1373-1376 full_clouds_ds: VoxelGrid(surf_leaf) of it
        LILI_CUDA(c, c->vg_count.ensure(16));
        LILI_TRY(voxelgrid_dev_sync(c, full, n, stride, bp->surf_leaf, tail, c->vg_count.as<int>(), nullptr, m));
    }
    return LILIOM_OK;
}

// Records a keyframe whose scan half (me edge + ms surf points) kf_scan_dev has written; returns its id
static int kf_push(liliom_ctx* c, int me, int ms) {
    c->kfs.push_back(KfEntry{c->kf_used, c->kf_used + me, me, ms});
    c->kf_used += (long long)me + ms;
    return (int)c->kfs.size() - 1;
}
// ... and its full cloud (m points) that kf_full_dev has written
static void kf_push_full(liliom_ctx* c, int kf_id, int m) {
    c->kfs[kf_id].full_off = c->kf_full_used;
    c->kfs[kf_id].n_full = m;
    c->kf_full_used += m;
}

// liliom_kf_add_resident in parts, run by the solo call and by the batch (liliom_kf_add_resident_batch): kf_res_begin (validation,
// nothing changes on an error; the source's clouds), their sizes (feat_sizes), kf_res_reserve (both arenas before any write), the
// VoxelGrid chain of each cloud (kf_scan_dev and kf_full_dev on the solo path), kf_res_finish (the keyframe's records).
struct KfResJob {
    liliom_ctx* c = nullptr;                 // the backend
    const liliom_backend_params* bp = nullptr;
    FeatCloud f[3];                          // the source's surf, edge and cut (ROT: laserCloud)
    int m[3] = {0, 0, 0};                    // their sizes
    int me = 0, ms = 0, mf = 0;              // points stored: edge, surf, full
};

static int kf_res_begin(liliom_ctx* c, const liliom_backend_params* bp, liliom_ctx* src, KfResJob& j) {
    if (!src) return LILIOM_E_ARG;
    LILI_TRY(backend_check(c, bp));
    if (src->nranks > 1) { c->last_error = "the source context has a communicator: the backend keyframe store is single-GPU"; return LILIOM_E_ARG; }
    if (src->prm.point_stride != c->prm.point_stride || src->device != c->device) return LILIOM_E_ARG;
    j = KfResJob{};
    j.c = c; j.bp = bp;
    return feat_clouds(src, j.f);
}

static int kf_res_reserve(const KfResJob& j) {
    liliom_ctx* c = j.c;
    LILI_TRY(kf_reserve(c, c->kf_arena, c->kf_used, c->kf_used + (long long)j.m[1] + j.m[0]));
    return kf_reserve(c, c->kf_full, c->kf_full_used, c->kf_full_used + j.m[2]);
}

static void kf_res_finish(const KfResJob& j, int* kf_id, int* n_edge_ds, int* n_surf_ds, int* n_full_stored) {
    *kf_id = kf_push(j.c, j.me, j.ms);
    kf_push_full(j.c, *kf_id, j.mf);
    if (n_edge_ds) *n_edge_ds = j.me;
    if (n_surf_ds) *n_surf_ds = j.ms;
    if (n_full_stored) *n_full_stored = j.mf;
}

// liliom_bmap_build in parts, run by the solo calls and by the batches (liliom_bmap_build(_batch)(_multi)): bmap_check (validation,
// nothing changes on an error), bmap_tables (the keyframe table, uploaded, and the buffers of both layers), the gather of the table
// into bmap_raw, per
// layer voxelgrid_dev's chain into bmap_ds[l] and bmap[l].xyzw, each layer's cell grid, the surf layer's reflectivity (48-byte
// points), bmap_finish (the counts).
struct BmapJob {
    liliom_ctx* c = nullptr;
    const liliom_backend_params* bp = nullptr;
    int rows = 0;                        // keyframe table rows: edge rows (destinations from 0) and surf rows (from E), list order
    long long largest = 0;               // the largest keyframe cloud (the gather's grid)
    long long n[2] = {0, 0};             // points of each layer's concatenation: E (edge), S (surf, behind the edge points)
    int m[2] = {0, 0};                   // the layers' points (VoxelGrid output counts)
    GridJob g[2];                        // the layers' cell grids (the batch's grid_begin .. grid_finish)
    bool grid[2] = {false, false};       // the batch: layer l's cell grid is begun and its launches are still to run
    unsigned long long launches_surf_box = 0;      // the batch: launches before the surf layer's box pass
};

static float bmap_leaf(const BmapJob& j, int l) { return l == 0 ? j.bp->edge_leaf : j.bp->surf_leaf; }
// :1543 sqdist[4] < 1.0 (edge), :1615 sqdist[4] < kd_max_radius (surf)
static float bmap_cell(const BmapJob& j, int l) { return l == 0 ? gate_cell(1.0) : gate_cell(j.bp->kd_max_radius); }
static const unsigned char* bmap_in(const BmapJob& j, int l) {
    return (const unsigned char*)j.c->bmap_raw.p + (l == 0 ? 0 : (size_t)j.n[0] * j.c->prm.point_stride);
}
static dim3 bmap_gather_grid(const BmapJob& j) { return kf_row_grid(j.rows, j.largest, j.c->sm_count * 4); }

// Validation, nothing changes on an error (the previous layers stay): the entries' keyframes are c's own (KfRow, stores unused)
// or each of its entry's store (KfRowM, liliom_bmap_build_multi)
template <class Row>
static int bmap_check(liliom_ctx* c, const liliom_backend_params* bp, liliom_ctx* const* stores, const int* kf_ids, const double* poses7,
                      int k) {
    constexpr bool multi = std::is_same<Row, KfRowM>::value;
    if (k < 0 || (k > 0 && (!kf_ids || !poses7 || (multi && !stores)))) return LILIOM_E_ARG;
    LILI_TRY(backend_check(c, bp));
    return kf_list_ok<Row>(c, stores, kf_ids, k) ? LILIOM_OK : LILIOM_E_ARG;
}

// After bmap_check: the keyframe table (rows of the table's type, read from each entry's store), uploaded, and the buffers of both
// layers.  Every call over either row type runs this one builder (kf_bmap_rows), largest-cloud rule and sizing.
template <class Row>
static int bmap_tables(liliom_ctx* c, const liliom_backend_params* bp, KfStores s, const int* kf_ids, const double* poses7, int k,
                       BmapJob& j) {
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    c->bmap_built = false;
    j = BmapJob{};
    j.c = c; j.bp = bp;
    std::vector<Row> tab;
    kf_bmap_rows(
        [&](int i) {
            const KfEntry& f = s[i]->kfs[kf_ids[i]];
            return KfClouds{s[i]->kf_arena.p, f.edge_off, f.surf_off, f.n_edge, f.n_surf};
        },
        poses7, k, tab, j.n, &j.largest);
    j.rows = (int)tab.size();
    LILI_CUDA(c, c->bmap_raw.ensure((size_t)std::max(j.n[0] + j.n[1], 1LL) * stride));
    if (j.rows > 0) LILI_TRY(kf_upload_table(c, tab));
    LILI_CUDA(c, c->vg_count.ensure(16));
    for (int l = 0; l < 2; ++l) {                                 // the centroid kernel also writes the float4 points
        LILI_CUDA(c, c->bmap_ds[l].ensure((size_t)std::max(j.n[l], 1LL) * stride));
        LILI_CUDA(c, c->bmap[l].xyzw.ensure((size_t)std::max(j.n[l], 1LL) * sizeof(float4)));
        if (j.n[l] > 0) LILI_TRY(vg_chain_ensure(c, j.n[l], 4));   // voxelgrid_dev's buffers at 32-bit keys
    }
    return LILIOM_OK;
}

static void bmap_finish(const BmapJob& j, int* n_edge_map, int* n_surf_map) {
    liliom_ctx* c = j.c;
    c->bmap_n[0] = j.m[0]; c->bmap_n[1] = j.m[1];
    c->bmap_built = true;
    if (n_edge_map) *n_edge_map = j.m[0];
    if (n_surf_map) *n_surf_map = j.m[1];
}

}  // namespace lili

using namespace lili;

extern "C" void liliom_backend_default_params(liliom_backend_params* p, int variant) {
    if (!p) return;
    memset(p, 0, sizeof(*p));
    p->variant = variant == 1 ? 1 : 0;
    p->edge_leaf = 0.2f;                 // L/config/config_fr_iosb.yaml edge_ds; R/src/BackendFusion.cpp:491
    p->surf_leaf = 0.4f;                 // L/config/config_fr_iosb.yaml surf_ds; R/src/BackendFusion.cpp:492
    p->kd_max_radius = 1.0;              // both config_fr_iosb.yaml
    p->surf_dist_thres = 0.12;           // both config_fr_iosb.yaml
    p->w_gate = variant == 1 ? 0.3 : 0.2;              // R/src/BackendFusion.cpp:1504, L/src/BackendFusion.cpp:1665
    p->lidar_const = variant == 1 ? 7.5 : 20.0;        // R/ and L/ config_fr_iosb.yaml
    p->reflect_thres = 15.0;             // L/config/config_fr_iosb.yaml (variant 0 only)
    p->cauchy_b = 1.0;                   // L/src/BackendFusion.cpp:845
    if (variant == 1) {                  // R/config/config_fr_iosb.yaml ql2b_*, tl2b_*
        p->q_lb[0] = 0.7071; p->q_lb[3] = 0.7071;
        p->t_lb[0] = -0.18; p->t_lb[2] = -0.095;
    } else {                             // L/config/config_fr_iosb.yaml ql2b_*, tl2b_*
        p->q_lb[3] = 1.0;
        p->t_lb[0] = -0.0265; p->t_lb[1] = 0.0202; p->t_lb[2] = 0.05309;
    }
}

extern "C" int liliom_kf_add(liliom_ctx* c, const liliom_backend_params* bp, const void* edge_last, int n_edge, const void* surf_last, int n_surf,
                             int* kf_id, void* edge_ds_out, int edge_cap, int* n_edge_ds, void* surf_ds_out, int surf_cap, int* n_surf_ds) {
    if (!c || !bp || !kf_id || n_edge < 0 || n_surf < 0 || (n_edge > 0 && !edge_last) || (n_surf > 0 && !surf_last)) return LILIOM_E_ARG;
    LILI_TRY(backend_check(c, bp));
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    const long long n = (long long)n_edge + n_surf;
    LILI_TRY(kf_reserve(c, c->kf_arena, c->kf_used, c->kf_used + n));          // VoxelGrid never outputs more points than it reads
    LILI_CUDA(c, c->raw.ensure((size_t)(n > 0 ? n : 1) * stride));
    unsigned char* raw = (unsigned char*)c->raw.p;
    if (n_edge) LILI_CUDA(c, cudaMemcpyAsync(raw, edge_last, (size_t)n_edge * stride, cudaMemcpyHostToDevice, c->stream));
    if (n_surf) LILI_CUDA(c, cudaMemcpyAsync(raw + (size_t)n_edge * stride, surf_last, (size_t)n_surf * stride, cudaMemcpyHostToDevice, c->stream));
    int me = 0, ms = 0;
    LILI_TRY(kf_scan_dev(c, bp, raw, n_edge, raw + (size_t)n_edge * stride, n_surf, &me, &ms));
    if (n_edge_ds) *n_edge_ds = me;
    if (n_surf_ds) *n_surf_ds = ms;
    if ((edge_ds_out && me > edge_cap) || (surf_ds_out && ms > surf_cap)) return LILIOM_E_CAPACITY;   // nothing stored
    const unsigned char* tail = (const unsigned char*)c->kf_arena.p + (size_t)c->kf_used * stride;
    if (edge_ds_out && me) LILI_CUDA(c, cudaMemcpyAsync(edge_ds_out, tail, (size_t)me * stride, cudaMemcpyDeviceToHost, c->stream));
    if (surf_ds_out && ms) LILI_CUDA(c, cudaMemcpyAsync(surf_ds_out, c->vg_out.p, (size_t)ms * stride, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    *kf_id = kf_push(c, me, ms);
    return LILIOM_OK;
}

// publishCloudLast -> BackendFusion's keyframe without the host: the scan half and the full cloud from the clouds an extraction
// left resident on src (surf_last, edge_last, full_cloud), on c's stream ordered after src's, in one all-or-nothing call.
extern "C" int liliom_kf_add_resident(liliom_ctx* c, const liliom_backend_params* bp, liliom_ctx* src, int* kf_id, int* n_edge_ds,
                                      int* n_surf_ds, int* n_full_stored) {
    if (!c || !bp || !src || !kf_id) return LILIOM_E_ARG;
    KfResJob j;
    LILI_TRY(kf_res_begin(c, bp, src, j));
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_TRY(feat_sizes(src, j.f, j.m));                          // they size the arenas and the filters
    LILI_TRY(batch_join_in(c, {src}));                            // src's work so far before c's reads of its clouds
    LILI_TRY(kf_res_reserve(j));
    LILI_TRY(kf_scan_dev(c, bp, j.f[1].buf->p, j.m[1], j.f[0].buf->p, j.m[0], &j.me, &j.ms));
    LILI_TRY(kf_full_dev(c, bp, j.f[2].buf->p, j.m[2], &j.mf));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    kf_res_finish(j, kf_id, n_edge_ds, n_surf_ds, n_full_stored);
    return LILIOM_OK;
}

extern "C" int liliom_kf_count(const liliom_ctx* c) { return c ? (int)c->kfs.size() : 0; }

extern "C" int liliom_kf_clear(liliom_ctx* c) {
    if (!c) return LILIOM_E_ARG;
    c->kfs.clear();
    c->kf_used = 0;                      // the arenas keep their allocations
    c->kf_full_used = 0;
    c->bmap_built = false; c->bmap_n[0] = c->bmap_n[1] = 0;
    c->bmap[0].ready = c->bmap[1].ready = false;
    c->win_k = 0;
    return LILIOM_OK;
}

namespace lili {

// The solo call after bmap_tables: the gather (of c's own arena, or of the arena each KfRowM row names), both layers' VoxelGrid
// chains and cell grids, the reflectivity, one wait at the end
template <class Row>
static int bmap_run(BmapJob& j, int* n_edge_map, int* n_surf_map) {
    liliom_ctx* c = j.c;
    const int stride = c->prm.point_stride;
    if (j.rows > 0) {
        KfKern<Row>::gather<<<bmap_gather_grid(j), 256, 0, c->stream>>>((const unsigned char*)c->kf_arena.p, c->kf_tab.as<Row>(), j.rows,
                                                                        stride, (unsigned char*)c->bmap_raw.p);
        LILI_TRY(launch_check(c, "k_kf_gather"));
    }
    for (int l = 0; l < 2; ++l)                                   // :1486-1492
        LILI_TRY(voxelgrid_dev_sync(c, bmap_in(j, l), (int)j.n[l], stride, bmap_leaf(j, l), c->bmap_ds[l].p, c->vg_count.as<int>() + l,
                                    c->bmap[l].xyzw.as<float4>(), &j.m[l]));
    for (int l = 0; l < 2; ++l) LILI_TRY(grid_build(c, c->bmap[l], bmap_cell(j, l), j.m[l]));
    if (stride == 48) {                                                         // reflectivity of the surf layer (:1617-1638)
        LILI_CUDA(c, c->bmap[1].refl.ensure((size_t)std::max(j.m[1], 1) * sizeof(float)));
        if (j.m[1] > 0) {
            k_kf_refl<<<cdiv(j.m[1], 256), 256, 0, c->stream>>>((const unsigned char*)c->bmap_ds[1].p, j.m[1], c->bmap[1].refl.as<float>());
            LILI_TRY(launch_check(c, "k_kf_refl"));
        }
    }
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    bmap_finish(j, n_edge_map, n_surf_map);
    return LILIOM_OK;
}

}  // namespace lili

extern "C" int liliom_bmap_build(liliom_ctx* c, const liliom_backend_params* bp, const int* kf_ids, const double* poses7, int k,
                                 int* n_edge_map, int* n_surf_map) {
    if (!c || !bp) return LILIOM_E_ARG;
    LILI_TRY(bmap_check<KfRow>(c, bp, nullptr, kf_ids, poses7, k));
    BmapJob j;
    LILI_TRY(bmap_tables<KfRow>(c, bp, KfStores{c}, kf_ids, poses7, k, j));
    return bmap_run<KfRow>(j, n_edge_map, n_surf_map);
}

// liliom_bmap_build over keyframes of several stores: rows that name their store's arena, the rest unchanged on c
extern "C" int liliom_bmap_build_multi(liliom_ctx* c, const liliom_backend_params* bp, liliom_ctx* const* stores, const int* kf_ids,
                                       const double* poses7, int k, int* n_edge_map, int* n_surf_map) {
    if (!c || !bp) return LILIOM_E_ARG;
    LILI_TRY(bmap_check<KfRowM>(c, bp, stores, kf_ids, poses7, k));
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_TRY(kf_join_stores(c, {{stores, k}}));
    BmapJob j;
    LILI_TRY(bmap_tables<KfRowM>(c, bp, KfStores{c, stores}, kf_ids, poses7, k, j));
    return bmap_run<KfRowM>(j, n_edge_map, n_surf_map);
}

extern "C" int liliom_bmap_download(liliom_ctx* c, int layer, void* out, int cap, int* m_out) {
    if (!c || !m_out || (layer != 0 && layer != 1)) return LILIOM_E_ARG;
    if (!c->bmap_built) return LILIOM_E_NOMAP;
    LILI_CUDA(c, cudaSetDevice(c->device));
    return download_sized(c, c->bmap_ds[layer], c->bmap_n[layer], c->prm.point_stride, out, cap, m_out);
}

extern "C" int liliom_kf_cloud(liliom_ctx* c, const int* kf_ids, const double* poses7, int k, float leaf, void* out, int cap, int* n_out) {
    if (!c || !n_out || k < 0 || (k > 0 && (!kf_ids || !poses7)) || !(leaf > 0)) return LILIOM_E_ARG;
    LILI_TRY(backend_check(c, nullptr));
    if (!kf_ids_ok(c, kf_ids, k)) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    *n_out = 0;
    LILI_CUDA(c, c->vg_count.ensure(16));
    long long off = 0;
    int m = 0;
    LILI_TRY(kf_cloud_dev(c, kf_ids, poses7, k, leaf, c->vg_count.as<int>(), &off, &m));
    if (off == 0) return LILIOM_OK;
    return download_sized(c, c->vg_out, m, stride, out, cap, n_out);
}

// detectLoopClosure + performLoopClosure's alignment (:2473-2582) without leaving the device: the history cloud goes into the
// loop index (its own cell grid: the odometry map, the local map and every resident correspondence stay), the latest cloud into
// loop_src, and the ICP runs on them (icp.cu).  Scratch shared with the other calls: bmap_raw, vg_out, the sort chain, grid_keys*,
// partials.  The call is written in parts so that the solo calls and the batched ones (liliom_loop_align(_batch)(_multi)) run the
// same code: loop_check and loop_tables, then per cloud the gather, the VoxelGrid chain and the repack, then grid_begin ..
// grid_finish of the target's cell grid, then icp_begin .. icp_finish.
namespace lili {

struct LoopJob {
    liliom_ctx* c = nullptr;
    int rows[2] = {0, 0};                // keyframe table rows of the target [0] and the source [1]; the source's follow the target's
    long long off[2] = {0, 0};           // points of each concatenation
    long long largest[2] = {0, 0};       // the largest keyframe cloud of each (the gather's grid)
    float leaf = 0.0f;
    double max_corr_dist = 0.0, trans_eps = 0.0, fit_eps = 0.0;
    int max_iter = 0;
    int m[2] = {0, 0};                   // VoxelGrid output counts
    GridJob g;
    IcpJob icp;
};

static float loop_cell(const liliom_ctx* c) { return gate_cell(c->prm.knn_max_sqdist); }   // the cell of liliom_icp_align's target
static float4* loop_dst(liliom_ctx* c, int k) { return k == 0 ? c->loop.xyzw.as<float4>() : c->loop_src.as<float4>(); }

// liliom_loop_align's arguments, the keyframe lists aside
static bool loop_args_ok(const int* src_ids, const double* src_poses7, int k_src, const int* tgt_ids, const double* tgt_poses7, int k_tgt,
                         float leaf, double max_corr_dist, int max_iter) {
    return k_src >= 0 && k_tgt >= 0 && (k_src == 0 || (src_ids && src_poses7)) && (k_tgt == 0 || (tgt_ids && tgt_poses7)) && leaf > 0 &&
           max_corr_dist > 0 && max_iter >= 1;
}

// After validation: the keyframe tables of both clouds in one upload (so that both stay valid until their gathers have run), rows
// of the table's type read from each entry's store, and every buffer of the clouds' chains.
template <class Row>
static int loop_tables(liliom_ctx* c, KfStores src, const int* src_ids, const double* src_poses7, int k_src, KfStores tgt, const int* tgt_ids,
                       const double* tgt_poses7, int k_tgt, float leaf, double max_corr_dist, int max_iter, double trans_eps, double fit_eps,
                       LoopJob& j) {
    LILI_CUDA(c, cudaSetDevice(c->device));
    j = LoopJob{};
    j.c = c; j.leaf = leaf; j.max_corr_dist = max_corr_dist; j.max_iter = max_iter; j.trans_eps = trans_eps; j.fit_eps = fit_eps;
    std::vector<Row> tab;
    // :2502-2547 his_key_frames_ds (the target), :2476-2497 latest_key_frames_ds (the source)
    j.off[0] = kf_cloud_rows(tgt, tgt_ids, tgt_poses7, k_tgt, tab, &j.largest[0]);
    j.rows[0] = (int)tab.size();
    j.off[1] = kf_cloud_rows(src, src_ids, src_poses7, k_src, tab, &j.largest[1]);
    j.rows[1] = (int)tab.size() - j.rows[0];
    const long long n = std::max(j.off[0], j.off[1]);
    const int stride = c->prm.point_stride;
    LILI_CUDA(c, c->vg_count.ensure(16));
    if (n > 0) {
        LILI_TRY(kf_upload_table(c, tab));
        LILI_CUDA(c, c->bmap_raw.ensure((size_t)n * stride));   // scratch: the local map's layers live in bmap_ds / bmap
        c->n_ds_resident = -1;      // vg_out is rewritten: no scan for liliom_map_update_resident
        LILI_CUDA(c, c->vg_out.ensure((size_t)n * stride));
        LILI_TRY(vg_chain_ensure(c, n, 4));                       // voxelgrid_dev's buffers at 32-bit keys
    }
    LILI_CUDA(c, c->loop.xyzw.ensure((size_t)std::max(j.off[0], 1LL) * sizeof(float4)));
    LILI_CUDA(c, c->loop_src.ensure((size_t)std::max(j.off[1], 1LL) * sizeof(float4)));
    return LILIOM_OK;
}

// Validation before loop_tables, nothing changes on an error: both lists' keyframes are c's own (KfRow, the stores unused) or each
// of its entry's store (KfRowM, liliom_loop_align_multi: also fewer than 2^31 points per cloud)
template <class Row>
static int loop_check(liliom_ctx* c, liliom_ctx* const* src_stores, const int* src_ids, const double* src_poses7, int k_src,
                      liliom_ctx* const* tgt_stores, const int* tgt_ids, const double* tgt_poses7, int k_tgt, float leaf, double max_corr_dist,
                      int max_iter) {
    constexpr bool multi = std::is_same<Row, KfRowM>::value;
    if (!loop_args_ok(src_ids, src_poses7, k_src, tgt_ids, tgt_poses7, k_tgt, leaf, max_corr_dist, max_iter) ||
        (multi && ((k_src > 0 && !src_stores) || (k_tgt > 0 && !tgt_stores))))
        return LILIOM_E_ARG;
    LILI_TRY(backend_check(c, nullptr));
    if (!kf_list_ok<Row>(c, src_stores, src_ids, k_src) || !kf_list_ok<Row>(c, tgt_stores, tgt_ids, k_tgt)) return LILIOM_E_ARG;
    if constexpr (multi)
        for (const auto& [st, ids, k] : {std::make_tuple(src_stores, src_ids, k_src), std::make_tuple(tgt_stores, tgt_ids, k_tgt)}) {
            long long N = 0;
            for (int i = 0; i < k; ++i) N += (long long)st[i]->kfs[ids[i]].n_edge + st[i]->kfs[ids[i]].n_surf;
            LILI_TRY(kf_points_ok(c, N));
        }
    return LILIOM_OK;
}

// the gather's grid for cloud k (kf_row_grid)
static dim3 loop_gather_grid(const LoopJob& j, int k) { return kf_row_grid(j.rows[k], j.largest[k], j.c->sm_count * 4); }
template <class Row = KfRow>
static const Row* loop_rows(const LoopJob& j, int k) { return j.c->kf_tab.as<Row>() + (k == 0 ? 0 : j.rows[0]); }

// Cloud k (0 target, 1 source) on the solo path: gather, VoxelGrid with its count read back (voxelgrid_dev_sync: wide keys where
// the index wraps), repack into the loop index's points or loop_src (the count read on the device).
template <class Row>
static int loop_cloud(LoopJob& j, int k) {
    liliom_ctx* c = j.c;
    const int stride = c->prm.point_stride;
    int* cnt = c->vg_count.as<int>() + k;
    if (j.off[k] > 0) {
        KfKern<Row>::gather<<<loop_gather_grid(j, k), 256, 0, c->stream>>>((const unsigned char*)c->kf_arena.p, loop_rows<Row>(j, k), j.rows[k],
                                                                           stride, (unsigned char*)c->bmap_raw.p);
        LILI_TRY(launch_check(c, "k_kf_gather"));
        LILI_TRY(voxelgrid_dev_sync(c, c->bmap_raw.p, (int)j.off[k], stride, j.leaf, c->vg_out.p, cnt, nullptr, &j.m[k]));
    }
    return repack_to_f4(c, c->vg_out.p, (int)j.off[k], stride, loop_dst(c, k), cnt);
}

// The solo call after loop_check and loop_tables: both clouds, the target's cell grid, the ICP
template <class Row>
static int loop_run(LoopJob& j, double T16[16], double* fitness, int* converged, int* iters, int* n_src, int* n_tgt) {
    liliom_ctx* c = j.c;
    LILI_TRY(loop_cloud<Row>(j, 0));      // :2502-2547 his_key_frames_ds -> the loop index's points (float4, w = index)
    LILI_TRY(loop_cloud<Row>(j, 1));      // :2476-2497 latest_key_frames_ds -> the source
    if (n_src) *n_src = j.m[1];
    if (n_tgt) *n_tgt = j.m[0];
    LILI_TRY(grid_build(c, c->loop, loop_cell(c), j.m[0]));
    return icp_align(c, c->loop, c->loop_src.as<float4>(), j.m[1], j.max_corr_dist, j.max_iter, j.trans_eps, j.fit_eps, T16, fitness,
                     converged, iters);
}

static int loop_icp_begin(LoopJob& j) {
    liliom_ctx* c = j.c;
    return icp_begin(c, c->loop, c->loop_src.as<float4>(), j.m[1], j.max_corr_dist, j.max_iter, j.trans_eps, j.fit_eps, j.icp);
}

// ---- the loop closure of several sessions (liliom_loop_align_batch): one launch per stage for up to kBatchMax sessions.
// Everything one session's stages read or write, on its own buffers.
struct LoopEntry {
    // a cloud: the gather of its table rows into bmap_raw, the VoxelGrid chain of its n points into vg_out, the repack into xyzw
    // (the local map's chain has no repack: its centroid stage writes the float4 points into xyzw, as voxelgrid_dev's d_feats;
    // every other chain runs with xyzw null)
    const unsigned char* arena; const KfRow* tab; int rows, gx, gy;
    const unsigned char* raw; unsigned char* raw_out; int n, stride; float leaf; int* mm; int mm_blocks; VgParams* pp;
    uint32_t* keys; int* vals; const uint32_t* keys2; const int* vals2; int* flags; int* rank; unsigned char* ds; int* count;
    float4* xyzw;
    // the target's cell grid over its m points
    int m; GridDesc g; uint32_t* gkeys; int* gvals; float4* sorted; int* cell_start;
};

// The stages (k_stage_batch, ctx.cuh), each with the block size, the blocks and the body of its solo launch
LILI_STAGE(LoopStGather, LoopEntry, 256, e.gx * e.gy, kf_gather_at(e.arena, e.tab, e.rows, e.stride, e.raw_out, KfGridAt{(unsigned)(bx % e.gx), (unsigned)(bx / e.gx), (unsigned)e.gx, (unsigned)e.gy}))
LILI_STAGE(LoopStBoxInit, LoopEntry, 32, 1, vg_box_init(e.mm))
LILI_STAGE(LoopStBox, LoopEntry, 256, e.mm_blocks, vg_minmax_body(e.raw, e.n, nullptr, e.stride, e.mm, SessionBlock{bx, (unsigned)e.mm_blocks}))
LILI_STAGE(LoopStParams, LoopEntry, 32, 1, vg_params_at(e.mm, e.leaf, e.pp))
LILI_STAGE(LoopStKeys, LoopEntry, 256, stage_blocks(e.n, 256), vg_keys_at<uint32_t>(e.raw, e.n, nullptr, e.stride, e.pp, e.keys, e.vals, i))
LILI_STAGE(LoopStHeads, LoopEntry, 256, stage_blocks(e.n + 1, 256), vg_heads_at(e.keys2, e.n, &e.pp->n_finite, e.flags, i))
LILI_STAGE(LoopStCentroid48, LoopEntry, 128, stage_blocks(e.n, 128),
           (vg_centroid_at<48, uint32_t>)(e.raw, e.keys2, e.vals2, e.flags, e.rank, e.n, nullptr, e.pp, e.ds, e.count, nullptr, i))
LILI_STAGE(LoopStCentroid32, LoopEntry, 128, stage_blocks(e.n, 128),
           (vg_centroid_at<32, uint32_t>)(e.raw, e.keys2, e.vals2, e.flags, e.rank, e.n, nullptr, e.pp, e.ds, e.count, nullptr, i))
// ... and those that also write the float4 points into xyzw (the local map's chain; the others keep the stages without the store)
LILI_STAGE(LoopStCentroidXyzw48, LoopEntry, 128, stage_blocks(e.n, 128),
           (vg_centroid_at<48, uint32_t>)(e.raw, e.keys2, e.vals2, e.flags, e.rank, e.n, nullptr, e.pp, e.ds, e.count, e.xyzw, i))
LILI_STAGE(LoopStCentroidXyzw32, LoopEntry, 128, stage_blocks(e.n, 128),
           (vg_centroid_at<32, uint32_t>)(e.raw, e.keys2, e.vals2, e.flags, e.rank, e.n, nullptr, e.pp, e.ds, e.count, e.xyzw, i))
LILI_STAGE(LoopStRepack, LoopEntry, 256, stage_blocks(e.n, 256), repack_f4_at(e.ds, e.n, e.count, e.stride, e.xyzw, i))
LILI_STAGE(LoopStGridBox, LoopEntry, 256, e.mm_blocks,
           vg_minmax_body((const unsigned char*)e.xyzw, e.m, nullptr, (int)sizeof(float4), e.mm, SessionBlock{bx, (unsigned)e.mm_blocks}))
LILI_STAGE(LoopStCellKeys, LoopEntry, 256, stage_blocks(e.m, 256), cell_keys_at(e.xyzw, e.m, e.g, e.gkeys, e.gvals, nullptr, i))
LILI_STAGE(LoopStGatherSorted, LoopEntry, 256, stage_blocks(e.m, 256), gather_sorted_at(e.xyzw, e.vals2, e.m, e.sorted, i))
LILI_STAGE(LoopStRunEnds, LoopEntry, 256, stage_blocks(e.m, 256), cell_run_ends_at(e.keys2, e.m, e.cell_start, i))

// LoopStGather's body over a table of rows that each name their store's arena (KfRowM: the batched multi-store calls).  An entry
// of its own, so that LoopEntry and every LoopSt* stage keep their parameters.
struct KfGatherMEntry {
    const KfRowM* tab; int rows, gx, gy, stride; unsigned char* out;
};
LILI_STAGE(KfStGatherM, KfGatherMEntry, 256, e.gx * e.gy, kf_gather_at((const unsigned char*)nullptr, e.tab, e.rows, e.stride, e.out, KfGridAt{(unsigned)(bx % e.gx), (unsigned)(bx / e.gx), (unsigned)e.gx, (unsigned)e.gy}))

// One session's gather in a batched launch, as its solo launch takes it: rows of c's keyframe table, its grid, the output
template <class Row>
struct KfGatherAt {
    liliom_ctx* c; const Row* tab; int rows; dim3 grid; void* out;
};
// The gathers of the sessions `which` (at(i): session i's KfGatherAt) on c0's stream: LoopStGather over c's own arena (KfRow),
// KfStGatherM over the arenas the rows name (KfRowM)
template <class Row, class At>
static int kf_gather_batch(liliom_ctx* c0, const std::vector<int>& which, At at) {
    if constexpr (std::is_same<Row, KfRow>::value)
        return stage_batch<LoopStGather>(c0, which, [&](LoopEntry& e, int i) {
            const KfGatherAt<KfRow> a = at(i);
            e = LoopEntry{};
            e.arena = (const unsigned char*)a.c->kf_arena.p; e.tab = a.tab; e.rows = a.rows; e.gx = (int)a.grid.x; e.gy = (int)a.grid.y;
            e.stride = a.c->prm.point_stride; e.raw_out = (unsigned char*)a.out;
            return a.c;
        });
    else
        return stage_batch<KfStGatherM>(c0, which, [&](KfGatherMEntry& e, int i) {
            const KfGatherAt<KfRowM> a = at(i);
            e = KfGatherMEntry{a.tab, a.rows, (int)a.grid.x, (int)a.grid.y, a.c->prm.point_stride, (unsigned char*)a.out};
            return a.c;
        });
}

// The entry of voxelgrid_dev's chain at 32-bit keys on c's buffers: n points at `in` -> `out`, the count at `count` (the stages
// LoopStBoxInit .. LoopStCentroidXyzw32; the keyframe store's and the local map's batches run them too)
static LoopEntry vg_chain_entry(liliom_ctx* c, const void* in, int n, float leaf, void* out, int* count) {
    LoopEntry e{};
    e.raw = (const unsigned char*)in; e.n = n; e.stride = c->prm.point_stride; e.leaf = leaf;
    e.mm = c->vg_minmax.as<int>(); e.mm_blocks = box_blocks(e.n, c->sm_count); e.pp = c->vg_params.as<VgParams>();
    e.keys = c->vg_keys.as<uint32_t>(); e.vals = c->vg_vals.as<int>(); e.keys2 = c->vg_keys2.as<uint32_t>(); e.vals2 = c->vg_vals2.as<int>();
    e.flags = c->vg_flags.as<int>(); e.rank = c->vg_rank.as<int>(); e.ds = (unsigned char*)out; e.count = count;
    return e;
}

// Session j's gather of cloud k (0 target, 1 source) and its chain's entry, as loop_cloud's launches take their arguments (the
// repack's output aside: loop_repack_entry)
template <class Row>
static KfGatherAt<Row> loop_gather_at(const LoopJob& j, int k) {
    return KfGatherAt<Row>{j.c, loop_rows<Row>(j, k), j.rows[k], loop_gather_grid(j, k), j.c->bmap_raw.p};
}
static LoopEntry loop_cloud_entry(const LoopJob& j, int k) {
    liliom_ctx* c = j.c;
    return vg_chain_entry(c, c->bmap_raw.p, (int)j.off[k], j.leaf, c->vg_out.p, c->vg_count.as<int>() + k);
}
static LoopEntry loop_repack_entry(const LoopJob& j, int k) {
    LoopEntry e = loop_cloud_entry(j, k);
    e.xyzw = loop_dst(j.c, k);
    return e;
}
// The launches of grid_build over index mi's m points (grid_begin has sized it)
static LoopEntry grid_entry(liliom_ctx* c, MapIndex& mi, int m) {
    LoopEntry e{};
    e.xyzw = mi.xyzw.as<float4>(); e.m = m; e.mm = c->vg_minmax.as<int>(); e.mm_blocks = box_blocks(e.m, c->sm_count);
    e.g = mi.grid; e.gkeys = c->grid_keys.as<uint32_t>(); e.gvals = c->grid_vals.as<int>();
    e.keys2 = c->grid_keys2.as<uint32_t>(); e.vals2 = c->grid_vals2.as<int>(); e.sorted = mi.sorted.as<float4>();
    e.cell_start = mi.cell_start.as<int>();
    return e;
}
// ... the target's cell grid
static LoopEntry loop_grid_entry(const LoopJob& j) { return grid_entry(j.c, j.c->loop, j.m[0]); }

namespace {

template <class St, class Make>
int loop_stage(liliom_ctx* c0, std::vector<LoopJob>& J, const std::vector<int>& which, Make make) {
    return stage_batch<St>(c0, which, [&](LoopEntry& e, int i) { e = make(J[i]); return J[i].c; });
}

// voxelgrid_dev's chain at 32-bit keys (box, parameters, keys, sort, heads, scan, centroids) of the sessions sel() on c0's stream:
// session i's cloud is entry(i) (vg_chain_entry) on ctx(i)'s buffers.  One k_stage_batch launch per stage for up to kBatchMax
// sessions; the library sort and scan per session, in order.  fail(i, rc): session i's sort or scan was not queued (sel() leaves it
// out from then on).
template <class Sel, class Make, class Ctx, class Fail>
int vg_chain_batch(liliom_ctx* c0, Sel sel, Make entry, Ctx ctx, Fail fail) {
    auto stage = [&](auto st, const std::vector<int>& which) -> int {
        return stage_batch<decltype(st)>(c0, which, [&](LoopEntry& e, int i) { e = entry(i); return ctx(i); });
    };
    auto of_kind = [&](bool s48, bool xyzw) {
        std::vector<int> v;
        for (int i : sel()) if ((ctx(i)->prm.point_stride == 48) == s48 && (entry(i).xyzw != nullptr) == xyzw) v.push_back(i);
        return v;
    };
    LILI_TRY(stage(LoopStBoxInit{}, sel()));
    LILI_TRY(stage(LoopStBox{}, sel()));
    LILI_TRY(stage(LoopStParams{}, sel()));
    LILI_TRY(stage(LoopStKeys{}, sel()));
    for (int i : sel()) {
        liliom_ctx* c = ctx(i);
        if (const int rc = sort_pairs_u32(c, c->vg_keys.as<uint32_t>(), c->vg_keys2.as<uint32_t>(), c->vg_vals.as<int>(), c->vg_vals2.as<int>(),
                                          entry(i).n, 32); rc != LILIOM_OK)
            fail(i, rc);
    }
    LILI_TRY(stage(LoopStHeads{}, sel()));
    for (int i : sel()) {
        liliom_ctx* c = ctx(i);
        if (const int rc = exclusive_scan_i32(c, c->vg_flags.as<int>(), c->vg_rank.as<int>(), entry(i).n); rc != LILIOM_OK) fail(i, rc);
    }
    LILI_TRY(stage(LoopStCentroid48{}, of_kind(true, false)));
    LILI_TRY(stage(LoopStCentroid32{}, of_kind(false, false)));
    LILI_TRY(stage(LoopStCentroidXyzw48{}, of_kind(true, true)));
    return stage(LoopStCentroidXyzw32{}, of_kind(false, true));
}

// The shared phases of loop_align_batch, every session's stream pointing at c0's.  Each phase: the solo call's host part per
// session, the stage launches for all of them, every session's read-back words into its own pinned block, ONE synchronise.
// wide[i]: session i's index wrapped in one of its clouds (vg_wide_keys); it leaves the shared path after phase 1.  Row: the
// keyframe tables' row type (KfRow: each session's own store; KfRowM: rows naming their stores).
template <class Row>
int loop_batch_run(liliom_ctx* c0, std::vector<LoopJob>& J, std::vector<char>& live, std::vector<char>& wide, liliom_loop_result* res,
                   int* status) {
    const int B = (int)J.size();
    auto fail = [&](int i, int rc) { status[i] = rc; live[i] = 0; };
    auto sel = [&](auto pred) {
        std::vector<int> v;
        for (int i = 0; i < B; ++i) if (live[i] && pred(J[i])) v.push_back(i);
        return v;
    };
    auto copy_back = [&](int i, size_t at, const void* src, size_t bytes) {
        if (cudaError_t err = cudaMemcpyAsync(J[i].c->h_pin->scratch + at, src, bytes, cudaMemcpyDeviceToHost, c0->stream); err != cudaSuccess)
            fail(i, fail_cuda(J[i].c, err, "loop closure batch: read-back"));
    };
    // 1. both clouds of every session (target, then source: they share bmap_raw, vg_out and the sort chain) -> counts, VgParams
    for (int k = 0; k < 2; ++k) {
        auto has = [k](const LoopJob& j) { return j.off[k] > 0; };
        auto cloud = [k](const LoopJob& j) { return loop_cloud_entry(j, k); };
        LILI_TRY(kf_gather_batch<Row>(c0, sel(has), [&](int i) { return loop_gather_at<Row>(J[i], k); }));
        LILI_TRY(vg_chain_batch(c0, [&] { return sel(has); }, [&](int i) { return cloud(J[i]); }, [&](int i) { return J[i].c; }, fail));
        LILI_TRY(loop_stage<LoopStRepack>(c0, J, sel(has), [k](const LoopJob& j) { return loop_repack_entry(j, k); }));
        for (int i : sel(has)) copy_back(i, k * sizeof(VgParams), J[i].c->vg_params.p, sizeof(VgParams));
    }
    for (int i : sel([](const LoopJob& j) { return j.off[0] > 0 || j.off[1] > 0; }))
        copy_back(i, 2 * sizeof(VgParams), J[i].c->vg_count.p, 2 * sizeof(int));
    LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
    for (int i : sel([](const LoopJob&) { return true; })) {
        const unsigned char* s = J[i].c->h_pin->scratch;
        for (int k = 0; k < 2; ++k) {
            if (J[i].off[k] <= 0) continue;
            VgParams vp;
            memcpy(&vp, s + k * sizeof(VgParams), sizeof(VgParams));
            memcpy(&J[i].m[k], s + 2 * sizeof(VgParams) + k * sizeof(int), sizeof(int));
            if (vg_wide_keys(vp)) { wide[i] = 1; live[i] = 0; }      // the solo path redoes this cloud with wide keys
        }
        if (live[i]) { res[i].n_src = J[i].m[1]; res[i].n_tgt = J[i].m[0]; }
    }
    // 2. the targets' boxes -> every session's cell grid (grid_begin)
    {
        auto has = [](const LoopJob& j) { return j.m[0] > 0; };
        LILI_TRY(loop_stage<LoopStBoxInit>(c0, J, sel(has), loop_grid_entry));
        LILI_TRY(loop_stage<LoopStGridBox>(c0, J, sel(has), loop_grid_entry));
        for (int i : sel(has)) copy_back(i, 0, J[i].c->vg_minmax.p, kBoxInts * sizeof(int));
        LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
        for (int i : sel([](const LoopJob&) { return true; })) {
            LoopJob& j = J[i];
            liliom_ctx* c = j.c;
            int hb[kBoxInts];
            memcpy(hb, c->h_pin->scratch, sizeof(hb));
            const int rc = j.m[0] > 0 ? grid_begin_exact(c, c->loop, loop_cell(c), j.m[0], hb, j.g) : grid_begin(c, c->loop, loop_cell(c), 0, nullptr, j.g);
            if (rc != LILIOM_OK) { fail(i, rc); continue; }
            if (const int rc2 = loop_icp_begin(j); rc2 != LILIOM_OK) fail(i, rc2);
        }
    }
    // 3. the targets' cell grids, the ICP launches -> every session's results
    {
        auto grid = [](const LoopJob& j) { return !j.g.done; };
        LILI_TRY(loop_stage<LoopStCellKeys>(c0, J, sel(grid), loop_grid_entry));
        for (int i : sel(grid)) if (const int rc = grid_sort(J[i].g); rc != LILIOM_OK) fail(i, rc);
        LILI_TRY(loop_stage<LoopStGatherSorted>(c0, J, sel(grid), loop_grid_entry));
        for (int i : sel(grid)) if (const int rc = grid_clear(J[i].g); rc != LILIOM_OK) fail(i, rc);
        LILI_TRY(loop_stage<LoopStRunEnds>(c0, J, sel(grid), loop_grid_entry));
        for (int i : sel(grid)) if (const int rc = grid_scan(J[i].g); rc != LILIOM_OK) fail(i, rc);
        for (int i : sel(grid)) if (const int rc = grid_finish(J[i].g, 0); rc != LILIOM_OK) fail(i, rc);
        std::vector<IcpJob*> jobs;
        for (int i : sel([](const LoopJob& j) { return !j.icp.done; })) jobs.push_back(&J[i].icp);
        LILI_TRY(icp_batch_launch(c0, jobs));
        LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
        for (int i : sel([](const LoopJob&) { return true; })) {
            liliom_loop_result& r = res[i];
            icp_finish(J[i].icp, r.T16, &r.fitness, &r.converged, &r.iters);
            status[i] = LILIOM_OK;
        }
    }
    return LILIOM_OK;
}

}  // namespace

// liliom_loop_align of several sessions.  Shared launches and waits on cs[0]'s stream (the other sessions' streams joined before
// and after with events); every buffer, library sort and scan and host decision stays the session's own, made by the solo
// call's parts from the session's own read-back words.  Row: KfRow, each session's keyframes from its own store (src_stores and
// tgt_stores NULL), or KfRowM, session i's from the stores src_stores[i] / tgt_stores[i] list, whose streams are joined in too.
template <class Row>
int loop_align_batch(liliom_ctx* const* cs, int B, liliom_ctx* const* const* src_stores, const int* const* src_ids,
                     const double* const* src_poses7, const int* k_src, liliom_ctx* const* const* tgt_stores, const int* const* tgt_ids,
                     const double* const* tgt_poses7, const int* k_tgt, const liliom_loop_params* prm, liliom_loop_result* res, int* status) {
    constexpr bool multi = std::is_same<Row, KfRowM>::value;
    auto stores = [](liliom_ctx* const* const* s, int i) { return multi ? s[i] : nullptr; };
    liliom_ctx* c0 = cs[0];
    std::vector<LoopJob> J(B);
    std::vector<char> live(B, 0), wide(B, 0);
    std::vector<std::pair<unsigned long long, unsigned long long>> launches0(B);
    const std::vector<liliom_ctx*> all(cs, cs + B);
    std::vector<liliom_ctx*> joined(all);
    for (int i = 0; i < B; ++i) {
        const liliom_loop_params& p = prm[i];
        launches0[i] = {cs[i]->cnt.launches, cs[i]->cnt.lib_launches};
        status[i] = loop_check<Row>(cs[i], stores(src_stores, i), src_ids[i], src_poses7[i], k_src[i], stores(tgt_stores, i), tgt_ids[i],
                                    tgt_poses7[i], k_tgt[i], p.leaf, p.max_corr_dist, p.max_iter);
        live[i] = status[i] == LILIOM_OK;
        if (multi && live[i]) {
            kf_add_stores(joined, stores(src_stores, i), k_src[i]);
            kf_add_stores(joined, stores(tgt_stores, i), k_tgt[i]);
        }
    }
    LILI_TRY(batch_join_in(c0, joined));
    int rc;
    {
        const BatchStreams on_c0(all, c0->stream);
        for (int i = 0; i < B; ++i) {
            if (!live[i]) continue;
            const liliom_loop_params& p = prm[i];
            status[i] = loop_tables<Row>(cs[i], KfStores{cs[i], stores(src_stores, i)}, src_ids[i], src_poses7[i], k_src[i],
                                         KfStores{cs[i], stores(tgt_stores, i)}, tgt_ids[i], tgt_poses7[i], k_tgt[i], p.leaf, p.max_corr_dist,
                                         p.max_iter, p.trans_eps, p.fit_eps, J[i]);
            live[i] = status[i] == LILIOM_OK;
        }
        rc = loop_batch_run<Row>(c0, J, live, wide, res, status);
        // sessions whose index wrapped finish on their solo path, which takes the wide keys: the whole solo call, its counters
        // counted from where the batch found them (what this call launched for the session is redone there)
        for (int i = 0; rc == LILIOM_OK && i < B; ++i) {
            if (!wide[i]) continue;
            liliom_ctx* c = cs[i];
            c->cnt.launches = launches0[i].first; c->cnt.lib_launches = launches0[i].second;
            const liliom_loop_params& p = prm[i];
            liliom_loop_result& r = res[i];
            if constexpr (multi)
                status[i] = liliom_loop_align_multi(c, src_stores[i], src_ids[i], src_poses7[i], k_src[i], tgt_stores[i], tgt_ids[i], tgt_poses7[i],
                                                    k_tgt[i], p.leaf, p.max_corr_dist, p.max_iter, p.trans_eps, p.fit_eps, r.T16, &r.fitness,
                                                    &r.converged, &r.iters, &r.n_src, &r.n_tgt);
            else
                status[i] = liliom_loop_align(c, src_ids[i], src_poses7[i], k_src[i], tgt_ids[i], tgt_poses7[i], k_tgt[i], p.leaf,
                                              p.max_corr_dist, p.max_iter, p.trans_eps, p.fit_eps, r.T16, &r.fitness, &r.converged, &r.iters,
                                              &r.n_src, &r.n_tgt);
        }
    }
    LILI_TRY(batch_join_out(c0, all));
    return rc;
}

// ---- the keyframe hand-off of several sessions (liliom_kf_add_resident_batch): the solo call's parts per session, the VoxelGrid
// chains of every session in shared launches (vg_chain_batch), three waits for all of them.
namespace {

// Cloud k of session j's source (0 surf, 1 edge, 2 cut / laserCloud) is filtered: the scan half's two, variant 1's full cloud
bool kf_filtered(const KfResJob& j, int k) { return k != 2 || j.bp->variant == 1; }

// ... and its chain's entry, writing where kf_scan_dev / kf_full_dev write: the edge cloud behind the stored points of kf_arena (its
// count in vg_count[0]), the surf cloud into vg_out (vg_count[1]), the full cloud behind those of kf_full (vg_count[0])
LoopEntry kf_cloud_entry(const KfResJob& j, int k) {
    liliom_ctx* c = j.c;
    const size_t stride = (size_t)c->prm.point_stride;
    int* cnt = c->vg_count.as<int>();
    if (k == 1) return vg_chain_entry(c, j.f[1].buf->p, j.m[1], j.bp->edge_leaf, (unsigned char*)c->kf_arena.p + (size_t)c->kf_used * stride, cnt);
    if (k == 0) return vg_chain_entry(c, j.f[0].buf->p, j.m[0], j.bp->surf_leaf, c->vg_out.p, cnt + 1);
    return vg_chain_entry(c, j.f[2].buf->p, j.m[2], j.bp->surf_leaf, (unsigned char*)c->kf_full.p + (size_t)c->kf_full_used * stride, cnt);
}

// The buffers the solo call's filters size, in its order (kf_scan_dev, then voxelgrid_dev per cloud, kf_full_dev)
int kf_res_buffers(const KfResJob& j) {
    liliom_ctx* c = j.c;
    c->n_ds_resident = -1;      // vg_out is rewritten: no scan for liliom_map_update_resident
    LILI_CUDA(c, c->vg_out.ensure((size_t)(j.m[0] > 0 ? j.m[0] : 1) * c->prm.point_stride));
    LILI_CUDA(c, c->vg_count.ensure(16));
    for (int k : {1, 0, 2})
        if (kf_filtered(j, k) && j.m[k] > 0) LILI_TRY(vg_chain_ensure(c, j.m[k], 4));
    return LILIOM_OK;
}

// The shared phases, every backend's stream pointing at c0's.  Session i's read-back words land in its backend's pinned scratch:
// the sizes, then per filtered cloud k its VgParams and count at k * kSlot.  wide[i]: session i's index wrapped in one of its
// clouds (vg_wide_keys); it leaves the shared path after the counts.
int kf_batch_run(liliom_ctx* c0, std::vector<KfResJob>& J, std::vector<char>& live, std::vector<char>& wide, int* status) {
    constexpr size_t kSlot = sizeof(VgParams) + sizeof(int);
    static_assert(3 * kSlot <= sizeof(PinBlock::scratch), "the three clouds' words fit the pinned scratch");
    const int B = (int)J.size();
    auto fail = [&](int i, int rc) { status[i] = rc; live[i] = 0; };
    auto sel = [&](auto pred) {
        std::vector<int> v;
        for (int i = 0; i < B; ++i) if (live[i] && pred(J[i])) v.push_back(i);
        return v;
    };
    auto any = [](const KfResJob&) { return true; };
    auto copy_back = [&](int i, size_t at, const void* src, size_t bytes) {
        if (cudaError_t err = cudaMemcpyAsync(J[i].c->h_pin->scratch + at, src, bytes, cudaMemcpyDeviceToHost, c0->stream); err != cudaSuccess)
            fail(i, fail_cuda(J[i].c, err, "keyframe batch: read-back"));
    };
    // 1. the sizes only on the device (a resident Horizon extraction's): every such source's, one wait; then both arenas
    auto on_device = [](const KfResJob& j) { return j.f[0].d_n != nullptr; };
    for (int i : sel(any))
        for (int k = 0; k < 3; ++k) J[i].m[k] = J[i].f[k].n;
    if (!sel(on_device).empty()) {
        for (int i : sel(on_device))
            for (int k = 0; k < 3; ++k) copy_back(i, k * sizeof(int), J[i].f[k].d_n, sizeof(int));
        LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
        for (int i : sel(on_device)) memcpy(J[i].m, J[i].c->h_pin->scratch, 3 * sizeof(int));
    }
    for (int i : sel(any)) {
        int rc = kf_res_reserve(J[i]);
        if (rc == LILIOM_OK) rc = kf_res_buffers(J[i]);
        if (rc != LILIOM_OK) fail(i, rc);
    }
    // 2. the edge chains, the surf chains, the full chains (variant 1; variant 0 copies the cloud) -> counts, VgParams; one wait
    for (int k : {1, 0, 2}) {
        for (int i : sel([k](const KfResJob& j) { return k != 2 && j.m[k] == 0; }))      // voxelgrid_dev's count of an empty cloud
            if (cudaError_t err = cudaMemsetAsync(kf_cloud_entry(J[i], k).count, 0, sizeof(int), c0->stream); err != cudaSuccess)
                fail(i, fail_cuda(J[i].c, err, "keyframe batch: empty count"));
        auto has = [k](const KfResJob& j) { return kf_filtered(j, k) && j.m[k] > 0; };
        LILI_TRY(vg_chain_batch(c0, [&] { return sel(has); }, [&](int i) { return kf_cloud_entry(J[i], k); }, [&](int i) { return J[i].c; }, fail));
        for (int i : sel(has)) {
            copy_back(i, k * kSlot, J[i].c->vg_params.p, sizeof(VgParams));
            copy_back(i, k * kSlot + sizeof(VgParams), kf_cloud_entry(J[i], k).count, sizeof(int));
        }
    }
    for (int i : sel([](const KfResJob& j) { return !kf_filtered(j, 2) && j.m[2] > 0; })) {      // L:1498-1500 as received
        liliom_ctx* c = J[i].c;
        const size_t stride = (size_t)c->prm.point_stride;
        if (cudaError_t err = cudaMemcpyAsync((unsigned char*)c->kf_full.p + (size_t)c->kf_full_used * stride, J[i].f[2].buf->p,
                                              (size_t)J[i].m[2] * stride, cudaMemcpyDeviceToDevice, c0->stream); err != cudaSuccess)
            fail(i, fail_cuda(c, err, "keyframe batch: full cloud"));
    }
    LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
    for (int i : sel(any)) {
        KfResJob& j = J[i];
        int cnt[3] = {0, 0, j.m[2]};
        for (int k = 0; k < 3; ++k) {
            if (!kf_filtered(j, k) || j.m[k] == 0) continue;
            const unsigned char* s = j.c->h_pin->scratch + k * kSlot;
            VgParams vp;
            memcpy(&vp, s, sizeof(VgParams));
            memcpy(&cnt[k], s + sizeof(VgParams), sizeof(int));
            if (vg_wide_keys(vp)) { wide[i] = 1; live[i] = 0; }       // the solo path redoes the session with wide keys
        }
        j.ms = cnt[0]; j.me = cnt[1]; j.mf = cnt[2];
    }
    // 3. the surf points behind the edge points; one wait
    for (int i : sel(any))
        if (const int rc = kf_surf_behind(J[i].c, J[i].me, J[i].ms); rc != LILIOM_OK) fail(i, rc);
    LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
    return LILIOM_OK;
}

}  // namespace

// liliom_kf_add_resident of several sessions.  Shared launches and waits on cs[0]'s stream (every backend's and source's stream
// joined before, every backend's after, with events); every buffer, library sort and scan and host decision stays the backend's
// own, made by the solo call's parts from the session's own read-back words.  The sources are only read, and every size is read
// before any session writes: the result is that of the solo calls in any order.
int kf_add_resident_batch(liliom_ctx* const* cs, int B, const liliom_backend_params* bps, liliom_ctx* const* srcs, int* kf_id, int* n_edge_ds,
                          int* n_surf_ds, int* n_full_stored, int* status) {
    liliom_ctx* c0 = cs[0];
    std::vector<KfResJob> J(B);
    std::vector<char> live(B, 0), wide(B, 0);
    std::vector<std::pair<unsigned long long, unsigned long long>> launches0(B);
    const std::vector<liliom_ctx*> all(cs, cs + B);
    std::vector<liliom_ctx*> joined(all);
    for (int i = 0; i < B; ++i) {
        launches0[i] = {cs[i]->cnt.launches, cs[i]->cnt.lib_launches};
        status[i] = kf_res_begin(cs[i], bps + i, srcs[i], J[i]);
        live[i] = status[i] == LILIOM_OK;
        if (live[i] && std::find(joined.begin(), joined.end(), srcs[i]) == joined.end()) joined.push_back(srcs[i]);
    }
    LILI_TRY(batch_join_in(c0, joined));
    int rc;
    {
        const BatchStreams on_c0(all, c0->stream);
        rc = kf_batch_run(c0, J, live, wide, status);
        for (int i = 0; rc == LILIOM_OK && i < B; ++i) {
            auto at = [i](int* p) { return p ? p + i : nullptr; };
            if (live[i]) {
                kf_res_finish(J[i], kf_id + i, at(n_edge_ds), at(n_surf_ds), at(n_full_stored));
            } else if (wide[i]) {
                // the whole solo call, which takes the wide keys, its counters counted from where the batch found them
                liliom_ctx* c = cs[i];
                c->cnt.launches = launches0[i].first; c->cnt.lib_launches = launches0[i].second;
                status[i] = liliom_kf_add_resident(c, bps + i, srcs[i], kf_id + i, at(n_edge_ds), at(n_surf_ds), at(n_full_stored));
            }
        }
    }
    LILI_TRY(batch_join_out(c0, all));
    return rc;
}

// ---- the backend local map of several sessions (liliom_bmap_build_batch): the solo call's parts per session, the gather, the
// VoxelGrid chains, the box passes and the cell grids of every session in shared launches, three waits for all of them.
struct BmapReflEntry {
    const unsigned char* pts; int n; float* out;
};
LILI_STAGE(BmapStRefl, BmapReflEntry, 256, stage_blocks(e.n, 256), kf_refl_at(e.pts, e.n, e.out, i))

namespace {

// Session j's entries, as the solo call's launches take their arguments: the gather of its table, layer l's chain (the float4 points
// into bmap[l].xyzw, as voxelgrid_dev's d_feats) and its cell grid
template <class Row>
KfGatherAt<Row> bmap_gather_at(const BmapJob& j) {
    return KfGatherAt<Row>{j.c, j.c->kf_tab.as<Row>(), j.rows, bmap_gather_grid(j), j.c->bmap_raw.p};
}
LoopEntry bmap_layer_entry(const BmapJob& j, int l) {
    liliom_ctx* c = j.c;
    LoopEntry e = vg_chain_entry(c, bmap_in(j, l), (int)j.n[l], bmap_leaf(j, l), c->bmap_ds[l].p, c->vg_count.as<int>() + l);
    e.xyzw = c->bmap[l].xyzw.as<float4>();
    return e;
}
LoopEntry bmap_grid_entry(const BmapJob& j, int l) { return grid_entry(j.c, j.c->bmap[l], j.m[l]); }

// The shared phases, every session's stream pointing at c0's.  Session i's read-back words land in its pinned scratch: per layer l
// its VgParams and count at l * kSlot (phase 1), its grid box at l * kBox (phase 2).  wide[i]: session i's index wrapped in one of
// its layers (vg_wide_keys); it leaves the shared path after phase 1.  Row: the keyframe tables' row type, as in loop_batch_run.
template <class Row>
int bmap_batch_run(liliom_ctx* c0, std::vector<BmapJob>& J, std::vector<char>& live, std::vector<char>& wide, int* status) {
    constexpr size_t kSlot = sizeof(VgParams) + sizeof(int), kBox = kBoxInts * sizeof(int);
    static_assert(2 * kSlot <= sizeof(PinBlock::scratch) && 2 * kBox <= sizeof(PinBlock::scratch), "both layers' words fit the pinned scratch");
    const int B = (int)J.size();
    auto fail = [&](int i, int rc) { status[i] = rc; live[i] = 0; J[i].grid[0] = J[i].grid[1] = false; };
    auto sel = [&](auto pred) {
        std::vector<int> v;
        for (int i = 0; i < B; ++i) if (live[i] && pred(J[i])) v.push_back(i);
        return v;
    };
    auto any = [](const BmapJob&) { return true; };
    auto copy_back = [&](int i, size_t at, const void* src, size_t bytes) {
        if (cudaError_t err = cudaMemcpyAsync(J[i].c->h_pin->scratch + at, src, bytes, cudaMemcpyDeviceToHost, c0->stream); err != cudaSuccess)
            fail(i, fail_cuda(J[i].c, err, "local map batch: read-back"));
    };
    // 1. every table's gather, the edge chains, then the surf chains (they share each session's sort chain) -> counts, VgParams
    LILI_TRY(kf_gather_batch<Row>(c0, sel([](const BmapJob& j) { return j.rows > 0; }), [&](int i) { return bmap_gather_at<Row>(J[i]); }));
    for (int l = 0; l < 2; ++l) {
        for (int i : sel([l](const BmapJob& j) { return j.n[l] == 0; }))      // voxelgrid_dev's count of an empty layer
            if (cudaError_t err = cudaMemsetAsync(J[i].c->vg_count.as<int>() + l, 0, sizeof(int), c0->stream); err != cudaSuccess)
                fail(i, fail_cuda(J[i].c, err, "local map batch: empty count"));
        auto has = [l](const BmapJob& j) { return j.n[l] > 0; };
        LILI_TRY(vg_chain_batch(c0, [&] { return sel(has); }, [&](int i) { return bmap_layer_entry(J[i], l); }, [&](int i) { return J[i].c; }, fail));
        for (int i : sel(has)) {
            copy_back(i, l * kSlot, J[i].c->vg_params.p, sizeof(VgParams));
            copy_back(i, l * kSlot + sizeof(VgParams), J[i].c->vg_count.as<int>() + l, sizeof(int));
        }
    }
    LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
    for (int i : sel(any)) {
        for (int l = 0; l < 2; ++l) {
            if (J[i].n[l] <= 0) continue;
            const unsigned char* s = J[i].c->h_pin->scratch + l * kSlot;
            VgParams vp;
            memcpy(&vp, s, sizeof(VgParams));
            memcpy(&J[i].m[l], s + sizeof(VgParams), sizeof(int));
            if (vg_wide_keys(vp)) { wide[i] = 1; live[i] = 0; }      // the solo path redoes the session with wide keys
        }
    }
    // 2. each layer's box (vg_minmax in stream order) -> both cell grids of every session (grid_begin)
    for (int l = 0; l < 2; ++l) {
        auto has = [l](const BmapJob& j) { return j.m[l] > 0; };
        if (l == 1) for (int i : sel(any)) J[i].launches_surf_box = J[i].c->cnt.launches;
        LILI_TRY(stage_batch<LoopStBoxInit>(c0, sel(has), [&](LoopEntry& e, int i) { e = bmap_grid_entry(J[i], l); return J[i].c; }));
        LILI_TRY(stage_batch<LoopStGridBox>(c0, sel(has), [&](LoopEntry& e, int i) { e = bmap_grid_entry(J[i], l); return J[i].c; }));
        for (int i : sel(has)) copy_back(i, l * kBox, J[i].c->vg_minmax.p, kBox);
    }
    LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
    for (int i : sel(any)) {
        BmapJob& j = J[i];
        liliom_ctx* c = j.c;
        for (int l = 0; l < 2; ++l) {
            int hb[kBoxInts];
            memcpy(hb, c->h_pin->scratch + l * kBox, sizeof(hb));
            const int rc = j.m[l] > 0 ? grid_begin_exact(c, c->bmap[l], bmap_cell(j, l), j.m[l], hb, j.g[l])
                                      : grid_begin(c, c->bmap[l], bmap_cell(j, l), 0, nullptr, j.g[l]);
            if (rc != LILIOM_OK) {
                const bool edge_built = l == 1 && j.grid[0];
                fail(i, rc);
                j.grid[0] = edge_built;           // the solo call builds the edge grid before it meets the surf layer's error
                if (l == 0) c->cnt.launches = j.launches_surf_box;     // ... and never reaches the surf layer's box
                break;
            }
            j.grid[l] = !j.g[l].done;
        }
    }
    // 3. every begun cell grid, edge then surf, then the reflectivity of the 48-byte surf layers; one wait
    for (int l = 0; l < 2; ++l) {
        auto grid = [&]() {
            std::vector<int> v;
            for (int i = 0; i < B; ++i) if (J[i].grid[l]) v.push_back(i);
            return v;
        };
        auto entry = [&](LoopEntry& e, int i) { e = bmap_grid_entry(J[i], l); return J[i].c; };
        LILI_TRY(stage_batch<LoopStCellKeys>(c0, grid(), entry));
        for (int i : grid()) if (const int rc = grid_sort(J[i].g[l]); rc != LILIOM_OK) fail(i, rc);
        LILI_TRY(stage_batch<LoopStGatherSorted>(c0, grid(), entry));
        for (int i : grid()) if (const int rc = grid_clear(J[i].g[l]); rc != LILIOM_OK) fail(i, rc);
        LILI_TRY(stage_batch<LoopStRunEnds>(c0, grid(), entry));
        for (int i : grid()) if (const int rc = grid_scan(J[i].g[l]); rc != LILIOM_OK) fail(i, rc);
        for (int i : grid()) if (const int rc = grid_finish(J[i].g[l], 0); rc != LILIOM_OK) fail(i, rc);
    }
    auto s48 = [](const BmapJob& j) { return j.c->prm.point_stride == 48; };
    for (int i : sel(s48))
        if (cudaError_t err = J[i].c->bmap[1].refl.ensure((size_t)std::max(J[i].m[1], 1) * sizeof(float)); err != cudaSuccess)
            fail(i, fail_cuda(J[i].c, err, "local map batch: reflectivity"));
    LILI_TRY(stage_batch<BmapStRefl>(c0, sel([&](const BmapJob& j) { return s48(j) && j.m[1] > 0; }), [&](BmapReflEntry& e, int i) {
        liliom_ctx* c = J[i].c;
        e = BmapReflEntry{(const unsigned char*)c->bmap_ds[1].p, J[i].m[1], c->bmap[1].refl.as<float>()};
        return c;
    }));
    LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
    return LILIOM_OK;
}

}  // namespace

// liliom_bmap_build of several sessions.  Shared launches and waits on cs[0]'s stream (the other sessions' streams joined before and
// after with events); every buffer, library sort and scan and host decision stays the session's own, made by the solo call's parts
// from the session's own read-back words.  Row: KfRow, each session's keyframes from its own store (stores NULL), or KfRowM,
// session i's from the stores stores[i] lists, whose streams are joined in too.
template <class Row>
int bmap_build_batch(liliom_ctx* const* cs, int B, const liliom_backend_params* bps, liliom_ctx* const* const* stores, const int* const* kf_ids,
                     const double* const* poses7, const int* k, int* n_edge_map, int* n_surf_map, int* status) {
    constexpr bool multi = std::is_same<Row, KfRowM>::value;
    auto stores_of = [stores](int i) { return multi ? stores[i] : nullptr; };
    liliom_ctx* c0 = cs[0];
    std::vector<BmapJob> J(B);
    std::vector<char> live(B, 0), wide(B, 0);
    std::vector<std::pair<unsigned long long, unsigned long long>> launches0(B);
    const std::vector<liliom_ctx*> all(cs, cs + B);
    std::vector<liliom_ctx*> joined(all);
    for (int i = 0; i < B; ++i) {
        launches0[i] = {cs[i]->cnt.launches, cs[i]->cnt.lib_launches};
        status[i] = bmap_check<Row>(cs[i], bps + i, stores_of(i), kf_ids[i], poses7[i], k[i]);
        live[i] = status[i] == LILIOM_OK;
        if (multi && live[i]) kf_add_stores(joined, stores_of(i), k[i]);
    }
    LILI_TRY(batch_join_in(c0, joined));
    int rc;
    {
        const BatchStreams on_c0(all, c0->stream);
        for (int i = 0; i < B; ++i) {
            if (!live[i]) continue;
            status[i] = bmap_tables<Row>(cs[i], bps + i, KfStores{cs[i], stores_of(i)}, kf_ids[i], poses7[i], k[i], J[i]);
            live[i] = status[i] == LILIOM_OK;
        }
        rc = bmap_batch_run<Row>(c0, J, live, wide, status);
        for (int i = 0; rc == LILIOM_OK && i < B; ++i) {
            auto at = [i](int* p) { return p ? p + i : nullptr; };
            if (live[i]) {
                bmap_finish(J[i], at(n_edge_map), at(n_surf_map));
            } else if (wide[i]) {
                // the whole solo call, which takes the wide keys, its counters counted from where the batch found them
                liliom_ctx* c = cs[i];
                c->cnt.launches = launches0[i].first; c->cnt.lib_launches = launches0[i].second;
                if constexpr (multi)
                    status[i] = liliom_bmap_build_multi(c, bps + i, stores[i], kf_ids[i], poses7[i], k[i], at(n_edge_map), at(n_surf_map));
                else
                    status[i] = liliom_bmap_build(c, bps + i, kf_ids[i], poses7[i], k[i], at(n_edge_map), at(n_surf_map));
            }
        }
    }
    LILI_TRY(batch_join_out(c0, all));
    return rc;
}

}  // namespace lili

extern "C" int liliom_loop_align(liliom_ctx* c, const int* src_ids, const double* src_poses7, int k_src, const int* tgt_ids,
                                 const double* tgt_poses7, int k_tgt, float leaf, double max_corr_dist, int max_iter, double trans_eps,
                                 double fit_eps, double T16[16], double* fitness, int* converged, int* iters, int* n_src, int* n_tgt) {
    if (!c || !T16 || !fitness || !converged || !iters) return LILIOM_E_ARG;
    LILI_TRY(loop_check<KfRow>(c, nullptr, src_ids, src_poses7, k_src, nullptr, tgt_ids, tgt_poses7, k_tgt, leaf, max_corr_dist, max_iter));
    LoopJob j;
    LILI_TRY(loop_tables<KfRow>(c, KfStores{c}, src_ids, src_poses7, k_src, KfStores{c}, tgt_ids, tgt_poses7, k_tgt, leaf, max_corr_dist,
                                max_iter, trans_eps, fit_eps, j));
    return loop_run<KfRow>(j, T16, fitness, converged, iters, n_src, n_tgt);
}

extern "C" int liliom_loop_align_batch(liliom_ctx* const* ctxs, int B, const int* const* src_ids, const double* const* src_poses7,
                                       const int* k_src, const int* const* tgt_ids, const double* const* tgt_poses7, const int* k_tgt,
                                       const liliom_loop_params* prm, liliom_loop_result* res, int* status) {
    if (!batch_ctxs_ok(ctxs, B) || !src_ids || !src_poses7 || !k_src || !tgt_ids || !tgt_poses7 || !k_tgt || !prm || !res || !status)
        return LILIOM_E_ARG;
    LILI_CUDA(ctxs[0], cudaSetDevice(ctxs[0]->device));
    return loop_align_batch<KfRow>(ctxs, B, nullptr, src_ids, src_poses7, k_src, nullptr, tgt_ids, tgt_poses7, k_tgt, prm, res, status);
}

extern "C" int liliom_loop_align_batch_multi(liliom_ctx* const* ctxs, int B, liliom_ctx* const* const* src_stores, const int* const* src_ids,
                                             const double* const* src_poses7, const int* k_src, liliom_ctx* const* const* tgt_stores,
                                             const int* const* tgt_ids, const double* const* tgt_poses7, const int* k_tgt,
                                             const liliom_loop_params* prm, liliom_loop_result* res, int* status) {
    if (!batch_ctxs_ok(ctxs, B) || !src_stores || !src_ids || !src_poses7 || !k_src || !tgt_stores || !tgt_ids || !tgt_poses7 || !k_tgt ||
        !prm || !res || !status)
        return LILIOM_E_ARG;
    LILI_CUDA(ctxs[0], cudaSetDevice(ctxs[0]->device));
    return loop_align_batch<KfRowM>(ctxs, B, src_stores, src_ids, src_poses7, k_src, tgt_stores, tgt_ids, tgt_poses7, k_tgt, prm, res, status);
}

extern "C" int liliom_kf_add_resident_batch(liliom_ctx* const* ctxs, int B, const liliom_backend_params* bps, liliom_ctx* const* srcs,
                                            int* kf_id, int* n_edge_ds, int* n_surf_ds, int* n_full_stored, int* status) {
    if (!batch_ctxs_ok(ctxs, B) || !bps || !srcs || !kf_id || !status) return LILIOM_E_ARG;
    LILI_CUDA(ctxs[0], cudaSetDevice(ctxs[0]->device));
    return kf_add_resident_batch(ctxs, B, bps, srcs, kf_id, n_edge_ds, n_surf_ds, n_full_stored, status);
}

extern "C" int liliom_bmap_build_batch(liliom_ctx* const* ctxs, int B, const liliom_backend_params* bps, const int* const* kf_ids,
                                       const double* const* poses7, const int* k, int* n_edge_map, int* n_surf_map, int* status) {
    if (!batch_ctxs_ok(ctxs, B) || !bps || !kf_ids || !poses7 || !k || !status) return LILIOM_E_ARG;
    LILI_CUDA(ctxs[0], cudaSetDevice(ctxs[0]->device));
    return bmap_build_batch<KfRow>(ctxs, B, bps, nullptr, kf_ids, poses7, k, n_edge_map, n_surf_map, status);
}

extern "C" int liliom_bmap_build_batch_multi(liliom_ctx* const* ctxs, int B, const liliom_backend_params* bps, liliom_ctx* const* const* stores,
                                             const int* const* kf_ids, const double* const* poses7, const int* k, int* n_edge_map,
                                             int* n_surf_map, int* status) {
    if (!batch_ctxs_ok(ctxs, B) || !bps || !stores || !kf_ids || !poses7 || !k || !status) return LILIOM_E_ARG;
    LILI_CUDA(ctxs[0], cudaSetDevice(ctxs[0]->device));
    return bmap_build_batch<KfRowM>(ctxs, B, bps, stores, kf_ids, poses7, k, n_edge_map, n_surf_map, status);
}

extern "C" int liliom_kf_add_full(liliom_ctx* c, const liliom_backend_params* bp, int kf_id, const void* full, int n, int* n_stored) {
    if (!c || !bp || n < 0 || (n > 0 && !full)) return LILIOM_E_ARG;
    LILI_TRY(backend_check(c, bp));
    if (!kf_ids_ok(c, &kf_id, 1)) return LILIOM_E_ARG;
    if (c->kfs[kf_id].n_full >= 0) {
        c->last_error = "keyframe " + std::to_string(kf_id) + " already has its full cloud";
        return LILIOM_E_ARG;
    }
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    LILI_TRY(kf_reserve(c, c->kf_full, c->kf_full_used, c->kf_full_used + n));     // VoxelGrid never outputs more points than it reads
    const void* in = full;                                        // variant 0 copies the host cloud straight into the arena
    if (n > 0 && bp->variant == 1) {                              // variant 1 filters it on the device
        LILI_CUDA(c, c->raw.ensure((size_t)n * stride));
        LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, full, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream));
        in = c->raw.p;
    }
    int m = 0;
    LILI_TRY(kf_full_dev(c, bp, in, n, &m));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    kf_push_full(c, kf_id, m);
    if (n_stored) *n_stored = m;
    return LILIOM_OK;
}

namespace lili {

// Every listed keyframe of kind LILIOM_KF_FULL has its full cloud (ids known to their stores)
static bool kf_full_ok(liliom_ctx* c, KfStores s, int kind, const int* kf_ids, int k) {
    for (int i = 0; i < k && kind == LILIOM_KF_FULL; ++i)
        if (s[i]->kfs[kf_ids[i]].n_full < 0) {
            c->last_error = "keyframe " + std::to_string(kf_ids[i]) + " has no full cloud (liliom_kf_add_full)";
            if (s.per) c->last_error += " in store " + std::to_string(i);
            return false;
        }
    return true;
}

// The global map's table (:2652-2662 list order, one cloud per keyframe): the stored cloud of `kind` of every entry, transformed by
// pre7s + pre_step * i (none when pre7s is null; pre_step 0: one for every entry) and then by its pose.  Returns the points.
template <class Row>
static long long gmap_rows(KfStores s, int kind, const int* kf_ids, const double* poses7, int k, const double* pre7s, size_t pre_step,
                           std::vector<Row>& tab, long long* largest) {
    long long N = 0;
    *largest = 0;
    for (int i = 0; i < k; ++i) {
        const KfEntry& f = s[i]->kfs[kf_ids[i]];
        const DevBuf& arena = kind == LILIOM_KF_FULL ? s[i]->kf_full : s[i]->kf_arena;
        const long long off = kind == LILIOM_KF_FULL ? f.full_off : f.surf_off;
        const int m = kind == LILIOM_KF_FULL ? f.n_full : f.n_surf;
        if (m) tab.push_back(kf_row_in<Row>(arena.p, off, N, m, poses7 + 7 * (size_t)i, pre7s ? pre7s + pre_step * i : nullptr));
        N += m;
        *largest = std::max(*largest, (long long)m);
    }
    return N;
}

// The global map without a concatenation buffer: box, voxel keys and centroids read the stored clouds through the keyframe table
// and transform every point on load (kf_table.h); the sort chain in between is voxelgrid_dev's (the sort at the key width of the
// box, k_vg_heads, the scan).  Device memory: the table, 16 bytes per listed point for keys and values (sort included; 24 with
// the wide keys), and
// the output; only PCL's declined case writes the transformed concatenation, which is then the output.
// arena: the store KfRow rows read (KfRowM rows name their own); N <= 2^31 - 1 points (kf_points_ok).
template <class Row>
static int gmap_run(liliom_ctx* c, const unsigned char* arena, const std::vector<Row>& tab, long long N, long long largest, float leaf,
                    void* out, int cap, int* n) {
    if (N == 0) { *n = 0; return LILIOM_OK; }
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    const int rows = (int)tab.size();
    LILI_TRY(kf_upload_table(c, tab));
    const Row* d_tab = c->kf_tab.as<Row>();
    // box of the transformed concatenation (pcl::getMinMax3D), read back: the overflow test and the key width are decided here
    LILI_CUDA(c, c->vg_minmax.ensure(8 * sizeof(int)));
    int* mm = c->vg_minmax.as<int>();
    int* empty = reinterpret_cast<int*>(c->h_pin->scratch);       // pinned staging of the empty box; the stream orders the read-back after it
    for (int w = 0; w < kBoxInts; ++w) empty[w] = vg_box_empty(w);
    LILI_CUDA(c, cudaMemcpyAsync(mm, empty, kBoxInts * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    KfKern<Row>::box<<<kf_row_grid(tab.size(), largest, 8, 1024), 256, 0, c->stream>>>(arena, d_tab, rows, stride, mm);
    LILI_TRY(launch_check(c, "k_kf_box"));
    int box[kBoxInts];
    LILI_TRY(read_back(c, {{box, mm, sizeof(box)}}));
    const VgParams p = vg_params(box, leaf);
    if (p.overflow)                                               // PCL declines the filter and publishes its input
        return download_sized(c, c->vg_out, (int)N, stride, out, cap, n, [&]() -> int {
            c->n_ds_resident = -1;      // vg_out is rewritten: no scan for liliom_map_update_resident
            LILI_CUDA(c, c->vg_out.ensure((size_t)N * stride));
            return kf_gather(c, arena, tab, largest, c->vg_out.p);
        });
    const int n_fin = p.n_finite;
    if (n_fin == 0) { *n = 0; return LILIOM_OK; }
    const int key_bits = vg_chain_key_bits(box, leaf);            // the wide keys (64-bit) when the index wraps
    const size_t kb = key_bits > 32 ? 8 : 4;
    LILI_CUDA(c, c->vg_keys.ensure((size_t)N * kb));
    LILI_CUDA(c, c->vg_vals.ensure((size_t)N * 4));
    LILI_CUDA(c, c->vg_keys2.ensure((size_t)N * kb));
    LILI_CUDA(c, c->vg_vals2.ensure((size_t)N * 4));
    LILI_CUDA(c, c->vg_flags.ensure(((size_t)n_fin + 2) * 4));
    LILI_CUDA(c, c->vg_rank.ensure(((size_t)n_fin + 2) * 4));
    auto chain = [&](auto* keys, auto* keys2) -> int {
        using K = std::remove_pointer_t<decltype(keys)>;
        const auto k_keys = KfKern<Row>::template keys<K>;
        k_keys<<<kf_row_grid(tab.size(), largest, 8), 256, 0, c->stream>>>(arena, d_tab, rows, stride, p, keys, c->vg_vals.as<int>());
        LILI_TRY(launch_check(c, "k_kf_keys"));
        // non-finite points carry the sentinel key and sort last: the first n_fin sorted entries are the finite points
        if constexpr (sizeof(K) == 4) LILI_TRY(sort_pairs_u32(c, keys, keys2, c->vg_vals.as<int>(), c->vg_vals2.as<int>(), (int)N, key_bits));
        else LILI_TRY(sort_pairs_u64(c, keys, keys2, c->vg_vals.as<int>(), c->vg_vals2.as<int>(), (int)N, key_bits));
        k_vg_heads<<<cdiv(n_fin + 1LL, 256), 256, 0, c->stream>>>(keys2, n_fin, nullptr, c->vg_flags.as<int>());
        LILI_TRY(launch_check(c, "k_vg_heads"));
        LILI_TRY(exclusive_scan_i32(c, c->vg_flags.as<int>(), c->vg_rank.as<int>(), n_fin));
        int m = 0;
        LILI_TRY(read_back(c, {{&m, c->vg_rank.as<int>() + n_fin, sizeof(int)}}));
        return download_sized(c, c->vg_out, m, stride, out, cap, n, [&]() -> int {
            c->n_ds_resident = -1;      // vg_out is rewritten: no scan for liliom_map_update_resident
            LILI_CUDA(c, c->vg_out.ensure((size_t)m * stride));
            const auto k_centroid = stride == 48 ? KfKern<Row>::template centroid<48, K> : KfKern<Row>::template centroid<32, K>;
            k_centroid<<<cdiv(n_fin, 128), 128, 0, c->stream>>>(arena, d_tab, rows, keys2, c->vg_vals2.as<int>(), c->vg_flags.as<int>(),
                                                                c->vg_rank.as<int>(), n_fin, (unsigned char*)c->vg_out.p);
            return launch_check(c, "k_kf_centroid");
        });
    };
    if (key_bits > 32) return chain(c->vg_keys.as<unsigned long long>(), c->vg_keys2.as<unsigned long long>());
    return chain(c->vg_keys.as<uint32_t>(), c->vg_keys2.as<uint32_t>());
}

}  // namespace lili

extern "C" int liliom_global_map(liliom_ctx* c, int kind, const int* kf_ids, const double* poses7, int k, const double pre7[7],
                                 float leaf, void* out, int cap, int* n) {
    if (!c || !n || k < 0 || (k > 0 && (!kf_ids || !poses7)) || (kind != LILIOM_KF_FULL && kind != LILIOM_KF_SURF) || !(leaf > 0))
        return LILIOM_E_ARG;
    LILI_TRY(backend_check(c, nullptr));
    if (!kf_ids_ok(c, kf_ids, k) || !kf_full_ok(c, KfStores{c}, kind, kf_ids, k)) return LILIOM_E_ARG;
    std::vector<KfRow> tab;
    long long largest = 0;
    const long long N = gmap_rows(KfStores{c}, kind, kf_ids, poses7, k, pre7, 0, tab, &largest);
    LILI_TRY(kf_points_ok(c, N));
    const unsigned char* arena = (const unsigned char*)(kind == LILIOM_KF_FULL ? c->kf_full.p : c->kf_arena.p);
    return gmap_run(c, arena, tab, N, largest, leaf, out, cap, n);
}

// liliom_global_map over keyframes of several stores: rows that name their store's arena, the rest unchanged on c
extern "C" int liliom_global_map_multi(liliom_ctx* c, int kind, liliom_ctx* const* stores, const int* kf_ids, const double* poses7, int k,
                                       const double* pre7s, float leaf, void* out, int cap, int* n) {
    if (!c || !n || k < 0 || (k > 0 && (!stores || !kf_ids || !poses7)) || (kind != LILIOM_KF_FULL && kind != LILIOM_KF_SURF) || !(leaf > 0))
        return LILIOM_E_ARG;
    LILI_TRY(backend_check(c, nullptr));
    if (!kf_stores_ok(c, stores, kf_ids, k) || !kf_full_ok(c, KfStores{c, stores}, kind, kf_ids, k)) return LILIOM_E_ARG;
    std::vector<KfRowM> tab;
    long long largest = 0;
    const long long N = gmap_rows(KfStores{c, stores}, kind, kf_ids, poses7, k, pre7s, 7, tab, &largest);
    LILI_TRY(kf_points_ok(c, N));
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_TRY(kf_join_stores(c, {{stores, k}}));
    return gmap_run(c, (const unsigned char*)c->kf_arena.p, tab, N, largest, leaf, out, cap, n);
}

// liliom_loop_align over keyframes of several stores: both clouds' rows name their store's arena, the rest unchanged on c
extern "C" int liliom_loop_align_multi(liliom_ctx* c, liliom_ctx* const* src_stores, const int* src_ids, const double* src_poses7, int k_src,
                                       liliom_ctx* const* tgt_stores, const int* tgt_ids, const double* tgt_poses7, int k_tgt, float leaf,
                                       double max_corr_dist, int max_iter, double trans_eps, double fit_eps, double T16[16], double* fitness,
                                       int* converged, int* iters, int* n_src, int* n_tgt) {
    if (!c || !T16 || !fitness || !converged || !iters) return LILIOM_E_ARG;
    LILI_TRY(loop_check<KfRowM>(c, src_stores, src_ids, src_poses7, k_src, tgt_stores, tgt_ids, tgt_poses7, k_tgt, leaf, max_corr_dist,
                                max_iter));
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_TRY(kf_join_stores(c, {{src_stores, k_src}, {tgt_stores, k_tgt}}));
    LoopJob j;
    LILI_TRY(loop_tables<KfRowM>(c, KfStores{c, src_stores}, src_ids, src_poses7, k_src, KfStores{c, tgt_stores}, tgt_ids, tgt_poses7, k_tgt,
                                 leaf, max_corr_dist, max_iter, trans_eps, fit_eps, j));
    return loop_run<KfRowM>(j, T16, fitness, converged, iters, n_src, n_tgt);
}
