// SURVEY.md §8 (f5): the backend's keyframe clouds and local map on the device.
//   keyframe store   BackendFusion::downSampleCloud, scan half (L/src/BackendFusion.cpp:1502-1514) + the clouds of
//                    saveKeyFramesAndFactors (:1688-1695): VoxelGrid of the received body-frame clouds, appended to one arena
//   local map        buildLocalMapWithLandMark (:1387-1484) + downSampleCloud, map half (:1486-1492): transform + concatenate
//                    the listed keyframes in ONE launch, VoxelGrid per layer, a cell grid per layer (MapIndex)
//   loop closure     detectLoopClosure's clouds (:2473-2547): edge then surf per keyframe, transformed, VoxelGrid; with
//                    performLoopClosure's ICP (:2552-2582) on them in the same call (liliom_loop_align)
//   full clouds      downSampleCloud, full-cloud half (:1494-1500; R:1373-1376): the /full_point_cloud of a keyframe, stored
//   global map       publishCompleteMap (:2644-2685) and save_pcd's map (:2703-2718): listed keyframes transformed, concatenated,
//                    VoxelGrid, in a VoxelGrid that reads the store through the keyframe table (kf_table.h): no concatenation
// The deque policy of the local map (:1407-1477) stays with the caller: every call lists the keyframes and the poses to use.
// Compiled with --fmad=false (the VoxelGrid centroids and the transform are bit-exact with the reference's arithmetic).
#include "ctx.cuh"
#include "dev_math.cuh"
#include "kf_table.h"

namespace lili {

// The table kernels: blockIdx.y walks the rows (grid-strided past 65535 rows), the blocks of a row stream through its points.
// The table lives in device memory, so one launch serves any number of keyframes (the odometry map's ConcatTab holds 64).
static dim3 kf_row_grid(size_t rows, long long largest, int bx_max, int by_max = 65535) {
    return dim3(std::max(1, std::min(cdiv(largest, 256), bx_max)), (unsigned)std::min<size_t>(rows, by_max));
}

// the transformed concatenation of the rows
__global__ void k_kf_gather(const unsigned char* __restrict__ arena, const KfRow* __restrict__ tab, int rows, int stride,
                            unsigned char* __restrict__ out) {
    for (int y = blockIdx.y; y < rows; y += gridDim.y) {
        const KfRow& r = tab[y];
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < r.n; i += gridDim.x * blockDim.x)
            kf_row_point(r, arena + (size_t)(r.src_off + i) * stride, stride, out + (size_t)(r.dst_off + i) * stride);
    }
}

// box (vg_box.h) of the finite transformed points of the rows, joined into mm
__global__ void k_kf_box(const unsigned char* __restrict__ arena, const KfRow* __restrict__ tab, int rows, int stride, int* __restrict__ mm) {
    int box[kBoxInts];
#pragma unroll
    for (int k = 0; k < kBoxInts; ++k) box[k] = vg_box_empty(k);
    for (int y = blockIdx.y; y < rows; y += gridDim.y) {
        const KfRow& r = tab[y];
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < r.n; i += gridDim.x * blockDim.x) {
            const VgXyz p = kf_row_xyz(r, arena + (size_t)(r.src_off + i) * stride);
            if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) vg_box_add(box, p.x, p.y, p.z);
        }
    }
    vg_box_commit(box, mm);
}

// PCL's relative voxel index of every transformed point (all-ones: not finite), value = its index in the concatenation
__global__ void k_kf_keys(const unsigned char* __restrict__ arena, const KfRow* __restrict__ tab, int rows, int stride, const VgParams p,
                          uint32_t* __restrict__ keys, int* __restrict__ vals) {
    for (int y = blockIdx.y; y < rows; y += gridDim.y) {
        const KfRow& r = tab[y];
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < r.n; i += gridDim.x * blockDim.x) {
            const VgXyz x = kf_row_xyz(r, arena + (size_t)(r.src_off + i) * stride);
            const long long d = r.dst_off + i;
            keys[d] = (isfinite(x.x) && isfinite(x.y) && isfinite(x.z)) ? vg_rel_index(p, x.x, x.y, x.z) : 0xffffffffu;
            vals[d] = (int)d;
        }
    }
}

// centroid of every voxel of the sorted keys (the first n_fin entries are the finite points), members transformed on load
template <int STRIDE>
__global__ void k_kf_centroid(const unsigned char* __restrict__ arena, const KfRow* __restrict__ tab, int rows, const uint32_t* __restrict__ keys,
                              const int* __restrict__ vals, const int* __restrict__ flags, const int* __restrict__ rank, int n_fin,
                              unsigned char* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_fin || !flags[i]) return;
    const VgAcc<STRIDE> a = vg_walk<STRIDE>(keys, i, n_fin, [&](int j) { return vals[j]; }, KfRowLoader<STRIDE>{arena, tab, rows});
    vg_write<STRIDE>(a.s, a.n, out + (size_t)rank[i] * STRIDE);
}

// reflectivity (curvature = 0.1 * reflectivity, L/src/FormatConvert.cpp:21) of 48-byte points
__global__ void k_kf_refl(const unsigned char* __restrict__ pts, int n, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = reinterpret_cast<const float*>(pts + (size_t)i * 48)[9];
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

static int kf_upload_table(liliom_ctx* c, const std::vector<KfRow>& tab) {
    LILI_CUDA(c, c->kf_tab.ensure(tab.size() * sizeof(KfRow)));
    LILI_CUDA(c, cudaMemcpyAsync(c->kf_tab.p, tab.data(), tab.size() * sizeof(KfRow), cudaMemcpyHostToDevice, c->stream));
    return LILIOM_OK;
}

// Transform + concatenate rows of `arena` into `out` (one launch).
static int kf_gather(liliom_ctx* c, const void* arena, const std::vector<KfRow>& tab, long long largest, void* out) {
    if (tab.empty() || largest <= 0) return LILIOM_OK;
    LILI_TRY(kf_upload_table(c, tab));
    k_kf_gather<<<kf_row_grid(tab.size(), largest, c->sm_count * 4), 256, 0, c->stream>>>(
        (const unsigned char*)arena, c->kf_tab.as<KfRow>(), (int)tab.size(), c->prm.point_stride, (unsigned char*)out);
    return launch_check(c, "k_kf_gather");
}

// a table row: n points from src -> dst, transformed by pre7 (optional) and then by pose7
static KfRow kf_row(long long src, long long dst, int n, const double* pose7, const double* pre7 = nullptr) {
    KfRow e{};
    e.src_off = src; e.dst_off = dst; e.n = n;
    e.q = Q4{pose7[0], pose7[1], pose7[2], pose7[3]};
    e.t = D3{pose7[4], pose7[5], pose7[6]};
    if (pre7) {
        e.pre = 1;
        e.pq = Q4{pre7[0], pre7[1], pre7[2], pre7[3]};
        e.pt = D3{pre7[4], pre7[5], pre7[6]};
    }
    return e;
}

// detectLoopClosure's cloud of the listed keyframes (:2476-2497, :2502-2547): edge then surf of each, transformed by its pose,
// concatenated into bmap_raw (one launch), VoxelGrid(leaf) into vg_out with its count at d_count (device).  *n_in: the points
// read (0: nothing was launched and d_count is not written).
static int kf_cloud_dev(liliom_ctx* c, const int* kf_ids, const double* poses7, int k, float leaf, int* d_count, long long* n_in) {
    const int stride = c->prm.point_stride;
    std::vector<KfRow> tab;
    long long off = 0, largest = 0;
    for (int i = 0; i < k; ++i) {                                 // :2492-2493 / :2519-2520: *edge_frames[i] then *surf_frames[i]
        const KfEntry& f = c->kfs[kf_ids[i]];
        if (f.n_edge) tab.push_back(kf_row(f.edge_off, off, f.n_edge, poses7 + 7 * (size_t)i));
        off += f.n_edge;
        if (f.n_surf) tab.push_back(kf_row(f.surf_off, off, f.n_surf, poses7 + 7 * (size_t)i));
        off += f.n_surf;
        largest = std::max(largest, (long long)std::max(f.n_edge, f.n_surf));
    }
    *n_in = off;
    if (off == 0) return LILIOM_OK;
    LILI_CUDA(c, c->bmap_raw.ensure((size_t)off * stride));      // scratch: the local map's layers live in bmap_ds / bmap
    LILI_CUDA(c, c->vg_out.ensure((size_t)off * stride));
    LILI_TRY(kf_gather(c, c->kf_arena.p, tab, largest, c->bmap_raw.p));
    return voxelgrid_dev(c, c->bmap_raw.p, (int)off, nullptr, stride, leaf, c->vg_out.p, d_count);
}

static int backend_check(liliom_ctx* c, const liliom_backend_params* bp) {
    if (c->nranks > 1) { c->last_error = "the backend keyframe store is single-GPU"; return LILIOM_E_ARG; }
    if (bp && (!(bp->edge_leaf > 0) || !(bp->surf_leaf > 0) || !(bp->kd_max_radius > 0) || (bp->variant != 0 && bp->variant != 1)))
        return LILIOM_E_ARG;
    return LILIOM_OK;
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
    LILI_CUDA(c, c->vg_out.ensure((size_t)(n_surf > 0 ? n_surf : 1) * stride));
    LILI_CUDA(c, c->vg_count.ensure(16));
    unsigned char* raw = (unsigned char*)c->raw.p;
    if (n_edge) LILI_CUDA(c, cudaMemcpyAsync(raw, edge_last, (size_t)n_edge * stride, cudaMemcpyHostToDevice, c->stream));
    if (n_surf) LILI_CUDA(c, cudaMemcpyAsync(raw + (size_t)n_edge * stride, surf_last, (size_t)n_surf * stride, cudaMemcpyHostToDevice, c->stream));
    unsigned char* tail = (unsigned char*)c->kf_arena.p + (size_t)c->kf_used * stride;
    int* cnt = c->vg_count.as<int>();
    LILI_TRY(voxelgrid_dev(c, raw, n_edge, nullptr, stride, bp->edge_leaf, tail, cnt));                                           // :1502-1507
    LILI_TRY(voxelgrid_dev(c, raw + (size_t)n_edge * stride, n_surf, nullptr, stride, bp->surf_leaf, c->vg_out.p, cnt + 1));     // :1509-1514
    int m[2];
    LILI_TRY(read_back(c, {{m, cnt, sizeof(m)}}));
    const int me = m[0], ms = m[1];
    if (n_edge_ds) *n_edge_ds = me;
    if (n_surf_ds) *n_surf_ds = ms;
    if ((edge_ds_out && me > edge_cap) || (surf_ds_out && ms > surf_cap)) return LILIOM_E_CAPACITY;   // nothing stored
    if (ms) LILI_CUDA(c, cudaMemcpyAsync(tail + (size_t)me * stride, c->vg_out.p, (size_t)ms * stride, cudaMemcpyDeviceToDevice, c->stream));
    if (edge_ds_out && me) LILI_CUDA(c, cudaMemcpyAsync(edge_ds_out, tail, (size_t)me * stride, cudaMemcpyDeviceToHost, c->stream));
    if (surf_ds_out && ms) LILI_CUDA(c, cudaMemcpyAsync(surf_ds_out, c->vg_out.p, (size_t)ms * stride, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    c->kfs.push_back(KfEntry{c->kf_used, c->kf_used + me, me, ms});
    c->kf_used += (long long)me + ms;
    *kf_id = (int)c->kfs.size() - 1;
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

extern "C" int liliom_bmap_build(liliom_ctx* c, const liliom_backend_params* bp, const int* kf_ids, const double* poses7, int k,
                                 int* n_edge_map, int* n_surf_map) {
    if (!c || !bp || k < 0 || (k > 0 && (!kf_ids || !poses7))) return LILIOM_E_ARG;
    LILI_TRY(backend_check(c, bp));
    if (!kf_ids_ok(c, kf_ids, k)) return LILIOM_E_ARG;           // before anything changes: the previous layers stay
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    c->bmap_built = false;
    long long E = 0, S = 0, largest = 0;
    for (int i = 0; i < k; ++i) { const KfEntry& f = c->kfs[kf_ids[i]]; E += f.n_edge; S += f.n_surf; largest = std::max(largest, (long long)std::max(f.n_edge, f.n_surf)); }
    std::vector<KfRow> tab;
    tab.reserve(2 * (size_t)k);
    long long de = 0, ds = E;
    for (int i = 0; i < k; ++i) {                                 // :1479-1483 edge and surf layers, list order
        const KfEntry& f = c->kfs[kf_ids[i]];
        if (f.n_edge) tab.push_back(kf_row(f.edge_off, de, f.n_edge, poses7 + 7 * (size_t)i));
        if (f.n_surf) tab.push_back(kf_row(f.surf_off, ds, f.n_surf, poses7 + 7 * (size_t)i));
        de += f.n_edge; ds += f.n_surf;
    }
    LILI_CUDA(c, c->bmap_raw.ensure((size_t)std::max(E + S, 1LL) * stride));
    LILI_TRY(kf_gather(c, c->kf_arena.p, tab, largest, c->bmap_raw.p));
    const long long nl[2] = {E, S};
    const float leaf[2] = {bp->edge_leaf, bp->surf_leaf};
    const unsigned char* src[2] = {(const unsigned char*)c->bmap_raw.p, (const unsigned char*)c->bmap_raw.p + (size_t)E * stride};
    LILI_CUDA(c, c->vg_count.ensure(16));
    int* cnt = c->vg_count.as<int>();
    for (int l = 0; l < 2; ++l) {                                 // :1486-1492; the centroid kernel also writes the float4 points
        LILI_CUDA(c, c->bmap_ds[l].ensure((size_t)std::max(nl[l], 1LL) * stride));
        LILI_CUDA(c, c->bmap[l].xyzw.ensure((size_t)std::max(nl[l], 1LL) * sizeof(float4)));
        LILI_TRY(voxelgrid_dev(c, src[l], (int)nl[l], nullptr, stride, leaf[l], c->bmap_ds[l].p, cnt + l, c->bmap[l].xyzw.as<float4>()));
    }
    int m[2];
    LILI_TRY(read_back(c, {{m, cnt, sizeof(m)}}));
    LILI_TRY(grid_build(c, c->bmap[0], gate_cell(1.0), m[0]));                 // :1543 sqdist[4] < 1.0
    LILI_TRY(grid_build(c, c->bmap[1], gate_cell(bp->kd_max_radius), m[1]));   // :1615 sqdist[4] < kd_max_radius
    if (stride == 48) {                                                         // reflectivity of the surf layer (:1617-1638)
        LILI_CUDA(c, c->bmap[1].refl.ensure((size_t)std::max(m[1], 1) * sizeof(float)));
        if (m[1] > 0) {
            k_kf_refl<<<cdiv(m[1], 256), 256, 0, c->stream>>>((const unsigned char*)c->bmap_ds[1].p, m[1], c->bmap[1].refl.as<float>());
            LILI_TRY(launch_check(c, "k_kf_refl"));
        }
    }
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    c->bmap_n[0] = m[0]; c->bmap_n[1] = m[1];
    c->bmap_built = true;
    if (n_edge_map) *n_edge_map = m[0];
    if (n_surf_map) *n_surf_map = m[1];
    return LILIOM_OK;
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
    LILI_TRY(kf_cloud_dev(c, kf_ids, poses7, k, leaf, c->vg_count.as<int>(), &off));
    if (off == 0) return LILIOM_OK;
    int m = 0;
    LILI_TRY(read_back(c, {{&m, c->vg_count.p, sizeof(int)}}));
    return download_sized(c, c->vg_out, m, stride, out, cap, n_out);
}

// detectLoopClosure + performLoopClosure's alignment (:2473-2582) without leaving the device: the history cloud goes into the
// loop index (its own cell grid: the odometry map, the local map and every resident correspondence stay), the latest cloud into
// loop_src, and the ICP runs on them (icp.cu).  Scratch shared with the other calls: bmap_raw, vg_out, the sort chain, grid_keys*,
// partials.  Two stream synchronises: the cloud sizes (the grid build needs the target's on the host), and the grid's box.
extern "C" int liliom_loop_align(liliom_ctx* c, const int* src_ids, const double* src_poses7, int k_src, const int* tgt_ids,
                                 const double* tgt_poses7, int k_tgt, float leaf, double max_corr_dist, int max_iter, double trans_eps,
                                 double fit_eps, double T16[16], double* fitness, int* converged, int* iters, int* n_src, int* n_tgt) {
    if (!c || k_src < 0 || k_tgt < 0 || (k_src > 0 && (!src_ids || !src_poses7)) || (k_tgt > 0 && (!tgt_ids || !tgt_poses7)) ||
        !(leaf > 0) || !(max_corr_dist > 0) || max_iter < 1 || !T16 || !fitness || !converged || !iters)
        return LILIOM_E_ARG;
    LILI_TRY(backend_check(c, nullptr));
    if (!kf_ids_ok(c, src_ids, k_src) || !kf_ids_ok(c, tgt_ids, k_tgt)) return LILIOM_E_ARG;     // before anything changes
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    LILI_CUDA(c, c->vg_count.ensure(16));
    int* cnt = c->vg_count.as<int>();
    long long off_t = 0, off_s = 0;
    // :2502-2547 his_key_frames_ds -> the loop index's points (float4, w = index), as liliom_icp_align installs a target
    LILI_TRY(kf_cloud_dev(c, tgt_ids, tgt_poses7, k_tgt, leaf, cnt, &off_t));
    LILI_CUDA(c, c->loop.xyzw.ensure((size_t)std::max(off_t, 1LL) * sizeof(float4)));
    LILI_TRY(repack_to_f4(c, c->vg_out.p, (int)off_t, stride, c->loop.xyzw.as<float4>(), cnt));
    // :2476-2497 latest_key_frames_ds -> the source
    LILI_TRY(kf_cloud_dev(c, src_ids, src_poses7, k_src, leaf, cnt + 1, &off_s));
    LILI_CUDA(c, c->loop_src.ensure((size_t)std::max(off_s, 1LL) * sizeof(float4)));
    LILI_TRY(repack_to_f4(c, c->vg_out.p, (int)off_s, stride, c->loop_src.as<float4>(), cnt + 1));
    int m[2];
    LILI_TRY(read_back(c, {{m, cnt, sizeof(m)}}));
    const int m_t = off_t ? m[0] : 0, m_s = off_s ? m[1] : 0;
    if (n_src) *n_src = m_s;
    if (n_tgt) *n_tgt = m_t;
    LILI_TRY(grid_build(c, c->loop, gate_cell(c->prm.knn_max_sqdist), m_t));      // the cell of liliom_icp_align's target
    return icp_align(c, c->loop, c->loop_src.as<float4>(), m_s, max_corr_dist, max_iter, trans_eps, fit_eps, T16, fitness, converged, iters);
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
    unsigned char* tail = (unsigned char*)c->kf_full.p + (size_t)c->kf_full_used * stride;
    int m = n;
    if (n > 0 && bp->variant == 0) {                              // L:1498-1500 full_clouds: the cloud as received
        LILI_CUDA(c, cudaMemcpyAsync(tail, full, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream));
        LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    } else if (n > 0) {                                           // R:1373-1376 full_clouds_ds: VoxelGrid(surf_leaf) of it
        LILI_CUDA(c, c->raw.ensure((size_t)n * stride));
        LILI_CUDA(c, c->vg_count.ensure(16));
        LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, full, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream));
        LILI_TRY(voxelgrid_dev(c, c->raw.p, n, nullptr, stride, bp->surf_leaf, tail, c->vg_count.as<int>()));
        LILI_TRY(read_back(c, {{&m, c->vg_count.p, sizeof(int)}}));
    }
    c->kfs[kf_id].full_off = c->kf_full_used;
    c->kfs[kf_id].n_full = m;
    c->kf_full_used += m;
    if (n_stored) *n_stored = m;
    return LILIOM_OK;
}

// The global map without a concatenation buffer: box, voxel keys and centroids read the stored clouds through the keyframe table
// and transform every point on load (kf_table.h); the sort chain in between is voxelgrid_dev's (sort_pairs_u32 at the key width of
// the box, k_vg_heads, the scan).  Device memory: the table, 16 bytes per listed point for keys and values (sort included), and
// the output; only PCL's declined case writes the transformed concatenation, which is then the output.
extern "C" int liliom_global_map(liliom_ctx* c, int kind, const int* kf_ids, const double* poses7, int k, const double pre7[7],
                                 float leaf, void* out, int cap, int* n) {
    if (!c || !n || k < 0 || (k > 0 && (!kf_ids || !poses7)) || (kind != LILIOM_KF_FULL && kind != LILIOM_KF_SURF) || !(leaf > 0))
        return LILIOM_E_ARG;
    LILI_TRY(backend_check(c, nullptr));
    if (!kf_ids_ok(c, kf_ids, k)) return LILIOM_E_ARG;
    for (int i = 0; i < k && kind == LILIOM_KF_FULL; ++i)
        if (c->kfs[kf_ids[i]].n_full < 0) {
            c->last_error = "keyframe " + std::to_string(kf_ids[i]) + " has no full cloud (liliom_kf_add_full)";
            return LILIOM_E_ARG;
        }
    const int stride = c->prm.point_stride;
    std::vector<KfRow> tab;
    long long N = 0, largest = 0;
    for (int i = 0; i < k; ++i) {                                 // :2652-2662 list order, one cloud per keyframe
        const KfEntry& f = c->kfs[kf_ids[i]];
        const long long off = kind == LILIOM_KF_FULL ? f.full_off : f.surf_off;
        const int m = kind == LILIOM_KF_FULL ? f.n_full : f.n_surf;
        if (m) tab.push_back(kf_row(off, N, m, poses7 + 7 * (size_t)i, pre7));
        N += m;
        largest = std::max(largest, (long long)m);
    }
    if (N >= (1LL << 31)) {                                       // the sort chain's values and PCL's indices are ints
        c->last_error = "the listed keyframes hold " + std::to_string(N) + " points (at most 2^31 - 1)";
        return LILIOM_E_CAPACITY;
    }
    if (N == 0) { *n = 0; return LILIOM_OK; }
    LILI_CUDA(c, cudaSetDevice(c->device));
    const unsigned char* arena = (const unsigned char*)(kind == LILIOM_KF_FULL ? c->kf_full.p : c->kf_arena.p);
    const int rows = (int)tab.size();
    LILI_TRY(kf_upload_table(c, tab));
    const KfRow* d_tab = c->kf_tab.as<KfRow>();
    // box of the transformed concatenation (pcl::getMinMax3D), read back: the overflow test and the key width are decided here
    LILI_CUDA(c, c->vg_minmax.ensure(8 * sizeof(int)));
    int* mm = c->vg_minmax.as<int>();
    int* empty = reinterpret_cast<int*>(c->h_pin->scratch);       // pinned staging of the empty box; the stream orders the read-back after it
    for (int w = 0; w < kBoxInts; ++w) empty[w] = vg_box_empty(w);
    LILI_CUDA(c, cudaMemcpyAsync(mm, empty, kBoxInts * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    k_kf_box<<<kf_row_grid(tab.size(), largest, 8, 1024), 256, 0, c->stream>>>(arena, d_tab, rows, stride, mm);
    LILI_TRY(launch_check(c, "k_kf_box"));
    int box[kBoxInts];
    LILI_TRY(read_back(c, {{box, mm, sizeof(box)}}));
    const VgParams p = vg_params(box, leaf);
    if (p.overflow)                                               // PCL declines the filter and publishes its input
        return download_sized(c, c->vg_out, (int)N, stride, out, cap, n, [&]() -> int {
            LILI_CUDA(c, c->vg_out.ensure((size_t)N * stride));
            return kf_gather(c, arena, tab, largest, c->vg_out.p);
        });
    const int n_fin = p.n_finite;
    if (n_fin == 0) { *n = 0; return LILIOM_OK; }
    LILI_CUDA(c, c->vg_keys.ensure((size_t)N * 4));
    LILI_CUDA(c, c->vg_vals.ensure((size_t)N * 4));
    LILI_CUDA(c, c->vg_keys2.ensure((size_t)N * 4));
    LILI_CUDA(c, c->vg_vals2.ensure((size_t)N * 4));
    LILI_CUDA(c, c->vg_flags.ensure(((size_t)n_fin + 2) * 4));
    LILI_CUDA(c, c->vg_rank.ensure(((size_t)n_fin + 2) * 4));
    k_kf_keys<<<kf_row_grid(tab.size(), largest, 8), 256, 0, c->stream>>>(arena, d_tab, rows, stride, p, c->vg_keys.as<uint32_t>(),
                                                                             c->vg_vals.as<int>());
    LILI_TRY(launch_check(c, "k_kf_keys"));
    // non-finite points carry the all-ones key and sort last: the first n_fin sorted entries are the finite points
    LILI_TRY(sort_pairs_u32(c, c->vg_keys.as<uint32_t>(), c->vg_keys2.as<uint32_t>(), c->vg_vals.as<int>(), c->vg_vals2.as<int>(), (int)N,
                            vg_key_bits(box, leaf)));
    k_vg_heads<<<cdiv(n_fin + 1LL, 256), 256, 0, c->stream>>>(c->vg_keys2.as<uint32_t>(), n_fin, nullptr, c->vg_flags.as<int>());
    LILI_TRY(launch_check(c, "k_vg_heads"));
    LILI_TRY(exclusive_scan_i32(c, c->vg_flags.as<int>(), c->vg_rank.as<int>(), n_fin));
    int m = 0;
    LILI_TRY(read_back(c, {{&m, c->vg_rank.as<int>() + n_fin, sizeof(int)}}));
    return download_sized(c, c->vg_out, m, stride, out, cap, n, [&]() -> int {
        LILI_CUDA(c, c->vg_out.ensure((size_t)m * stride));
        if (stride == 48)
            k_kf_centroid<48><<<cdiv(n_fin, 128), 128, 0, c->stream>>>(arena, d_tab, rows, c->vg_keys2.as<uint32_t>(), c->vg_vals2.as<int>(),
                                                                       c->vg_flags.as<int>(), c->vg_rank.as<int>(), n_fin, (unsigned char*)c->vg_out.p);
        else
            k_kf_centroid<32><<<cdiv(n_fin, 128), 128, 0, c->stream>>>(arena, d_tab, rows, c->vg_keys2.as<uint32_t>(), c->vg_vals2.as<int>(),
                                                                       c->vg_flags.as<int>(), c->vg_rank.as<int>(), n_fin, (unsigned char*)c->vg_out.p);
        return launch_check(c, "k_kf_centroid");
    });
}
