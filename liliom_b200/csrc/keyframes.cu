// SURVEY.md §8 (f5): the backend's keyframe clouds and local map on the device.
//   keyframe store   BackendFusion::downSampleCloud, scan half (L/src/BackendFusion.cpp:1502-1514) + the clouds of
//                    saveKeyFramesAndFactors (:1688-1695): VoxelGrid of the received body-frame clouds, appended to one arena
//   local map        buildLocalMapWithLandMark (:1387-1484) + downSampleCloud, map half (:1486-1492): transform + concatenate
//                    the listed keyframes in ONE launch, VoxelGrid per layer, a cell grid per layer (MapIndex)
//   loop closure     detectLoopClosure's clouds (:2473-2547): edge then surf per keyframe, transformed, VoxelGrid
// The deque policy of the local map (:1407-1477) stays with the caller: every call lists the keyframes and the poses to use.
// Compiled with --fmad=false (the VoxelGrid centroids and the transform are bit-exact with the reference's arithmetic).
#include "ctx.cuh"
#include "dev_math.cuh"

namespace lili {

// One row of the gather table: n points of the arena at src_off, transformed by (q, t), written at dst_off of the output.
struct GatherEnt { long long src_off, dst_off; Q4 q; D3 t; int n, pad; };

// blockIdx.y = table row; the blocks of a row stream through that row's points.  The table lives in device memory, so one
// launch serves any number of keyframes (the odometry map's ConcatTab parameter holds 64).
__global__ void k_kf_gather(const unsigned char* __restrict__ arena, const GatherEnt* __restrict__ tab, int stride, unsigned char* __restrict__ out) {
    const GatherEnt& e = tab[blockIdx.y];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < e.n; i += gridDim.x * blockDim.x)
        pcl_transform_point(arena + (size_t)(e.src_off + i) * stride, stride, e.q, e.t, out + (size_t)(e.dst_off + i) * stride);
}

// reflectivity (curvature = 0.1 * reflectivity, L/src/FormatConvert.cpp:21) of 48-byte points
__global__ void k_kf_refl(const unsigned char* __restrict__ pts, int n, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = reinterpret_cast<const float*>(pts + (size_t)i * 48)[9];
}

void backend_release(liliom_ctx* c) {
    DevBuf* bufs[] = {&c->kf_arena, &c->kf_tab, &c->bmap_raw, &c->bmap_ds[0], &c->bmap_ds[1], &c->win_valid[0], &c->win_valid[1],
                      &c->win_line, &c->win_plane, &c->win_score, &c->win_cnt, &c->win_tab};
    for (DevBuf* b : bufs) b->release();
    c->bmap[0].release(); c->bmap[1].release();
}

// Room for `pts` points in the arena.  Grows geometrically and COPIES the stored keyframes (DevBuf::ensure would discard them);
// the cudaFree of the old block synchronises, which only happens on growth.
static int kf_reserve(liliom_ctx* c, long long pts) {
    const size_t stride = (size_t)c->prm.point_stride;
    const size_t need = (size_t)pts * stride;
    if (need <= c->kf_arena.cap) return LILIOM_OK;
    size_t want = std::max(need + need / 2, std::max(c->kf_arena.cap * 2, (size_t)1 << 20));
    void* p = nullptr;
    LILI_CUDA(c, cudaMalloc(&p, want));
    if (c->kf_used > 0) {
        const cudaError_t e = cudaMemcpyAsync(p, c->kf_arena.p, (size_t)c->kf_used * stride, cudaMemcpyDeviceToDevice, c->stream);
        if (e != cudaSuccess) { cudaFree(p); return fail_cuda(c, e, "kf_reserve copy"); }
        LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    }
    c->kf_arena.release();
    c->kf_arena.p = p; c->kf_arena.cap = want;
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

// Transform + concatenate rows of the store into `out` (one launch).  rows: {keyframe list index, layer 0 edge / 1 surf}.
static int kf_gather(liliom_ctx* c, const std::vector<GatherEnt>& tab, long long largest, void* out) {
    if (tab.empty() || largest <= 0) return LILIOM_OK;
    LILI_CUDA(c, c->kf_tab.ensure(tab.size() * sizeof(GatherEnt)));
    LILI_CUDA(c, cudaMemcpyAsync(c->kf_tab.p, tab.data(), tab.size() * sizeof(GatherEnt), cudaMemcpyHostToDevice, c->stream));
    const int bx = std::max(1, std::min(cdiv(largest, 256), c->sm_count * 4));
    k_kf_gather<<<dim3(bx, (unsigned)tab.size()), 256, 0, c->stream>>>((const unsigned char*)c->kf_arena.p, c->kf_tab.as<GatherEnt>(),
                                                                      c->prm.point_stride, (unsigned char*)out);
    return launch_check(c, "k_kf_gather");
}

static GatherEnt gather_row(long long src, long long dst, int n, const double* pose7) {
    GatherEnt e{};
    e.src_off = src; e.dst_off = dst; e.n = n;
    e.q = Q4{pose7[0], pose7[1], pose7[2], pose7[3]};
    e.t = D3{pose7[4], pose7[5], pose7[6]};
    return e;
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
    LILI_TRY(kf_reserve(c, c->kf_used + n));          // VoxelGrid never outputs more points than it reads
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
    LILI_CUDA(c, cudaMemcpyAsync(c->h_pin->bk_cnt, cnt, 2 * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    const int me = c->h_pin->bk_cnt[0], ms = c->h_pin->bk_cnt[1];
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
    c->kf_used = 0;                      // the arena keeps its allocation
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
    std::vector<GatherEnt> tab;
    tab.reserve(2 * (size_t)k);
    long long de = 0, ds = E;
    for (int i = 0; i < k; ++i) {                                 // :1479-1483 edge and surf layers, list order
        const KfEntry& f = c->kfs[kf_ids[i]];
        if (f.n_edge) tab.push_back(gather_row(f.edge_off, de, f.n_edge, poses7 + 7 * (size_t)i));
        if (f.n_surf) tab.push_back(gather_row(f.surf_off, ds, f.n_surf, poses7 + 7 * (size_t)i));
        de += f.n_edge; ds += f.n_surf;
    }
    LILI_CUDA(c, c->bmap_raw.ensure((size_t)std::max(E + S, 1LL) * stride));
    LILI_TRY(kf_gather(c, tab, largest, c->bmap_raw.p));
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
    LILI_CUDA(c, cudaMemcpyAsync(c->h_pin->bk_cnt, cnt, 2 * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    const int m[2] = {c->h_pin->bk_cnt[0], c->h_pin->bk_cnt[1]};
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
    const int m = c->bmap_n[layer];
    *m_out = m;
    if (!out) return LILIOM_OK;
    if (m > cap) return LILIOM_E_CAPACITY;
    if (m) LILI_CUDA(c, cudaMemcpyAsync(out, c->bmap_ds[layer].p, (size_t)m * c->prm.point_stride, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

extern "C" int liliom_kf_cloud(liliom_ctx* c, const int* kf_ids, const double* poses7, int k, float leaf, void* out, int cap, int* n_out) {
    if (!c || !n_out || k < 0 || (k > 0 && (!kf_ids || !poses7)) || !(leaf > 0)) return LILIOM_E_ARG;
    LILI_TRY(backend_check(c, nullptr));
    if (!kf_ids_ok(c, kf_ids, k)) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    *n_out = 0;
    std::vector<GatherEnt> tab;
    long long off = 0, largest = 0;
    for (int i = 0; i < k; ++i) {                                 // :2492-2493 / :2519-2520: *edge_frames[i] then *surf_frames[i]
        const KfEntry& f = c->kfs[kf_ids[i]];
        if (f.n_edge) tab.push_back(gather_row(f.edge_off, off, f.n_edge, poses7 + 7 * (size_t)i));
        off += f.n_edge;
        if (f.n_surf) tab.push_back(gather_row(f.surf_off, off, f.n_surf, poses7 + 7 * (size_t)i));
        off += f.n_surf;
        largest = std::max(largest, (long long)std::max(f.n_edge, f.n_surf));
    }
    if (off == 0) return LILIOM_OK;
    LILI_CUDA(c, c->bmap_raw.ensure((size_t)off * stride));      // scratch: the local map's layers live in bmap_ds / bmap
    LILI_CUDA(c, c->vg_out.ensure((size_t)off * stride));
    LILI_CUDA(c, c->vg_count.ensure(16));
    LILI_TRY(kf_gather(c, tab, largest, c->bmap_raw.p));
    LILI_TRY(voxelgrid_dev(c, c->bmap_raw.p, (int)off, nullptr, stride, leaf, c->vg_out.p, c->vg_count.as<int>()));
    LILI_CUDA(c, cudaMemcpyAsync(c->h_pin->bk_cnt, c->vg_count.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    const int m = c->h_pin->bk_cnt[0];
    *n_out = m;
    if (!out) return LILIOM_OK;
    if (m > cap) return LILIOM_E_CAPACITY;
    if (m) LILI_CUDA(c, cudaMemcpyAsync(out, c->vg_out.p, (size_t)m * stride, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}
