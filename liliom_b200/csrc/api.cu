// C ABI of libliliom_b200.so (see include/liliom.h for the contract and reference citations).
#include "ctx.cuh"
#include "dev_math.cuh"
#include "pc2_fields.h"
#include "wire_decode.h"
#include <new>
#include <cstdlib>

namespace lili {
void nccl_destroy(liliom_ctx* c);

// LidarOdometry::undistortion (L/src/LidarOdometry.cpp:178-199), in place on device clouds: one segment per cloud, segment s owns
// blocks [off[s], off[s + 1]) of the grid (batch.h).  A segment's size is n, or min(*d_n, n) when it is only on the device (n:
// a host upper bound).  liliom_undistort launches one segment, liliom_undistort_resident the three resident clouds,
// liliom_undistort_resident_batch the three of each of up to kBatchMax sessions (k_undistort_batch).
struct UndistortSeg {
    unsigned char* pts;
    int n;
    const int* d_n;
};
typedef BatchTab<UndistortSeg, 3> UndistortTab;

// point i of segment s (:181-197)
__device__ __forceinline__ void undistort_at(const UndistortSeg& s, int i, int stride, const D3& trans, const Q4& quat) {
    if (i >= (s.d_n ? min(*s.d_n, s.n) : s.n)) return;
    unsigned char* pts = s.pts;
    float4* p0 = reinterpret_cast<float4*>(pts + (size_t)i * stride);
    float4 a = p0[0];
    const float intensity = *reinterpret_cast<const float*>(pts + (size_t)i * stride + (stride == 48 ? 32 : 16));
    const int line = scan_id_of(intensity);                                             // :181 (x86's int(float))
    const double dt_i = (double)fsubx(intensity, (float)line);                         // :182 float - int -> float, then widened
    double ratio_i = dt_i / 0.1;                                                        // :183
    if (ratio_i > 1) ratio_i = 1;                                                       // :185-186
    const Q4 q_si = qslerp_x(Q4{1.0, 0.0, 0.0, 0.0}, ratio_i, quat);                    // :188-189
    const D3 r = qrot_x(q_si, D3{(double)a.x, (double)a.y, (double)a.z});               // :193
    a.x = (float)addx(r.x, mulx(ratio_i, trans.x));                                    // :191, :193-197
    a.y = (float)addx(r.y, mulx(ratio_i, trans.y));
    a.z = (float)addx(r.z, mulx(ratio_i, trans.z));
    p0[0] = a;
}

__global__ void k_undistort(const __grid_constant__ UndistortTab tab, int stride, D3 trans, Q4 quat) {
    const BatchSlot at = batch_slot(tab);
    undistort_at(tab.s[at.s], at.blk.bi() * blockDim.x + threadIdx.x, stride, trans, quat);
}

// a segment of the batched launch: the session's stride and motion travel with each of its clouds, so that Horizon and ROT
// sessions share a launch
struct UndistortBatchSeg {
    UndistortSeg seg;
    int stride;
    D3 trans;
    Q4 quat;
};
typedef BatchTab<UndistortBatchSeg, 3 * kBatchMax> UndistortBatchTab;
static_assert(sizeof(UndistortBatchTab) <= 32764, "a batched launch's session table must fit in the kernel parameter space");

__global__ void k_undistort_batch(const __grid_constant__ UndistortBatchTab tab) {
    const BatchSlot at = batch_slot(tab);
    const UndistortBatchSeg& s = tab.s[at.s];
    undistort_at(s.seg, at.blk.bi() * blockDim.x + threadIdx.x, s.stride, s.trans, s.quat);
}

// k_undistort over k <= 3 segments on the context's stream (segments without points get no blocks; none at all: no launch)
static int undistort_launch(liliom_ctx* c, const UndistortSeg* segs, int k, const double trans[3], const double quat_wxyz[4]) {
    UndistortTab tab{};
    tab.n = k;
    for (int s = 0; s < k; ++s) {
        tab.s[s] = segs[s];
        tab.off[s + 1] = tab.off[s] + stage_blocks(segs[s].n, 256);
    }
    if (tab.off[k] == 0) return LILIOM_OK;
    k_undistort<<<tab.off[k], 256, 0, c->stream>>>(tab, c->prm.point_stride, D3{trans[0], trans[1], trans[2]},
                                                   Q4{quat_wxyz[0], quat_wxyz[1], quat_wxyz[2], quat_wxyz[3]});
    return launch_check(c, "k_undistort");
}

// the three resident clouds of c as undistort segments (feat_clouds: LILIOM_E_ARG when nothing is resident)
static int undistort_resident_segs(liliom_ctx* c, UndistortSeg segs[3]) {
    FeatCloud f[3];
    LILI_TRY(feat_clouds(c, f));
    for (int k = 0; k < 3; ++k) segs[k] = UndistortSeg{f[k].buf->as<unsigned char>(), f[k].n_max, f[k].d_n};
    return LILIOM_OK;
}

static int upload_feats(liliom_ctx* c, const void* feats, int n, int stride) {
    c->d_nfeats = nullptr;
    if (n < 0 || (n > 0 && !feats)) return LILIOM_E_ARG;
    if (stride != 16 && stride != 32 && stride != 48) return LILIOM_E_ARG;
    c->n_feats = n;
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

}  // namespace lili

using namespace lili;

extern "C" void liliom_default_params(liliom_params* p, int variant) {
    if (!p) return;
    memset(p, 0, sizeof(*p));
    p->abi_version = LILIOM_ABI_VERSION;
    p->point_stride = variant == 1 ? 32 : 48;
    p->surf_thres = 0.2;         // L/config/config_fr_iosb.yaml:5
    p->edge_thres = 4.0;         // L/config/config_fr_iosb.yaml:6
    p->line_num = 64;            // R/config/config_fr_iosb.yaml
    p->ds_rate = variant == 1 ? 4 : 1;
    p->rot_ds_leaf = 0.6f;       // R/src/Preprocessing.cpp:14
    p->leaf_scan = 0.4f;         // L/src/LidarOdometry.cpp:155
    p->leaf_map = 0.4f;          // L/src/LidarOdometry.cpp:156
    p->knn_max_sqdist = 1.0;     // :365
    p->plane_thres = 0.06;       // :389
    p->weight_gate = 0.4;        // :400
    p->huber_a = 0.1;            // :507
    p->max_map_frames = 20;      // :290
    p->max_scan_points = 400000; // R/src/Preprocessing.cpp:9-12
    p->max_map_points = 2000000;
}

extern "C" const char* liliom_strerror(int code) {
    switch (code) {
        case LILIOM_OK: return "ok";
        case LILIOM_E_ARG: return "invalid argument";
        case LILIOM_E_CUDA: return "CUDA error (see liliom_last_error)";
        case LILIOM_E_FEWMAP: return "not enough feature points from the map (< 10): pose unchanged";
        case LILIOM_E_CAPACITY: return "buffer capacity too small";
        case LILIOM_E_GRID: return "map extent too large for the dense cell grid";
        case LILIOM_E_LINES: return "wrong scan number (line_num must be 16, 32 or 64, or 1..128 with LILIOM_RING_FIELD)";
        case LILIOM_E_NCCL: return "NCCL error (see liliom_last_error)";
        case LILIOM_E_NOMAP: return "no map installed";
        default: return "unknown error";
    }
}

extern "C" const char* liliom_last_error(const liliom_ctx* c) { return c ? c->last_error.c_str() : ""; }
extern "C" int liliom_point_stride(const liliom_ctx* c) { return c ? c->prm.point_stride : 0; }

extern "C" int liliom_create(liliom_ctx** out, const liliom_params* p, int device) {
    if (!out || !p) return LILIOM_E_ARG;
    *out = nullptr;
    if (p->abi_version != LILIOM_ABI_VERSION) return LILIOM_E_ARG;
    if (p->point_stride != 48 && p->point_stride != 32) return LILIOM_E_ARG;
    if (!(p->knn_max_sqdist > 0) || p->knn_max_sqdist > 4.0) return LILIOM_E_ARG;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) return LILIOM_E_CUDA;   // no CPU fallback
    liliom_ctx* c = new (std::nothrow) liliom_ctx();
    if (!c) return LILIOM_E_ARG;
    c->prm = *p;
    c->device = device;
    cudaError_t e = cudaSetDevice(device);
    cudaDeviceProp prop;
    if (e == cudaSuccess && cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->sm_count = prop.multiProcessorCount;
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking);
    c->stream = c->own_stream;
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_ready, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_copied, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_batch, cudaEventDisableTiming);
    c->h_pin_bytes = sizeof(PinBlock) + (1 << 20);      // the header + 1 MiB of per-iteration stats (3276 iterations)
    if (e == cudaSuccess) e = cudaHostAlloc((void**)&c->h_pin, c->h_pin_bytes, cudaHostAllocDefault);
    if (e != cudaSuccess) { liliom_destroy(c); return LILIOM_E_CUDA; }      // tears down whatever was created
    // the GN kernel writes its results straight into this block when the device can address it (UVA: always, in practice)
    if (cudaHostGetDevicePointer((void**)&c->h_pin_dev, c->h_pin, 0) != cudaSuccess) { c->h_pin_dev = nullptr; (void)cudaGetLastError(); }
    if (const char* e1 = getenv("LILIOM_KNN_LANES")) { int v = atoi(e1); if (v == 1 || v == 2 || v == 4 || v == 8 || v == 16) c->force_lanes = v; }
    c->dbg_timing = getenv("LILIOM_DEBUG_TIMING") != nullptr;
    c->rot_slow_walk = getenv("LILIOM_ROT_SLOW_WALK") != nullptr;
    if (const char* e9 = getenv("LILIOM_HZ_CHAIN")) c->hz_chain = atoi(e9) != 0;
    c->test_shrink_box = getenv("LILIOM_TEST_SHRINK_BOX") != nullptr;
    if (const char* e10 = getenv("LILIOM_TEST_ICP_BLOCKS")) c->test_icp_blocks = std::max(0, atoi(e10));
    if (const char* e8 = getenv("LILIOM_KNN_TMA")) c->knn_tma = atoi(e8) != 0;
    if (const char* e4 = getenv("LILIOM_SHARD_BLOCK")) {      // shard block edge in metres (power of two, 8..256): larger blocks = thinner halos
        int v = atoi(e4);
        if (v >= 8 && v <= 256 && (v & (v - 1)) == 0) c->shard_inv_block = 1.0f / (float)v;
    }
    if (const char* e2 = getenv("LILIOM_KNN_ROUNDS")) { int v = atoi(e2); if (v >= 1 && v <= 32) c->force_rounds = v; }
    if (const char* e11 = getenv("LILIOM_TEST_LOOPBACK")) {      // <group>:<rank>/<nranks>; a malformed value refuses the context
        const char* colon = strrchr(e11, ':');
        int r = -1, nr = 0, used = 0;
        if (!colon || colon == e11 || sscanf(colon + 1, "%d/%d%n", &r, &nr, &used) != 2 || colon[1 + used] != '\0' || nr < 2 ||
            nr > kMaxPeers || r < 0 || r >= nr) { liliom_destroy(c); return LILIOM_E_ARG; }
        c->loopback_group.assign(e11, colon - e11);
        c->nranks = nr; c->rank = r;
        if (const char* e12 = getenv("LILIOM_TEST_LOOPBACK_MS")) c->loopback_ms = std::max(1, atoi(e12));
    }
    *out = c;
    return LILIOM_OK;
}

extern "C" void liliom_destroy(liliom_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    nccl_destroy(c);
    for (cudaEvent_t e : c->ev_pool) cudaEventDestroy(e);
    if (c->h_pin) cudaFreeHost(c->h_pin);
    if (c->ev_ready) cudaEventDestroy(c->ev_ready);
    if (c->ev_copied) cudaEventDestroy(c->ev_copied);
    if (c->ev_batch) cudaEventDestroy(c->ev_batch);
    if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    delete c;      // the device buffers (DevBuf members, frames, indices) free themselves here, with the device still current
}

// ===================== L1 =====================
// Shared tail of the Horizon entry points: c->raw holds n 48-byte points (upload already queued on the stream).
static int extract_horizon_from_raw(liliom_ctx* c, int n, const double q_imu[4],
                                    liliom_pt48* surf_out, int surf_cap, int* n_surf, liliom_pt48* edge_out, int edge_cap, int* n_edge,
                                    liliom_pt48* cut_out, int cut_cap, int* n_cut) {
    int ns = 0, ne = 0, nc = 0;
    // The cutted cloud is complete after the de-skew kernel: its D2H runs on the copy stream under the patch kernels.
    // It is issued before the count is known, so min(n, cut_cap) slots are copied; slots past *n_cut are unspecified.
    c->early_cut_dst = cut_out; c->early_cut_cap = cut_cap; c->early_cut_issued = false;
    const int rc_x = horizon_extract_dev(c, n, q_imu, &ns, &ne, &nc);
    c->early_cut_dst = nullptr;
    if (rc_x != LILIOM_OK) { if (c->early_cut_issued) cudaStreamSynchronize(c->copy_stream); return rc_x; }
    const bool over = (surf_out && ns > surf_cap) || (edge_out && ne > edge_cap) || (cut_out && nc > cut_cap);
    if (!over) {
        if (surf_out && ns) LILI_CUDA(c, cudaMemcpyAsync(surf_out, c->surf.p, (size_t)ns * 48, cudaMemcpyDeviceToHost, c->stream));
        if (edge_out && ne) LILI_CUDA(c, cudaMemcpyAsync(edge_out, c->edge.p, (size_t)ne * 48, cudaMemcpyDeviceToHost, c->stream));
        if (cut_out && nc && !c->early_cut_issued)
            LILI_CUDA(c, cudaMemcpyAsync(cut_out, c->cut.p, (size_t)nc * 48, cudaMemcpyDeviceToHost, c->stream));
    }
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    if (c->early_cut_issued) LILI_CUDA(c, cudaStreamSynchronize(c->copy_stream));   // c->cut is reused by the next call
    if (over) return LILIOM_E_CAPACITY;
    *n_surf = ns; *n_edge = ne; *n_cut = nc;
    return LILIOM_OK;
}

extern "C" int liliom_extract_horizon(liliom_ctx* c, const liliom_pt48* pts, int n, const double q_imu[4],
                                      liliom_pt48* surf_out, int surf_cap, int* n_surf, liliom_pt48* edge_out, int edge_cap, int* n_edge,
                                      liliom_pt48* cut_out, int cut_cap, int* n_cut) {
    if (!c || n < 0 || (n > 0 && !pts) || !q_imu || !n_surf || !n_edge || !n_cut) return LILIOM_E_ARG;
    if (c->prm.point_stride != 48) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_CUDA(c, c->raw.ensure((size_t)(n > 0 ? n : 1) * 48));
    if (n > 0) LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, pts, (size_t)n * 48, cudaMemcpyHostToDevice, c->stream));
    return extract_horizon_from_raw(c, n, q_imu, surf_out, surf_cap, n_surf, edge_out, edge_cap, n_edge, cut_out, cut_cap, n_cut);
}

// ---- (f3) FormatConvert on the device: livox_ros_driver::CustomPoint[] -> pcl::PointXYZINormal[] (L/src/FormatConvert.cpp:11-24;
// the per-point body: wire_decode.h; the decode: wire_decode below)
namespace lili {
// the Livox calls' refusals
static bool livox_args_ok(const liliom_ctx* c, const void* custom_pts, int n, int stride) {
    return c && n >= 0 && (n == 0 || custom_pts) && (stride == 19 || stride == 20) && c->prm.point_stride == 48;
}

// The end of a convert call that leaves n points of `stride` bytes resident: the resident count, and the download to out
// (NULL: none) on the context's stream.
static int resident_finish(liliom_ctx* c, int n, int stride, void* out) {
    c->n_raw_scan = n;
    if (out && n) LILI_CUDA(c, cudaMemcpyAsync(out, c->raw_scan.p, (size_t)n * stride, cudaMemcpyDeviceToHost, c->stream));
    return LILIOM_OK;
}
}  // namespace lili

static int extract_rot_from_raw(liliom_ctx* c, int n, const double q_imu[4], const double q_lb[4],
                                liliom_pt32* surf_out, int surf_cap, int* n_surf, liliom_pt32* edge_out, int edge_cap, int* n_edge,
                                liliom_pt32* cut_out, int cut_cap, int* n_cut, const uint16_t* rings = nullptr,
                                const double* times = nullptr);

extern "C" int liliom_extract_rot(liliom_ctx* c, const liliom_pt32* pts, int n, const double q_imu[4], const double q_lb[4],
                                  liliom_pt32* surf_out, int surf_cap, int* n_surf, liliom_pt32* edge_out, int edge_cap, int* n_edge,
                                  liliom_pt32* cut_out, int cut_cap, int* n_cut) {
    if (!c || n < 0 || (n > 0 && !pts) || !q_imu || !q_lb || !n_surf || !n_edge || !n_cut) return LILIOM_E_ARG;
    if (c->prm.point_stride != 32) return LILIOM_E_ARG;
    if (c->ring_source == LILIOM_RING_FIELD) return LILIOM_E_ARG;     // host 32-byte points carry no ring
    if (c->time_source == LILIOM_TIME_FIELD) return LILIOM_E_ARG;     // ... and no time
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_CUDA(c, c->raw.ensure((size_t)(n > 0 ? n : 1) * 32));
    if (n > 0) LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, pts, (size_t)n * 32, cudaMemcpyHostToDevice, c->stream));
    return extract_rot_from_raw(c, n, q_imu, q_lb, surf_out, surf_cap, n_surf, edge_out, edge_cap, n_edge, cut_out, cut_cap, n_cut);
}

// ---- (f3) pcl::fromROSMsg(PointCloud2 -> pcl::PointXYZI) on the device (R/src/Preprocessing.cpp:277); field matching: pc2_fields.h,
// the per-point body: wire_decode.h
namespace lili {
// pc2_match under the context's sources: the `ring` field under LILIOM_RING_FIELD, the named time field under LILIOM_TIME_FIELD
static int pc2_match_ctx(const liliom_ctx* c, const liliom_pc2_msg* msg, Pc2Map* m) {
    return pc2_match(msg, m, c->ring_source == LILIOM_RING_FIELD, c->time_source == LILIOM_TIME_FIELD ? c->time_name : nullptr);
}
static size_t pc2_bytes(const liliom_pc2_msg* msg) { return (size_t)msg->height * msg->row_step; }
// the side buffers the decode writes: those of the channels m matched (nullptr for the others)
static uint16_t* pc2_ring_out(const Pc2Map& m, Pc2Side& side) { return m.ring_src >= 0 ? side.ring.as<uint16_t>() : nullptr; }
static double* pc2_time_out(const Pc2Map& m, Pc2Side& side) { return m.time_src >= 0 ? side.time.as<double>() : nullptr; }

// ---- the decode of driver messages, one session (the solo calls) or many (liliom_convert_batch): the stages (k_stage_batch),
// each session's decode as one thread per point; a block belongs to one session, so the ring / time branches stay uniform.
// The PointCloud2 decode is kept a pass of its own rather than fused into the ROT chain's first stage: the chain reads the
// decoded sweep again.
struct LivoxEntry {
    const unsigned char* in;
    int n, stride;
    unsigned char* out;
};
struct Pc2Entry {
    const unsigned char* in;
    int n;
    Pc2Wire w;
    unsigned char* out;
    uint16_t* ring_out;
    double* time_out;
};
LILI_STAGE(WireStLivox, LivoxEntry, 256, stage_blocks(e.n, 256), livox_point_at(e.in, e.n, e.stride, e.out, i))
LILI_STAGE(WireStPc2, Pc2Entry, 256, stage_blocks(e.n, 256), pc2_point_at(e.in, e.n, e.w, e.out, e.ring_out, e.time_out, i))

// One accepted message of a session: what pc2_match_ctx made of it (PC2), its points, where they go and their download.
struct WireJob {
    liliom_ctx* c;
    const liliom_wire_msg* msg;
    Pc2Map m;
    int n;
    void* out;                  // the convert calls' download (NULL: none)
    DevBuf* dst;                // the decoded points: the resident sweep (the convert calls) or the extractor's input
    Pc2Side* side;              // their side channels (NULL: left as they are, liliom_extract_horizon_livox)
};

// The solo convert call's refusals of session c's message, in its order; on LILIOM_OK, j describes the session, decoded into
// the resident sweep.  A PC2 message refused for capacity reports its size in *n, as liliom_convert_pc2 does.
static int wire_accept(liliom_ctx* c, const liliom_wire_msg& w, void* out, int cap, int* n, WireJob& j) {
    j = WireJob{c, &w, Pc2Map{}, 0, out, nullptr, nullptr};
    if (w.kind == LILIOM_WIRE_LIVOX) {
        if (!livox_args_ok(c, w.custom_pts, w.n, w.stride)) return LILIOM_E_ARG;
        if (out && w.n > cap) return LILIOM_E_CAPACITY;
        j.n = w.n;
    } else {
        if (w.kind != LILIOM_WIRE_PC2 || pc2_match_ctx(c, w.pc2, &j.m) != LILIOM_OK) return LILIOM_E_ARG;
        if (c->prm.point_stride != 32) return LILIOM_E_ARG;
        if (out && j.m.n > cap) { *n = j.m.n; return LILIOM_E_CAPACITY; }
        j.n = j.m.n;
    }
    j.dst = &c->raw_scan;
    j.side = &c->raw_scan_side;
    return LILIOM_OK;
}
static bool wire_is_livox(const WireJob& j) { return j.msg->kind == LILIOM_WIRE_LIVOX; }

// The buffers of an accepted job: dst for its points, side cleared and sized for the channels it matched, wire_in for the payload
static int wire_begin(const WireJob& j) {
    liliom_ctx* c = j.c;
    const size_t n = (size_t)(j.n > 0 ? j.n : 1);
    if (wire_is_livox(j)) {
        if (j.side) j.side->clear();
        LILI_CUDA(c, j.dst->ensure(n * 48));
        if (j.n > 0) LILI_CUDA(c, c->wire_in.ensure((size_t)j.n * j.msg->stride));
        return LILIOM_OK;
    }
    LILI_CUDA(c, j.dst->ensure(n * 32));
    j.side->clear();
    if (j.m.ring_src >= 0) LILI_CUDA(c, j.side->ring.ensure(n * sizeof(uint16_t)));
    if (j.m.time_src >= 0) LILI_CUDA(c, j.side->time.ensure(n * sizeof(double)));
    if (j.n > 0) LILI_CUDA(c, c->wire_in.ensure(pc2_bytes(j.msg->pc2)));
    return LILIOM_OK;
}

// The decode of jobs past wire_begin, on c0's stream (every job's context stream is c0's): each payload into its context's
// wire_in, the stages, then each PointCloud2 job's side records the channels it now holds (none when the decode fails).
static int wire_decode(liliom_ctx* c0, const std::vector<WireJob>& jobs) {
    std::vector<int> livox, pc2;        // jobs with points, by kind
    for (size_t k = 0; k < jobs.size(); ++k) {
        const WireJob& j = jobs[k];
        if (j.n <= 0) continue;
        const void* src = wire_is_livox(j) ? j.msg->custom_pts : j.msg->pc2->data;
        const size_t bytes = wire_is_livox(j) ? (size_t)j.n * j.msg->stride : pc2_bytes(j.msg->pc2);
        LILI_CUDA(j.c, cudaMemcpyAsync(j.c->wire_in.p, src, bytes, cudaMemcpyHostToDevice, c0->stream));
        (wire_is_livox(j) ? livox : pc2).push_back((int)k);
    }
    LILI_TRY(stage_batch<WireStLivox>(c0, livox, [&](LivoxEntry& e, int k) {
        const WireJob& j = jobs[k];
        e = LivoxEntry{j.c->wire_in.as<const unsigned char>(), j.n, j.msg->stride, j.dst->as<unsigned char>()};
        return j.c;
    }));
    LILI_TRY(stage_batch<WireStPc2>(c0, pc2, [&](Pc2Entry& e, int k) {
        const WireJob& j = jobs[k];
        e = Pc2Entry{j.c->wire_in.as<const unsigned char>(), j.n, pc2_wire(j.msg->pc2, j.m), j.dst->as<unsigned char>(),
                     pc2_ring_out(j.m, *j.side), pc2_time_out(j.m, *j.side)};
        return j.c;
    }));
    for (const WireJob& j : jobs) {
        if (wire_is_livox(j)) continue;
        j.side->has_ring = j.m.ring_src >= 0;
        j.side->has_time = j.m.time_src >= 0;
    }
    return LILIOM_OK;
}

// One session's decode on its own stream (the solo calls)
static int wire_decode_one(const WireJob& j) {
    LILI_TRY(wire_begin(j));
    return wire_decode(j.c, {j});
}

// A solo convert call: the decode into the resident sweep, its download, one synchronise; *n (PC2): the point count
static int wire_convert(liliom_ctx* c, const liliom_wire_msg& w, void* out, int cap, int* n) {
    WireJob j;
    LILI_TRY(wire_accept(c, w, out, cap, n, j));
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_TRY(wire_decode_one(j));
    LILI_TRY(resident_finish(c, j.n, wire_is_livox(j) ? 48 : 32, out));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    if (n) *n = j.n;
    return LILIOM_OK;
}
}  // namespace lili

extern "C" int liliom_convert_livox(liliom_ctx* c, const void* custom_pts, int n, int stride, liliom_pt48* out, int cap) {
    const liliom_wire_msg w{LILIOM_WIRE_LIVOX, custom_pts, n, stride, nullptr};
    return wire_convert(c, w, out, cap, nullptr);
}

extern "C" int liliom_convert_pc2(liliom_ctx* c, const liliom_pc2_msg* msg, liliom_pt32* out, int cap, int* n) {
    if (!c || !n) return LILIOM_E_ARG;
    const liliom_wire_msg w{LILIOM_WIRE_PC2, nullptr, 0, 0, msg};
    return wire_convert(c, w, out, cap, n);
}

extern "C" int liliom_extract_horizon_livox(liliom_ctx* c, const void* custom_pts, int n, int stride, const double q_imu[4],
                                            liliom_pt48* surf_out, int surf_cap, int* n_surf, liliom_pt48* edge_out, int edge_cap, int* n_edge,
                                            liliom_pt48* cut_out, int cut_cap, int* n_cut) {
    if (!q_imu || !n_surf || !n_edge || !n_cut) return LILIOM_E_ARG;
    const liliom_wire_msg w{LILIOM_WIRE_LIVOX, custom_pts, n, stride, nullptr};
    WireJob j;
    LILI_TRY(wire_accept(c, w, nullptr, 0, nullptr, j));
    j.dst = &c->raw;
    j.side = nullptr;
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_TRY(wire_decode_one(j));
    return extract_horizon_from_raw(c, n, q_imu, surf_out, surf_cap, n_surf, edge_out, edge_cap, n_edge, cut_out, cut_cap, n_cut);
}

extern "C" int liliom_extract_rot_pc2(liliom_ctx* c, const liliom_pc2_msg* msg, const double q_imu[4], const double q_lb[4],
                                      liliom_pt32* surf_out, int surf_cap, int* n_surf, liliom_pt32* edge_out, int edge_cap, int* n_edge,
                                      liliom_pt32* cut_out, int cut_cap, int* n_cut) {
    if (!c || !q_imu || !q_lb || !n_surf || !n_edge || !n_cut) return LILIOM_E_ARG;
    const liliom_wire_msg w{LILIOM_WIRE_PC2, nullptr, 0, 0, msg};
    WireJob j;
    LILI_TRY(wire_accept(c, w, nullptr, 0, nullptr, j));
    if (c->ring_source == LILIOM_RING_FIELD && !rot_lines_ok(c->prm.line_num, true)) return LILIOM_E_LINES;
    j.dst = &c->raw;
    j.side = &c->raw_side;
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_TRY(wire_decode_one(j));
    return extract_rot_from_raw(c, j.n, q_imu, q_lb, surf_out, surf_cap, n_surf, edge_out, edge_cap, n_edge, cut_out, cut_cap, n_cut,
                                c->raw_side.rings(), c->raw_side.times());
}

extern "C" int liliom_convert_batch(liliom_ctx* const* ctxs, int B, const liliom_wire_msg* msgs, void* const* out, const int* cap, int* n,
                                    int* status) {
    if (!batch_ctxs_ok(ctxs, B) || !msgs || !n || !status) return LILIOM_E_ARG;
    liliom_ctx* c0 = ctxs[0];
    LILI_CUDA(c0, cudaSetDevice(c0->device));
    const std::vector<liliom_ctx*> all(ctxs, ctxs + B);
    std::vector<WireJob> jobs;
    std::vector<int> at;                    // index of each job's session in ctxs
    for (int i = 0; i < B; ++i) {
        WireJob j;
        status[i] = wire_accept(ctxs[i], msgs[i], out ? out[i] : nullptr, cap ? cap[i] : 0, n + i, j);
        if (status[i] == LILIOM_OK) status[i] = wire_begin(j);
        if (status[i] != LILIOM_OK) continue;
        jobs.push_back(j);
        at.push_back(i);
    }
    // every session's work so far is ordered before the copies into its buffers; they, the decodes and the downloads then
    // queue back to back on ctxs[0]'s stream
    LILI_TRY(batch_join_in(c0, all));
    {
        const BatchStreams on_c0(all, c0->stream);
        LILI_TRY(wire_decode(c0, jobs));
        for (const WireJob& j : jobs) LILI_TRY(resident_finish(j.c, j.n, wire_is_livox(j) ? 48 : 32, j.out));
    }
    // one synchronise for the whole call
    LILI_TRY(batch_join_out(c0, all));
    LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
    for (size_t k = 0; k < jobs.size(); ++k) n[at[k]] = jobs[k].n;
    return LILIOM_OK;
}

// Shared tail of the ROT entry points: c->raw holds n 32-byte points (upload / decode already queued on the stream); rings: their
// ring ids (LILIOM_RING_FIELD) or nullptr (elevation tables); times: their times (LILIOM_TIME_FIELD) or nullptr (azimuth rule).
static int extract_rot_from_raw(liliom_ctx* c, int n, const double q_imu[4], const double q_lb[4],
                                liliom_pt32* surf_out, int surf_cap, int* n_surf, liliom_pt32* edge_out, int edge_cap, int* n_edge,
                                liliom_pt32* cut_out, int cut_cap, int* n_cut, const uint16_t* rings, const double* times) {
    int ns = 0, ne = 0, nc = 0;
    LILI_TRY(rot_extract_dev(c, n, q_imu, q_lb, &ns, &ne, &nc, rings, times));
    if ((surf_out && ns > surf_cap) || (edge_out && ne > edge_cap) || (cut_out && nc > cut_cap)) return LILIOM_E_CAPACITY;
    if (surf_out && ns) LILI_CUDA(c, cudaMemcpyAsync(surf_out, c->surf.p, (size_t)ns * 32, cudaMemcpyDeviceToHost, c->stream));
    if (edge_out && ne) LILI_CUDA(c, cudaMemcpyAsync(edge_out, c->edge.p, (size_t)ne * 32, cudaMemcpyDeviceToHost, c->stream));
    if (cut_out && nc) LILI_CUDA(c, cudaMemcpyAsync(cut_out, c->rot_cloud.p, (size_t)nc * 32, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    *n_surf = ns; *n_edge = ne; *n_cut = nc;
    return LILIOM_OK;
}

extern "C" int liliom_extract_rot_labels(liliom_ctx* c, int* label_out, float* curv_out, int cap) {
    if (!c) return LILIOM_E_ARG;
    const int n = c->n_rot_cloud;
    if (n > cap) return LILIOM_E_CAPACITY;
    LILI_CUDA(c, cudaSetDevice(c->device));
    if (label_out && n) LILI_CUDA(c, cudaMemcpyAsync(label_out, c->rot_label.p, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
    if (curv_out && n) LILI_CUDA(c, cudaMemcpyAsync(curv_out, c->rot_curv.p, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

extern "C" int liliom_voxelgrid(liliom_ctx* c, const void* pts, int n, int stride, float leaf, void* out, int cap, int* n_out) {
    if (!c || n < 0 || (n > 0 && !pts) || !n_out || !(leaf > 0)) return LILIOM_E_ARG;
    if (stride != 48 && stride != 32) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    *n_out = 0;
    if (n == 0) return LILIOM_OK;
    LILI_CUDA(c, c->raw.ensure((size_t)n * stride));
    c->n_ds_resident = -1;      // vg_out is rewritten: no scan for liliom_map_update_resident
    LILI_CUDA(c, c->vg_out.ensure((size_t)n * stride));
    LILI_CUDA(c, c->vg_count.ensure(16));
    LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, pts, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream));
    bool coop = false;
    LILI_TRY(voxelgrid_coop(c, c->raw.p, n, nullptr, stride, leaf, c->vg_out.p, c->vg_count.as<int>(), nullptr, &coop));
    int m = 0, key_bits = 32;
    if (coop) {      // the cooperative filter may decline the input: its verdict comes back with the count and the box's parameters
        VgParams vp;
        LILI_TRY(read_back(c, {{&m, c->vg_count.p, sizeof(int)}, {&vp, c->vg_params.p, sizeof(VgParams)}}));
        if (vp.bail) coop = false;
        if (vg_wide_keys(vp)) key_bits = kVgWideKeyBits;
    }
    if (!coop) LILI_TRY(voxelgrid_dev_sync(c, c->raw.p, n, stride, leaf, c->vg_out.p, c->vg_count.as<int>(), nullptr, &m, key_bits));
    if (out && m > cap) return LILIOM_E_CAPACITY;
    if (out && m) {
        LILI_CUDA(c, cudaMemcpyAsync(out, c->vg_out.p, (size_t)m * stride, cudaMemcpyDeviceToHost, c->stream));
        LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    }
    *n_out = m;
    return LILIOM_OK;
}

// SURVEY §8 (f3): LidarOdometry::undistortion on the device (L/src/LidarOdometry.cpp:178-199; publishCloudLast :624-632)
extern "C" int liliom_undistort(liliom_ctx* c, void* pts_inout, int n, const double trans[3], const double quat_wxyz[4]) {
    if (!c || n < 0 || (n > 0 && !pts_inout) || !trans || !quat_wxyz) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    if (n == 0) return LILIOM_OK;
    const int stride = c->prm.point_stride;
    LILI_CUDA(c, c->raw.ensure((size_t)n * stride));
    LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, pts_inout, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream));
    const UndistortSeg seg{c->raw.as<unsigned char>(), n, nullptr};
    LILI_TRY(undistort_launch(c, &seg, 1, trans, quat_wxyz));
    LILI_CUDA(c, cudaMemcpyAsync(pts_inout, c->raw.p, (size_t)n * stride, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

// publishCloudLast's undistortion (:624-632) of the three clouds the last extraction left resident, in place, in one launch;
// a resident Horizon extraction's sizes are read on the device
extern "C" int liliom_undistort_resident(liliom_ctx* c, const double trans[3], const double quat_wxyz[4]) {
    if (!c || !trans || !quat_wxyz) return LILIOM_E_ARG;
    UndistortSeg segs[3];
    LILI_TRY(undistort_resident_segs(c, segs));
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_TRY(undistort_launch(c, segs, 3, trans, quat_wxyz));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

// liliom_undistort_resident of several sessions: the three clouds of up to kBatchMax sessions per k_undistort_batch launch, each
// segment with its solo launch's blocks; a session whose clouds have no points takes part in no launch, as in its solo call
extern "C" int liliom_undistort_resident_batch(liliom_ctx* const* ctxs, int B, const double* trans, const double* quat_wxyz, int* status) {
    if (!batch_ctxs_ok(ctxs, B) || !trans || !quat_wxyz || !status) return LILIOM_E_ARG;
    liliom_ctx* c0 = ctxs[0];
    LILI_CUDA(c0, cudaSetDevice(c0->device));
    std::vector<UndistortBatchSeg> segs;    // three per session that launches
    std::vector<liliom_ctx*> who;
    for (int i = 0; i < B; ++i) {
        liliom_ctx* c = ctxs[i];
        UndistortSeg s[3];
        status[i] = undistort_resident_segs(c, s);
        if (status[i] != LILIOM_OK || stage_blocks(s[0].n, 256) + stage_blocks(s[1].n, 256) + stage_blocks(s[2].n, 256) == 0) continue;
        const double* t = trans + 3 * (size_t)i;
        const double* q = quat_wxyz + 4 * (size_t)i;
        for (int k = 0; k < 3; ++k) segs.push_back(UndistortBatchSeg{s[k], c->prm.point_stride, D3{t[0], t[1], t[2]}, Q4{q[0], q[1], q[2], q[3]}});
        who.push_back(c);
    }
    const std::vector<liliom_ctx*> all(ctxs, ctxs + B);
    LILI_TRY(batch_join_in(c0, all));
    for (size_t first = 0; first < who.size(); first += kBatchMax) {
        const int n = (int)std::min(who.size() - first, (size_t)kBatchMax);
        UndistortBatchTab tab{};
        tab.n = 3 * n;
        for (int m = 0; m < 3 * n; ++m) {
            tab.s[m] = segs[3 * first + m];
            tab.off[m + 1] = tab.off[m] + stage_blocks(tab.s[m].seg.n, 256);
        }
        k_undistort_batch<<<tab.off[3 * n], 256, 0, c0->stream>>>(tab);
        LILI_CUDA(c0, cudaGetLastError());
        for (int m = 0; m < n; ++m) who[first + m]->cnt.launches++;
    }
    LILI_TRY(batch_join_out(c0, all));
    LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
    return LILIOM_OK;
}

// ===================== L2: scan-to-map =====================
extern "C" int liliom_upload_feats(liliom_ctx* c, const void* feats, int n, int stride) {
    if (!c) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_TRY(upload_feats(c, feats, n, stride));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

extern "C" int liliom_scan_to_map_resident(liliom_ctx* c, double pose7[7], int match_cnt, int max_num_iter, int mode, liliom_iter_stats* stats) {
    if (!c || !pose7 || (mode != LILIOM_MODE_CERES && mode != LILIOM_MODE_GN) || match_cnt < 0) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    return s2m_run(c, pose7, match_cnt, max_num_iter, mode, stats, false, nullptr);
}

extern "C" int liliom_scan_to_map(liliom_ctx* c, const void* feats, int n, int stride, double pose7[7], int match_cnt, int max_num_iter,
                                  int mode, liliom_iter_stats* stats) {
    if (!c || !pose7 || (mode != LILIOM_MODE_CERES && mode != LILIOM_MODE_GN) || match_cnt < 0) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    if (!c->map.ready) return LILIOM_E_NOMAP;
    if (c->map_n_global < 10) return LILIOM_E_FEWMAP;
    LILI_TRY(upload_feats(c, feats, n, stride));
    return s2m_run(c, pose7, match_cnt, max_num_iter, mode, stats, false, nullptr);
}

static int odometry_on_resident_surf(liliom_ctx* c, double pose7[7], int match_cnt, int max_num_iter, int mode, liliom_iter_stats* stats,
                                     void* ds_out, int ds_cap, int* n_ds, bool spec_failed = false);

extern "C" int liliom_odometry(liliom_ctx* c, const void* surf_feats, int n, double pose7[7], int match_cnt, int max_num_iter, int mode,
                               liliom_iter_stats* stats, void* ds_out, int ds_cap, int* n_ds) {
    if (!c || !pose7 || n < 0 || (n > 0 && !surf_feats) || (mode != LILIOM_MODE_CERES && mode != LILIOM_MODE_GN) || match_cnt < 0) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    LILI_CUDA(c, c->surf.ensure((size_t)(n > 0 ? n : 1) * stride));
    if (n > 0) LILI_CUDA(c, cudaMemcpyAsync(c->surf.p, surf_feats, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream));
    c->n_surf_dev = n;
    c->feat_ready = false;         // the caller's surf features replace the extracted ones
    return odometry_on_resident_surf(c, pose7, match_cnt, max_num_iter, mode, stats, ds_out, ds_cap, n_ds);
}

extern "C" int liliom_set_stream(liliom_ctx* c, void* cuda_stream) {
    if (!c) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    c->stream = cuda_stream ? (cudaStream_t)cuda_stream : c->own_stream;
    return LILIOM_OK;
}

extern "C" int liliom_upload_scan(liliom_ctx* c, const void* pts, int n) {
    if (!c || n < 0 || (n > 0 && !pts)) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    LILI_CUDA(c, c->raw_scan.ensure((size_t)(n > 0 ? n : 1) * stride));
    if (n > 0) LILI_CUDA(c, cudaMemcpyAsync(c->raw_scan.p, pts, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    c->n_raw_scan = n;
    c->raw_scan_side.clear();
    return LILIOM_OK;
}

extern "C" int liliom_set_ring_source(liliom_ctx* c, int source) {
    if (!c || (source != LILIOM_RING_ELEVATION && source != LILIOM_RING_FIELD)) return LILIOM_E_ARG;
    if (source == LILIOM_RING_FIELD && c->prm.point_stride != 32) return LILIOM_E_ARG;
    if (source != c->ring_source) c->raw_scan_side.has_ring = false;   // the resident sweep was decoded under the other source
    c->ring_source = source;
    return LILIOM_OK;
}

extern "C" int liliom_set_time_source(liliom_ctx* c, int source, const char* field_name) {
    if (!c || (source != LILIOM_TIME_AZIMUTH && source != LILIOM_TIME_FIELD)) return LILIOM_E_ARG;
    if (source == LILIOM_TIME_FIELD) {
        if (c->prm.point_stride != 32 || !field_name) return LILIOM_E_ARG;
        const size_t len = strnlen(field_name, sizeof(c->time_name));
        if (len >= sizeof(c->time_name)) return LILIOM_E_ARG;
        memset(c->time_name, 0, sizeof(c->time_name));
        memcpy(c->time_name, field_name, len);
    }
    c->raw_scan_side.has_time = false;   // any call: the resident sweep's times (if any) may belong to another field
    c->time_source = source;
    return LILIOM_OK;
}

// The side channels a ROT extraction of the resident sweep reads under the context's sources: LILIOM_E_ARG when the sweep was
// not decoded with one of them.
static int resident_side(const liliom_ctx* c, const uint16_t** rings, const double** times) {
    const bool field = c->ring_source == LILIOM_RING_FIELD;
    const bool timed = c->time_source == LILIOM_TIME_FIELD;
    const lili::Pc2Side& side = c->raw_scan_side;
    if (field && !side.has_ring) return LILIOM_E_ARG;       // no ring ids decoded with the resident sweep
    if (timed && !side.has_time) return LILIOM_E_ARG;       // no times decoded with the resident sweep
    *rings = field ? side.rings() : nullptr;
    *times = timed ? side.times() : nullptr;
    return LILIOM_OK;
}

static const double kIdentityQ[4] = {1, 0, 0, 0};

extern "C" int liliom_extract_resident(liliom_ctx* c, const double q_imu[4], const double q_lb[4], int* n_surf, int* n_edge, int* n_cut) {
    if (!c || !q_imu || !n_surf || !n_edge || !n_cut) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    const int n = c->n_raw_scan;
    // the extractors only read their input: they take the resident sweep in place (no device-to-device copy)
    c->raw_src = n > 0 ? c->raw_scan.p : nullptr;
    int rc;
    if (stride == 48) rc = horizon_extract_dev(c, n, q_imu, n_surf, n_edge, n_cut, /*sync_counts=*/false);
    else {
        const uint16_t* rings = nullptr;
        const double* times = nullptr;
        rc = resident_side(c, &rings, &times);
        if (rc == LILIOM_OK) rc = rot_extract_dev(c, n, q_imu, q_lb ? q_lb : kIdentityQ, n_surf, n_edge, n_cut, rings, times);
    }
    c->raw_src = nullptr;
    return rc;
}

// The contexts of a batched call: distinct, single-GPU, on one device.
bool lili::batch_ctxs_ok(liliom_ctx* const* ctxs, int B) {
    if (B < 1 || !ctxs) return false;
    for (int i = 0; i < B; ++i) {
        const liliom_ctx* c = ctxs[i];
        if (!c || c->device != ctxs[0]->device || c->nranks > 1 || c->nccl_comm || c->peer_ready) return false;
        for (int j = 0; j < i; ++j) if (ctxs[j] == c) return false;
    }
    return true;
}

extern "C" int liliom_extract_resident_batch(liliom_ctx* const* ctxs, int B, const double* q_imu, const double* q_lb, int* n_surf,
                                             int* n_edge, int* n_cut, int* status) {
    if (!batch_ctxs_ok(ctxs, B) || !q_imu || !n_surf || !n_edge || !n_cut || !status) return LILIOM_E_ARG;
    liliom_ctx* c0 = ctxs[0];
    LILI_CUDA(c0, cudaSetDevice(c0->device));
    std::vector<HzBatchSession> hz;
    std::vector<RotBatchSession> rot;
    std::vector<int> hz_at, rot_at;         // index of each session in ctxs
    for (int i = 0; i < B; ++i) {
        liliom_ctx* c = ctxs[i];
        const int n = c->n_raw_scan;
        // the extractors only read their input: they take the resident sweep in place
        if (c->prm.point_stride == 48) {
            c->raw_src = n > 0 ? c->raw_scan.p : nullptr;
            hz.push_back(HzBatchSession{c, n, q_imu + 4 * i, n_surf + i, n_edge + i, n_cut + i, LILIOM_OK});
            hz_at.push_back(i);
            continue;
        }
        RotBatchSession s{c, n, q_imu + 4 * i, q_lb ? q_lb + 4 * i : kIdentityQ, nullptr, nullptr, n_surf + i, n_edge + i, n_cut + i,
                          LILIOM_OK, false};
        status[i] = resident_side(c, &s.rings, &s.times);
        if (status[i] != LILIOM_OK) continue;
        c->raw_src = n > 0 ? c->raw_scan.p : nullptr;
        rot.push_back(s);
        rot_at.push_back(i);
    }
    int rc = horizon_batch_queue(c0, hz);
    if (rc == LILIOM_OK) rc = rot_batch_queue(c0, rot);
    for (const HzBatchSession& s : hz) s.c->raw_src = nullptr;
    for (const RotBatchSession& s : rot) s.c->raw_src = nullptr;
    LILI_TRY(rc);
    for (size_t k = 0; k < hz.size(); ++k) status[hz_at[k]] = hz[k].status;
    // one synchronise for the whole call: every session's stream joins ctxs[0]'s
    LILI_TRY(batch_join_in(c0, std::vector<liliom_ctx*>(ctxs, ctxs + B)));
    LILI_CUDA(c0, cudaStreamSynchronize(c0->stream));
    for (size_t k = 0; k < rot.size(); ++k) status[rot_at[k]] = rot[k].pending ? rot_batch_finish(rot[k]) : rot[k].status;
    return LILIOM_OK;
}

extern "C" int liliom_features_download(liliom_ctx* c, void* surf, int surf_cap, int* n_surf, void* edge, int edge_cap, int* n_edge,
                                        void* cut, int cut_cap, int* n_cut) {
    if (!c || !n_surf || !n_edge || !n_cut) return LILIOM_E_ARG;
    FeatCloud f[3];
    LILI_TRY(feat_clouds(c, f));
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    int m[3];
    LILI_TRY(feat_sizes(c, f, m));
    *n_surf = m[0]; *n_edge = m[1]; *n_cut = m[2];
    void* out[3] = {surf, edge, cut};
    const int cap[3] = {surf_cap, edge_cap, cut_cap};
    for (int k = 0; k < 3; ++k) if (out[k] && m[k] > cap[k]) return LILIOM_E_CAPACITY;
    for (int k = 0; k < 3; ++k)
        if (out[k] && m[k] > 0) LILI_CUDA(c, cudaMemcpyAsync(out[k], f[k].buf->p, (size_t)m[k] * stride, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

// liliom_odometry_resident in three parts, shared by the solo and the batched call.
// 1. The scan VoxelGrid of the resident surf features into the queries.  *step: LILIOM_OK when the step may run, or the map's
//    refusal (LILIOM_E_NOMAP / LILIOM_E_FEWMAP).
static int odo_filter(liliom_ctx* c, bool spec_failed, int* step) {
    const int stride = c->prm.point_stride;
    // surf count: exact on the host (n_surf_dev >= 0) or only on the device (resident pipeline, no round trip)
    const int n_max = c->n_surf_dev >= 0 ? c->n_surf_dev : c->n_surf_max;
    const int* d_n = c->n_surf_dev >= 0 ? nullptr : c->d_nsurf;
    c->n_ds_resident = -1;      // until odo_finish: a call that fails before it leaves no scan for liliom_map_update_resident
    LILI_CUDA(c, c->vg_out.ensure((size_t)(n_max > 0 ? n_max : 1) * stride));
    LILI_CUDA(c, c->vg_count.ensure(16));
    LILI_CUDA(c, c->feats.ensure((size_t)(n_max > 0 ? n_max : 1) * sizeof(float4)));
    if (c->prm.leaf_scan > 0.0f) {
        // L/src/LidarOdometry.cpp:321-322; the centroid kernel also emits the float4 queries
        // speculate that the scan's voxel box has < 2^24 cells (a 200 m sweep at 0.4 m: ~2^21-2^23): one radix pass
        // less.  The box is read back with the pose; on a miss the step is redone with full-width keys, which are the wide ones
        // when the box's index wraps (vg_wide_keys).
        const int key_bits = spec_failed ? (c->vg_wide ? kVgWideKeyBits : 32) : n_max > 24576 ? 32 : 24;
        // scan-sized clouds take the single-launch cooperative filter; it may decline (VgParams::bail, read back with the pose)
        bool coop = false;
        if (!spec_failed)
            LILI_TRY(voxelgrid_coop(c, c->surf.p, n_max, d_n, stride, c->prm.leaf_scan, c->vg_out.p, c->vg_count.as<int>(), c->feats.as<float4>(), &coop));
        if (!coop)
            LILI_TRY(voxelgrid_dev(c, c->surf.p, n_max, d_n, stride, c->prm.leaf_scan, c->vg_out.p, c->vg_count.as<int>(), c->feats.as<float4>(), key_bits));
        c->d_nfeats = c->vg_count.as<int>();
        c->vg_used24 = !coop && key_bits < 32;
        c->vg_check = n_max > 0 && (coop || key_bits <= 32);   // an empty scan writes no vg_params: nothing of this call to read back
        c->vg_bail = false;
        c->vg_wide = false;
    } else {   // leaf_scan == 0: benchmark mode, every surf feature is a query
        if (n_max > 0) LILI_CUDA(c, cudaMemcpyAsync(c->vg_out.p, c->surf.p, (size_t)n_max * stride, cudaMemcpyDeviceToDevice, c->stream));
        LILI_TRY(repack_to_f4(c, c->surf.p, n_max, stride, c->feats.as<float4>(), d_n));
        c->d_nfeats = d_n;
    }
    c->n_feats = n_max;
    *step = !c->map.ready ? LILIOM_E_NOMAP : c->map_n_global < 10 ? LILIOM_E_FEWMAP : LILIOM_OK;
    return LILIOM_OK;
}

// 2. After a step that ran and returned rc: true when the VoxelGrid's speculation missed, and the call must be redone from its
//    start pose with the sort chain and full-width keys (spec_failed): 32-bit ones, or the wide ones when the box's index wraps.
//    Clears the check either way.
static bool odo_spec_missed(liliom_ctx* c, int rc, bool spec_failed) {
    const bool miss = rc == LILIOM_OK && c->vg_check &&
                      ((!spec_failed && (c->vg_bail || (c->vg_used24 && c->vg_ncells >= (1LL << 24) - 1))) || c->vg_wide);
    c->vg_check = false;
    if (miss) c->d_nfeats = nullptr;
    return miss;
}

// 3. The query count of a step that did not run (ran = false), and surf_last_ds: *n_ds and the optional download.
static int odo_finish(liliom_ctx* c, bool ran, int rc, void* ds_out, int ds_cap, int* n_ds) {
    if (!ran) {   // still report surf_last_ds: read the count back
        if (c->d_nfeats) {
            int nq = 0;
            LILI_TRY(read_back(c, {{&nq, c->d_nfeats, sizeof(int)}}));
            c->n_feats_actual = min(nq, c->n_feats);
        } else c->n_feats_actual = c->n_feats;
    }
    c->d_nfeats = nullptr;
    const int m = c->n_feats_actual;
    c->n_ds_resident = (!ran || rc == LILIOM_OK) ? m : -1;      // vg_out holds surf_last_ds, m points (liliom_map_update_resident)
    if (n_ds) *n_ds = m;
    if (ds_out) {
        if (m > ds_cap) return LILIOM_E_CAPACITY;
        if (m) {
            LILI_CUDA(c, cudaMemcpyAsync(ds_out, c->vg_out.p, (size_t)m * c->prm.point_stride, cudaMemcpyDeviceToHost, c->stream));
            LILI_CUDA(c, cudaStreamSynchronize(c->stream));
        }
    }
    return rc;
}

static int odometry_on_resident_surf(liliom_ctx* c, double pose7[7], int match_cnt, int max_num_iter, int mode, liliom_iter_stats* stats,
                                     void* ds_out, int ds_cap, int* n_ds, bool spec_failed) {
    if (!c || !pose7 || (mode != LILIOM_MODE_CERES && mode != LILIOM_MODE_GN) || match_cnt < 0) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    int rc = LILIOM_OK;
    LILI_TRY(odo_filter(c, spec_failed, &rc));
    const bool ran = rc == LILIOM_OK;
    double pose_in[7];
    memcpy(pose_in, pose7, sizeof(pose_in));
    if (ran) {
        rc = s2m_run(c, pose7, match_cnt, max_num_iter, mode, stats, false, nullptr);
        if (odo_spec_missed(c, rc, spec_failed)) {
            memcpy(pose7, pose_in, sizeof(pose_in));
            return odometry_on_resident_surf(c, pose7, match_cnt, max_num_iter, mode, stats, ds_out, ds_cap, n_ds, true);
        }
    }
    return odo_finish(c, ran, rc, ds_out, ds_cap, n_ds);
}

extern "C" int liliom_odometry_resident(liliom_ctx* c, double pose7[7], int match_cnt, int max_num_iter, int mode, liliom_iter_stats* stats,
                                        void* ds_out, int ds_cap, int* n_ds) {
    return odometry_on_resident_surf(c, pose7, match_cnt, max_num_iter, mode, stats, ds_out, ds_cap, n_ds);
}

// The whole-call refusals of the batched steps: nothing is touched when one holds.
static bool batch_args_ok(liliom_ctx* const* ctxs, int B, const double* poses7, const int* match_cnt, const int* max_num_iter, int mode,
                          const int* status) {
    if (!batch_ctxs_ok(ctxs, B) || !poses7 || !status || !match_cnt) return false;
    if (mode != LILIOM_MODE_CERES && mode != LILIOM_MODE_GN) return false;
    if (mode == LILIOM_MODE_CERES && !max_num_iter) return false;
    for (int i = 0; i < B; ++i)
        if (match_cnt[i] < 0) return false;
    return true;
}

extern "C" int liliom_scan_to_map_resident_batch_ex(liliom_ctx* const* ctxs, int B, double* poses7_inout, const int* match_cnt,
                                                    const int* max_num_iter, int mode, liliom_iter_stats* const* stats, int* status) {
    if (!batch_args_ok(ctxs, B, poses7_inout, match_cnt, max_num_iter, mode, status)) return LILIOM_E_ARG;
    LILI_CUDA(ctxs[0], cudaSetDevice(ctxs[0]->device));
    for (int i = 0; i < B; ++i) status[i] = LILIOM_OK;
    return s2m_batch(ctxs, B, poses7_inout, match_cnt, max_num_iter, mode, stats, status);
}

extern "C" int liliom_odometry_resident_batch_ex(liliom_ctx* const* ctxs, int B, double* poses7_inout, const int* match_cnt,
                                                 const int* max_num_iter, int mode, liliom_iter_stats* const* stats, void* const* ds_out,
                                                 const int* ds_cap, int* n_ds, int* status) {
    if (!batch_args_ok(ctxs, B, poses7_inout, match_cnt, max_num_iter, mode, status)) return LILIOM_E_ARG;
    LILI_CUDA(ctxs[0], cudaSetDevice(ctxs[0]->device));
    std::vector<int> step(B, LILIOM_OK);
    std::vector<char> filtered(B, 0);
    for (int i = 0; i < B; ++i) {
        status[i] = odo_filter(ctxs[i], false, &step[i]);
        filtered[i] = status[i] == LILIOM_OK;
        if (!filtered[i]) step[i] = status[i];
    }
    const std::vector<double> pose_in(poses7_inout, poses7_inout + (size_t)7 * B);
    std::vector<int> ran(step);
    LILI_TRY(s2m_batch(ctxs, B, poses7_inout, match_cnt, max_num_iter, mode, stats, step.data()));
    for (int i = 0; i < B; ++i) {
        if (!filtered[i]) continue;
        liliom_ctx* c = ctxs[i];
        double* pose = poses7_inout + 7 * i;
        liliom_iter_stats* st = stats ? stats[i] : nullptr;
        void* out = ds_out ? ds_out[i] : nullptr;
        const int cap = ds_cap ? ds_cap[i] : 0;
        int* nd = n_ds ? n_ds + i : nullptr;
        const bool did_run = ran[i] == LILIOM_OK;
        if (did_run && odo_spec_missed(c, step[i], false)) {       // the session's solo call redone from its start pose
            memcpy(pose, pose_in.data() + 7 * i, 7 * sizeof(double));
            status[i] = odometry_on_resident_surf(c, pose, match_cnt[i], max_num_iter ? max_num_iter[i] : 0, mode, st, out, cap, nd, true);
        } else status[i] = odo_finish(c, did_run, step[i], out, cap, nd);
    }
    return LILIOM_OK;
}

// The uniform-count GN calls: liliom_*_batch_ex with match_cnt for every session and stats + i*match_cnt.
struct UniformBatch {
    std::vector<int> cnt;
    std::vector<liliom_iter_stats*> st;
    UniformBatch(int B, int match_cnt, liliom_iter_stats* stats) : cnt(B, match_cnt), st(B) {
        for (int i = 0; i < B; ++i) st[i] = stats ? stats + (size_t)i * match_cnt : nullptr;
    }
};

extern "C" int liliom_scan_to_map_resident_batch(liliom_ctx* const* ctxs, int B, double* poses7_inout, int match_cnt,
                                                 liliom_iter_stats* stats, int* status) {
    if (B < 1 || match_cnt < 0) return LILIOM_E_ARG;
    const UniformBatch u(B, match_cnt, stats);
    return liliom_scan_to_map_resident_batch_ex(ctxs, B, poses7_inout, u.cnt.data(), nullptr, LILIOM_MODE_GN, stats ? u.st.data() : nullptr,
                                                status);
}

extern "C" int liliom_odometry_resident_batch(liliom_ctx* const* ctxs, int B, double* poses7_inout, int match_cnt,
                                              liliom_iter_stats* stats, void* const* ds_out, const int* ds_cap, int* n_ds, int* status) {
    if (B < 1 || match_cnt < 0) return LILIOM_E_ARG;
    const UniformBatch u(B, match_cnt, stats);
    return liliom_odometry_resident_batch_ex(ctxs, B, poses7_inout, u.cnt.data(), nullptr, LILIOM_MODE_GN, stats ? u.st.data() : nullptr,
                                             ds_out, ds_cap, n_ds, status);
}

extern "C" int liliom_find_surf_corr(liliom_ctx* c, const void* feats, int n, int stride, const double pose7[7], unsigned char* valid,
                                     float* plane, int* nn_idx, float* sqd, double out29[29]) {
    if (!c || !pose7) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    if (!c->map.ready) return LILIOM_E_NOMAP;
    if (c->map_n_global < 10) return LILIOM_E_FEWMAP;
    LILI_TRY(upload_feats(c, feats, n, stride));
    double p[7];
    memcpy(p, pose7, sizeof(p));
    LILI_TRY(s2m_run(c, p, 0, 0, LILIOM_MODE_GN, nullptr, true, out29));
    if (n > 0) {
        if (valid) LILI_CUDA(c, cudaMemcpyAsync(valid, c->corr_valid.p, (size_t)n, cudaMemcpyDeviceToHost, c->stream));
        if (plane) LILI_CUDA(c, cudaMemcpyAsync(plane, c->corr_plane.p, (size_t)n * 16, cudaMemcpyDeviceToHost, c->stream));
        if (nn_idx) LILI_CUDA(c, cudaMemcpyAsync(nn_idx, c->nn_idx.p, (size_t)n * 20, cudaMemcpyDeviceToHost, c->stream));
        if (sqd) LILI_CUDA(c, cudaMemcpyAsync(sqd, c->nn_sqd.p, (size_t)n * 20, cudaMemcpyDeviceToHost, c->stream));
        LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    }
    return LILIOM_OK;
}

// ===================== SURVEY §8 (f4): loop-closure alignment =====================
extern "C" int liliom_icp_align(liliom_ctx* c, const void* src, int n_src, const void* tgt, int n_tgt, int stride, double max_corr_dist,
                                int max_iter, double trans_eps, double fit_eps, double T16[16], double* fitness, int* converged, int* iters) {
    if (!c || n_src < 0 || n_tgt < 0 || (n_src > 0 && !src) || (n_tgt > 0 && !tgt) || !T16 || !fitness || !converged || !iters) return LILIOM_E_ARG;
    if ((stride != 16 && stride != 32 && stride != 48) || !(max_corr_dist > 0) || max_iter < 1) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    if (c->nranks > 1) { c->last_error = "liliom_icp_align is single-GPU"; return LILIOM_E_ARG; }
    // target -> the context's map (cell grid), source -> the resident query array
    c->inc_valid = false;
    LILI_TRY(map_install_host(c, tgt, n_tgt, stride, false));
    LILI_TRY(upload_feats(c, src, n_src, stride));
    return icp_align(c, c->map, c->feats.as<float4>(), n_src, max_corr_dist, max_iter, trans_eps, fit_eps, T16, fitness, converged, iters);
}

// ===================== wire format, publishing side =====================
// PCL's field tables (pc2_fields.h) as pcl::toROSMsg lists them
extern "C" int liliom_pc2_layout(int point_stride, liliom_pc2_field* fields, int cap, int* point_step) {
    if (point_stride != 48 && point_stride != 32) return LILIOM_E_ARG;
    const Pc2Name* src = point_stride == 48 ? kPc2Fields48 : kPc2Fields32;
    const int n = point_stride == 48 ? (int)(sizeof(kPc2Fields48) / sizeof(kPc2Fields48[0])) : kPc2Fields32N;
    if (point_step) *point_step = point_stride;
    if (!fields) return n;
    if (cap < n) return LILIOM_E_CAPACITY;
    for (int i = 0; i < n; ++i) {
        memset(&fields[i], 0, sizeof(fields[i]));
        strncpy(fields[i].name, src[i].name, sizeof(fields[i].name) - 1);
        fields[i].offset = src[i].offset; fields[i].datatype = kPc2Float32; fields[i].count = 1;
    }
    return n;
}

// ===================== instrumentation =====================
extern "C" int liliom_get_counters(liliom_ctx* c, liliom_counters* out, int reset) {
    if (!c || !out) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    unsigned long long dev[2] = {0, 0};       // examined candidates, searched queries: counted by the kernels themselves
    if (c->counter.p) {
        LILI_CUDA(c, cudaMemcpyAsync(dev, c->counter.as<unsigned char>() + 16, sizeof(dev), cudaMemcpyDeviceToHost, c->stream));
        LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    }
    c->cnt.knn_candidates = dev[0];
    c->cnt.knn_queries = dev[1];
    *out = c->cnt;
    if (reset) {
        c->cnt = liliom_counters{};
        if (c->counter.p) LILI_CUDA(c, cudaMemsetAsync(c->counter.as<unsigned char>() + 16, 0, 16, c->stream));
    }
    return LILIOM_OK;
}

extern "C" int liliom_knn_block_stats(liliom_ctx* c, const double pose7[7], unsigned long long out2[2]) {
    if (!c || !pose7 || !out2) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    return block27_stats(c, pose7, out2);
}

extern "C" int liliom_set_kernel_timing(liliom_ctx* c, int on) {
    if (!c) return LILIOM_E_ARG;
    c->time_kernels = on != 0;
    c->time_every = on > 1 ? on : 1;
    c->time_calls = 0;
    return LILIOM_OK;
}
