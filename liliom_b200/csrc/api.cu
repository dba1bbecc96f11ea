// C ABI of libliliom_b200.so (see include/liliom.h for the contract and reference citations).
#include "ctx.cuh"
#include "dev_math.cuh"
#include "knn_core.cuh"
#include "pc2_fields.h"
#include <new>
#include <cstdlib>
#include <ctime>

namespace lili {
void nccl_destroy(liliom_ctx* c);
int nccl_allreduce_sum_f64(liliom_ctx* c, double* buf, int count);

// ---- map sharding (multi-GPU): keep a point when any shard block (cube of 1/inv_block metres, default 16 m) touched by its
// halo box is owned by `rank` (same hash as owner_of() in knn_core.cuh)
__global__ void k_shard_flags(const float4* __restrict__ p, int n, float halo, float inv_block, int nranks, int rank, int* __restrict__ flags) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    int f = 0;
    if (i < n) {
        float4 v = p[i];
        for (int c = 0; c < 8 && !f; ++c) {
            float x = v.x + ((c & 1) ? halo : -halo), y = v.y + ((c & 2) ? halo : -halo), z = v.z + ((c & 4) ? halo : -halo);
            if (owner_of(x, y, z, nranks, inv_block) == rank) f = 1;
        }
    }
    flags[i] = f;
}
// same rule on PCL-layout points (stride bytes): used by the sharded liliom_map_push_frame
__global__ void k_shard_flags_strided(const unsigned char* __restrict__ p, int n, int stride, float halo, float inv_block, int nranks, int rank,
                                      int* __restrict__ flags) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    int f = 0;
    if (i < n) {
        const float4 v = *reinterpret_cast<const float4*>(p + (size_t)i * stride);
        for (int c = 0; c < 8 && !f; ++c) {
            float x = v.x + ((c & 1) ? halo : -halo), y = v.y + ((c & 2) ? halo : -halo), z = v.z + ((c & 4) ? halo : -halo);
            if (owner_of(x, y, z, nranks, inv_block) == rank) f = 1;
        }
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

__global__ void k_compact_f4(const float4* __restrict__ in, const int* __restrict__ flags, const int* __restrict__ pos, int n, float4* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && flags[i]) out[pos[i]] = in[i];
}

// transformCloud (L/src/LidarOdometry.cpp:246-278; R/src/LidarOdometry.cpp:239-264)
__global__ void k_transform_cloud(const unsigned char* __restrict__ in, int n, int stride, Q4 q, D3 t, unsigned char* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    pcl_transform_point(in + (size_t)i * stride, stride, q, t, out + (size_t)i * stride);
}

// Concatenation of the FIFO frames (L/src/LidarOdometry.cpp:301-302) in ONE launch: blockIdx.y = frame, the blocks of a row
// stream that frame's 16-byte words to its offset in the concatenated cloud.  (20 cudaMemcpyAsync calls cost a fixed
// latency per copy whatever the size, which a single launch does not.)
constexpr int kConcatMax = 64;
struct ConcatTab { const float4* src[kConcatMax]; long long off[kConcatMax + 1]; };      // offsets in 16-byte words
__global__ void k_concat_frames(const __grid_constant__ ConcatTab tab, float4* __restrict__ out) {
    const int f = blockIdx.y;
    const long long n16 = tab.off[f + 1] - tab.off[f];
    const float4* __restrict__ src = tab.src[f];
    float4* __restrict__ dst = out + tab.off[f];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i];
}
// sharded rebuild: the shard filter and the repack to float4 {x,y,z,index} in one pass over the VoxelGrid output
__global__ void k_compact_repack(const unsigned char* __restrict__ in, const int* __restrict__ flags, const int* __restrict__ pos, int n, int stride,
                                 float4* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !flags[i]) return;
    float4 v = *reinterpret_cast<const float4*>(in + (size_t)i * stride);
    v.w = __int_as_float(i);
    out[pos[i]] = v;
}

// LidarOdometry::undistortion (L/src/LidarOdometry.cpp:178-199), in place on device points
__global__ void k_undistort(unsigned char* __restrict__ pts, int n, int stride, D3 trans, Q4 quat) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float4* p0 = reinterpret_cast<float4*>(pts + (size_t)i * stride);
    float4 a = p0[0];
    const float intensity = *reinterpret_cast<const float*>(pts + (size_t)i * stride + (stride == 48 ? 32 : 16));
    const int line = (int)intensity;                                                    // :181
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

static int install_map_from_xyzw(liliom_ctx* c, int m) {
    // c->map.xyzw holds m float4 (w = global index).  Shard when a communicator is attached.
    c->map_n_global = m;
    if (c->nranks > 1 && m > 0) {
        LILI_CUDA(c, c->flags.ensure(((size_t)m + 2) * 4));
        LILI_CUDA(c, c->idx_a.ensure(((size_t)m + 2) * 4));
        LILI_CUDA(c, c->map_ds.ensure((size_t)m * sizeof(float4)));
        const float cell = gate_cell(c->prm.knn_max_sqdist);
        k_shard_flags<<<cdiv(m + 1, 256), 256, 0, c->stream>>>(c->map.xyzw.as<float4>(), m, cell, c->shard_inv_block, c->nranks, c->rank, c->flags.as<int>());
        LILI_TRY(launch_check(c, "k_shard_flags"));
        LILI_TRY(exclusive_scan_i32(c, c->flags.as<int>(), c->idx_a.as<int>(), m));
        k_compact_f4<<<cdiv(m, 256), 256, 0, c->stream>>>(c->map.xyzw.as<float4>(), c->flags.as<int>(), c->idx_a.as<int>(), m, c->map_ds.as<float4>());
        LILI_TRY(launch_check(c, "k_compact_f4"));
        int local = 0;
        LILI_TRY(read_back(c, {{&local, c->idx_a.as<int>() + m, sizeof(int)}}));
        LILI_CUDA(c, cudaMemcpyAsync(c->map.xyzw.p, c->map_ds.p, (size_t)local * sizeof(float4), cudaMemcpyDeviceToDevice, c->stream));
        m = local;
    }
    return grid_build(c, m);
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
    c->h_pin_bytes = sizeof(PinBlock) + (1 << 20);      // the header + 1 MiB of per-iteration stats (3276 iterations)
    if (e == cudaSuccess) e = cudaHostAlloc((void**)&c->h_pin, c->h_pin_bytes, cudaHostAllocDefault);
    if (e != cudaSuccess) { liliom_destroy(c); return LILIOM_E_CUDA; }      // tears down whatever was created
    // the GN kernel writes its results straight into this block when the device can address it (UVA: always, in practice)
    if (cudaHostGetDevicePointer((void**)&c->h_pin_dev, c->h_pin, 0) != cudaSuccess) { c->h_pin_dev = nullptr; (void)cudaGetLastError(); }
    if (const char* e1 = getenv("LILIOM_KNN_LANES")) { int v = atoi(e1); if (v == 1 || v == 2 || v == 4 || v == 8 || v == 16) c->force_lanes = v; }
    c->dbg_timing = getenv("LILIOM_DEBUG_TIMING") != nullptr;
    c->rot_slow_walk = getenv("LILIOM_ROT_SLOW_WALK") != nullptr;
    c->test_shrink_box = getenv("LILIOM_TEST_SHRINK_BOX") != nullptr;
    if (const char* e8 = getenv("LILIOM_KNN_TMA")) c->knn_tma = atoi(e8) != 0;
    if (const char* e5 = getenv("LILIOM_GN_SYNC")) { int v = atoi(e5); if (v == 0 || v == 1 || v == 3) c->gn_sync = v; }
    if (const char* e4 = getenv("LILIOM_SHARD_BLOCK")) {      // shard block edge in metres (power of two, 8..256): larger blocks = thinner halos
        int v = atoi(e4);
        if (v >= 8 && v <= 256 && (v & (v - 1)) == 0) c->shard_inv_block = 1.0f / (float)v;
    }
    if (const char* e2 = getenv("LILIOM_KNN_ROUNDS")) { int v = atoi(e2); if (v >= 1 && v <= 32) c->force_rounds = v; }
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

// ---- (f3) FormatConvert on the device: livox_ros_driver::CustomPoint[] -> pcl::PointXYZINormal[] (L/src/FormatConvert.cpp:11-24)
namespace lili {
// little-endian 32-bit word assembled from bytes: sensor payloads carry fields at any byte offset, never read them wider
__device__ __forceinline__ unsigned rd32(const unsigned char* p) {
    return (unsigned)p[0] | ((unsigned)p[1] << 8) | ((unsigned)p[2] << 16) | ((unsigned)p[3] << 24);
}
__global__ void k_livox_to_pt48(const unsigned char* __restrict__ in, int n, int stride, float4* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned time_end = rd32(in + (size_t)(n - 1) * stride);                       // :13 points.back().offset_time
    const unsigned char* p = in + (size_t)i * stride;
    const unsigned off = rd32(p);
    const float x = __uint_as_float(rd32(p + 4)), y = __uint_as_float(rd32(p + 8)), z = __uint_as_float(rd32(p + 12));
    const unsigned refl = p[16], line = p[18];
    const float s = __fdiv_rn(__uint2float_rn(off), __uint2float_rn(time_end));          // :19 float(offset_time / (float)time_end)
    const float intensity = (float)addx((double)line, mulx((double)s, 0.1));            // :20
    const float curvature = (float)mulx(0.1, (double)refl);                             // :21
    out[3 * (size_t)i] = make_float4(x, y, z, 1.0f);                                    // pcl::PointXYZINormal default ctor: data[3] = 1
    out[3 * (size_t)i + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
    out[3 * (size_t)i + 2] = make_float4(intensity, curvature, 0.f, 0.f);
}
static int livox_to_dev(liliom_ctx* c, const void* custom_pts, int n, int stride, void* d_out48) {
    if (n <= 0) return LILIOM_OK;
    LILI_CUDA(c, c->wire_in.ensure((size_t)n * stride));
    LILI_CUDA(c, cudaMemcpyAsync(c->wire_in.p, custom_pts, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream));
    k_livox_to_pt48<<<cdiv(n, 256), 256, 0, c->stream>>>((const unsigned char*)c->wire_in.p, n, stride, (float4*)d_out48);
    return launch_check(c, "k_livox_to_pt48");
}
}  // namespace lili

extern "C" int liliom_convert_livox(liliom_ctx* c, const void* custom_pts, int n, int stride, liliom_pt48* out, int cap) {
    if (!c || n < 0 || (n > 0 && !custom_pts) || (stride != 19 && stride != 20)) return LILIOM_E_ARG;
    if (c->prm.point_stride != 48) return LILIOM_E_ARG;
    if (out && n > cap) return LILIOM_E_CAPACITY;
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_CUDA(c, c->raw_scan.ensure((size_t)(n > 0 ? n : 1) * 48));
    LILI_TRY(livox_to_dev(c, custom_pts, n, stride, c->raw_scan.p));
    c->n_raw_scan = n;
    c->raw_scan_rings = false;
    c->raw_scan_times = false;
    if (out && n) LILI_CUDA(c, cudaMemcpyAsync(out, c->raw_scan.p, (size_t)n * 48, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

extern "C" int liliom_extract_horizon_livox(liliom_ctx* c, const void* custom_pts, int n, int stride, const double q_imu[4],
                                            liliom_pt48* surf_out, int surf_cap, int* n_surf, liliom_pt48* edge_out, int edge_cap, int* n_edge,
                                            liliom_pt48* cut_out, int cut_cap, int* n_cut) {
    if (!c || n < 0 || (n > 0 && !custom_pts) || (stride != 19 && stride != 20) || !q_imu || !n_surf || !n_edge || !n_cut) return LILIOM_E_ARG;
    if (c->prm.point_stride != 48) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_CUDA(c, c->raw.ensure((size_t)(n > 0 ? n : 1) * 48));
    LILI_TRY(livox_to_dev(c, custom_pts, n, stride, c->raw.p));
    return extract_horizon_from_raw(c, n, q_imu, surf_out, surf_cap, n_surf, edge_out, edge_cap, n_edge, cut_out, cut_cap, n_cut);
}

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

// ---- (f3) pcl::fromROSMsg(PointCloud2 -> pcl::PointXYZI) on the device (R/src/Preprocessing.cpp:277); field matching: pc2_fields.h
namespace lili {
// One thread per point, row-major over (row, column).  src = Pc2Map::src of x, y, z, intensity (-1: unmapped -> 0).
// Kept a pass of its own rather than fused into k_rot_pre: k_rot_hp and k_rot_build read the decoded sweep again.
// ring_out (LILIOM_RING_FIELD only; nullptr otherwise, a uniform branch): the point's `ring` field (Pc2Map::ring_src / ring_bytes).
// time_out (LILIOM_TIME_FIELD only; nullptr otherwise, a uniform branch): the point's time field as double (Pc2Map::time_src /
// time_type).
__global__ void k_pc2_to_pt32(const unsigned char* __restrict__ in, int n, unsigned width, unsigned point_step, unsigned row_step, int4 src,
                              float4* __restrict__ out, int2 ring, uint16_t* __restrict__ ring_out, int2 tm, double* __restrict__ time_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned r = (unsigned)i / width, col = (unsigned)i - r * width;
    const unsigned char* p = in + (size_t)r * row_step + (size_t)col * point_step;
    auto fld = [p](int off) { return off < 0 ? 0.0f : __uint_as_float(rd32(p + off)); };
    out[2 * (size_t)i] = make_float4(fld(src.x), fld(src.y), fld(src.z), 1.0f);          // pcl::PointXYZI default ctor: data[3] = 1
    out[2 * (size_t)i + 1] = make_float4(fld(src.w), 0.f, 0.f, 0.f);
    if (ring_out) ring_out[i] = (uint16_t)pc2_ring_value(p, ring.x, ring.y);
    if (time_out) time_out[i] = pc2_time_value(p, tm.x, tm.y);
}
// msg already accepted by pc2_match (m): stage the payload, decode into d_out32 (m.n points of 32 bytes) and, when d_ring is
// given (m matched with want_ring), the ring ids into d_ring (m.n u16), when d_time is given (m matched with a time name), the
// times into d_time (m.n double)
static int pc2_to_dev(liliom_ctx* c, const liliom_pc2_msg* msg, const Pc2Map& m, void* d_out32, uint16_t* d_ring, double* d_time) {
    if (m.n <= 0) return LILIOM_OK;
    const size_t bytes = (size_t)msg->height * msg->row_step;
    LILI_CUDA(c, c->wire_in.ensure(bytes));
    LILI_CUDA(c, cudaMemcpyAsync(c->wire_in.p, msg->data, bytes, cudaMemcpyHostToDevice, c->stream));
    k_pc2_to_pt32<<<cdiv(m.n, 256), 256, 0, c->stream>>>((const unsigned char*)c->wire_in.p, m.n, msg->width, msg->point_step, msg->row_step,
                                                          make_int4(m.src[0], m.src[1], m.src[2], m.src[3]), (float4*)d_out32,
                                                          make_int2(m.ring_src, m.ring_bytes), d_ring, make_int2(m.time_src, m.time_type),
                                                          d_time);
    return launch_check(c, "k_pc2_to_pt32");
}
}  // namespace lili

// the name of the time field a context reads (LILIOM_TIME_FIELD), or nullptr (LILIOM_TIME_AZIMUTH: no time field is looked at)
static const char* time_field_of(const liliom_ctx* c) {
    return c && c->time_source == LILIOM_TIME_FIELD ? c->time_name : nullptr;
}

extern "C" int liliom_convert_pc2(liliom_ctx* c, const liliom_pc2_msg* msg, liliom_pt32* out, int cap, int* n) {
    Pc2Map m;
    const bool field = c && c->ring_source == LILIOM_RING_FIELD;
    const char* tname = time_field_of(c);
    if (!c || !n || pc2_match(msg, &m, field, tname) != LILIOM_OK) return LILIOM_E_ARG;
    if (c->prm.point_stride != 32) return LILIOM_E_ARG;
    if (out && m.n > cap) { *n = m.n; return LILIOM_E_CAPACITY; }
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_CUDA(c, c->raw_scan.ensure((size_t)(m.n > 0 ? m.n : 1) * 32));
    c->raw_scan_rings = false;
    c->raw_scan_times = false;
    if (field) LILI_CUDA(c, c->raw_scan_ring.ensure((size_t)(m.n > 0 ? m.n : 1) * sizeof(uint16_t)));
    if (tname) LILI_CUDA(c, c->raw_scan_time.ensure((size_t)(m.n > 0 ? m.n : 1) * sizeof(double)));
    LILI_TRY(pc2_to_dev(c, msg, m, c->raw_scan.p, field ? c->raw_scan_ring.as<uint16_t>() : nullptr,
                        tname ? c->raw_scan_time.as<double>() : nullptr));
    c->n_raw_scan = m.n;
    c->raw_scan_rings = field;
    c->raw_scan_times = tname != nullptr;
    if (out && m.n) LILI_CUDA(c, cudaMemcpyAsync(out, c->raw_scan.p, (size_t)m.n * 32, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    *n = m.n;
    return LILIOM_OK;
}

extern "C" int liliom_extract_rot_pc2(liliom_ctx* c, const liliom_pc2_msg* msg, const double q_imu[4], const double q_lb[4],
                                      liliom_pt32* surf_out, int surf_cap, int* n_surf, liliom_pt32* edge_out, int edge_cap, int* n_edge,
                                      liliom_pt32* cut_out, int cut_cap, int* n_cut) {
    Pc2Map m;
    const bool field = c && c->ring_source == LILIOM_RING_FIELD;
    const char* tname = time_field_of(c);
    if (!c || !q_imu || !q_lb || !n_surf || !n_edge || !n_cut || pc2_match(msg, &m, field, tname) != LILIOM_OK) return LILIOM_E_ARG;
    if (c->prm.point_stride != 32) return LILIOM_E_ARG;
    if (field && !rot_lines_ok(c->prm.line_num, true)) return LILIOM_E_LINES;
    LILI_CUDA(c, cudaSetDevice(c->device));
    LILI_CUDA(c, c->raw.ensure((size_t)(m.n > 0 ? m.n : 1) * 32));
    if (field) LILI_CUDA(c, c->raw_ring.ensure((size_t)(m.n > 0 ? m.n : 1) * sizeof(uint16_t)));
    if (tname) LILI_CUDA(c, c->raw_time.ensure((size_t)(m.n > 0 ? m.n : 1) * sizeof(double)));
    uint16_t* rings = field ? c->raw_ring.as<uint16_t>() : nullptr;
    double* times = tname ? c->raw_time.as<double>() : nullptr;
    LILI_TRY(pc2_to_dev(c, msg, m, c->raw.p, rings, times));
    return extract_rot_from_raw(c, m.n, q_imu, q_lb, surf_out, surf_cap, n_surf, edge_out, edge_cap, n_edge, cut_out, cut_cap, n_cut, rings,
                                times);
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
    LILI_CUDA(c, c->vg_out.ensure((size_t)n * stride));
    LILI_CUDA(c, c->vg_count.ensure(16));
    LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, pts, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream));
    bool coop = false;
    LILI_TRY(voxelgrid_coop(c, c->raw.p, n, nullptr, stride, leaf, c->vg_out.p, c->vg_count.as<int>(), nullptr, &coop));
    int m = 0;
    if (coop) {      // the cooperative filter may decline the input: its verdict comes back with the count
        VgParams vp;
        LILI_TRY(read_back(c, {{&m, c->vg_count.p, sizeof(int)}, {&vp, c->vg_params.p, sizeof(VgParams)}}));
        if (vp.bail) coop = false;
    }
    if (!coop) {
        LILI_TRY(voxelgrid_dev(c, c->raw.p, n, nullptr, stride, leaf, c->vg_out.p, c->vg_count.as<int>()));
        LILI_TRY(read_back(c, {{&m, c->vg_count.p, sizeof(int)}}));
    }
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
    k_undistort<<<cdiv(n, 256), 256, 0, c->stream>>>((unsigned char*)c->raw.p, n, stride, D3{trans[0], trans[1], trans[2]},
                                                    Q4{quat_wxyz[0], quat_wxyz[1], quat_wxyz[2], quat_wxyz[3]});
    LILI_TRY(launch_check(c, "k_undistort"));
    LILI_CUDA(c, cudaMemcpyAsync(pts_inout, c->raw.p, (size_t)n * stride, cudaMemcpyDeviceToHost, c->stream));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

// ===================== L2: map =====================
extern "C" int liliom_map_clear(liliom_ctx* c) {
    if (!c) return LILIOM_E_ARG;
    c->frames.clear();
    c->inc_valid = false;
    c->map.ready = false; c->map.n = 0; c->map_n_global = 0;
    return LILIOM_OK;
}

// Shared body of the two push_frame entry points: d_src = n body-frame points of point_stride bytes ON THE DEVICE.
static int push_frame_from_device(liliom_ctx* c, const void* d_src, int n, const double pose7[7], bool keep_inc = false) {
    const int stride = c->prm.point_stride;
    if (!keep_inc) c->inc_valid = false;        // the entry array of liliom_map_update no longer describes the FIFO
    Frame f;
    f.slot = (int)c->frames.size();
    if ((int)c->frames.size() >= c->prm.max_map_frames && !c->frames.empty()) {      // L/src/LidarOdometry.cpp:293-296 pop_front
        f.buf = std::move(c->frames.front().buf);   // the popped frame's allocation is recycled: cudaFree + cudaMalloc per scan cost
        f.slot = c->frames.front().slot;        // more than the whole map maintenance of a 10 M-point map (cudaFree synchronises)
        c->frames.erase(c->frames.begin());
    }
    f.n = n;
    int rc = LILIOM_OK;
    if (n > 0) {
        Q4 q{pose7[0], pose7[1], pose7[2], pose7[3]};
        D3 t{pose7[4], pose7[5], pose7[6]};
        auto body = [&]() -> int {
            LILI_CUDA(c, f.buf.ensure((size_t)n * stride));
            if (c->nranks == 1) {
                k_transform_cloud<<<cdiv(n, 256), 256, 0, c->stream>>>((const unsigned char*)d_src, n, stride, q, t, (unsigned char*)f.buf.p);
                LILI_TRY(launch_check(c, "k_transform_cloud"));
                LILI_TRY(vg_minmax_dev(c, f.buf.p, n, nullptr, stride));                 // the frame's box, for the rebuilds it takes part in
                return read_back(c, {{f.mm, c->vg_minmax.p, 7 * sizeof(int)}});
            }
            // sharded map maintenance: every rank receives the frame, keeps the points within (search radius + one voxel
            // diagonal) of a block it owns — every voxel that can reach an owned query's 1 m ball is then complete locally —
            // and voxel-filters / indexes only its shard.  No inter-rank traffic.
            LILI_CUDA(c, c->map_ds.ensure((size_t)n * stride));
            LILI_CUDA(c, c->flags.ensure(((size_t)n + 2) * 4));
            LILI_CUDA(c, c->idx_a.ensure(((size_t)n + 2) * 4));
            k_transform_cloud<<<cdiv(n, 256), 256, 0, c->stream>>>((const unsigned char*)d_src, n, stride, q, t, (unsigned char*)c->map_ds.p);
            LILI_TRY(launch_check(c, "k_transform_cloud"));
            const float halo = gate_cell(c->prm.knn_max_sqdist) + 1.7320508f * c->prm.leaf_map + 0.05f;
            k_shard_flags_strided<<<cdiv(n + 1, 256), 256, 0, c->stream>>>((const unsigned char*)c->map_ds.p, n, stride, halo, c->shard_inv_block, c->nranks, c->rank, c->flags.as<int>());
            LILI_TRY(launch_check(c, "k_shard_flags_strided"));
            LILI_TRY(exclusive_scan_i32(c, c->flags.as<int>(), c->idx_a.as<int>(), n));
            k_compact_strided<<<cdiv(n, 256), 256, 0, c->stream>>>((const unsigned char*)c->map_ds.p, c->flags.as<int>(), c->idx_a.as<int>(), n, stride,
                                                                  (unsigned char*)f.buf.p);
            LILI_TRY(launch_check(c, "k_compact_strided"));
            LILI_TRY(vg_minmax_dev(c, f.buf.p, n, c->idx_a.as<int>() + n, stride));     // box of the points this rank keeps
            return read_back(c, {{&f.n, c->idx_a.as<int>() + n, sizeof(int)}, {f.mm, c->vg_minmax.p, 7 * sizeof(int)}});
        };
        rc = body();
    }
    if (rc != LILIOM_OK) return rc;
    c->frames.push_back(std::move(f));
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

namespace lili {
// tail shared by the rebuild and the incremental update (single GPU): c->map_ds holds m filtered points
void frames_box(const liliom_ctx* c, int mm[kBoxInts]) {
    for (int k = 0; k < kBoxInts; ++k) mm[k] = vg_box_empty(k);
    for (const auto& f : c->frames) vg_box_merge(mm, f.mm);
}

int map_finish_from_ds(liliom_ctx* c, int m) {
    const int stride = c->prm.point_stride;
    LILI_CUDA(c, c->map.xyzw.ensure((size_t)(m > 0 ? m : 1) * sizeof(float4)));
    c->map_n_global = m;
    LILI_TRY(repack_to_f4(c, c->map_ds.p, m, stride, c->map.xyzw.as<float4>()));
    int mm[7];
    frames_box(c, mm);
    LILI_TRY(grid_build(c, m, mm[6] > 0 ? mm : nullptr));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}
}  // namespace lili

extern "C" int liliom_map_rebuild(liliom_ctx* c, int* n_map_out);

// SURVEY §8 (f2): push + incremental refresh (map_inc.cu); same result as liliom_map_push_frame + liliom_map_rebuild
static int map_update_from_device(liliom_ctx* c, const void* d_src, int n, const double pose7[7], int* n_map_out) {
    if (n_map_out) *n_map_out = 0;
    const bool incremental = c->nranks == 1 && c->prm.max_map_frames <= 64 && n < (1 << 24);
    int popped_slot = -1, popped_nfin = 0;
    if ((int)c->frames.size() >= c->prm.max_map_frames && !c->frames.empty()) { popped_slot = c->frames.front().slot; popped_nfin = c->frames.front().mm[6]; }
    LILI_TRY(push_frame_from_device(c, d_src, n, pose7, incremental));
    if (incremental) {
        c->map.ready = false; c->map.n = 0; c->map_n_global = 0;
        int m = 0;
        const int rc = map_inc_update(c, popped_slot, popped_nfin, &m);
        if (rc == LILIOM_OK) {
            LILI_TRY(map_finish_from_ds(c, m));
            if (n_map_out) *n_map_out = m;
            return LILIOM_OK;
        }
        c->inc_valid = false;
        if (rc != LILIOM_E_GRID) return rc;       // E_GRID: keys not representable / PCL's overflow case -> the sort chain decides
    }
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

// surf_from_map_ds as a point cloud (all fields), in liliom_map_download order
extern "C" int liliom_map_download_cloud(liliom_ctx* c, void* out, int cap, int* m_out) {
    if (!c || !m_out) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    if (c->nranks > 1) { c->last_error = "liliom_map_download_cloud is single-GPU"; return LILIOM_E_ARG; }
    return download_sized(c, c->map_ds, c->map_n_global, c->prm.point_stride, out, cap, m_out);
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
    c->map.ready = false; c->map.n = 0; c->map_n_global = 0;
    if (n_map_out) *n_map_out = 0;
    if (total == 0 && c->nranks == 1) { c->map.ready = true; return LILIOM_OK; }
    LILI_CUDA(c, c->map_raw.ensure((total > 0 ? total : 1) * stride));
    LILI_CUDA(c, c->map_ds.ensure((total > 0 ? total : 1) * stride));
    LILI_CUDA(c, c->vg_count.ensure(16));
    // bounding box and finite count of the concatenation = union over the frames (each measured once, at its push)
    int box[7];
    frames_box(c, box);
    // single GPU: the centroid kernel writes the float4 map itself (no repack pass); at most `total` voxels
    if (c->nranks == 1) LILI_CUDA(c, c->map.xyzw.ensure((total > 0 ? total : 1) * sizeof(float4)));
    size_t off = 0;
    if (c->frames.size() <= (size_t)kConcatMax && total > 0) {
        ConcatTab tab{};
        int k = 0;
        size_t largest = 0;
        for (auto& f : c->frames) {
            tab.src[k] = (const float4*)f.buf.p; tab.off[k] = (long long)(off * (stride / 16));
            off += (size_t)f.n; largest = f.n > (int)largest ? (size_t)f.n : largest; ++k;
        }
        for (; k <= kConcatMax; ++k) tab.off[k] = (long long)(off * (stride / 16));
        const int bx = max(1, min(cdiv((long long)largest * (stride / 16), 256 * 4), c->sm_count * 4));
        k_concat_frames<<<dim3(bx, (unsigned)c->frames.size()), 256, 0, c->stream>>>(tab, (float4*)c->map_raw.p);
        LILI_TRY(launch_check(c, "k_concat_frames"));
    } else
    for (auto& f : c->frames) {                                                    // :301-302 concatenation, oldest first
        if (f.n) LILI_CUDA(c, cudaMemcpyAsync((unsigned char*)c->map_raw.p + off * stride, f.buf.p, (size_t)f.n * stride, cudaMemcpyDeviceToDevice, c->stream));
        off += (size_t)f.n;
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
    if (c->nranks > 1) {
        // Every rank ENTERS the all-reduce whatever happened locally (a rank that returned early would leave its peers waiting
        // in the collective): the local status travels as a second scalar and all ranks fail together.
        // Shard filter: drops the (possibly incomplete) voxels beyond the 1-cell halo, fused with the repack to float4.
        auto shard_and_index = [&]() -> int {
            int local = 0;
            if (m > 0) {
                LILI_CUDA(c, c->flags.ensure(((size_t)m + 2) * 4));
                LILI_CUDA(c, c->idx_a.ensure(((size_t)m + 2) * 4));
                k_shard_flags_strided<<<cdiv(m + 1, 256), 256, 0, c->stream>>>((const unsigned char*)c->map_ds.p, m, stride, gate_cell(c->prm.knn_max_sqdist),
                                                                             c->shard_inv_block, c->nranks, c->rank, c->flags.as<int>());
                LILI_TRY(launch_check(c, "k_shard_flags_strided"));
                LILI_TRY(exclusive_scan_i32(c, c->flags.as<int>(), c->idx_a.as<int>(), m));
                k_compact_repack<<<cdiv(m, 256), 256, 0, c->stream>>>((const unsigned char*)c->map_ds.p, c->flags.as<int>(), c->idx_a.as<int>(), m, stride,
                                                                     c->map.xyzw.as<float4>());
                LILI_TRY(launch_check(c, "k_compact_repack"));
                LILI_TRY(read_back(c, {{&local, c->idx_a.as<int>() + m, sizeof(int)}}));
            }
            return grid_build(c, local, box[6] > 0 ? box : nullptr);
        };
        const int rc_local = shard_and_index();
        mark();  // [3] shard filter + cell grid
        // the "< 10 map points" guard (L/src/LidarOdometry.cpp:485-488) is about the whole map: sum the owned-voxel counts
        LILI_CUDA(c, c->neq.ensure(32 * sizeof(double)));
        double* pin = c->h_pin->map_status;
        pin[0] = rc_local == LILIOM_OK ? (double)c->map.n : 0.0;
        pin[1] = rc_local == LILIOM_OK ? 0.0 : 1.0;
        LILI_CUDA(c, cudaMemcpyAsync(c->neq.p, pin, 2 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
        LILI_TRY(nccl_allreduce_sum_f64(c, c->neq.as<double>(), 2));
        LILI_CUDA(c, cudaMemcpyAsync(pin + 2, c->neq.p, 2 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        LILI_CUDA(c, cudaStreamSynchronize(c->stream));
        if (rc_local != LILIOM_OK) return rc_local;
        if (pin[3] != 0.0) { c->map.ready = false; c->last_error = "liliom_map_rebuild failed on another rank"; return LILIOM_E_NCCL; }
        c->map_n_global = (int)pin[2];                  // halo voxels are counted on several ranks: an upper bound >= the true size
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

extern "C" int liliom_map_set_points(liliom_ctx* c, const liliom_f4* xyzw, int m) {
    if (!c || m < 0 || (m > 0 && !xyzw)) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    c->map.refl.release();
    c->map.ready = false;
    LILI_CUDA(c, c->map.xyzw.ensure((size_t)(m > 0 ? m : 1) * sizeof(float4)));
    LILI_CUDA(c, c->raw.ensure((size_t)(m > 0 ? m : 1) * sizeof(float4)));
    if (m > 0) {
        LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, xyzw, (size_t)m * sizeof(float4), cudaMemcpyHostToDevice, c->stream));
        LILI_TRY(repack_to_f4(c, c->raw.p, m, 16, c->map.xyzw.as<float4>()));
    }
    LILI_TRY(install_map_from_xyzw(c, m));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

// Install a PCL-layout cloud as the map, keeping its reflectivity channel for the Horizon backend variant.
extern "C" int liliom_map_set_cloud(liliom_ctx* c, const void* pts, int m, int stride) {
    if (!c || m < 0 || (m > 0 && !pts) || (stride != 48 && stride != 32)) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    if (c->nranks > 1) { c->last_error = "liliom_map_set_cloud is single-GPU"; return LILIOM_E_ARG; }
    c->map.ready = false;
    LILI_CUDA(c, c->map.xyzw.ensure((size_t)(m > 0 ? m : 1) * sizeof(float4)));
    LILI_CUDA(c, c->map.refl.ensure((size_t)(m > 0 ? m : 1) * sizeof(float)));
    LILI_CUDA(c, c->raw.ensure((size_t)(m > 0 ? m : 1) * stride));
    if (m > 0) {
        LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, pts, (size_t)m * stride, cudaMemcpyHostToDevice, c->stream));
        LILI_TRY(repack_to_f4(c, c->raw.p, m, stride, c->map.xyzw.as<float4>()));
        if (stride == 48) {
            k_kf_refl<<<cdiv(m, 256), 256, 0, c->stream>>>((const unsigned char*)c->raw.p, m, c->map.refl.as<float>());
            LILI_TRY(launch_check(c, "k_kf_refl"));
        } else LILI_CUDA(c, cudaMemsetAsync(c->map.refl.p, 0, (size_t)m * sizeof(float), c->stream));
    }
    LILI_TRY(install_map_from_xyzw(c, m));
    LILI_CUDA(c, cudaStreamSynchronize(c->stream));
    return LILIOM_OK;
}

extern "C" int liliom_map_size(const liliom_ctx* c) { return c ? c->map.n : 0; }

extern "C" int liliom_map_download(liliom_ctx* c, liliom_f4* out, int cap, int* m_out) {
    if (!c || !m_out) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    return download_sized(c, c->map.xyzw, c->map.n, sizeof(float4), out, cap, m_out);
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
    c->raw_scan_rings = false;
    c->raw_scan_times = false;
    return LILIOM_OK;
}

extern "C" int liliom_set_ring_source(liliom_ctx* c, int source) {
    if (!c || (source != LILIOM_RING_ELEVATION && source != LILIOM_RING_FIELD)) return LILIOM_E_ARG;
    if (source == LILIOM_RING_FIELD && c->prm.point_stride != 32) return LILIOM_E_ARG;
    if (source != c->ring_source) c->raw_scan_rings = false;       // the resident sweep was decoded under the other source
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
    c->raw_scan_times = false;       // any call: the resident sweep's times (if any) may belong to another field
    c->time_source = source;
    return LILIOM_OK;
}

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
        const double ident[4] = {1, 0, 0, 0};
        const bool field = c->ring_source == LILIOM_RING_FIELD;
        const bool timed = c->time_source == LILIOM_TIME_FIELD;
        if (field && !c->raw_scan_rings) rc = LILIOM_E_ARG;       // no ring ids decoded with the resident sweep
        else if (timed && !c->raw_scan_times) rc = LILIOM_E_ARG;  // no times decoded with the resident sweep
        else rc = rot_extract_dev(c, n, q_imu, q_lb ? q_lb : ident, n_surf, n_edge, n_cut, field ? c->raw_scan_ring.as<uint16_t>() : nullptr,
                                  timed ? c->raw_scan_time.as<double>() : nullptr);
    }
    c->raw_src = nullptr;
    return rc;
}

static int odometry_on_resident_surf(liliom_ctx* c, double pose7[7], int match_cnt, int max_num_iter, int mode, liliom_iter_stats* stats,
                                     void* ds_out, int ds_cap, int* n_ds, bool spec_failed) {
    if (!c || !pose7 || (mode != LILIOM_MODE_CERES && mode != LILIOM_MODE_GN) || match_cnt < 0) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    const int stride = c->prm.point_stride;
    // surf count: exact on the host (n_surf_dev >= 0) or only on the device (resident pipeline, no round trip)
    const int n_max = c->n_surf_dev >= 0 ? c->n_surf_dev : c->n_surf_max;
    const int* d_n = c->n_surf_dev >= 0 ? nullptr : c->d_nsurf;
    LILI_CUDA(c, c->vg_out.ensure((size_t)(n_max > 0 ? n_max : 1) * stride));
    LILI_CUDA(c, c->vg_count.ensure(16));
    LILI_CUDA(c, c->feats.ensure((size_t)(n_max > 0 ? n_max : 1) * sizeof(float4)));
    if (c->prm.leaf_scan > 0.0f) {
        // L/src/LidarOdometry.cpp:321-322; the centroid kernel also emits the float4 queries
        // speculate that the scan's voxel box has < 2^24 cells (a 200 m sweep at 0.4 m: ~2^21-2^23): one radix pass
        // less.  The box is read back with the pose; on a miss the step is redone with full-width keys.
        const int key_bits = (n_max > 24576 || spec_failed) ? 32 : 24;
        // scan-sized clouds take the single-launch cooperative filter; it may decline (VgParams::bail, read back with the pose)
        bool coop = false;
        if (!spec_failed)
            LILI_TRY(voxelgrid_coop(c, c->surf.p, n_max, d_n, stride, c->prm.leaf_scan, c->vg_out.p, c->vg_count.as<int>(), c->feats.as<float4>(), &coop));
        if (!coop)
            LILI_TRY(voxelgrid_dev(c, c->surf.p, n_max, d_n, stride, c->prm.leaf_scan, c->vg_out.p, c->vg_count.as<int>(), c->feats.as<float4>(), key_bits));
        c->d_nfeats = c->vg_count.as<int>();
        c->vg_used24 = !coop && key_bits < 32;
        c->vg_check = coop || key_bits < 32;
        c->vg_bail = false;
    } else {   // leaf_scan == 0: benchmark mode, every surf feature is a query
        if (n_max > 0) LILI_CUDA(c, cudaMemcpyAsync(c->vg_out.p, c->surf.p, (size_t)n_max * stride, cudaMemcpyDeviceToDevice, c->stream));
        LILI_TRY(repack_to_f4(c, c->surf.p, n_max, stride, c->feats.as<float4>(), d_n));
        c->d_nfeats = d_n;
    }
    c->n_feats = n_max;
    int rc = LILIOM_OK;
    if (!c->map.ready) rc = LILIOM_E_NOMAP;
    else if (c->map_n_global < 10) rc = LILIOM_E_FEWMAP;
    double pose_in[7];
    memcpy(pose_in, pose7, sizeof(pose_in));
    if (rc == LILIOM_OK) {
        rc = s2m_run(c, pose7, match_cnt, max_num_iter, mode, stats, false, nullptr);
        if (rc == LILIOM_OK && c->vg_check && !spec_failed &&
            (c->vg_bail || (c->vg_used24 && c->vg_ncells >= (1LL << 24) - 1))) {   // speculation missed: redo with the sort chain, 32-bit keys
            c->vg_check = false;
            c->d_nfeats = nullptr;
            memcpy(pose7, pose_in, sizeof(pose_in));
            return odometry_on_resident_surf(c, pose7, match_cnt, max_num_iter, mode, stats, ds_out, ds_cap, n_ds, true);
        }
        c->vg_check = false;
    } else {   // still report surf_last_ds: read the count back
        if (c->d_nfeats) {
            int nq = 0;
            LILI_TRY(read_back(c, {{&nq, c->d_nfeats, sizeof(int)}}));
            c->n_feats_actual = min(nq, n_max);
        } else c->n_feats_actual = n_max;
    }
    c->d_nfeats = nullptr;
    const int m = c->n_feats_actual;
    if (n_ds) *n_ds = m;
    if (ds_out) {
        if (m > ds_cap) return LILIOM_E_CAPACITY;
        if (m) {
            LILI_CUDA(c, cudaMemcpyAsync(ds_out, c->vg_out.p, (size_t)m * stride, cudaMemcpyDeviceToHost, c->stream));
            LILI_CUDA(c, cudaStreamSynchronize(c->stream));
        }
    }
    return rc;
}

extern "C" int liliom_odometry_resident(liliom_ctx* c, double pose7[7], int match_cnt, int max_num_iter, int mode, liliom_iter_stats* stats,
                                        void* ds_out, int ds_cap, int* n_ds) {
    return odometry_on_resident_surf(c, pose7, match_cnt, max_num_iter, mode, stats, ds_out, ds_cap, n_ds);
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
    c->map.refl.release();
    c->map.ready = false;
    c->inc_valid = false;
    LILI_CUDA(c, c->map.xyzw.ensure((size_t)(n_tgt > 0 ? n_tgt : 1) * sizeof(float4)));
    LILI_CUDA(c, c->raw.ensure((size_t)(n_tgt > 0 ? n_tgt : 1) * stride));
    if (n_tgt > 0) {
        LILI_CUDA(c, cudaMemcpyAsync(c->raw.p, tgt, (size_t)n_tgt * stride, cudaMemcpyHostToDevice, c->stream));
        LILI_TRY(repack_to_f4(c, c->raw.p, n_tgt, stride, c->map.xyzw.as<float4>()));
    }
    LILI_TRY(install_map_from_xyzw(c, n_tgt));
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
