// pcl::VoxelGrid<PointT>::filter on the device (L/src/LidarOdometry.cpp:315-323 leaf 0.4;
// R/src/Preprocessing.cpp:502-508 leaf 0.6): bounding box -> integer voxel index
// (idx = i + j*dx + k*dx*dy, fp32 floor(p*inv_leaf) - min_b) -> stable sort by index ->
// per-voxel centroid of all fields in ascending index order.  PCL's std::sort leaves the
// within-voxel order unspecified; here it is the original point order, so the fp32 sums are
// reproducible and equal to the oracle's.  Compiled with --fmad=false.
// The box / divisions are computed on the device (VgParams): no host round trip inside the call.
#include "ctx.cuh"
#include <climits>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <type_traits>

namespace lili {

__global__ void k_vg_init(int* mm) { vg_box_init(mm); }

// box of the finite points (vg_box.h; the body in ctx.cuh)
__global__ void k_vg_minmax(const unsigned char* __restrict__ pts, int n_max, const int* __restrict__ d_n, int stride, int* __restrict__ mm) {
    vg_minmax_body(pts, n_max, d_n, stride, mm, SoloBlock{});
}

struct VgBox { int mm[kBoxInts]; };      // a box (vg_box.h) by value

__global__ void k_vg_params(const int* __restrict__ mm, float leaf, VgParams* __restrict__ out) {
    vg_params_at(mm, leaf, out);
}
// the bounding box is already known on the host (map rebuild: the union of the frames' boxes, kept since their push)
__global__ void k_vg_params_box(const VgBox b, float leaf, VgParams* __restrict__ out) {
    if (threadIdx.x == 0) *out = vg_params(b.mm, leaf);
}

// the key and centroid kernels: bodies in ctx.cuh (the batched loop closure runs them too)
template <typename K>
__global__ void k_vg_keys(const unsigned char* __restrict__ pts, int n_max, const int* __restrict__ d_n, int stride, const VgParams* __restrict__ pp,
                          K* __restrict__ keys, int* __restrict__ vals) {
    vg_keys_at<K>(pts, n_max, d_n, stride, pp, keys, vals, blockIdx.x * blockDim.x + threadIdx.x);
}

template <int STRIDE, typename K>
__global__ void k_vg_centroid(const unsigned char* __restrict__ pts, const K* __restrict__ keys, const int* __restrict__ vals,
                              const int* __restrict__ flags, const int* __restrict__ rank, int n_max, const int* __restrict__ d_n,
                              const VgParams* __restrict__ pp, unsigned char* __restrict__ out, int* __restrict__ count_out,
                              float4* __restrict__ feats_out) {
    vg_centroid_at<STRIDE, K>(pts, keys, vals, flags, rank, n_max, d_n, pp, out, count_out, feats_out, blockIdx.x * blockDim.x + threadIdx.x);
}

// ---------------------------------------------------------------------------------------
// Scan-sized VoxelGrid in ONE cooperative launch, without a sort (n <= VGC_NCAP points).
// The sort chain above costs ~13 dependent launches (~95 us for a 13k-point /surf_features cloud, almost
// all of it launch latency and three onesweep passes).  PCL only needs (a) which points share a voxel,
// (b) the voxels in ascending index order, (c) each voxel's members summed in a fixed order.  With
// idx = i + j*dx + k*dx*dy and 0 <= i < dx, 0 <= j < dy, ascending idx is lexicographic (k, j, i) order, and
// i/j/k differ from the absolute cell coordinate floor(p*inv_leaf) only by the box minimum (exact in fp32
// below 2^24), so neither (a) nor (b) needs the bounding box:
//   phase 1  every point inserts its absolute (kz, jy, ix) key into a hash table (64-bit CAS), the first
//            writer appends the key to a dense list; the point's arrival number in its voxel (atomicAdd on
//            the slot's count) places its index in the slot's fixed-size member bucket; box partials
//   -------- the one grid barrier
//   phase 2  every block reduces the box partials itself (VgParams: PCL's overflow test) and stages the key
//            list in shared memory
//   phase 3  one warp per voxel: output rank = number of listed keys below its key (all pairs); members read
//            from the slot's bucket and ordered by original index (rank by counting in shared memory), fp32
//            sums in that order — the order of the sort chain and of the oracle — centroid written at the rank
// Inputs it declines (|cell coordinate| >= 2^20, PCL's index overflow, a voxel with more than VGC_VCAP members, a box
// whose PCL index wraps: VgParams::wraps, where absolute-key order is not PCL's order and distinct cells can share an
// index) set VgParams::bail and an output count of 0; the box's own parameters are left with the bail mark, so the caller
// knows which key width the sort chain needs.  Semantics otherwise identical to k_vg_* above.
// One barrier is enough because every bail condition is final when it is passed: bits 0 (unrepresentable
// key) and 1 (arrival number VGC_VCAP, i.e. a voxel over VGC_VCAP members) are only set in phase 1, and the
// overflow and wrap tests (bits 2 and 3) read the box partials, which phase 1 completes.  So every block takes the same decision, and
// no block decides to bail on a bit that another block can still set (a block that bailed on a late bit would
// never reach a later barrier, and the blocks waiting there would spin forever).  After the barrier a warp
// touches only its own voxel's slot (count, bucket, and handing the slot back) plus data no block writes any
// more (key list, slots, box partials), so no second barrier is needed either.
// ---------------------------------------------------------------------------------------
constexpr int VGC_NCAP = 32768;       // point indices fit the 16-bit bucket entries
constexpr int VGC_T = 65536;          // hash slots (load factor <= 0.5)
constexpr int VGC_THREADS = 512;      // 132 x 16 warps: one voxel round covers a down-sampled 24k sweep (1-2k voxels)
constexpr int VGC_WARPS = VGC_THREADS / 32;
constexpr int VGC_VCAP = 256;         // members per voxel handled in shared memory (= bucket size)
constexpr unsigned long long VGC_EMPTY = ~0ull;

struct VgCoopBufs {
    unsigned long long* hkey;   // [T]   voxel key per slot (VGC_EMPTY when free; restored by the kernel itself)
    int* hcnt;                  // [T]   members per slot (0 when free; restored by the kernel itself)
    unsigned short* bucket;     // [T][VCAP] point indices of the slot's members, in arrival order
    unsigned long long* ukey;   // [NCAP] dense list of occupied keys (arbitrary order)
    int* uslot;                 // [NCAP] their slots
    int* mmpart;                // [7][grid] per-block box partials
    unsigned int* ctl;          // [4][4] rotating {barrier arrivals, bail flags, #voxels, spare}; slot = call & 3
};

static size_t vgc_layout(VgCoopBufs& B, unsigned char* base, int grid) {
    size_t off = 0;
    auto take = [&](size_t bytes) { unsigned char* p = base ? base + off : nullptr; off += (bytes + 255) & ~(size_t)255; return p; };
    B.hkey = (unsigned long long*)take((size_t)VGC_T * 8);
    B.hcnt = (int*)take((size_t)VGC_T * 4);
    B.bucket = (unsigned short*)take((size_t)VGC_T * VGC_VCAP * 2);
    B.ukey = (unsigned long long*)take((size_t)VGC_NCAP * 8);
    B.uslot = (int*)take((size_t)VGC_NCAP * 4);
    B.mmpart = (int*)take((size_t)7 * grid * 4);
    B.ctl = (unsigned int*)take(16 * 4);
    return off;
}

constexpr int VGC_UKEYS = 8192;    // occupied-voxel keys a block holds in shared memory for the ranks (more: read through L2)
struct VgCoopSmem {
    int   red[7][VGC_WARPS];
    int   mm[kBoxInts];
    unsigned int bail;
    int   mem[VGC_WARPS][VGC_VCAP];     // a voxel's members in arrival order
    int   sidx[VGC_WARPS][VGC_VCAP];    // ... in ascending original index
    float stage[VGC_WARPS][32][8];
    unsigned long long ukeys[VGC_UKEYS];
};

template <int STRIDE>
__global__ void __launch_bounds__(VGC_THREADS, 1) k_vg_coop(const unsigned char* __restrict__ pts, int n_max, const int* __restrict__ d_n, float leaf,
                                                         VgCoopBufs B, unsigned int call, VgParams* __restrict__ pp,
                                                         unsigned char* __restrict__ out, int* __restrict__ count_out, float4* __restrict__ feats_out) {
    extern __shared__ __align__(16) unsigned char vgc_smem[];
    VgCoopSmem& S = *reinterpret_cast<VgCoopSmem*>(vgc_smem);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned int G = gridDim.x;
    const int gtid = blockIdx.x * VGC_THREADS + tid, gthreads = G * VGC_THREADS;
    const int gwarp = blockIdx.x * VGC_WARPS + warp, gwarps = G * VGC_WARPS;
    // bit 31 of `call` (LILIOM_DEBUG_TIMING): block 0 leaves clock64 stamps of the phase boundaries behind the 16 control words
    long long* stamp = ((call >> 31) != 0u && blockIdx.x == 0 && tid == 0) ? reinterpret_cast<long long*>(B.ctl + 16) : nullptr;
    call &= 0x7fffffffu;
    if (stamp) { stamp[0] = clock64(); stamp[5] = (long long)globaltimer_ns(); }
    unsigned int* ctl = B.ctl + 4 * (call & 3u);          // [0] barrier, [1] bail, [2] #voxels
    if (blockIdx.x == 0 && tid < 4) B.ctl[4 * ((call + 1u) & 3u) + tid] = 0u;   // the next launch's slot (nobody uses it now)
    const int n = d_n ? min(*d_n, n_max) : n_max;
    const float inv_leaf = 1.0f / leaf;

    // ---- phase 1: hash insert, member buckets, bounding box partials
    int box[kBoxInts];
#pragma unroll
    for (int k = 0; k < kBoxInts; ++k) box[k] = vg_box_empty(k);
    // (warp-uniform trip count: the first writers of a warp append to the voxel list with ONE atomic per warp — 1-2k atomics on a
    // single counter were a serial chain of their own.  Warp w of block b takes the 32 points of global warp w*G + b: a ~10k-point
    // scan spreads its loads and atomics over every SM instead of queueing 512 points on each of the first 20 blocks)
    for (int i0 = (warp * (int)G + (int)blockIdx.x) * 32; i0 < n; i0 += gthreads) {
        const int i = i0 + lane;
        const bool active = i < n;
        float4 v = make_float4(NAN, 0.f, 0.f, 0.f);
        if (active) v = *reinterpret_cast<const float4*>(pts + (size_t)i * STRIDE);
        int slot = -1;
        bool won = false;
        unsigned long long wkey = 0;
        if (isfinite(v.x) && isfinite(v.y) && isfinite(v.z)) {
            vg_box_add(box, v.x, v.y, v.z);
            unsigned long long key;
            if (!vg_abs_key(v.x, v.y, v.z, inv_leaf, &key)) {
                atomicOr(&ctl[1], 1u);
            } else {
                unsigned int s = (unsigned int)((key * 0x9E3779B97F4A7C15ull) >> 48) & (VGC_T - 1);
                while (true) {
                    const unsigned long long prev = atomicCAS(&B.hkey[s], VGC_EMPTY, key);
                    if (prev == VGC_EMPTY) { won = true; wkey = key; break; }
                    if (prev == key) break;
                    s = (s + 1) & (VGC_T - 1);
                }
                slot = (int)s;
                const int pos = atomicAdd(&B.hcnt[s], 1);
                if (pos < VGC_VCAP) B.bucket[(size_t)s * VGC_VCAP + pos] = (unsigned short)i;
                else if (pos == VGC_VCAP) atomicOr(&ctl[1], 2u);      // more members than a warp orders in shared memory
            }
        }
        const unsigned wm = __ballot_sync(0xffffffffu, won);
        if (wm) {
            const int leader = __ffs(wm) - 1;
            unsigned int ubase = 0;
            if (lane == leader) ubase = atomicAdd(&ctl[2], (unsigned int)__popc(wm));
            ubase = __shfl_sync(0xffffffffu, ubase, leader);
            if (won) { const unsigned int u = ubase + (unsigned int)__popc(wm & ((1u << lane) - 1u)); B.ukey[u] = wkey; B.uslot[u] = slot; }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int k = 0; k < kBoxInts; ++k) box[k] = vg_box_join(k, box[k], __shfl_xor_sync(0xffffffffu, box[k], o));
    }
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < kBoxInts; ++k) S.red[k][warp] = box[k];
    }
    __syncthreads();
    if (tid < kBoxInts) {
        int v = S.red[tid][0];
        for (int w = 1; w < VGC_WARPS; ++w) v = vg_box_join(tid, v, S.red[tid][w]);
        B.mmpart[tid * G + blockIdx.x] = v;
    }
    grid_barrier<kFenced>(&ctl[0], G);
    if (stamp) stamp[1] = clock64();

    // ---- phase 2: box parameters (every block, warp 0) and the key list in shared memory (the other warps)
    const int U = (int)*reinterpret_cast<volatile unsigned int*>(&ctl[2]);
    unsigned int bail = *reinterpret_cast<volatile unsigned int*>(&ctl[1]);    // final (see above)
    // rank by counting over ALL listed keys: from shared memory when the list fits (a down-sampled 24k sweep lists 1-2k voxels)
    const bool in_smem = U <= VGC_UKEYS;
    if (warp == 0) {
        int mm[kBoxInts];
#pragma unroll
        for (int k = 0; k < kBoxInts; ++k) mm[k] = vg_box_empty(k);
        for (unsigned int b = lane; b < G; b += 32) {
#pragma unroll
            for (int k = 0; k < kBoxInts; ++k) mm[k] = vg_box_join(k, mm[k], __ldcg(&B.mmpart[k * G + b]));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
            for (int k = 0; k < kBoxInts; ++k) mm[k] = vg_box_join(k, mm[k], __shfl_xor_sync(0xffffffffu, mm[k], o));
        }
        if (lane == 0) {
            VgParams p = vg_params(mm, leaf);
            if (p.overflow) bail |= 4u;                                  // PCL copies the input: sort chain
            if (p.wraps) bail |= 8u;                                     // PCL's index wraps: not the absolute keys' order
            if (blockIdx.x == 0) {
                if (bail) p.bail = 1;
                *pp = p;
                *count_out = bail ? 0 : U;
            }
            S.bail = bail;
        }
    } else if (!bail && in_smem) {
        for (int v = tid - 32; v < U; v += VGC_THREADS - 32) S.ukeys[v] = __ldcg(&B.ukey[v]);
    }
    __syncthreads();
    bail = S.bail;
    if (stamp) stamp[2] = clock64();
    if (bail) {
        // declined (the bail mark and an empty result are written above): leave the table clean for the next launch
        for (int s = gtid; s < VGC_T; s += gthreads) { B.hkey[s] = VGC_EMPTY; B.hcnt[s] = 0; }
        return;
    }

    // ---- phase 3: one warp per voxel — output rank, members in ascending original index, sequential fp32 sums
    constexpr int NF = kVgFields<STRIDE>;
    int* mem = S.mem[warp];
    int* sidx = S.sidx[warp];
    for (int u = gwarp; u < U; u += gwarps) {
        const int s = __ldcg(&B.uslot[u]);
        const int c = __ldcg(&B.hcnt[s]);                    // <= VGC_VCAP (bit 1 otherwise)
        const unsigned long long my = in_smem ? S.ukeys[u] : __ldcg(&B.ukey[u]);
        int o = 0;
        if (in_smem) {
#pragma unroll 4
            for (int v = lane; v < U; v += 32) o += (S.ukeys[v] < my) ? 1 : 0;
        } else {
#pragma unroll 4
            for (int v = lane; v < U; v += 32) o += (__ldcg(&B.ukey[v]) < my) ? 1 : 0;
        }
#pragma unroll
        for (int k = 16; k > 0; k >>= 1) o += __shfl_xor_sync(0xffffffffu, o, k);
        if (stamp && u == gwarp) stamp[3] = clock64();
        for (int j = lane; j < c; j += 32) mem[j] = __ldcg(&B.bucket[(size_t)s * VGC_VCAP + j]);
        __syncwarp();
        // order by counting (indices are distinct)
        for (int j = lane; j < c; j += 32) {
            const int m = mem[j];
            int below = 0;
            for (int k = 0; k < c; ++k) below += (mem[k] < m) ? 1 : 0;
            sidx[below] = m;
        }
        __syncwarp();
        float acc = 0.f;       // lane f < NF owns field f
        for (int base = 0; base < c; base += 32) {
            const int j = base + lane;
            if (j < c) vg_load<STRIDE>(pts + (size_t)sidx[j] * STRIDE, S.stage[warp][lane]);
            __syncwarp();
            if (lane < NF) {
                const int m = min(32, c - base);
                for (int k = 0; k < m; ++k) acc += S.stage[warp][k][lane];
            }
            __syncwarp();
        }
        float f[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) f[k] = __shfl_sync(0xffffffffu, acc, k);
        if (lane == 0) {
            const VgXyz cxyz = vg_write<STRIDE>(f, c, out + (size_t)o * STRIDE);
            if (feats_out) feats_out[o] = make_float4(cxyz.x, cxyz.y, cxyz.z, __int_as_float(o));
            B.hkey[s] = VGC_EMPTY;      // hand the slot back
            B.hcnt[s] = 0;
        }
        __syncwarp();
    }
    if (stamp) { stamp[4] = clock64(); stamp[6] = (long long)globaltimer_ns(); }
}

// stage stamps of the last k_vg_coop launch (LILIOM_DEBUG_TIMING); nullptr before the first launch
const long long* vg_coop_stamps(liliom_ctx* c) {
    if (!c->vg_coop.p) return nullptr;
    VgCoopBufs B;
    vgc_layout(B, (unsigned char*)c->vg_coop.p, c->sm_count);
    return reinterpret_cast<const long long*>(B.ctl + 16);
}

// Returns LILIOM_OK after enqueueing the cooperative filter; the caller must look at VgParams::bail (vg_params)
// after its next sync and fall back to voxelgrid_dev when it is set.  *used = false: not applicable, nothing enqueued.
int voxelgrid_coop(liliom_ctx* c, const void* d_in, int n_max, const int* d_n, int stride, float leaf, void* d_out, int* d_count,
                   float4* d_feats, bool* used) {
    *used = false;
    if ((stride != 48 && stride != 32) || n_max <= 0 || n_max > VGC_NCAP) return LILIOM_OK;
    const int grid = c->sm_count;
    VgCoopBufs B;
    const size_t bytes = vgc_layout(B, nullptr, grid);
    if (!c->vg_coop.p) {
        LILI_CUDA(c, c->vg_coop.ensure(bytes));
        vgc_layout(B, (unsigned char*)c->vg_coop.p, grid);
        LILI_CUDA(c, cudaMemsetAsync(c->vg_coop.p, 0, c->vg_coop.cap, c->stream));
        LILI_CUDA(c, cudaMemsetAsync(B.hkey, 0xff, (size_t)VGC_T * 8, c->stream));
        c->vg_coop_calls = 0;
        LILI_CUDA(c, cudaFuncSetAttribute(k_vg_coop<48>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(VgCoopSmem)));
        LILI_CUDA(c, cudaFuncSetAttribute(k_vg_coop<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(VgCoopSmem)));
    }
    vgc_layout(B, (unsigned char*)c->vg_coop.p, grid);
    LILI_CUDA(c, c->vg_params.ensure(sizeof(VgParams)));
    const unsigned char* in = (const unsigned char*)d_in;
    unsigned char* outp = (unsigned char*)d_out;
    VgParams* pp = c->vg_params.as<VgParams>();
    unsigned int call = (c->vg_coop_calls & 0x7fffffffu) | (c->dbg_timing ? 0x80000000u : 0u);
    void* kargs[] = {&in, &n_max, &d_n, &leaf, &B, &call, &pp, &outp, &d_count, &d_feats};
    const void* fn = stride == 48 ? (const void*)k_vg_coop<48> : (const void*)k_vg_coop<32>;
    LILI_CUDA(c, cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(VGC_THREADS), kargs, sizeof(VgCoopSmem), c->stream));
    LILI_TRY(launch_check(c, "k_vg_coop"));
    c->vg_coop_calls++;
    *used = true;
    return LILIOM_OK;
}

// box of the finite points of a device cloud, left in c->vg_minmax (7 ints, vg_box.h); no sync
int vg_minmax_dev(liliom_ctx* c, const void* d_in, int n_max, const int* d_n, int stride) {
    LILI_CUDA(c, c->vg_minmax.ensure(8 * sizeof(int)));
    int* mm = c->vg_minmax.as<int>();
    k_vg_init<<<1, 32, 0, c->stream>>>(mm);
    LILI_TRY(launch_check(c, "k_vg_init"));
    if (n_max > 0) {
        k_vg_minmax<<<box_blocks(n_max, c->sm_count), 256, 0, c->stream>>>((const unsigned char*)d_in, n_max, d_n, stride, mm);
        LILI_TRY(launch_check(c, "k_vg_minmax"));
    }
    return LILIOM_OK;
}

// the buffers of voxelgrid_dev's chain over n points at kb-byte keys
int vg_chain_ensure(liliom_ctx* c, long long n, size_t kb) {
    LILI_CUDA(c, c->vg_minmax.ensure(8 * sizeof(int)));
    LILI_CUDA(c, c->vg_params.ensure(sizeof(VgParams)));
    LILI_CUDA(c, c->vg_keys.ensure((size_t)n * kb));
    LILI_CUDA(c, c->vg_vals.ensure((size_t)n * 4));
    LILI_CUDA(c, c->vg_keys2.ensure((size_t)n * kb));
    LILI_CUDA(c, c->vg_vals2.ensure((size_t)n * 4));
    LILI_CUDA(c, c->vg_flags.ensure(((size_t)n + 2) * 4));
    LILI_CUDA(c, c->vg_rank.ensure(((size_t)n + 2) * 4));
    return LILIOM_OK;
}

// key_bits < 32: the caller speculates that the voxel index fits that width (one onesweep pass less per 8 bits) and must check
// `ncells <= 2^key_bits - 1` afterwards (vg_params stays on the device).  key_bits = 32 assumes the index does not wrap: the
// caller checks vg_wide_keys on the VgParams it reads back and redoes the call with key_bits = kVgWideKeyBits (64-bit keys) on
// a hit (voxelgrid_dev_sync).  host_mm (optional): the cloud's box and finite count already known on the host -> no pass over
// the input for it, and the key width follows from the box (vg_chain_key_bits).
int voxelgrid_dev(liliom_ctx* c, const void* d_in, int n_max, const int* d_n, int stride, float leaf, void* d_out, int* d_count,
                  float4* d_feats, int key_bits, const int* host_mm) {
    if (stride != 48 && stride != 32) return LILIOM_E_ARG;
    if (host_mm) key_bits = vg_chain_key_bits(host_mm, leaf);
    if (n_max <= 0) {
        LILI_CUDA(c, cudaMemsetAsync(d_count, 0, sizeof(int), c->stream));
        return LILIOM_OK;
    }
    const unsigned char* in = (const unsigned char*)d_in;
    const int n = n_max;
    const bool wide = key_bits > 32;
    LILI_TRY(vg_chain_ensure(c, n, wide ? 8 : 4));
    int* mm = c->vg_minmax.as<int>();
    VgParams* pp = c->vg_params.as<VgParams>();
    if (host_mm) {
        VgBox b;
        for (int k = 0; k < kBoxInts; ++k) b.mm[k] = host_mm[k];
        k_vg_params_box<<<1, 32, 0, c->stream>>>(b, leaf, pp);
        LILI_TRY(launch_check(c, "k_vg_params_box"));
    } else {
        k_vg_init<<<1, 32, 0, c->stream>>>(mm);
        LILI_TRY(launch_check(c, "k_vg_init"));
        k_vg_minmax<<<min(cdiv(n, 256), c->sm_count * 8), 256, 0, c->stream>>>(in, n, d_n, stride, mm);
        LILI_TRY(launch_check(c, "k_vg_minmax"));
        k_vg_params<<<1, 32, 0, c->stream>>>(mm, leaf, pp);
        LILI_TRY(launch_check(c, "k_vg_params"));
    }
    // keys -> sort -> heads -> ranks -> centroids at key type K; non-finite points carry the sentinel key (the all-ones 32-bit key,
    // folded to the sort's width, or bit 32 of a wide key) and sort last; VgParams::n_finite excludes them
    auto chain = [&](auto* keys, auto* keys2, int end_bit) -> int {
        using K = std::remove_pointer_t<decltype(keys)>;
        k_vg_keys<K><<<cdiv(n, 256), 256, 0, c->stream>>>(in, n, d_n, stride, pp, keys, c->vg_vals.as<int>());
        LILI_TRY(launch_check(c, "k_vg_keys"));
        if constexpr (sizeof(K) == 4) LILI_TRY(sort_pairs_u32(c, keys, keys2, c->vg_vals.as<int>(), c->vg_vals2.as<int>(), n, end_bit));
        else LILI_TRY(sort_pairs_u64(c, keys, keys2, c->vg_vals.as<int>(), c->vg_vals2.as<int>(), n, end_bit));
        k_vg_heads<<<cdiv(n + 1, 256), 256, 0, c->stream>>>(keys2, n, &pp->n_finite, c->vg_flags.as<int>());
        LILI_TRY(launch_check(c, "k_vg_heads"));
        LILI_TRY(exclusive_scan_i32(c, c->vg_flags.as<int>(), c->vg_rank.as<int>(), n));
        if (stride == 48)
            k_vg_centroid<48, K><<<cdiv(n, 128), 128, 0, c->stream>>>(in, keys2, c->vg_vals2.as<int>(), c->vg_flags.as<int>(), c->vg_rank.as<int>(), n,
                                                                      d_n, pp, (unsigned char*)d_out, d_count, d_feats);
        else
            k_vg_centroid<32, K><<<cdiv(n, 128), 128, 0, c->stream>>>(in, keys2, c->vg_vals2.as<int>(), c->vg_flags.as<int>(), c->vg_rank.as<int>(), n,
                                                                      d_n, pp, (unsigned char*)d_out, d_count, d_feats);
        return launch_check(c, "k_vg_centroid");
    };
    if (wide) return chain(c->vg_keys.as<unsigned long long>(), c->vg_keys2.as<unsigned long long>(), kVgWideKeyBits);
    return chain(c->vg_keys.as<uint32_t>(), c->vg_keys2.as<uint32_t>(), key_bits);
}

// voxelgrid_dev of n points (n known on the host) with its output count read back at once: the count and VgParams come back in
// one sync, and the filter is redone with wide keys when the index wraps.  key_bits: 32, or kVgWideKeyBits when the caller
// already knows the index wraps.  *m: the output count.
int voxelgrid_dev_sync(liliom_ctx* c, const void* d_in, int n, int stride, float leaf, void* d_out, int* d_count, float4* d_feats, int* m,
                       int key_bits) {
    *m = 0;
    LILI_TRY(voxelgrid_dev(c, d_in, n, nullptr, stride, leaf, d_out, d_count, d_feats, key_bits));
    if (n <= 0) return LILIOM_OK;
    VgParams vp;
    LILI_TRY(read_back(c, {{m, d_count, sizeof(int)}, {&vp, c->vg_params.p, sizeof(VgParams)}}));
    if (key_bits > 32 || !vg_wide_keys(vp)) return LILIOM_OK;
    LILI_TRY(voxelgrid_dev(c, d_in, n, nullptr, stride, leaf, d_out, d_count, d_feats, kVgWideKeyBits));
    return read_back(c, {{m, d_count, sizeof(int)}});
}

}  // namespace lili
