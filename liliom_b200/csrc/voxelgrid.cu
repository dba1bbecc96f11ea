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

namespace lili {

__global__ void k_vg_init(int* mm) {
    if (threadIdx.x < kBoxInts) mm[threadIdx.x] = vg_box_empty(threadIdx.x);
}

// box of the finite points (vg_box.h)
__global__ void k_vg_minmax(const unsigned char* __restrict__ pts, int n_max, const int* __restrict__ d_n, int stride, int* __restrict__ mm) {
    const int n = d_n ? min(*d_n, n_max) : n_max;
    int box[kBoxInts];
#pragma unroll
    for (int k = 0; k < kBoxInts; ++k) box[k] = vg_box_empty(k);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float4 v = *reinterpret_cast<const float4*>(pts + (size_t)i * stride);
        if (!(isfinite(v.x) && isfinite(v.y) && isfinite(v.z))) continue;
        vg_box_add(box, v.x, v.y, v.z);
    }
    vg_box_commit(box, mm);
}

struct VgBox { int mm[kBoxInts]; };      // a box (vg_box.h) by value

__global__ void k_vg_params(const int* __restrict__ mm, float leaf, VgParams* __restrict__ out) {
    if (threadIdx.x == 0) *out = vg_params(mm, leaf);
}
// the bounding box is already known on the host (map rebuild: the union of the frames' boxes, kept since their push)
__global__ void k_vg_params_box(const VgBox b, float leaf, VgParams* __restrict__ out) {
    if (threadIdx.x == 0) *out = vg_params(b.mm, leaf);
}

__global__ void k_vg_keys(const unsigned char* __restrict__ pts, int n_max, const int* __restrict__ d_n, int stride, const VgParams* __restrict__ pp,
                          uint32_t* __restrict__ keys, int* __restrict__ vals) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max) return;
    const int n = d_n ? min(*d_n, n_max) : n_max;
    const VgParams p = *pp;
    float4 v = make_float4(NAN, 0.f, 0.f, 0.f);
    if (i < n) v = *reinterpret_cast<const float4*>(pts + (size_t)i * stride);
    uint32_t key = 0xffffffffu;
    if (isfinite(v.x) && isfinite(v.y) && isfinite(v.z)) key = vg_rel_index(p, v.x, v.y, v.z);
    keys[i] = key;
    vals[i] = i;
}

template <int STRIDE>
__global__ void k_vg_centroid(const unsigned char* __restrict__ pts, const uint32_t* __restrict__ keys, const int* __restrict__ vals,
                              const int* __restrict__ flags, const int* __restrict__ rank, int n_max, const int* __restrict__ d_n,
                              const VgParams* __restrict__ pp, unsigned char* __restrict__ out, int* __restrict__ count_out,
                              float4* __restrict__ feats_out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
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

// ---------------------------------------------------------------------------------------
// Scan-sized VoxelGrid in ONE cooperative launch, without a sort (n <= VGC_NCAP points).
// The sort chain above costs ~13 dependent launches (~95 us for a 13k-point /surf_features cloud, almost
// all of it launch latency and three onesweep passes).  PCL only needs (a) which points share a voxel,
// (b) the voxels in ascending index order, (c) each voxel's members summed in a fixed order.  With
// idx = i + j*dx + k*dx*dy and 0 <= i < dx, 0 <= j < dy, ascending idx is lexicographic (k, j, i) order, and
// i/j/k differ from the absolute cell coordinate floor(p*inv_leaf) only by the box minimum (exact in fp32
// below 2^24), so neither (a) nor (b) needs the bounding box:
//   phase 1  every point inserts its absolute (kz, jy, ix) key into a hash table (64-bit CAS), the first
//            writer appends the key to a dense list; per-slot member count by atomicAdd; box partials
//   phase 2  output rank of a voxel = number of listed keys below its key (all pairs, one warp per voxel,
//            the list is a few KB and L1-resident); member segment start by atomicAdd (scratch order)
//   phase 3  every point drops its index into its voxel's segment
//   phase 4  one warp per voxel: members ordered by original index (rank by counting), fp32 sums in that
//            order — the order of the sort chain and of the oracle — centroid written at the voxel's rank
// Three grid barriers instead of twelve launch boundaries.  Inputs it declines (|cell coordinate| >= 2^20,
// PCL's index overflow, a voxel with more than VGC_VCAP members) set VgParams::bail and an output count
// of 0; the caller re-runs the sort chain.  Semantics otherwise identical to k_vg_* above.
// ---------------------------------------------------------------------------------------
constexpr int VGC_NCAP = 32768;
constexpr int VGC_T = 65536;          // hash slots (load factor <= 0.5)
constexpr int VGC_THREADS = 256;
constexpr int VGC_WARPS = VGC_THREADS / 32;
constexpr int VGC_VCAP = 256;         // members per voxel handled in shared memory
constexpr unsigned long long VGC_EMPTY = ~0ull;

struct VgCoopBufs {
    unsigned long long* hkey;   // [T]   voxel key per slot (VGC_EMPTY when free; restored by the kernel itself)
    int* hcnt;                  // [T]   members per slot (0 when free; restored by the kernel itself)
    int* hoff;                  // [T]   start of the slot's member segment
    unsigned long long* ukey;   // [NCAP] dense list of occupied keys (arbitrary order)
    int* uslot;                 // [NCAP] their slots
    int* urank;                 // [NCAP] their output ranks
    int* pslot;                 // [NCAP] slot of point i (-1: not finite)
    int* ppos;                  // [NCAP] arrival number of point i inside its voxel
    int* members;               // [NCAP] point indices grouped by voxel
    int* mmpart;                // [7][grid] per-block box partials
    unsigned int* ctl;          // [4][4] rotating {barrier arrivals, bail flag, #voxels, segment cursor}; slot = call & 3
};

static size_t vgc_layout(VgCoopBufs& B, unsigned char* base, int grid) {
    size_t off = 0;
    auto take = [&](size_t bytes) { unsigned char* p = base ? base + off : nullptr; off += (bytes + 255) & ~(size_t)255; return p; };
    B.hkey = (unsigned long long*)take((size_t)VGC_T * 8);
    B.hcnt = (int*)take((size_t)VGC_T * 4);
    B.hoff = (int*)take((size_t)VGC_T * 4);
    B.ukey = (unsigned long long*)take((size_t)VGC_NCAP * 8);
    B.uslot = (int*)take((size_t)VGC_NCAP * 4);
    B.urank = (int*)take((size_t)VGC_NCAP * 4);
    B.pslot = (int*)take((size_t)VGC_NCAP * 4);
    B.ppos = (int*)take((size_t)VGC_NCAP * 4);
    B.members = (int*)take((size_t)VGC_NCAP * 4);
    B.mmpart = (int*)take((size_t)7 * grid * 4);
    B.ctl = (unsigned int*)take(16 * 4);
    return off;
}

__device__ __forceinline__ void vgc_barrier(unsigned int* bar, unsigned int target) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        atomicAdd(bar, 1u);
        while ((int)(*reinterpret_cast<volatile unsigned int*>(bar) - target) < 0) { }
        __threadfence();
    }
    __syncthreads();
}

constexpr int VGC_UKEYS = 4032;    // occupied-voxel keys a block can hold in shared memory for phase 2 (static smem limit: 48 KB)
struct VgCoopSmem {
    int   red[7][VGC_WARPS];
    int   sidx[VGC_WARPS][VGC_VCAP];
    float stage[VGC_WARPS][32][8];
    unsigned long long ukeys[VGC_UKEYS];
};

template <int STRIDE>
__global__ void __launch_bounds__(VGC_THREADS) k_vg_coop(const unsigned char* __restrict__ pts, int n_max, const int* __restrict__ d_n, float leaf,
                                                         VgCoopBufs B, unsigned int call, VgParams* __restrict__ pp,
                                                         unsigned char* __restrict__ out, int* __restrict__ count_out, float4* __restrict__ feats_out) {
    __shared__ VgCoopSmem S;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned int G = gridDim.x;
    const int gtid = blockIdx.x * VGC_THREADS + tid, gthreads = G * VGC_THREADS;
    const int gwarp = blockIdx.x * VGC_WARPS + warp, gwarps = G * VGC_WARPS;
    // bit 31 of `call` (LILIOM_DEBUG_TIMING): block 0 leaves clock64 stamps of the phase boundaries behind the 16 control words
    long long* stamp = ((call >> 31) != 0u && blockIdx.x == 0 && tid == 0) ? reinterpret_cast<long long*>(B.ctl + 16) : nullptr;
    call &= 0x7fffffffu;
    if (stamp) { stamp[0] = clock64(); stamp[5] = (long long)globaltimer_ns(); }
    unsigned int* ctl = B.ctl + 4 * (call & 3u);          // [0] barrier, [1] bail, [2] #voxels, [3] segment cursor
    if (blockIdx.x == 0 && tid < 4) B.ctl[4 * ((call + 1u) & 3u) + tid] = 0u;   // the next launch's slot (nobody uses it now)
    const int n = d_n ? min(*d_n, n_max) : n_max;
    const float inv_leaf = 1.0f / leaf;

    // ---- phase 1: hash insert + bounding box partials
    int box[kBoxInts];
#pragma unroll
    for (int k = 0; k < kBoxInts; ++k) box[k] = vg_box_empty(k);
    // (warp-uniform trip count: the first writers of a warp append to the voxel list with ONE atomic per warp — 1-2k atomics on a
    // single counter were a serial chain of their own)
    for (int i0 = gtid - lane; i0 < n; i0 += gthreads) {
        const int i = i0 + lane;
        const bool active = i < n;
        float4 v = make_float4(NAN, 0.f, 0.f, 0.f);
        if (active) v = *reinterpret_cast<const float4*>(pts + (size_t)i * STRIDE);
        int slot = -1, pos = 0;
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
                pos = atomicAdd(&B.hcnt[s], 1);
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
        if (active) { B.pslot[i] = slot; B.ppos[i] = pos; }
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
    vgc_barrier(&ctl[0], G);
    if (stamp) stamp[1] = clock64();

    int U = (int)*reinterpret_cast<volatile unsigned int*>(&ctl[2]);
    // Only bit 0 (set in phase 1) is final before barrier 1.  Bits 1 and 2 are set DURING phase 2, so a block that leaves the
    // barrier late could already see them: were it to take the bail path here it would never arrive at barrier 2 and the
    // blocks that read 0 would spin there forever.  Every block therefore decides on bit 0 alone; the full word is read
    // again after barrier 2, when it is final for all blocks.
    unsigned int bail = *reinterpret_cast<volatile unsigned int*>(&ctl[1]) & 1u;
    if (!bail) {
        // ---- phase 2: box parameters (block 0), output ranks and member segments
        if (blockIdx.x == 0 && warp == 0) {
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
                if (p.overflow) { p.bail = 1; atomicOr(&ctl[1], 4u); }   // PCL copies the input: sort chain
                *pp = p;
                *count_out = p.bail ? 0 : U;
            }
        }
        // rank by counting over ALL listed keys: from shared memory when the list fits (a down-sampled 24k sweep lists 1-2k
        // voxels): when every compare re-read the list through L2 this phase was ~50 dependent L2 round trips per voxel
        // (LILIOM_DEBUG_TIMING shows the phase's cycles)
        const bool in_smem = U <= VGC_UKEYS;
        if (in_smem) {
            for (int v = tid; v < U; v += VGC_THREADS) S.ukeys[v] = __ldcg(&B.ukey[v]);
            __syncthreads();
        }
        // (block-uniform trip count: the member segments of a block's voxels are carved out of the cursor with ONE atomic per block
        // and iteration instead of one per voxel on the same word)
        for (int ub = 0; ub < U; ub += gwarps) {
            const int u = ub + gwarp;
            const bool valid = u < U;
            int below = 0, s = 0, c = 0;
            if (valid) {
                const unsigned long long my = in_smem ? S.ukeys[u] : __ldcg(&B.ukey[u]);
                if (in_smem) {
#pragma unroll 4
                    for (int v = lane; v < U; v += 32) below += (S.ukeys[v] < my) ? 1 : 0;
                } else {
#pragma unroll 4
                    for (int v = lane; v < U; v += 32) below += (__ldcg(&B.ukey[v]) < my) ? 1 : 0;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) below += __shfl_xor_sync(0xffffffffu, below, o);
                if (lane == 0) {
                    s = __ldcg(&B.uslot[u]);
                    c = __ldcg(&B.hcnt[s]);
                    if (c > VGC_VCAP) atomicOr(&ctl[1], 2u);
                }
            }
            if (lane == 0) S.red[0][warp] = c;                 // (the box partials in S.red were consumed before barrier 1)
            __syncthreads();
            if (tid == 0) {
                int tot = 0;
                for (int w = 0; w < VGC_WARPS; ++w) tot += S.red[0][w];
                S.red[1][0] = tot ? (int)atomicAdd(&ctl[3], (unsigned int)tot) : 0;
            }
            __syncthreads();
            if (valid && lane == 0) {
                int off = S.red[1][0];
                for (int w = 0; w < warp; ++w) off += S.red[0][w];
                B.hoff[s] = off;
                B.urank[u] = below;
            }
            __syncthreads();
        }
        vgc_barrier(&ctl[0], 2u * G);
        if (stamp) stamp[2] = clock64();
        bail = *reinterpret_cast<volatile unsigned int*>(&ctl[1]);
    }
    if (bail) {
        // declined: leave the table clean for the next launch and report an empty result with the bail mark
        for (int s = gtid; s < VGC_T; s += gthreads) { B.hkey[s] = VGC_EMPTY; B.hcnt[s] = 0; }
        if (blockIdx.x == 0 && tid == 0) {
            VgParams p;
            p.inv_leaf = inv_leaf;
            for (int k = 0; k < 3; ++k) { p.min_b[k] = 0; p.div_b[k] = 1; p.mul[k] = 1; }
            p.overflow = 0; p.n_finite = 0; p.bail = 1;
            *pp = p;
            *count_out = 0;
        }
        return;
    }

    // ---- phase 3: group the point indices by voxel
    for (int i = gtid; i < n; i += gthreads) {
        const int s = __ldcg(&B.pslot[i]);
        if (s >= 0) B.members[__ldcg(&B.hoff[s]) + __ldcg(&B.ppos[i])] = i;
    }
    vgc_barrier(&ctl[0], 3u * G);
    if (stamp) stamp[3] = clock64();

    // ---- phase 4: one warp per voxel — members in ascending original index, sequential fp32 sums
    constexpr int NF = kVgFields<STRIDE>;
    for (int u = gwarp; u < U; u += gwarps) {
        const int s = __ldcg(&B.uslot[u]);
        const int c = __ldcg(&B.hcnt[s]);
        const int off = __ldcg(&B.hoff[s]);
        const int o = __ldcg(&B.urank[u]);
        // order by counting (indices are distinct)
        for (int j = lane; j < c; j += 32) {
            const int m = __ldcg(&B.members[off + j]);
            int below = 0;
            for (int k = 0; k < c; ++k) below += (__ldcg(&B.members[off + k]) < m) ? 1 : 0;
            S.sidx[warp][below] = m;
        }
        __syncwarp();
        float acc = 0.f;       // lane f < NF owns field f
        for (int base = 0; base < c; base += 32) {
            const int j = base + lane;
            if (j < c) vg_load<STRIDE>(pts + (size_t)S.sidx[warp][j] * STRIDE, S.stage[warp][lane]);
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
    }
    vgc_layout(B, (unsigned char*)c->vg_coop.p, grid);
    LILI_CUDA(c, c->vg_params.ensure(sizeof(VgParams)));
    const unsigned char* in = (const unsigned char*)d_in;
    unsigned char* outp = (unsigned char*)d_out;
    VgParams* pp = c->vg_params.as<VgParams>();
    unsigned int call = (c->vg_coop_calls & 0x7fffffffu) | (c->dbg_timing ? 0x80000000u : 0u);
    void* kargs[] = {&in, &n_max, &d_n, &leaf, &B, &call, &pp, &outp, &d_count, &d_feats};
    const void* fn = stride == 48 ? (const void*)k_vg_coop<48> : (const void*)k_vg_coop<32>;
    LILI_CUDA(c, cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(VGC_THREADS), kargs, 0, c->stream));
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
        k_vg_minmax<<<min(cdiv(n_max, 256), c->sm_count * 8), 256, 0, c->stream>>>((const unsigned char*)d_in, n_max, d_n, stride, mm);
        LILI_TRY(launch_check(c, "k_vg_minmax"));
    }
    return LILIOM_OK;
}

// key_bits < 32: the caller speculates that the voxel index fits that width (one onesweep pass less per 8 bits) and must check
// `ncells <= 2^key_bits - 1` afterwards (vg_params stays on the device).  host_mm (optional): the cloud's box and finite count
// already known on the host -> no pass over the input for it, and the key width follows from the box (vg_key_bits).
int voxelgrid_dev(liliom_ctx* c, const void* d_in, int n_max, const int* d_n, int stride, float leaf, void* d_out, int* d_count,
                  float4* d_feats, int key_bits, const int* host_mm) {
    if (stride != 48 && stride != 32) return LILIOM_E_ARG;
    if (host_mm) key_bits = vg_key_bits(host_mm, leaf);
    if (n_max <= 0) {
        LILI_CUDA(c, cudaMemsetAsync(d_count, 0, sizeof(int), c->stream));
        return LILIOM_OK;
    }
    const unsigned char* in = (const unsigned char*)d_in;
    const int n = n_max;
    LILI_CUDA(c, c->vg_minmax.ensure(8 * sizeof(int)));
    LILI_CUDA(c, c->vg_params.ensure(sizeof(VgParams)));
    LILI_CUDA(c, c->vg_keys.ensure((size_t)n * 4));
    LILI_CUDA(c, c->vg_vals.ensure((size_t)n * 4));
    LILI_CUDA(c, c->vg_keys2.ensure((size_t)n * 4));
    LILI_CUDA(c, c->vg_vals2.ensure((size_t)n * 4));
    LILI_CUDA(c, c->vg_flags.ensure(((size_t)n + 2) * 4));
    LILI_CUDA(c, c->vg_rank.ensure(((size_t)n + 2) * 4));
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
    k_vg_keys<<<cdiv(n, 256), 256, 0, c->stream>>>(in, n, d_n, stride, pp, c->vg_keys.as<uint32_t>(), c->vg_vals.as<int>());
    LILI_TRY(launch_check(c, "k_vg_keys"));
    // non-finite points carry the all-ones key (folded to the sort's width) and sort last; VgParams::n_finite excludes them
    LILI_TRY(sort_pairs_u32(c, c->vg_keys.as<uint32_t>(), c->vg_keys2.as<uint32_t>(), c->vg_vals.as<int>(), c->vg_vals2.as<int>(), n, key_bits));
    k_vg_heads<<<cdiv(n + 1, 256), 256, 0, c->stream>>>(c->vg_keys2.as<uint32_t>(), n, &pp->n_finite, c->vg_flags.as<int>());
    LILI_TRY(launch_check(c, "k_vg_heads"));
    LILI_TRY(exclusive_scan_i32(c, c->vg_flags.as<int>(), c->vg_rank.as<int>(), n));
    if (stride == 48)
        k_vg_centroid<48><<<cdiv(n, 128), 128, 0, c->stream>>>(in, c->vg_keys2.as<uint32_t>(), c->vg_vals2.as<int>(), c->vg_flags.as<int>(),
                                                               c->vg_rank.as<int>(), n, d_n, pp, (unsigned char*)d_out, d_count, d_feats);
    else
        k_vg_centroid<32><<<cdiv(n, 128), 128, 0, c->stream>>>(in, c->vg_keys2.as<uint32_t>(), c->vg_vals2.as<int>(), c->vg_flags.as<int>(),
                                                               c->vg_rank.as<int>(), n, d_n, pp, (unsigned char*)d_out, d_count, d_feats);
    LILI_TRY(launch_check(c, "k_vg_centroid"));
    return LILIOM_OK;
}

}  // namespace lili
