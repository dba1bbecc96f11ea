// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.h).  Pinned to the reference's own code: DESIGN.md §6.
// pcl::VoxelGrid, exact 5-NN (pcl::KdTreeFLANN semantics) and transformCloud restated.
#include "oracle_api.h"
#include "oracle_math.h"
#include <vector>
#include <cstring>
#include <climits>
#include <limits>
#include <numeric>
#ifdef _OPENMP
#include <omp.h>
#endif

using namespace orc;

// ---------------------------------------------------------------------------------------
// from-knowledge: pcl::VoxelGrid<PointT>::applyFilter (PCL 1.8-1.10), downsample_all_data
// = true, min_points_per_voxel = 0.  Within-voxel order: PCL uses an unstable std::sort on
// the voxel index; the restatement DEFINES it as original-index order (stable sort).
// Centroid (pcl::CentroidPoint, PCL >= 1.8): xyz, intensity, curvature = fp32 sum / n;
// normal = fp32 sum, then normalised (no division).
// Call sites: LiLi-OM/src/LidarOdometry.cpp:315-323 (leaf 0.4, :155-156),
//             LiLi-OM-ROT/src/Preprocessing.cpp:502-508 (leaf 0.6).
// ---------------------------------------------------------------------------------------
template <class P> struct Traits;
template <> struct Traits<orc_pt48> { static constexpr bool has_normal = true; };
template <> struct Traits<orc_pt32> { static constexpr bool has_normal = false; };

// int(float) and int64_t(float) as PCL's x86-64 build converts them (cvttss2si): truncation, or INT_MIN / INT64_MIN for NaN,
// +-inf and every value out of range (a far cluster: |x| / leaf >= 2^31 sends every x index to INT_MIN).  Written out: the
// plain conversion is undefined in C++ out of range.
static inline int x86_int(float v) { return scan_id_of(v); }
static inline int64_t x86_int64(float v) {
    return (v >= -9223372036854775808.0f && v < 9223372036854775808.0f) ? (int64_t)v : INT64_MIN;
}
static inline int64_t wrap_add(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); }
static inline int64_t wrap_mul(int64_t a, int64_t b) { return (int64_t)((uint64_t)a * (uint64_t)b); }
static inline int wrap_add32(int a, int b) { return (int)((unsigned)a + (unsigned)b); }
static inline int wrap_mul32(int a, int b) { return (int)((unsigned)a * (unsigned)b); }

template <class P>
static int voxelgrid_t(const P* in, int n, float leaf, P* out, int cap) {
    if (n <= 0) return 0;
    const float inv = 1.0f / leaf;
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    int nfinite = 0;
    for (int i = 0; i < n; ++i) {
        const P& p = in[i];
        if (!std::isfinite(p.x) || !std::isfinite(p.y) || !std::isfinite(p.z)) continue;
        ++nfinite;
        mn[0] = std::min(mn[0], p.x); mx[0] = std::max(mx[0], p.x);
        mn[1] = std::min(mn[1], p.y); mx[1] = std::max(mx[1], p.y);
        mn[2] = std::min(mn[2], p.z); mx[2] = std::max(mx[2], p.z);
    }
    if (nfinite == 0) return 0;
    int64_t dx = wrap_add(x86_int64((mx[0] - mn[0]) * inv), 1);
    int64_t dy = wrap_add(x86_int64((mx[1] - mn[1]) * inv), 1);
    int64_t dz = wrap_add(x86_int64((mx[2] - mn[2]) * inv), 1);
    if (wrap_mul(wrap_mul(dx, dy), dz) > (int64_t)INT_MAX) {
        // "Leaf size is too small for the input dataset. Integer indices would overflow." -> output = input
        int m = std::min(n, cap);
        std::memcpy(out, in, sizeof(P) * (size_t)m);
        return n;
    }
    int min_b[3], max_b[3], div_b[3];
    for (int a = 0; a < 3; ++a) {
        min_b[a] = x86_int(std::floor(mn[a] * inv));
        max_b[a] = x86_int(std::floor(mx[a] * inv));
        div_b[a] = wrap_add32(wrap_add32(max_b[a], -min_b[a]), 1);
    }
    const int mul[3] = {1, div_b[0], wrap_mul32(div_b[0], div_b[1])};
    std::vector<std::pair<unsigned, int>> iv;
    iv.reserve(n);
    for (int i = 0; i < n; ++i) {
        const P& p = in[i];
        if (!std::isfinite(p.x) || !std::isfinite(p.y) || !std::isfinite(p.z)) continue;
        int i0 = x86_int(std::floor(p.x * inv) - (float)min_b[0]);
        int i1 = x86_int(std::floor(p.y * inv) - (float)min_b[1]);
        int i2 = x86_int(std::floor(p.z * inv) - (float)min_b[2]);
        int idx = wrap_add32(wrap_add32(wrap_mul32(i0, mul[0]), wrap_mul32(i1, mul[1])), wrap_mul32(i2, mul[2]));
        iv.emplace_back((unsigned)idx, i);
    }
    std::stable_sort(iv.begin(), iv.end(),
                     [](const std::pair<unsigned, int>& a, const std::pair<unsigned, int>& b) { return a.first < b.first; });
    int nout = 0;
    size_t i = 0;
    while (i < iv.size()) {
        size_t j = i + 1;
        while (j < iv.size() && iv[j].first == iv[i].first) ++j;
        float sx = 0, sy = 0, sz = 0, si = 0, sc = 0, snx = 0, sny = 0, snz = 0;
        for (size_t k = i; k < j; ++k) {
            const P& p = in[iv[k].second];
            sx += p.x; sy += p.y; sz += p.z; si += p.intensity;
            if constexpr (Traits<P>::has_normal) {
                sc += p.curvature; snx += p.nx; sny += p.ny; snz += p.nz;
            }
        }
        const float cnt = (float)(j - i);
        if (nout < cap) {
            P o;
            std::memset(&o, 0, sizeof(P));
            o.x = sx / cnt; o.y = sy / cnt; o.z = sz / cnt; o.w = 1.0f;
            o.intensity = si / cnt;
            if constexpr (Traits<P>::has_normal) {
                o.curvature = sc / cnt;
                // Eigen normalize(): v /= sqrt(squaredNorm) if squaredNorm > 0
                float n2 = snx * snx + sny * sny + snz * snz;
                if (n2 > 0.0f) {
                    float nn = std::sqrt(n2);
                    o.nx = snx / nn; o.ny = sny / nn; o.nz = snz / nn;
                } else {
                    o.nx = snx; o.ny = sny; o.nz = snz;
                }
                o.nw = 0.0f;
            }
            out[nout] = o;
        }
        ++nout;
        i = j;
    }
    return nout;
}

extern "C" int orc_voxelgrid(const void* pts, int n, int stride, float leaf, void* out, int cap) {
    if (stride == 48) return voxelgrid_t<orc_pt48>((const orc_pt48*)pts, n, leaf, (orc_pt48*)out, cap);
    if (stride == 32) return voxelgrid_t<orc_pt32>((const orc_pt32*)pts, n, leaf, (orc_pt32*)out, cap);
    return -1;
}

// ---------------------------------------------------------------------------------------
// from-knowledge: FLANN KDTreeSingleIndex + L2_Simple<float> through pcl::KdTreeFLANN:
// exact K nearest, squared distance accumulated in fp32 as ((dx*dx)+dy*dy)+dz*dz, sorted
// ascending.  Tie order in FLANN is traversal order (unspecified); DEFINED here as
// ascending point index.  The tree below is our own (median split, bucket leaves); only
// the result set is specified by the reference, not the tree shape.
// ---------------------------------------------------------------------------------------
namespace {

struct KdNode {
    int lo, hi;        // point range [lo, hi) in the permuted array
    int left, right;   // children (-1 for leaf)
    int dim;
    float split_lo, split_hi;  // max of the left child / min of the right child along dim
};

struct KdTree {
    std::vector<float> px, py, pz;  // permuted coordinates
    std::vector<int> id;            // permuted -> original index
    std::vector<KdNode> nodes;
    int m = 0;
};

static inline float sqdist3(float ax, float ay, float az, float bx, float by, float bz) {
    float dx = ax - bx, dy = ay - by, dz = az - bz;
    float r = dx * dx;
    r += dy * dy;
    r += dz * dz;
    return r;
}

struct Top5 {
    float d[5];
    int i[5];
    int cnt = 0;
    Top5() { for (int k = 0; k < 5; ++k) { d[k] = std::numeric_limits<float>::infinity(); i[k] = -1; } }
    static inline bool less(float da, int ia, float db, int ib) { return da < db || (da == db && ia < ib); }
    inline float worst() const { return d[4]; }
    inline void push(float dist, int idx) {
        if (!(cnt < 5 || less(dist, idx, d[4], i[4]))) return;
        int k = cnt < 5 ? cnt : 4;
        while (k > 0 && less(dist, idx, d[k - 1], i[k - 1])) {
            d[k] = d[k - 1]; i[k] = i[k - 1]; --k;
        }
        d[k] = dist; i[k] = idx;
        if (cnt < 5) ++cnt;
    }
};

static int build_rec(KdTree& t, const float* xyzw, std::vector<int>& order, int lo, int hi) {
    int me = (int)t.nodes.size();
    t.nodes.push_back({lo, hi, -1, -1, 0, 0.f, 0.f});
    if (hi - lo <= 12) return me;
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int k = lo; k < hi; ++k) {
        const float* p = xyzw + 4 * (size_t)order[k];
        for (int a = 0; a < 3; ++a) { mn[a] = std::min(mn[a], p[a]); mx[a] = std::max(mx[a], p[a]); }
    }
    int dim = 0;
    if (mx[1] - mn[1] > mx[dim] - mn[dim]) dim = 1;
    if (mx[2] - mn[2] > mx[dim] - mn[dim]) dim = 2;
    if (!(mx[dim] > mn[dim])) return me;  // all points identical -> leaf
    int mid = (lo + hi) / 2;
    std::nth_element(order.begin() + lo, order.begin() + mid, order.begin() + hi, [&](int a, int b) {
        float va = xyzw[4 * (size_t)a + dim], vb = xyzw[4 * (size_t)b + dim];
        return va < vb || (va == vb && a < b);
    });
    float slo = -FLT_MAX, shi = FLT_MAX;
    for (int k = lo; k < mid; ++k) slo = std::max(slo, xyzw[4 * (size_t)order[k] + dim]);
    for (int k = mid; k < hi; ++k) shi = std::min(shi, xyzw[4 * (size_t)order[k] + dim]);
    int l = build_rec(t, xyzw, order, lo, mid);
    int r = build_rec(t, xyzw, order, mid, hi);
    t.nodes[me].left = l; t.nodes[me].right = r; t.nodes[me].dim = dim;
    t.nodes[me].split_lo = slo; t.nodes[me].split_hi = shi;
    return me;
}

static void search_rec(const KdTree& t, int ni, const float q[3], Top5& top) {
    const KdNode& nd = t.nodes[ni];
    if (nd.left < 0) {
        for (int k = nd.lo; k < nd.hi; ++k) top.push(sqdist3(q[0], q[1], q[2], t.px[k], t.py[k], t.pz[k]), t.id[k]);
        return;
    }
    float qv = q[nd.dim];
    // distance (fp32, squared) from q to each child's slab along dim; 0 when inside
    float dl = qv > nd.split_lo ? (qv - nd.split_lo) * (qv - nd.split_lo) : 0.f;
    float dr = qv < nd.split_hi ? (nd.split_hi - qv) * (nd.split_hi - qv) : 0.f;
    int first = nd.left, second = nd.right;
    float dsecond = dr;
    if (dr < dl) { first = nd.right; second = nd.left; dsecond = dl; }
    search_rec(t, first, q, top);
    if (top.cnt < 5 || dsecond <= top.worst()) search_rec(t, second, q, top);
}

}  // namespace

extern "C" void* orc_kdtree_build(const float* map_xyzw, int m) {
    KdTree* t = new KdTree();
    t->m = m;
    std::vector<int> order(m);
    std::iota(order.begin(), order.end(), 0);
    t->nodes.reserve(m / 4 + 16);
    if (m > 0) build_rec(*t, map_xyzw, order, 0, m);
    t->px.resize(m); t->py.resize(m); t->pz.resize(m); t->id.resize(m);
    for (int k = 0; k < m; ++k) {
        const float* p = map_xyzw + 4 * (size_t)order[k];
        t->px[k] = p[0]; t->py[k] = p[1]; t->pz[k] = p[2]; t->id[k] = order[k];
    }
    return t;
}

extern "C" void orc_kdtree_free(void* tree) { delete (KdTree*)tree; }

extern "C" void orc_knn5(const void* tree, const float* q_xyzw, int nq, int* idx, float* sqd, int nthreads) {
    const KdTree& t = *(const KdTree*)tree;
    (void)nthreads;
#pragma omp parallel for schedule(dynamic, 256) num_threads(nthreads > 0 ? nthreads : 1)
    for (int i = 0; i < nq; ++i) {
        Top5 top;
        if (t.m > 0) search_rec(t, 0, q_xyzw + 4 * (size_t)i, top);
        for (int k = 0; k < 5; ++k) { idx[5 * (size_t)i + k] = top.i[k]; sqd[5 * (size_t)i + k] = top.d[k]; }
    }
}

extern "C" void orc_knn5_brute(const float* map_xyzw, int m, const float* q_xyzw, int nq, int* idx, float* sqd) {
    for (int i = 0; i < nq; ++i) {
        Top5 top;
        const float* q = q_xyzw + 4 * (size_t)i;
        for (int k = 0; k < m; ++k) {
            const float* p = map_xyzw + 4 * (size_t)k;
            top.push(sqdist3(q[0], q[1], q[2], p[0], p[1], p[2]), k);
        }
        for (int k = 0; k < 5; ++k) { idx[5 * (size_t)i + k] = top.i[k]; sqd[5 * (size_t)i + k] = top.d[k]; }
    }
}

// internal helper used by oracle_s2m.cpp / oracle_backend.cpp
namespace orc {
void knn5_one(const void* tree, const float q[3], int idx[5], float sqd[5]) {
    const KdTree& t = *(const KdTree*)tree;
    Top5 top;
    if (t.m > 0) search_rec(t, 0, q, top);
    for (int k = 0; k < 5; ++k) { idx[k] = top.i[k]; sqd[k] = top.d[k]; }
}
}  // namespace orc

// ---------------------------------------------------------------------------------------
// LidarOdometry::undistortion — LiLi-OM/src/LidarOdometry.cpp:178-199: every point of a keyframe cloud is moved to the end of
// the sweep, p' = slerp(I, quat; ratio) * p + ratio * trans with ratio = min(frac(intensity) / 0.1, 1).  In place; only
// x, y, z change.  (publishCloudLast :624-632 calls it with quat = identity and trans = the relative translation.)
// ---------------------------------------------------------------------------------------
extern "C" void orc_undistort(void* pts, int n, int stride, const double trans[3], const double quat_wxyz[4]) {
    const Quat quat{quat_wxyz[0], quat_wxyz[1], quat_wxyz[2], quat_wxyz[3]};
    const double dt = 0.1;
    for (int i = 0; i < n; ++i) {
        float* p = reinterpret_cast<float*>((unsigned char*)pts + (size_t)i * stride);
        const float intensity = stride == 48 ? p[8] : p[4];
        const int line = scan_id_of(intensity);
        const double dt_i = intensity - line;
        double ratio_i = dt_i / dt;
        if (ratio_i > 1) ratio_i = 1;
        const Quat q_si = qslerp(Quat{1, 0, 0, 0}, ratio_i, quat);
        const V3 pt_s = qrot(q_si, V3{p[0], p[1], p[2]}) + V3{ratio_i * trans[0], ratio_i * trans[1], ratio_i * trans[2]};
        p[0] = (float)pt_s.x; p[1] = (float)pt_s.y; p[2] = (float)pt_s.z;
    }
}

// ---------------------------------------------------------------------------------------
// LidarOdometry::transformCloud — LiLi-OM/src/LidarOdometry.cpp:246-278 (48 B: rotates the
// normal, copies intensity+curvature); LiLi-OM-ROT/src/LidarOdometry.cpp:239-264 (32 B).
// ---------------------------------------------------------------------------------------
extern "C" void orc_transform_cloud(const void* in, int n, int stride, const double pose7[7], void* out) {
    Quat q{pose7[0], pose7[1], pose7[2], pose7[3]};
    V3 t{pose7[4], pose7[5], pose7[6]};
    for (int i = 0; i < n; ++i) {
        if (stride == 48) {
            const orc_pt48& p = ((const orc_pt48*)in)[i];
            orc_pt48 o;
            std::memset(&o, 0, sizeof(o));
            V3 po = qrot(q, V3{p.x, p.y, p.z}) + t;
            V3 no = qrot(q, V3{p.nx, p.ny, p.nz});
            o.x = (float)po.x; o.y = (float)po.y; o.z = (float)po.z; o.w = 1.0f;
            o.intensity = p.intensity; o.curvature = p.curvature;
            o.nx = (float)no.x; o.ny = (float)no.y; o.nz = (float)no.z;
            ((orc_pt48*)out)[i] = o;
        } else {
            const orc_pt32& p = ((const orc_pt32*)in)[i];
            orc_pt32 o;
            std::memset(&o, 0, sizeof(o));
            V3 po = qrot(q, V3{p.x, p.y, p.z}) + t;
            o.x = (float)po.x; o.y = (float)po.y; o.z = (float)po.z; o.w = 1.0f;
            o.intensity = p.intensity;
            ((orc_pt32*)out)[i] = o;
        }
    }
}
