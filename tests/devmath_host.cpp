// TEST INFRASTRUCTURE: host build of the device scalar routines (liliom_b200/csrc/dev_math.cuh) so that the CPU test tier can
// exercise the SAME SOURCE the kernels compile — plane fit (fast path + rank-revealing QR fallback), plane gates, residual rows,
// Huber / Cauchy correctors and the 29-sum fold, 6x6 LDL^T, Ceres' Plus, the 3x3 symmetric eigensolver — against NumPy and
// against the oracle's independent copies.  The round-to-nearest intrinsics become plain operators (this file is compiled with
// -ffp-contract=off, so nothing is fused either).
#include <cmath>
#include <cfloat>
#include <cstring>
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fsqrt_rn(float a) { return std::sqrt(a); }
using std::isfinite;
#include <cuda_runtime.h>
#ifndef __noinline__
#define __noinline__
#endif
#include "../liliom_b200/csrc/dev_math.cuh"

using namespace lili;

extern "C" {
int dm_plane_fit5(const float* m20, double nv[3]) {          // returns 1 when the fast path produced the answer, 0 for the QR fallback
    float4 m[5];
    for (int j = 0; j < 5; ++j) m[j] = make_float4(m20[4 * j], m20[4 * j + 1], m20[4 * j + 2], m20[4 * j + 3]);
    double kS, kA2, cn;
    if (plane_fit5_fast(m, nv, kS, kA2, cn)) return 1;
    plane_fit5_qr(m, nv);
    return 0;
}
// n neighbourhoods (m20: n x 5 x 4 floats, s3: n x 3 transformed queries) through plane_fit_gate, as phase B of the GN pass runs
// it, at the thresholds plane_thres[i] and w_gate[i]: ok[i], path[i] (0 fast, 1 declined, 2 guard band), pl4 / weight (left as passed in when refused).  When fit is given, also
// the fast path's own normal (fit[4 i .. 4 i + 2], un-normalised; fit[4 i + 3] = 1 when the fast path took the set) and its
// fit-error bound rho (plane_fit_gate's, NaN when the fast path declined) in rho[i].
void dm_fit_gate_batch(const float* m20, const float* s3, int n, const double* plane_thres, const double* w_gate, unsigned char* ok, int* path,
                       float* pl4, float* weight, double* fit, double* rho) {
    for (int i = 0; i < n; ++i) {
        float4 m[5];
        const float* p = m20 + 20 * (size_t)i;
        for (int j = 0; j < 5; ++j) m[j] = make_float4(p[4 * j], p[4 * j + 1], p[4 * j + 2], p[4 * j + 3]);
        const float* s = s3 + 3 * (size_t)i;
        float4 pl = make_float4(pl4[4 * i], pl4[4 * i + 1], pl4[4 * i + 2], pl4[4 * i + 3]);
        ok[i] = plane_fit_gate(m, s[0], s[1], s[2], plane_thres[i], w_gate[i], pl, weight[i], path[i]) ? 1 : 0;
        pl4[4 * i] = pl.x; pl4[4 * i + 1] = pl.y; pl4[4 * i + 2] = pl.z; pl4[4 * i + 3] = pl.w;
        if (fit) {
            double nv[3], kS, kA2, cn;
            const bool fast = plane_fit5_fast(m, nv, kS, kA2, cn);
            for (int k = 0; k < 3; ++k) fit[4 * (size_t)i + k] = fast ? nv[k] : 0.0;
            fit[4 * (size_t)i + 3] = fast ? 1.0 : 0.0;
            if (fast) {       // plane_fit_gate's rho from the same quantities
                double n[3] = {nv[0], nv[1], nv[2]};
                double nn;
                const double ninv = gate_normalise(n, nn);
                double dmax = 0.0;
                for (int j = 0; j < 5; ++j) dmax = fmax(dmax, gate_dist(n, ninv, m[j].x, m[j].y, m[j].z));
                rho[i] = fit_err_bound(kS, kA2, cn, nn, dmax);
            } else {
                rho[i] = NAN;
            }
        }
    }
}
int dm_solve6(const double s21[21], const double rhs[6], double x[6]) { return solve6_ldlt(s21, rhs, x) ? 1 : 0; }
int dm_gn_safe_step(const double s21[21], const double rhs[6], double d[6]) { return gn_safe_step(s21, rhs, d) ? 1 : 0; }
void dm_pose_plus(const double x[7], const double d[6], double out[7]) { pose_plus(x, d, out); }
void dm_eigen_sym3(const double a[6], double ev[3], double evec[9]) {     // a = {a00, a10, a20, a11, a21, a22}
    double v[3][3];
    eigen_sym3(a[0], a[1], a[2], a[3], a[4], a[5], ev, v);
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) evec[3 * r + c] = v[r][c];
}
void dm_colpiv_qr(const double A15[15], const double b5[5], double x[3]) {
    double A[5][3], b[5];
    for (int j = 0; j < 5; ++j) { for (int k = 0; k < 3; ++k) A[j][k] = A15[3 * j + k]; b[j] = b5[j]; }
    colpiv_qr_solve_5x3(A, b, x);
}
void dm_qslerp_identity(const double q[4], double t, double out[4]) {     // slerp(Identity -> q; t), not re-normalised
    const Q4 r = qslerp_x(Q4{1.0, 0.0, 0.0, 0.0}, t, Q4{q[0], q[1], q[2], q[3]});
    out[0] = r.w; out[1] = r.x; out[2] = r.y; out[3] = r.z;
}
int dm_scan_id_of(float x) { return scan_id_of(x); }
void dm_qrot(const double q[4], const double v[3], double out[3]) {
    D3 r = qrot_x(Q4{q[0], q[1], q[2], q[3]}, D3{v[0], v[1], v[2]});
    out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
// plane_gate on the fitted nv (normalised in place) of the neighbours m20 and the query s3; pl4 / weight are left as passed in
// when the plane is refused
int dm_plane_gate(double nv[3], const float* m20, const float s3[3], double plane_thres, double w_gate, int refuse, float pl4[4],
                  float* weight) {
    float4 m[5];
    for (int j = 0; j < 5; ++j) m[j] = make_float4(m20[4 * j], m20[4 * j + 1], m20[4 * j + 2], m20[4 * j + 3]);
    float4 pl = make_float4(pl4[0], pl4[1], pl4[2], pl4[3]);
    const bool ok = plane_gate(nv, m, s3[0], s3[1], s3[2], plane_thres, w_gate, refuse != 0, pl, *weight);
    pl4[0] = pl.x; pl4[1] = pl.y; pl4[2] = pl.z; pl4[3] = pl.w;
    return ok ? 1 : 0;
}
// the 29 sums of the scan-to-map rows (plane_row + huber_correct + add_row29) of the valid correspondences at pose7
void dm_plane_neq(const float* feats4, int n, const unsigned char* valid, const float* plane4, const double pose7[7], double huber_a,
                  double out29[29]) {
    const Q4 q{pose7[0], pose7[1], pose7[2], pose7[3]};
    const D3 t{pose7[4], pose7[5], pose7[6]};
    for (int k = 0; k < 29; ++k) out29[k] = 0.0;
    for (int i = 0; i < n; ++i) {
        if (!valid[i]) continue;
        const float* f = feats4 + 4 * (size_t)i;
        Row R = plane_row(q, t, f[0], f[1], f[2], make_float4(plane4[4 * i], plane4[4 * i + 1], plane4[4 * i + 2], plane4[4 * i + 3]));
        huber_correct(R, huber_a);
        add_row29(out29, R);
    }
}
// the 29 sums of n raw rows (J6[6 * i ..], r[i]) through cauchy_correct + add_row29
void dm_cauchy_fold(const double* J6, const double* r, int n, double cauchy_b, double out29[29]) {
    const double b2 = cauchy_b * cauchy_b, c2 = 1.0 / b2;
    for (int k = 0; k < 29; ++k) out29[k] = 0.0;
    for (int i = 0; i < n; ++i) {
        Row R;
        for (int k = 0; k < 6; ++k) R.J[k] = J6[6 * (size_t)i + k];
        R.r = r[i];
        cauchy_correct(R, b2, c2);
        add_row29(out29, R);
    }
}
}
