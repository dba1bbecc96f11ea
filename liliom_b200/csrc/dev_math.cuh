// Device scalar routines of the LiLi-OM hot path (sm_90a).
// The *_x ("exact") helpers spell every operation with round-to-nearest intrinsics so that
// nvcc never contracts them into FMAs: they reproduce bit-for-bit what the reference's
// generic x86-64 build computes (no FMA; SURVEY.md Appendix C.2), which is what makes the
// label / index outputs bit-exact.  Routines without _x may be contracted; they only feed
// tolerance-checked fp64 results.
#pragma once
#include <cuda_runtime.h>
#include <cfloat>
#include "pcl_xform.h"      // D3, Q4, mulx / addx / subx, cross_x, qrot_x, pcl_transform_point (shared with the host)

namespace lili {

__device__ __forceinline__ float fmulx(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float faddx(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsubx(float a, float b) { return __fsub_rn(a, b); }

// Hamilton product, Eigen operand order (a * b), exact ops.
__device__ __forceinline__ Q4 qmul_x(Q4 a, Q4 b) {
    Q4 r;
    r.w = subx(subx(subx(mulx(a.w, b.w), mulx(a.x, b.x)), mulx(a.y, b.y)), mulx(a.z, b.z));
    r.x = subx(addx(addx(mulx(a.w, b.x), mulx(a.x, b.w)), mulx(a.y, b.z)), mulx(a.z, b.y));
    r.y = subx(addx(addx(mulx(a.w, b.y), mulx(a.y, b.w)), mulx(a.z, b.x)), mulx(a.x, b.z));
    r.z = subx(addx(addx(mulx(a.w, b.z), mulx(a.z, b.w)), mulx(a.x, b.y)), mulx(a.y, b.x));
    return r;
}

// Eigen::Quaterniond::inverse()
__device__ __forceinline__ Q4 qinv_x(Q4 q) {
    double n2 = addx(addx(addx(mulx(q.w, q.w), mulx(q.x, q.x)), mulx(q.y, q.y)), mulx(q.z, q.z));
    if (n2 > 0) return {q.w / n2, -q.x / n2, -q.y / n2, -q.z / n2};
    return {0, 0, 0, 0};
}

// Eigen::Quaterniond::slerp(t, other) from `a`, result not re-normalised
// (L/src/Preprocessing.cpp:114-115).  acos/sin are CUDA's fp64 routines (<= 1-2 ulp from
// glibc's); their results are narrowed to fp32 point coordinates downstream.
__device__ __forceinline__ Q4 qslerp_x(Q4 a, double t, Q4 b) {
    const double one = 1.0 - DBL_EPSILON;
    double d = addx(addx(addx(mulx(a.w, b.w), mulx(a.x, b.x)), mulx(a.y, b.y)), mulx(a.z, b.z));
    double absD = fabs(d);
    double s0, s1;
    if (absD >= one) {
        s0 = subx(1.0, t);
        s1 = t;
    } else {
        double theta = acos(absD);
        double sinTheta = sin(theta);
        s0 = sin(mulx(subx(1.0, t), theta)) / sinTheta;
        s1 = sin(mulx(t, theta)) / sinTheta;
    }
    if (d < 0) s1 = -s1;
    return {addx(mulx(s0, a.w), mulx(s1, b.w)), addx(mulx(s0, a.x), mulx(s1, b.x)),
            addx(mulx(s0, a.y), mulx(s1, b.y)), addx(mulx(s0, a.z), mulx(s1, b.z))};
}

// ---------------------------------------------------------------------------------------
// 3x3 symmetric eigen-decomposition following the algorithm of
// Eigen::SelfAdjointEigenSolver<Matrix3d> (iterative path): max-abs scaling, closed-form 3x3
// Householder tridiagonalisation, implicit symmetric QR with Wilkinson shift, ascending order.
// Following the same algorithm (rather than an analytic solver) keeps eigenvector SIGNS equal
// to the reference's, which end up in the published normal_x/y/z fields
// (L/src/Preprocessing.cpp:354-360, 368-376).  Compile the including TU with --fmad=false
// when bit-stable labels are required.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void givens_rot(double p, double q, double& c, double& s) {
    if (q == 0.0) {
        c = p < 0 ? -1.0 : 1.0; s = 0.0;
    } else if (p == 0.0) {
        c = 0.0; s = q < 0 ? 1.0 : -1.0;
    } else if (fabs(p) > fabs(q)) {
        double t = q / p;
        double u = sqrt(1.0 + t * t);
        if (p < 0) u = -u;
        c = 1.0 / u; s = -t * c;
    } else {
        double t = p / q;
        double u = sqrt(1.0 + t * t);
        if (q < 0) u = -u;
        s = -1.0 / u; c = -t * s;
    }
}

__device__ __forceinline__ double hypot_pos(double x, double y) {
    double ax = fabs(x), ay = fabs(y);
    double p = ax > ay ? ax : ay;
    if (p == 0.0) return 0.0;
    double qp = (ax > ay ? ay : ax) / p;
    return p * sqrt(1.0 + qp * qp);
}

// a: symmetric, lower triangle read (a00,a10,a20,a11,a21,a22). evec[r][c] = component r of eigenvector c.
// The 3x3 case is written out on SCALARS (d0..d2, s0, s1, q00..q22): the same operations in the same order as the generic
// loops of the algorithm, but nothing is indexed at run time, so everything lives in registers (the indexed version kept
// diag/sub/Q in local memory: the patch stage of the Horizon extractor spent ~44k cycles per patch mostly there).
struct Eig3State { double d0, d1, d2, s0, s1, q00, q01, q02, q10, q11, q12, q20, q21, q22; };

// one Givens step of the implicit symmetric QR sweep on rows/columns (k, k+1); FIRST: k == start (no update of sub[k-1]),
// LAST: k == end-1 (no bulge into sub[k+1]).  K = 0 or 1 selects the scalars.
template <int K>
__device__ __forceinline__ void eig3_step(Eig3State& S, double& x, double& z, bool first, bool last) {
    double c, s;
    givens_rot(x, z, c, s);
    double& dk = K == 0 ? S.d0 : S.d1;
    double& dk1 = K == 0 ? S.d1 : S.d2;
    double& sk = K == 0 ? S.s0 : S.s1;
    const double sdk = s * dk + c * sk;
    const double dkp1 = s * sk + c * dk1;
    dk = c * (c * dk - s * sk) - s * (c * sk - s * dk1);
    dk1 = s * sdk + c * dkp1;
    sk = c * sdk - s * dkp1;
    if (!first) { if (K == 1) S.s0 = c * S.s0 - s * z; }      // sub[k-1] (only k = 1 has one)
    x = sk;
    if (!last) { if (K == 0) { z = -s * S.s1; S.s1 = c * S.s1; } }      // bulge (only k = 0 can have a successor)
    if (K == 0) {
        double a, b;
        a = S.q00; b = S.q01; S.q00 = c * a - s * b; S.q01 = s * a + c * b;
        a = S.q10; b = S.q11; S.q10 = c * a - s * b; S.q11 = s * a + c * b;
        a = S.q20; b = S.q21; S.q20 = c * a - s * b; S.q21 = s * a + c * b;
    } else {
        double a, b;
        a = S.q01; b = S.q02; S.q01 = c * a - s * b; S.q02 = s * a + c * b;
        a = S.q11; b = S.q12; S.q11 = c * a - s * b; S.q12 = s * a + c * b;
        a = S.q21; b = S.q22; S.q21 = c * a - s * b; S.q22 = s * a + c * b;
    }
}

// Returns the eigenvalues (ascending) in d0..d2 and eigenvector c in column c of q: a value, so that a caller that picks a
// column at run time does not force the result through local memory (eigen_sym3 below is the array form).
__device__ __forceinline__ Eig3State eigen_sym3_s(double a00, double a10, double a20, double a11, double a21, double a22) {
    double scale = fmax(fmax(fmax(fabs(a00), fabs(a10)), fmax(fabs(a20), fabs(a11))), fmax(fabs(a21), fabs(a22)));
    if (scale == 0.0) scale = 1.0;
    a00 /= scale; a10 /= scale; a20 /= scale; a11 /= scale; a21 /= scale; a22 /= scale;
    Eig3State S;
    S.d0 = a00;
    const double v1norm2 = a20 * a20;
    if (v1norm2 <= DBL_MIN) {
        S.d1 = a11; S.d2 = a22; S.s0 = a10; S.s1 = a21;
        S.q00 = 1; S.q01 = 0; S.q02 = 0; S.q10 = 0; S.q11 = 1; S.q12 = 0; S.q20 = 0; S.q21 = 0; S.q22 = 1;
    } else {
        const double beta = sqrt(a10 * a10 + v1norm2);
        const double invBeta = 1.0 / beta;
        const double m01 = a10 * invBeta;
        const double m02 = a20 * invBeta;
        const double q = 2.0 * m01 * a21 + m02 * (a22 - a11);
        S.d1 = a11 + m02 * q;
        S.d2 = a22 - m02 * q;
        S.s0 = beta;
        S.s1 = a21 - m01 * q;
        S.q00 = 1; S.q01 = 0;   S.q02 = 0;
        S.q10 = 0; S.q11 = m01; S.q12 = m02;
        S.q20 = 0; S.q21 = m02; S.q22 = -m01;
    }
    int end = 2, start = 0, iter = 0;
    const double precision_inv = 1.0 / DBL_EPSILON;
    while (end > 0) {
        // deflation test on sub[start..end)
        if (start <= 0 && 0 < end) {
            if (fabs(S.s0) < DBL_MIN) S.s0 = 0.0;
            else { const double ss = precision_inv * S.s0; if (ss * ss <= (fabs(S.d0) + fabs(S.d1))) S.s0 = 0.0; }
        }
        if (start <= 1 && 1 < end) {
            if (fabs(S.s1) < DBL_MIN) S.s1 = 0.0;
            else { const double ss = precision_inv * S.s1; if (ss * ss <= (fabs(S.d1) + fabs(S.d2))) S.s1 = 0.0; }
        }
        while (end > 0 && (end == 2 ? S.s1 : S.s0) == 0.0) end--;
        if (end <= 0) break;
        iter++;
        if (iter > 90) break;
        start = end - 1;
        while (start > 0 && (start == 2 ? S.s1 : S.s0) != 0.0) start--;        // sub[start-1]
        const double dEm1 = end == 2 ? S.d1 : S.d0, dE = end == 2 ? S.d2 : S.d1;
        const double td = (dEm1 - dE) * 0.5;
        const double e = end == 2 ? S.s1 : S.s0;
        double mu = dE;
        if (td == 0.0) {
            mu -= fabs(e);
        } else if (e != 0.0) {
            const double e2 = e * e;
            const double h = hypot_pos(td, e);
            if (e2 == 0.0) mu -= e / ((td + (td > 0 ? h : -h)) / e);
            else mu -= e2 / (td + (td > 0 ? h : -h));
        }
        double x = (start == 0 ? S.d0 : S.d1) - mu;
        double z = start == 0 ? S.s0 : S.s1;
        if (start == 0) {
            if (z != 0.0) {
                eig3_step<0>(S, x, z, true, end == 1);
                if (end == 2 && z != 0.0) eig3_step<1>(S, x, z, false, true);
            }
        } else {      // start == 1, end == 2
            if (z != 0.0) eig3_step<1>(S, x, z, true, true);
        }
    }
    // ascending selection sort of (eigenvalue, column), as the generic two-pass loop does it
    {
        int k = 0;
        if (S.d1 < S.d0) k = 1;
        if (S.d2 < (k == 1 ? S.d1 : S.d0)) k = 2;
        if (k == 1) { double t = S.d0; S.d0 = S.d1; S.d1 = t; t = S.q00; S.q00 = S.q01; S.q01 = t; t = S.q10; S.q10 = S.q11; S.q11 = t; t = S.q20; S.q20 = S.q21; S.q21 = t; }
        else if (k == 2) { double t = S.d0; S.d0 = S.d2; S.d2 = t; t = S.q00; S.q00 = S.q02; S.q02 = t; t = S.q10; S.q10 = S.q12; S.q12 = t; t = S.q20; S.q20 = S.q22; S.q22 = t; }
        if (S.d2 < S.d1) { double t = S.d1; S.d1 = S.d2; S.d2 = t; t = S.q01; S.q01 = S.q02; S.q02 = t; t = S.q11; S.q11 = S.q12; S.q12 = t; t = S.q21; S.q21 = S.q22; S.q22 = t; }
    }
    S.d0 = S.d0 * scale; S.d1 = S.d1 * scale; S.d2 = S.d2 * scale;
    return S;
}

__device__ inline void eigen_sym3(double a00, double a10, double a20, double a11, double a21, double a22,
                                  double eval[3], double evec[3][3]) {
    const Eig3State S = eigen_sym3_s(a00, a10, a20, a11, a21, a22);
    eval[0] = S.d0; eval[1] = S.d1; eval[2] = S.d2;
    evec[0][0] = S.q00; evec[0][1] = S.q01; evec[0][2] = S.q02;
    evec[1][0] = S.q10; evec[1][1] = S.q11; evec[1][2] = S.q12;
    evec[2][0] = S.q20; evec[2][1] = S.q21; evec[2][2] = S.q22;
}

// ---------------------------------------------------------------------------------------
// 5x3 least squares  A n = b  by column-pivoted Householder QR in fp64 (the algorithm of
// Eigen::ColPivHouseholderQR, L/src/LidarOdometry.cpp:375): map points sit hundreds of metres
// from the origin with sub-metre spread, so normal equations (condition squared) would cost
// ~1e-4 m in the plane offset — QR keeps it at ~1e-9 m.
// Everything is register-resident (fully unrolled, column permutation via swaps).
// kEigenOrder: apply each reflector to the trailing columns as Eigen's applyHouseholderOnTheLeft does (essential^T * bottom
// first, then the head row), the order of the oracle's copy, so that without contraction the bits are the oracle's
// (backend_corr.cu).  false keeps the head-row-first order the scan-to-map kernel (grid_knn.cu, compiled with contraction)
// has always used; moving it is a change of that kernel's results and belongs with its own bit-stability work.
// ---------------------------------------------------------------------------------------
template <bool kEigenOrder = true>
__device__ inline void colpiv_qr_solve_5x3(double A[5][3], double b[5], double x[3]) {
    double nu[3], ndir[3], tau[3];
    int perm[3] = {0, 1, 2};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        double s = 0;
#pragma unroll
        for (int i = 0; i < 5; ++i) s += A[i][k] * A[i][k];
        nu[k] = ndir[k] = sqrt(s);
    }
    double maxn = fmax(nu[0], fmax(nu[1], nu[2]));
    double th = maxn * DBL_EPSILON;
    const double threshold_helper = th * th / 5.0;
    const double downdate_thr = 1.4901161193847656e-08;   // sqrt(DBL_EPSILON)
    int nonzero = 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        int big = k;
        double bigv = nu[k];
#pragma unroll
        for (int j = k + 1; j < 3; ++j) if (nu[j] > bigv) { bigv = nu[j]; big = j; }
        double big_sq = bigv * bigv;
        if (nonzero == 3 && big_sq < threshold_helper * double(5 - k)) nonzero = k;
        if (big != k) {
#pragma unroll
            for (int j = k + 1; j < 3; ++j) {
                if (j == big) {
#pragma unroll
                    for (int i = 0; i < 5; ++i) { double t = A[i][k]; A[i][k] = A[i][j]; A[i][j] = t; }
                    double t = nu[k]; nu[k] = nu[j]; nu[j] = t;
                    t = ndir[k]; ndir[k] = ndir[j]; ndir[j] = t;
                    int p = perm[k]; perm[k] = perm[j]; perm[j] = p;
                }
            }
        }
        double tail = 0;
#pragma unroll
        for (int i = k + 1; i < 5; ++i) tail += A[i][k] * A[i][k];
        double c0 = A[k][k], beta, tk;
        if (tail <= DBL_MIN) {
            tk = 0; beta = c0;
#pragma unroll
            for (int i = k + 1; i < 5; ++i) A[i][k] = 0;
        } else {
            beta = sqrt(c0 * c0 + tail);
            if (c0 >= 0) beta = -beta;
            double inv = c0 - beta;
#pragma unroll
            for (int i = k + 1; i < 5; ++i) A[i][k] = A[i][k] / inv;
            tk = (beta - c0) / beta;
        }
        A[k][k] = beta;
        tau[k] = tk;
        if (tk != 0) {
#pragma unroll
            for (int j = k + 1; j < 3; ++j) {
                double tmp = kEigenOrder ? 0.0 : A[k][j];
#pragma unroll
                for (int i = k + 1; i < 5; ++i) tmp += A[i][k] * A[i][j];
                if (kEigenOrder) tmp += A[k][j];
                A[k][j] -= tk * tmp;
#pragma unroll
                for (int i = k + 1; i < 5; ++i) A[i][j] -= tk * A[i][k] * tmp;
            }
        }
#pragma unroll
        for (int j = k + 1; j < 3; ++j) {
            if (nu[j] != 0) {
                double temp = fabs(A[k][j]) / nu[j];
                temp = (1.0 + temp) * (1.0 - temp);
                temp = temp < 0 ? 0 : temp;
                double r = nu[j] / ndir[j];
                double temp2 = temp * r * r;
                if (temp2 <= downdate_thr) {
                    double s = 0;
#pragma unroll
                    for (int i = k + 1; i < 5; ++i) s += A[i][j] * A[i][j];
                    ndir[j] = sqrt(s);
                    nu[j] = ndir[j];
                } else {
                    nu[j] *= sqrt(temp);
                }
            }
        }
    }
    x[0] = x[1] = x[2] = 0;
    if (nonzero == 0) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (k < nonzero && tau[k] != 0) {
            double tmp = b[k];
#pragma unroll
            for (int i = k + 1; i < 5; ++i) tmp += A[i][k] * b[i];
            b[k] -= tau[k] * tmp;
#pragma unroll
            for (int i = k + 1; i < 5; ++i) b[i] -= tau[k] * A[i][k] * tmp;
        }
    }
    double c[3] = {b[0], b[1], b[2]};
#pragma unroll
    for (int i = 2; i >= 0; --i) {
        if (i < nonzero) {
            double s = c[i];
#pragma unroll
            for (int j = i + 1; j < 3; ++j) if (j < nonzero) s -= A[i][j] * c[j];
            c[i] = s / A[i][i];
        }
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        if (i < nonzero) {
            // scatter through the permutation without dynamic register indexing
            if (perm[i] == 0) x[0] = c[i];
            else if (perm[i] == 1) x[1] = c[i];
            else x[2] = c[i];
        }
    }
}

// ---------------------------------------------------------------------------------------
// Fast path of the same least-squares plane  min || A n + 1 ||  (A = the 5 neighbours):
// with c = centroid, q_j = p_j - c and S = sum q_j q_j^T,   A^T A = S + 5 c c^T,  A^T 1 = 5 c,
// so by Sherman-Morrison   n = -5 u / (1 + 5 c.u),   u = S^-1 c.
// S is built from CENTRED coordinates (differences of fp32 values are exact in fp64), so its
// conditioning is the patch's own spread ratio (~1e3..1e6) instead of (|p|/spread)^2 of the
// raw normal equations; a 3x3 LDL^T (stable for SPD without pivoting) then gives the same
// minimiser as the Householder QR to ~1e-12 relative, in ~1/8 of the fp64 instructions.
// Returns false when S is numerically singular (collinear / coincident / exactly coplanar
// neighbours): the caller then takes the rank-revealing QR path, which reproduces Eigen's
// behaviour for those cases.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ bool plane_fit5_fast(const float4 m[5], double nv[3]) {
    const double cx = ((double)m[0].x + (double)m[1].x + (double)m[2].x + (double)m[3].x + (double)m[4].x) * 0.2;
    const double cy = ((double)m[0].y + (double)m[1].y + (double)m[2].y + (double)m[3].y + (double)m[4].y) * 0.2;
    const double cz = ((double)m[0].z + (double)m[1].z + (double)m[2].z + (double)m[3].z + (double)m[4].z) * 0.2;
    double s00 = 0, s01 = 0, s02 = 0, s11 = 0, s12 = 0, s22 = 0;
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        const double qx = (double)m[j].x - cx, qy = (double)m[j].y - cy, qz = (double)m[j].z - cz;
        s00 += qx * qx; s01 += qx * qy; s02 += qx * qz; s11 += qy * qy; s12 += qy * qz; s22 += qz * qz;
    }
    const double tr = s00 + s11 + s22;
    const double tiny = 1e-9 * tr;
    // LDL^T of S
    const double d0 = s00;
    if (!(d0 > tiny)) return false;
    const double i0 = 1.0 / d0;
    const double l10 = s01 * i0, l20 = s02 * i0;
    const double d1 = s11 - l10 * s01;
    if (!(d1 > tiny)) return false;
    const double i1 = 1.0 / d1;
    const double t21 = s12 - l20 * s01;
    const double l21 = t21 * i1;
    const double d2 = s22 - l20 * s02 - l21 * t21;
    if (!(d2 > tiny)) return false;
    // u = S^-1 c
    const double y0 = cx, y1 = cy - l10 * y0, y2 = cz - l20 * y0 - l21 * y1;
    const double z2 = y2 / d2;
    const double z1 = y1 * i1 - l21 * z2;
    const double z0 = y0 * i0 - l10 * z1 - l20 * z2;
    const double den = 1.0 + 5.0 * (cx * z0 + cy * z1 + cz * z2);
    const double sc = -5.0 / den;
    nv[0] = sc * z0; nv[1] = sc * z1; nv[2] = sc * z2;
    return isfinite(nv[0]) && isfinite(nv[1]) && isfinite(nv[2]);
}

static __device__ __noinline__ void plane_fit5_qr(const float4 m[5], double nv[3]) {
    double A[5][3], B[5];
#pragma unroll
    for (int j = 0; j < 5; ++j) { A[j][0] = m[j].x; A[j][1] = m[j].y; A[j][2] = m[j].z; B[j] = -1.0; }
    colpiv_qr_solve_5x3<false>(A, B, nv);
}

// 6x6 SPD solve (LDL^T), H given as the 21-scalar upper triangle (row-major), rhs b.
// Fully unrolled so that every array lives in registers: this runs on ONE thread at the tail of
// the iteration kernel, where local-memory round trips would be pure exposed latency.
// Returns false on a non-finite / zero pivot.  `lambda` is added to every diagonal entry (Levenberg damping); with
// piv_min >= 0 a pivot that is not above piv_min also fails (relative conditioning test of the GN step, see gn_safe_step).
__device__ __forceinline__ bool solve6_ldlt(const double* s21, const double* rhs, double x[6], double lambda = 0.0, double piv_min = -1.0) {
    double H[6][6];
    {
        int k = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a)
#pragma unroll
            for (int b = a; b < 6; ++b) { H[a][b] = s21[k]; H[b][a] = s21[k]; ++k; }
    }
    double L[6][6], D[6], Dinv[6];
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        double d = H[j][j] + lambda;
#pragma unroll
        for (int m = 0; m < j; ++m) d -= L[j][m] * L[j][m] * D[m];
        if (!(fabs(d) > 1e-300) || !isfinite(d) || (piv_min >= 0.0 && !(d > piv_min))) ok = false;
        D[j] = d;
        const double inv = 1.0 / d;
        Dinv[j] = inv;
#pragma unroll
        for (int i = j + 1; i < 6; ++i) {
            double s = H[i][j];
#pragma unroll
            for (int m = 0; m < j; ++m) s -= L[i][m] * L[j][m] * D[m];
            L[i][j] = s * inv;
        }
    }
    double y[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        double s = rhs[i];
#pragma unroll
        for (int m = 0; m < i; ++m) s -= L[i][m] * y[m];
        y[i] = s;
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) y[i] *= Dinv[i];
#pragma unroll
    for (int i = 5; i >= 0; --i) {
        double s = y[i];
#pragma unroll
        for (int m = i + 1; m < 6; ++m) s -= L[m][i] * x[m];
        x[i] = s;
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) if (!isfinite(x[i])) ok = false;
    return ok;
}

static __device__ __noinline__ bool solve6_ldlt_damped(const double* s21, const double* rhs, double x[6], double lambda) {
    return solve6_ldlt(s21, rhs, x, lambda, 0.0);
}

// Gauss-Newton step of LILIOM_MODE_GN with the two safeguards an undamped step lacks (ADVICE r1; the reference's own solver is
// Ceres' trust-region LM, L/src/LidarOdometry.cpp:527-537 = LILIOM_MODE_CERES):
//   (1) conditioning: when a pivot of H = J^T J falls below 1e-10 * max diag(H) the scan does not constrain some direction
//       (a narrow-FoV sweep facing one wall, a corridor); the step is then taken from the Levenberg-damped system
//       (H + 1e-6 * max diag * I) d = -g, which moves the constrained directions and leaves the others (nearly) alone;
//   (2) trust region: a step of more than kGnMaxRot rad / kGnMaxTrans m is scaled back onto that bound.
// Neither triggers on a well-posed scan, where the step is the plain LDL^T solution.  oracle_s2m.cpp::gn_safe_step is the same.
constexpr double kGnPivotRel = 1e-10, kGnDampRel = 1e-6, kGnMaxRot = 0.35, kGnMaxTrans = 5.0;
__device__ __forceinline__ bool gn_safe_step(const double* s21, const double* rhs, double d[6]) {
    const double maxd = fmax(fmax(fmax(s21[0], s21[6]), fmax(s21[11], s21[15])), fmax(s21[18], s21[20]));
    if (!(maxd > 0.0) || !isfinite(maxd)) return false;
    bool ok = solve6_ldlt(s21, rhs, d, 0.0, kGnPivotRel * maxd);
    if (!ok) ok = solve6_ldlt_damped(s21, rhs, d, kGnDampRel * maxd);      // cold path, not inlined
    if (!ok) return false;
    // (this runs on ONE thread at the tail of every GN pass: the common case must stay two multiply-add chains and two compares)
    const double rot2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2], tr2 = d[3] * d[3] + d[4] * d[4] + d[5] * d[5];
    if (rot2 > kGnMaxRot * kGnMaxRot || tr2 > kGnMaxTrans * kGnMaxTrans) {
        const double rot = sqrt(rot2), tr = sqrt(tr2);
        double sc = 1.0;
        if (rot > kGnMaxRot) sc = kGnMaxRot / rot;
        if (tr * sc > kGnMaxTrans) sc = kGnMaxTrans / tr;
#pragma unroll
        for (int k = 0; k < 6; ++k) d[k] *= sc;
    }
    return true;
}

// ceres::QuaternionParameterization::Plus on q, identity on t.
__device__ inline void pose_plus(const double x[7], const double d[6], double out[7]) {
    double nd = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    if (nd > 0.0) {
        double sbd, cs;
        if (nd < 0.25) {
            // GN steps are small: Taylor series of sin(x)/x and cos(x) to x^16 (truncation < 1e-22 at x = 0.25),
            // a short FMA chain instead of the generic argument-reduction path on the single-thread tail
            const double x2 = nd * nd;
            sbd = 1.0 + x2 * (-1.0 / 6 + x2 * (1.0 / 120 + x2 * (-1.0 / 5040 + x2 * (1.0 / 362880 + x2 * (-1.0 / 39916800 +
                  x2 * (1.0 / 6227020800.0 + x2 * (-1.0 / 1307674368000.0)))))));
            cs = 1.0 + x2 * (-0.5 + x2 * (1.0 / 24 + x2 * (-1.0 / 720 + x2 * (1.0 / 40320 + x2 * (-1.0 / 3628800 +
                 x2 * (1.0 / 479001600 + x2 * (-1.0 / 87178291200.0 + x2 * (1.0 / 20922789888000.0))))))));
        } else {
            double sn;
            sincos(nd, &sn, &cs);
            sbd = sn / nd;
        }
        double dw = cs, dx = sbd * d[0], dy = sbd * d[1], dz = sbd * d[2];
        out[0] = dw * x[0] - dx * x[1] - dy * x[2] - dz * x[3];
        out[1] = dw * x[1] + dx * x[0] + dy * x[3] - dz * x[2];
        out[2] = dw * x[2] + dy * x[0] + dz * x[1] - dx * x[3];
        out[3] = dw * x[3] + dz * x[0] + dx * x[2] - dy * x[1];
    } else {
        out[0] = x[0]; out[1] = x[1]; out[2] = x[2]; out[3] = x[3];
    }
    out[4] = x[4] + d[3]; out[5] = x[5] + d[4]; out[6] = x[6] + d[5];
}

// ---- correspondence arithmetic of the GN pass, the LM solve (grid_knn.cu) and the backend kernels (backend_corr.cu) ----

// The gates of a fitted plane  nv . p + 1 = 0  of the five neighbours m (L/src/LidarOdometry.cpp:376-405, R/src/BackendFusion.cpp:
// 1486-1504) in the reference's mixed fp32/fp64 widths: normalise nv, every neighbour within plane_thres, then the fp32 weight of the
// transformed query (sx, sy, sz) above w_gate.  `refuse` rejects the plane after the distance test (the backend's reflectivity gate).
// On acceptance pl = weight * [n, 1/|nv|] and `weight` are set; otherwise neither is touched.
__device__ __forceinline__ bool plane_gate(double nv[3], const float4 m[5], float sx, float sy, float sz, double plane_thres,
                                           double w_gate, bool refuse, float4& pl, float& weight) {
    const double n2 = nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2];
    const double nn = sqrt(n2);
    const double normInverse = 1.0 / nn;                                                                      // :376
    if (n2 > 0) { nv[0] /= nn; nv[1] /= nn; nv[2] /= nn; }                                                    // :377
    bool planeValid = true;
#pragma unroll
    for (int j = 0; j < 5; ++j)                                                                                // :386-393
        if (fabs(nv[0] * m[j].x + nv[1] * m[j].y + nv[2] * m[j].z + normInverse) > plane_thres) planeValid = false;
    if (refuse) planeValid = false;
    bool ok = false;
    if (planeValid) {
        // :397-398; exact ops keep the fp32 roundings stable
        const float pd = (float)addx(addx(addx(mulx(nv[0], (double)sx), mulx(nv[1], (double)sy)), mulx(nv[2], (double)sz)), normInverse);
        const float rng = __fsqrt_rn(__fsqrt_rn(faddx(faddx(fmulx(sx, sx), fmulx(sy, sy)), fmulx(sz, sz))));
        const float w = (float)subx(1.0, mulx(0.9, (double)fabsf(pd)) / (double)rng);
        if ((double)w > w_gate) {                                                                              // :400
            pl = make_float4((float)mulx((double)w, nv[0]), (float)mulx((double)w, nv[1]),                     // :402-405
                             (float)mulx((double)w, nv[2]), (float)mulx((double)w, normInverse));
            weight = w;
            ok = true;
        }
    }
    return ok;
}

struct Row { double J[6]; double r; double half_rho; };     // Jacobian row, residual and (after a corrector) rho / 2

// LidarPlaneNormIncreFactor (LidarKeyframeFactor.h:118-128) in closed form, before the loss:
//   r = n~ . (R p + t) + d~ ;  J = [ 2 (R p x n~)^T , n~^T ]   (tangent order [rot, t]; SURVEY.md Appendix A)
__device__ __forceinline__ Row plane_row(const Q4& q, const D3& t, float x, float y, float z, const float4& pl) {
    const D3 rp = qrot_x(q, D3{(double)x, (double)y, (double)z});
    const double nx = pl.x, ny = pl.y, nz = pl.z;
    Row R;
    R.r = nx * (rp.x + t.x) + ny * (rp.y + t.y) + nz * (rp.z + t.z) + (double)pl.w;
    R.J[0] = 2.0 * (rp.y * nz - rp.z * ny);
    R.J[1] = 2.0 * (rp.z * nx - rp.x * nz);
    R.J[2] = 2.0 * (rp.x * ny - rp.y * nx);
    R.J[3] = nx; R.J[4] = ny; R.J[5] = nz;
    return R;
}

// ceres::HuberLoss(a) and ceres::CauchyLoss(b) with Ceres' Corrector on a raw row: J and r scaled by sqrt(rho'), rho / 2 kept.
// Both have rho'' <= 0, the branch in which the Corrector is that scaling alone.  The Cauchy form takes the caller's loop
// invariants b2 = b^2 and inv_b2 = 1 / b^2.
__device__ __forceinline__ void huber_correct(Row& R, double a) {
    const double s2 = R.r * R.r, b2 = a * a;
    double rho0 = s2, rho1 = 1.0;
    if (s2 > b2) { const double rt = sqrt(s2); rho0 = 2.0 * a * rt - b2; rho1 = fmax(DBL_MIN, a / rt); }
    const double sr = sqrt(rho1);
#pragma unroll
    for (int k = 0; k < 6; ++k) R.J[k] *= sr;
    R.r *= sr;
    R.half_rho = 0.5 * rho0;
}
__device__ __forceinline__ void cauchy_correct(Row& R, double b2, double inv_b2) {
    const double sum = 1.0 + R.r * R.r * inv_b2;
    const double rho0 = b2 * log(sum);
    const double sr = sqrt(fmax(DBL_MIN, 1.0 / sum));
#pragma unroll
    for (int k = 0; k < 6; ++k) R.J[k] *= sr;
    R.r *= sr;
    R.half_rho = 0.5 * rho0;
}

// Fold one corrected row into the 29 sums.  This order defines the layout every consumer of the sums reads.
__device__ __forceinline__ void add_row29(double acc[29], const Row& R) {
    int k = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = i; j < 6; ++j) acc[k++] += R.J[i] * R.J[j];
#pragma unroll
    for (int i = 0; i < 6; ++i) acc[21 + i] += R.J[i] * R.r;
    acc[27] += R.half_rho;
    acc[28] += 1.0;
}

#ifdef __CUDACC__
// Block sum of every thread's acc[29] in a fixed order: an xor tree inside each warp, then the nwarps warp sums in warp order
// through red[nwarps][29] in shared memory.  Thread k < 29 gets the total of scalar k; every thread must call it.
__device__ __forceinline__ double block_sum29(const double acc[29], double (*red)[29], int nwarps) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 29; ++k) {
        double v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) red[warp][k] = v;
    }
    __syncthreads();
    double v = 0;
    if (threadIdx.x < 29)
        for (int w = 0; w < nwarps; ++w) v += red[w][threadIdx.x];
    return v;
}
#endif

}  // namespace lili
