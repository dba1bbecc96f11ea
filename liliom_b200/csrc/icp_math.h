// The arithmetic of PCL's IterativeClosestPoint loop (icp.cu; from-knowledge, PCL 1.8-1.10 registration/impl/icp.hpp,
// transformation_estimation_svd.hpp, default_convergence_criteria.hpp), shared by host and device: the 3x3 SVD, the Umeyama
// step from the 17 correspondence sums, the composition final = incremental * final and the convergence test.
// Every fp64 operation is spelled with round-to-nearest intrinsics on the device and as a plain operator on the host, as in
// pcl_xform.h: icp.cu is compiled with FMA contraction (its transform of the source points must keep its bits), so a plain
// expression there could be contracted, while the intrinsics never are.  The kernel, the host build in tests/icp_math_host.cpp
// (-ffp-contract=off) and the earlier host loop of icp.cu give the same bits.
#pragma once
#include <cfloat>
#include "pcl_xform.h"

namespace lili {

constexpr int kIcpSums = 17;      // sum p (3), sum q (3), sum p q^T (9, row = p, col = q), sum d2, count

#ifdef __CUDA_ARCH__
VGB_HD double divx(double a, double b) { return __ddiv_rn(a, b); }
VGB_HD double sqrtx(double a) { return __dsqrt_rn(a); }
#else
VGB_HD double divx(double a, double b) { return a / b; }
VGB_HD double sqrtx(double a) { return std::sqrt(a); }
#endif

// 3x3 SVD by one-sided Jacobi (Hestenes), A = U diag(s) V^T; singular values unsorted, U completed to an orthonormal basis
VGB_HD void svd3(const double A[3][3], double U[3][3], double s[3], double V[3][3]) {
    double B[3][3];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { B[i][j] = A[i][j]; V[i][j] = i == j ? 1.0 : 0.0; }
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                double alpha = 0, beta = 0, gamma = 0;
                for (int i = 0; i < 3; ++i) {
                    alpha = addx(alpha, mulx(B[i][p], B[i][p]));
                    beta = addx(beta, mulx(B[i][q], B[i][q]));
                    gamma = addx(gamma, mulx(B[i][p], B[i][q]));
                }
                off = fmax(off, divx(fabs(gamma), sqrtx(addx(mulx(alpha, beta), 1e-300))));
                if (fabs(gamma) < 1e-300) continue;
                const double zeta = divx(subx(beta, alpha), mulx(2.0, gamma));
                const double t = divx(zeta >= 0 ? 1.0 : -1.0, addx(fabs(zeta), sqrtx(addx(1.0, mulx(zeta, zeta)))));
                const double c = divx(1.0, sqrtx(addx(1.0, mulx(t, t)))), sn = mulx(c, t);
                for (int i = 0; i < 3; ++i) {
                    const double bp = B[i][p], bq = B[i][q];
                    B[i][p] = subx(mulx(c, bp), mulx(sn, bq)); B[i][q] = addx(mulx(sn, bp), mulx(c, bq));
                    const double vp = V[i][p], vq = V[i][q];
                    V[i][p] = subx(mulx(c, vp), mulx(sn, vq)); V[i][q] = addx(mulx(sn, vp), mulx(c, vq));
                }
            }
        if (off < 1e-15) break;
    }
    for (int j = 0; j < 3; ++j) {
        s[j] = sqrtx(addx(addx(mulx(B[0][j], B[0][j]), mulx(B[1][j], B[1][j])), mulx(B[2][j], B[2][j])));
        for (int i = 0; i < 3; ++i) U[i][j] = s[j] > 1e-300 ? divx(B[i][j], s[j]) : 0.0;
    }
    // a zero singular value leaves a zero column in U: complete it to an orthonormal basis (cross product of the other two)
    for (int j = 0; j < 3; ++j) {
        if (s[j] > 1e-300) continue;
        const int a = (j + 1) % 3, b = (j + 2) % 3;
        U[0][j] = subx(mulx(U[1][a], U[2][b]), mulx(U[2][a], U[1][b]));
        U[1][j] = subx(mulx(U[2][a], U[0][b]), mulx(U[0][a], U[2][b]));
        U[2][j] = subx(mulx(U[0][a], U[1][b]), mulx(U[1][a], U[0][b]));
    }
}

VGB_HD double det3(const double M[3][3]) {
    return addx(subx(mulx(M[0][0], subx(mulx(M[1][1], M[2][2]), mulx(M[1][2], M[2][1]))),
                     mulx(M[0][1], subx(mulx(M[1][0], M[2][2]), mulx(M[1][2], M[2][0])))),
                mulx(M[0][2], subx(mulx(M[1][0], M[2][1]), mulx(M[1][1], M[2][0]))));
}

// Umeyama without scale on the matched pairs (p = transformed source, q = target) from their 17 sums (count s[16] >= 3):
// R = U S V^T of sigma = 1/n sum (q - mq)(p - mp)^T, S = diag(1,1,sign det), t = mq - R mp
VGB_HD void icp_umeyama(const double s[kIcpSums], double R[3][3], double t[3]) {
    const double cnt = s[16];
    const double mp[3] = {divx(s[0], cnt), divx(s[1], cnt), divx(s[2], cnt)}, mq[3] = {divx(s[3], cnt), divx(s[4], cnt), divx(s[5], cnt)};
    double Sg[3][3];                                              // dst x src^T
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Sg[i][j] = subx(divx(s[6 + 3 * j + i], cnt), mulx(mq[i], mp[j]));
    double U[3][3], sv[3], V[3][3];
    svd3(Sg, U, sv, V);
    const double sgn = mulx(det3(U), det3(V)) < 0 ? -1.0 : 1.0;
    // the reflection fix belongs to the SMALLEST singular value (Eigen sorts them descending and flips the last)
    int jmin = 0;
    for (int j = 1; j < 3; ++j) if (sv[j] < sv[jmin]) jmin = j;
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
        double acc = 0.0;
        for (int k = 0; k < 3; ++k) acc = addx(acc, mulx(mulx(U[i][k], k == jmin ? sgn : 1.0), V[j][k]));
        R[i][j] = acc;
    }
    for (int i = 0; i < 3; ++i) t[i] = subx(mq[i], addx(addx(mulx(R[i][0], mp[0]), mulx(R[i][1], mp[1])), mulx(R[i][2], mp[2])));
}

// final = incremental * final (row 3 of both stays 0 0 0 1)
VGB_HD void icp_compose(const double R[3][3], const double t[3], double F[4][4]) {
    double N[3][4];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 4; ++j)
            N[i][j] = addx(addx(addx(mulx(R[i][0], F[0][j]), mulx(R[i][1], F[1][j])), mulx(R[i][2], F[2][j])), j == 3 ? t[i] : 0.0);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 4; ++j) F[i][j] = N[i][j];
    F[3][0] = F[3][1] = F[3][2] = 0.0; F[3][3] = 1.0;
}

// DefaultConvergenceCriteria::hasConverged with max_iterations_similar_transforms_ = 0, after iteration `it` (1-based)
VGB_HD bool icp_converged(int it, int max_iter, const double R[3][3], const double t[3], double mse, double prev_mse, double trans_eps,
                          double fit_eps) {
    if (it >= max_iter) return true;
    const double cos_angle = mulx(0.5, subx(addx(addx(R[0][0], R[1][1]), R[2][2]), 1.0));
    const double tr2 = addx(addx(mulx(t[0], t[0]), mulx(t[1], t[1])), mulx(t[2], t[2]));
    if (cos_angle >= subx(1.0, trans_eps) && tr2 <= trans_eps) return true;
    if (divx(fabs(subx(mse, prev_mse)), prev_mse) < fit_eps) return true;
    if (fabs(subx(mse, prev_mse)) < 1e-12) return true;
    return false;
}

// The state of one alignment and one step of it from the sums of a correspondence pass at the current F.
struct IcpState {
    double F[4][4];
    double prev_mse;
    int it;
};
enum { kIcpGo = 0, kIcpConverged = 1, kIcpStuck = 2 };      // stuck: fewer than 3 correspondences (icp.hpp: not converged)

VGB_HD void icp_init(IcpState& st) {
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) st.F[i][j] = i == j ? 1.0 : 0.0;
    st.prev_mse = DBL_MAX;
    st.it = 0;
}

VGB_HD int icp_step(IcpState& st, const double s[kIcpSums], int max_iter, double trans_eps, double fit_eps) {
    const double cnt = s[16];
    if (cnt < 3.0) return kIcpStuck;
    double R[3][3], t[3];
    icp_umeyama(s, R, t);
    icp_compose(R, t, st.F);
    ++st.it;
    const double mse = divx(s[15], cnt);
    if (icp_converged(st.it, max_iter, R, t, mse, st.prev_mse, trans_eps, fit_eps)) return kIcpConverged;
    st.prev_mse = mse;
    return kIcpGo;
}

// getFitnessScore(): mean squared NN distance of the aligned source (sums of the pass without a cut-off)
VGB_HD double icp_fitness(const double s[kIcpSums]) { return s[16] > 0 ? divx(s[15], s[16]) : DBL_MAX; }

}  // namespace lili
