// TEST INFRASTRUCTURE: host build of liliom_b200/csrc/icp_math.h (the 3x3 SVD, the Umeyama step from the 17 sums, the
// composition and PCL's convergence test), so that the CPU test tier checks the SAME SOURCE k_icp_persistent runs, and the
// whole ICP loop composed from it with a brute-force 1-NN that ranks candidates as the kernel does (squared fp32 distance,
// then the target index).
#include "../liliom_b200/csrc/icp_math.h"
#include <cstdint>
#include <cstring>

using namespace lili;

extern "C" void im_svd3(const double* a9, double* u9, double* s3, double* v9) {
    double A[3][3], U[3][3], V[3][3];
    memcpy(A, a9, sizeof(A));
    svd3(A, U, s3, V);
    memcpy(u9, U, sizeof(U));
    memcpy(v9, V, sizeof(V));
}

extern "C" double im_det3(const double* m9) {
    double M[3][3];
    memcpy(M, m9, sizeof(M));
    return det3(M);
}

extern "C" void im_umeyama(const double* s17, double* r9, double* t3) {
    double R[3][3];
    icp_umeyama(s17, R, t3);
    memcpy(r9, R, sizeof(R));
}

extern "C" int im_converged(int it, int max_iter, const double* r9, const double* t3, double mse, double prev_mse, double trans_eps,
                            double fit_eps) {
    double R[3][3];
    memcpy(R, r9, sizeof(R));
    return icp_converged(it, max_iter, R, t3, mse, prev_mse, trans_eps, fit_eps) ? 1 : 0;
}

// one step from the sums on state (F16, prev_mse, it): returns kIcpGo / kIcpConverged / kIcpStuck and the updated state
extern "C" int im_step(double* f16, double* prev_mse, int* it, const double* s17, int max_iter, double trans_eps, double fit_eps) {
    IcpState st;
    memcpy(st.F, f16, sizeof(st.F));
    st.prev_mse = *prev_mse;
    st.it = *it;
    const int v = icp_step(st, s17, max_iter, trans_eps, fit_eps);
    memcpy(f16, st.F, sizeof(st.F));
    *prev_mse = st.prev_mse;
    *it = st.it;
    return v;
}

// the 17 sums of one pass: src (n x 4 floats) under F, nearest target point (m x 4 floats) kept when d2 <= max_d2 (max_d2 < 0: all)
static void pass(const float* src, int n, const float* tgt, int m, const double F[4][4], float max_d2, double s[kIcpSums]) {
    for (int k = 0; k < kIcpSums; ++k) s[k] = 0.0;
    for (int i = 0; i < n; ++i) {
        const float* p = src + 4 * i;
        const double px = F[0][0] * p[0] + F[0][1] * p[1] + F[0][2] * p[2] + F[0][3];
        const double py = F[1][0] * p[0] + F[1][1] * p[1] + F[1][2] * p[2] + F[1][3];
        const double pz = F[2][0] * p[0] + F[2][1] * p[1] + F[2][2] * p[2] + F[2][3];
        const float sx = (float)px, sy = (float)py, sz = (float)pz;
        uint64_t best = ~0ull;
        for (int j = 0; j < m; ++j) {
            const float dx = sx - tgt[4 * j], dy = sy - tgt[4 * j + 1], dz = sz - tgt[4 * j + 2];
            const float d = dx * dx + dy * dy + dz * dz;
            uint32_t bits;
            memcpy(&bits, &d, 4);
            const uint64_t key = ((uint64_t)bits << 32) | (uint32_t)j;
            if (key < best) best = key;
        }
        if (best == ~0ull) continue;
        float d;
        const uint32_t bits = (uint32_t)(best >> 32);
        memcpy(&d, &bits, 4);
        if (max_d2 >= 0.f && !(d <= max_d2)) continue;
        const float* q = tgt + 4 * (uint32_t)best;
        const double v[kIcpSums] = {px, py, pz, q[0], q[1], q[2], px * q[0], px * q[1], px * q[2], py * q[0], py * q[1], py * q[2],
                                    pz * q[0], pz * q[1], pz * q[2], (double)d, 1.0};
        for (int k = 0; k < kIcpSums; ++k) s[k] += v[k];
    }
}

// the whole loop (k_icp_persistent's sequence): passes and steps until a verdict, then the fitness pass
extern "C" void im_icp(const float* src, int n, const float* tgt, int m, double max_corr_dist, int max_iter, double trans_eps, double fit_eps,
                       double* t16, double* fitness, int* converged, int* iters) {
    IcpState st;
    icp_init(st);
    double s[kIcpSums];
    int verdict = kIcpStuck;
    *fitness = 0.0;
    if (n > 0 && m > 0) {
        const float max_d2 = (float)(max_corr_dist * max_corr_dist);
        do {
            pass(src, n, tgt, m, st.F, max_d2, s);
            verdict = icp_step(st, s, max_iter, trans_eps, fit_eps);
        } while (verdict == kIcpGo);
        pass(src, n, tgt, m, st.F, -1.0f, s);
        *fitness = icp_fitness(s);
    }
    memcpy(t16, st.F, sizeof(st.F));
    *converged = verdict == kIcpConverged ? 1 : 0;
    *iters = st.it;
}
