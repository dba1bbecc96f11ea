// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.h).  Pinned to the reference's own code: DESIGN.md §6.
// Scan-to-map step of LidarOdometry restated: LiLi-OM/src/LidarOdometry.cpp:221-244
// (transformPoint), :352-413 (findCorrespondingSurfFeatures), :483-561
// (updateTransformationWithCeres), LiLi-OM/include/factors/LidarKeyframeFactor.h:111-139
// (LidarPlaneNormIncreFactor).  Ceres 2.0 (README.md:36-41) is absent: its trust-region
// Levenberg-Marquardt loop, Huber corrector, QuaternionParameterization and DENSE_QR are
// restated from knowledge ("from-knowledge" marks).
#include "oracle_api.h"
#include "oracle_math.h"
#include <vector>
#include <cstring>
#include <limits>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace orc { void knn5_one(const void* tree, const float q[3], int idx[5], float sqd[5]); }
using namespace orc;

// LidarOdometry.cpp:221-244 — p_w = q * p + t in fp64, narrowed to fp32 on store.
static inline void transform_point(const double pose7[7], const float p[3], float out[3]) {
    Quat q{pose7[0], pose7[1], pose7[2], pose7[3]};
    V3 o = qrot(q, V3{p[0], p[1], p[2]}) + V3{pose7[4], pose7[5], pose7[6]};
    out[0] = (float)o.x; out[1] = (float)o.y; out[2] = (float)o.z;
}

// LidarOdometry.cpp:369-405 on the five neighbours mp[j].  Returns 1 when a correspondence is
// emitted and fills plane[4] = {w*nx, w*ny, w*nz, w*d}; nv_out (optional) gets the QR's
// un-normalised normal.
static inline int fit_gate_one(const float* const mp[5], const float sel[3], double plane_thres, double w_gate, float plane[4],
                               float* weight_out, double* nv_out) {
    double A[15], B[5];
    for (int j = 0; j < 5; ++j) {
        A[3 * j + 0] = mp[j][0]; A[3 * j + 1] = mp[j][1]; A[3 * j + 2] = mp[j][2];   // :369-371
        B[j] = -1.0;                                                  // :363
    }
    double nv[3];
    colpiv_qr_solve_nx3(5, A, B, nv);                                 // :375
    if (nv_out) for (int k = 0; k < 3; ++k) nv_out[k] = nv[k];
    double nn = std::sqrt(nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2]);
    double normInverse = 1 / nn;                                      // :376
    double n2 = nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2];
    if (n2 > 0) { double s = std::sqrt(n2); nv[0] /= s; nv[1] /= s; nv[2] /= s; }   // :377 normalize()
    for (int j = 0; j < 5; ++j) {                                     // :386-393
        if (std::fabs(nv[0] * mp[j][0] + nv[1] * mp[j][1] + nv[2] * mp[j][2] + normInverse) > plane_thres) return 0;
    }
    // :397-398 — mixed widths exactly as written (fabs/sqrt resolve to the float overloads)
    float pd = nv[0] * sel[0] + nv[1] * sel[1] + nv[2] * sel[2] + normInverse;
    float weight = 1 - 0.9 * std::fabs(pd) / std::sqrt(std::sqrt(sel[0] * sel[0] + sel[1] * sel[1] + sel[2] * sel[2]));
    if (!(weight > w_gate)) return 0;                                 // :400
    plane[0] = weight * nv[0];                                        // :402-405
    plane[1] = weight * nv[1];
    plane[2] = weight * nv[2];
    plane[3] = weight * normInverse;
    if (weight_out) *weight_out = weight;
    return 1;
}

// LidarOdometry.cpp:362-410 for one feature, given its 5-NN.
static inline int surf_corr_one(const float* map_xyzw, const float sel[3], const int idx[5], const float sqd[5],
                                double max_sqd, double plane_thres, double w_gate, float plane[4], float* weight_out) {
    if (!((double)sqd[4] < max_sqd)) return 0;                       // :365
    const float* mp[5];
    for (int j = 0; j < 5; ++j) mp[j] = map_xyzw + 4 * (size_t)idx[j];
    return fit_gate_one(mp, sel, plane_thres, w_gate, plane, weight_out, nullptr);
}

// :369-405 for n neighbourhoods m20 (n x 5 x 4 floats) and transformed queries s3 (n x 3), at the thresholds plane_thres[i], w_gate[i]:
// ok[i], plane (zero when refused), weight and the QR's un-normalised normal nv3 (n x 3).
extern "C" void orc_fit_gate_batch(const float* m20, const float* s3, int n, const double* plane_thres, const double* w_gate, unsigned char* ok,
                                   float* plane4, float* weight, double* nv3) {
    for (int i = 0; i < n; ++i) {
        const float* mp[5];
        for (int j = 0; j < 5; ++j) mp[j] = m20 + 20 * (size_t)i + 4 * j;
        float pl[4] = {0, 0, 0, 0};
        float w = 0.0f;
        ok[i] = (unsigned char)fit_gate_one(mp, s3 + 3 * (size_t)i, plane_thres[i], w_gate[i], pl, &w, nv3 + 3 * (size_t)i);
        for (int k = 0; k < 4; ++k) plane4[4 * (size_t)i + k] = pl[k];
        weight[i] = w;
    }
}

extern "C" int orc_find_surf_corr(const void* tree, const float* map_xyzw, int m, const float* feats_xyzw, int n,
                                  const double pose7[7], unsigned char* corr_valid, float* corr_plane,
                                  int* nn_idx, float* pw, int nthreads) {
    (void)m;
    int cnt = 0;
#pragma omp parallel for schedule(dynamic, 128) reduction(+ : cnt) num_threads(nthreads > 0 ? nthreads : 1)
    for (int i = 0; i < n; ++i) {
        float sel[3];
        transform_point(pose7, feats_xyzw + 4 * (size_t)i, sel);
        int idx[5]; float sqd[5];
        knn5_one(tree, sel, idx, sqd);
        float plane[4] = {0, 0, 0, 0};
        int ok = (idx[4] >= 0) ? surf_corr_one(map_xyzw, sel, idx, sqd, 1.0, 0.06, 0.4, plane, nullptr) : 0;
        corr_valid[i] = (unsigned char)ok;
        for (int k = 0; k < 4; ++k) corr_plane[4 * (size_t)i + k] = plane[k];
        if (nn_idx) for (int k = 0; k < 5; ++k) nn_idx[5 * (size_t)i + k] = idx[k];
        if (pw) { pw[4 * (size_t)i] = sel[0]; pw[4 * (size_t)i + 1] = sel[1]; pw[4 * (size_t)i + 2] = sel[2]; pw[4 * (size_t)i + 3] = 1.0f; }
        cnt += ok;
    }
    return cnt;
}

// ---------------------------------------------------------------------------------------
// One residual of LidarPlaneNormIncreFactor (LidarKeyframeFactor.h:118-128) and the row
// Ceres would assemble for it: autodiff <1,4,3> wrt (q, t), the q block chained with
// from-knowledge ceres::QuaternionParameterization::ComputeJacobian (4x3), the row then
// scaled by the from-knowledge Huber corrector (sqrt(rho'), rho'' <= 0 branch;
// cf. the in-repo copy LiLi-OM/src/MarginalizationFactor.cpp:44-70).
// J[0..2] = rotation tangent, J[3..5] = translation.  Returns rho(s) (cost = rho/2).
// ---------------------------------------------------------------------------------------
static inline double plane_row(const double x[7], const float p[4], const float pl[4], double a, double J[6], double& r_out) {
    const double w = x[0];
    V3 qv{x[1], x[2], x[3]};
    V3 v{p[0], p[1], p[2]};
    V3 nrm{pl[0], pl[1], pl[2]};
    double nd = pl[3];
    // Eigen q * v
    V3 uv = cross(qv, v); uv = uv + uv;
    V3 pwv = v + w * uv + cross(qv, uv) + V3{x[4], x[5], x[6]};
    double r = dot(nrm, pwv) + nd;
    // d(point_w)/dq, exactly differentiating the expression above
    double jq[4];
    jq[0] = dot(nrm, uv);
    const V3 e[3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int k = 0; k < 3; ++k) {
        V3 duv = 2.0 * cross(e[k], v);
        V3 df = w * duv + cross(e[k], uv) + cross(qv, duv);
        jq[k + 1] = dot(nrm, df);
    }
    // QuaternionParameterization::ComputeJacobian (row-major 4x3), x = (w,x,y,z)
    const double P[4][3] = {{-x[1], -x[2], -x[3]}, {x[0], x[3], -x[2]}, {-x[3], x[0], x[1]}, {x[2], -x[1], x[0]}};
    for (int c = 0; c < 3; ++c) J[c] = jq[0] * P[0][c] + jq[1] * P[1][c] + jq[2] * P[2][c] + jq[3] * P[3][c];
    J[3] = nrm.x; J[4] = nrm.y; J[5] = nrm.z;
    // HuberLoss(a)::Evaluate + Corrector
    double s = r * r, rho0, rho1;
    const double b = a * a;
    if (s > b) {
        double rt = std::sqrt(s);
        rho0 = 2.0 * a * rt - b;
        rho1 = std::max(std::numeric_limits<double>::min(), a / rt);
    } else {
        rho0 = s; rho1 = 1.0;
    }
    double sr = std::sqrt(rho1);
    for (int c = 0; c < 6; ++c) J[c] *= sr;
    r_out = sr * r;
    return rho0;
}

static void accumulate(const float* feats, int n, const unsigned char* valid, const float* plane, const double x[7],
                       double a, double out29[29]) {
    for (int k = 0; k < 29; ++k) out29[k] = 0;
    for (int i = 0; i < n; ++i) {
        if (!valid[i]) continue;
        double J[6], r;
        double rho = plane_row(x, feats + 4 * (size_t)i, plane + 4 * (size_t)i, a, J, r);
        int k = 0;
        for (int aidx = 0; aidx < 6; ++aidx)
            for (int bidx = aidx; bidx < 6; ++bidx) out29[k++] += J[aidx] * J[bidx];
        for (int aidx = 0; aidx < 6; ++aidx) out29[21 + aidx] += J[aidx] * r;
        out29[27] += 0.5 * rho;
        out29[28] += 1.0;
    }
}

extern "C" void orc_normal_equations(const float* feats_xyzw, int n, const unsigned char* corr_valid,
                                     const float* corr_plane, const double pose7[7], double huber_a, double out29[29]) {
    accumulate(feats_xyzw, n, corr_valid, corr_plane, pose7, huber_a, out29);
}

// from-knowledge: ceres::QuaternionParameterization::Plus + identity Plus on t.
static inline void pose_plus(const double x[7], const double d[6], double out[7]) {
    double nd = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    if (nd > 0.0) {
        double sbd = std::sin(nd) / nd;
        Quat dq{std::cos(nd), sbd * d[0], sbd * d[1], sbd * d[2]};
        Quat r = qmul(dq, Quat{x[0], x[1], x[2], x[3]});
        out[0] = r.w; out[1] = r.x; out[2] = r.y; out[3] = r.z;
    } else {
        for (int k = 0; k < 4; ++k) out[k] = x[k];
    }
    for (int k = 0; k < 3; ++k) out[4 + k] = x[4 + k] + d[3 + k];
}

// LidarOdometry.cpp:539-549 + math_tools.h:165-173
static inline void unify(double x[7]) {
    if (x[0] < 0) { x[0] = -x[0]; x[1] = -x[1]; x[2] = -x[2]; x[3] = -x[3]; }
}

static void unpack_sym(const double s[27], double H[6][6], double g[6]) {
    int k = 0;
    for (int a = 0; a < 6; ++a) for (int b = a; b < 6; ++b) { H[a][b] = H[b][a] = s[k++]; }
    for (int a = 0; a < 6; ++a) g[a] = s[21 + a];
}

// dense symmetric positive (semi)definite 6x6 solve by LDL^T with a tiny-pivot guard; lambda is added to the diagonal,
// piv_min >= 0 additionally rejects pivots that are not above it
static bool solve6(const double Hin[6][6], const double bin[6], double x[6], double lambda = 0.0, double piv_min = -1.0) {
    double L[6][6] = {{0}}, D[6];
    for (int j = 0; j < 6; ++j) {
        double d = Hin[j][j] + lambda;
        for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k] * D[k];
        if (!(std::fabs(d) > 1e-300) || !std::isfinite(d) || (piv_min >= 0.0 && !(d > piv_min))) return false;
        D[j] = d;
        L[j][j] = 1;
        for (int i = j + 1; i < 6; ++i) {
            double s = Hin[i][j];
            for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k] * D[k];
            L[i][j] = s / d;
        }
    }
    double y[6];
    for (int i = 0; i < 6; ++i) { double s = bin[i]; for (int k = 0; k < i; ++k) s -= L[i][k] * y[k]; y[i] = s; }
    for (int i = 0; i < 6; ++i) y[i] /= D[i];
    for (int i = 5; i >= 0; --i) { double s = y[i]; for (int k = i + 1; k < 6; ++k) s -= L[k][i] * x[k]; x[i] = s; }
    for (int i = 0; i < 6; ++i) if (!std::isfinite(x[i])) return false;
    return true;
}

// The GN mode's step (NOT the reference's solver, which is Ceres LM = orc_scan_to_map_ceres): plain LDL^T solution of
// H d = -g, with (1) a Levenberg-damped re-solve when a pivot is below 1e-10 * max diag(H) (unconstrained direction) and
// (2) a trust region of 0.35 rad / 5 m on the step.  Same constants as dev_math.cuh::gn_safe_step.
static bool gn_safe_step(const double H[6][6], const double nb[6], double d[6]) {
    double maxd = 0;
    for (int k = 0; k < 6; ++k) maxd = std::fmax(maxd, H[k][k]);
    if (!(maxd > 0.0) || !std::isfinite(maxd)) return false;
    if (!solve6(H, nb, d, 0.0, 1e-10 * maxd) && !solve6(H, nb, d, 1e-6 * maxd, 0.0)) return false;
    const double rot = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), tr = std::sqrt(d[3] * d[3] + d[4] * d[4] + d[5] * d[5]);
    double sc = 1.0;
    if (rot > 0.35) sc = 0.35 / rot;
    if (tr * sc > 5.0) sc = 5.0 / tr;
    if (sc < 1.0) for (int k = 0; k < 6; ++k) d[k] *= sc;
    return true;
}

extern "C" int orc_scan_to_map_gn(const void* tree, const float* map_xyzw, int m, const float* feats_xyzw, int n,
                                  double pose7[7], int iters, orc_iter_stats* stats, int nthreads) {
    if (m < 10) return -1;   // LidarOdometry.cpp:485-488
    std::vector<unsigned char> valid(n);
    std::vector<float> plane(4 * (size_t)n);
    double x[7];
    std::memcpy(x, pose7, sizeof(x));
    for (int it = 0; it < iters; ++it) {
        int nc = orc_find_surf_corr(tree, map_xyzw, m, feats_xyzw, n, x, valid.data(), plane.data(), nullptr, nullptr, nthreads);
        double s29[29];
        accumulate(feats_xyzw, n, valid.data(), plane.data(), x, 0.1, s29);
        double H[6][6], g[6], d[6], nb[6];
        unpack_sym(s29, H, g);
        for (int k = 0; k < 6; ++k) nb[k] = -g[k];
        double xn[7];
        if (nc > 0 && gn_safe_step(H, nb, d)) pose_plus(x, d, xn); else std::memcpy(xn, x, sizeof(xn));
        unify(xn);
        if (stats) {
            stats[it].n_corr = nc; stats[it].lm_iters = 1; stats[it].cost = s29[27];
            std::memcpy(stats[it].jtj_jtr, s29, 27 * sizeof(double));
            std::memcpy(stats[it].pose7, xn, sizeof(xn));
        }
        std::memcpy(x, xn, sizeof(x));
    }
    std::memcpy(pose7, x, sizeof(x));
    return 0;
}

// ---------------------------------------------------------------------------------------
// from-knowledge: ceres::Solve with Solver::Options defaults of Ceres 2.0 except the four
// set at LidarOdometry.cpp:528-534 (DENSE_QR, max_num_iterations, max_solver_time 15 ms —
// DISABLED here, it makes the reference non-deterministic — no progress output).
// TrustRegionMinimizer + LevenbergMarquardtStrategy:
//   jacobi scaling 1/(1+||col||) fixed at iteration 0; D = sqrt(clamp(diag(J^T J),1e-6,1e32)/radius);
//   radius0 = 1e4, max 1e16, min 1e-32; min_relative_decrease 1e-3; function_tolerance 1e-6;
//   parameter_tolerance 1e-8; gradient_tolerance 1e-10; monotonic steps.
//   The start counts as a successful step (TrustRegionMinimizer::IterationZero), so the gradient test runs before
//   iteration 1 too; the gradient's size is |x - Plus(x, -g)|_inf (EvaluateGradientAndJacobian); an invalid step is
//   LevenbergMarquardtStrategy::StepIsInvalid = StepRejected(0): radius / decrease_factor, decrease_factor doubled,
//   diagonal kept.  tests/lm_reference.py restates the same rules with their sources.
// ---------------------------------------------------------------------------------------
namespace {
struct Corr { float p[4]; float pl[4]; };

struct Lin {
    std::vector<double> J;   // nres x 6 (robustified, unscaled)
    std::vector<double> r;   // nres
    double cost;
    double g[6];             // J^T r (unscaled)
};

static void linearise(const std::vector<Corr>& c, const double x[7], Lin& L, bool with_jac) {
    size_t nr = c.size();
    L.r.resize(nr);
    if (with_jac) L.J.resize(nr * 6);
    double cost = 0;
    for (int k = 0; k < 6; ++k) L.g[k] = 0;
    for (size_t i = 0; i < nr; ++i) {
        double J[6], r;
        double rho = plane_row(x, c[i].p, c[i].pl, 0.1, J, r);
        cost += 0.5 * rho;
        L.r[i] = r;
        if (with_jac) for (int k = 0; k < 6; ++k) { L.J[6 * i + k] = J[k]; L.g[k] += J[k] * r; }
    }
    L.cost = cost;
}

// min || [Js; diag(D)] y - [r; 0] ||  by Householder QR (from-knowledge: Ceres DenseQRSolver ->
// Eigen::HouseholderQR on the augmented system).  Js is nr x 6 already column-scaled.
static bool dense_qr_solve(const std::vector<double>& Js, const std::vector<double>& r, const double D[6], double y[6]) {
    size_t nr = r.size();
    size_t rows = nr + 6;
    std::vector<double> A(rows * 6, 0.0), b(rows, 0.0);
    for (size_t i = 0; i < nr; ++i) { for (int k = 0; k < 6; ++k) A[6 * i + k] = Js[6 * i + k]; b[i] = r[i]; }
    for (int k = 0; k < 6; ++k) A[6 * (nr + k) + k] = D[k];
    for (int k = 0; k < 6; ++k) {
        double tail = 0;
        for (size_t i = k + 1; i < rows; ++i) tail += A[6 * i + k] * A[6 * i + k];
        double c0 = A[6 * k + k], beta, tau;
        if (tail <= DBL_MIN) { tau = 0; beta = c0; }
        else {
            beta = std::sqrt(c0 * c0 + tail);
            if (c0 >= 0) beta = -beta;
            for (size_t i = k + 1; i < rows; ++i) A[6 * i + k] /= (c0 - beta);
            tau = (beta - c0) / beta;
        }
        A[6 * k + k] = beta;
        if (tau != 0) {
            for (int j = k + 1; j < 6; ++j) {
                double tmp = A[6 * k + j];
                for (size_t i = k + 1; i < rows; ++i) tmp += A[6 * i + k] * A[6 * i + j];
                A[6 * k + j] -= tau * tmp;
                for (size_t i = k + 1; i < rows; ++i) A[6 * i + j] -= tau * A[6 * i + k] * tmp;
            }
            double tmp = b[k];
            for (size_t i = k + 1; i < rows; ++i) tmp += A[6 * i + k] * b[i];
            b[k] -= tau * tmp;
            for (size_t i = k + 1; i < rows; ++i) b[i] -= tau * A[6 * i + k] * tmp;
        }
    }
    for (int i = 5; i >= 0; --i) {
        double s = b[i];
        for (int j = i + 1; j < 6; ++j) s -= A[6 * i + j] * y[j];
        if (A[6 * i + i] == 0) return false;
        y[i] = s / A[6 * i + i];
    }
    for (int k = 0; k < 6; ++k) if (!std::isfinite(y[k])) return false;
    return true;
}

static int ceres_lm(const std::vector<Corr>& c, double x[7], int max_num_iter, double* final_cost) {
    const double function_tolerance = 1e-6, parameter_tolerance = 1e-8, gradient_tolerance = 1e-10;
    const double min_relative_decrease = 1e-3, min_radius = 1e-32, max_radius = 1e16;
    const double min_diag = 1e-6, max_diag = 1e32;
    double radius = 1e4, decrease_factor = 2.0;
    bool reuse_diagonal = false;
    double diagonal[6];
    Lin L;
    if (c.empty()) { if (final_cost) *final_cost = 0; return 0; }   // nothing to minimise
    // iteration 0
    linearise(c, x, L, true);
    double x_cost = L.cost;
    double scaling[6];
    size_t nr = c.size();
    for (int k = 0; k < 6; ++k) {
        double s = 0;
        for (size_t i = 0; i < nr; ++i) s += L.J[6 * i + k] * L.J[6 * i + k];
        scaling[k] = 1.0 / (1.0 + std::sqrt(s));
    }
    std::vector<double> Js(nr * 6);
    auto scale_jac = [&]() { for (size_t i = 0; i < nr; ++i) for (int k = 0; k < 6; ++k) Js[6 * i + k] = L.J[6 * i + k] * scaling[k]; };
    scale_jac();
    double x_norm = 0; for (int k = 0; k < 7; ++k) x_norm += x[k] * x[k]; x_norm = std::sqrt(x_norm);
    int iteration = 0, invalid = 0;
    bool last_successful = true;        // IterationZero marks the start a successful step
    for (;;) {
        // FinalizeIterationAndCheckIfMinimizerCanContinue
        if (iteration >= max_num_iter) break;
        if (last_successful) {           // GradientToleranceReached on |x - Plus(x, -g)|_inf
            double ng[6], xg[7], gmax = 0;
            for (int k = 0; k < 6; ++k) ng[k] = -L.g[k];
            pose_plus(x, ng, xg);
            for (int k = 0; k < 7; ++k) gmax = std::max(gmax, std::fabs(x[k] - xg[k]));
            if (gmax <= gradient_tolerance) break;
        }
        if (radius < min_radius) break;
        ++iteration;
        last_successful = false;
        // ComputeTrustRegionStep (LevenbergMarquardtStrategy::ComputeStep)
        if (!reuse_diagonal) {
            for (int k = 0; k < 6; ++k) {
                double s = 0;
                for (size_t i = 0; i < nr; ++i) s += Js[6 * i + k] * Js[6 * i + k];
                diagonal[k] = std::min(std::max(s, min_diag), max_diag);
            }
        }
        double D[6], y[6], step[6];
        for (int k = 0; k < 6; ++k) D[k] = std::sqrt(diagonal[k] / radius);
        bool ok = dense_qr_solve(Js, L.r, D, y);
        reuse_diagonal = true;
        double model_cost_change = 0;
        if (ok) {
            for (int k = 0; k < 6; ++k) step[k] = -y[k];
            // model_cost_change = -(Js step) . (r + Js step / 2)
            for (size_t i = 0; i < nr; ++i) {
                double mr = 0;
                for (int k = 0; k < 6; ++k) mr += Js[6 * i + k] * step[k];
                model_cost_change -= mr * (L.r[i] + mr / 2.0);
            }
        }
        if (!ok || !(model_cost_change > 0.0)) {
            // HandleInvalidStep -> StepIsInvalid = StepRejected(0)
            if (++invalid >= 5) break;
            radius = radius / decrease_factor;
            decrease_factor *= 2.0;
            continue;
        }
        invalid = 0;
        for (int k = 0; k < 6; ++k) step[k] *= scaling[k];
        double xc[7];
        pose_plus(x, step, xc);
        Lin Lc;
        linearise(c, xc, Lc, false);
        double candidate_cost = Lc.cost;
        // ParameterToleranceReached
        double sn = 0; for (int k = 0; k < 7; ++k) sn += (x[k] - xc[k]) * (x[k] - xc[k]); sn = std::sqrt(sn);
        if (sn <= parameter_tolerance * (x_norm + parameter_tolerance)) break;
        // FunctionToleranceReached
        double cost_change = x_cost - candidate_cost;
        if (std::fabs(cost_change) <= function_tolerance * x_cost) break;
        double relative_decrease = cost_change / model_cost_change;
        if (relative_decrease > min_relative_decrease) {
            // HandleSuccessfulStep
            std::memcpy(x, xc, sizeof(xc));
            x_norm = 0; for (int k = 0; k < 7; ++k) x_norm += x[k] * x[k]; x_norm = std::sqrt(x_norm);
            linearise(c, x, L, true);
            scale_jac();
            x_cost = L.cost;
            last_successful = true;
            double q = 2.0 * relative_decrease - 1.0;
            radius = radius / std::max(1.0 / 3.0, 1.0 - q * q * q);
            radius = std::min(max_radius, radius);
            decrease_factor = 2.0;
            reuse_diagonal = false;
        } else {
            // HandleUnsuccessfulStep
            radius = radius / decrease_factor;
            decrease_factor *= 2.0;
            reuse_diagonal = true;
        }
    }
    if (final_cost) *final_cost = x_cost;
    return iteration;
}
}  // namespace

extern "C" int orc_ceres_solve(const float* feats_xyzw, int n, const unsigned char* corr_valid, const float* corr_plane,
                               double pose7[7], int max_num_iter, double* final_cost) {
    std::vector<Corr> c;
    for (int i = 0; i < n; ++i) if (corr_valid[i]) {
        Corr k;
        std::memcpy(k.p, feats_xyzw + 4 * (size_t)i, 16);
        std::memcpy(k.pl, corr_plane + 4 * (size_t)i, 16);
        c.push_back(k);
    }
    return ceres_lm(c, pose7, max_num_iter, final_cost);
}

extern "C" int orc_scan_to_map_ceres(const void* tree, const float* map_xyzw, int m, const float* feats_xyzw, int n,
                                     double pose7[7], int match_cnt, int max_num_iter, orc_iter_stats* stats, int nthreads) {
    if (m < 10) return -1;   // LidarOdometry.cpp:485-488
    std::vector<unsigned char> valid(n);
    std::vector<float> plane(4 * (size_t)n);
    double x[7];
    std::memcpy(x, pose7, sizeof(x));            // transformInc, :492-498
    for (int it = 0; it < match_cnt; ++it) {     // :506
        int nc = orc_find_surf_corr(tree, map_xyzw, m, feats_xyzw, n, x, valid.data(), plane.data(), nullptr, nullptr, nthreads);  // :513
        double s29[29];
        accumulate(feats_xyzw, n, valid.data(), plane.data(), x, 0.1, s29);
        double fc = 0;
        int lm = orc_ceres_solve(feats_xyzw, n, valid.data(), plane.data(), x, max_num_iter, &fc);  // :528-537
        unify(x);                                 // :539-549
        if (stats) {
            stats[it].n_corr = nc; stats[it].lm_iters = lm; stats[it].cost = s29[27];
            std::memcpy(stats[it].jtj_jtr, s29, 27 * sizeof(double));
            std::memcpy(stats[it].pose7, x, sizeof(x));
        }
    }
    std::memcpy(pose7, x, sizeof(x));            // :554-560
    return 0;
}

// ---- host glue -----------------------------------------------------------------------
// math_tools.h:125-138 deltaQ (un-normalised, w = 1) and Preprocessing.cpp:129-133.
extern "C" void orc_solve_rotation(double q_wxyz[4], const double gyr0[3], const double gyr1[3], double dt) {
    double un[3];
    for (int k = 0; k < 3; ++k) un[k] = 0.5 * (gyr0[k] + gyr1[k]);
    double th[3] = {un[0] * dt, un[1] * dt, un[2] * dt};
    Quat dq{1.0, th[0] / 2.0, th[1] / 2.0, th[2] / 2.0};
    Quat r = qmul(Quat{q_wxyz[0], q_wxyz[1], q_wxyz[2], q_wxyz[3]}, dq);
    q_wxyz[0] = r.w; q_wxyz[1] = r.x; q_wxyz[2] = r.y; q_wxyz[3] = r.z;
}

// LidarOdometry.cpp:415-442
extern "C" void orc_pose_compose(const double a[7], const double r[7], double o[7]) {
    Quat q0{a[0], a[1], a[2], a[3]};
    V3 t0{a[4], a[5], a[6]};
    Quat dq{r[0], r[1], r[2], r[3]};
    V3 dt{r[4], r[5], r[6]};
    V3 t = qrot(q0, dt) + t0;
    Quat q = qmul(q0, dq);
    o[0] = q.w; o[1] = q.x; o[2] = q.y; o[3] = q.z; o[4] = t.x; o[5] = t.y; o[6] = t.z;
}

// LidarOdometry.cpp:444-480
extern "C" void orc_pose_relative(const double p[7], const double c[7], double o[7]) {
    Quat q1{p[0], p[1], p[2], p[3]}, q2{c[0], c[1], c[2], c[3]};
    V3 t1{p[4], p[5], p[6]}, t2{c[4], c[5], c[6]};
    Quat qi = qinv(q1);
    Quat qr = qmul(qi, q2);
    V3 tr = qrot(qi, t2 - t1);
    o[0] = qr.w; o[1] = qr.x; o[2] = qr.y; o[3] = qr.z; o[4] = tr.x; o[5] = tr.y; o[6] = tr.z;
}

// ---- test hooks -------------------------------------------------------------------------
extern "C" void orc_eigen_sym3(const double a[9], double eval[3], double evec[9]) {
    double A[3][3], V[3][3];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) A[i][j] = a[3 * i + j];
    eigen_sym3(A, eval, V);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) evec[3 * i + j] = V[i][j];
}
extern "C" void orc_colpiv_qr_solve(int rows, const double* A, const double* b, double x[3]) { colpiv_qr_solve_nx3(rows, A, b, x); }
extern "C" void orc_slerp_identity(const double q[4], double t, double out[4]) {
    Quat r = qslerp(Quat{1, 0, 0, 0}, t, Quat{q[0], q[1], q[2], q[3]});
    out[0] = r.w; out[1] = r.x; out[2] = r.y; out[3] = r.z;
}
