// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
// legs may build, load or call anything under oracle/.
//
// PARITY UNPINNED: the reference (KIT-ISAS/lili-om) ships no tests, golden vectors or
// fixtures for this path, and cannot be built here (needs ROS, PCL, Eigen, Ceres, glog —
// none present, no network).  This file restates, from knowledge, the third-party
// numerical routines the reference calls on the hot path (marked "from-knowledge"),
// so that the rest of the oracle can follow the reference source expression by
// expression.  Citations are relative to the reference repository's root.
//
// Compile with -O3 -ffp-contract=off (the reference builds with -O3 for generic x86-64:
// no FMA contraction, LiLi-OM/CMakeLists.txt:5).
#pragma once
#include <cmath>
#include <cfloat>
#include <cstdint>
#include <algorithm>

namespace orc {

struct V3 { double x, y, z; };
static inline V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
static inline V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
static inline V3 operator*(double s, V3 a) { return {s * a.x, s * a.y, s * a.z}; }
static inline double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
static inline V3 cross(V3 a, V3 b) {
    return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
static inline double norm(V3 a) { return std::sqrt(dot(a, a)); }

// Quaternion in Eigen's constructor order (w, x, y, z).
struct Quat { double w, x, y, z; };

// from-knowledge: Eigen::Quaterniond * Eigen::Quaterniond (Hamilton product).
static inline Quat qmul(Quat a, Quat b) {
    return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z,
            a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
            a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}

// from-knowledge: Eigen::Quaterniond * Vector3d (QuaternionBase::_transformVector):
//   uv = q.vec x v; uv += uv; return v + w*uv + q.vec x uv     (no normalisation)
// Call sites: LiLi-OM/src/LidarOdometry.cpp:231,261; LiLi-OM/src/Preprocessing.cpp:118.
static inline V3 qrot(Quat q, V3 v) {
    V3 qv{q.x, q.y, q.z};
    V3 uv = cross(qv, v);
    uv = uv + uv;
    return v + q.w * uv + cross(qv, uv);
}

// from-knowledge: Eigen::Quaterniond::inverse(): conjugate / squaredNorm (zero if n2 == 0).
static inline Quat qinv(Quat q) {
    double n2 = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z;
    if (n2 > 0) return {q.w / n2, -q.x / n2, -q.y / n2, -q.z / n2};
    return {0, 0, 0, 0};
}

// from-knowledge: Eigen::Quaterniond::slerp(t, other) — result NOT re-normalised.
// Call site: LiLi-OM/src/Preprocessing.cpp:114-115 (q0 = Identity, other = q_iMU).
static inline Quat qslerp(Quat a, double t, Quat b) {
    const double one = 1.0 - DBL_EPSILON;
    double d = a.w * b.w + a.x * b.x + a.y * b.y + a.z * b.z;
    double absD = std::fabs(d);
    double s0, s1;
    if (absD >= one) {
        s0 = 1.0 - t;
        s1 = t;
    } else {
        double theta = std::acos(absD);
        double sinTheta = std::sin(theta);
        s0 = std::sin((1.0 - t) * theta) / sinTheta;
        s1 = std::sin(t * theta) / sinTheta;
    }
    if (d < 0) s1 = -s1;
    return {s0 * a.w + s1 * b.w, s0 * a.x + s1 * b.x, s0 * a.y + s1 * b.y, s0 * a.z + s1 * b.z};
}

// ---------------------------------------------------------------------------------------
// from-knowledge: Eigen::SelfAdjointEigenSolver<Matrix3d>::compute (iterative path, Eigen
// 3.3.7+/3.4): scale by max-abs of the lower triangle, closed-form 3x3 Householder
// tridiagonalisation, implicit symmetric QR steps with Wilkinson shift, ascending sort.
// Call sites: LiLi-OM/src/Preprocessing.cpp:298,351; LiLi-OM/src/BackendFusion.cpp:1568.
// A is symmetric, row-major a[3][3]; only the lower triangle is read.
// evec[r][c]: component r of eigenvector c (columns match eval[c]).
// ---------------------------------------------------------------------------------------
static inline void givens(double p, double q, double& c, double& s) {
    if (q == 0.0) {
        c = p < 0 ? -1.0 : 1.0;
        s = 0.0;
    } else if (p == 0.0) {
        c = 0.0;
        s = q < 0 ? 1.0 : -1.0;
    } else if (std::fabs(p) > std::fabs(q)) {
        double t = q / p;
        double u = std::sqrt(1.0 + t * t);
        if (p < 0) u = -u;
        c = 1.0 / u;
        s = -t * c;
    } else {
        double t = p / q;
        double u = std::sqrt(1.0 + t * t);
        if (q < 0) u = -u;
        s = -1.0 / u;
        c = -t * s;
    }
}

static inline double eig_hypot(double x, double y) {
    double ax = std::fabs(x), ay = std::fabs(y);
    double p = ax > ay ? ax : ay;
    if (p == 0.0) return 0.0;
    double qp = (ax > ay ? ay : ax) / p;
    return p * std::sqrt(1.0 + qp * qp);
}

static inline void eigen_sym3(const double a[3][3], double eval[3], double evec[3][3]) {
    double m00 = a[0][0], m10 = a[1][0], m20 = a[2][0], m11 = a[1][1], m21 = a[2][1], m22 = a[2][2];
    double scale = 0.0;
    {
        const double l[6] = {m00, m10, m20, m11, m21, m22};
        for (double v : l) scale = std::max(scale, std::fabs(v));
    }
    if (scale == 0.0) scale = 1.0;
    m00 /= scale; m10 /= scale; m20 /= scale; m11 /= scale; m21 /= scale; m22 /= scale;

    double diag[3], sub[2];
    double Q[3][3];
    const double tol = DBL_MIN;
    diag[0] = m00;
    double v1norm2 = m20 * m20;
    if (v1norm2 <= tol) {
        diag[1] = m11; diag[2] = m22; sub[0] = m10; sub[1] = m21;
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Q[i][j] = (i == j);
    } else {
        double beta = std::sqrt(m10 * m10 + v1norm2);
        double invBeta = 1.0 / beta;
        double m01 = m10 * invBeta;
        double m02 = m20 * invBeta;
        double q = 2.0 * m01 * m21 + m02 * (m22 - m11);
        diag[1] = m11 + m02 * q;
        diag[2] = m22 - m02 * q;
        sub[0] = beta;
        sub[1] = m21 - m01 * q;
        Q[0][0] = 1; Q[0][1] = 0;   Q[0][2] = 0;
        Q[1][0] = 0; Q[1][1] = m01; Q[1][2] = m02;
        Q[2][0] = 0; Q[2][1] = m02; Q[2][2] = -m01;
    }

    const int n = 3;
    int end = n - 1, start = 0, iter = 0;
    const int maxIter = 30;
    const double considerAsZero = DBL_MIN;
    const double precision_inv = 1.0 / DBL_EPSILON;
    while (end > 0) {
        for (int i = start; i < end; ++i) {
            if (std::fabs(sub[i]) < considerAsZero) {
                sub[i] = 0.0;
            } else {
                double ss = precision_inv * sub[i];
                if (ss * ss <= (std::fabs(diag[i]) + std::fabs(diag[i + 1]))) sub[i] = 0.0;
            }
        }
        while (end > 0 && sub[end - 1] == 0.0) end--;
        if (end <= 0) break;
        iter++;
        if (iter > maxIter * n) break;
        start = end - 1;
        while (start > 0 && sub[start - 1] != 0.0) start--;

        // tridiagonal_qr_step
        double td = (diag[end - 1] - diag[end]) * 0.5;
        double e = sub[end - 1];
        double mu = diag[end];
        if (td == 0.0) {
            mu -= std::fabs(e);
        } else if (e != 0.0) {
            double e2 = e * e;
            double h = eig_hypot(td, e);
            if (e2 == 0.0) mu -= e / ((td + (td > 0 ? h : -h)) / e);
            else mu -= e2 / (td + (td > 0 ? h : -h));
        }
        double x = diag[start] - mu;
        double z = sub[start];
        for (int k = start; k < end && z != 0.0; ++k) {
            double c, s;
            givens(x, z, c, s);
            double sdk = s * diag[k] + c * sub[k];
            double dkp1 = s * sub[k] + c * diag[k + 1];
            diag[k] = c * (c * diag[k] - s * sub[k]) - s * (c * sub[k] - s * diag[k + 1]);
            diag[k + 1] = s * sdk + c * dkp1;
            sub[k] = c * sdk - s * dkp1;
            if (k > start) sub[k - 1] = c * sub[k - 1] - s * z;
            x = sub[k];
            if (k < end - 1) {
                z = -s * sub[k + 1];
                sub[k + 1] = c * sub[k + 1];
            }
            // Q = Q * G : columns k, k+1
            for (int r = 0; r < 3; ++r) {
                double qk = Q[r][k], qk1 = Q[r][k + 1];
                Q[r][k] = c * qk - s * qk1;
                Q[r][k + 1] = s * qk + c * qk1;
            }
        }
    }
    // ascending selection sort, swapping eigenvector columns
    for (int i = 0; i < n - 1; ++i) {
        int k = i;
        for (int j = i + 1; j < n; ++j) if (diag[j] < diag[k]) k = j;
        if (k != i) {
            std::swap(diag[i], diag[k]);
            for (int r = 0; r < 3; ++r) std::swap(Q[r][i], Q[r][k]);
        }
    }
    for (int i = 0; i < 3; ++i) {
        eval[i] = diag[i] * scale;
        for (int r = 0; r < 3; ++r) evec[r][i] = Q[r][i];
    }
}

// ---------------------------------------------------------------------------------------
// from-knowledge: Eigen::Matrix<double,5,3>::colPivHouseholderQr().solve(b) (Eigen 3.3):
// column-pivoted Householder QR with LAPACK-style norm down-dating, solution over the
// first `nonzero_pivots` pivoted columns, remaining components zero.
// Call sites: LiLi-OM/src/LidarOdometry.cpp:375; LiLi-OM/src/BackendFusion.cpp:1641.
// A is rows x 3 row-major (rows <= 8).
// ---------------------------------------------------------------------------------------
static inline void colpiv_qr_solve_nx3(int rows, const double* Ain, const double* bin, double xout[3]) {
    const int cols = 3;
    double A[8][3];
    double c[8];
    for (int i = 0; i < rows; ++i) {
        for (int j = 0; j < 3; ++j) A[i][j] = Ain[i * 3 + j];
        c[i] = bin[i];
    }
    double normsUpd[3], normsDir[3], hcoef[3];
    int perm[3] = {0, 1, 2};
    for (int k = 0; k < cols; ++k) {
        double s = 0;
        for (int i = 0; i < rows; ++i) s += A[i][k] * A[i][k];
        normsUpd[k] = normsDir[k] = std::sqrt(s);
    }
    double maxn = std::max(normsUpd[0], std::max(normsUpd[1], normsUpd[2]));
    double th = maxn * DBL_EPSILON;
    const double threshold_helper = th * th / double(rows);
    const double norm_downdate_threshold = std::sqrt(DBL_EPSILON);
    int nonzero_pivots = cols;
    for (int k = 0; k < cols; ++k) {
        int big = k;
        for (int j = k + 1; j < cols; ++j) if (normsUpd[j] > normsUpd[big]) big = j;
        double big_sq = normsUpd[big] * normsUpd[big];
        if (nonzero_pivots == cols && big_sq < threshold_helper * double(rows - k)) nonzero_pivots = k;
        if (k != big) {
            for (int i = 0; i < rows; ++i) std::swap(A[i][k], A[i][big]);
            std::swap(normsUpd[k], normsUpd[big]);
            std::swap(normsDir[k], normsDir[big]);
            std::swap(perm[k], perm[big]);
        }
        // makeHouseholderInPlace on A[k..rows-1][k]
        double tailSq = 0;
        for (int i = k + 1; i < rows; ++i) tailSq += A[i][k] * A[i][k];
        double c0 = A[k][k];
        double tau, beta;
        if (tailSq <= DBL_MIN) {
            tau = 0; beta = c0;
            for (int i = k + 1; i < rows; ++i) A[i][k] = 0;
        } else {
            beta = std::sqrt(c0 * c0 + tailSq);
            if (c0 >= 0) beta = -beta;
            for (int i = k + 1; i < rows; ++i) A[i][k] = A[i][k] / (c0 - beta);
            tau = (beta - c0) / beta;
        }
        A[k][k] = beta;
        hcoef[k] = tau;
        // apply H = I - tau v v^T (v = [1; essential]) to the trailing columns
        if (tau != 0) {
            for (int j = k + 1; j < cols; ++j) {
                double tmp = 0;
                for (int i = k + 1; i < rows; ++i) tmp += A[i][k] * A[i][j];
                tmp += A[k][j];
                A[k][j] -= tau * tmp;
                for (int i = k + 1; i < rows; ++i) A[i][j] -= tau * A[i][k] * tmp;
            }
        }
        for (int j = k + 1; j < cols; ++j) {
            if (normsUpd[j] != 0) {
                double temp = std::fabs(A[k][j]) / normsUpd[j];
                temp = (1.0 + temp) * (1.0 - temp);
                temp = temp < 0 ? 0 : temp;
                double r = normsUpd[j] / normsDir[j];
                double temp2 = temp * r * r;
                if (temp2 <= norm_downdate_threshold) {
                    double s = 0;
                    for (int i = k + 1; i < rows; ++i) s += A[i][j] * A[i][j];
                    normsDir[j] = std::sqrt(s);
                    normsUpd[j] = normsDir[j];
                } else {
                    normsUpd[j] *= std::sqrt(temp);
                }
            }
        }
    }
    xout[0] = xout[1] = xout[2] = 0;
    if (nonzero_pivots == 0) return;
    // c = Q^T b : apply H_0 .. H_{nonzero_pivots-1}
    for (int k = 0; k < nonzero_pivots; ++k) {
        double tau = hcoef[k];
        if (tau == 0) continue;
        double tmp = c[k];
        for (int i = k + 1; i < rows; ++i) tmp += A[i][k] * c[i];
        c[k] -= tau * tmp;
        for (int i = k + 1; i < rows; ++i) c[i] -= tau * A[i][k] * tmp;
    }
    // back-substitution on the leading nonzero_pivots block
    for (int i = nonzero_pivots - 1; i >= 0; --i) {
        double s = c[i];
        for (int j = i + 1; j < nonzero_pivots; ++j) s -= A[i][j] * c[j];
        c[i] = s / A[i][i];
    }
    for (int i = 0; i < nonzero_pivots; ++i) xout[perm[i]] = c[i];
}

}  // namespace orc
