// Compile-only stand-in for the Ceres (and glog) names the odometry's translation units mention.  No cost functor is
// instantiated, and ceres::Solve aborts: the harnesses never drive updateTransformationWithCeres.
#pragma once
#include <cstdlib>

namespace google { inline void InitGoogleLogging(const char*) {} }

namespace ceres {
struct CostFunction { virtual ~CostFunction() {} };
struct LossFunction { virtual ~LossFunction() {} };
struct HuberLoss : LossFunction { explicit HuberLoss(double) {} };
struct CauchyLoss : LossFunction { explicit CauchyLoss(double) {} };
struct LocalParameterization { virtual ~LocalParameterization() {} };
struct QuaternionParameterization : LocalParameterization {};
template <class F, int... Sizes> struct AutoDiffCostFunction : CostFunction {
    explicit AutoDiffCostFunction(F* f) : functor(f) {}
    ~AutoDiffCostFunction() { delete functor; }
    F* functor;
};
struct Problem {
    void AddParameterBlock(double*, int, LocalParameterization* = nullptr) {}
    template <class... B> void AddResidualBlock(CostFunction*, LossFunction*, B*...) {}
};
enum LinearSolverType { DENSE_QR, DENSE_SCHUR, SPARSE_NORMAL_CHOLESKY, SPARSE_SCHUR };
struct Solver {
    struct Options {
        LinearSolverType linear_solver_type = DENSE_QR;
        int max_num_iterations = 50;
        double max_solver_time_in_seconds = 1e9;
        bool minimizer_progress_to_stdout = false;
        bool check_gradients = false;
        double gradient_check_relative_precision = 1e-8;
    };
    struct Summary {};
};
inline void Solve(const Solver::Options&, Problem*, Solver::Summary*) { std::abort(); }
template <class T> void QuaternionRotatePoint(const T q[4], const T pt[3], T result[3]);
template <class T> void UnitQuaternionRotatePoint(const T q[4], const T pt[3], T result[3]);
template <class T> void QuaternionProduct(const T z[4], const T w[4], T zw[4]);
}  // namespace ceres
