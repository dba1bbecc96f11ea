// The trust-region state machine of the Ceres-faithful LM (Ceres 2.0's TrustRegionMinimizer + LevenbergMarquardtStrategy, as
// tests/lm_reference.py settles its rules), apart from the evaluations it asks for.  One home for the decisions of the solve:
// the single-GPU kernels (grid_knn.cu: k_lm_solve, k_lm_solve_batch) run them on thread 0 between block-wide evaluations, the
// collective LM of a sharded context (k_lm_advance, k_lm_end) between all-reduced evaluations, and tests/lm_tr_host.cpp on the
// host.  Every function reads and writes only the LmState and the 29 sums it is given (21 upper-triangle J^T J, 6 J^T r, cost,
// count), so the same sums give the same bits wherever it runs.  Like dev_math.cuh, whose pose_plus and solve6_ldlt it calls,
// it is device code that also compiles for the host (tests/lm_tr_host.cpp: plain operators, -ffp-contract=off).
//
// The loop, as the single-GPU kernel runs it:
//     st.x = start; st.max_num_iter = ...; S0 = eval(st.x); lm_begin(st, S0);
//     while (lm_propose(st)) { Sc = eval(st.xc); if (!lm_judge(st, Sc)) break; }
//     lm_end(st, pose, stats, neq0);
// lm_propose stops before evaluating anything more than max_num_iter candidates, so a driver that runs exactly
// 1 + max(0, max_num_iter) evaluation rounds (the start, then one candidate per round, no-op rounds once `done` is set) is
// always done by its last round.
#pragma once
#include "dev_math.cuh"

namespace lili {

// Why a solve stopped (LmState::done); 0 while it runs.
enum LmStop : int { kLmRunning = 0, kLmNoCorrespondences, kLmIterationCap, kLmGradient, kLmRadiusFloor, kLmFiveInvalid,
                    kLmParameter, kLmFunction };

struct LmState {
    double x[7];                 // the iterate (set by the caller before lm_begin)
    double S[29];                // the sums at x
    double radius, decrease_factor;
    bool reuse_diagonal, last_successful;
    double diagonal[6], scaling[6];      // the LM diagonal; the Jacobi scaling, fixed at iteration 0
    double x_cost, count0;               // cost at x; correspondences at the start
    int iteration, invalid;              // iterations counted (Ceres' count: invalid steps included); invalid steps in a row
    double model_cost_change;            // of the candidate
    double xc[7];                        // the candidate lm_propose asks to evaluate
    int done;                            // LmStop
    int max_num_iter;                    // set by the caller before lm_begin
};

// Part k of one row of the per-iteration stats (kStatsDoubles doubles: n_corr, lm_iters, cost, the 27 sums, pose7, pad).
// Part k < 29 is scalar k of the sums s; part 29 is the LM iteration count and the pose xn after the step.  The block kernels
// store one part per thread, the one-thread kernels every part.
__device__ __forceinline__ void write_stats(double* st, int k, const double* s, double lm_iters, const double* xn) {
    if (k < 29) st[k < 27 ? 3 + k : k == 27 ? 2 : 0] = s[k];
    else {
        st[1] = lm_iters;
#pragma unroll
        for (int j = 0; j < 7; ++j) st[30 + j] = xn[j];
    }
}

// From the sums S0 at the start st.x: the Jacobi scaling, the initial radius, and the start counted as a successful step
// (TrustRegionMinimizer::IterationZero), so that the gradient test also runs before iteration 1.
__device__ __forceinline__ void lm_begin(LmState& st, const double S0[29]) {
    for (int k = 0; k < 29; ++k) st.S[k] = S0[k];
    st.radius = 1e4; st.decrease_factor = 2.0;
    st.reuse_diagonal = false; st.last_successful = true;
    st.x_cost = S0[27];
    st.iteration = 0; st.invalid = 0;
    int kk = 0;
    for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) { if (i == j) st.scaling[i] = 1.0 / (1.0 + sqrt(S0[kk])); ++kk; }
    st.count0 = S0[28];
    st.model_cost_change = 0;
    st.done = kLmRunning;
}

// Proposes the next candidate in st.xc (true) or stops (false, st.done set).  Invalid steps (the damped system not solved, or
// no decrease predicted) are counted and rejected here without an evaluation: radius / decrease_factor, which doubles, the
// diagonal kept (LevenbergMarquardtStrategy::StepIsInvalid -> StepRejected(0)); five in a row stop the solve.
__device__ __forceinline__ bool lm_propose(LmState& st) {
    for (;;) {
        if (st.count0 <= 0.0) { st.done = kLmNoCorrespondences; return false; }
        if (st.iteration >= st.max_num_iter) { st.done = kLmIterationCap; return false; }
        if (st.last_successful) {      // |x - Plus(x, -g)|_inf
            // the translation part first, as Plus forms it: when it alone exceeds the tolerance the decision is made, and the
            // quaternion part (sincos on a single thread for a large g) is only formed near a stop
            double tmax = 0;
            for (int k = 0; k < 3; ++k) tmax = fmax(tmax, fabs(st.x[4 + k] - (st.x[4 + k] + -st.S[24 + k])));
            if (tmax <= 1e-10) {
                double ng[6], xg[7], gmax = 0;
                for (int k = 0; k < 6; ++k) ng[k] = -st.S[21 + k];
                pose_plus(st.x, ng, xg);
                for (int k = 0; k < 7; ++k) gmax = fmax(gmax, fabs(st.x[k] - xg[k]));
                if (gmax <= 1e-10) { st.done = kLmGradient; return false; }
            }
        }
        if (st.radius < 1e-32) { st.done = kLmRadiusFloor; return false; }
        ++st.iteration;
        st.last_successful = false;
        // scaled normal equations  Hs = S H S, gs = S g
        double Hs[21], gs[6];
        int kk = 0;
        for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) { Hs[kk] = st.S[kk] * st.scaling[i] * st.scaling[j]; ++kk; }
        for (int i = 0; i < 6; ++i) gs[i] = st.S[21 + i] * st.scaling[i];
        if (!st.reuse_diagonal) {
            kk = 0;
            for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) { if (i == j) st.diagonal[i] = fmin(fmax(Hs[kk], 1e-6), 1e32); ++kk; }
        }
        double Ha[21];
        kk = 0;
        for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) { Ha[kk] = Hs[kk] + (i == j ? st.diagonal[i] / st.radius : 0.0); ++kk; }
        double y[6];
        bool ok = solve6_ldlt(Ha, gs, y);
        st.reuse_diagonal = true;
        double step[6];
        st.model_cost_change = 0;
        if (ok) {
            for (int k = 0; k < 6; ++k) step[k] = -y[k];
            // -(step.gs + 1/2 step^T Hs step)
            double Hfull[6][6];
            kk = 0;
            for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) { Hfull[i][j] = Hs[kk]; Hfull[j][i] = Hs[kk]; ++kk; }
            double sg = 0, shs = 0;
            for (int i = 0; i < 6; ++i) {
                sg += step[i] * gs[i];
                double hv = 0;
                for (int j = 0; j < 6; ++j) hv += Hfull[i][j] * step[j];
                shs += step[i] * hv;
            }
            st.model_cost_change = -(sg + 0.5 * shs);
        }
        if (!ok || !(st.model_cost_change > 0.0)) {
            if (++st.invalid >= 5) { st.done = kLmFiveInvalid; return false; }
            st.radius = st.radius / st.decrease_factor;      // StepIsInvalid = StepRejected(0)
            st.decrease_factor *= 2.0;
            continue;
        }
        st.invalid = 0;
        double step_keep[6];
        for (int k = 0; k < 6; ++k) step_keep[k] = step[k] * st.scaling[k];
        pose_plus(st.x, step_keep, st.xc);
        return true;
    }
}

// Judges the candidate st.xc from its sums Sc: the parameter and function tolerances stop the solve (false, st.done set);
// otherwise the step is accepted on a relative decrease above 1e-3 (radius grown by the rho rule) or rejected (radius divided
// by decrease_factor, which doubles), and the solve goes on (true).
__device__ __forceinline__ bool lm_judge(LmState& st, const double Sc[29]) {
    double candidate_cost = Sc[27];
    double xn = 0, sn = 0;
    for (int k = 0; k < 7; ++k) { xn += st.x[k] * st.x[k]; sn += (st.x[k] - st.xc[k]) * (st.x[k] - st.xc[k]); }
    xn = sqrt(xn); sn = sqrt(sn);
    double cost_change = st.x_cost - candidate_cost;
    if (sn <= 1e-8 * (xn + 1e-8)) { st.done = kLmParameter; return false; }                 // parameter tolerance
    if (fabs(cost_change) <= 1e-6 * st.x_cost) { st.done = kLmFunction; return false; }     // function tolerance
    double relative_decrease = cost_change / st.model_cost_change;
    if (relative_decrease > 1e-3) {
        for (int k = 0; k < 7; ++k) st.x[k] = st.xc[k];
        for (int k = 0; k < 29; ++k) st.S[k] = Sc[k];
        st.x_cost = candidate_cost;
        st.last_successful = true;
        double qd = 2.0 * relative_decrease - 1.0;
        st.radius = st.radius / fmax(1.0 / 3.0, 1.0 - qd * qd * qd);
        st.radius = fmin(1e16, st.radius);
        st.decrease_factor = 2.0;
        st.reuse_diagonal = false;
    } else {
        st.radius = st.radius / st.decrease_factor;
        st.decrease_factor *= 2.0;
        st.reuse_diagonal = true;
    }
    return true;
}

// The result: the quaternion with w >= 0 (L/src/LidarOdometry.cpp:539-549) into pose, and, when stats is given, the outer
// iteration's stats row from the linearisation sums neq0 with the iteration count and the pose.
__device__ __forceinline__ void lm_end(LmState& st, double* pose, double* stats, const double* neq0) {
    if (st.x[0] < 0) { st.x[0] = -st.x[0]; st.x[1] = -st.x[1]; st.x[2] = -st.x[2]; st.x[3] = -st.x[3]; }
    for (int k = 0; k < 7; ++k) pose[k] = st.x[k];
    if (stats) {
#pragma unroll
        for (int k = 0; k <= 29; ++k) write_stats(stats, k, neq0, (double)st.iteration, st.x);
    }
}

}  // namespace lili
