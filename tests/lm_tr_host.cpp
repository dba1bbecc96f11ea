// TEST INFRASTRUCTURE: host build of the LM's trust-region state machine (liliom_b200/csrc/lm_tr.cuh), driven the two ways
// the device drives it: the single-GPU kernel's loop (lm_solve_body: evaluate, then propose / evaluate / judge until a stop)
// and the collective LM's fixed rounds (k_lm_eval_part / k_lm_advance: exactly 1 + max(0, max_num_iter) rounds, no-op rounds
// once done).  The evaluations come from the caller (a callback: the sums at a pose), so both drivers see the same sums.
// The round-to-nearest intrinsics become plain operators (this file is compiled with -ffp-contract=off: nothing is fused).
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
#include "../liliom_b200/csrc/lm_tr.cuh"

using namespace lili;

extern "C" {
typedef void (*lmtr_eval_fn)(const double* x7, double* out29);

// What one drive of the state machine leaves: the pose and stats row lm_end writes, the iteration count, the stop, and every
// pose it asked the sums of (log: 7 doubles each, at most cap of them; n_eval counts them all).
struct LmtrResult {
    double pose[7];
    double stats[40];
    int iteration, done, n_eval, rounds;
};

static void logged(lmtr_eval_fn ev, const double* x, double* S, double* log, int cap, LmtrResult* r) {
    if (r->n_eval < cap) memcpy(log + 7 * (size_t)r->n_eval, x, 7 * sizeof(double));
    ++r->n_eval;
    ev(x, S);
}

// lm_solve_body's loop order.
void lmtr_loop(const double* x0, int max_num_iter, const double* neq0, lmtr_eval_fn ev, double* log, int cap, LmtrResult* r) {
    memset(r, 0, sizeof(*r));
    LmState st;
    memcpy(st.x, x0, sizeof(st.x));
    st.max_num_iter = max_num_iter;
    double S[29];
    logged(ev, st.x, S, log, cap, r);
    lm_begin(st, S);
    while (lm_propose(st)) {
        double Sc[29];
        logged(ev, st.xc, Sc, log, cap, r);
        if (!lm_judge(st, Sc)) break;
    }
    r->iteration = st.iteration; r->done = st.done;
    lm_end(st, r->pose, r->stats, neq0);
}

// The collective LM's rounds on one rank, whose all-reduce returns the callback's sums: round 0 evaluates at the start and
// runs lm_begin + lm_propose, every later round evaluates the candidate (zeros once done) and runs lm_judge + lm_propose
// unless done.  rounds < 0: 1 + max(0, max_num_iter), as the host sequence runs them.  r->done is the state after the last round.
void lmtr_rounds(const double* x0, int max_num_iter, int rounds, const double* neq0, lmtr_eval_fn ev, double* log, int cap,
                 LmtrResult* r) {
    memset(r, 0, sizeof(*r));
    if (rounds < 0) rounds = 1 + (max_num_iter > 0 ? max_num_iter : 0);
    LmState st;
    memset(&st, 0xff, sizeof(st));          // whatever an earlier call left: round 0 must not read it
    double sums[29];
    for (int round = 0; round < rounds; ++round) {
        // k_lm_eval_part
        if (round == 0) {
            memcpy(st.x, x0, sizeof(st.x));
            st.done = kLmRunning;
            logged(ev, st.x, sums, log, cap, r);
        } else if (st.done != kLmRunning) {
            for (double& v : sums) v = 0.0;
        } else {
            logged(ev, st.xc, sums, log, cap, r);
        }
        // k_lm_advance
        if (round == 0) {
            st.max_num_iter = max_num_iter;
            lm_begin(st, sums);
            lm_propose(st);
        } else if (st.done == kLmRunning) {
            if (lm_judge(st, sums)) lm_propose(st);
        }
    }
    r->rounds = rounds;
    r->iteration = st.iteration; r->done = st.done;
    lm_end(st, r->pose, r->stats, neq0);        // k_lm_end
}
}
