"""TEST INFRASTRUCTURE: Ceres 2.0's TrustRegionMinimizer + LevenbergMarquardtStrategy restated in NumPy for the scan-to-map
problem on frozen correspondences (features and their planes), with a trace of every iteration.

Sums.  Each row is built in fp64 the way dev_math.cuh::plane_row and huber_correct build it (r = n.(Rp + t) + d,
J = [2 (Rp x n), n], both scaled by sqrt(rho') of HuberLoss(0.1)), and every one of the 29 scalars is summed with math.fsum:
correctly rounded, independent of order.  Next to each sum the sum of its |terms| is kept; the device's 512-thread block
reduction is within gamma_d of it per scalar (d = the depth of that reduction, see reduction_bound).

Two step solvers, both reported on every iteration: "normal" (the device's: Hs + diag(D^2) solved as a dense system) and "qr"
(Ceres' DENSE_QR: least squares on [Js; diag(D)] against [r; 0]).  The trace follows one of them (`solver`).

Ceres rules, settled from the Ceres 2.0 source (ceres/internal/trust_region_minimizer.cc, levenberg_marquardt_strategy.cc):
  * Invalid step.  LevenbergMarquardtStrategy::StepIsInvalid() is `StepRejected(0.0)`: radius /= decrease_factor,
    decrease_factor *= 2, reuse_diagonal = true.  (The oracle and the kernel used to halve the radius and recompute the
    diagonal; a sequence invalid -> rejected then shrinks the radius by 2 * 2 instead of 2 * 4.)
  * Gradient size.  TrustRegionMinimizer::EvaluateGradientAndJacobian sets gradient_max_norm = |x - Plus(x, -g)|_inf in the
    ambient coordinates (7 here: the quaternion and t), not max|g| in the tangent space.
  * Gradient test at the start.  TrustRegionMinimizer::IterationZero ends with step_is_successful = true, and
    FinalizeIterationAndCheckIfMinimizerCanContinue runs GradientToleranceReached (which only looks at a successful step)
    before the first iteration as after every other.  So a start with a zero gradient stops after 0 iterations.  (The oracle
    and the kernel used to test the gradient only after a step had been accepted: such a start then took five invalid steps.)
  * Model cost change.  ComputeTrustRegionStep: model_cost_change = -(Js s).(r + Js s / 2), over the residuals.  The kernel
    uses -(s.gs + s^T Hs s / 2), equal in exact arithmetic.  Both are reported; the trace's decision uses its solver's formula.
  * Order of the stops: iteration cap, gradient (after a successful step or at the start), radius < 1e-32 before a step;
    after it, invalid (five in a row stop), parameter tolerance |x - x_c| <= 1e-8 (|x| + 1e-8), function tolerance
    |cost change| <= 1e-6 cost, then accept on relative decrease > 1e-3.

The radius floor needs about 15 consecutive rejections (1e4 / 2^(1+2+...+15) < 1e-32).  A rejection shrinks the next step with
the radius, and the parameter tolerance stops the solve once a step is shorter than 1e-8 |x| (|x| >= 1: the quaternion),
long before then: no world of tests/lm_adversarial.py reaches it, and none pretends to.  Invalid steps are out of reach too,
under the settled rules: with g != 0 (the gradient test has passed) the normal formula is >= (s.gs)/2 > 0 to rounding, and
Hs + D^2 is positive definite -- on well-conditioned input.  When the damped system is ill-conditioned (a rank-deficient
J^T J with the radius far beyond 1e4, so the damping 1e-6 / radius is below the rounding of Hs) s.gs can cancel and an LDL^T
pivot can fail; no world here reaches that.  An exactly zero gradient let through by the old start rule was what produced
invalid steps before.

Decisions.  Every comparison with a threshold is recorded with its distance from the threshold and a rounding bound derived
from the |terms| of what it compares plus, after a step, the one-step bound of the candidate (a device's candidate may lie
that far from the reference's).  A decision whose distance is within its bound is OPEN: `traces` follows both outcomes and
returns every admissible trace; `follow` (the device check) takes at an open decision whichever outcome the device's iterates
show.
"""
from __future__ import annotations

import copy
import math

import numpy as np

U = np.finfo(np.float64).eps / 2
HUBER_A = 0.1
RADIUS0, MAX_RADIUS, MIN_RADIUS = 1e4, 1e16, 1e-32
MIN_DIAG, MAX_DIAG = 1e-6, 1e32
FUNCTION_TOL, PARAMETER_TOL, GRADIENT_TOL, MIN_REL_DECREASE = 1e-6, 1e-8, 1e-10, 1e-3
MAX_INVALID = 5
LM_BLOCK = 512          # grid_knn.cu::kLmBlock
ROW_ULPS = 16           # a row's own rounding (device closed form vs this one): a few u per term, rounded up
PLUS_ULPS = 8           # rounding of Plus (as reanchor.PLUS_ULPS)
STOPS = ("iteration_cap", "gradient", "parameter", "function", "five_invalid", "radius_floor", "no_correspondences")
BRANCHES = ("accepted", "rejected", "invalid")

# the rules of Ceres 2.0 (see the module docstring); a planted fault replaces one
CERES = dict(gradient_at_start=True, gradient_ambient=True, invalid="ceres", reject_double=True, reject_div=None,
             rescale_each_accept=False, mcc_half=True, grow=None, reset_df=True)


def gamma(n):
    return n * U / (1 - n * U)


def unpack(s29):
    H = np.zeros((6, 6))
    H[np.triu_indices(6)] = s29[:21]
    H = H + np.triu(H, 1).T
    return H, np.asarray(s29[21:27], np.float64)


def plus(x, d):
    """ceres::QuaternionParameterization::Plus on q, identity on t."""
    nd = float(np.linalg.norm(d[:3]))
    out = np.array(x, np.float64)
    if nd > 0:
        aw, ax, ay, az = math.cos(nd), *(math.sin(nd) / nd * np.asarray(d[:3], np.float64))
        bw, bx, by, bz = x[:4]
        out[:4] = [aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                   aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx]
    out[4:] = np.asarray(x[4:], np.float64) + np.asarray(d[3:], np.float64)
    return out


def unify(x):
    x = np.array(x, np.float64)
    if x[0] < 0:
        x[:4] = -x[:4]
    return x


def _rotmat(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def f4(feats):
    """n x 4 fp32 features from an array or a PCL point array (x, y, z fields)."""
    feats = np.asarray(feats)
    if feats.dtype.fields is not None:
        out = np.ones((len(feats), 4), np.float32)
        out[:, 0] = feats["x"]; out[:, 1] = feats["y"]; out[:, 2] = feats["z"]
        return out
    return np.asarray(feats, np.float32).reshape(-1, 4)


def rows(feats, valid, plane, x, a=HUBER_A):
    """The corrected rows of the valid correspondences at x: (J (n x 6), r (n), rho / 2 (n), outer (n: Huber's outer region))."""
    sel = np.asarray(valid) != 0
    f = f4(feats)[sel, :3].astype(np.float64)
    pl = np.asarray(plane, np.float32).reshape(-1, 4)[sel].astype(np.float64)
    rp = f @ _rotmat(x[:4]).T
    n = pl[:, :3]
    r = n[:, 0] * (rp[:, 0] + x[4]) + n[:, 1] * (rp[:, 1] + x[5]) + n[:, 2] * (rp[:, 2] + x[6]) + pl[:, 3]
    J = np.empty((len(r), 6))
    J[:, 0] = 2 * (rp[:, 1] * n[:, 2] - rp[:, 2] * n[:, 1])
    J[:, 1] = 2 * (rp[:, 2] * n[:, 0] - rp[:, 0] * n[:, 2])
    J[:, 2] = 2 * (rp[:, 0] * n[:, 1] - rp[:, 1] * n[:, 0])
    J[:, 3:] = n
    s2, b2 = r * r, a * a
    outer = s2 > b2
    rt = np.sqrt(s2)
    rho0 = np.where(outer, 2 * a * rt - b2, s2)
    with np.errstate(divide="ignore"):
        rho1 = np.where(outer, np.maximum(np.finfo(np.float64).tiny, a / np.where(outer, rt, 1.0)), 1.0)
    sr = np.sqrt(rho1)
    return J * sr[:, None], r * sr, 0.5 * rho0, outer


def sums(J, r, half):
    """The 29 scalars (normal_equations order) summed with math.fsum, and the sums of their |terms|."""
    iu = np.triu_indices(6)
    cols = [J[:, i] * J[:, j] for i, j in zip(*iu)] + [J[:, i] * r for i in range(6)] + [half, np.ones(len(r))]
    return (np.array([math.fsum(c) for c in cols]), np.array([float(np.abs(c).sum()) for c in cols]))


def reduction_bound(n_rows, abs29):
    """|device sum - fsum| per scalar: the block reduction's depth d = ceil(n / 512) serial adds per thread, 5 xor levels in the
    warp, 16 warp sums in order, each a relative u; each term's own rounding ROW_ULPS u."""
    d = -(-max(int(n_rows), 1) // LM_BLOCK) + 5 + LM_BLOCK // 32
    return (gamma(d) + ROW_ULPS * U) * np.asarray(abs29)


class Problem:
    """Frozen correspondences: evaluates sums at a pose (cached)."""

    def __init__(self, feats, valid, plane):
        self.feats, self.valid, self.plane = feats, valid, plane
        self.n = int((np.asarray(valid) != 0).sum())
        self._cache = {}

    def at(self, x):
        key = np.asarray(x, np.float64).tobytes()
        if key not in self._cache:
            J, r, half, outer = rows(self.feats, self.valid, self.plane, x)
            S, A = sums(J, r, half)
            self._cache[key] = dict(S=S, A=A, dS=reduction_bound(self.n, A), J=J, r=r, outer=outer)
        return self._cache[key]


def minimiser(P, x, steps=30):
    """Newton's method on the fsum sums (Plus of the full step) until the step stops shrinking: the minimiser to rounding."""
    x = np.array(x, np.float64)
    for _ in range(steps):
        H, g = unpack(P.at(x)["S"])
        d = -np.linalg.solve(H, g)
        x = plus(x, d)
        if np.abs(d).max() < 1e-15:
            break
    return x


def _ldl(A):
    n = len(A)
    L = np.eye(n); D = np.zeros(n)
    for j in range(n):
        D[j] = A[j, j] - np.sum(L[j, :j] ** 2 * D[:j])
        for i in range(j + 1, n):
            L[i, j] = (A[i, j] - np.sum(L[i, :j] * L[j, :j] * D[:j])) / D[j] if D[j] != 0 else np.inf
    return L, D


def _gnorm(x, g, ambient):
    if not ambient:
        return float(np.max(np.abs(g)))
    return float(np.max(np.abs(np.asarray(x) - plus(x, -np.asarray(g)))))


class State:
    def __init__(self, P, start, rules):
        self.P, self.rules = P, rules
        self.x = np.array(start, np.float64)
        e = P.at(self.x)
        H, _ = unpack(e["S"])
        self.scaling = 1.0 / (1.0 + np.sqrt(np.diag(H)))
        self.radius, self.df, self.reuse, self.diag = RADIUS0, 2.0, False, None
        self.last_ok = bool(rules["gradient_at_start"])
        self.it, self.invalid = 0, 0
        self.rel_r = 0.0        # relative uncertainty of the radius carried (from the relative decreases that set it)
        self.done = None        # stop reason


def _decide(rec, ov, name, value, thr, bound, le):
    """value <= thr (le) or value > thr; open when |value - thr| <= bound.  ov: overrides of open decisions by name."""
    out = (value <= thr) if le else (value > thr)
    margin = float(value - thr)
    is_open = bool(np.isfinite(bound) and abs(margin) <= bound) or not np.isfinite(margin)
    if is_open and name in ov:
        out = ov[name]
    rec["decisions"].append(dict(name=name, value=float(value), threshold=float(thr), margin=margin, bound=float(bound),
                                 outcome=bool(out), open=is_open))
    if is_open:
        rec["open"].append(name)
    return out


def iterate(st: State, ov=None, solver="normal"):
    """One pass of the loop from st (not modified): returns (next state, record).  record: it, x_before, x_after, branch
    (accepted / rejected / invalid / None), stop (one of STOPS / None), pre (stopped before counting an iteration),
    the step by both solvers, both model cost changes, the one-step bound, decisions and the names of the open ones."""
    ov = ov or {}
    s = copy.copy(st)
    R = s.rules
    e = s.P.at(s.x)
    S, dS = e["S"], e["dS"]
    rec = dict(it=s.it + 1, x_before=s.x.copy(), x_after=s.x.copy(), branch=None, stop=None, pre=False, radius=s.radius,
               decrease_factor=s.df, decisions=[], open=[])
    if not S[28] > 0:
        s.done = rec["stop"] = "no_correspondences"; rec["pre"] = True; rec["it"] = s.it
        return s, rec
    if s.it >= s.P_max:
        s.done = rec["stop"] = "iteration_cap"; rec["pre"] = True; rec["it"] = s.it
        return s, rec
    H, g = unpack(S)
    if s.last_ok:
        gn = _gnorm(s.x, g, R["gradient_ambient"])
        gb = float(np.max(dS[21:27])) + PLUS_ULPS * U * max(1.0, float(np.abs(s.x).max()))
        if _decide(rec, ov, "gradient", gn, GRADIENT_TOL, gb, True):
            s.done = rec["stop"] = "gradient"; rec["pre"] = True; rec["it"] = s.it
            return s, rec
    if s.radius < MIN_RADIUS:
        s.done = rec["stop"] = "radius_floor"; rec["pre"] = True; rec["it"] = s.it
        return s, rec
    s.it += 1
    s.last_ok = False
    sc = s.scaling
    Hs = H * np.outer(sc, sc); gs = g * sc
    if not s.reuse:
        s.diag = np.clip(np.diag(Hs), MIN_DIAG, MAX_DIAG)
    s.reuse = True
    Dd = s.diag / s.radius
    A = Hs + np.diag(Dd)
    Js = e["J"] * sc[None, :]
    try:
        y_n = np.linalg.solve(A, gs)
    except np.linalg.LinAlgError:
        y_n = np.full(6, np.nan)
    aug = np.vstack([Js, np.diag(np.sqrt(Dd))])
    y_q = np.linalg.lstsq(aug, np.concatenate([e["r"], np.zeros(6)]), rcond=None)[0]
    y = y_n if solver == "normal" else y_q
    ok = bool(np.all(np.isfinite(y)))
    step = -y
    half = 0.5 if R["mcc_half"] else 1.0
    mcc_n = -(step @ gs + half * step @ Hs @ step)
    mcc_nb = gamma(14) * (np.abs(step) @ np.abs(gs) + 0.5 * np.abs(step) @ np.abs(Hs) @ np.abs(step)) + \
        np.abs(step) @ (dS[21:27] * sc) + 0.5 * np.abs(step) @ (np.abs(unpack(dS)[0]) * np.outer(sc, sc)) @ np.abs(step)
    mr = Js @ step
    mcc_q = -math.fsum(mr * (e["r"] + half * mr))
    mcc_qb = gamma(8) * float(np.sum(np.abs(mr) * (np.abs(e["r"]) + 0.5 * np.abs(mr))))
    mcc, mcc_b = (mcc_n, mcc_nb) if solver == "normal" else (mcc_q, mcc_qb)
    # the one-step bound: the reduction's sums error, LDL^T's backward error, the radius carried
    dH, dg = unpack(dS)
    dHs = dH * np.outer(sc, sc)
    dA = np.linalg.norm(dHs) + float(np.max(np.diag(dHs))) / s.radius
    Ainv = np.linalg.norm(np.linalg.inv(A), 2) if ok else np.inf
    Lf, Df = _ldl(A)
    bwd = gamma(3 * 6 + 1) * np.linalg.norm(np.abs(Lf) @ np.diag(np.abs(Df)) @ np.abs(Lf).T)
    dy = Ainv * (np.linalg.norm(dg * sc) + (dA + bwd) * np.linalg.norm(y)) + \
        (np.linalg.norm(np.linalg.solve(A, Dd * y)) * s.rel_r if ok else np.inf)
    delta = step * sc
    step_bound = float(np.max(sc) * dy + PLUS_ULPS * U * max(1.0, float(np.linalg.norm(s.x[4:]) + np.linalg.norm(delta[3:]))))
    rec.update(y_normal=y_n, y_qr=y_q, mcc_normal=float(mcc_n), mcc_qr=float(mcc_q), mcc_bound=float(mcc_b),
               mcc_normal_bound=float(mcc_nb), mcc_qr_bound=float(mcc_qb),
               mcc_disagree=bool((mcc_n > 0) != (mcc_q > 0)), step_bound=step_bound, cond=float(np.linalg.cond(A)),
               cond_aug=float(np.linalg.cond(aug)), y_bound=float(dy))
    valid = ok and _decide(rec, ov, "valid", mcc, 0.0, mcc_b, False)
    if not valid:
        s.invalid += 1
        rec["branch"] = "invalid"
        if s.invalid >= MAX_INVALID:
            s.done = rec["stop"] = "five_invalid"
            return s, rec
        if R["invalid"] == "ceres":
            s.radius /= s.df; s.df *= 2.0
        elif R["invalid"] == "halve":
            s.radius *= 0.5; s.reuse = False
        # "keep": the radius left as it was (a planted fault)
        return s, rec
    s.invalid = 0
    xc = plus(s.x, delta)
    ec = s.P.at(xc)
    rec["candidate"] = xc
    xn = float(np.linalg.norm(s.x)); sn = float(np.linalg.norm(s.x - xc))
    if _decide(rec, ov, "parameter", sn, PARAMETER_TOL * (xn + PARAMETER_TOL), step_bound * math.sqrt(7) + 4 * U * xn, True):
        s.done = rec["stop"] = "parameter"
        return s, rec
    cost, cc_cost = S[27], ec["S"][27]
    cc = cost - cc_cost
    gc = np.linalg.norm(ec["S"][21:27])
    cc_b = dS[27] + ec["dS"][27] + 2 * U * (abs(cost) + abs(cc_cost)) + gc * step_bound * math.sqrt(7) + \
        0.5 * np.linalg.norm(unpack(ec["S"])[0], 2) * 7 * step_bound ** 2
    if _decide(rec, ov, "function", abs(cc), FUNCTION_TOL * cost, cc_b + FUNCTION_TOL * dS[27], True):
        s.done = rec["stop"] = "function"
        return s, rec
    rd = cc / mcc
    # rounding of the relative decrease at this candidate, and (for a decision) the candidate's own uncertainty on top
    rd_round = (dS[27] + ec["dS"][27] + 2 * U * (abs(cost) + abs(cc_cost)) + abs(rd) * mcc_b) / abs(mcc) + 4 * U * abs(rd)
    rd_b = rd_round + (cc_b - dS[27] - ec["dS"][27] - 2 * U * (abs(cost) + abs(cc_cost))) / abs(mcc)
    rec.update(relative_decrease=float(rd), rd_bound=float(rd_b), rd_round=float(rd_round), cost_change=float(cc),
               rel_r=s.rel_r, mcc=float(mcc), cost=float(cost), dcost=float(dS[27]),
               dmcc_step=float(np.linalg.norm(Dd * y) * dy + 0.5 * np.linalg.norm(A, 2) * dy ** 2))
    if _decide(rec, ov, "accept", rd, MIN_REL_DECREASE, rd_b, False):
        rec["branch"] = "accepted"
        s.x = xc
        s.last_ok = True
        if R["rescale_each_accept"]:
            Hn, _ = unpack(ec["S"])
            s.scaling = 1.0 / (1.0 + np.sqrt(np.diag(Hn)))
        s.radius, s.rel_r = _grow(R, rec["radius"], s.rel_r, rd, rd_round)
        s.df = 2.0 if R["reset_df"] else s.df
        s.reuse = False
        rec["x_after"] = xc.copy()
    else:
        rec["branch"] = "rejected"
        if R["reject_div"] is not None:
            s.radius /= R["reject_div"]
        else:
            s.radius /= s.df
        if R["reject_double"]:
            s.df *= 2.0
        s.reuse = True
    return s, rec


def _grow(R, radius, rel_r, rd, rd_b):
    """StepAccepted: radius / max(1/3, 1 - (2 rd - 1)^3), at most 1e16.  The radius's relative uncertainty grows by the rule's
    sensitivity 6 (2 rd - 1)^2 / (1 - (2 rd - 1)^3) times rd's ROUNDING bound rd_b.  Only rounding: the relative decrease that
    sets a device's radius is the one at the device's own accepted iterate, which follow() knows (it is x_j), so the candidate's
    position uncertainty never enters the radius and the bound cannot feed on itself."""
    qd = 2 * rd - 1
    den = 1 - qd ** 3
    if den > 1 / 3:
        rel_r += 6 * qd ** 2 / den * rd_b
    return min(MAX_RADIUS, radius / max(1 / 3, den) if R["grow"] is None else R["grow"](radius, rd)), rel_r


def _start(feats, valid, plane, start, max_num_iter, rules):
    P = Problem(feats, valid, plane)
    st = State(P, start, dict(CERES, **(rules or {})))
    st.P_max = max_num_iter
    return st


State.P_max = 15


def run(feats, valid, plane, start, max_num_iter=15, solver="normal", rules=None, ov_seq=None):
    """One trace: at every open decision the nominal outcome unless ov_seq (a list of dicts, one per iteration) overrides it.
    Returns dict(iters, stop, x (unified), records)."""
    st = _start(feats, valid, plane, start, max_num_iter, rules)
    recs = []
    while st.done is None:
        ov = ov_seq[len(recs)] if ov_seq and len(recs) < len(ov_seq) else None
        st, rec = iterate(st, ov, solver)
        recs.append(rec)
    return dict(iters=st.it, stop=st.done, x=unify(st.x), records=recs)


def traces(feats, valid, plane, start, max_num_iter=15, solver="normal", rules=None, cap=64):
    """Every admissible trace: both outcomes at every open decision (depth-first, at most `cap` traces)."""
    out, stack = [], [[]]
    while stack and len(out) < cap:
        seq = stack.pop()
        t = run(feats, valid, plane, start, max_num_iter, solver, rules, seq)
        out.append(t)
        for i in range(len(seq), len(t["records"])):
            rec = t["records"][i]
            for name in rec["open"]:
                taken = next(d["outcome"] for d in rec["decisions"] if d["name"] == name)
                pre = [dict((dd["name"], dd["outcome"]) for dd in r["decisions"] if dd["open"]) for r in t["records"][:i]]
                cur = dict((dd["name"], dd["outcome"]) for dd in rec["decisions"] if dd["open"] and dd["name"] != name)
                cur[name] = not taken
                stack.append(pre + [cur])
    return out


def open_decisions(trace):
    return [(r["it"], d) for r in trace["records"] for d in r["decisions"] if d["open"]]


class TraceError(AssertionError):
    pass


def follow(feats, valid, plane, start, iterates, stop_iter, max_num_iter=15, rules=None):
    """The per-iteration check of one device solve on frozen correspondences.

    iterates[j] is the device's iterate after j iterations (the pose its call with max_num_iter = j returned; iterates[0] is
    the start) for j = 0 .. stop_iter (+1 if available); stop_iter is the device's iteration count of the uncapped call.  The
    reference's trust-region state is carried along the DEVICE's iterates: at iteration j the reference computes its step from
    x_{j-1}; an unmoved x_j is a rejected or invalid step or a stop, a moved one an accepted step, which must lie within the
    one-step bound of the reference's candidate.  A closed decision must match the device's; at an open one the outcome the
    device shows is taken.  Raises TraceError; returns dict(records, ratio (largest deviation / bound), branches, stop)."""
    st = _start(feats, valid, plane, start, max_num_iter, rules)
    recs, ratio, worst = [], 0.0, (0.0, 0.0)
    while st.done is None:
        j = st.it + 1
        moved = None
        if j < len(iterates):
            moved = not np.array_equal(np.asarray(iterates[j]), np.asarray(iterates[j - 1]))
        want_stop_before = stop_iter == j - 1
        # enumerate overrides of this iteration's open decisions until one agrees with what the device shows
        nxt, rec = iterate(st, None)
        cands = [(nxt, rec)]
        if rec["open"]:
            names = rec["open"]
            for mask in range(1, 2 ** len(names)):
                base = {d["name"]: d["outcome"] for d in rec["decisions"] if d["open"]}
                ov = {n: (not base[n]) if (mask >> i) & 1 else base[n] for i, n in enumerate(names)}
                cands.append(iterate(st, ov))
        chosen = None
        for n_, r_ in cands:
            if r_["pre"]:
                ok = want_stop_before
            else:
                is_moved = r_["branch"] == "accepted"
                ok = (moved is None or moved == is_moved) and (stop_iter == j if r_["stop"] is not None else stop_iter >= j)
            if ok:
                chosen = (n_, r_)
                break
        if chosen is None:
            dev = "stopped" if want_stop_before else ("moved" if moved else "kept its pose") + \
                (" and stopped" if stop_iter == j else "")
            raise TraceError(f"LM iteration {j}: the device {dev}, the reference takes {rec['branch'] or rec['stop']}"
                             f" (decisions {[(d['name'], d['outcome'], d['margin'], d['bound']) for d in rec['decisions']]})")
        st, rec = chosen
        if rec["branch"] == "accepted" and moved:
            x_dev = unify(iterates[j])
            want = unify(rec["candidate"])
            dev = float(np.abs(x_dev - want).max())
            if not dev <= rec["step_bound"]:
                raise TraceError(f"LM iteration {j}: accepted step differs from the reference's by {dev:.3e} > "
                                 f"{rec['step_bound']:.3e}\n  device {x_dev.tolist()}\n  ref    {want.tolist()}")
            rec["dev"] = dev
            rec["dev_qr"] = float(np.abs(x_dev - unify(plus(rec["x_before"], -rec["y_qr"] * st.scaling))).max())
            if dev / rec["step_bound"] > ratio:
                ratio = dev / rec["step_bound"]
                worst = (dev, rec["step_bound"])
            # carry the state along the device's own iterate: x, and the radius from the relative decrease AT x_j (the device's
            # step moves its model cost change by at most dmcc_step); the device accepted, so that decrease must admit it
            st.x = np.array(iterates[j], np.float64)
            e_dev = st.P.at(st.x)
            cost_dev = e_dev["S"][27]
            rd_dev = (rec["cost"] - cost_dev) / rec["mcc"]
            rd_dev_b = (rec["dcost"] + e_dev["dS"][27] + 2 * U * (abs(rec["cost"]) + abs(cost_dev)) +
                        abs(rd_dev) * (rec["mcc_bound"] + rec["dmcc_step"])) / abs(rec["mcc"]) + 4 * U * abs(rd_dev)
            if not rd_dev + rd_dev_b > MIN_REL_DECREASE:
                raise TraceError(f"LM iteration {j}: the device accepted a step whose relative decrease at its own iterate is "
                                 f"{rd_dev:.6e} (+- {rd_dev_b:.2e}), not above {MIN_REL_DECREASE}")
            st.radius, st.rel_r = _grow(st.rules, rec["radius"], rec["rel_r"], rd_dev, rd_dev_b)
            rec["rd_device"], rec["rd_device_bound"] = float(rd_dev), float(rd_dev_b)
        recs.append(rec)
    if st.it != stop_iter:
        raise TraceError(f"the device takes {stop_iter} LM iterations, the reference along its iterates {st.it}")
    return dict(records=recs, ratio=ratio, dev=worst[0], bound=worst[1], stop=st.done,
                branches=[r["branch"] for r in recs if r["branch"]])
