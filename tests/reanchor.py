"""Re-anchored pass check of the scan-to-map solve: every pass of one device call re-run on the CPU from the device's own start pose.

A trajectory check (each pass's pose within 1e-4 of the oracle's) cannot see a step that is a little wrong: Gauss-Newton and LM
re-linearise at the next pass and converge to the same fixed point anyway.  This checker takes the per-pass stats of ONE call
(liliom_iter_stats: n_corr, lm_iters, cost, the 27 sums, the pose after the pass) and re-runs each pass k from the pose the device
started it from: the guess for k = 0, st[k-1].pose7 after that.  So every pass is compared with an independent fp64 computation of
that pass alone, and an error in one pass cannot hide behind the passes after it.

GN mode (check_gn), every pass k from start_k:
  (a) oracle.find_surf_corr at start_k: its count equals st[k].n_corr exactly (both sides transform with the same non-contracted
      fp64 expression, so at the same pose every accept decision is the same);
  (b) oracle.normal_equations at start_k equals st[k].jtj_jtr and the cost at rtol 1e-9, the suite's level for sums.  Given a
      probe of the device's own correspondences at a pose (the GPU tier passes one), the sums are reduced by the oracle from the
      device's planes, and those planes are held to the oracle's first: accept flags exact, planes at rtol 2e-6 (see _oracle_pass);
  (c) st[k].pose7 equals the GN step computed on the host from the device's OWN 29 sums and start_k, twice: with the host build of
      dev_math.cuh (gn_safe_step + pose_plus, tests/devmath_host.cpp) and with the NumPy restatement below.  Tolerance: see
      step_tolerance.
  (d) the branch the host took on every pass (plain, damped, clipped, refused) is reported, so a test can assert it was covered.

Ceres-faithful mode (check_ceres), every outer iteration k from start_k: the oracle's correspondences at start_k (count exact, sums
at rtol 1e-9; the device's planes when probed, as in (b)), then oracle.ceres_solve on them from start_k must take exactly
st[k].lm_iters iterations and land within ceres_tolerance of st[k].pose7.

Per LM iteration (check_ceres with `truncated`): a match_cnt = 1 call stops as soon as its iteration count reaches
max_num_iter and freezes its correspondences at its start, so the calls truncated(start_k, j) for j = 0 .. lm_iters + 1
return the device's iterate after each iteration, bit for bit the computation of the full pass.  lm_reference.follow carries
Ceres' trust-region state along those iterates: every decision (moved = accepted; unmoved = rejected, invalid or stopped)
must match an admissible reference trace, the stop iteration exactly, and every accepted step must land within the one-step
bound of the reference's candidate (the block reduction's gamma_d sum(|terms|) per scalar, the damped system's conditioning
and LDL^T's backward error, and the radius carried).  The distance from the QR step is reported next to it.

Both raise ReanchorError (an AssertionError) naming the pass and the check that failed, and return a report of the largest
deviations seen, each next to its bound.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

U = np.finfo(np.float64).eps / 2         # unit roundoff of fp64, 2^-53
SUMS_RTOL = SUMS_ATOL = 1e-9
GN_PIVOT_REL, GN_DAMP_REL, GN_MAX_ROT, GN_MAX_TRANS = 1e-10, 1e-6, 0.35, 5.0     # dev_math.cuh::gn_safe_step
STEP_ULPS = 32          # c * n * u with n = 6 and c = 2 for each of the two eliminations compared, rounded up to a power of two
PLUS_ULPS = 8           # rounding of Plus itself: a 4-term quaternion product and one addition per translation component
LM_ULPS = 64            # per LM step: normal equations by LDL^T (device) against the augmented system by Householder QR (oracle)


class ReanchorError(AssertionError):
    pass


def _fail(msg):
    raise ReanchorError(msg)


def start_poses(guess, st):
    """The pose the device started each pass from: the guess, then the pose the previous pass wrote."""
    return [np.asarray(guess, np.float64)] + [np.array(s.pose7, np.float64) for s in st[:-1]]


def sums29(s):
    """The 29 scalars of one stats row in normal_equations order: 21 upper-triangle J^T J, 6 J^T r, cost, count."""
    return np.array(list(s.jtj_jtr) + [s.cost, float(s.n_corr)], np.float64)


def unpack(s29):
    H = np.zeros((6, 6))
    H[np.triu_indices(6)] = s29[:21]
    H = H + np.triu(H, 1).T
    return H, np.asarray(s29[21:27], np.float64)


def unify(x):
    """LidarOdometry.cpp:539-549: the quaternion with w >= 0."""
    x = np.array(x, np.float64)
    if x[0] < 0:
        x[:4] = -x[:4]
    return x


def ceres_plus(x, d):
    """ceres::QuaternionParameterization::Plus on q, identity on t (restated from knowledge, as in test_oracle_cpu.py)."""
    nd = np.linalg.norm(d[:3])
    out = np.array(x, np.float64)
    if nd > 0:
        aw, ax, ay, az = np.cos(nd), *(np.sin(nd) / nd * np.asarray(d[:3]))
        bw, bx, by, bz = x[:4]
        out[:4] = [aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                   aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx]
    out[4:] = np.asarray(x[4:]) + d[3:]
    return out


def _ldl_pivots(A):
    """Pivots of the unpivoted LDL^T of A, in the order dev_math.cuh::solve6_ldlt forms them."""
    n = len(A)
    L = np.eye(n); D = np.zeros(n)
    for j in range(n):
        D[j] = A[j, j] - np.sum(L[j, :j] ** 2 * D[:j])
        for i in range(j + 1, n):
            L[i, j] = (A[i, j] - np.sum(L[i, :j] * L[j, :j] * D[:j])) / D[j] if D[j] != 0 else np.inf
    return D


def _pivots_ok(A, piv_min):
    D = _ldl_pivots(A)
    return bool(np.all(np.isfinite(D)) and np.all(np.abs(D) > 1e-300) and (piv_min < 0 or np.all(D > piv_min)))


def gn_step(s29, start):
    """The GN pass's step restated in NumPy (the rules test_gn_safe_step_device_copy states): plain solution of H d = -g; the
    Levenberg-damped system H + 1e-6 max diag(H) I when a pivot is not above 1e-10 max diag(H); the step scaled back onto
    0.35 rad / 5 m; refused (pose kept) on a zero or non-finite system or without correspondences.  Returns
    (pose after the pass, branch, d, the solved system A)."""
    H, g = unpack(s29)
    maxd = float(np.max(np.diag(H)))
    if not (maxd > 0.0) or not np.isfinite(maxd) or not np.all(np.isfinite(s29[:27])):
        return unify(start), "refused", np.zeros(6), None
    A, branch = H, "plain"
    if not _pivots_ok(H, GN_PIVOT_REL * maxd):
        A, branch = H + GN_DAMP_REL * maxd * np.eye(6), "damped"
        if not _pivots_ok(A, 0.0):
            return unify(start), "refused", np.zeros(6), None
    d = np.linalg.solve(A, -g)
    if not np.all(np.isfinite(d)):
        return unify(start), "refused", np.zeros(6), None
    rot, tr = np.linalg.norm(d[:3]), np.linalg.norm(d[3:])
    sc = 1.0
    if rot > GN_MAX_ROT:
        sc = GN_MAX_ROT / rot
    if tr * sc > GN_MAX_TRANS:
        sc = GN_MAX_TRANS / tr
    if sc < 1.0:
        d = d * sc
        branch = "clipped" if branch == "plain" else branch + "+clipped"
    if not s29[28] > 0:
        return unify(start), "empty", d, A
    return unify(ceres_plus(start, d)), branch, d, A


def step_tolerance(start, d, A):
    """Per-component bound on |device pose - host pose| for one GN pass, derived, not tuned.

    The device and the host solve the same system A d = -g (A = H, or H + lambda I on the damped branch) from the SAME 29 sums,
    by the same unpivoted LDL^T; only the rounding differs (grid_knn.cu is built with FMA contraction, the host builds are not,
    and NumPy solves by pivoted LU).  Each elimination is backward stable on this SPD system, so each computed step is within
    c * n * u * cond(A) * |d| of the exact one at first order (n = 6, u = 2^-53, c a small constant); two of them differ by at
    most twice that, which STEP_ULPS * u * cond(A) * |d| covers with c = 2.  The trust-region scale 0.35 / |d_rot| adds a
    relative O(u) and the sign rule is exact.  Plus is 1-Lipschitz in d for a unit quaternion, so the step error passes to the
    pose unamplified, and Plus adds its own rounding: PLUS_ULPS * u relative to the larger of 1 and the translation.  (The
    Taylor series of the device's Plus truncates below 1e-22.)"""
    if A is None:
        return PLUS_ULPS * U * max(1.0, float(np.abs(start).max()))
    return STEP_ULPS * U * float(np.linalg.cond(A)) * float(np.linalg.norm(d)) + \
        PLUS_ULPS * U * max(1.0, float(np.linalg.norm(start[4:]) + np.linalg.norm(d[3:])))


def devmath_step(dm, s29, start):
    """The same pass through the host build of dev_math.cuh: gn_safe_step + pose_plus + the sign rule of grid_knn.cu::gn_step."""
    dp = C.POINTER(C.c_double)
    s21 = np.ascontiguousarray(s29[:21], np.float64)
    nb = np.ascontiguousarray(-np.asarray(s29[21:27], np.float64))
    d = np.zeros(6); out = np.zeros(7)
    x = np.ascontiguousarray(start, np.float64)
    ok = dm.dm_gn_safe_step(s21.ctypes.data_as(dp), nb.ctypes.data_as(dp), d.ctypes.data_as(dp))
    if s29[28] > 0 and ok:
        dm.dm_pose_plus(x.ctypes.data_as(dp), d.ctypes.data_as(dp), out.ctypes.data_as(dp))
    else:
        out[:] = x
    return unify(out)


def _check_sums(k, got, want, what):
    """At rtol 1e-9 (plus atol 1e-9 for the scalars near zero), the suite's level for sums.  Returns the largest deviation as a
    share of that bound."""
    err = np.abs(got - want)
    lim = SUMS_ATOL + SUMS_RTOL * np.abs(want)
    if not np.all(err <= lim):
        j = int(np.argmax(err / lim))
        _fail(f"{what} pass {k}: sums differ from the oracle's at the device's start pose: scalar {j} {got[j]!r} vs {want[j]!r}")
    return float(np.max(err / lim))


def normwise_deviation(got, want):
    """The relative perturbation of the linear system the sums describe: max(|dH|_F / |H|_F, |dg| / |g|), at least u."""
    def rel(a, b):
        nb = float(np.linalg.norm(b))
        return float(np.linalg.norm(a - b)) / nb if nb > 0 else (0.0 if not np.any(a - b) else np.inf)
    return max(rel(got[:21], want[:21]), rel(got[21:27], want[21:27]), U)


def _oracle_pass(oracle, tree, feats, start, st_k, k, nthreads, what, probe, rep):
    """(a) and (b) of one pass.  Returns the correspondences the pass's sums are held to (the device's planes when `probe` is
    given) and the normwise deviation of the pass's sums from their fp64 reduction."""
    cnt, valid, plane, _, _ = oracle.find_surf_corr(tree, feats, start, nthreads)
    if cnt != st_k.n_corr:
        _fail(f"{what} pass {k}: n_corr {st_k.n_corr} but the oracle finds {cnt} correspondences at the device's start pose")
    got = sums29(st_k)
    if probe is not None:
        # The device fits each plane by its closed form and the oracle by column-pivoting QR, both in fp64, and both store it in
        # fp32: a coefficient can land one fp32 rounding apart.  Over 10^4..10^5 correspondences near convergence, where J^T r is
        # a small difference of large terms, those roundings move a sum by more than 1e-9 of its value.  So the sums are held to
        # the oracle's fp64 reduction of the DEVICE's correspondences, and those to the oracle's: accept flags exact, planes at
        # the suite's plane tolerance (rtol 2e-6, atol 1e-7).  The sums' distance from the oracle's own reduction is reported
        # (sum_ratio_oracle_planes: the largest deviation as a share of the 1e-9 bound), not asserted.
        v_d, pl_d = probe(start)
        if not np.array_equal(v_d, valid):
            bad = np.nonzero(v_d != valid)[0]
            _fail(f"{what} pass {k}: accept flags differ from the oracle's at the device's start pose at {len(bad)} queries {bad[:5]}")
        close = np.abs(pl_d - plane) <= 1e-7 + 2e-6 * np.abs(plane)
        if not close.all():
            bad = np.nonzero(~close.all(1))[0]
            _fail(f"{what} pass {k}: planes differ from the oracle's at {len(bad)} queries {bad[:5]}")
        want_o = oracle.normal_equations(feats, valid, plane, start)
        ratio_o = float(np.max(np.abs(got[:28] - want_o[:28]) / (SUMS_ATOL + SUMS_RTOL * np.abs(want_o[:28]))))
        rep["sum_ratio_oracle_planes"] = max(rep.get("sum_ratio_oracle_planes", 0.0), ratio_o)
        plane = pl_d
    want = oracle.normal_equations(feats, valid, plane, start)
    rep["sum_ratio"] = max(rep["sum_ratio"], _check_sums(k, got[:28], want[:28], what))
    return valid, plane, normwise_deviation(got, want)


def check_gn(oracle, tree, feats, guess, st, dm, nthreads=1, what="GN", probe=None):
    """Check every pass of one GN-mode call (see the module docstring).  probe(pose) -> (accept flags, planes): the device's own
    correspondences at a pose (see _oracle_pass).  Returns a report: per-pass branches, the largest sum deviation as a share of its
    bound, and the largest step deviation of each host computation with the bound it was held to."""
    rep = dict(branches=[], sum_ratio=0.0, step_dev=0.0, step_bound=0.0, step_ratio=0.0, n_corr=[s.n_corr for s in st])
    for k, (start, s) in enumerate(zip(start_poses(guess, st), st)):
        _oracle_pass(oracle, tree, feats, start, s, k, nthreads, what, probe, rep)
        s29 = sums29(s)
        want, branch, d, A = gn_step(s29, start)
        tol = step_tolerance(start, d, A)
        got = np.array(s.pose7, np.float64)
        for name, ref in (("NumPy", want), ("dev_math host build", devmath_step(dm, s29, start))):
            dev = float(np.abs(got - ref).max())
            if not dev <= tol:
                _fail(f"{what} pass {k} ({branch}): pose differs from the {name} step on the device's own sums by {dev:.3e} > {tol:.3e}"
                      f"\n  device {got.tolist()}\n  host   {ref.tolist()}")
            if dev > rep["step_dev"]:
                rep["step_dev"], rep["step_bound"] = dev, tol
            rep["step_ratio"] = max(rep["step_ratio"], dev / tol)
        rep["branches"].append(branch)
    return rep


def ceres_tolerance(start, pose_o, s29, lm_iters, e):
    """Bound on |device pose - oracle pose| after one outer iteration of the Ceres-faithful mode, derived, not tuned.

    Both run the same Levenberg-Marquardt loop on the same frozen correspondences (the device's own, when probed) from the same
    start and take the same accept / reject decisions (lm_iters is compared exactly).  What differs: (1) the device's sums, a
    relative perturbation e of the system measured at the start (normwise_deviation against the fp64 reduction of the same
    correspondences: only the summation order differs), taken as the perturbation at every iterate of the loop; (2) each step,
    solved by LDL^T on the damped scaled normal equations on the device and by Householder QR on the augmented Jacobian in the
    oracle, LM_ULPS * u relative apart.  A relative perturbation of the system moves its solution by at most 2 (e + LM_ULPS u)
    cond(H) |step| at first order (damping only lowers the condition number, so cond of the undamped H at start_k bounds every
    step's).  Summed over the lm_iters steps, each taken no longer than the whole move |pose_o - start| (no step overshoots the
    minimum), plus the rounding of Plus.  On a rank-deficient H (one feature, a single plane) cond(H) is unbounded and so is this
    bound: there the iteration count and the sums are what bind."""
    H, _ = unpack(s29)
    move = float(np.linalg.norm(np.asarray(pose_o) - np.asarray(start)))
    kappa = float(np.linalg.cond(H)) if np.all(np.isfinite(H)) and np.any(H) else 1.0
    return max(lm_iters, 1) * 2 * (e + LM_ULPS * U) * kappa * move + \
        PLUS_ULPS * U * max(lm_iters, 1) * max(1.0, float(np.linalg.norm(np.asarray(start)[4:])) + move)


def trace_pass(feats, valid, plane, start, lm_iters, truncated, max_num_iter, k, what, rep):
    """The per-iteration check of one outer pass (see the module docstring): truncated(start, j) -> (pose after j LM
    iterations, the call's iteration count)."""
    import lm_reference as LR
    iterates = [np.asarray(start, np.float64)]
    for j in range(1, lm_iters + 2):
        if j > max_num_iter:
            break
        pose, it = truncated(start, j)
        if it != min(j, lm_iters):
            _fail(f"{what} pass {k}: the call capped at {j} LM iterations reports {it}, the uncapped one {lm_iters}")
        iterates.append(np.asarray(pose, np.float64))
    try:
        tr = LR.follow(feats, valid, plane, start, iterates, lm_iters, max_num_iter)
    except LR.TraceError as e:
        _fail(f"{what} pass {k}: trace: {e}")
    rep["trace_ratio"] = max(rep.get("trace_ratio", 0.0), tr["ratio"])
    if tr["ratio"] >= rep.get("trace_ratio", 0.0):
        rep["trace_dev"], rep["trace_bound"] = tr["dev"], tr["bound"]
    rep.setdefault("branches", []).extend(tr["branches"])
    rep.setdefault("stops", []).append(tr["stop"])
    qr = [r["dev_qr"] for r in tr["records"] if "dev_qr" in r]
    if qr:
        rep["qr_dev"] = max(rep.get("qr_dev", 0.0), max(qr))
        # what a QR solve itself meets on the augmented system: u (kappa + kappa^2 |res| / (|A| |y|)) |y|, first order
        rep["qr_bound"] = max(rep.get("qr_bound", 0.0), max(U * (r["cond_aug"] + r["cond_aug"] ** 2) * float(np.linalg.norm(r["y_qr"]))
                                                              for r in tr["records"] if "dev_qr" in r))
    acc = [r for r in tr["records"] if r["branch"] == "accepted" and "candidate" in r]
    rep["bound_over_step"] = max([rep.get("bound_over_step", 0.0)] +
                                 [r["step_bound"] / max(float(np.linalg.norm(r["candidate"] - r["x_before"])), 1e-300) for r in acc])
    rep["mcc_gap"] = max([rep.get("mcc_gap", 0.0)] + [abs(r["mcc_normal"] - r["mcc_qr"]) / abs(r["mcc_normal"])
                                                      for r in tr["records"] if "mcc_qr" in r and r["mcc_normal"] != 0])
    rep["open_decisions"] = rep.get("open_decisions", 0) + sum(len(r["open"]) for r in tr["records"])
    rep["step_bound_sum"] = max(rep.get("step_bound_sum", 0.0), sum(r.get("step_bound", 0.0) for r in tr["records"] if r["branch"] == "accepted"))
    return tr


def check_ceres(oracle, tree, feats, guess, st, max_num_iter, nthreads=1, what="CERES", probe=None, truncated=None,
                trace_passes=None):
    """Check every outer iteration of one Ceres-faithful call.  Returns the largest sum deviation as a share of its bound and the
    largest pose deviation with the bound it was held to.  With truncated(start, j) (the device's match_cnt = 1 call capped at
    j LM iterations from `start`), the passes in trace_passes (all by default) are also checked iteration by iteration."""
    rep = dict(sum_ratio=0.0, pose_dev=0.0, pose_bound=0.0, pose_ratio=0.0, lm_iters=[s.lm_iters for s in st])
    for k, (start, s) in enumerate(zip(start_poses(guess, st), st)):
        valid, plane, e = _oracle_pass(oracle, tree, feats, start, s, k, nthreads, what, probe, rep)
        it, pose_o, _ = oracle.ceres_solve(feats, valid, plane, start, max_num_iter)
        pose_o = unify(pose_o)
        if it != s.lm_iters:
            _fail(f"{what} pass {k}: {s.lm_iters} LM iterations but the oracle's LM from the device's start pose takes {it}")
        got = np.array(s.pose7, np.float64)
        tol = ceres_tolerance(start, pose_o, sums29(s), it, e)
        dev = float(np.abs(got - pose_o).max())
        if not dev <= tol:
            _fail(f"{what} pass {k}: pose differs from the oracle's LM from the device's start pose by {dev:.3e} > {tol:.3e}"
                  f"\n  device {got.tolist()}\n  oracle {pose_o.tolist()}")
        if dev > rep["pose_dev"]:
            rep["pose_dev"], rep["pose_bound"] = dev, tol
        rep["pose_ratio"] = max(rep["pose_ratio"], dev / tol)
        if truncated is not None and (trace_passes is None or k in trace_passes):
            trace_pass(feats, valid, plane, start, s.lm_iters, truncated, max_num_iter, k, what, rep)
    return rep
