"""CPU tier of the per-iteration LM check: the NumPy restatement of Ceres' trust-region loop (tests/lm_reference.py) against the
oracle's LM on every adversarial world (tests/lm_adversarial.py) and on the horizon_ds world, its fsum sums against the oracle's,
every world's branch clear of its threshold, and the trace checker (lm_reference.follow) accepting the oracle's own truncated
solves and rejecting each planted fault of a rewrite of the trust-region bookkeeping, with a note of which of those faults the
end-of-pass check (reanchor.check_ceres) would have let through."""
import numpy as np
import pytest

import lm_adversarial as LA
import lm_reference as LR
import reanchor as RA
from test_reanchor_cpu import PLANE_WORLDS

NAMES = list(LA.WORLDS)


@pytest.fixture(scope="module")
def worlds(oracle):
    """name -> (feats, valid, plane, guess, max_num_iter): the correspondences the oracle finds at each world's guess."""
    out = {}
    for name, (fn, mni, _, _) in LA.WORLDS.items():
        m, q, g = fn()
        cnt, v, pl, _, _ = oracle.find_surf_corr(oracle.KdTree(m), q, g)
        out[name] = (q, v, pl, g, mni)
    from liliom_b200 import synth
    m, _ = synth.make_map(100_000, seed=20260923)
    T = synth.default_true_pose()
    pts, qi = synth.make_horizon_sweep(T)
    surf, _, _ = oracle.extract_horizon(pts, qi)
    ds, g = oracle.voxelgrid(surf, 0.4), synth.perturbed_pose(T)
    cnt, v, pl, _, _ = oracle.find_surf_corr(oracle.KdTree(m), ds, g)
    out["horizon_ds"] = (ds, v, pl, g, 15)
    m, q, g = PLANE_WORLDS["tilted_flat_plane"][0]()
    _, v, pl, _, _ = oracle.find_surf_corr(oracle.KdTree(m), q, g)
    out["tilted_flat_plane"] = (q, v, pl, g, 15)
    return out


def _truncated(oracle, feats, valid, plane, start, max_num_iter):
    """The oracle's solve capped at j = 0 .. its iteration count + 1 (the iterates a device trace check reads)."""
    n, _, _ = oracle.ceres_solve(feats, valid, plane, start, max_num_iter)
    its = [np.asarray(start, np.float64)]
    for j in range(1, min(n + 1, max_num_iter) + 1):
        its.append(RA.unify(oracle.ceres_solve(feats, valid, plane, start, j)[1]))
    return its, n


@pytest.mark.parametrize("name", NAMES + ["horizon_ds"])
def test_reference_matches_oracle(oracle, worlds, name):
    """The same iteration count and stop on every world, the pose within the reference's summed one-step bounds, and the fsum
    sums at the guess equal to the oracle's reduction at rtol 1e-9."""
    feats, v, pl, g, mni = worlds[name]
    t = LR.run(feats, v, pl, g, mni)
    it, pose, _ = oracle.ceres_solve(feats, v, pl, g, mni)
    assert it == t["iters"], (name, it, t["iters"], t["stop"])
    bound = sum(r.get("step_bound", 0.0) for r in t["records"] if r["branch"] == "accepted")
    # the oracle solves by QR and sums in order: its pose is within the QR steps' distance from the normal ones plus the bound
    qr_gap = sum(float(np.abs((r["y_qr"] - r["y_normal"])).max()) for r in t["records"] if r["branch"] == "accepted")
    assert np.abs(RA.unify(pose) - t["x"]).max() <= bound + qr_gap + RA.PLUS_ULPS * RA.U, name
    S = oracle.normal_equations(feats, v, pl, g)
    e = LR.Problem(feats, v, pl).at(g)
    assert np.all(np.abs(S[:28] - e["S"][:28]) <= 1e-9 + 1e-9 * np.abs(e["S"][:28])), name
    assert S[28] == e["S"][28]


@pytest.mark.parametrize("name", NAMES)
def test_world_takes_its_branch(worlds, name):
    """Every world's intended stop and branches with every decision of its trace closed (clear of its threshold by more than
    its rounding bound), and every accepted step's bound far below the step (bound / |step| < 1e-6: the bound stays a
    statement about rounding, not a licence); parameter_edge has exactly one open decision, genuinely at its threshold."""
    feats, v, pl, g, mni = worlds[name]
    t = LR.run(feats, v, pl, g, mni)
    _, _, stop, branches = LA.WORLDS[name]
    if stop:
        assert t["stop"] == stop, (name, t["stop"])
    got = [r["branch"] for r in t["records"]]
    for b in branches:
        assert b in got, (name, got)
    if name == "rotation":
        # two rejections in a row (decrease_factor doubles), acceptances after them
        assert any(a == b == "rejected" for a, b in zip(got, got[1:])), got
        assert any(r["decrease_factor"] == 4.0 for r in t["records"])
        assert got[0] == "rejected" and "accepted" in got
    ops = LR.open_decisions(t)
    if name == "parameter_edge":
        assert [(it, d["name"]) for it, d in ops] == [(1, "parameter")], ops
        d = ops[0][1]
        assert abs(d["margin"]) <= d["bound"] < 1e-6 * d["threshold"]
    else:
        assert not ops, (name, ops)
    for r in t["records"]:
        if r["branch"] == "accepted":
            assert r["step_bound"] < 1e-6 * np.linalg.norm(r["candidate"] - r["x_before"]), (name, r["it"])
    if name == "zero_residual":
        assert t["iters"] == 0 and np.array_equal(t["x"], g)
    if name == "gradient":
        assert t["iters"] == 1 and t["records"][-1]["decisions"][0]["value"] < 0.5 * LR.GRADIENT_TOL


@pytest.mark.parametrize("name", NAMES + ["horizon_ds"])
def test_model_cost_change_formulas(worlds, name, capsys):
    """The kernel's -(s.gs + s^T Hs s / 2) against Ceres' -(Js s).(r + Js s / 2) on every iteration: within the sum of their
    rounding bounds, never of different sign; the largest relative gap is printed."""
    feats, v, pl, g, mni = worlds[name]
    t = LR.run(feats, v, pl, g, mni)
    gap = 0.0
    for r in t["records"]:
        if "mcc_qr" in r:
            d = abs(r["mcc_normal"] - r["mcc_qr"])
            assert d <= r["mcc_normal_bound"] + r["mcc_qr_bound"], (name, r["it"], d)
            assert not r["mcc_disagree"]
            gap = max(gap, d / abs(r["mcc_normal"]))
    with capsys.disabled():
        print(f"\nmodel_cost_change {name}: largest |normal - qr| / |normal| = {gap:.2e}")


def test_admissible_traces_fork_at_open_decisions(oracle, worlds):
    """At parameter_edge's open decision both outcomes are followed: two admissible traces, the pose kept (parameter stop) or
    the step accepted (gradient stop after it).  A device showing either is accepted by follow, through its override path;
    a device that moved AND kept going is not admissible."""
    feats, v, pl, g, mni = worlds["parameter_edge"]
    ts = LR.traces(feats, v, pl, g, mni)
    assert sorted(t["stop"] for t in ts) == ["gradient", "parameter"] and all(t["iters"] == 1 for t in ts)
    for t in ts:
        moved = t["stop"] == "gradient"
        assert moved != np.array_equal(t["x"], LR.unify(g))
        tr = LR.follow(feats, v, pl, g, [np.asarray(g), t["x"], t["x"]], 1, mni)
        assert tr["stop"] == t["stop"]
    with pytest.raises(LR.TraceError):
        LR.follow(feats, v, pl, g, [np.asarray(g), next(t["x"] for t in ts if t["stop"] == "gradient")], 2, mni)


@pytest.mark.parametrize("name", NAMES + ["horizon_ds"])
def test_follow_accepts_the_oracle_truncated_solves(oracle, worlds, name):
    feats, v, pl, g, mni = worlds[name]
    its, n = _truncated(oracle, feats, v, pl, g, mni)
    tr = LR.follow(feats, v, pl, g, its, n, mni)
    # the oracle solves by QR: its accepted steps are held to the normal-equation bound plus nothing else, and meet it
    assert tr["ratio"] <= 1.0
    assert tr["stop"] == LR.run(feats, v, pl, g, mni)["stop"] or LR.open_decisions(LR.run(feats, v, pl, g, mni))


def test_old_start_rule_fails():
    """The rule the oracle and the kernel used to follow (the gradient tested only after an accepted step) takes a step on the
    zero-residual world (|g| near 1e-13), where Ceres (IterationZero marks the start successful) stops after none."""
    m, q, g = LA.zero_residual()
    import oracle_lib as O
    _, v, pl, _, _ = O.find_surf_corr(O.KdTree(m), q, g)
    old = LR.run(q, v, pl, g, 15, rules=dict(gradient_at_start=False, invalid="halve"))
    assert old["iters"] == 1 and old["stop"] == "parameter"
    new = LR.run(q, v, pl, g, 15)
    assert new["iters"] == 0 and new["stop"] == "gradient"
    assert O.ceres_solve(q, v, pl, g, 15)[0] == 0          # the oracle follows Ceres


# fault name -> (world, the rules it replaces, whether the end-of-pass check lets it through there)
FAULTS = {
    "reject_keeps_decrease_factor": ("rotation", dict(reject_double=False), False),
    "reject_always_halves": ("rotation", dict(reject_div=2.0, reject_double=False), False),
    "gradient_only_after_a_success": ("zero_residual", dict(gradient_at_start=False), False),
    "model_cost_change_without_half": ("rotation", dict(mcc_half=False), False),
    # on the exactly flat tilted plane the iteration count is unchanged and ceres_tolerance is unbounded (rank-deficient H):
    # only the per-iteration check sees these
    "model_cost_change_without_half_flat": ("tilted_flat_plane", dict(mcc_half=False), True),
    "radius_grown_half_again_too_far": ("tilted_flat_plane", dict(grow=lambda r, rd: 1.5 * r / max(1 / 3, 1 - (2 * rd - 1) ** 3)), True),
}


@pytest.mark.parametrize("fault", list(FAULTS))
def test_follow_rejects_planted_fault(oracle, worlds, fault, capsys):
    """A device whose trust-region bookkeeping has the fault: its truncated iterates are the faulty reference's, capped at each
    j.  The per-iteration check must reject it; whether the end-of-pass check (iteration count exact, pose within
    ceres_tolerance of the oracle's) would have is printed.  Not planted, because they cannot change an outcome: an invalid
    step that leaves the radius unchanged (under Ceres' rules no world reaches an invalid step, see lm_reference), and the
    Jacobi scaling recomputed after every accepted step (it cancels from the step: (S H S + S diag(H) S / radius) y = -S g
    gives S y = -(H + diag(H) / radius)^-1 g, except where the 1e-6 clamp of the diagonal binds, which no world reaches)."""
    name, rules, end_missed = FAULTS[fault]
    feats, v, pl, g, mni = worlds[name]
    full = LR.run(feats, v, pl, g, mni, rules=rules)
    its = [np.asarray(g, np.float64)] + [LR.run(feats, v, pl, g, j, rules=rules)["x"]
                                         for j in range(1, min(full["iters"] + 1, mni) + 1)]
    with pytest.raises(LR.TraceError):
        LR.follow(feats, v, pl, g, its, full["iters"], mni)
    it_o, pose_o, _ = oracle.ceres_solve(feats, v, pl, g, mni)
    s29 = oracle.normal_equations(feats, v, pl, g)
    tol = RA.ceres_tolerance(g, RA.unify(pose_o), s29, it_o, RA.U)
    end_ok = full["iters"] == it_o and float(np.abs(full["x"] - RA.unify(pose_o)).max()) <= tol
    with capsys.disabled():
        print(f"\nplanted fault {fault} on {name}: per-iteration check rejects; end-of-pass check "
              f"{'ACCEPTS (missed)' if end_ok else 'rejects'}")
    assert end_ok == end_missed, (fault, end_ok)
