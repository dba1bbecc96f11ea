"""Every adversarial LM world of tests/lm_adversarial.py on the device, checked LM iteration by LM iteration
(reanchor.trace_pass / lm_reference.follow) through scan_to_map and through upload_feats + scan_to_map_resident, and the union of
the branches and stops the device takes over all worlds.  Every decision must be closed (clear of its threshold) except the one
parameter_edge is built to leave open, and every accepted step's bound stays below 1e-6 of the step.  The gap between the two
model_cost_change formulas is printed; on the weak worlds so is the device's distance from the QR step, next to the
normal-equation bound it is held to and the bound a QR solve itself would meet, and the whole call is held to the 1e-4
pose-parity level against the QR reference wherever the summed one-step bounds say that level is attainable."""
import json

import numpy as np
import pytest

import lm_adversarial as LA
import lm_reference as LR
import reanchor as RA
from test_gpu_reanchored import probe_of, truncated_of

pytestmark = pytest.mark.gpu


def _resident_truncated(ctx, feats):
    import liliom_b200 as L
    ctx.upload_feats(feats)

    def run(start, j):
        pose, st = ctx.scan_to_map_resident(start, 1, max_num_iter=j, mode=L.MODE_CERES, want_stats=True)
        return pose, st[0].lm_iters
    return run


def _device_world(oracle, name):
    import liliom_b200 as L
    fn, mni, _, _ = LA.WORLDS[name]
    m, feats, guess = fn()
    tree = oracle.KdTree(m)
    c, pc, rc = L.Context(variant=0), L.Context(variant=0), L.Context(variant=0)
    try:
        for x in (c, pc, rc):
            x.map_set_points(m)
        pr = probe_of(pc, feats)
        pose, st = c.scan_to_map(feats, guess, 1, max_num_iter=mni, mode=L.MODE_CERES)
        rep = RA.check_ceres(oracle, tree, feats, guess, st, mni, 8, f"lm/{name}", pr, truncated_of(pc, feats))
        c.upload_feats(feats)
        pose_r, st_r = c.scan_to_map_resident(guess, 1, max_num_iter=mni, mode=L.MODE_CERES, want_stats=True)
        assert pose_r.tobytes() == pose.tobytes()
        rep_r = RA.check_ceres(oracle, tree, feats, guess, st_r, mni, 8, f"lm/{name}/resident", pr, _resident_truncated(rc, feats))
        qr_call = None
        if name in LA.WEAK:
            vd, pld = pr(guess)
            qr_call = float(np.abs(RA.unify(pose) - LR.run(feats, vd, pld, guess, mni, solver="qr")["x"]).max())
        return dict(rep=rep, rep_r=rep_r, pose=pose, guess=guess, lm_iters=st[0].lm_iters, qr_call=qr_call)
    finally:
        c.close(); pc.close(); rc.close()


@pytest.fixture(scope="module")
def device_runs(oracle):
    return {name: _device_world(oracle, name) for name in LA.WORLDS}


@pytest.mark.parametrize("name", list(LA.WORLDS))
def test_lm_world_every_iteration(device_runs, name):
    _, _, stop, branches = LA.WORLDS[name]
    d = device_runs[name]
    rep = d["rep"]
    for r in (rep, d["rep_r"]):
        assert r.get("bound_over_step", 0.0) < 1e-6, r
        assert r.get("open_decisions", 0) == (1 if name == "parameter_edge" else 0), r
    if stop:
        assert rep["stops"] == [stop], rep["stops"]
    for b in branches:
        assert b in rep["branches"], rep["branches"]
    if name == "zero_residual":
        assert np.array_equal(d["pose"], d["guess"]) and d["lm_iters"] == 0
    keep = ("trace_ratio", "trace_dev", "trace_bound", "bound_over_step", "mcc_gap", "qr_dev", "qr_bound", "pose_ratio",
            "step_bound_sum")
    out = {k: v for k, v in rep.items() if k in keep}
    out.update(stops=rep.get("stops"), branches=sorted(set(rep.get("branches", []))), lm_iters=rep["lm_iters"])
    if d["qr_call"] is not None:
        out["call_dev_from_qr"] = d["qr_call"]
        if rep["step_bound_sum"] < 1e-4:
            assert d["qr_call"] <= 1e-4, out
    print(f"lm_trace {name} {json.dumps(out)}")


def test_lm_branch_coverage(device_runs):
    """Over every world: the device took every reachable branch and stop.  Invalid steps, five invalid steps in a row and the
    radius floor are out of reach under Ceres' rules on well-conditioned input (lm_reference's docstring)."""
    branches, stops = set(), set()
    for d in device_runs.values():
        for r in (d["rep"], d["rep_r"]):
            branches.update(r.get("branches", []))
            stops.update(r.get("stops", []))
    assert {"accepted", "rejected"} <= branches, branches
    assert {"iteration_cap", "function", "parameter", "gradient", "no_correspondences"} <= stops, stops
    print(f"lm_coverage {json.dumps(dict(branches=sorted(branches), stops=sorted(stops)))}")
