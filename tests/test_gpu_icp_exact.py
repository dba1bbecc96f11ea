"""GPU tier for the loop-closure ICP (k_icp_persistent, liliom_icp_align / liliom_loop_align) against tests/icp_reference.py's
icp_trace bit for bit: the final T (16 doubles), the fitness over every source point, the verdict and the iteration count; and pass
by pass, since PCL's loop under a cap of k iterations is the first k passes of the uncapped loop.  The adversarial world at 1 m and
2 m cells and four cut-offs (cell corners and faces, ties, a clump, source points far outside the target's grid on every face,
pairs on the correspondence cut), the default loop-closure world at every source size that changes the launch and in all three
point layouts, and one loop-closure call from the keyframe store."""
import numpy as np
import pytest

import icp_reference as R

pytestmark = pytest.mark.gpu

F32 = np.float32
LEAF = 0.4


def _ctx(cell=1.0, variant=0):
    import liliom_b200 as L
    p = L.default_params(variant)
    p.knn_max_sqdist = cell * cell                # the target's grid: cells of gate_cell(knn_max_sqdist) metres
    return L.Context(params=p)


def _check(got, tr, what):
    T, fit, conv, it = got
    assert (conv, it) == (tr["converged"], tr["iters"]), (what, (conv, it), (tr["converged"], tr["iters"]), tr["end"])
    assert T.tobytes() == tr["T"].tobytes(), (what, np.abs(T - tr["T"]).max())
    assert np.float64(fit).tobytes() == np.float64(tr["fitness"]).tobytes(), (what, fit, tr["fitness"])


def _check_passes(c, src, tgt, tr, max_corr, what):
    """max_iter = k for k = 1 .. iterations: T equals the trace's F after pass k; names the first pass that differs"""
    steps = [p for p in tr["passes"] if p["mse"] is not None and p["n_corr"] >= 3]
    for k in range(1, tr["iters"] + 1):
        T, fit, conv, it = c.icp_align(src, tgt, max_corr_dist=max_corr, max_iter=k)
        want = steps[k - 1]
        if T.tobytes() != want["F"].tobytes() or it != k or not conv:
            s = want["sums"]
            pytest.fail(f"{what}: pass {k} differs (reference n_corr {want['n_corr']}, |T - F_k| max {np.abs(T - want['F']).max():.3e}, "
                        f"iterations {it}, reference sums up to {np.abs(s).max():.6e})")


@pytest.fixture(scope="module", params=[1.0, 2.0], ids=["cell1", "cell2"])
def adv(request):
    cell = request.param
    src, tgt, notes = R.adversarial_icp_world(0, cell)
    c = _ctx(cell)
    yield c, src, tgt, notes, cell
    c.close()


@pytest.mark.parametrize("max_corr", R.MAX_CORRS)
def test_adversarial_world_bit_for_bit_and_pass_by_pass(adv, max_corr):
    c, src, tgt, notes, cell = adv
    tr = R.icp_trace(src, tgt, max_corr)
    _check(c.icp_align(src, tgt, max_corr_dist=max_corr), tr, f"cell {cell} max_corr {max_corr}")
    _check_passes(c, src, tgt, tr, max_corr, f"cell {cell} max_corr {max_corr}")
    # the cut at PCL's threshold: pass 1 leaves out the pairs at exactly fp32(max_corr^2) and keeps those one float below
    if max_corr in (0.3, 1.7):
        idx = tr["passes"][0]["idx"]
        assert (idx[notes["gate"][(max_corr, "at")]] < 0).all() and (idx[notes["gate"][(max_corr, "below")]] >= 0).all()
        _, d, _ = R.reference_nn1(src[:, :3], tgt, None)
        assert tr["passes"][0]["n_corr"] == int((d <= F32(max_corr * max_corr)).sum()) - len(notes["gate"][(max_corr, "at")])
    # points beyond the grid's largest dimension are part of the fitness (a mean over all n points)
    assert tr["fitness"] > 4000.0 ** 2 / len(src)


@pytest.mark.parametrize("max_corr", [1.0, 30.0])
def test_adversarial_world_far_from_the_origin(max_corr):
    """the same world moved to (5000, -3000, 20) m, where an fp32 step is 0.5 mm"""
    src, tgt, _ = R.adversarial_icp_world(1, 1.0, offset=(5000.0, -3000.0, 20.0))
    c = _ctx(1.0)
    try:
        tr = R.icp_trace(src, tgt, max_corr)
        _check(c.icp_align(src, tgt, max_corr_dist=max_corr), tr, f"offset max_corr {max_corr}")
        _check_passes(c, src, tgt, tr, max_corr, f"offset max_corr {max_corr}")
    finally:
        c.close()


def default_world(world_small, n, seed=4):
    """test_loop_closure_icp's world: 30 000 target points from the synthetic map, a source of n points seen from a frame off
    by 2.5 deg / (0.6, -0.4, 0.1) m with 1 cm noise"""
    rng = np.random.default_rng(seed)
    m = world_small["map"]
    near = m[(np.abs(m[:, 0]) < 45) & (np.abs(m[:, 1]) < 45)]
    tgt = near[rng.permutation(len(near))[:30000]].copy()
    ang = np.deg2rad(2.5)
    Rz = np.array([[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1.0]])
    pick = near[rng.integers(0, len(near), n)]
    src = R.as_f4(((pick[:, :3].astype(np.float64) - np.array([0.6, -0.4, 0.1])) @ Rz + rng.normal(0, 0.01, (n, 3))).astype(F32))
    return src, R.as_f4(tgt)


def _layout(a, stride):
    import liliom_b200 as L
    if stride == 16:
        return np.ascontiguousarray(a, F32)
    out = np.zeros(len(a), L.PT32 if stride == 32 else L.PT48)
    out["x"], out["y"], out["z"] = a[:, 0], a[:, 1], a[:, 2]
    return out


@pytest.mark.parametrize("n", [1, 2, 3, 255, 256, 257, 12000, 300000])
def test_default_world_at_every_launch_shape(world_small, n):
    """1 and 2 points: stuck at once, then the fitness pass; 255 / 256 / 257: one virtual block, full, one more; 300 000: more
    virtual blocks than co-resident blocks.  Every point layout gives the same bits."""
    src, tgt = default_world(world_small, n)
    tr = R.icp_trace(src, tgt)
    c = _ctx(1.0)
    try:
        for stride in (16, 32, 48):
            _check(c.icp_align(_layout(src, stride), _layout(tgt, stride)), tr, f"n {n} stride {stride}")
    finally:
        c.close()
    if n < 3:
        assert tr["end"] == R.STUCK_END


def test_far_source_has_a_finite_fitness():
    """a source 500 m from the target with a 5 m cut: no correspondence, not converged, identity; the fitness is the mean squared
    distance of every point (as PCL's getFitnessScore), not DBL_MAX"""
    src, tgt, _ = R.adversarial_icp_world(0, 1.0)
    far = src.copy(); far[:, 0] += 500.0
    tr = R.icp_trace(far, tgt, 5.0)
    assert tr["end"] == R.STUCK_END and np.isfinite(tr["fitness"]) and tr["fitness"] > 400.0 ** 2
    c = _ctx(1.0)
    try:
        got = c.icp_align(far, tgt, max_corr_dist=5.0)
    finally:
        c.close()
    assert not got[2] and got[3] == 0 and np.array_equal(got[0], np.eye(4))
    _check(got, tr, "far source")


@pytest.mark.parametrize("stride", [48, 32])
def test_loop_align_from_the_store(stride):
    """one liliom_loop_align call equals the trace on that call's two liliom_kf_cloud outputs (the target indexed in kf_cloud
    order), with a keyframe whose clouds reach 300 m beyond the rest"""
    import liliom_b200 as L
    from liliom_b200 import synth
    n_hist = 21
    seq = synth.make_keyframe_sequence(n_hist, stride=stride, revisit=1)
    e5, s5, p5 = seq[5]
    far_s = s5.copy(); far_s["x"] += 300.0; far_s["z"] -= 40.0
    seq.append((e5, np.concatenate([s5, far_s]), p5))
    bp = L.backend_default_params(0 if stride == 48 else 1)
    c = L.Context(variant=0 if stride == 48 else 1)
    try:
        for i, (e, s, _) in enumerate(seq):
            assert c.kf_add(bp, e, s, download=False)[0] == i
        poses = [p for _, _, p in seq]
        far_id = len(seq) - 1
        for si, ti in (([n_hist], list(range(n_hist))), ([far_id], list(range(10)))):
            sp, tp = [poses[i] for i in si], [poses[i] for i in ti]
            got = c.loop_align(si, sp, ti, tp, LEAF)
            src, tgt = c.kf_cloud(si, sp, LEAF), c.kf_cloud(ti, tp, LEAF)
            assert got[4:] == (len(src), len(tgt))
            tr = R.icp_trace(R.as_f4(np.c_[src["x"], src["y"], src["z"]]), R.as_f4(np.c_[tgt["x"], tgt["y"], tgt["z"]]))
            _check(got[:4], tr, f"loop_align {si} onto {len(ti)} keyframes")
    finally:
        c.close()


def test_every_way_the_loop_ends_is_exercised(world_small):
    """the cases of this file end the loop by the cap, rotation+translation, relative mse and too few correspondences: asserted
    here on the device, so that an edit of the worlds cannot quietly make them benign"""
    src, tgt, _ = R.adversarial_icp_world(0, 1.0)
    dsrc, dtgt = default_world(world_small, 12000)
    cases = [(src, tgt, dict(max_corr=1.0)), (src, tgt, dict(max_corr=1.0, max_iter=2)), (src[:2], tgt, {}),
             (dsrc, dtgt, {}), (dsrc[:3000], dtgt, dict(fit_eps=1e-3))]
    ends = set()
    c = _ctx(1.0)
    try:
        for s, t, kw in cases:
            tr = R.icp_trace(s, t, **kw)
            kwd = dict(max_corr_dist=kw.get("max_corr", 30.0), max_iter=kw.get("max_iter", 100), fit_eps=kw.get("fit_eps", 1e-6))
            _check(c.icp_align(s, t, **kwd), tr, f"{len(s)} points {kw}")
            ends.add(tr["end"])
    finally:
        c.close()
    assert {R.CAP, R.ROT_TRANS, R.REL_MSE, R.STUCK_END} <= ends, ends
