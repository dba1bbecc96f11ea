"""CPU tier of the re-anchored pass checker (tests/reanchor.py): it accepts the oracle's own GN and Ceres-faithful trajectories, and
it rejects each planted fault of the kind a rewrite of the device's GN step could introduce: the step solved in fp32, the trust
region skipped, damping where the system is well posed, one pass's sums taken from the previous pass, n_corr off by one, and a
quaternion left with w < 0.  Each fault is planted in one pass of a trajectory the checker accepts, and must be rejected at that
pass by the check that covers it."""
import numpy as np
import pytest

import lm_reference as LR
import reanchor as RA
from test_devmath_host import dm  # noqa: F401  (the host build of dev_math.cuh, a fixture)

ITERS = 10


def single_plane(seed=3, flat=False):
    """test_gn_step_stays_bounded_on_a_single_plane's world: the map is the plane z = 0 with 5 mm of noise, the features a patch of
    ground 1.5 m below the sensor.  The noise tilts every fitted normal a little, which constrains x, y and yaw weakly: the
    smallest LDL^T pivot stays near 3e-6 of the largest and every pass takes the PLAIN step.
    flat=True: the plane z = -2 exactly (a plane the fit's a x + b y + c z = -1 can represent), features and guess moved with it.
    Every fitted normal is then (0, 0, 1) to rounding, x, y and yaw are unobservable, and every pass takes the DAMPED step."""
    rng = np.random.default_rng(seed)
    g = np.arange(-30.0, 30.0, 0.4)
    X, Y = np.meshgrid(g, g)
    m = np.ones((X.size, 4), np.float32)
    m[:, 0] = X.ravel() + rng.uniform(-0.1, 0.1, X.size); m[:, 1] = Y.ravel() + rng.uniform(-0.1, 0.1, X.size)
    m[:, 2] = rng.normal(0, 0.005, X.size)
    feats = np.ones((1500, 4), np.float32)
    feats[:, 0] = rng.uniform(-20, 20, 1500); feats[:, 1] = rng.uniform(-20, 20, 1500); feats[:, 2] = -1.5
    half = np.deg2rad(1.0) / 2
    guess = np.array([np.cos(half), np.sin(half), 0.0, 0.0, 0.3, -0.2, 1.42])
    if flat:
        m[:, 2] = -2.0
        guess[6] -= 2.0
    return m, feats, guess


def flat_plane():
    return single_plane(flat=True)


def tilted_plane(seed=4, flat=False, tilt=0.8):
    """The single plane with features near the sensor (within 1.2 m of it horizontally) and a guess rolled 0.8 rad: the first GN
    step wants more roll than the 0.35 rad trust region lets it take (CLIPPED; DAMPED+CLIPPED on the flat plane)."""
    m, _, _ = single_plane(seed, flat)
    rng = np.random.default_rng(seed)
    r = 1.2 * np.sqrt(rng.uniform(0, 1, 800)); a = rng.uniform(0, 2 * np.pi, 800)
    feats = np.ones((800, 4), np.float32)
    feats[:, 0] = r * np.cos(a); feats[:, 1] = r * np.sin(a); feats[:, 2] = -1.5
    half = tilt / 2
    guess = np.array([np.cos(half), np.sin(half), 0.0, 0.0, 0.1, 0.2, -0.5 if flat else 1.5])
    return m, feats, guess


def tilted_flat_plane():
    return tilted_plane(flat=True)


# the branch every world's first GN pass takes, and whether a later pass takes another
PLANE_WORLDS = {"single_plane": (single_plane, "plain"), "flat_plane": (flat_plane, "damped"),
                "tilted_plane": (tilted_plane, "clipped"), "tilted_flat_plane": (tilted_flat_plane, "damped+clipped")}


def copy_stats(oracle, st):
    return [oracle.IterStats.from_buffer_copy(s) for s in st]


@pytest.fixture(scope="module")
def worlds(oracle):
    """(name, tree, features, guess) of the seeded worlds: world_small's Horizon sweep (down-sampled and every surf feature), a
    second seeded map with an HDL sweep through the ROT extractor, the single plane and the tilted plane."""
    from liliom_b200 import synth
    out = []
    for seed, kind in ((20260923, "horizon"), (11, "hdl")):
        m, _ = synth.make_map(100_000, seed=seed)
        T = synth.default_true_pose()
        if kind == "horizon":
            pts, q = synth.make_horizon_sweep(T)
            surf, _, _ = oracle.extract_horizon(pts, q)
        else:
            pts, q = synth.make_hdl64_sweep(T, seed=5)
            _, surf, _, _, _, _ = oracle.extract_rot(pts, q, (1.0, 0, 0, 0), 64, 4)
        tree = oracle.KdTree(m)
        out.append((f"{kind}_ds", tree, oracle.voxelgrid(surf, 0.4), synth.perturbed_pose(T)))
        if kind == "horizon":
            out.append(("horizon_surf", tree, surf, synth.perturbed_pose(T)))
    for name, (fn, _) in PLANE_WORLDS.items():
        m, feats, guess = fn()
        out.append((name, oracle.KdTree(m), feats, guess))
    return {w[0]: w[1:] for w in out}


@pytest.fixture(scope="module")
def gn_runs(oracle, worlds):
    runs = {}
    for name, (tree, feats, guess) in worlds.items():
        rc, _, st = oracle.scan_to_map_gn(tree, feats, guess, ITERS)
        assert rc == 0
        runs[name] = st
    return runs


@pytest.mark.parametrize("name", ["horizon_ds", "horizon_surf", "hdl_ds"] + list(PLANE_WORLDS))
def test_accepts_the_oracle_gn_trajectory(oracle, dm, worlds, gn_runs, name):  # noqa: F811
    tree, feats, guess = worlds[name]
    st = gn_runs[name]
    rep = RA.check_gn(oracle, tree, feats, guess, st, dm)
    assert rep["sum_ratio"] == 0.0                # the oracle's own sums at the oracle's own poses: the same computation
    assert st[0].n_corr > 100
    first = PLANE_WORLDS[name][1] if name in PLANE_WORLDS else "plain"
    assert rep["branches"][0] == first, rep["branches"]
    later = {"flat_plane": "damped", "tilted_flat_plane": "damped", "tilted_plane": "plain"}.get(name, first)
    assert set(rep["branches"][1:]) == {later}, rep["branches"]
    # the oracle's LDL^T divides by the pivot, the device's multiplies by its inverse: not bit-identical, but inside the bound
    assert rep["step_ratio"] <= 1.0


@pytest.mark.parametrize("name", ["horizon_ds", "hdl_ds", "single_plane"])
def test_accepts_the_oracle_ceres_trajectory(oracle, worlds, name):
    tree, feats, guess = worlds[name]
    rc, _, st = oracle.scan_to_map_ceres(tree, feats, guess, 3, 15)
    assert rc == 0
    rep = RA.check_ceres(oracle, tree, feats, guess, st, 15)
    assert rep["pose_dev"] == 0.0 and rep["sum_ratio"] == 0.0
    assert all(s.lm_iters > 0 for s in st)


def test_gn_step_restatement_matches_oracle_branches(oracle, dm, worlds, gn_runs):  # noqa: F811
    """The NumPy step and the dev_math host build agree with each other on every pass of every world, including the damped and
    clipped ones, within the derived bound."""
    for name, (tree, feats, guess) in worlds.items():
        st = gn_runs[name]
        for start, s in zip(RA.start_poses(guess, st), st):
            s29 = RA.sums29(s)
            want, branch, d, A = RA.gn_step(s29, start)
            assert np.abs(RA.devmath_step(dm, s29, start) - want).max() <= RA.step_tolerance(start, d, A), (name, branch)


# ---------------------------------------------------------------------------------------------- planted faults
def _plant_pose(st, k, pose):
    for j in range(7):
        st[k].pose7[j] = pose[j]


def _first(branches, want):
    return next(k for k, b in enumerate(branches) if b == want)


def fault_fp32_step(oracle, st, guess):
    k = 0
    start = RA.start_poses(guess, st)[k]
    H, g = RA.unpack(RA.sums29(st[k]))
    d = np.linalg.solve(H.astype(np.float32), -g.astype(np.float32)).astype(np.float64)
    _plant_pose(st, k, RA.unify(RA.ceres_plus(start, d)))
    return k, "NumPy step"


def fault_damped_when_well_posed(oracle, st, guess):
    k = 0
    start = RA.start_poses(guess, st)[k]
    H, g = RA.unpack(RA.sums29(st[k]))
    d = np.linalg.solve(H + RA.GN_DAMP_REL * H.diagonal().max() * np.eye(6), -g)
    _plant_pose(st, k, RA.unify(RA.ceres_plus(start, d)))
    return k, "NumPy step"


def fault_stale_sums(oracle, st, guess):
    """Pass 1 reduces pass 0's partials: its sums, cost and count are pass 0's and its step is taken from them."""
    k = 1
    start = RA.start_poses(guess, st)[k]
    for j in range(27):
        st[k].jtj_jtr[j] = st[k - 1].jtj_jtr[j]
    st[k].cost = st[k - 1].cost
    st[k].n_corr = st[k - 1].n_corr
    want, _, _, _ = RA.gn_step(RA.sums29(st[k]), start)
    _plant_pose(st, k, want)
    return k, "sums differ|n_corr"


def fault_n_corr_off_by_one(oracle, st, guess):
    k = 2
    st[k].n_corr += 1
    return k, "n_corr"


def fault_quaternion_not_unified(oracle, st, guess):
    k = 1
    p = np.array(st[k].pose7)
    assert p[0] > 0
    p[:4] = -p[:4]
    _plant_pose(st, k, p)
    return k, "NumPy step"


@pytest.mark.parametrize("fault", [fault_fp32_step, fault_damped_when_well_posed, fault_stale_sums, fault_n_corr_off_by_one,
                                   fault_quaternion_not_unified], ids=lambda f: f.__name__[6:])
@pytest.mark.parametrize("name", ["horizon_ds", "hdl_ds"])
def test_rejects_planted_fault(oracle, dm, worlds, gn_runs, fault, name):  # noqa: F811
    tree, feats, guess = worlds[name]
    st = copy_stats(oracle, gn_runs[name])
    RA.check_gn(oracle, tree, feats, guess, st, dm)                            # the unplanted copy passes
    k, why = fault(oracle, st, guess)
    with pytest.raises(RA.ReanchorError, match=rf"pass {k}\b.*({why})"):
        RA.check_gn(oracle, tree, feats, guess, st, dm)


@pytest.mark.parametrize("name", ["tilted_plane", "tilted_flat_plane"])
def test_rejects_skipped_trust_region(oracle, dm, worlds, gn_runs, name):  # noqa: F811
    """On the clipped pass: the pose moved by the whole step the branch solved for, unclipped."""
    tree, feats, guess = worlds[name]
    st = copy_stats(oracle, gn_runs[name])
    rep = RA.check_gn(oracle, tree, feats, guess, st, dm)
    k = _first(rep["branches"], PLANE_WORLDS[name][1])
    start = RA.start_poses(guess, st)[k]
    H, g = RA.unpack(RA.sums29(st[k]))
    if "damped" in rep["branches"][k]:
        H = H + RA.GN_DAMP_REL * H.diagonal().max() * np.eye(6)
    d = np.linalg.solve(H, -g)
    assert np.linalg.norm(d[:3]) > 1.1 * RA.GN_MAX_ROT
    _plant_pose(st, k, RA.unify(RA.ceres_plus(start, d)))
    with pytest.raises(RA.ReanchorError, match=rf"pass {k}\b.*NumPy step"):
        RA.check_gn(oracle, tree, feats, guess, st, dm)


def test_rejects_damping_skipped(oracle, dm, worlds, gn_runs):  # noqa: F811
    """On the flat plane's damped pass: the pose moved by the least-squares solution of the singular system instead."""
    tree, feats, guess = worlds["flat_plane"]
    st = copy_stats(oracle, gn_runs["flat_plane"])
    k = 0
    start = RA.start_poses(guess, st)[k]
    H, g = RA.unpack(RA.sums29(st[k]))
    d = np.linalg.lstsq(H, -g, rcond=None)[0]
    _plant_pose(st, k, RA.unify(RA.ceres_plus(start, d)))
    with pytest.raises(RA.ReanchorError, match=rf"pass {k}\b.*NumPy step"):
        RA.check_gn(oracle, tree, feats, guess, st, dm)


def lm_restated(oracle, feats, valid, plane, start, max_num_iter, grow=None):
    """The Ceres-faithful LM restated in NumPy (tests/lm_reference.py); grow(radius, relative_decrease) replaces the radius
    update after a successful step, to plant a fault.  Returns (iterations, pose)."""
    t = LR.run(feats, valid, plane, start, max_num_iter, rules=dict(grow=grow))
    return t["iters"], t["x"]


def test_lm_restatement_matches_oracle_lm(oracle, worlds):
    """The restated LM takes the oracle's iteration count on every outer iteration and lands within the checker's bound."""
    tree, feats, guess = worlds["horizon_ds"]
    rc, _, st = oracle.scan_to_map_ceres(tree, feats, guess, 3, 15)
    for start, s in zip(RA.start_poses(guess, st), st):
        _, valid, plane, _, _ = oracle.find_surf_corr(tree, feats, start)
        it, pose = lm_restated(oracle, feats, valid, plane, start, 15)
        assert it == s.lm_iters
        assert np.abs(pose - np.array(s.pose7)).max() <= RA.ceres_tolerance(start, np.array(s.pose7), RA.sums29(s), it, RA.U)


RADIUS_FAULTS = {"radius_kept": lambda r, rd: r, "radius_update_halved": lambda r, rd: r / max(1 / 3, 1 - (2 * rd - 1) ** 3) / 2}


@pytest.mark.parametrize("fault", ["lm_iters", "sums"] + list(RADIUS_FAULTS))
def test_ceres_check_rejects_planted_fault(oracle, worlds, fault):
    """The Ceres-faithful check: one LM iteration more, the previous iteration's sums, or the trust-region radius updated wrongly
    after a successful step (not grown; grown by half the rule's factor) with the iteration count unchanged."""
    tree, feats, guess = worlds["horizon_ds"]
    rc, _, st = oracle.scan_to_map_ceres(tree, feats, guess, 3, 15)
    RA.check_ceres(oracle, tree, feats, guess, st, 15)
    k = 0 if fault in RADIUS_FAULTS else 1
    if fault == "lm_iters":
        st[k].lm_iters += 1
        why = "LM iterations"
    elif fault == "sums":
        for j in range(27):
            st[k].jtj_jtr[j] = st[k - 1].jtj_jtr[j]
        why = "sums differ"
    else:
        start = RA.start_poses(guess, st)[k]
        _, valid, plane, _, _ = oracle.find_surf_corr(tree, feats, start)
        it, pose = lm_restated(oracle, feats, valid, plane, start, 15, RADIUS_FAULTS[fault])
        assert it == st[k].lm_iters and it > 1         # only the pose can tell
        _plant_pose(st, k, pose)
        why = "pose differs"
    with pytest.raises(RA.ReanchorError, match=rf"pass {k}\b.*{why}"):
        RA.check_ceres(oracle, tree, feats, guess, st, 15)
