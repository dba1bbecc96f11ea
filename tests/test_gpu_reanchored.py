"""Every scan-to-map pass of the device checked against the oracle from the device's OWN start pose (tests/reanchor.py).

The trajectory checks of test_gpu_at_size.py / test_gpu_parity.py hold each pass's pose within 1e-4 of the oracle's; a step that is
a little wrong converges to the same fixed point and passes them.  Here each pass k of a device call is re-run on the CPU from the
pose the device started it from: the oracle's correspondence count and accept flags must equal the device's exactly, the device's
planes must equal the oracle's at rtol 2e-6, the device's sums must equal the oracle's fp64 reduction of those planes at rtol 1e-9,
and the device's pose after the pass must equal the GN step computed on the host from the device's own sums within a bound
derived from the condition number of the solved system (or, in the Ceres-faithful mode, the oracle's LM on the same
correspondences from the same start must take the same number of iterations and land within a derived bound).

Covered: world_small's down-sampled scan, every surf feature, 3000 of them, 40 and one, through scan_to_map and through
upload_feats + scan_to_map_resident; every forced search shape of test_gpu_knn_exact.py, on the persistent launch and on per-pass
launches, and the 16-lane persistent launch with bulk-copy staging (LILIOM_KNN_TMA=1, one round and three); odometry_resident after extract_resident (Horizon and ROT), whose want_stats=False pose must carry the same bits; the
single plane (plain step), the exactly flat plane (damped step), and a guess rolled 0.8 rad over both (trust-region clip); and
BASELINE configs 1 and 2 at size (1 M and 2 M maps).  In the Ceres-faithful mode the scan_to_map calls are also checked LM
iteration by LM iteration (reanchor.trace_pass; configs 1 and 2 on their first outer pass).  Each check prints one `reanchor`
line with its largest deviations and bounds."""
import json

import numpy as np
import pytest

import knn_reference as R
import reanchor as RA
from test_devmath_host import dm  # noqa: F401  (the host build of dev_math.cuh, a fixture)
from test_gpu_knn_exact import KWARPS, SHAPES, _ctx, _ids, _per_task, _plan_grid, _sm_count
from test_reanchor_cpu import PLANE_WORLDS

pytestmark = pytest.mark.gpu

ITERS = 10
CERES_OUTER, CERES_LM = 3, 15


def _same_points(a, b):
    """Every field of the PCL point type (x, y, z, intensity, and normal and curvature in the 48-byte layout) bit for bit."""
    assert len(a) == len(b), (len(a), len(b))
    for f in ("x", "y", "z", "intensity") + (("nx", "ny", "nz", "curvature") if "nx" in a.dtype.names else ()):
        assert np.array_equal(a[f].view(np.uint32), b[f].view(np.uint32)), f


def _say(what, rep):
    keep = {k: (round(float(v), 4) if k.endswith("ratio") else float(v)) for k, v in rep.items()
            if k not in ("branches", "n_corr", "lm_iters", "stops")}
    if "stops" in rep:
        keep["stops"] = sorted(set(rep["stops"]))
    if "branches" in rep:
        keep["branches"] = sorted(set(rep["branches"]))
    print(f"reanchor {what} {json.dumps(keep)}")


def probe_of(ctx, feats):
    """The device's own correspondences of `feats` at a pose, from a context that holds the same map (and the same search shape)
    as the one under test, so that probing changes nothing the tested context remembers between calls."""
    return lambda pose: ctx.find_surf_corr(feats, pose)[:2]


def _gn(oracle, dm, tree, feats, guess, st, what, probe, nthreads=8):  # noqa: F811
    rep = RA.check_gn(oracle, tree, feats, guess, st, dm, nthreads, what, probe)
    _say(what, rep)
    return rep


def truncated_of(ctx, feats):
    """The device's match_cnt = 1 Ceres-faithful call from `start` capped at j LM iterations: (pose, its iteration count).
    From a context like probe_of's, so the call under test is not disturbed."""
    import liliom_b200 as L

    def run(start, j):
        pose, st = ctx.scan_to_map(feats, start, 1, max_num_iter=j, mode=L.MODE_CERES)
        return pose, st[0].lm_iters
    return run


def _ceres(oracle, tree, feats, guess, st, what, probe, nthreads=8, truncated=None, trace_passes=None):
    """The end-of-pass check and, given truncated (truncated_of), every LM iteration of the passes in trace_passes."""
    rep = RA.check_ceres(oracle, tree, feats, guess, st, CERES_LM, nthreads, what, probe, truncated, trace_passes)
    _say(what, rep)
    return rep


@pytest.fixture(scope="module")
def ws(oracle, world_small):
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    return dict(surf=surf, ds=ds, tree=oracle.KdTree(world_small["map"]), map=world_small["map"], guess=world_small["guess"])


FEATURE_SETS = {"ds": lambda w: w["ds"], "surf": lambda w: w["surf"], "surf3000": lambda w: w["surf"][:3000],
                "ds40": lambda w: w["ds"][:40], "one": lambda w: w["ds"][:1]}


@pytest.mark.parametrize("fs", list(FEATURE_SETS))
def test_world_small_every_pass(oracle, dm, ws, fs):  # noqa: F811
    """scan_to_map and upload_feats + scan_to_map_resident, GN and Ceres-faithful, every pass re-anchored; the resident call
    without stats returns the same pose bits as with them."""
    import liliom_b200 as L
    feats = FEATURE_SETS[fs](ws)
    tree, guess = ws["tree"], ws["guess"]
    c, pc = L.Context(variant=0), L.Context(variant=0)
    try:
        c.map_set_points(ws["map"]); pc.map_set_points(ws["map"])
        pr = probe_of(pc, feats)
        pose, st = c.scan_to_map(feats, guess, ITERS, mode=L.MODE_GN)
        rep = _gn(oracle, dm, tree, feats, guess, st, f"world_small/{fs}/scan_to_map", pr)
        assert np.array_equal(pose, np.array(st[-1].pose7))
        if fs in ("ds", "surf", "surf3000"):
            assert st[0].n_corr > 0.5 * len(feats) and set(rep["branches"]) == {"plain"}
        c.upload_feats(feats)
        pose_r, st_r = c.scan_to_map_resident(guess, ITERS, mode=L.MODE_GN, want_stats=True)
        _gn(oracle, dm, tree, feats, guess, st_r, f"world_small/{fs}/resident", pr)
        pose_n, none = c.scan_to_map_resident(guess, ITERS, mode=L.MODE_GN, want_stats=False)
        assert none is None and pose_n.tobytes() == pose_r.tobytes()
        pose, st = c.scan_to_map(feats, guess, CERES_OUTER, max_num_iter=CERES_LM, mode=L.MODE_CERES)
        _ceres(oracle, tree, feats, guess, st, f"world_small/{fs}/scan_to_map", pr, truncated=truncated_of(pc, feats))
        pose_r, st_r = c.scan_to_map_resident(guess, CERES_OUTER, max_num_iter=CERES_LM, mode=L.MODE_CERES, want_stats=True)
        _ceres(oracle, tree, feats, guess, st_r, f"world_small/{fs}/resident", pr)
    finally:
        c.close(); pc.close()


@pytest.mark.parametrize("shape", SHAPES, ids=_ids)
def test_forced_search_shapes_every_pass(oracle, dm, ws, shape):  # noqa: F811
    """Every forced lane shape / rounds of the 5-NN search (and the plan's own choice): the persistent launch on the down-sampled
    scan, per-pass launches on a query set whose grid exceeds one block per SM, and the Ceres-faithful mode."""
    import liliom_b200 as L
    sm = _sm_count()
    tree, guess = ws["tree"], ws["guess"]
    f4 = oracle._f4(ws["ds"])
    per_task = 32 if shape is None else _per_task(shape)
    big = np.resize(f4, (sm * KWARPS * per_task + 1001, 4))
    if shape is not None:
        assert _plan_grid(len(f4), shape, sm) <= sm < _plan_grid(len(big), shape, sm)
    c, pc = _ctx(shape), _ctx(shape)
    try:
        c.map_set_points(ws["map"]); pc.map_set_points(ws["map"])
        _, st = c.scan_to_map(f4, guess, ITERS, mode=L.MODE_GN)
        _gn(oracle, dm, tree, f4, guess, st, f"shape {_ids(shape)}/persistent", probe_of(pc, f4))
        _, st = c.scan_to_map(big, guess, 4, mode=L.MODE_GN)
        _gn(oracle, dm, tree, big, guess, st, f"shape {_ids(shape)}/per_pass", probe_of(pc, big))
        _, st = c.scan_to_map(f4, guess, CERES_OUTER, max_num_iter=CERES_LM, mode=L.MODE_CERES)
        _ceres(oracle, tree, f4, guess, st, f"shape {_ids(shape)}/ceres", probe_of(pc, f4), truncated=truncated_of(pc, f4))
    finally:
        c.close(); pc.close()


@pytest.mark.parametrize("rounds", [1, 3])
def test_bulk_copy_staging_every_pass(oracle, dm, ws, rounds):  # noqa: F811
    """The 16-lane persistent launch with every run staged by one bulk copy (k_gn_persistent<16, true>, LILIOM_KNN_TMA=1), as
    test_bulk_copy_staging_bit_identical runs it: world_small's down-sampled scan, and the adversarial map of test_gpu_knn_exact.py
    (an 80-point clump: runs longer than a staging tile) from a slightly rotated start; GN and Ceres-faithful."""
    import liliom_b200 as L
    sm = _sm_count()
    am, aq, _ = R.adversarial_world(0)
    q = np.array([1.0, 0.002, -0.003, 0.001]); q /= np.linalg.norm(q)
    cases = [("world_small", ws["map"], ws["tree"], oracle._f4(ws["ds"]), ws["guess"]),
             ("adversarial", am, oracle.KdTree(am), aq, np.concatenate([q, [0.05, -0.04, 0.02]]))]
    for name, m, tree, feats, guess in cases:
        assert _plan_grid(len(feats), (16, rounds), sm) <= sm          # persistent: the bulk-copy instantiation
        c, pc = _ctx((16, rounds), tma=True), _ctx((16, rounds), tma=True)
        try:
            c.map_set_points(m); pc.map_set_points(m)
            pr = probe_of(pc, feats)
            _, st = c.scan_to_map(feats, guess, ITERS, mode=L.MODE_GN)
            rep = _gn(oracle, dm, tree, feats, guess, st, f"tma 16x{rounds}/{name}", pr)
            assert st[0].n_corr > 0 and "refused" not in rep["branches"]
            _, st = c.scan_to_map(feats, guess, CERES_OUTER, max_num_iter=CERES_LM, mode=L.MODE_CERES)
            _ceres(oracle, tree, feats, guess, st, f"tma 16x{rounds}/{name}/ceres", pr)
        finally:
            c.close(); pc.close()


@pytest.mark.parametrize("variant", [0, 1], ids=["horizon", "rot"])
def test_odometry_resident_every_pass(oracle, dm, world_small, variant):  # noqa: F811
    """upload_scan + extract_resident + odometry_resident, as the bench's resident leg calls them: the first call (launches sized
    from the upper bound), the second (one persistent launch sized from the first), and the same call without stats, which writes
    the pose straight into the pinned block: the same bits."""
    import liliom_b200 as L
    if variant == 0:
        pts, q = world_small["hz"], world_small["q_hz"]
        surf_o, _, _ = oracle.extract_horizon(pts, q)
    else:
        pts, q = world_small["hdl"], world_small["q_hdl"]
        _, surf_o, _, _, _, _ = oracle.extract_rot(pts, q, (1.0, 0, 0, 0), 64, 4)
    ds_o = oracle.voxelgrid(surf_o, 0.4)
    tree, guess = oracle.KdTree(world_small["map"]), world_small["guess"]
    c, pc = L.Context(variant=variant), L.Context(variant=variant)
    try:
        c.map_set_points(world_small["map"]); pc.map_set_points(world_small["map"])
        pr = probe_of(pc, ds_o)
        poses = []
        for call in range(2):
            c.upload_scan(pts)
            c.extract_resident(q)
            pose, st, ds = c.odometry_resident(guess, ITERS, mode=L.MODE_GN, want_ds=True, cap=len(pts))
            _same_points(ds, ds_o)
            _gn(oracle, dm, tree, ds_o, guess, st, f"odometry_resident/{'horizon' if variant == 0 else 'rot'}/call{call}", pr)
            poses.append(pose)
        c.upload_scan(pts)
        c.extract_resident(q)
        pose_n, none, nds = c.odometry_resident(guess, ITERS, mode=L.MODE_GN, want_stats=False)
        assert none is None and nds == len(ds_o)
        assert pose_n.tobytes() == poses[1].tobytes()
        c.upload_scan(pts)
        c.extract_resident(q)
        _, st, _ = c.odometry_resident(guess, CERES_OUTER, max_num_iter=CERES_LM, mode=L.MODE_CERES)
        _ceres(oracle, tree, ds_o, guess, st, f"odometry_resident/{'horizon' if variant == 0 else 'rot'}/ceres", pr)
    finally:
        c.close(); pc.close()


@pytest.mark.parametrize("name", list(PLANE_WORLDS))
def test_degenerate_geometry_branches(oracle, dm, name):  # noqa: F811
    """The GN step's rarely used branches on the device: the exactly flat plane takes the damped step on every pass, the 0.8 rad
    roll the trust-region clip on its first pass (damped and clipped on the flat plane).  The noisy single plane of
    test_gn_step_stays_bounded_on_a_single_plane stays on the plain step: its fitted normals constrain x, y and yaw weakly."""
    import liliom_b200 as L
    fn, first = PLANE_WORLDS[name]
    m, feats, guess = fn()
    tree = oracle.KdTree(m)
    c, pc = L.Context(variant=0), L.Context(variant=0)
    try:
        c.map_set_points(m); pc.map_set_points(m)
        pr = probe_of(pc, feats)
        pose, st = c.scan_to_map(feats, guess, ITERS, mode=L.MODE_GN)
        rep = _gn(oracle, dm, tree, feats, guess, st, f"plane/{name}", pr)
        assert rep["branches"][0] == first, rep["branches"]
        if name == "flat_plane":
            assert set(rep["branches"]) == {"damped"}
        assert np.all(np.isfinite(pose))
        _, st = c.scan_to_map(feats, guess, CERES_OUTER, max_num_iter=CERES_LM, mode=L.MODE_CERES)
        _ceres(oracle, tree, feats, guess, st, f"plane/{name}/ceres", pr, truncated=truncated_of(pc, feats))
    finally:
        c.close(); pc.close()


@pytest.mark.parametrize("config", [1, 2])
def test_configs_at_size_every_pass(oracle, dm, config):  # noqa: F811
    """BASELINE config 1 (24k Horizon sweep vs 1 M map) and config 2 (130k HDL-64E sweep through the ROT extractor vs 2 M map):
    scan_to_map on the oracle's down-sampled scan and the node-facing odometry call, GN and Ceres-faithful."""
    import liliom_b200 as L
    from liliom_b200 import synth
    m, _ = synth.make_map(1_000_000 if config == 1 else 2_000_000)
    T = synth.default_true_pose()
    guess = synth.perturbed_pose(T)
    if config == 1:
        pts, q = synth.make_horizon_sweep(T)
        surf_o, _, _ = oracle.extract_horizon(pts, q)
    else:
        pts, q = synth.make_hdl64_sweep(T)
        _, surf_o, _, _, _, _ = oracle.extract_rot(pts, q, (1.0, 0, 0, 0), 64, 4)
    ds_o = oracle.voxelgrid(surf_o, 0.4)
    tree = oracle.KdTree(m)
    c, pc = L.Context(variant=0 if config == 1 else 1), L.Context(variant=0 if config == 1 else 1)
    try:
        c.map_set_points(m); pc.map_set_points(m)
        pr = probe_of(pc, ds_o)
        _, st = c.scan_to_map(ds_o, guess, ITERS, mode=L.MODE_GN)
        _gn(oracle, dm, tree, ds_o, guess, st, f"config{config}/scan_to_map", pr)
        _, st, ds = c.odometry(surf_o, guess, ITERS, mode=L.MODE_GN)
        _same_points(ds, ds_o)
        _gn(oracle, dm, tree, ds_o, guess, st, f"config{config}/odometry", pr)
        _, st = c.scan_to_map(ds_o, guess, 2, max_num_iter=CERES_LM, mode=L.MODE_CERES)
        _ceres(oracle, tree, ds_o, guess, st, f"config{config}/ceres", pr, truncated=truncated_of(pc, ds_o), trace_passes=(0,))
    finally:
        c.close(); pc.close()
