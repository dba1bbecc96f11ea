"""The scan-to-map 5-NN search on the device against a plain reference, at every lane shape and on every GN pass.

The search has five shapes (one thread per query, 2, 4, 8 or 16 lanes per query) and a number of rounds per warp task; the launch
plan picks them from the query count, LILIOM_KNN_LANES / LILIOM_KNN_ROUNDS force them.  For each forced shape and the unforced plan:
  (a) find_surf_corr at the identity pose returns, for EVERY query, the five (fp32 distance, map index) keys of
      tests/knn_reference.py (kd-tree ball, no cell grid), including queries with fewer than five points inside the gate;
      decisions and planes equal the oracle's; the 29 sums equal the oracle's normal equations;
  (b) from the second pass of a call every query starts its search at a coherence bound instead of the gate: pass k of
      scan_to_map must give exactly the count and the bits of the sums of a full search from the gate at pass k's start pose;
  (c) bulk-copy staging of the 16-lane search (LILIOM_KNN_TMA=1) changes no bit, with one round and with three;
  (d) upload_feats + scan_to_map_resident equals scan_to_map."""
import os

import numpy as np
import pytest

import knn_reference as R

pytestmark = pytest.mark.gpu

KWARPS = 8
# (LILIOM_KNN_LANES, LILIOM_KNN_ROUNDS); None: the plan's own choice.  (2, 4) is clamped by the plan to 32 queries per task.
SHAPES = [(1, 1), (2, 1), (2, 4), (4, 1), (4, 3), (8, 1), (8, 2), (16, 1), (16, 3), None]
IDENT = np.array([1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0])


def _ctx(shape, tma=False):
    import liliom_b200 as L
    env = {"LILIOM_KNN_LANES": str(shape[0]) if shape else None, "LILIOM_KNN_ROUNDS": str(shape[1]) if shape else None,
           "LILIOM_KNN_TMA": "1" if tma else "0"}
    old = {k: os.environ.get(k) for k in env}
    try:
        for k, v in env.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        return L.Context(variant=0)             # the switches are read at liliom_create
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _cdiv(a, b):
    return -(-a // b)


def _per_task(shape):
    """Queries per warp task of a forced shape (s2m_plan clamps it to 32)."""
    lanes, rounds = shape
    return min((32 // lanes) * rounds, 32)


def _plan_grid(n, shape, sm):
    """Blocks of a forced shape for n queries with a host-side count (s2m_plan); the launch is persistent when this is <= sm."""
    return min(max(_cdiv(_cdiv(n, _per_task(shape)), KWARPS), 1), 2 * sm)


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ids(shape):
    return "plan" if shape is None else f"{shape[0]}x{shape[1]}"


@pytest.fixture(scope="module")
def adv(oracle):
    """The adversarial map, its queries, and a long query list (the adversarial ones first, then the dense region, the sparse region
    and beyond the grid) long enough that one thread per query loops over its warp tasks."""
    m, qs, notes = R.adversarial_world(0)
    if len(qs) % 2 == 0:                         # every per_task is even: an odd count is never a multiple
        qs = qs[:-1]
        notes["outside"] = (notes["outside"][0], min(notes["outside"][1], len(qs)))
    rng = np.random.default_rng(5)
    n_big = 2 * _sm_count() * KWARPS * 32 + 500
    fill = np.ones((n_big - len(qs), 4), np.float32)
    k = len(fill)
    fill[:, :3] = np.concatenate([
        np.array([20.0, -8.0, 1.0]) + rng.uniform(-0.5, 1.05, (k - k // 5, 3)) * np.array([10.0, 8.0, 4.0]),
        np.array([40.0, -7.0, 1.0]) + rng.uniform(0, 1, (k // 5, 3)) * np.array([110.0, 15.0, 5.0]),
    ])
    big = np.concatenate([qs, fill.astype(np.float32)])
    tau0 = R.gate_tau(1.0)
    idx, sqd, _ = R.reference_knn5(big, m, tau0)
    o0, o1 = notes["outside"]                    # the map is what the cases need: beyond the grid, with and without neighbours
    assert (idx[o0:o1, 0] < 0).any() and (idx[o0:o1, 0] >= 0).any()
    tree = oracle.KdTree(m)
    return dict(map=m, qs=qs, big=big, idx=idx, sqd=sqd, tree=tree, notes=notes)


def _check_corr(oracle, c, adv, n):
    feats = adv["big"][:n]
    valid, plane, idx, sqd, s29 = c.find_surf_corr(feats, IDENT)
    want_idx, want_sqd = adv["idx"][:n], adv["sqd"][:n]
    bad = np.nonzero((idx != want_idx).any(1))[0]
    assert len(bad) == 0, (n, len(bad), bad[:5], idx[bad[:3]], want_idx[bad[:3]])
    has = want_idx >= 0
    assert np.array_equal(sqd[has].view(np.uint32), want_sqd[has].view(np.uint32)), n
    cnt, valid_o, plane_o, idx_o, _ = oracle.find_surf_corr(adv["tree"], feats, IDENT, nthreads=8)
    assert np.array_equal(valid, valid_o), (n, np.nonzero(valid != valid_o)[0][:5])
    np.testing.assert_allclose(plane, plane_o, rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(s29, oracle.normal_equations(feats, valid_o, plane_o, IDENT), rtol=1e-9, atol=1e-9)
    return int(has.all(1).sum()), int((~has).all(1).sum())


@pytest.mark.parametrize("shape", SHAPES, ids=_ids)
def test_neighbour_sets_every_query(oracle, adv, shape):
    """(a) One query, an odd count, and more than two warp tasks per warp of the grid: every key of every query."""
    c = _ctx(shape)
    try:
        c.map_set_points(adv["map"])
        per_task = 32 if shape is None else _per_task(shape)
        sizes = [1, len(adv["qs"]), 2 * _sm_count() * KWARPS * per_task + 500]
        for n in sizes:
            full, none = _check_corr(oracle, c, adv, n)
            if n > 1:
                assert full > 0 and none > 0
    finally:
        c.close()


@pytest.fixture(scope="module")
def cases(oracle, world_small):
    """(name, map, feats, start pose, iterations) of the coherence scenarios."""
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    f4 = oracle._f4(ds)
    guess, T = world_small["guess"], world_small["T"]
    far = guess.copy(); far[4:] += np.array([0.4, -0.3, 0.15])
    # duplicates under the queries: at the identity start the world-frame queries sit on five copies each (fifth distance 0)
    fw = oracle._f4(oracle.transform_cloud(ds, T))
    dup_map = np.concatenate([world_small["map"], np.repeat(fw[:400], 5, 0)])
    # one plane (z = 0): x, y and yaw are unobservable; a step the safeguard refuses leaves the pose, so the bound moves by 0
    rng = np.random.default_rng(3)
    g = np.arange(-30.0, 30.0, 0.4)
    X, Y = np.meshgrid(g, g)
    pm = np.ones((X.size, 4), np.float32)
    pm[:, 0] = X.ravel() + rng.uniform(-0.1, 0.1, X.size); pm[:, 1] = Y.ravel() + rng.uniform(-0.1, 0.1, X.size)
    pm[:, 2] = rng.normal(0, 0.005, X.size)
    pf = np.ones((1500, 4), np.float32)
    pf[:, 0] = rng.uniform(-20, 20, 1500); pf[:, 1] = rng.uniform(-20, 20, 1500); pf[:, 2] = -1.5
    half = np.deg2rad(1.0) / 2
    pguess = np.array([np.cos(half), np.sin(half), 0.0, 0.0, 0.3, -0.2, 1.42])
    m, qs, _ = R.adversarial_world(0)
    return [
        ("world_small", world_small["map"], f4, guess, 6),
        ("half_metre_off", world_small["map"], f4, far, 6),
        ("duplicates", dup_map, fw, IDENT, 5),
        ("single_plane", pm, pf, pguess, 5),
        # pass 0 (a full search) leaves fifth distances exactly at the gate, so pass 1 starts from a previous d5 == tau0 and the
        # bound clamps to the gate; how tight the bound itself is, is checked on the host (test_knncore_host.py)
        ("gate", m, qs, IDENT, 4),
    ]


def _assert_pass_equals_full_search(c, feats, pose0, st, exact, what):
    starts = [pose0] + [np.array(s.pose7) for s in st[:-1]]
    for k, (s, p) in enumerate(zip(st, starts)):
        _, _, _, _, s29 = c.find_surf_corr(feats, p)
        assert s.n_corr == int(s29[28]), (what, k, s.n_corr, s29[28])
        got = np.array(list(s.jtj_jtr) + [s.cost])
        want = np.concatenate([s29[:27], s29[27:28]])
        if exact:
            assert got.tobytes() == want.tobytes(), (what, k, got - want)
        else:
            np.testing.assert_allclose(got, want, rtol=1e-12, atol=0, err_msg=f"{what} pass {k}")


@pytest.mark.parametrize("shape", SHAPES, ids=_ids)
def test_coherence_is_exact_pass_by_pass(cases, shape):
    """(b) Every GN pass of scan_to_map (persistent launch, and per-pass launches on a query set whose grid exceeds the SM count)
    and every outer iteration in CERES mode against a full search from the gate at the same start pose: count and sums bit for
    bit.  Forced shapes run the same lanes, rounds and grid in both calls; the unforced plan may pick another shape for the
    correspondence call, so its sums are compared at 1e-12 (counts stay exact)."""
    import liliom_b200 as L
    sm = _sm_count()
    exact = shape is not None
    c = _ctx(shape)
    try:
        for name, m, feats, pose0, iters in cases:
            c.map_set_points(m)
            pose, st = c.scan_to_map(feats, pose0, iters, mode=L.MODE_GN)
            assert np.all(np.isfinite(pose)) and (st[0].n_corr > 0 or name == "gate"), name
            _assert_pass_equals_full_search(c, feats, pose0, st, exact, (shape, name))
        # per-pass launches: the surf sweep cycled to more queries than one block per SM can hold
        name, m, feats, pose0, iters = cases[0]
        per_task = 32 if shape is None else _per_task(shape)
        n_pp = sm * KWARPS * per_task + 1001
        big = np.resize(feats, (n_pp, 4))
        if shape is not None:
            assert _plan_grid(n_pp, shape, sm) > sm
        c.map_set_points(m)
        pose, st = c.scan_to_map(big, pose0, 4, mode=L.MODE_GN)
        _assert_pass_equals_full_search(c, big, pose0, st, exact, (shape, "per_pass"))
        # CERES: outer iteration k linearises at the pose the LM solve of iteration k-1 left
        pose, st = c.scan_to_map(feats, pose0, 3, max_num_iter=15, mode=L.MODE_CERES)
        _assert_pass_equals_full_search(c, feats, pose0, st, exact, (shape, "ceres"))
    finally:
        c.close()


def _stats_bytes(st):
    return [bytes(s) for s in st]


@pytest.mark.parametrize("rounds", [1, 3])
def test_bulk_copy_staging_bit_identical(adv, rounds):
    """(c) The 16-lane search with every run staged by one bulk copy against the same shape through registers, on the adversarial
    map (an 80-point clump: runs longer than a staging tile) and the persistent launch: poses and every pass's sums."""
    import liliom_b200 as L
    qs = adv["qs"]
    assert _plan_grid(len(qs), (16, rounds), _sm_count()) <= _sm_count()      # persistent
    q = np.array([1.0, 0.002, -0.003, 0.001]); q /= np.linalg.norm(q)
    starts = [IDENT, np.concatenate([q, [0.05, -0.04, 0.02]])]
    out = []
    for tma in (False, True):
        c = _ctx((16, rounds), tma=tma)
        try:
            c.map_set_points(adv["map"])
            res = []
            for p0 in starts:
                pose, st = c.scan_to_map(qs, p0, 6, mode=L.MODE_GN)
                res.append((pose.tobytes(), _stats_bytes(st)))
            out.append(res)
        finally:
            c.close()
    assert out[0] == out[1]


@pytest.mark.parametrize("shape", [None, (1, 1), (16, 3)], ids=_ids)
def test_resident_entry_points(cases, shape):
    """(d) upload_feats + scan_to_map_resident(want_stats=True) against scan_to_map on the same features and context."""
    import liliom_b200 as L
    name, m, feats, pose0, iters = cases[0]
    c = _ctx(shape)
    try:
        c.map_set_points(m)
        for mode in (L.MODE_GN, L.MODE_CERES):
            pose_a, st_a = c.scan_to_map(feats, pose0, iters, mode=mode)
            c.upload_feats(feats)
            pose_b, st_b = c.scan_to_map_resident(pose0, iters, mode=mode, want_stats=True)
            assert pose_a.tobytes() == pose_b.tobytes(), mode
            assert _stats_bytes(st_a) == _stats_bytes(st_b), mode
            assert st_a[0].n_corr > 100
    finally:
        c.close()
