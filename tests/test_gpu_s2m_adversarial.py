"""The scan-to-map plane stage (phase B of grid_knn.cu: plane fit, plane-distance gate, weight gate) on the device against the
oracle, bit for bit in its decisions, on neighbourhoods built one float step either side of the plane gate.

Each case sits at its own site, 4 m from every other, so its 5-NN set is exactly the five points built for it.  A patch is a
noisy plane 300 m out; its out-of-plane offsets are scaled by t, and t is bisected with the oracle deciding (plane_thres 0.06)
until the two sides are neighbouring floats; even sites take the kept side, odd sites the refused one.  Without the guard band of
dev_math.cuh::plane_fit_gate the fast fit decides a large share of these pairs differently from the oracle's QR."""
import numpy as np
import pytest

from test_gpu_knn_exact import IDENT, SHAPES, _ctx, _ids

pytestmark = pytest.mark.gpu

PLANE_THRES = 0.06


def _pairs(oracle, n, seed):
    rng = np.random.default_rng(seed)
    g = np.arange(n)
    c = np.array([300.0, -120.0, 40.0]) + 4.0 * np.stack([g % 25, (g // 25) % 25, g // 625], 1) + rng.uniform(0.1, 0.3, (n, 3))
    nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    base = c[:, None, :] + rng.uniform(-0.3, 0.3, (n, 5, 3))
    base -= ((base - c[:, None, :]) * nrm[:, None, :]).sum(2, keepdims=True) * nrm[:, None, :]
    off = rng.uniform(-1, 1, (n, 5, 1)) * nrm[:, None, :]
    q = c.astype(np.float32)

    def make(t):
        m = np.ones((n, 5, 4), np.float32)
        m[:, :, :3] = base + t[:, None, None] * off
        return m

    def decide(t):
        return oracle.fit_gate(make(t), q, PLANE_THRES, -np.inf)[0]

    lo, hi = np.zeros(n), np.full(n, 0.3)
    use = (decide(lo) == 1) & (decide(hi) == 0)              # the sites whose fit does not absorb the offsets (most)
    assert use.sum() > 200
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        kept = decide(mid) == 1
        lo = np.where(kept, mid, lo); hi = np.where(kept, hi, mid)
    keep = g % 2 == 0                                       # even sites one float step inside the gate, odd ones one outside
    return np.where(keep[:, None, None], make(lo), make(hi))[use], q[use], keep[use]


@pytest.fixture(scope="module")
def world(oracle):
    m, q, keep = _pairs(oracle, 1200, 21)
    n = len(q)
    mp = m.reshape(-1, 4)
    feats = np.ones((n, 4), np.float32)
    feats[:, :3] = q
    tree = oracle.KdTree(mp)
    idx, _ = tree.knn5(feats)
    assert (np.sort(idx, 1) == np.arange(5 * n).reshape(n, 5)).all()      # each case's 5-NN set is the set built for it
    cnt, valid, plane, _, _ = oracle.find_surf_corr(tree, feats, IDENT, nthreads=8)
    assert np.array_equal(valid.astype(bool), keep)                       # each case lands on the side it was built for
    return dict(map=mp, feats=feats, tree=tree, valid=valid, plane=plane)


@pytest.mark.parametrize("shape", SHAPES, ids=_ids)
def test_plane_gate_pairs_decided_as_the_oracle(oracle, world, shape):
    """valid equal to the oracle's for every query; the 29 sums equal the oracle's normal equations at 1e-9 and the count exact."""
    c = _ctx(shape)
    try:
        c.map_set_points(world["map"])
        valid, plane, idx, sqd, s29 = c.find_surf_corr(world["feats"], IDENT)
        bad = np.nonzero(valid != world["valid"])[0]
        assert len(bad) == 0, (len(bad), bad[:8])
        assert int(s29[28]) == int(world["valid"].sum())
        ref = oracle.normal_equations(world["feats"], world["valid"], world["plane"], IDENT)
        np.testing.assert_allclose(s29, ref, rtol=1e-9, atol=1e-9)
    finally:
        c.close()


# ---- the adversarial worlds of tests/s2m_adversarial.py (both poses, every case class) ----

import s2m_adversarial as S  # noqa: E402
import reanchor as RA  # noqa: E402
from test_devmath_host import dm, fit_gate_device  # noqa: E402,F401  (the host build of dev_math.cuh, a fixture)


@pytest.fixture(scope="module")
def adv_worlds(oracle, dm):  # noqa: F811
    """Each world with the oracle's correspondences at its pose and, from the host build of plane_fit_gate on the same neighbour
    sets, the cases the exact path decides (every degenerate set and the gate cases inside the guard band)."""
    out = {}
    for w in S.WORLDS:
        W = S.s2m_world(w)
        tree = oracle.KdTree(W["map"])
        _, valid, plane, idx, pw = oracle.find_surf_corr(tree, W["feats"], W["pose"])
        _, path, _, _, _, _, _ = fit_gate_device(dm, W["map"][idx], pw[:, :3], PLANE_THRES, 0.4)
        out[w] = dict(W, tree=tree, valid=valid, plane=plane, idx=idx, exact=path != 0)
    return out


@pytest.mark.parametrize("world", S.WORLDS)
@pytest.mark.parametrize("shape", SHAPES, ids=_ids)
def test_adversarial_world_every_shape(oracle, adv_worlds, world, shape):
    """find_surf_corr at the world's pose: valid and the neighbour sets equal the oracle's for every query; plane bits equal the
    oracle's on every exact-path case; the other planes within the suite's plane tolerance; the sums at 1e-9, the count exact."""
    A = adv_worlds[world]
    c = _ctx(shape)
    try:
        c.map_set_points(A["map"])
        valid, plane, idx, _, s29 = c.find_surf_corr(A["feats"], A["pose"])
        bad = np.nonzero(valid != A["valid"])[0]
        assert len(bad) == 0, (world, bad[:8])
        assert np.array_equal(np.sort(idx, 1), np.sort(A["idx"], 1))
        ex = A["exact"]
        assert ex[S.s2m_world(world)["notes"]["coincident"]].all()
        assert plane[ex].tobytes() == A["plane"][ex].tobytes(), np.nonzero((plane != A["plane"]).any(1) & ex)[0]
        np.testing.assert_allclose(plane, A["plane"], rtol=2e-6, atol=1e-7)
        assert int(s29[28]) == int(A["valid"].sum())
        ref = oracle.normal_equations(A["feats"], A["valid"], A["plane"], A["pose"])
        np.testing.assert_allclose(s29, ref, rtol=1e-9, atol=1e-9)
    finally:
        c.close()


@pytest.mark.parametrize("world", S.WORLDS)
def test_adversarial_world_gn_and_ceres_pass_by_pass(oracle, dm, adv_worlds, world):  # noqa: F811
    """One GN and one Ceres-mode scan_to_map from the world's pose, every pass re-run by the oracle from the device's own start
    pose (reanchor.check_gn / check_ceres): counts exact, flags exact, sums at 1e-9."""
    import liliom_b200 as L
    A = adv_worlds[world]
    c, p = _ctx(None), _ctx(None)
    try:
        c.map_set_points(A["map"]); p.map_set_points(A["map"])
        probe = (lambda pose: p.find_surf_corr(A["feats"], pose)[:2])
        _, st = c.scan_to_map(A["feats"], A["pose"], 4, mode=L.MODE_GN)
        RA.check_gn(oracle, A["tree"], A["feats"], A["pose"], st, dm, 8, f"{world} GN", probe)
        _, st = c.scan_to_map(A["feats"], A["pose"], 3, max_num_iter=15, mode=L.MODE_CERES)
        RA.check_ceres(oracle, A["tree"], A["feats"], A["pose"], st, 15, 8, f"{world} CERES", probe)
    finally:
        c.close(); p.close()


def test_adversarial_sessions_in_a_batch_equal_solo(adv_worlds):
    """scan_to_map_resident_batch_ex with both adversarial sessions beside an ordinary one, in both modes: every session's pose and
    per-pass stats bit-identical to its own solo call."""
    import knn_reference as KR
    import liliom_b200 as L
    m0, q0, _ = KR.adversarial_world(0)
    sessions = [(adv_worlds["near"]["map"], adv_worlds["near"]["feats"], adv_worlds["near"]["pose"]), (m0, q0, IDENT),
                (adv_worlds["far"]["map"], adv_worlds["far"]["feats"], adv_worlds["far"]["pose"])]

    def fresh():
        cs = []
        for m, f, _ in sessions:
            c = _ctx(None); c.map_set_points(m); c.upload_feats(f); cs.append(c)
        return cs
    for mode in (L.MODE_GN, L.MODE_CERES):
        cs = fresh()
        try:
            poses, status, sts = L.scan_to_map_resident_batch_ex(cs, [s[2] for s in sessions], 3, 15, mode=mode, want_stats=True)
            assert (np.asarray(status) == 0).all()
        finally:
            for c in cs:
                c.close()
        cs = fresh()
        try:
            for k, (c, s) in enumerate(zip(cs, sessions)):
                pose, st = c.scan_to_map_resident(s[2], 3, 15, mode=mode, want_stats=True)
                assert pose.tobytes() == np.asarray(poses[k]).tobytes(), (mode, k)
                assert [bytes(x) for x in st] == [bytes(x) for x in sts[k]], (mode, k)
        finally:
            for c in cs:
                c.close()


def test_guard_band_rate_on_benchmark_sweep(oracle, dm):  # noqa: F811
    """How often plane_fit_gate leaves the fast fit on the benchmark's workload (bench.py: a Livox-Horizon sweep against the
    1 M-point synthetic map): every GN pass's own neighbour sets, read back from the device (find_surf_corr at the pass's start
    pose), through the host build of plane_fit_gate.  Reported, and held to be a cold path."""
    import bench
    import liliom_b200 as L
    m, sweeps = bench.make_workload("horizon", 1_000_000, 1)
    sw = sweeps[0]
    surf, _, _ = oracle.extract_horizon(sw["pts"], sw["q"])
    feats = oracle._f4(oracle.voxelgrid(surf, 0.4))
    body = np.zeros(len(feats), oracle.PT48)
    body["x"], body["y"], body["z"], body["w"] = feats[:, 0], feats[:, 1], feats[:, 2], 1.0
    c = _ctx(None)
    try:
        c.map_set_points(m)
        _, st = c.scan_to_map(feats, sw["guess"], 6, mode=L.MODE_GN)
        counts = np.zeros(3, np.int64)
        for start in RA.start_poses(sw["guess"], st):
            _, _, idx, sqd, _ = c.find_surf_corr(feats, start)
            live = (idx >= 0).all(1) & (sqd[:, 4] < 1.0)
            w = oracle.transform_cloud(body, start)
            pw = np.stack([w["x"], w["y"], w["z"]], 1)[live]
            mm = np.ascontiguousarray(m, np.float32).reshape(-1, 4)[idx[live]]
            _, path, _, _, _, _, _ = fit_gate_device(dm, mm, pw, PLANE_THRES, 0.4)
            counts += np.bincount(path, minlength=3)
    finally:
        c.close()
    n = int(counts.sum())
    print(f"guard band on the benchmark sweep: {n} fits over 6 passes, fast {counts[0]}, declined {counts[1]}, "
          f"guard band {counts[2]} ({counts[2] / n:.3%})")
    assert n > 5000 and counts[2] < 0.05 * n
