"""GPU parity AT THE BASELINE SIZES (VERDICT r1 "What's weak" #1): the CUDA path against the CPU oracle on the
configs' own workloads — not only on the 100 k-point toy world.
  configs[1]  24k-pt Horizon sweep vs 1 M-pt map, 10 GN iterations (and the Ceres-faithful mode)
  configs[2]  130k-pt HDL-64E sweep through the ROT extractor (ds_rate 4) vs 2 M-pt map
  configs[3]  24k-pt sweep vs 5 M-pt map on ONE GPU (the sharded runs are compared with this pose by tools/multi_check.py)
Bit-exact: feature clouds, down-sampled scan, accepted 5-NN index sets, accept flags, correspondence counts.
Tolerance (BASELINE.json): pose within 1e-4 m / 1e-4 rad at equal iteration count."""
import numpy as np
import pytest

from test_devmath_host import dm  # noqa: F401  (the host build of dev_math.cuh, a fixture)
from test_gpu_reanchored import _gn, probe_of

pytestmark = pytest.mark.gpu

F48 = ["x", "y", "z", "nx", "ny", "nz", "intensity", "curvature"]
F32 = ["x", "y", "z", "intensity"]


def _fields_equal(a, b, fields):
    assert len(a) == len(b), (len(a), len(b))
    for f in fields:
        assert np.array_equal(a[f].view(np.uint32), b[f].view(np.uint32)), f


def _rot_angle(qa, qb):
    qa = np.asarray(qa) / np.linalg.norm(qa); qb = np.asarray(qb) / np.linalg.norm(qb)
    return 2.0 * np.arccos(min(1.0, abs(float(np.dot(qa, qb)))))


def _pose_close(a, b, tol_t=1e-4, tol_r=1e-4):
    assert np.linalg.norm(np.asarray(a)[4:] - np.asarray(b)[4:]) < tol_t, (a, b)
    assert _rot_angle(a[:4], b[:4]) < tol_r, (a, b)


def _s2m_parity(c, oracle, tree, ds_o, guess, T, iters=10, nthreads=8):
    import liliom_b200 as L
    # correspondences at the start pose: accept flags, accepted index sets and squared distances exact
    cnt, valid_o, plane_o, idx_o, pw_o = oracle.find_surf_corr(tree, ds_o, guess, nthreads)
    valid, plane, idx, sqd, s29 = c.find_surf_corr(ds_o, guess)
    _, sqd_o = tree.knn5(pw_o, nthreads)
    inside = sqd_o[:, 4] < 1.0
    assert inside.sum() > 0.5 * len(ds_o)
    assert np.array_equal(idx[inside], idx_o[inside])
    assert np.array_equal(sqd[inside].view(np.uint32), sqd_o[inside].view(np.uint32))
    assert np.array_equal(valid, valid_o) and int(valid.sum()) == cnt
    np.testing.assert_allclose(plane, plane_o, rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(s29, oracle.normal_equations(ds_o, valid_o, plane_o, guess), rtol=1e-9, atol=1e-9)
    # GN mode, iteration by iteration
    rc, pose_o, st_o = oracle.scan_to_map_gn(tree, ds_o, guess, iters, nthreads)
    pose, st = c.scan_to_map(ds_o, guess, iters, mode=L.MODE_GN)
    assert rc == 0 and st[0].n_corr == st_o[0].n_corr
    for a, b in zip(st, st_o):
        assert abs(a.n_corr - b.n_corr) <= 2        # a gate sitting on its threshold may flip once the poses differ by 1e-12
        _pose_close(np.array(a.pose7), np.array(b.pose7))
    _pose_close(pose, pose_o)
    _pose_close(pose, T, tol_t=0.03, tol_r=0.01)
    # Ceres-faithful mode: same LM iteration counts, same correspondences
    rc, pose_c, st_c = oracle.scan_to_map_ceres(tree, ds_o, guess, 2, 15, nthreads)
    pose2, st2 = c.scan_to_map(ds_o, guess, 2, max_num_iter=15, mode=L.MODE_CERES)
    assert [s.lm_iters for s in st2] == [s.lm_iters for s in st_c]
    assert [s.n_corr for s in st2] == [s.n_corr for s in st_c]
    _pose_close(pose2, pose_c)
    return pose


def test_config1_horizon_sweep_vs_1m_map(oracle):
    import liliom_b200 as L
    from liliom_b200 import synth
    m, _ = synth.make_map(1_000_000)
    T = synth.default_true_pose()
    pts, q = synth.make_horizon_sweep(T)
    guess = synth.perturbed_pose(T)
    c = L.Context(variant=0)
    c.map_set_points(m)
    surf, edge, cut = c.extract_horizon(pts, q)
    surf_o, edge_o, cut_o = oracle.extract_horizon(pts, q)
    _fields_equal(surf, surf_o, F48); _fields_equal(edge, edge_o, F48); _fields_equal(cut, cut_o, F48)
    ds_o = oracle.voxelgrid(surf_o, 0.4)
    tree = oracle.KdTree(m)
    pose = _s2m_parity(c, oracle, tree, ds_o, guess, T)
    # the node-facing call (VoxelGrid + persistent GN kernel with the device-side query count) gives the same pose bits
    pose_n, st, ds = c.odometry(surf, guess, 10, mode=L.MODE_GN)
    _fields_equal(ds, ds_o, F48)
    _pose_close(pose_n, pose, 1e-9, 1e-9)
    # dense: every surf feature a query (the roofline micro-run's shape, one thread per query)
    rc, pose_o, _ = oracle.scan_to_map_gn(tree, surf_o, guess, 6, 8)
    pose_d, _ = c.scan_to_map(surf, guess, 6, mode=L.MODE_GN)
    _pose_close(pose_d, pose_o)
    c.close()


def test_config2_hdl64_sweep_vs_2m_map(oracle):
    import liliom_b200 as L
    from liliom_b200 import synth
    m, _ = synth.make_map(2_000_000)
    T = synth.default_true_pose()
    pts, q = synth.make_hdl64_sweep(T)
    assert len(pts) > 120_000
    guess = synth.perturbed_pose(T)
    c = L.Context(variant=1)                      # LiLi-OM-ROT defaults: 32-byte points, 64 lines, ds_rate 4
    c.map_set_points(m)
    rc, surf_o, edge_o, cut_o, lab_o, cur_o = oracle.extract_rot(pts, q, (1.0, 0, 0, 0), 64, 4)
    surf, edge, cut = c.extract_rot(pts, q)
    lab, cur = c.extract_rot_labels(len(cut))
    _fields_equal(cut, cut_o, F32); _fields_equal(edge, edge_o, F32); _fields_equal(surf, surf_o, F32)
    assert np.array_equal(lab, lab_o) and np.array_equal(cur.view(np.uint32), cur_o.view(np.uint32))
    ds_o = oracle.voxelgrid(surf_o, 0.4)
    tree = oracle.KdTree(m)
    _s2m_parity(c, oracle, tree, ds_o, guess, T)
    pose_n, st, ds = c.odometry(surf, guess, 10, mode=L.MODE_GN)
    _fields_equal(ds, ds_o, F32)
    rc, pose_o, _ = oracle.scan_to_map_gn(tree, ds_o, guess, 10, 8)
    _pose_close(pose_n, pose_o)
    c.close()


def test_config3_horizon_sweep_vs_5m_map_single_gpu(oracle):
    import liliom_b200 as L
    from liliom_b200 import synth
    m, _ = synth.make_map(5_000_000)
    T = synth.default_true_pose()
    pts, q = synth.make_horizon_sweep(T)
    guess = synth.perturbed_pose(T)
    c = L.Context(variant=0)
    c.map_set_points(m)
    surf_o, _, _ = oracle.extract_horizon(pts, q)
    ds_o = oracle.voxelgrid(surf_o, 0.4)
    tree = oracle.KdTree(m)
    _s2m_parity(c, oracle, tree, ds_o, guess, T)
    c.close()


def test_rot_extract_32_lines(oracle, world_small):
    """The 32-line ring table (R/src/Preprocessing.cpp:325-331): scanID = int((angle + 92/3) * 3/4)."""
    import liliom_b200 as L
    p = L.default_params(1); p.line_num = 32; p.ds_rate = 1
    c = L.Context(p)
    pts = world_small["hdl"][::2].copy()
    q_lb = np.array([0.9995, -0.02, 0.01, 0.015]); q_lb /= np.linalg.norm(q_lb)
    rc, surf_o, edge_o, cut_o, lab_o, cur_o = oracle.extract_rot(pts, world_small["q_hdl"], q_lb, 32, 1)
    assert rc == 0
    rings = np.floor(cut_o["intensity"]).astype(int)
    assert rings.min() >= 0 and rings.max() <= 31 and len(np.unique(rings)) >= 12      # the table is exercised over many rings
    surf, edge, cut = c.extract_rot(pts, world_small["q_hdl"], q_lb)
    lab, cur = c.extract_rot_labels(len(cut))
    _fields_equal(cut, cut_o, F32)
    assert np.array_equal(lab, lab_o) and np.array_equal(cur.view(np.uint32), cur_o.view(np.uint32))
    _fields_equal(edge, edge_o, F32); _fields_equal(surf, surf_o, F32)
    assert len(edge) > 20 and len(surf) > 500
    # points outside the table's range are dropped (scanID < 0 or > 31), in both
    hi = pts.copy(); hi["z"][::5] = np.abs(hi["z"][::5]) + 0.5 * np.hypot(hi["x"][::5], hi["y"][::5])
    rc, surf_o, edge_o, cut_o, _, _ = oracle.extract_rot(hi, world_small["q_hdl"], q_lb, 32, 1)
    surf, edge, cut = c.extract_rot(hi, world_small["q_hdl"], q_lb)
    _fields_equal(cut, cut_o, F32); _fields_equal(edge, edge_o, F32); _fields_equal(surf, surf_o, F32)
    c.close()


def test_gn_step_stays_bounded_on_a_single_plane(oracle):
    """ADVICE r1: the GN mode's step on degenerate geometry.  The map is ONE plane (z = 0): translation in x/y and yaw are
    unobservable, J^T J is singular up to rounding.  The undamped LDL^T step used to be free to return anything; with the
    conditioning test + Levenberg re-solve + trust region the pose must stay near the guess in the unobservable directions,
    converge in the observable ones (z, roll, pitch), and agree with the oracle's identical safeguard."""
    import liliom_b200 as L
    rng = np.random.default_rng(3)
    g = np.arange(-30.0, 30.0, 0.4)
    X, Y = np.meshgrid(g, g)
    m = np.ones((X.size, 4), np.float32)
    m[:, 0] = (X.ravel() + rng.uniform(-0.1, 0.1, X.size)); m[:, 1] = (Y.ravel() + rng.uniform(-0.1, 0.1, X.size))
    m[:, 2] = rng.normal(0, 0.005, X.size)
    feats = np.ones((1500, 4), np.float32)
    feats[:, 0] = rng.uniform(-20, 20, 1500); feats[:, 1] = rng.uniform(-20, 20, 1500); feats[:, 2] = -1.5      # body frame: ground 1.5 m below
    half = np.deg2rad(1.0) / 2
    guess = np.array([np.cos(half), np.sin(half), 0.0, 0.0, 0.3, -0.2, 1.42])       # true pose: identity rotation, t = (0, 0, 1.5)
    c = L.Context(variant=0)
    c.map_set_points(m)
    tree = oracle.KdTree(m)
    pose, st = c.scan_to_map(feats, guess, 10, mode=L.MODE_GN)
    rc, pose_o, st_o = oracle.scan_to_map_gn(tree, feats, guess, 10)
    assert st[0].n_corr > 1000
    assert np.all(np.isfinite(pose))
    assert abs(pose[6] - 1.5) < 0.01 and abs(pose[1]) < 2e-3 and abs(pose[2]) < 2e-3          # observable: height, roll, pitch
    assert abs(pose[4] - guess[4]) < 1.0 and abs(pose[5] - guess[5]) < 1.0 and abs(pose[3]) < 0.2   # unobservable: bounded
    assert abs(pose[6] - pose_o[6]) < 1e-4 and abs(pose[1] - pose_o[1]) < 1e-5 and abs(pose[2] - pose_o[2]) < 1e-5
    for s in st:
        assert np.all(np.isfinite(np.array(s.pose7)))
    c.close()


def test_persistent_barrier_stress(oracle, dm, world_small):  # noqa: F811
    """VERDICT r1 'What's weak' #7: the persistent GN kernel's grid barrier.  Many launches with varying grid sizes and
    iteration counts, six times over: every repetition's poses and per-iteration sums must equal the first's bit for bit, and
    every pass of the first is re-anchored against the oracle (tests/reanchor.py) with the device's own correspondences from a
    second context's find_surf_corr, the per-pass kernel, which has no grid barrier.  A stale or missing block partial read past
    the barrier would show up as a differing sum: it cannot meet the sums' rtol of 1e-9."""
    import liliom_b200 as L
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    tree, guess = oracle.KdTree(world_small["map"]), world_small["guess"]
    rng = np.random.default_rng(17)
    scans = [ds[rng.permutation(len(ds))[: int(n)]] for n in rng.integers(40, len(ds), 24)]
    c, pc = L.Context(variant=0), L.Context(variant=0)
    try:
        c.map_set_points(world_small["map"]); pc.map_set_points(world_small["map"])
        ref = []
        for rep in range(6):
            for k, f in enumerate(scans):
                pose, st = c.scan_to_map(f, guess, 3 + (k % 9), mode=L.MODE_GN)
                out = pose.tobytes() + b"".join(np.array(s.jtj_jtr).tobytes() for s in st)
                if rep == 0:
                    ref.append(out)
                    _gn(oracle, dm, tree, f, guess, st, f"barrier stress/scan {k} ({len(f)} queries)", probe_of(pc, f))
                else:
                    assert out == ref[k], (rep, k)
    finally:
        c.close(); pc.close()
