"""CPU tests of the oracle (no GPU): the from-knowledge restatements of Eigen / PCL / FLANN / Ceres
against independent NumPy / SciPy implementations, and the committed golden vectors.
The reference ships no tests or fixtures ("parity unpinned"): these checks are what pins the oracle."""
import os

import numpy as np
import pytest
from scipy.optimize import least_squares
from scipy.spatial import cKDTree

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def ceres_plus(x, d):
    nd = np.linalg.norm(d[:3])
    out = np.array(x, float)
    if nd > 0:
        dq = np.concatenate([[np.cos(nd)], np.sin(nd) / nd * d[:3]])
        aw, ax, ay, az = dq; bw, bx, by, bz = x[:4]
        out[:4] = [aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                   aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx]
    out[4:] = x[4:] + d[3:]
    return out


def test_eigen_sym3_matches_numpy(oracle):
    rng = np.random.default_rng(0)
    for k in range(200):
        B = rng.normal(size=(3, 3)) * 10.0 ** rng.integers(-3, 3)
        A = B @ B.T if k % 2 else (B + B.T)
        ev, vec = oracle.eigen_sym3(A)
        w, v = np.linalg.eigh(A)
        np.testing.assert_allclose(ev, w, rtol=1e-10, atol=1e-12 * np.abs(w).max())
        assert np.all(np.diff(ev) >= 0)
        np.testing.assert_allclose(A @ vec, vec * ev, atol=1e-9 * max(1.0, np.abs(w).max()))
        np.testing.assert_allclose(vec.T @ vec, np.eye(3), atol=1e-12)
    ev, vec = oracle.eigen_sym3(np.zeros((3, 3)))
    assert np.all(ev == 0)
    ev, vec = oracle.eigen_sym3(np.diag([3.0, 1.0, 2.0]))
    np.testing.assert_allclose(ev, [1, 2, 3])


def test_colpiv_qr_matches_lstsq(oracle):
    rng = np.random.default_rng(1)
    for _ in range(200):
        c = rng.uniform(-300, 300, 3)
        n = rng.normal(size=3); n /= np.linalg.norm(n)
        P = c + rng.uniform(-0.6, 0.6, (5, 3))
        P -= np.outer((P - c) @ n, n) * 0.98          # nearly planar patch far from the origin
        x = oracle.colpiv_qr_solve(P, -np.ones(5))
        ref, *_ = np.linalg.lstsq(P, -np.ones(5), rcond=None)
        np.testing.assert_allclose(x, ref, rtol=1e-6, atol=1e-9)
    # rank-deficient (collinear) input: solution has a zero component, like Eigen's nonzero_pivots handling
    t = np.linspace(0, 1, 5)[:, None]
    P = np.array([10.0, 5.0, 1.0]) + t * np.array([0.0, 0.0, 1.0])
    x = oracle.colpiv_qr_solve(P, -np.ones(5))
    assert np.isfinite(x).all() and (x == 0).sum() >= 1
    np.testing.assert_allclose(P @ x, -1, atol=1e-9)


def test_slerp_matches_closed_form(oracle):
    q = np.array([0.99995, 0.0, 0.0, 0.0099995])
    for t in (0.0, 0.3, 1.0):
        out = oracle.slerp_identity(q, t)
        th = np.arccos(q[0])          # q is (almost) unit
        np.testing.assert_allclose(out[0], np.sin((1 - t) * th) / np.sin(th) + np.sin(t * th) / np.sin(th) * q[0], rtol=1e-12)
    np.testing.assert_allclose(oracle.slerp_identity([1, 0, 0, 0], 0.4), [1, 0, 0, 0])


def test_voxelgrid_matches_numpy(oracle, world_small):
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    for leaf in (0.4, 0.6):
        got = oracle.voxelgrid(surf, leaf)
        inv = np.float32(1.0) / np.float32(leaf)
        xyz = np.stack([surf["x"], surf["y"], surf["z"]], 1)
        ijk = np.floor(xyz * inv).astype(np.int64)
        mn = ijk.min(0); div = ijk.max(0) - mn + 1
        idx = (ijk[:, 0] - mn[0]) + (ijk[:, 1] - mn[1]) * div[0] + (ijk[:, 2] - mn[2]) * div[0] * div[1]
        uniq, inv_idx, counts = np.unique(idx, return_inverse=True, return_counts=True)
        assert len(got) == len(uniq)
        for f in ("x", "y", "z", "intensity", "curvature"):
            acc = np.zeros(len(uniq), np.float32)
            np.add.at(acc, inv_idx, surf[f])            # sequential fp32 accumulation in index order
            np.testing.assert_array_equal(got[f], acc / counts.astype(np.float32))
        nrm = np.sqrt(got["nx"] ** 2 + got["ny"] ** 2 + got["nz"] ** 2)
        np.testing.assert_allclose(nrm, 1.0, atol=1e-5)


def test_kdtree_matches_scipy_and_brute(oracle, world_small):
    m = world_small["map"][:20000]
    rng = np.random.default_rng(3)
    q = m[rng.integers(0, len(m), 500)].copy()
    q[:, :3] += rng.normal(0, 0.3, (500, 3)).astype(np.float32)
    tree = oracle.KdTree(m)
    idx, sqd = tree.knn5(q)
    bidx, bsqd = oracle.knn5_brute(m, q)
    assert np.array_equal(idx, bidx) and np.array_equal(sqd.view(np.uint32), bsqd.view(np.uint32))
    d, ii = cKDTree(m[:, :3].astype(np.float64)).query(q[:, :3].astype(np.float64), k=5)
    assert (np.sort(idx, 1) == np.sort(ii, 1)).all(1).mean() > 0.995   # fp32-vs-fp64 near-ties only
    np.testing.assert_allclose(np.sqrt(sqd), d, rtol=1e-4, atol=1e-5)
    assert np.all(np.diff(sqd, axis=1) >= 0)
    # fewer than 5 points: padded with -1 / inf
    t3 = oracle.KdTree(m[:3])
    i3, d3 = t3.knn5(q[:2])
    assert (i3[:, 3:] == -1).all() and np.isinf(d3[:, 3:]).all()


def test_gradient_matches_finite_differences(oracle, world_small):
    """J^T r from the closed-form/autodiff-faithful rows == d(cost)/d(delta) through ceres Plus."""
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    tree = oracle.KdTree(world_small["map"])
    pose = world_small["guess"]
    cnt, valid, plane, idx, pw = oracle.find_surf_corr(tree, ds, pose)
    s = oracle.normal_equations(ds, valid, plane, pose)
    g = s[21:27]
    h = 1e-6
    for k in range(6):
        d = np.zeros(6); d[k] = h
        cp = oracle.normal_equations(ds, valid, plane, ceres_plus(pose, d))[27]
        cm = oracle.normal_equations(ds, valid, plane, ceres_plus(pose, -d))[27]
        assert abs((cp - cm) / (2 * h) - g[k]) < 1e-5 * max(1.0, abs(g[k])), (k, (cp - cm) / (2 * h), g[k])
    assert s[28] == cnt


def test_ceres_lm_matches_scipy_huber(oracle, world_small):
    """ceres::Solve restatement vs scipy least_squares(loss='huber', f_scale=0.1) on the same frozen correspondences."""
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    tree = oracle.KdTree(world_small["map"])
    pose0 = world_small["guess"]
    cnt, valid, plane, _, _ = oracle.find_surf_corr(tree, ds, pose0)
    iters, pose_c, cost_c = oracle.ceres_solve(ds, valid, plane, pose0, 50)
    P = np.stack([ds["x"], ds["y"], ds["z"]], 1).astype(np.float64)[valid == 1]
    N = plane[valid == 1, :3].astype(np.float64); D = plane[valid == 1, 3].astype(np.float64)

    def res(d):
        x = ceres_plus(pose0, d)
        qv = x[1:4]
        uv = 2.0 * np.cross(qv, P)
        pw = P + x[0] * uv + np.cross(qv, uv) + x[4:]
        return (N * pw).sum(1) + D
    sol = least_squares(res, np.zeros(6), loss="huber", f_scale=0.1, xtol=1e-14, ftol=1e-14, gtol=1e-14)
    pose_s = ceres_plus(pose0, sol.x)
    assert np.linalg.norm(pose_c[4:] - pose_s[4:]) < 2e-5
    assert abs(abs(np.dot(pose_c[:4], pose_s[:4])) - 1.0) < 1e-9
    assert abs(cost_c - sol.cost) < 1e-6 * max(1.0, sol.cost)
    assert 1 <= iters <= 50


def test_scan_to_map_recovers_true_pose(oracle, world_small):
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    tree = oracle.KdTree(world_small["map"])
    T = world_small["T"]
    rc, pose, st = oracle.scan_to_map_gn(tree, ds, world_small["guess"], 10)
    assert rc == 0 and np.linalg.norm(pose[4:] - T[4:]) < 0.02
    rc, pose2, st2 = oracle.scan_to_map_ceres(tree, ds, world_small["guess"], 2, 15)
    assert rc == 0 and np.linalg.norm(pose2[4:] - T[4:]) < 0.02 and pose2[0] > 0
    rc, pose3, _ = oracle.scan_to_map_gn(oracle.KdTree(world_small["map"][:5]), ds, world_small["guess"], 2)
    assert rc == -1 and np.array_equal(pose3, world_small["guess"])      # < 10 map points: pose untouched


def test_horizon_extractor_structure(oracle, world_small):
    surf, edge, cut = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    assert len(cut) == len(world_small["hz"])
    assert len(surf) > 5000 and 0 < len(edge) < len(surf)
    assert (surf["curvature"] > 0).all() and (edge["curvature"] > 0).all()
    for c in (surf, edge):
        n = np.sqrt(c["nx"] ** 2 + c["ny"] ** 2 + c["nz"] ** 2)
        np.testing.assert_allclose(n, 1.0, atol=1e-5)
    # surf points of one patch share one normal and lie on a plane through the patch
    line = surf["intensity"].astype(np.int32)
    assert set(np.unique(line)) <= set(range(6))


def test_rot_extractor_structure(oracle, world_small):
    rc, surf, edge, cut, lab, cur = oracle.extract_rot(world_small["hdl"], world_small["q_hdl"], (1, 0, 0, 0), 64, 1)
    assert rc == 0 and len(cut) > 80000
    ring = cut["intensity"].astype(np.int32)
    assert np.all(np.diff(ring) >= -1) and ring.max() <= 50          # bucketed by ring, rings > 50 dropped
    assert set(np.unique(lab)) <= {-1, 0, 1, 2}
    assert (lab == 2).sum() <= 2 * 6 * 51 and (lab == -1).sum() <= 4 * 6 * 51
    assert (cur[lab > 0] > 2.0).all() and (cur[lab == -1] < 0.1).all()
    assert len(edge) == (lab > 0).sum()
    assert oracle.extract_rot(world_small["hdl"], world_small["q_hdl"], (1, 0, 0, 0), 20, 1)[0] == -2


# ---------------------------------------------------------------- golden vectors (tests/golden, made by tests/make_golden.py)
def _same(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape
    assert a.tobytes() == b.tobytes()


def test_golden_horizon(oracle):
    g = np.load(os.path.join(GOLD, "horizon_small.npz"))
    surf, edge, cut = oracle.extract_horizon(g["pts"].view(oracle.PT48).reshape(-1), g["q_imu"], float(g["surf_thres"]), float(g["edge_thres"]))
    _same(surf.view(np.uint8), g["surf"]); _same(edge.view(np.uint8), g["edge"]); _same(cut.view(np.uint8), g["cut"])
    _same(oracle.voxelgrid(surf, 0.4).view(np.uint8), g["surf_ds"])


def test_golden_rot(oracle):
    g = np.load(os.path.join(GOLD, "rot_small.npz"))
    rc, surf, edge, cut, lab, cur = oracle.extract_rot(g["pts"].view(oracle.PT32).reshape(-1), g["q_imu"], g["q_lb"], int(g["line_num"]), int(g["ds_rate"]))
    _same(surf.view(np.uint8), g["surf"]); _same(edge.view(np.uint8), g["edge"]); _same(cut.view(np.uint8), g["cut"])
    _same(lab, g["label"]); _same(cur, g["curv"])


def test_golden_scan_to_map(oracle):
    g = np.load(os.path.join(GOLD, "s2m_small.npz"))
    tree = oracle.KdTree(g["map"])
    cnt, valid, plane, idx, pw = oracle.find_surf_corr(tree, g["feats"], g["pose0"])
    _same(valid, g["valid"]); _same(plane, g["plane"]); _same(idx, g["nn_idx"])
    np.testing.assert_allclose(oracle.normal_equations(g["feats"], valid, plane, g["pose0"]), g["neq29"], rtol=1e-13)
    rc, pose, st = oracle.scan_to_map_gn(tree, g["feats"], g["pose0"], 6)
    np.testing.assert_allclose(pose, g["pose_gn6"], rtol=0, atol=1e-12)
    rc, pose, st = oracle.scan_to_map_ceres(tree, g["feats"], g["pose0"], 2, 15)
    np.testing.assert_allclose(pose, g["pose_ceres"], rtol=0, atol=1e-12)
    assert [s.lm_iters for s in st] == list(g["ceres_lm_iters"])


def test_kdtree_matches_real_flann_kdtree_single(oracle, world_small):
    """Third-party pin: OpenCV vendors the FLANN sources (cv::flann), including the very index class PCL's KdTreeFLANN
    instantiates — KDTreeSingleIndex (algorithm 4), leaf_max_size 15 by default in PCL, SearchParams(checks=-1, eps=0,
    sorted=true) (L/src/LidarOdometry.cpp:490,360 through pcl::KdTreeFLANN).  The oracle's from-knowledge kd-tree must
    return the same neighbours in the same order with bit-identical fp32 squared distances, except where FLANN's own
    tie order (equal distances) is unspecified."""
    cv2 = pytest.importorskip("cv2")
    if not hasattr(cv2, "flann_Index"):
        pytest.skip("this OpenCV build has no flann module")
    m = world_small["map"][:60000]
    xyz = np.ascontiguousarray(m[:, :3], dtype=np.float32)
    rng = np.random.default_rng(11)
    q = m[rng.integers(0, len(m), 3000)].copy()
    q[:, :3] += rng.normal(0, 0.35, (3000, 3)).astype(np.float32)
    index = cv2.flann_Index(xyz, dict(algorithm=4, leaf_max_size=15, reorder=True))       # FLANN_INDEX_KDTREE_SINGLE
    fi, fd = index.knnSearch(np.ascontiguousarray(q[:, :3]), 5, params=dict(checks=-1, eps=0.0, sorted=True))
    idx, sqd = oracle.KdTree(m).knn5(q)
    # distances: FLANN's L2 functor accumulates (dx*dx + dy*dy) + dz*dz in fp32 — same bits as the oracle
    assert np.array_equal(sqd.view(np.uint32), fd.astype(np.float32).view(np.uint32))
    same = (idx == fi)
    tie = np.zeros_like(same)
    tie[:, 1:] |= sqd[:, 1:] == sqd[:, :-1]
    tie[:, :-1] |= sqd[:, :-1] == sqd[:, 1:]
    assert (same | tie).all()
    assert same.mean() > 0.999
    # the 5th-neighbour gate (:365) therefore decides identically
    assert np.array_equal(sqd[:, 4] < 1.0, fd[:, 4] < 1.0)


# ---------------------------------------------------------------- §8 (f1): backend LiDAR factor blocks
def _backend_case(oracle, world_small):
    """Edge + surf correspondences of one 'keyframe' against the small world, searched at the LiDAR pose."""
    surf, edge, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    tree = oracle.KdTree(world_small["map"])
    pose_l = world_small["guess"]
    ds = oracle.voxelgrid(surf, 0.4)
    sv, plane, score = oracle.correspond_surf_backend(tree, ds, pose_l, 1.0, 0.06, 0.2, 0.6)
    # line features: query the planar map with jittered copies of map points lying on the poles' neighbourhood
    ev, pa, pb = oracle.correspond_edge(tree, edge, pose_l, 0)
    return dict(ds=ds, sv=sv, plane=plane, score=score, edge=edge, ev=ev, pa=pa, pb=pb, pose_l=pose_l)


def _fd_gradient(block_fn, pose, h=1e-6):
    """d(cost)/d(delta) through Ceres' Plus, delta = [dt, drot] (parameter block order t, q)."""
    g = np.zeros(6)
    for k in range(6):
        d = np.zeros(6); d[k] = h
        # ceres_plus takes [rot, trans]
        dp = np.concatenate([d[3:], d[:3]])
        cp = block_fn(ceres_plus(pose, dp))[27]
        cm = block_fn(ceres_plus(pose, -dp))[27]
        g[k] = (cp - cm) / (2 * h)
    return g


def test_backend_surf_block_gradient_and_structure(oracle, world_small):
    c = _backend_case(oracle, world_small)
    assert c["sv"].sum() > 200
    q_lb = np.array([0.9990482, 0.0, 0.0436194, 0.0]); t_lb = np.array([0.05, -0.02, 0.10])     # 5 deg pitch + lever arm
    # body pose such that body∘extrinsic⁻¹ = lidar pose:  q_b = q_l*q_lb, t_b = t_l + q_l... keep it simple: evaluate anywhere
    pose_b = np.array(c["pose_l"])
    fn = lambda x: oracle.backend_surf_block(c["ds"], c["sv"], c["plane"], c["score"], x, q_lb, t_lb, 1.0)
    s = fn(pose_b)
    assert s[28] == c["sv"].sum() and s[27] > 0
    g = _fd_gradient(fn, pose_b)
    np.testing.assert_allclose(s[21:27], g, rtol=2e-5, atol=1e-7)
    # H is the Gauss-Newton block: symmetric PSD by construction
    H = np.zeros((6, 6)); H[np.triu_indices(6)] = s[:21]; H = H + np.triu(H, 1).T
    assert np.linalg.eigvalsh(H).min() > -1e-9
    # with identity extrinsics, score 1 and a huge Cauchy width the block equals the LidarOdometry plane block
    # (orc_normal_equations: Huber never active for |r| < a, tangent order [rot, trans])
    ones = np.ones(len(c["ds"]))
    s1 = oracle.backend_surf_block(c["ds"], c["sv"], c["plane"], ones, pose_b, (1, 0, 0, 0), (0, 0, 0), 1e9)
    s2 = oracle.normal_equations(c["ds"], c["sv"], c["plane"], pose_b, a=1e9)
    H2 = np.zeros((6, 6)); H2[np.triu_indices(6)] = s2[:21]; H2 = H2 + np.triu(H2, 1).T
    perm = [3, 4, 5, 0, 1, 2]
    H1 = np.zeros((6, 6)); H1[np.triu_indices(6)] = s1[:21]; H1 = H1 + np.triu(H1, 1).T
    np.testing.assert_allclose(H1, H2[np.ix_(perm, perm)], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(s1[21:27], s2[21:27][perm], rtol=1e-9, atol=1e-12)


def test_backend_edge_block_gradient(oracle, world_small):
    rng = np.random.default_rng(5)
    # synthetic lines: 400 features scattered around vertical segments, endpoints a/b = centre +- 0.1 u
    n = 400
    ctr = rng.uniform(-20, 20, (n, 3)); u = rng.normal(size=(n, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    pa = (ctr + 0.1 * u).astype(np.float32); pb = (ctr - 0.1 * u).astype(np.float32)
    pose = world_small["guess"]
    Rm = lambda q: np.array([[1 - 2 * (q[2] ** 2 + q[3] ** 2), 2 * (q[1] * q[2] - q[0] * q[3]), 2 * (q[1] * q[3] + q[0] * q[2])],
                             [2 * (q[1] * q[2] + q[0] * q[3]), 1 - 2 * (q[1] ** 2 + q[3] ** 2), 2 * (q[2] * q[3] - q[0] * q[1])],
                             [2 * (q[1] * q[3] - q[0] * q[2]), 2 * (q[2] * q[3] + q[0] * q[1]), 1 - 2 * (q[1] ** 2 + q[2] ** 2)]])
    world_pts = ctr + rng.uniform(-1, 1, (n, 1)) * u + rng.normal(0, 0.05, (n, 3))
    body = (world_pts - pose[4:]) @ Rm(pose[:4])          # R^T (p - t)
    feats = np.ones((n, 4), np.float32); feats[:, :3] = body
    valid = (rng.random(n) < 0.8).astype(np.uint8)
    fn = lambda x: oracle.backend_edge_block(feats, valid, pa, pb, 0.6, x, 1.0)
    s = fn(pose)
    assert s[28] == valid.sum()
    # residual = s * point-to-line distance: check the cost against a direct evaluation
    lp = feats[valid == 1, :3].astype(np.float64) @ Rm(pose[:4]).T + pose[4:]
    a = pa[valid == 1].astype(np.float64); b = pb[valid == 1].astype(np.float64)
    r = 0.6 * np.linalg.norm(np.cross(lp - a, lp - b), axis=1) / np.linalg.norm(a - b, axis=1)
    np.testing.assert_allclose(s[27], 0.5 * np.log1p(r * r).sum(), rtol=1e-10)
    np.testing.assert_allclose(s[21:27], _fd_gradient(fn, pose), rtol=2e-5, atol=1e-7)


# ---------------------------------------------------------------- §8 (f3): FormatConvert
def test_convert_livox_matches_formula(oracle):
    rng = np.random.default_rng(9)
    n = 5000
    a = np.zeros(n, oracle.LIVOX20)
    a["offset_time"] = np.sort(rng.integers(0, 99_999_000, n)).astype(np.uint32)
    a["x"], a["y"], a["z"] = rng.uniform(-50, 50, (3, n)).astype(np.float32)
    a["reflectivity"] = rng.integers(0, 256, n); a["line"] = rng.integers(0, 6, n); a["tag"] = rng.integers(0, 256, n)
    out = oracle.convert_livox(a)
    s = a["offset_time"].astype(np.float32) / np.float32(a["offset_time"][-1])        # fp32 division (:19)
    np.testing.assert_array_equal(out["intensity"], (a["line"].astype(np.float64) + s.astype(np.float64) * 0.1).astype(np.float32))
    np.testing.assert_array_equal(out["curvature"], (0.1 * a["reflectivity"].astype(np.float64)).astype(np.float32))
    np.testing.assert_array_equal(out["x"], a["x"]); assert (out["w"] == 1).all() and (out["nx"] == 0).all()
    # serialised (19-byte) wire layout gives the same cloud
    wire = np.ascontiguousarray(a.view(np.uint8).reshape(n, 20)[:, :19])
    out19 = oracle.convert_livox(wire.reshape(-1), stride=19)
    assert out19.tobytes() == out.tobytes()
    # the converted cloud is what the Horizon extractor expects: line = int(intensity), frac in [0, 0.1]
    assert ((out["intensity"] - np.floor(out["intensity"])) <= 0.1 + 1e-6).all()


def test_golden_backend_blocks_and_livox(oracle):
    g = np.load(os.path.join(GOLD, "backend_small.npz")); s2m = np.load(os.path.join(GOLD, "s2m_small.npz"))
    tree = oracle.KdTree(s2m["map"]); feats = s2m["feats"]
    sv, plane, score = oracle.correspond_surf_backend(tree, feats, g["pose_l"], 1.0, 0.06, 0.2, 0.6)
    _same(sv, g["surf_valid"]); _same(plane, g["surf_plane"]); _same(score, g["surf_score"])
    np.testing.assert_allclose(oracle.backend_surf_block(feats, sv, plane, score, g["pose_b"], g["q_lb"], g["t_lb"], 1.0), g["surf_block"], rtol=1e-13)
    ev, pa, pb = oracle.correspond_edge(tree, feats, g["pose_l"], 0)
    _same(ev, g["edge_valid"]); _same(pa, g["edge_pa"]); _same(pb, g["edge_pb"])
    np.testing.assert_allclose(oracle.backend_edge_block(feats, ev, pa, pb, 0.6, g["pose_b"], 1.0), g["edge_block"], rtol=1e-13)
    lv = np.load(os.path.join(GOLD, "livox_small.npz"))
    _same(oracle.convert_livox(lv["records"].view(oracle.LIVOX20).reshape(-1)).view(np.uint8), lv["cloud"])


def test_incremental_local_map_is_bit_exact(oracle, world_small):
    """Design check for SURVEY §8 (f2): a local map maintained INCREMENTALLY (append the newest frame's points to their
    voxels, drop the oldest frame's, re-sum only the voxels whose membership changed from the front) equals
    pcl::VoxelGrid of the concatenated <= 20 frames bit for bit, because (i) PCL's voxel of a point is floor(p/leaf)
    whatever the bounding box, (ii) its output order (ascending i + j*dx + k*dx*dy) is the lexicographic (k, j, i) order of
    those absolute coordinates, (iii) the centroid is a sequential fp32 sum in concatenation order, which an append extends."""
    rng = np.random.default_rng(4)
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    base = oracle.voxelgrid(surf, 0.4)
    leaf = np.float32(0.4); inv = np.float32(1.0) / leaf
    frames = []                       # (frame cloud) oldest first
    vox = {}                          # (kz, ky, kx) -> list of [frame_serial, running fp32 sums per field..., count]; kept as member lists
    fields = ["x", "y", "z", "nx", "ny", "nz", "intensity", "curvature"]

    def keys_of(cloud):
        k = np.floor(np.stack([cloud["x"], cloud["y"], cloud["z"]], 1) * inv).astype(np.int64)
        return [tuple(r[::-1]) for r in k]                     # (kz, ky, kx)

    members = {}                      # key -> list of (serial, point record), concatenation order
    serial = 0
    for step in range(26):
        f = base.copy()
        f["x"] += np.float32(0.11 * step) + rng.normal(0, 0.02, len(f)).astype(np.float32)
        f["y"] += np.float32(-0.03 * step)
        if len(frames) >= 20:                                   # FIFO eviction (LidarOdometry.cpp:290-299)
            old = frames.pop(0)
            for kk in set(keys_of(old[1])):
                members[kk] = [mm for mm in members[kk] if mm[0] != old[0]]
                if not members[kk]:
                    del members[kk]
        frames.append((serial, f))
        for kk, rec in zip(keys_of(f), f):
            members.setdefault(kk, []).append((serial, rec))
        serial += 1
        if step % 5 != 0 and step < 24:
            continue
        ref = oracle.voxelgrid(np.concatenate([c for _, c in frames]), float(leaf))
        order = sorted(members)
        assert len(order) == len(ref)
        got = np.zeros(len(order), oracle.PT48)
        for o, kk in enumerate(order):
            acc = {fl: np.float32(0) for fl in fields}
            for _, rec in members[kk]:
                for fl in fields:
                    acc[fl] = np.float32(acc[fl] + rec[fl])
            n = np.float32(len(members[kk]))
            for fl in ("x", "y", "z", "intensity", "curvature"):
                got[fl][o] = acc[fl] / n
            got["w"][o] = 1.0
            nx, ny, nz = acc["nx"], acc["ny"], acc["nz"]
            n2 = np.float32(np.float32(nx * nx + ny * ny) + nz * nz)
            if n2 > 0:
                nn = np.sqrt(n2)
                nx, ny, nz = nx / nn, ny / nn, nz / nn
            got["nx"][o], got["ny"][o], got["nz"][o] = nx, ny, nz
        for fl in ("x", "y", "z", "intensity", "curvature"):
            assert got[fl].tobytes() == ref[fl].tobytes(), (step, fl)
        np.testing.assert_allclose(np.stack([got["nx"], got["ny"], got["nz"]], 1), np.stack([ref["nx"], ref["ny"], ref["nz"]], 1), atol=2e-7)


def test_horizon_extractor_second_restatement(oracle, world_small):
    """An independent NumPy restatement of the binning + patch classifier (L/src/Preprocessing.cpp:238-383), written from the
    reference source and not from oracle_horizon.cpp, must select the same surf / edge points in the same order.  It starts
    from the oracle's de-skewed cloud (the slerp is covered elsewhere) and uses numpy's eigvalsh for the two PCA gates, so
    only a ratio within rounding of a threshold could differ (none does on these sweeps)."""
    from liliom_b200 import synth
    for seed in (1, 7):
        T = np.array(world_small["T"]); T[4] += 0.9 * seed
        pts, q = synth.make_horizon_sweep(T, seed=seed)
        surf_o, edge_o, cut_o = oracle.extract_horizon(pts, q, 0.2, 4.0)
        N_SCANS, H_SCANS = 6, 4000
        t_interval = 0.1 / (H_SCANS - 1)
        mat = np.zeros((N_SCANS, H_SCANS), oracle.PT48)                       # zero-initialised like PointXYZINormal mat[][] (+ curvature 0 = empty)
        for p in cut_o:                                                       # :242-268 (scan_id >= 0 always for the synthetic sweep)
            scan_id = int(p["intensity"])
            dep = np.float32(np.float32(p["x"] * p["x"] + p["y"] * p["y"]) + p["z"] * p["z"])       # float products, summed in float (:259)
            if dep > 40000.0 or dep < 4.0 or p["curvature"] < 0.05 or p["curvature"] > 25.45:
                continue
            col = int(np.round(float(np.float32(p["intensity"] - np.float32(scan_id))) / t_interval))   # float - int -> float, / double
            if col >= H_SCANS or col < 0:
                continue
            if mat[scan_id, col]["curvature"] != 0:
                continue
            mat[scan_id, col] = p
        depth = np.sqrt((mat["x"] * mat["x"] + mat["y"] * mat["y"] + mat["z"] * mat["z"]).astype(np.float32)).astype(np.float64)   # getDepth: float
        curv = mat["curvature"].copy()
        xyz = np.stack([mat["x"], mat["y"], mat["z"]], -1).astype(np.float64)
        surf_sel, edge_sel = [], []
        for i in range(5, H_SCANS - 12, 6):
            cells = [(k, i + j) for j in range(6) for k in range(N_SCANS) if curv[k, i + j] > 0]
            if len(cells) < 25:
                continue
            P = np.array([xyz[c] for c in cells]); ctr = P.mean(0)
            ev = np.linalg.eigvalsh((P - ctr).T @ (P - ctr))
            ids = []
            for k in range(N_SCANS):
                max_s, idx = 0.0, i
                for j in range(6):
                    if curv[k, i + j] <= 0:
                        continue
                    d = depth[k]
                    g1 = d[i + j - 4] + d[i + j - 3] + d[i + j - 2] + d[i + j - 1] - 8 * d[i + j] + d[i + j + 1] + d[i + j + 2] + d[i + j + 3] + d[i + j + 4]
                    g1 = g1 / (8 * d[i + j] + 1e-3)
                    if g1 > 0.06 and g1 > max_s:
                        max_s, idx = g1, i + j
                if max_s != 0:
                    ids.append((k, idx))
            if len(ids) > 3:
                E = np.array([xyz[c] for c in ids]); ce = E.mean(0)
                eve = np.linalg.eigvalsh((E - ce).T @ (E - ce))
                if eve[2] > 4.0 * eve[1]:
                    for c in ids:
                        if curv[c] <= 0 and mat[c]["intensity"] <= 0:
                            continue
                        edge_sel.append(c); curv[c] *= -1
            if ev[0] < 0.2 * ev[1]:
                for j in range(6):
                    for k in range(N_SCANS):
                        if curv[k, i + j] > 0:
                            surf_sel.append((k, i + j)); curv[k, i + j] *= -1
        assert len(surf_sel) == len(surf_o) and len(edge_sel) == len(edge_o), (len(surf_sel), len(surf_o), len(edge_sel), len(edge_o))
        for sel, out in ((surf_sel, surf_o), (edge_sel, edge_o)):
            got = np.array([[mat[c]["x"], mat[c]["y"], mat[c]["z"]] for c in sel], np.float32).reshape(-1, 3)
            ref = np.stack([out["x"], out["y"], out["z"]], 1)
            assert got.tobytes() == ref.tobytes()


def test_rot_labelling_second_restatement(oracle, world_small):
    """Independent NumPy restatement of the ROT curvature / per-segment sort / greedy labelling (R/src/Preprocessing.cpp:377-500),
    written from the reference source, on the oracle's ring-bucketed de-skewed cloud: curvature and labels bit-exact, the edge
    cloud (cornerPointsLessSharp) in the same order.  std::sort's tie order is defined as (curvature, index), as everywhere."""
    for ds_rate in (1, 4):
        rc, surf_o, edge_o, cut, lab_o, cur_o = oracle.extract_rot(world_small["hdl"], world_small["q_hdl"], (1, 0, 0, 0), 64, ds_rate)
        assert rc == 0
        n = len(cut)
        x, y, z = cut["x"], cut["y"], cut["z"]
        ring = cut["intensity"].astype(np.int32)
        N_SCANS = 64
        counts = np.bincount(ring, minlength=N_SCANS)
        ends = np.cumsum(counts); starts = ends - counts
        scanStart = starts + 5; scanEnd = ends - 6                                     # :378-382

        def stencil(a):
            i = np.arange(5, n - 5)
            s = a[i - 5] + a[i - 4]; s = s + a[i - 3]; s = s + a[i - 2]; s = s + a[i - 1]
            s = s - np.float32(10) * a[i]
            for k in (1, 2, 3, 4, 5):
                s = s + a[i + k]
            return s
        dx, dy, dz = stencil(x), stencil(y), stencil(z)
        curv = np.zeros(n, np.float32)
        curv[5:n - 5] = (dx * dx + dy * dy) + dz * dz                                  # :391
        picked = np.zeros(n + 8, np.int32); label = np.zeros(n, np.int32)
        r2 = (x * x + y * y) + z * z

        def gap2(a, b):
            ddx = x[a] - x[b]; ddy = y[a] - y[b]; ddz = z[a] - z[b]
            return np.float32(np.float32(ddx * ddx + ddy * ddy) + ddz * ddz)

        def suppress(ind):
            for l in range(1, 6):
                if gap2(ind + l, ind + l - 1) > 0.05:
                    break
                picked[ind + l] = 1
            for l in range(-1, -6, -1):
                if gap2(ind + l, ind + l + 1) > 0.05:
                    break
                picked[ind + l] = 1
        edge_order = []
        for i in range(N_SCANS):
            if scanEnd[i] - scanStart[i] < 6 or i % ds_rate != 0:
                continue
            for j in range(6):
                sp = scanStart[i] + (scanEnd[i] - scanStart[i]) * j // 6
                ep = scanStart[i] + (scanEnd[i] - scanStart[i]) * (j + 1) // 6 - 1
                seg = np.arange(sp, ep + 1)
                order = seg[np.lexsort((seg, curv[seg]))]
                big = 0
                for ind in order[::-1]:
                    if picked[ind] == 0 and curv[ind] > 2.0:
                        big += 1
                        if big <= 2:
                            label[ind] = 2
                        elif big <= 10:
                            label[ind] = 1
                        else:
                            break
                        edge_order.append(ind)
                        picked[ind] = 1
                        suppress(ind)
                small = 0
                for ind in order:
                    if r2[ind] < 0.25:
                        continue
                    if picked[ind] == 0 and curv[ind] < 0.1:
                        label[ind] = -1
                        small += 1
                        if small >= 4:
                            break
                        picked[ind] = 1
                        suppress(ind)
        assert curv.tobytes() == cur_o.tobytes()
        assert np.array_equal(label, lab_o), int((label != lab_o).sum())
        got = np.stack([x[edge_order], y[edge_order], z[edge_order]], 1)
        assert got.tobytes() == np.stack([edge_o["x"], edge_o["y"], edge_o["z"]], 1).tobytes()


def test_find_surf_corr_second_restatement_on_real_flann(oracle, world_small):
    """findCorrespondingSurfFeatures (L/src/LidarOdometry.cpp:352-413) restated a second time, from the reference source, on top
    of third-party code only: the 5-NN come from a real FLANN KDTreeSingleIndex (OpenCV's vendored FLANN, the class PCL wraps),
    the plane from numpy's least squares.  Accept flags must equal the oracle's, planes agree to fp32 rounding."""
    cv2 = pytest.importorskip("cv2")
    if not hasattr(cv2, "flann_Index"):
        pytest.skip("this OpenCV build has no flann module")
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    m = world_small["map"]
    pose = world_small["guess"]
    cnt, valid_o, plane_o, idx_o, pw_o = oracle.find_surf_corr(oracle.KdTree(m), ds, pose)
    # transformPoint (:221-244): Eigen q*p + t in double, stored as float
    P = np.stack([ds["x"], ds["y"], ds["z"]], 1).astype(np.float64)
    qv = pose[1:4]; uv = 2.0 * np.cross(qv, P)
    sel = (P + pose[0] * uv + np.cross(qv, uv) + pose[4:]).astype(np.float32)
    index = cv2.flann_Index(np.ascontiguousarray(m[:, :3]), dict(algorithm=4, leaf_max_size=15, reorder=True))
    nn, sqd = index.knnSearch(np.ascontiguousarray(sel), 5, params=dict(checks=-1, eps=0.0, sorted=True))
    valid = np.zeros(len(sel), np.uint8); plane = np.zeros((len(sel), 4), np.float32)
    for i in range(len(sel)):
        if not sqd[i, 4] < 1.0:                                                        # :365
            continue
        A = m[nn[i], :3].astype(np.float64)
        norm, *_ = np.linalg.lstsq(A, -np.ones(5), rcond=None)                         # :375
        nrm = np.linalg.norm(norm)
        if not nrm > 0:
            continue
        normInverse = 1.0 / nrm; norm = norm / nrm
        if (np.abs(A @ norm + normInverse) > 0.06).any():                              # :386-393
            continue
        s = sel[i]
        pd = np.float32(norm[0] * s[0] + norm[1] * s[1] + norm[2] * s[2] + normInverse)
        rng = np.sqrt(np.sqrt(np.float32(np.float32(s[0] * s[0] + s[1] * s[1]) + s[2] * s[2])))   # float overloads (SURVEY App. C.1)
        weight = np.float32(1 - 0.9 * abs(float(pd)) / float(rng))
        if weight > 0.4:
            valid[i] = 1
            plane[i] = [weight * norm[0], weight * norm[1], weight * norm[2], weight * normInverse]
    # identical decisions except where a gate sits within rounding of its threshold (different LS solver) or FLANN's tie order differs
    assert (valid != valid_o).sum() <= 2, int((valid != valid_o).sum())
    both = (valid == 1) & (valid_o == 1)
    assert both.sum() > 1000
    np.testing.assert_allclose(plane[both], plane_o[both], rtol=5e-6, atol=5e-7)


def test_backend_edge_corr_second_restatement_on_real_flann(oracle):
    """findCorrespondingCornerFeatures (L/src/BackendFusion.cpp:1531-1599; ROT variant adds the dist < 0.1 gate, R:1435-1443)
    restated from the reference source on real FLANN + numpy.linalg.eigh: same accept flags, same line end points to fp32."""
    cv2 = pytest.importorskip("cv2")
    if not hasattr(cv2, "flann_Index"):
        pytest.skip("this OpenCV build has no flann module")
    rng = np.random.default_rng(31)
    segs = []
    for px in range(-30, 31, 6):
        for py in (-8.0, 8.0):
            zz = np.arange(0.0, 6.0, 0.2)
            segs.append(np.stack([np.full_like(zz, px), np.full_like(zz, py), zz], 1))
        xx = np.arange(px, px + 6.0, 0.2)
        segs.append(np.stack([xx, np.full_like(xx, 10.0), np.full_like(xx, 3.0)], 1))
    m = np.concatenate(segs).astype(np.float32) + rng.normal(0, 0.01, (sum(len(s) for s in segs), 3)).astype(np.float32)
    m4 = np.ones((len(m), 4), np.float32); m4[:, :3] = m
    pose = np.array([1.0, 0, 0, 0, 0.0, 0.0, 0.0])
    feats = np.ones((1200, 4), np.float32)
    feats[:, :3] = m[rng.integers(0, len(m), 1200)] + rng.normal(0, 0.08, (1200, 3)).astype(np.float32)
    tree = oracle.KdTree(m4)
    index = cv2.flann_Index(np.ascontiguousarray(m), dict(algorithm=4, leaf_max_size=15, reorder=True))
    nn, sqd = index.knnSearch(np.ascontiguousarray(feats[:, :3]), 5, params=dict(checks=-1, eps=0.0, sorted=True))
    for variant in (0, 1):
        v_o, pa_o, pb_o = oracle.correspond_edge(tree, feats, pose, variant)
        v = np.zeros(len(feats), np.uint8); pa = np.zeros((len(feats), 3), np.float32); pb = np.zeros((len(feats), 3), np.float32)
        for i in range(len(feats)):
            if not sqd[i, 4] < 1.0:
                continue
            P = m[nn[i]].astype(np.float64)
            c = P.sum(0) / 5.0
            w, vec = np.linalg.eigh((P - c).T @ (P - c))
            if not w[2] > 3 * w[1]:
                continue
            u = vec[:, 2]
            A, B = c + 0.1 * u, c - 0.1 * u
            if variant == 1:
                lp = feats[i, :3].astype(np.float64)
                if not np.linalg.norm(np.cross(lp - A, lp - B)) / np.linalg.norm(A - B) < 0.1:
                    continue
            v[i] = 1; pa[i] = A; pb[i] = B
        assert (v != v_o).sum() <= 2 and v.sum() > 300
        both = (v == 1) & (v_o == 1)
        # the eigenvector's sign is arbitrary: the end points may be swapped
        same = np.abs(pa[both] - pa_o[both]).max(1) < 1e-5
        swapped = np.abs(pa[both] - pb_o[both]).max(1) < 1e-5
        assert (same | swapped).all()


def test_voxelgrid_adversarial_inputs_match_numpy(oracle):
    """pcl::VoxelGrid restatement on inputs the sweeps never produce: negative coordinates, points exactly on voxel faces,
    duplicates, non-finite points (dropped from the box and from the output), a single point, both strides."""
    rng = np.random.default_rng(8)
    for dt, leaf in ((oracle.PT48, 0.4), (oracle.PT32, 0.6), (oracle.PT48, 0.25)):
        n = 3000
        c = np.zeros(n, dt)
        xyz = rng.uniform(-7, 7, (n, 3)).astype(np.float32)
        xyz[:300] = np.round(xyz[:300] / np.float32(leaf)) * np.float32(leaf)        # exactly on voxel faces
        xyz[300:400] = xyz[:100]                                                     # duplicates
        c["x"], c["y"], c["z"] = xyz.T
        c["intensity"] = rng.uniform(0, 50, n).astype(np.float32)
        if dt is oracle.PT48:
            c["curvature"] = rng.uniform(0, 25, n).astype(np.float32)
        bad = rng.choice(n, 40, replace=False)
        c["x"][bad[:15]] = np.nan; c["y"][bad[15:30]] = np.inf; c["z"][bad[30:]] = -np.inf
        got = oracle.voxelgrid(c, leaf)
        ok = np.isfinite(c["x"]) & np.isfinite(c["y"]) & np.isfinite(c["z"])
        f = c[ok]
        inv = np.float32(1.0) / np.float32(leaf)
        ijk = np.floor(np.stack([f["x"], f["y"], f["z"]], 1) * inv).astype(np.int64)
        mn = ijk.min(0); div = ijk.max(0) - mn + 1
        idx = (ijk[:, 0] - mn[0]) + (ijk[:, 1] - mn[1]) * div[0] + (ijk[:, 2] - mn[2]) * div[0] * div[1]
        uniq, inv_idx, counts = np.unique(idx, return_inverse=True, return_counts=True)
        assert len(got) == len(uniq)
        for fld in ("x", "y", "z", "intensity"):
            acc = np.zeros(len(uniq), np.float32)
            np.add.at(acc, inv_idx, f[fld])
            np.testing.assert_array_equal(got[fld], acc / counts.astype(np.float32))
    one = np.zeros(1, oracle.PT48); one["x"] = 1.5; one["curvature"] = 3
    assert len(oracle.voxelgrid(one, 0.4)) == 1 and len(oracle.voxelgrid(one[:0], 0.4)) == 0


def test_horizon_deskew_second_restatement(oracle, world_small):
    """undistortion (L/src/Preprocessing.cpp:104-127) restated in NumPy from the reference source: slerp(Identity -> q_iMU) by the
    fractional part of `intensity` over 0.1 s, Eigen's un-normalised q * v.  The oracle's cutted cloud must agree to fp32 rounding
    (numpy's acos / sin are not glibc's bit for bit, so this is a 1-ulp-of-fp32 check, not a bit-exact one)."""
    pts, q = world_small["hz"], np.asarray(world_small["q_hz"], np.float64)
    _, _, cut = oracle.extract_horizon(pts, q)
    assert len(cut) == len(pts)                                   # no NaN / closer-than-0.1 m points in the synthetic sweep
    inten = pts["intensity"].astype(np.float64)
    ratio = np.minimum((inten - np.floor(inten)) / 0.1, 1.0)       # float intensity - int line, in double (:106-112)
    d = q[0]                                                       # Identity . q_iMU
    absd = abs(d)
    if absd >= 1.0 - np.finfo(np.float64).eps:
        s0, s1 = 1.0 - ratio, ratio
    else:
        th = np.arccos(absd); sth = np.sin(th)
        s0 = np.sin((1.0 - ratio) * th) / sth; s1 = np.sin(ratio * th) / sth
    if d < 0:
        s1 = -s1
    qs = np.stack([s0 + s1 * q[0], s1 * q[1], s1 * q[2], s1 * q[3]], 1)             # s0 * Identity + s1 * q_iMU, not re-normalised
    P = np.stack([pts["x"], pts["y"], pts["z"]], 1).astype(np.float64)
    uv = 2.0 * np.cross(qs[:, 1:], P)
    out = (P + qs[:, :1] * uv + np.cross(qs[:, 1:], uv)).astype(np.float32)
    ref = np.stack([cut["x"], cut["y"], cut["z"]], 1)
    assert np.abs(out.view(np.int32) - ref.view(np.int32)).max() <= 1              # within one fp32 ulp
    assert np.array_equal(cut["intensity"], pts["intensity"]) and np.array_equal(cut["curvature"], pts["curvature"])


def test_rot_ring_and_time_assignment_on_glibc(oracle, world_small):
    """R/src/Preprocessing.cpp:280-372 restated from the reference source with the float overloads resolved to glibc's own atanf /
    atan2f through ctypes (what `using namespace std` makes the reference call, tests/rot_restate.py): ring id, the halfPassed azimuth unwrapping and
    intensity = ring + 0.1 * relTime, bucketed by ring in input order, must equal the oracle's laserCloud bit for bit."""
    import rot_restate
    pts = world_small["hdl"]
    rc, _, _, cut, _, _ = oracle.extract_rot(pts, world_small["q_hdl"], (1, 0, 0, 0), 64, 1)
    got = rot_restate.assign(pts, 64)["intensity"]
    assert len(got) == len(cut)
    assert got.tobytes() == cut["intensity"].tobytes()


def test_pose_glue_second_restatement(oracle):
    """poseInitialization / computeRelative / transformCloud (L/src/LidarOdometry.cpp:415-480, 246-278) against plain NumPy
    quaternion algebra written from the reference source (Hamilton product, Eigen's q*v, inverse = conjugate / squared norm)."""
    import ctypes as C
    rng = np.random.default_rng(12)

    def qmul(a, b):
        return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                         a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3], a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]])

    def qrot(q, v):
        uv = 2.0 * np.cross(q[1:], v)
        return v + q[0] * uv + np.cross(q[1:], uv)
    L = oracle.lib()
    for _ in range(50):
        a = rng.normal(size=7); a[:4] /= np.linalg.norm(a[:4]) * rng.uniform(0.999, 1.001)     # almost-unit, as accumulated in the node
        r = rng.normal(size=7); r[:4] /= np.linalg.norm(r[:4])
        out = np.zeros(7)
        L.orc_pose_compose(oracle._d(a), oracle._d(r), oracle._d(out))                          # t0 = q0*dt + t0 ; q0 = q0*dq
        np.testing.assert_allclose(out[:4], qmul(a[:4], r[:4]), rtol=0, atol=1e-15)
        np.testing.assert_allclose(out[4:], qrot(a[:4], r[4:]) + a[4:], rtol=0, atol=1e-14)
        rel = np.zeros(7)
        L.orc_pose_relative(oracle._d(a), oracle._d(out), oracle._d(rel))                       # q1^-1 * q2 ; q1^-1 * (t2 - t1)
        qi = np.array([a[0], -a[1], -a[2], -a[3]]) / np.dot(a[:4], a[:4])
        np.testing.assert_allclose(rel[:4], qmul(qi, out[:4]), rtol=0, atol=1e-14)
        np.testing.assert_allclose(rel[4:], qrot(qi, out[4:] - a[4:]), rtol=0, atol=1e-13)
    # transformCloud: xyz rotated + translated (double, stored float), normals rotated only (48-byte layout)
    c = np.zeros(200, oracle.PT48)
    c["x"], c["y"], c["z"] = rng.uniform(-30, 30, (3, 200)).astype(np.float32)
    nrm = rng.normal(size=(200, 3)); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    c["nx"], c["ny"], c["nz"] = nrm.T.astype(np.float32)
    c["intensity"] = 3.5; c["curvature"] = 1.25
    pose = rng.normal(size=7); pose[:4] /= np.linalg.norm(pose[:4])
    t = oracle.transform_cloud(c, pose)
    P = np.stack([c["x"], c["y"], c["z"]], 1).astype(np.float64)
    N = np.stack([c["nx"], c["ny"], c["nz"]], 1).astype(np.float64)
    ref_p = np.array([qrot(pose[:4], p) + pose[4:] for p in P]).astype(np.float32)
    ref_n = np.array([qrot(pose[:4], v) for v in N]).astype(np.float32)
    assert np.abs(np.stack([t["x"], t["y"], t["z"]], 1).view(np.int32) - ref_p.view(np.int32)).max() <= 1
    np.testing.assert_allclose(np.stack([t["nx"], t["ny"], t["nz"]], 1), ref_n, atol=1e-6)
    assert (t["intensity"] == 3.5).all() and (t["curvature"] == 1.25).all()


def test_undistortion_matches_numpy_restatement(oracle):
    """LidarOdometry::undistortion (L/src/LidarOdometry.cpp:178-199) restated in NumPy from the reference source: ratio =
    min(frac(intensity)/0.1, 1); p' = slerp(I, quat; ratio) * p + ratio * trans.  With quat = identity (the only way the
    reference calls it, :626) the oracle must agree bit for bit; with a general quaternion to one fp32 ulp (acos/sin)."""
    rng = np.random.default_rng(12)
    pts = np.zeros(4000, oracle.PT48)
    pts["x"] = rng.uniform(-50, 50, 4000).astype(np.float32); pts["y"] = rng.uniform(-50, 50, 4000).astype(np.float32)
    pts["z"] = rng.uniform(-3, 8, 4000).astype(np.float32)
    pts["intensity"] = (rng.integers(0, 6, 4000) + rng.uniform(0, 0.13, 4000)).astype(np.float32)    # some ratios above 1: clamped
    pts["curvature"] = rng.uniform(0, 1, 4000).astype(np.float32); pts["nx"] = 1.0
    trans = np.array([0.31, -0.07, 0.02])
    line = pts["intensity"].astype(np.int32)
    ratio = np.minimum((pts["intensity"] - line.astype(np.float32)).astype(np.float64) / 0.1, 1.0)
    got = oracle.undistort(pts, trans)
    for k, f in enumerate(("x", "y", "z")):
        want = (pts[f].astype(np.float64) + ratio * trans[k]).astype(np.float32)
        assert np.array_equal(got[f].view(np.uint32), want.view(np.uint32)), f
    for f in ("intensity", "curvature", "nx", "w"):
        assert np.array_equal(got[f], pts[f])
    # general quaternion: Rodrigues with angle ratio*theta about the quaternion's axis
    half = 0.04
    axis = np.array([0.2, -0.5, 0.84]); axis /= np.linalg.norm(axis)
    quat = np.concatenate([[np.cos(half)], np.sin(half) * axis])
    got = oracle.undistort(pts, trans, quat)
    ang = 2 * half * ratio
    p = np.stack([pts["x"], pts["y"], pts["z"]], 1).astype(np.float64)
    rp = (p * np.cos(ang)[:, None] + np.cross(axis, p) * np.sin(ang)[:, None] + axis * (p @ axis)[:, None] * (1 - np.cos(ang))[:, None])
    want = rp + ratio[:, None] * trans
    for k, f in enumerate(("x", "y", "z")):
        np.testing.assert_allclose(got[f], want[:, k].astype(np.float32), rtol=3e-7, atol=2e-6)
    # 32-byte points carry the time in float #4
    p32 = np.zeros(100, oracle.PT32); p32["x"] = 1.0; p32["intensity"] = 3.05
    g32 = oracle.undistort(p32, trans)
    assert np.array_equal(g32["x"], (1.0 + np.float64(np.float32(3.05) - np.float32(3.0)) / 0.1 * trans[0]).astype(np.float32) * np.ones(100, np.float32))
