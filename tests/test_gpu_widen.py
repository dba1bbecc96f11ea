"""GPU parity for the SURVEY.md §8 (f) rows: (f1) backend LiDAR factor blocks, (f3) Livox CustomMsg ingest.
Same bar as tests/test_gpu_parity.py: the CUDA path through the C ABI against the CPU oracle on identical inputs."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _f4(cloud):
    out = np.ones((len(cloud), 4), np.float32)
    out[:, 0] = cloud["x"]; out[:, 1] = cloud["y"]; out[:, 2] = cloud["z"]
    return out


def _livox_sweep(world_small, L):
    """The synthetic Horizon sweep re-encoded as the livox CustomPoint records FormatConvert receives."""
    pts = world_small["hz"]
    n = len(pts)
    a = np.zeros(n, L.LIVOX20)
    line = np.floor(pts["intensity"]).astype(np.int64)
    frac = (pts["intensity"].astype(np.float64) - line) / 0.1
    a["offset_time"] = np.clip(np.round(frac * 99_000_000.0), 0, 99_000_000).astype(np.uint32)
    a["offset_time"][-1] = 99_000_000                                   # points.back() defines time_end
    a["x"], a["y"], a["z"] = pts["x"], pts["y"], pts["z"]
    a["reflectivity"] = np.clip(np.round(pts["curvature"].astype(np.float64) * 10.0), 0, 255).astype(np.uint8)
    a["line"] = line.astype(np.uint8)
    a["tag"] = 0x10
    return a


# ---------------------------------------------------------------- (f3) FormatConvert on the device
@pytest.mark.parametrize("stride", [20, 19])
def test_convert_livox_bit_exact(ctx48, oracle, world_small, stride):
    import liliom_b200 as L
    a = _livox_sweep(world_small, L)
    raw = a if stride == 20 else np.ascontiguousarray(a.view(np.uint8).reshape(len(a), 20)[:, :19]).reshape(-1)
    ref = oracle.convert_livox(raw, stride=stride if stride == 19 else None)
    got = ctx48.convert_livox(raw, stride=stride if stride == 19 else None)
    assert got.tobytes() == ref.tobytes()
    assert len(ctx48.convert_livox(a[:0])) == 0


def test_extract_horizon_from_livox_records(ctx48, oracle, world_small):
    import liliom_b200 as L
    a = _livox_sweep(world_small, L)
    cloud = oracle.convert_livox(a)
    surf_o, edge_o, cut_o = oracle.extract_horizon(cloud, world_small["q_hz"])
    surf, edge, cut = ctx48.extract_horizon_livox(a, world_small["q_hz"])
    assert len(surf_o) > 3000
    for got, ref in ((surf, surf_o), (edge, edge_o), (cut, cut_o)):
        assert len(got) == len(ref) and got.tobytes() == ref.tobytes()
    # resident flow: convert -> extract_resident gives the same counts
    n = ctx48.convert_livox(a, download=False)
    ctx48.extract_resident(world_small["q_hz"])          # counts stay on the device in the resident pipeline
    assert n == len(a)
    pose, st, ds = ctx48.odometry_resident(world_small["guess"], 0, want_ds=True, cap=len(a))     # surf count is device-side there
    assert len(ds) == len(oracle.voxelgrid(surf_o, 0.4))


# ---------------------------------------------------------------- (f1) backend LiDAR factor blocks
def test_backend_surf_block_matches_oracle(oracle, world_small):
    import liliom_b200 as L
    surf_o, edge_o, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf_o, 0.4)
    tree = oracle.KdTree(world_small["map"])
    pose_l = world_small["guess"]
    q_lb = np.array([0.9990482, 0.0, 0.0436194, 0.0]); t_lb = np.array([0.05, -0.02, 0.10])
    c = L.Context(variant=0)
    c.map_set_points(world_small["map"])
    v_o, pl_o, sc_o = oracle.correspond_surf_backend(tree, ds, pose_l, 1.0, 0.06, 0.2, 0.6)
    v, pl, sc = c.correspond_surf(ds, pose_l, 1.0, 0.06, 0.2, 0.6)
    assert np.array_equal(v, v_o) and v.sum() > 200
    assert pl.tobytes() == pl_o.tobytes() and sc.tobytes() == sc_o.tobytes()
    for k, pose_b in enumerate((pose_l, world_small["T"])):           # the block may be evaluated at any pose (LM iterations)
        ref = oracle.backend_surf_block(ds, v, pl, sc, pose_b, q_lb, t_lb, 1.0)
        got = c.backend_surf_block(pose_b, q_lb, t_lb, 1.0)
        assert got[28] == ref[28] == v.sum()
        np.testing.assert_allclose(got, ref, rtol=1e-9, atol=1e-9 * np.abs(ref[:21]).max())
    # the wrong kind resident -> argument error, not garbage
    with pytest.raises(L.LiliomError):
        c.backend_edge_block(pose_l, 0.6)
    c.close()


def test_backend_edge_block_matches_oracle(oracle, world_small):
    import liliom_b200 as L
    rng = np.random.default_rng(21)
    # an edge local map: points along vertical poles and horizontal rails (line-like 5-NN sets), 0.2 m spacing + noise
    poles = []
    for px in range(-30, 31, 6):
        for py in (-8.0, 8.0):
            z = np.arange(0.0, 6.0, 0.2)
            poles.append(np.stack([np.full_like(z, px), np.full_like(z, py), z], 1))
        x = np.arange(px, px + 6.0, 0.2)
        poles.append(np.stack([x, np.full_like(x, 10.0), np.full_like(x, 3.0)], 1))
    m = np.concatenate(poles).astype(np.float32)
    m += rng.normal(0, 0.01, m.shape).astype(np.float32)
    m4 = np.ones((len(m), 4), np.float32); m4[:, :3] = m
    pose = np.array([0.9990482, 0.0, 0.0, 0.0436194, 0.4, -0.3, 0.1])
    pose[:4] /= np.linalg.norm(pose[:4])      # unit like every pose Ceres' QuaternionParameterization produces (the closed-form row assumes it)
    # features: map points pulled into the body frame with noise
    sel = m[rng.integers(0, len(m), 1500)].astype(np.float64) + rng.normal(0, 0.08, (1500, 3))
    qw, qx, qy, qz = pose[:4]
    R = np.array([[1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qw * qz), 2 * (qx * qz + qw * qy)],
                  [2 * (qx * qy + qw * qz), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qw * qx)],
                  [2 * (qx * qz - qw * qy), 2 * (qy * qz + qw * qx), 1 - 2 * (qx * qx + qy * qy)]])
    feats = np.ones((1500, 4), np.float32); feats[:, :3] = (sel - pose[4:]) @ R
    tree = oracle.KdTree(m4)
    c = L.Context(variant=0)
    c.map_set_points(m4)
    for variant in (0, 1):
        v_o, pa_o, pb_o = oracle.correspond_edge(tree, feats, pose, variant)
        v, pa, pb = c.correspond_edge(feats, pose, variant)
        assert np.array_equal(v, v_o) and v.sum() > 300
        assert pa.tobytes() == pa_o.tobytes() and pb.tobytes() == pb_o.tobytes()
        pose_b = pose.copy(); pose_b[4:] += (0.02, -0.01, 0.03)
        ref = oracle.backend_edge_block(feats, v, pa, pb, 0.6, pose_b, 1.0)
        got = c.backend_edge_block(pose_b, 0.6, 1.0)
        assert got[28] == ref[28] == v.sum()
        np.testing.assert_allclose(got, ref, rtol=1e-8, atol=1e-9 * np.abs(ref[:21]).max())
    # empty feature set: zero block
    c.correspond_edge(feats[:0], pose, 0)
    assert not c.backend_edge_block(pose, 0.6).any()
    c.close()


def test_widen_rows_against_golden_fixtures(oracle):
    """(f1)/(f3) through the C ABI against the committed fixtures (tests/golden, generator tests/make_golden_widen.py)."""
    import os
    import liliom_b200 as L
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    g = np.load(os.path.join(gold, "backend_small.npz")); s2m = np.load(os.path.join(gold, "s2m_small.npz"))
    c = L.Context(variant=0)
    c.map_set_points(s2m["map"])
    feats = s2m["feats"]
    # The fixture was made by the oracle, and backend_corr.cu is compiled without contraction: the same flags and plane bits.
    v, pl, sc = c.correspond_surf(feats, g["pose_l"], 1.0, 0.06, 0.2, 0.6)
    assert np.array_equal(v, g["surf_valid"])
    assert pl.tobytes() == np.ascontiguousarray(g["surf_plane"], np.float32).tobytes()
    got = c.backend_surf_block(g["pose_b"], g["q_lb"], g["t_lb"], 1.0)
    want = g["surf_block"]
    np.testing.assert_allclose(got[:28], want[:28], rtol=2e-4, atol=2e-4 * np.abs(want[:21]).max())
    assert got[28] == want[28]
    ve, pa, pb = c.correspond_edge(feats, g["pose_l"], 0)
    assert np.array_equal(ve, g["edge_valid"])
    got = c.backend_edge_block(g["pose_b"], 0.6, 1.0)
    want = g["edge_block"]
    np.testing.assert_allclose(got[:28], want[:28], rtol=2e-4, atol=2e-4 * np.abs(want[:21]).max())
    assert got[28] == want[28]
    lv = np.load(os.path.join(gold, "livox_small.npz"))
    cloud = c.convert_livox(lv["records"].view(L.LIVOX20).reshape(-1))
    assert cloud.view(np.uint8).tobytes() == lv["cloud"].tobytes()
    c.close()


def test_undistortion_on_device(oracle, world_small):
    """(f3) LidarOdometry::undistortion (L/src/LidarOdometry.cpp:178-199) through the C ABI: bit-exact with quat = identity
    (how publishCloudLast calls it, :624-632), within one fp32 ulp for a general quaternion (fp64 acos/sin)."""
    import liliom_b200 as L
    surf, edge, cut = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    trans = np.array([0.27, -0.04, 0.015])
    c = L.Context(variant=0)
    for cloud in (cut, surf, edge, cut[:0]):
        got, want = c.undistort(cloud, trans), oracle.undistort(cloud, trans)
        assert got.view(np.uint8).tobytes() == want.view(np.uint8).tobytes()
    quat = np.array([0.9992, 0.01, -0.03, 0.02])
    got, want = c.undistort(cut, trans, quat), oracle.undistort(cut, trans, quat)
    for f in ("x", "y", "z"):
        np.testing.assert_allclose(got[f], want[f], rtol=2.5e-7, atol=1e-6)
    for f in ("intensity", "curvature", "nx", "ny", "nz"):
        assert np.array_equal(got[f].view(np.uint32), want[f].view(np.uint32))
    c.close()
    c32 = L.Context(variant=1)
    hdl = world_small["hdl"][:20000].copy()
    hdl["intensity"] = (np.arange(20000) % 64 + (np.arange(20000) % 97) / 970.0).astype(np.float32)
    assert c32.undistort(hdl, trans).view(np.uint8).tobytes() == oracle.undistort(hdl, trans).view(np.uint8).tobytes()
    c32.close()


def _icp_numpy(oracle, src, tgt, max_corr=30.0, max_iter=100, trans_eps=1e-6, fit_eps=1e-6):
    """PCL's IterativeClosestPoint loop restated on third-party numerics (from-knowledge, like icp.cu's header): exact NN from the
    oracle's kd-tree, Umeyama (no scale) with numpy's SVD, DefaultConvergenceCriteria."""
    tree = oracle.KdTree(tgt)
    F = np.eye(4)
    prev = np.finfo(np.float64).max
    it, conv = 0, False
    s3 = src[:, :3].astype(np.float64)
    while True:
        p = s3 @ F[:3, :3].T + F[:3, 3]
        q4 = np.ones((len(p), 4), np.float32); q4[:, :3] = p.astype(np.float32)
        idx, sqd = tree.knn5(q4)
        keep = sqd[:, 0] <= np.float32(max_corr * max_corr)
        if keep.sum() < 3:
            break
        P, Q = p[keep], tgt[idx[keep, 0], :3].astype(np.float64)
        mp, mq = P.mean(0), Q.mean(0)
        S = (Q - mq).T @ (P - mp) / len(P)
        U, D, Vt = np.linalg.svd(S)
        sg = np.ones(3)
        if np.linalg.det(U) * np.linalg.det(Vt) < 0:
            sg[2] = -1
        R = U @ np.diag(sg) @ Vt
        t = mq - R @ mp
        Ti = np.eye(4); Ti[:3, :3] = R; Ti[:3, 3] = t
        F = Ti @ F
        it += 1
        mse = float(sqd[keep, 0].astype(np.float64).mean())
        if it >= max_iter:
            conv = True; break
        if 0.5 * (np.trace(R) - 1.0) >= 1.0 - trans_eps and float(t @ t) <= trans_eps:
            conv = True; break
        if abs(mse - prev) / prev < fit_eps or abs(mse - prev) < 1e-12:
            conv = True; break
        prev = mse
    p = s3 @ F[:3, :3].T + F[:3, 3]
    q4 = np.ones((len(p), 4), np.float32); q4[:, :3] = p.astype(np.float32)
    _, sqd = tree.knn5(q4)
    return F, float(sqd[:, 0].astype(np.float64).mean()), conv, it


def test_loop_closure_icp(oracle, world_small):
    """(f4) liliom_icp_align with the reference's settings (L/src/BackendFusion.cpp:2566-2570) recovers a known loop-closure offset
    and follows the NumPy/kd-tree restatement of PCL's loop: same iteration count (+-1: a criterion sitting on its threshold),
    transform within 1e-6, same verdict; a source with nothing within reach does not converge."""
    import liliom_b200 as L
    rng = np.random.default_rng(4)
    m = world_small["map"]
    near = m[(np.abs(m[:, 0]) < 45) & (np.abs(m[:, 1]) < 45)]
    tgt = near[rng.permutation(len(near))[:30000]].copy()
    # source: a sub-sampled, noisy copy of part of the target seen from a frame that is off by 2.5 deg / (0.6, -0.4, 0.1) m
    ang = np.deg2rad(2.5)
    Rz = np.array([[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1.0]])
    t_true = np.array([0.6, -0.4, 0.1])
    pick = near[rng.permutation(len(near))[:12000]]
    src = np.ones((len(pick), 4), np.float32)
    src[:, :3] = ((pick[:, :3].astype(np.float64) - t_true) @ Rz + rng.normal(0, 0.01, (len(pick), 3))).astype(np.float32)   # R^T (q - t)
    c = L.Context(variant=0)
    T, fit, conv, it = c.icp_align(src, tgt)
    T_o, fit_o, conv_o, it_o = _icp_numpy(oracle, src, tgt)
    assert conv and conv_o and abs(it - it_o) <= 1 and 3 <= it < 100, (it, it_o)
    np.testing.assert_allclose(T, T_o, rtol=0, atol=2e-6 if it == it_o else 2e-4)
    assert abs(fit - fit_o) < 1e-6 * max(1.0, fit_o)
    # ... and it is the right answer: target <- source = (Rz, t_true) up to the noise and the sampling
    assert np.abs(T[:3, :3] - Rz).max() < 5e-3 and np.abs(T[:3, 3] - t_true).max() < 0.05 and fit < 0.3
    # 32-byte clouds go through the same call
    s32 = np.zeros(len(src), L.PT32); s32["x"], s32["y"], s32["z"] = src[:, 0], src[:, 1], src[:, 2]
    t32 = np.zeros(len(tgt), L.PT32); t32["x"], t32["y"], t32["z"] = tgt[:, 0], tgt[:, 1], tgt[:, 2]
    c32 = L.Context(variant=1)
    T2, fit2, conv2, it2 = c32.icp_align(s32, t32)
    assert it2 == it and np.array_equal(T2, T) and fit2 == fit
    c32.close()
    # nothing within the correspondence distance: "not enough correspondences" -> not converged, identity
    far = src.copy(); far[:, 0] += 500.0
    T3, fit3, conv3, it3 = c.icp_align(far, tgt, max_corr_dist=5.0)
    assert not conv3 and it3 == 0 and np.array_equal(T3, np.eye(4))
    c.close()
