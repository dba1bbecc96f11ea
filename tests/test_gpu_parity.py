"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle on identical inputs.
Bit-exact for index / label / fp32-cloud outputs, tolerance for fp64 reductions and poses
(BASELINE.json: pose within 1e-4 m / 1e-4 rad at equal iteration count)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _fields_equal(a, b, fields):
    assert len(a) == len(b), (len(a), len(b))
    for f in fields:
        fa, fb = a[f].view(np.uint32), b[f].view(np.uint32)
        bad = np.nonzero(fa != fb)[0]
        assert len(bad) == 0, f"field {f}: {len(bad)} of {len(a)} differ, first at {bad[:5]}: {a[f][bad[:5]]} vs {b[f][bad[:5]]}"


def _rot_angle(qa, qb):
    qa = np.asarray(qa) / np.linalg.norm(qa); qb = np.asarray(qb) / np.linalg.norm(qb)
    return 2.0 * np.arccos(min(1.0, abs(float(np.dot(qa, qb)))))


def _pose_close(a, b, tol_t=1e-4, tol_r=1e-4):
    assert np.linalg.norm(np.asarray(a)[4:] - np.asarray(b)[4:]) < tol_t, (a, b)
    assert _rot_angle(a[:4], b[:4]) < tol_r, (a, b)


# ---------------------------------------------------------------- VoxelGrid
@pytest.mark.parametrize("leaf", [0.4, 0.6])
def test_voxelgrid_pt48_bit_exact(ctx48, oracle, world_small, leaf):
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    want = oracle.voxelgrid(surf, leaf)
    got = ctx48.voxelgrid(surf, leaf)
    _fields_equal(got, want, ["x", "y", "z", "nx", "ny", "nz", "intensity", "curvature"])


def test_voxelgrid_pt32_bit_exact(ctx32, oracle, world_small):
    pts = world_small["hdl"][:40000]
    want = oracle.voxelgrid(pts, 0.6)
    got = ctx32.voxelgrid(pts, 0.6)
    _fields_equal(got, want, ["x", "y", "z", "intensity"])


def test_voxelgrid_edge_cases(ctx48, oracle):
    import liliom_b200 as L
    assert len(ctx48.voxelgrid(np.zeros(0, L.PT48), 0.4)) == 0
    one = np.zeros(1, L.PT48); one["x"] = 1.5; one["nx"] = 2.0; one["intensity"] = 3.0
    _fields_equal(ctx48.voxelgrid(one, 0.4), oracle.voxelgrid(one, 0.4), ["x", "y", "z", "nx", "intensity"])
    # overflow of the int32 voxel index: PCL returns the input unchanged
    far = np.zeros(3, L.PT48); far["x"] = [0.0, 1e6, -1e6]; far["y"] = [0, 1e6, 5]; far["z"] = [0, 3e5, 9]
    got, want = ctx48.voxelgrid(far, 0.01), oracle.voxelgrid(far, 0.01)
    assert len(want) == 3
    _fields_equal(got, want, ["x", "y", "z"])
    # non-finite points are dropped
    nf = np.zeros(4, L.PT48); nf["x"] = [0.1, np.nan, 0.2, np.inf]
    _fields_equal(ctx48.voxelgrid(nf, 0.4), oracle.voxelgrid(nf, 0.4), ["x", "y", "z"])


# ---------------------------------------------------------------- scan-to-map
@pytest.fixture(scope="module")
def s2m_case(ctx48, oracle, world_small):
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    tree = oracle.KdTree(world_small["map"])
    ctx48.map_set_points(world_small["map"])
    return dict(surf=surf, ds=ds, tree=tree)


def test_map_download_roundtrip(ctx48, world_small, s2m_case):
    got = ctx48.map_download()
    assert got.shape == world_small["map"].shape
    assert np.array_equal(got[:, :3].view(np.uint32), world_small["map"][:, :3].view(np.uint32))


@pytest.mark.parametrize("which", ["ds", "surf"])
def test_knn_and_correspondences_exact(ctx48, oracle, world_small, s2m_case, which):
    feats = s2m_case[which]
    pose = world_small["guess"]
    cnt, valid_o, plane_o, idx_o, pw_o = oracle.find_surf_corr(s2m_case["tree"], feats, pose)
    valid, plane, idx, sqd, s29 = ctx48.find_surf_corr(feats, pose)
    # (a) 5-NN index sets: exact wherever the oracle's 5th neighbour is inside the 1 m ball
    _, sqd_o = s2m_case["tree"].knn5(pw_o)
    inside = sqd_o[:, 4] < 1.0
    assert inside.sum() > 0.5 * len(feats)
    assert np.array_equal(idx[inside], idx_o[inside])
    assert np.array_equal(sqd[inside].view(np.uint32), sqd_o[inside].view(np.uint32))
    # (b) accept/reject decisions and weighted planes
    assert np.array_equal(valid, valid_o)
    assert int(valid.sum()) == cnt and cnt > 100
    np.testing.assert_allclose(plane, plane_o, rtol=2e-6, atol=1e-7)
    # (c) the 27 normal-equation scalars + cost + count (fp64 reduction order differs)
    want = oracle.normal_equations(feats, valid_o, plane_o, pose)
    np.testing.assert_allclose(s29, want, rtol=1e-9, atol=1e-9)


def test_scan_to_map_gn_pose(ctx48, oracle, world_small, s2m_case):
    rc, pose_o, st_o = oracle.scan_to_map_gn(s2m_case["tree"], s2m_case["ds"], world_small["guess"], 10)
    pose, st = ctx48.scan_to_map(s2m_case["ds"], world_small["guess"], 10, mode=1)
    assert rc == 0
    for a, b in zip(st, st_o):
        assert abs(a.n_corr - b.n_corr) <= 2
        _pose_close(np.array(a.pose7), np.array(b.pose7))
    np.testing.assert_allclose(np.array(st[0].jtj_jtr), np.array(st_o[0].jtj_jtr), rtol=1e-9, atol=1e-9)
    _pose_close(pose, pose_o)
    _pose_close(pose, world_small["T"], tol_t=0.02, tol_r=0.01)   # and it is the right answer


def test_scan_to_map_ceres_pose(ctx48, oracle, world_small, s2m_case):
    rc, pose_o, st_o = oracle.scan_to_map_ceres(s2m_case["tree"], s2m_case["ds"], world_small["guess"], 2, 15)
    pose, st = ctx48.scan_to_map(s2m_case["ds"], world_small["guess"], 2, max_num_iter=15, mode=0)
    assert [s.lm_iters for s in st] == [s.lm_iters for s in st_o]
    assert [s.n_corr for s in st] == [s.n_corr for s in st_o]
    _pose_close(pose, pose_o)


def test_few_map_points_leaves_pose(ctx48, world_small):
    import liliom_b200 as L
    c = L.Context(variant=0)
    c.map_set_points(world_small["map"][:5])
    with pytest.raises(L.LiliomError) as e:
        c.scan_to_map(world_small["map"][:100], world_small["guess"], 2)
    assert e.value.code == -3
    c.close()


def test_map_lifecycle_matches_reference_pipeline(oracle, world_small):
    """push_frame (transformCloud) + FIFO + VoxelGrid(0.4) == oracle concat + voxelgrid."""
    import liliom_b200 as L
    c = L.Context(variant=0)
    c.params.max_map_frames  # default 20
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    rng = np.random.default_rng(5)
    frames = []
    for k in range(23):
        pose = np.array(world_small["T"]); pose[4] += 0.3 * k; pose[5] += 0.05 * k
        sub = ds[rng.permutation(len(ds))[: len(ds) // 2]]
        c.map_push_frame(sub, pose)
        frames.append(oracle.transform_cloud(sub, pose))
    m = c.map_rebuild()
    want = oracle.voxelgrid(np.concatenate(frames[-20:]), 0.4)
    got = c.map_download()
    assert m == len(want) == len(got)
    for k, f in enumerate(("x", "y", "z")):                       # every channel the search reads; w carries the point's index
        assert np.array_equal(got[:, k].view(np.uint32), want[f].view(np.uint32)), f
    assert np.array_equal(got[:, 3].view(np.int32), np.arange(m, dtype=np.int32))
    # ... and the map a scan is matched against is that cloud: same correspondences as the oracle's kd-tree over it
    m4 = np.ones((m, 4), np.float32); m4[:, 0] = want["x"]; m4[:, 1] = want["y"]; m4[:, 2] = want["z"]
    tree = oracle.KdTree(m4)
    cnt, valid_o, plane_o, idx_o, pw_o = oracle.find_surf_corr(tree, ds, world_small["guess"])
    valid, plane, idx, sqd, s29 = c.find_surf_corr(ds, world_small["guess"])
    assert np.array_equal(valid, valid_o) and cnt > 100
    _, sqd_o = tree.knn5(pw_o)
    inside = sqd_o[:, 4] < 1.0
    assert np.array_equal(idx[inside], idx_o[inside])
    c.close()


def test_map_rebuild_box_escape_rebuilds_exact_grid(oracle, world_small, monkeypatch):
    """The rebuild takes the cell grid's box from the frames' boxes (no pass over the map).  A centroid outside that box must be
    noticed (k_cell_keys' escape flag) and the grid rebuilt from the exact min/max: forced here with a box shrunk to one cell in
    x (LILIOM_TEST_SHRINK_BOX), and the search must return exactly what it returns with the regular box."""
    import liliom_b200 as L
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    out = []
    for shrink in (False, True):
        if shrink:
            monkeypatch.setenv("LILIOM_TEST_SHRINK_BOX", "1")
        else:
            monkeypatch.delenv("LILIOM_TEST_SHRINK_BOX", raising=False)
        c = L.Context(variant=0)
        rng = np.random.default_rng(5)
        for k in range(6):
            pose = np.array(world_small["T"]); pose[4] += 0.3 * k; pose[5] += 0.05 * k
            c.map_push_frame(ds[rng.permutation(len(ds))[: len(ds) // 2]], pose)
        m = c.map_rebuild()
        got = c.map_download()
        valid, plane, idx, sqd, s29 = c.find_surf_corr(ds, world_small["guess"])
        pose, st = c.scan_to_map(ds, world_small["guess"], 5, mode=L.MODE_GN)
        out.append((m, got.copy(), valid.copy(), idx.copy(), sqd.copy(), s29.copy(), pose.copy()))
        c.close()
    monkeypatch.delenv("LILIOM_TEST_SHRINK_BOX", raising=False)
    a, b = out
    assert a[0] == b[0] and a[0] > 1000 and a[2].sum() > 100
    for x, y in zip(a[1:], b[1:]):
        assert x.tobytes() == y.tobytes()


# ---------------------------------------------------------------- extractors
def test_horizon_extract_bit_exact(ctx48, oracle, world_small):
    surf_o, edge_o, cut_o = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    surf, edge, cut = ctx48.extract_horizon(world_small["hz"], world_small["q_hz"])
    F = ["x", "y", "z", "nx", "ny", "nz", "intensity", "curvature"]
    _fields_equal(cut, cut_o, F)
    _fields_equal(edge, edge_o, F)
    _fields_equal(surf, surf_o, F)
    assert len(surf) > 5000 and len(edge) > 10


def test_horizon_extract_edge_cases(ctx48, oracle, world_small):
    import liliom_b200 as L
    F = ["x", "y", "z", "nx", "ny", "nz", "intensity", "curvature"]
    pts = world_small["hz"].copy()
    pts["x"][::97] = np.nan                   # removeNaN
    pts["x"][5::131] = 0.01; pts["y"][5::131] = 0.0; pts["z"][5::131] = 0.0   # removeClosedPointCloud
    pts["curvature"][7::53] = 0.0             # reflectivity gate
    pts["intensity"][11::211] = -1.0          # scan_id < 0
    pts["intensity"][13::223] = 6.02          # scan_id >= N_SCANS (reference UB, guarded in both)
    q = np.array([1.0, 0.001, -0.002, 0.01])
    for a, b in zip(ctx48.extract_horizon(pts, q), oracle.extract_horizon(pts, q)):
        _fields_equal(a, b, F)
    empty = np.zeros(0, L.PT48)
    s, e, c = ctx48.extract_horizon(empty, q)
    assert len(s) == len(e) == len(c) == 0
    # NaN q_iMU resets to identity (Preprocessing.cpp:232-234)
    qn = np.array([np.nan, 0, 0, 0])
    for a, b in zip(ctx48.extract_horizon(world_small["hz"], qn), oracle.extract_horizon(world_small["hz"], qn)):
        _fields_equal(a, b, F)


def test_horizon_extract_single_launch_shapes(ctx48, oracle, world_small):
    """The extractor runs as one cooperative launch; block b owns a contiguous slice of the sweep.  Sweeps longer than
    grid x 256 points give every thread several points (the stable compaction order must survive), tiny sweeps leave
    most blocks empty, and back-to-back calls alternate the barrier words."""
    F = ["x", "y", "z", "nx", "ny", "nz", "intensity", "curvature"]
    base = world_small["hz"]
    rng = np.random.default_rng(11)
    big = np.concatenate([base, base, base, base])       # ~4x the returns: later duplicates lose every cell claim
    big["x"][len(base):] += rng.normal(0, 0.01, len(big) - len(base)).astype(np.float32)
    big["x"][3::41] = np.nan
    q = world_small["q_hz"]
    for pts in (big, base[:700], base[:1], big[:50001], base):
        for a, b in zip(ctx48.extract_horizon(pts, q), oracle.extract_horizon(pts, q)):
            _fields_equal(a, b, F)


@pytest.mark.parametrize("ds_rate", [1, 4])
def test_rot_extract_bit_exact(oracle, world_small, ds_rate):
    import liliom_b200 as L
    p = L.default_params(1)
    p.ds_rate = ds_rate
    c = L.Context(p)
    q_lb = np.array([0.999, 0.01, -0.02, 0.03]); q_lb /= np.linalg.norm(q_lb)
    rc, surf_o, edge_o, cut_o, lab_o, cur_o = oracle.extract_rot(world_small["hdl"], world_small["q_hdl"], q_lb, 64, ds_rate)
    surf, edge, cut = c.extract_rot(world_small["hdl"], world_small["q_hdl"], q_lb)
    lab, cur = c.extract_rot_labels(len(cut))
    F = ["x", "y", "z", "intensity"]
    _fields_equal(cut, cut_o, F)
    assert np.array_equal(cur.view(np.uint32), cur_o.view(np.uint32))
    assert np.array_equal(lab, lab_o)
    _fields_equal(edge, edge_o, F)
    _fields_equal(surf, surf_o, F)
    assert len(edge) > 50 and len(surf) > 1000
    c.close()


def test_rot_extract_walk_paths_identical(oracle, world_small, monkeypatch):
    """k_rot_ring has two walks over a segment's sorted candidates: the availability-mask walk (segments up to 1024 points, every
    real sensor) and the general bitonic-sort + batch walk kept for longer segments.  LILIOM_ROT_SLOW_WALK forces the general one;
    both must give the oracle's features and labels bit for bit."""
    import liliom_b200 as L
    q_lb = np.array([0.999, 0.01, -0.02, 0.03]); q_lb /= np.linalg.norm(q_lb)
    F = ["x", "y", "z", "intensity"]
    for ds_rate in (1, 4):
        rc, surf_o, edge_o, cut_o, lab_o, cur_o = oracle.extract_rot(world_small["hdl"], world_small["q_hdl"], q_lb, 64, ds_rate)
        for slow in (False, True):
            if slow:
                monkeypatch.setenv("LILIOM_ROT_SLOW_WALK", "1")
            else:
                monkeypatch.delenv("LILIOM_ROT_SLOW_WALK", raising=False)
            p = L.default_params(1)
            p.ds_rate = ds_rate
            c = L.Context(p)
            surf, edge, cut = c.extract_rot(world_small["hdl"], world_small["q_hdl"], q_lb)
            lab, cur = c.extract_rot_labels(len(cut))
            c.close()
            _fields_equal(cut, cut_o, F)
            assert np.array_equal(lab, lab_o), (ds_rate, slow)
            _fields_equal(edge, edge_o, F)
            _fields_equal(surf, surf_o, F)
    monkeypatch.delenv("LILIOM_ROT_SLOW_WALK", raising=False)


def test_rot_extract_16_lines_and_errors(oracle, world_small):
    import liliom_b200 as L
    p = L.default_params(1); p.line_num = 16; p.ds_rate = 1
    c = L.Context(p)
    pts = world_small["hdl"][::3].copy()
    rc, surf_o, edge_o, cut_o, lab_o, cur_o = oracle.extract_rot(pts, world_small["q_hdl"], (1, 0, 0, 0), 16, 1)
    surf, edge, cut = c.extract_rot(pts, world_small["q_hdl"])
    F = ["x", "y", "z", "intensity"]
    _fields_equal(cut, cut_o, F); _fields_equal(edge, edge_o, F); _fields_equal(surf, surf_o, F)
    c.close()
    p.line_num = 20
    c = L.Context(p)
    with pytest.raises(L.LiliomError) as e:
        c.extract_rot(pts, world_small["q_hdl"])
    assert e.value.code == -6
    c.close()


# ---------------------------------------------------------------- backend kernel reuse
def test_backend_correspondences(ctx48, oracle, world_small, s2m_case):
    feats = s2m_case["ds"]
    pose = world_small["guess"]
    v_o, pl_o, sc_o = oracle.correspond_surf_backend(s2m_case["tree"], feats, pose, 1.0, 0.1, 0.3, 0.5)
    v, pl, sc = ctx48.correspond_surf(feats, pose, 1.0, 0.1, 0.3, 0.5)
    assert np.array_equal(v, v_o) and v.sum() > 100
    # backend_corr.cu is compiled without contraction: the same bits as the oracle
    assert pl.tobytes() == pl_o.tobytes() and sc.tobytes() == sc_o.tobytes()
    for variant in (0, 1):
        ve_o, pa_o, pb_o = oracle.correspond_edge(s2m_case["tree"], feats, pose, variant)
        ve, pa, pb = ctx48.correspond_edge(feats, pose, variant)
        assert np.array_equal(ve, ve_o)
        assert pa.tobytes() == pa_o.tobytes() and pb.tobytes() == pb_o.tobytes()


# ---------------------------------------------------------------- size-independent properties at BASELINE sizes
def test_full_size_properties():
    """1 M-point map, dense 20k-query sweep: (i) kNN equals scipy's exact kd-tree, (ii) GN is
    deterministic run to run, (iii) the pose error shrinks to the noise floor."""
    import liliom_b200 as L
    from liliom_b200 import synth
    from scipy.spatial import cKDTree
    m, _ = synth.make_map(1_000_000)
    T = synth.default_true_pose()
    hz, q = synth.make_horizon_sweep(T)
    c = L.Context(variant=0)
    c.map_set_points(m)
    surf, edge, cut = c.extract_horizon(hz, q)
    guess = synth.perturbed_pose(T)
    valid, plane, idx, sqd, s29 = c.find_surf_corr(surf, guess)
    # transformed queries via the same fp64 expression (numpy) -> fp32
    qv = np.asarray(guess[:4]); t = np.asarray(guess[4:])
    p = np.stack([surf["x"], surf["y"], surf["z"]], 1).astype(np.float64)
    uv = 2.0 * np.cross(qv[1:], p); pw = (p + qv[0] * uv + np.cross(qv[1:], uv) + t).astype(np.float32)
    d, ii = cKDTree(m[:, :3].astype(np.float64)).query(pw.astype(np.float64), k=5)
    inside = d[:, 4] < 0.999
    same = np.sort(idx[inside], 1) == np.sort(ii[inside].astype(np.int32), 1)
    assert same.all(1).mean() > 0.9999      # fp64 vs fp32 distance ties may reorder a handful
    p1, _ = c.scan_to_map(surf, guess, 10, mode=1)
    p2, _ = c.scan_to_map(surf, guess, 10, mode=1)
    assert np.array_equal(p1, p2)
    assert np.linalg.norm(p1[4:] - T[4:]) < 0.02
    c.close()


# ---------------------------------------------------------------- committed golden vectors (tests/golden)
def test_gpu_against_golden_fixtures(ctx48):
    import os
    import liliom_b200 as L
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    g = np.load(os.path.join(gold, "horizon_small.npz"))
    surf, edge, cut = ctx48.extract_horizon(g["pts"].view(L.PT48).reshape(-1), g["q_imu"])
    assert surf.view(np.uint8).tobytes() == g["surf"].tobytes()
    assert edge.view(np.uint8).tobytes() == g["edge"].tobytes()
    assert cut.view(np.uint8).tobytes() == g["cut"].tobytes()
    assert ctx48.voxelgrid(surf, 0.4).view(np.uint8).tobytes() == g["surf_ds"].tobytes()

    g = np.load(os.path.join(gold, "rot_small.npz"))
    p = L.default_params(1); p.ds_rate = int(g["ds_rate"]); p.line_num = int(g["line_num"])
    c = L.Context(p)
    surf, edge, cut = c.extract_rot(g["pts"].view(L.PT32).reshape(-1), g["q_imu"], g["q_lb"])
    lab, cur = c.extract_rot_labels(len(cut))
    assert cut.view(np.uint8).tobytes() == g["cut"].tobytes()
    assert np.array_equal(lab, g["label"]) and cur.tobytes() == g["curv"].tobytes()
    assert edge.view(np.uint8).tobytes() == g["edge"].tobytes()
    assert surf.view(np.uint8).tobytes() == g["surf"].tobytes()
    c.close()

    g = np.load(os.path.join(gold, "s2m_small.npz"))
    c = L.Context(variant=0)
    c.map_set_points(g["map"])
    valid, plane, idx, sqd, s29 = c.find_surf_corr(g["feats"], g["pose0"])
    assert np.array_equal(valid, g["valid"])
    ok = g["valid"] == 1
    assert np.array_equal(idx[ok], g["nn_idx"][ok])
    np.testing.assert_allclose(plane, g["plane"], rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(s29, g["neq29"], rtol=1e-9, atol=1e-9)
    pose, _ = c.scan_to_map(g["feats"], g["pose0"], 6, mode=L.MODE_GN)
    _pose_close(pose, g["pose_gn6"])
    pose, st = c.scan_to_map(g["feats"], g["pose0"], 2, max_num_iter=15, mode=L.MODE_CERES)
    _pose_close(pose, g["pose_ceres"])
    assert [s.lm_iters for s in st] == list(g["ceres_lm_iters"])
    c.close()


def test_odometry_call_and_sort_width_speculation(ctx48, oracle, world_small, s2m_case):
    """liliom_odometry = VoxelGrid(0.4) of the received surf cloud + scan-to-map.  The scan VoxelGrid sorts
    24-bit keys speculatively; a sweep whose voxel box has >= 2^24 cells must transparently redo with 32."""
    surf = s2m_case["surf"]
    for far in (False, True):
        cloud = surf.copy()
        if far:   # stretch the bounding box to ~520 x 520 x 80 voxels (> 2^24 cells)
            extra = np.zeros(4, cloud.dtype)
            extra["x"] = [-104.0, 104.0, 0.0, 0.0]; extra["y"] = [0.0, 0.0, -104.0, 104.0]; extra["z"] = [-16.0, 16.0, 0.0, 0.0]
            extra["curvature"] = 1.0
            cloud = np.concatenate([cloud, extra])
        ds_o = oracle.voxelgrid(cloud, 0.4)
        rc, pose_o, _ = oracle.scan_to_map_gn(s2m_case["tree"], ds_o, world_small["guess"], 5)
        pose, st, ds = ctx48.odometry(cloud, world_small["guess"], 5, mode=1)
        _fields_equal(ds, ds_o, ["x", "y", "z", "nx", "ny", "nz", "intensity", "curvature"])
        _pose_close(pose, pose_o)


def test_voxelgrid_cooperative_filter_paths(ctx48, ctx32, oracle, world_small, s2m_case):
    """Clouds of <= 32768 points take the single-launch cooperative filter (hash + rank by counting, no sort).
    It must give the sort chain's / oracle's bits, keep its hash table clean across calls, and hand inputs it
    declines (a voxel with > 256 members, cell coordinates beyond 2^20, PCL's index overflow) to the sort chain."""
    import liliom_b200 as L
    F48 = ["x", "y", "z", "nx", "ny", "nz", "intensity", "curvature"]
    rng = np.random.default_rng(5)
    surf = s2m_case["surf"]
    hdl = world_small["hdl"][:30000]
    dense = np.zeros(3000, L.PT48)                      # 3000 points in a handful of voxels: > 256 members each
    dense["x"] = rng.uniform(0.0, 0.8, 3000).astype(np.float32); dense["y"] = rng.uniform(0.0, 0.4, 3000).astype(np.float32)
    dense["z"] = rng.uniform(0.0, 0.4, 3000).astype(np.float32); dense["intensity"] = rng.uniform(0, 255, 3000).astype(np.float32)
    dense["nx"] = rng.normal(size=3000).astype(np.float32); dense["curvature"] = rng.uniform(0, 1, 3000).astype(np.float32)
    farpt = surf[:2000].copy(); farpt["x"][::7] += 600000.0      # |floor(x / 0.4)| > 2^20 for some points
    shifted = surf[:3000].copy(); shifted["x"] += np.float32(600000.0)   # small box, but cell coordinates beyond 2^20
    sparse = np.zeros(5000, L.PT48)                     # every point its own voxel, with NaNs sprinkled in
    sparse["x"] = rng.uniform(-80, 80, 5000).astype(np.float32); sparse["y"] = rng.uniform(-80, 80, 5000).astype(np.float32)
    sparse["z"] = rng.uniform(-5, 5, 5000).astype(np.float32); sparse["x"][::97] = np.nan; sparse["z"][5::131] = np.inf
    for rep in range(3):                                # alternate inputs: rotating control slots, table hand-back
        for cloud, leaf in ((surf, 0.4), (dense, 0.4), (sparse, 0.4), (farpt, 0.4), (shifted, 0.4), (surf, 0.2), (dense, 0.05)):
            _fields_equal(ctx48.voxelgrid(cloud, leaf), oracle.voxelgrid(cloud, leaf), F48)
        _fields_equal(ctx32.voxelgrid(hdl, 0.6), oracle.voxelgrid(hdl, 0.6), ["x", "y", "z", "intensity"])
    # the odometry entry point: declined inputs are redone transparently, then the next call is cooperative again
    for cloud in (surf, np.concatenate([surf, dense]), farpt, surf):
        ds_o = oracle.voxelgrid(cloud, 0.4)
        rc, pose_o, _ = oracle.scan_to_map_gn(s2m_case["tree"], ds_o, world_small["guess"], 3)
        pose, st, ds = ctx48.odometry(cloud, world_small["guess"], 3, mode=1)
        _fields_equal(ds, ds_o, F48)
        _pose_close(pose, pose_o)


def test_backend_reflectivity_weighted_planes(oracle, world_small, s2m_case):
    """Horizon BackendFusion variant (L/src/BackendFusion.cpp:1601-1681): reflectivity-weighted plane rows."""
    import liliom_b200 as L
    rng = np.random.default_rng(9)
    # a surf local map in the PCL layout with a reflectivity channel: the down-sampled features of the sweep, at the true pose
    ds = s2m_case["ds"].copy()
    map_cloud = oracle.transform_cloud(ds, world_small["T"])
    map_cloud["curvature"] = rng.uniform(1.0, 20.0, len(map_cloud)).astype(np.float32)
    map_cloud["curvature"][::17] = 5.0                                 # exact reflectivity ties -> 1/0 rows, as in the reference
    feats = ds.copy()
    feats["curvature"] = rng.uniform(1.0, 20.0, len(feats)).astype(np.float32)
    feats["curvature"][::17] = 5.0
    m4 = np.ones((len(map_cloud), 4), np.float32); m4[:, 0] = map_cloud["x"]; m4[:, 1] = map_cloud["y"]; m4[:, 2] = map_cloud["z"]
    tree = oracle.KdTree(m4)
    pose = world_small["guess"]
    c = L.Context(variant=0)
    c.map_set_cloud(map_cloud)
    for thres in (40.0, 25.0):
        v_o, pl_o, sc_o = oracle.correspond_surf_backend(tree, feats, pose, 1.0, 0.18, 0.2, 0.8, map_cloud["curvature"], feats["curvature"], thres)
        v, pl, sc = c.correspond_surf_refl(feats, pose, 1.0, 0.18, 0.2, 0.8, thres)
        assert np.array_equal(v, v_o)
        assert pl.tobytes() == pl_o.tobytes()
        # lidar_const * (weight + exp(-sum_w)): CUDA's exp is within 1 ulp and glibc may round the other way; times lidar_const
        # that is at most two ulps of the score (tests/test_gpu_backend_adversarial.py)
        assert np.all(np.abs(sc - sc_o) <= 2 * np.spacing(np.abs(sc_o)))
    assert v_o.sum() > 20
    c.close()


# ---------------------------------------------------------------- ROT package end to end (BASELINE configs[2] as a parity case)
def test_rot_pipeline_extract_downsample_scan_to_map(ctx32, oracle, world_small):
    """HDL-64E sweep -> LiLi-OM-ROT extractor -> VoxelGrid(0.4) -> scan-to-map on 32-byte points
    (R/src/Preprocessing.cpp + R/src/LidarOdometry.cpp), GN and Ceres-faithful modes."""
    import liliom_b200 as L
    rc, surf_o, edge_o, cut_o, lab_o, cur_o = oracle.extract_rot(world_small["hdl"], world_small["q_hdl"], (1, 0, 0, 0), 64, 4)
    surf, edge, cut = ctx32.extract_rot(world_small["hdl"], world_small["q_hdl"])
    _fields_equal(surf, surf_o, ["x", "y", "z", "intensity"])
    ctx32.map_set_points(world_small["map"])
    tree = oracle.KdTree(world_small["map"])
    ds_o = oracle.voxelgrid(surf_o, 0.4)
    for mode, run_o in ((1, lambda: oracle.scan_to_map_gn(tree, ds_o, world_small["guess"], 6)),
                        (0, lambda: oracle.scan_to_map_ceres(tree, ds_o, world_small["guess"], 2, 12))):
        rc, pose_o, st_o = run_o()
        pose, st, ds = ctx32.odometry(surf, world_small["guess"], 6 if mode == 1 else 2, max_num_iter=12, mode=mode)
        _fields_equal(ds, ds_o, ["x", "y", "z", "intensity"])
        _pose_close(pose, pose_o)
        assert [s.n_corr for s in st] == [s.n_corr for s in st_o] or mode == 1
    _pose_close(pose, world_small["T"], tol_t=0.03, tol_r=0.01)


# ---------------------------------------------------------------- ragged / degenerate inputs
def test_scan_to_map_edge_cases(ctx48, oracle, world_small, s2m_case):
    import liliom_b200 as L
    guess = world_small["guess"]
    # no features: the pose is returned unchanged in both modes
    for mode in (0, 1):
        pose, st = ctx48.scan_to_map(np.zeros((0, 4), np.float32), guess, 3, mode=mode)
        assert np.array_equal(pose, guess) and all(s.n_corr == 0 for s in st)
    # one feature, and features that are nowhere near the map (every 5th neighbour beyond 1 m): no correspondence, no step
    far = np.ones((64, 4), np.float32); far[:, :3] += 5000.0
    pose, st = ctx48.scan_to_map(far, guess, 2, mode=1)
    assert np.array_equal(pose, guess) and st[0].n_corr == 0
    one = s2m_case["ds"][:1]
    rc, pose_o, _ = oracle.scan_to_map_gn(s2m_case["tree"], one, guess, 2)
    pose, st = ctx48.scan_to_map(one, guess, 2, mode=1)
    assert np.all(np.isfinite(pose))
    # a map with exact duplicate points and a collinear run (rank-deficient plane fits take the QR path)
    m = world_small["map"][:20000].copy()
    m = np.concatenate([m, m[:500], np.stack([np.linspace(0, 30, 400), np.full(400, 3.0), np.full(400, 1.0), np.ones(400)], 1).astype(np.float32)])
    c = L.Context(variant=0)
    c.map_set_points(m)
    tree = oracle.KdTree(m)
    q = np.ones((300, 4), np.float32)
    q[:, 0] = np.linspace(0.2, 29.7, 300); q[:, 1] = 3.02; q[:, 2] = 1.01
    ident = np.array([1.0, 0, 0, 0, 0, 0, 0])
    cnt, valid_o, plane_o, idx_o, pw_o = oracle.find_surf_corr(tree, q, ident)
    valid, plane, idx, sqd, s29 = c.find_surf_corr(q, ident)
    _, sqd_o = tree.knn5(pw_o)
    inside = sqd_o[:, 4] < 1.0
    assert inside.sum() > 200 and np.array_equal(idx[inside], idx_o[inside])
    assert np.array_equal(valid, valid_o)
    ok = valid_o == 1
    np.testing.assert_allclose(plane[ok], plane_o[ok], rtol=1e-4, atol=1e-5)
    c.close()


def test_map_too_large_for_dense_grid():
    import liliom_b200 as L
    c = L.Context(variant=0)
    m = np.ones((16, 4), np.float32)
    m[:, 0] = np.linspace(-4e5, 4e5, 16); m[:, 1] = np.linspace(-4e5, 4e5, 16)
    with pytest.raises(L.LiliomError) as e:
        c.map_set_points(m)
    assert e.value.code == -5           # LILIOM_E_GRID: extent needs more than 2^29 one-metre cells
    for bad in (np.nan, np.inf):        # a non-finite map point is an argument error, not a point outside the box
        m = np.ones((16, 4), np.float32)
        m[7, 1] = bad
        with pytest.raises(L.LiliomError) as e:
            c.map_set_points(m)
        assert e.value.code == -1       # LILIOM_E_ARG
    c.close()


# ---------------------------------------------------------------- (f2) incremental device map
@pytest.mark.parametrize("variant", [0, 1])
def test_incremental_map_update_equals_rebuild_over_a_stream(oracle, world_small, variant):
    """liliom_map_update (push + incremental merge of the resident voxel entries, map.cu) against the oracle's
    concat + VoxelGrid(0.4) of the last 20 frames, every scan of a 46-scan stream, every field bit for bit; and against a second
    context that takes the two-step path (push_frame + rebuild): same cloud, same correspondences.  The stream has overlapping
    frames (most voxels hold points of several frames), an empty frame, non-finite points, a frame of exact duplicates, and a
    plain liliom_map_push_frame in the middle (the entry array must be rebuilt once after it)."""
    import liliom_b200 as L
    c = L.Context(variant=variant)
    two = L.Context(variant=variant)
    if variant == 0:
        surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
        F = ["x", "y", "z", "nx", "ny", "nz", "intensity", "curvature"]
    else:
        rc, surf, _, _, _, _ = oracle.extract_rot(world_small["hdl"], world_small["q_hdl"], (1.0, 0, 0, 0), 64, 4)
        F = ["x", "y", "z", "intensity"]
    ds = oracle.voxelgrid(surf, 0.4)
    rng = np.random.default_rng(31 + variant)
    frames = []
    for k in range(46):
        pose = np.array(world_small["T"]); pose[4] += 0.11 * k; pose[5] += 0.03 * k
        half = np.deg2rad(0.4 * k) / 2
        pose[:4] = [np.cos(half), 0.0, 0.0, np.sin(half)]
        sub = ds[np.sort(rng.permutation(len(ds))[: int(len(ds) * rng.uniform(0.3, 0.9))])].copy()
        if k == 7:
            sub = sub[:0]                                   # an empty frame
        if k == 11:
            sub["x"][::13] = np.nan; sub["z"][5::29] = np.inf   # non-finite points are dropped by the filter
        if k == 17:
            sub = np.concatenate([sub[:300]] * 3)           # exact duplicates: three members per voxel from one frame
        world = oracle.transform_cloud(sub, pose)
        frames.append(world)
        if k == 23:                                         # the two separate calls on the incremental context
            c.map_push_frame(sub, pose)
            m = c.map_rebuild()
        else:
            m = c.map_update(sub, pose)
        two.map_push_frame(sub, pose)
        m2 = two.map_rebuild()
        live = [f for f in frames[-20:] if len(f)]
        want = oracle.voxelgrid(np.concatenate(live), 0.4) if live else frames[0][:0]
        got = c.map_download_cloud()
        assert m == m2 == len(want) == len(got), (k, m, m2, len(want))
        _fields_equal(got, want, F)
        a, b = c.map_download(), two.map_download()
        assert a.view(np.uint32).tobytes() == b.view(np.uint32).tobytes(), k
        if k in (3, 19, 20, 21, 24, 45):                    # FIFO filling, first pops, after the rebuild-all, the end
            va, pa, ia, sa, na = c.find_surf_corr(ds, world_small["guess"])
            vb, pb, ib, sb, nb = two.find_surf_corr(ds, world_small["guess"])
            assert np.array_equal(va, vb) and np.array_equal(ia, ib) and pa.tobytes() == pb.tobytes() and na.tobytes() == nb.tobytes()
    c.close(); two.close()


def test_incremental_map_falls_back_when_keys_do_not_fit(oracle, world_small):
    """Voxel coordinates beyond 2^20 (or PCL's int32 index overflow) cannot be keyed absolutely: liliom_map_update must take
    the sort chain for such a FIFO and return to the incremental path once the offending frame has left it."""
    import liliom_b200 as L
    p = L.default_params(0); p.max_map_frames = 3
    c = L.Context(p)
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    ds = ds[(np.abs(ds["y"]) < 3.0) & (np.abs(ds["z"]) < 3.0)][:2000]      # a thin strip: the 1 m cell grid must still hold the stretched extent
    assert len(ds) > 200
    ident = np.array([1.0, 0, 0, 0, 0, 0, 0])
    frames = []
    for k in range(8):
        f = ds.copy(); f["x"] += np.float32(0.37 * k)
        if k == 2:
            f["x"][:5] += np.float32(600000.0)              # |floor(x / 0.4)| > 2^20
        frames.append(oracle.transform_cloud(f, ident))
        m = c.map_update(f, ident)
        want = oracle.voxelgrid(np.concatenate(frames[-3:]), 0.4)
        got = c.map_download_cloud()
        assert m == len(want) == len(got), k
        _fields_equal(got, want, ["x", "y", "z", "nx", "ny", "nz", "intensity", "curvature"])
    c.close()


def test_map_past_64_frames_equals_reference_pipeline(oracle, world_small):
    """A FIFO longer than one concatenation launch holds (max_map_frames 70, 64 frames per launch): liliom_map_rebuild and
    liliom_map_update (the two-step path at this FIFO length) against the oracle's VoxelGrid(0.4) of the concatenation, every
    field bit for bit, at 64 frames, 65, 70 and after four pops.  One frame of the second launch is empty."""
    import liliom_b200 as L
    p = L.default_params(0); p.max_map_frames = 70
    a, b = L.Context(p), L.Context(p)
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    fields = ["x", "y", "z", "nx", "ny", "nz", "intensity", "curvature"]
    rng = np.random.default_rng(41)
    frames = []
    for k in range(74):
        pose = np.array(world_small["T"]); pose[4] += 0.07 * k; pose[5] += 0.02 * k
        sub = ds[np.sort(rng.permutation(len(ds))[: int(len(ds) * rng.uniform(0.05, 0.3))])].copy()
        if k == 66:
            sub = sub[:0]
        frames.append(oracle.transform_cloud(sub, pose))
        a.map_push_frame(sub, pose)
        mb = b.map_update(sub, pose)
        if k in (63, 64, 69, 73):
            ma = a.map_rebuild()
            want = oracle.voxelgrid(np.concatenate(frames[-70:]), 0.4)
            assert ma == mb == len(want), (k, ma, mb, len(want))
            _fields_equal(a.map_download_cloud(), want, fields)
            _fields_equal(b.map_download_cloud(), want, fields)
            assert a.map_download().tobytes() == b.map_download().tobytes(), k
    a.close(); b.close()


def test_map_download_cloud_after_an_install_reports_no_map(oracle, world_small):
    """An installed map (liliom_map_set_points) has no filtered cloud behind it: liliom_map_download_cloud returns LILIOM_E_NOMAP,
    not the cloud of an earlier rebuild and not a copy from a buffer no rebuild has written.  The next rebuild brings the FIFO's
    cloud back, and after liliom_map_clear the cloud is empty.  Only size queries are made while the answer may be stale."""
    import ctypes as C
    import liliom_b200 as L
    lib = L._binding.lib()

    def size_query(c):
        n = C.c_int(-7)
        return lib.liliom_map_download_cloud(c._h, None, 0, C.byref(n)), n.value

    fresh = L.Context(variant=0)
    fresh.map_set_points(world_small["map"][:5000])
    assert size_query(fresh)[0] == L._binding.E_NOMAP
    assert "installed" in lib.liliom_last_error(fresh._h).decode()
    fresh.close()

    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    fields = ["x", "y", "z", "nx", "ny", "nz", "intensity", "curvature"]
    c = L.Context(variant=0)
    frames = []
    for k in range(4):
        pose = np.array(world_small["T"]); pose[4] += 0.3 * k
        c.map_push_frame(ds, pose)
        frames.append(oracle.transform_cloud(ds, pose))
    m = c.map_rebuild()
    want = oracle.voxelgrid(np.concatenate(frames), 0.4)
    _fields_equal(c.map_download_cloud(), want, fields)
    c.map_set_points(world_small["map"][: m // 2])
    assert size_query(c)[0] == L._binding.E_NOMAP
    with pytest.raises(L.LiliomError) as e:
        c.map_download_cloud()
    assert e.value.code == L._binding.E_NOMAP
    assert c.map_rebuild() == m
    _fields_equal(c.map_download_cloud(), want, fields)
    c.map_clear()
    assert size_query(c) == (L._binding.OK, 0)
    c.close()
