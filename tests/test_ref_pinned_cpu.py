"""The oracle pinned to the reference's own code: the reference's FormatConvert, both Preprocessing nodes and both LidarOdometry
translation units, compiled unmodified against the shim headers of oracle/ref/ (oracle/_ref/libref_*.so, tests/ref_lib.py), are
compared with the oracle's restatement of the same lines, every published field bit for bit.  The shims forward every Eigen, PCL
and FLANN routine to the oracle's own from-knowledge restatement, so what is checked here is the reading of the reference's lines:
comparisons, float/double widths, int(float) truncations, loop bounds, the order of the rules.  The libraries exist where build()
found the reference tree; elsewhere this module is skipped."""
import math
import os
import re
import subprocess

import numpy as np
import pytest

import ref_lib as R
from ref_cases import (DBL_EPS, Q_LB, hz_safe as _hz_safe, hz_sweeps as _hz_sweeps, imu_streams as _imu_streams,
                       quats as _quats, rot_cut_nonempty as _rot_cut_nonempty, rot_tied as _rot_tied)
import ref_cases as RC

pytestmark = pytest.mark.skipif(not R.available(), reason="oracle/_ref/ not built (build() needs the reference tree)")

F = np.float32


def _bytes_equal(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    if len(got) == 0:
        return
    # every field of both layouts is a float; a NaN equals any NaN (its sign and payload are the compiler's operand order)
    g = np.ascontiguousarray(got).view(np.float32).reshape(len(got), -1)
    w = np.ascontiguousarray(want).view(np.float32).reshape(len(want), -1)
    bad = np.flatnonzero(((g.view(np.uint32) != w.view(np.uint32)) & ~(np.isnan(g) & np.isnan(w))).any(1))
    assert len(bad) == 0, (what, f"{len(bad)} of {len(got)} points differ, first {bad[:5]}", got[bad[:2]], want[bad[:2]])


# ------------------------------------------------------------------------------------------------------------ FormatConvert
def _livox_cases():
    import hz_adversarial as H
    import oracle_lib as O
    out = list(H.livox_messages())
    normal = out[0][1]
    m = normal.copy(); m["line"][::7] = 255; m["reflectivity"][::5] = 255
    out.append(("line_refl_255", m, 20))
    m = normal.copy()
    m["x"][3] = np.nan; m["y"][11] = np.inf; m["z"][19] = -np.inf
    out.append(("nonfinite_xyz", m, 20))
    out.append(("one_point", normal[:1].copy(), 20))
    return out


def test_format_convert_matches_oracle(oracle, world_small):
    """livoxLidarHandler (LiLi-OM/src/FormatConvert.cpp) against orc_convert_livox on world_small's records and at every edge"""
    import hz_adversarial as H
    cases = _livox_cases()
    pts = world_small["hz"]
    pts = pts[np.isfinite(pts["intensity"]) & (pts["intensity"] >= 0) & (pts["intensity"] < 6)]
    r = np.zeros(len(pts), oracle.LIVOX20)
    r["x"], r["y"], r["z"] = pts["x"], pts["y"], pts["z"]
    frac = (pts["intensity"] - np.floor(pts["intensity"])).astype(np.float64)
    r["offset_time"] = np.minimum(np.round(frac / 0.1 * 1e8), 1e8).astype(np.uint32); r["offset_time"][-1] = 100_000_000
    r["line"] = np.floor(pts["intensity"]).astype(np.uint8); r["reflectivity"] = (np.arange(len(pts)) % 256).astype(np.uint8)
    cases.append(("world_small", r, 20))
    n_pts = 0
    for name, recs, stride in cases:
        got = R.convert_livox(recs, stride)
        want = oracle.convert_livox(recs, stride if stride != 20 else None)
        _bytes_equal(got, want, name)
        n_pts += len(got)
    print(f"FormatConvert: {len(cases)} messages, {n_pts} points bit for bit")


# ------------------------------------------------------------------------------------------------------------ Horizon node
def test_horizon_node_matches_oracle(oracle, world_small):
    """the node's cloudHandler (L/src/Preprocessing.cpp:194-408) against orc_extract_horizon given the q_iMU it published with"""
    n_sw = n_pts = n_surf = n_edge = 0
    for name, sw in _hz_sweeps(world_small):
        pts = _hz_safe(np.ascontiguousarray(sw["pts"], R.PT48))
        surf, edge, cut, q = R.node_run(R.HorizonNode(), pts, sw["q"])
        surf_o, edge_o, cut_o = oracle.extract_horizon(pts, q)
        _bytes_equal(cut, cut_o, f"{name} cutted"); _bytes_equal(surf, surf_o, f"{name} surf"); _bytes_equal(edge, edge_o, f"{name} edge")
        n_sw += 1; n_pts += len(pts); n_surf += len(surf); n_edge += len(edge)
    print(f"Horizon node: {n_sw} sweeps, {n_pts} points, {n_surf} surf / {n_edge} edge features bit for bit")


def _imu_chain(oracle, stream, t_cur):
    """processIMU (L/src/Preprocessing.cpp:135-171) after imuHandler (:173-192) over `stream`, on orc_solve_rotation"""
    import ctypes as C
    L = oracle.lib()
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    q = np.array([1.0, 0.0, 0.0, 0.0])
    gyr0 = np.array(stream[0][1], np.float64)
    cur = stream[0][0]
    r = np.zeros(3)
    i = 0
    while stream[i][0] < t_cur:
        t = stream[i][0]
        dt = t - cur
        cur = stream[i][0]
        r = np.array(stream[i][1], np.float64)
        L.orc_solve_rotation(dp(q), dp(gyr0), dp(r), dt); gyr0 = r
        i += 1
        if i >= len(stream):
            break
    if i < len(stream):
        dt1 = t_cur - cur
        dt2 = stream[i][0] - t_cur
        w1 = dt2 / (dt1 + dt2); w2 = dt1 / (dt1 + dt2)
        g = np.array(stream[i][1], np.float64)
        r = np.array([w1 * r[k] + w2 * g[k] for k in range(3)])
        L.orc_solve_rotation(dp(q), dp(gyr0), dp(r), dt1); gyr0 = r
    return q


def test_horizon_q_imu_matches_solve_rotation_chain(oracle, world_small):
    """q_iMU as the node integrates the gyro (imuHandler + processIMU + solveRotation + deltaQ) against orc_solve_rotation over
    irregular stamps, a stamp equal to the scan time, a single message and the interpolation branch; then the sweep against the
    oracle at that q"""
    t0, t_cur, streams = _imu_streams()
    for name, stream in streams.items():
        assert len(stream) <= 600
        node = R.HorizonNode()
        for st, gy in stream:
            node.imu(st, gy)
        assert node.cloud(t0, world_small["hz"]) is None
        assert node.cloud(t_cur, np.zeros(0, R.PT48)) is None
        surf, edge, cut, q = node.cloud(t_cur + 0.1, np.zeros(0, R.PT48))
        want = _imu_chain(oracle, stream, t_cur)
        assert np.array_equal(q.view(np.uint64), want.view(np.uint64)), (name, q, want)
        surf_o, edge_o, cut_o = oracle.extract_horizon(world_small["hz"], q)
        _bytes_equal(surf, surf_o, name); _bytes_equal(edge, edge_o, name); _bytes_equal(cut, cut_o, name)
        print(f"q_iMU {name}: {len(stream)} IMU messages, q = {q}")


# ------------------------------------------------------------------------------------------------------------ ROT node
def _rot_compare(oracle, name, pts, q_imu, q_lb, line_num, ds_rate, features=None):
    """the node against the oracle: the ring-ordered cloud always bit for bit, the features bit for bit unless a sort range holds
    tied candidates.  Returns (points, surf, edge, tied)."""
    pts = np.ascontiguousarray(pts, R.PT32)
    surf, edge, cut, q = R.node_run(R.RotNode(line_num, ds_rate, q_lb), pts, q_imu)
    rc, surf_o, edge_o, cut_o, _, curv = oracle.extract_rot(pts, q, q_lb, line_num, ds_rate)
    assert rc == 0
    _bytes_equal(cut, cut_o, f"{name} cloud")
    tied = _rot_tied(cut_o, curv, line_num)
    if features or (features is None and not tied):
        _bytes_equal(edge, edge_o, f"{name} edge"); _bytes_equal(surf, surf_o, f"{name} surf")
    return len(pts), len(surf), len(edge), tied


def test_rot_node_matches_oracle_world(oracle, world_small):
    """the ROT node's cloudHandler (R/src/Preprocessing.cpp:248-535) against orc_extract_rot on world_small's HDL-64 sweep at
    line_num 16, 32, 64, ds_rate 1-4, identity and non-identity q_lb"""
    tot = [0, 0, 0]
    for ln in (16, 32, 64):
        for ds in (1, 2, 3, 4):
            for qlb in ((1.0, 0.0, 0.0, 0.0), Q_LB):
                *got, tied = _rot_compare(oracle, f"world_small/{ln}/{ds}", world_small["hdl"], world_small["q_hdl"], qlb, ln, ds,
                                         features=True)
                tot = [a + b for a, b in zip(tot, got)]
    print(f"ROT node on world_small: 24 settings, {tot[0]} points, {tot[1]} surf / {tot[2]} edge features bit for bit")


def test_rot_node_matches_oracle_adversarial(oracle):
    """... and on every rot_adversarial sweep at its own settings, as built and with every coordinate jittered by a few ulps so
    that the lattice's equal curvatures (flat walls give exact zeros) split and the classifier's picks are compared too"""
    import rot_adversarial as RA
    rng = np.random.default_rng(31)
    n = 0; tot = [0, 0, 0]; skipped = []; tied = []
    for name, sw in RA.all_sweeps():
        if not _rot_cut_nonempty(sw["pts"]):      # the node reads points[0] of the cut cloud (:285)
            skipped.append(name); continue
        jit = np.ascontiguousarray(sw["pts"], R.PT32).copy()
        for f in ("x", "y", "z"):
            with np.errstate(all="ignore"):
                jit[f] = (jit[f] * (1.0 + rng.integers(-8, 9, len(jit)) * 2.0 ** -23)).astype(F)
        for tag, pts in (("", sw["pts"]), ("/jittered", jit)):
            *got, t = _rot_compare(oracle, name + tag, pts, sw["q_imu"], sw["q_lb"], sw["line_num"], sw["ds_rate"])
            if t:
                tied.append(name + tag)
            else:
                tot = [a + b for a, b in zip(tot, got)]
            n += 1
    print(f"ROT node: {n} adversarial sweeps, every ring-ordered cloud bit for bit; {n - len(tied)} without tied sort ranges, "
          f"{tot[0]} points, {tot[1]} surf / {tot[2]} edge features bit for bit; tied (features not compared): {tied}; "
          f"no point past the 3 m cut (not driven): {skipped}")
    assert n >= 60 and n - len(tied) >= 5


# ------------------------------------------------------------------------------------------------------------ LidarOdometry
@pytest.mark.parametrize("variant", [0, 1])
def test_undistortion_matches_oracle(oracle, variant):
    """LidarOdometry::undistortion (L/src/LidarOdometry.cpp:178-199, the ROT copy) against orc_undistort: intensities negative,
    integral, of fraction 0.1, >= 2^24, >= 2^31, NaN and +-inf; quaternions identity, |dot| either side of 1 - eps, negative w,
    180 degrees, non-unit"""
    od = R.Odometry(variant)
    pts = RC.lo_cloud(od.dtype, 200, 3 + variant)
    n = 0
    for name, q in _quats().items():
        for trans in ((0.0, 0.0, 0.0), (0.31, -1.7, 0.05)):
            got = od.undistort(pts, trans, q)
            want = oracle.undistort(pts, trans, q)
            _bytes_equal(got, want, f"{variant} {name} {trans}"); n += len(got)
    print(f"undistortion variant {variant}: {n} points bit for bit")


@pytest.mark.parametrize("variant", [0, 1])
def test_transform_cloud_and_point_match_oracle(oracle, variant):
    """transformCloud (both layouts) against orc_transform_cloud, and transformPoint's x, y, z (and normal) against it"""
    od = R.Odometry(variant)
    pts = RC.lo_cloud(od.dtype, 300, 11 + variant)
    rng = np.random.default_rng(5)
    n = 0
    for k in range(6):
        q = rng.normal(size=4) * (1.0 if k % 2 else 1.3); t = rng.uniform(-50, 50, 3)
        pose = np.concatenate([q, t])
        want = oracle.transform_cloud(pts, pose)
        _bytes_equal(od.transform_cloud(pts, pose), want, f"cloud {k}")
        tp = od.transform_point(pts, pose)
        for f in ("x", "y", "z") + (("nx", "ny", "nz", "intensity", "curvature") if variant == 0 else ("intensity",)):
            assert np.array_equal(tp[f].view(np.uint32), want[f].view(np.uint32)), f
        n += len(pts)
    print(f"transformCloud variant {variant}: {n} points bit for bit")


def _surf_compare(oracle, od, map4, feats4, pose, name):
    tree = oracle.KdTree(map4)
    cnt_o, valid, plane, _, _ = oracle.find_surf_corr(tree, feats4, pose)
    feats = od.points(feats4[:, :3])
    cnt, pts, nrm = od.find_surf_corr(od.points(map4[:, :3]), feats, pose)
    assert cnt == cnt_o, (name, cnt, cnt_o)
    _bytes_equal(pts, feats[valid.astype(bool)], f"{name} accepted points")
    ch = "intensity"
    got = np.stack([nrm["x"], nrm["y"], nrm["z"], nrm[ch]], 1)
    assert np.array_equal(got.view(np.uint32), plane[valid.astype(bool)].view(np.uint32)), name
    blank = od.points(np.zeros((cnt, 3), F)); blank["intensity"] = nrm["intensity"]
    blank["x"], blank["y"], blank["z"] = nrm["x"], nrm["y"], nrm["z"]
    _bytes_equal(nrm, blank, f"{name} normal points")   # every other field as PointType() leaves it
    return cnt


@pytest.mark.parametrize("variant", [0, 1])
def test_find_surf_corr_matches_oracle(oracle, world_small, variant):
    """findCorrespondingSurfFeatures (L/src/LidarOdometry.cpp:352-413) against orc_find_surf_corr on world_small and every
    s2m_adversarial world: the accepted set, its order, the planes and surf_res_cnt"""
    import s2m_adversarial as S
    od = R.Odometry(variant)
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    f4 = np.ones((len(ds), 4), F); f4[:, 0], f4[:, 1], f4[:, 2] = ds["x"], ds["y"], ds["z"]
    total = _surf_compare(oracle, od, np.ascontiguousarray(world_small["map"], F).reshape(-1, 4), f4, world_small["guess"], "world_small")
    nq = len(f4)
    for w in S.WORLDS:
        W = S.s2m_world(w)
        total += _surf_compare(oracle, od, np.ascontiguousarray(W["map"], F), np.ascontiguousarray(W["feats"], F), W["pose"], w)
        nq += len(W["feats"])
    print(f"findCorrespondingSurfFeatures variant {variant}: {nq} queries, {total} correspondences bit for bit")


def test_pose_composition_matches_oracle(oracle):
    """poseInitialization / computeRelative (L/src/LidarOdometry.cpp:415-480) against orc_pose_compose / orc_pose_relative"""
    import ctypes as C
    L = oracle.lib(); dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    rng = np.random.default_rng(9)
    n = 0
    for variant in (0, 1):
        od = R.Odometry(variant)
        for k in range(50):
            a = np.concatenate([rng.normal(size=4) * (1.0 if k % 3 else 0.7), rng.uniform(-100, 100, 3)])
            b = np.concatenate([rng.normal(size=4), rng.uniform(-2, 2, 3)])
            want = np.zeros(7); L.orc_pose_compose(dp(a), dp(b), dp(want))
            assert np.array_equal(od.pose_init(a, b).view(np.uint64), want.view(np.uint64)), k
            want = np.zeros(7); L.orc_pose_relative(dp(a), dp(b), dp(want))
            assert np.array_equal(od.compute_relative(a, b).view(np.uint64), want.view(np.uint64)), k
            ident = np.array([1.0, 0, 0, 0, 0, 0, 0])
            want = np.zeros(7); L.orc_pose_relative(dp(ident), dp(b), dp(want))
            assert np.array_equal(od.compute_relative(None, b).view(np.uint64), want.view(np.uint64)), k
            n += 3
    print(f"pose composition: {n} compositions bit for bit")


@pytest.mark.parametrize("variant", [0, 1])
def test_local_map_fifo_matches_oracle_pipeline(oracle, world_small, variant):
    """buildLocalMap + downSampleCloud (L/src/LidarOdometry.cpp:280-323) over 26 scans — the 20-frame FIFO fills and pops, one
    scan is empty — against the oracle's pipeline: VoxelGrid(0.4) of each scan, transformCloud by its saved pose, the map of scan
    k the VoxelGrid(0.4) of the frames saved at scans 1 .. k-1 (at most the last 20; scan 0 saves before any down-sampling, so
    its frame is empty and never enters), scan 1 matched against its own raw features"""
    od = R.Odometry(variant)
    dt = od.dtype
    if variant == 0:
        surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    else:
        _, surf, _, _, _, _ = oracle.extract_rot(world_small["hdl"], world_small["q_hdl"])
    surf = np.ascontiguousarray(surf, dt)
    rng = np.random.default_rng(21)
    saved = []
    n_maps = 0
    for k in range(26):
        s = surf[np.sort(rng.permutation(len(surf))[: len(surf) // 3])] if k != 7 else surf[:0]
        pose = np.array(world_small["T"], np.float64); pose[4] += 0.3 * k; pose[5] -= 0.07 * k
        got, ds = od.map_step(s, pose, cap=21 * len(surf) + 1)
        ds_o = oracle.voxelgrid(s, 0.4) if len(s) else s[:0]
        if k == 0:
            assert got is None
            saved.append(s[:0])
        else:
            _bytes_equal(ds, ds_o, f"scan {k} down-sampled")
            if k == 1:
                want = oracle.voxelgrid(s, 0.4)
            else:
                frames = [f for f in saved[1:]][-20:]
                cat = np.concatenate(frames) if frames else s[:0]
                want = oracle.voxelgrid(cat, 0.4) if len(cat) else cat
            _bytes_equal(got, want, f"scan {k} map"); n_maps += 1
            saved.append(oracle.transform_cloud(ds_o, pose) if len(ds_o) else ds_o)
    print(f"local map variant {variant}: {n_maps} maps bit for bit")


# ------------------------------------------------------------------------------------------------------------ fixture
def test_golden_digests_are_the_reference():
    """tests/golden/ref_pinned.json, which the device is checked against where oracle/_ref/ cannot be built, holds what the
    compiled reference publishes now, case for case (inputs included)"""
    import make_golden_ref
    want = RC.load_golden()
    got = make_golden_ref.build_entries()
    assert sorted(got) == sorted(want)
    bad = [k for k in got if got[k] != want[k]]
    assert not bad, bad[:10]
    print(f"fixture: {len(got)} cases match the compiled reference")


# ------------------------------------------------------------------------------------------------------------ copy guard
def _reference_dir():
    return os.environ.get("LILIOM_REFERENCE_DIR", os.path.join(os.path.dirname(R.ROOT), "reference"))


@pytest.mark.skipif(not os.path.isdir(os.path.join(_reference_dir(), "LiLi-OM")), reason="the reference tree is not here")
def test_no_tracked_file_copies_a_reference_line():
    """No tracked file holds a line of the reference's sources of 40 or more characters (whitespace ignored; #include lines
    exempt): the harnesses include the reference by name at build time, and the restatements are written, not pasted."""
    ref = _reference_dir()
    lines = set()
    for d, _, fs in os.walk(ref):
        for f in fs:
            if f.endswith((".cpp", ".h", ".hpp", ".py")):
                with open(os.path.join(d, f), errors="replace") as fh:
                    for ln in fh:
                        s = re.sub(r"\s+", "", ln)
                        if len(s) >= 40 and not s.startswith("#include"):
                            lines.add(s)
    files = subprocess.run(["git", "ls-files", "--cached", "--others", "--exclude-standard"], cwd=R.ROOT, capture_output=True, text=True, check=True).stdout.split()
    hits = []
    for f in files:
        p = os.path.join(R.ROOT, f)
        if not os.path.isfile(p) or f.startswith("tests/golden/"):
            continue
        with open(p, "rb") as fh:
            data = fh.read()
        if b"\0" in data[:4096]:
            continue
        for i, ln in enumerate(data.decode("utf-8", "replace").splitlines()):
            if re.sub(r"\s+", "", ln) in lines:
                hits.append(f"{f}:{i + 1}")
    print(f"copy guard: {len(lines)} reference lines, {len(files)} tracked files")
    assert not hits, hits[:20]
