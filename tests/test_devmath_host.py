"""CPU tier for the DEVICE scalar routines: liliom_b200/csrc/dev_math.cuh compiled for the host (tests/devmath_host.cpp) and
checked against NumPy and against the oracle's independent copies — the same source the kernels compile, without a GPU."""
import ctypes as C
import os

import numpy as np
import pytest

import host_build


@pytest.fixture(scope="module")
def dm():
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("CUDA headers not found")
    L = host_build.load("devmath_host", ["tests/devmath_host.cpp"],
                        ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-D_GNU_SOURCE", "-Wno-attributes", "-I", cuda_inc],
                        deps=[f"liliom_b200/csrc/{h}" for h in ("dev_math.cuh", "pcl_xform.h", "vg_box.h")])
    dp, fp = C.POINTER(C.c_double), C.POINTER(C.c_float)
    L.dm_plane_fit5.argtypes = [fp, dp]; L.dm_solve6.argtypes = [dp, dp, dp]; L.dm_gn_safe_step.argtypes = [dp, dp, dp]
    L.dm_pose_plus.argtypes = [dp, dp, dp]; L.dm_pose_plus.restype = None
    L.dm_eigen_sym3.argtypes = [dp, dp, dp]; L.dm_eigen_sym3.restype = None
    L.dm_colpiv_qr.argtypes = [dp, dp, dp]; L.dm_colpiv_qr.restype = None
    L.dm_qrot.argtypes = [dp, dp, dp]; L.dm_qrot.restype = None
    L.dm_qslerp_identity.argtypes = [dp, C.c_double, dp]; L.dm_qslerp_identity.restype = None
    L.dm_scan_id_of.argtypes = [C.c_float]; L.dm_scan_id_of.restype = C.c_int
    vp = C.c_void_p
    L.dm_plane_gate.argtypes = [dp, fp, fp, C.c_double, C.c_double, C.c_int, fp, fp]
    L.dm_plane_neq.argtypes = [vp, C.c_int, vp, vp, dp, C.c_double, dp]; L.dm_plane_neq.restype = None
    L.dm_cauchy_fold.argtypes = [dp, dp, C.c_int, C.c_double, dp]; L.dm_cauchy_fold.restype = None
    return L


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def test_plane_fit_fast_path_and_qr_fallback(dm, oracle):
    rng = np.random.default_rng(0)
    n_fast = 0
    for k in range(400):
        c = rng.uniform(-300, 300, 3)
        nrm = rng.normal(size=3); nrm /= np.linalg.norm(nrm)
        P = c + rng.uniform(-0.6, 0.6, (5, 3))
        P -= np.outer((P - c) @ nrm, nrm) * (1.0 if k % 7 == 0 else 0.98)            # every 7th patch exactly coplanar (in exact arithmetic)
        m = np.ones((5, 4), np.float32); m[:, :3] = P
        nv = np.zeros(3)
        fast = dm.dm_plane_fit5(m.ctypes.data_as(C.POINTER(C.c_float)), _d(nv))
        n_fast += fast
        A = m[:, :3].astype(np.float64)
        ref, *_ = np.linalg.lstsq(A, -np.ones(5), rcond=None)
        np.testing.assert_allclose(nv, ref, rtol=2e-6, atol=1e-9)
        np.testing.assert_allclose(nv, oracle.colpiv_qr_solve(A, -np.ones(5)), rtol=2e-6, atol=1e-9)      # the oracle's Eigen-style QR
    assert n_fast > 300
    # collinear neighbours: the fast path must decline (singular scatter) and the rank-revealing QR answer like the oracle's
    t = np.linspace(0, 1, 5)[:, None]
    m = np.ones((5, 4), np.float32); m[:, :3] = np.array([10.0, 5.0, 1.0]) + t * np.array([0.0, 0.0, 1.0])
    nv = np.zeros(3)
    assert dm.dm_plane_fit5(m.ctypes.data_as(C.POINTER(C.c_float)), _d(nv)) == 0
    np.testing.assert_allclose(nv, oracle.colpiv_qr_solve(m[:, :3].astype(np.float64), -np.ones(5)), rtol=1e-9, atol=1e-12)


def _adversarial_neighbour_sets(oracle):
    """the 5-NN sets of every adversarial backend query (tests/bk_adversarial.py), as the backend kernels see them: the edge
    sets' scatter matrices (k_backend_edge's operation order) and the surf sets' QR systems, plain and reflectivity-weighted"""
    import bk_adversarial as BK
    scat, qr = [], []
    for world in BK.WORLDS:
        W = BK.backend_world(world)
        for m4, q, edge in ((W["edge_map"], W["edge_q"], True), (BK.f4(W["surf_map"]), W["surf_q"], False)):
            w = oracle.transform_cloud(q, W["pose"])
            sel = np.stack([w["x"], w["y"], w["z"], np.ones(len(w), np.float32)], 1)
            idx, sqd = oracle.KdTree(m4).knn5(sel)
            for i in range(len(q)):
                if idx[i, 4] < 0:
                    continue
                P = m4[idx[i], :3].astype(np.float64)
                if edge:
                    c = [0.0, 0.0, 0.0]
                    for j in range(5):
                        c = [c[k] + P[j, k] for k in range(3)]
                    c = [v / 5.0 for v in c]
                    a = [0.0] * 6                     # a00 a10 a20 a11 a21 a22
                    for j in range(5):
                        z = [P[j, k] - c[k] for k in range(3)]
                        for t, (r, s) in enumerate(((0, 0), (1, 0), (2, 0), (1, 1), (2, 1), (2, 2))):
                            a[t] = a[t] + z[r] * z[s]
                    scat.append(np.array(a))
                else:
                    qr.append((P, -np.ones(5)))
                    fr = q["curvature"][i]
                    tw = np.abs(fr - W["surf_map"]["curvature"][idx[i]]).astype(np.float64)
                    sw = 0.0
                    for v in tw:
                        sw = sw + v
                    with np.errstate(divide="ignore", invalid="ignore"):
                        wv = (1.0 / tw) / sw
                        if np.isfinite(wv).all():
                            qr.append((wv[:, None] * P, -wv))
    return scat, qr


def _full3(a):
    return np.array([[a[0], a[1], a[2]], [a[1], a[3], a[4]], [a[2], a[4], a[5]]])


def test_colpiv_qr_device_copy_equals_oracle_copy(dm, oracle):
    """the device's ColPivHouseholderQR (k_backend_surf's plane fit) and the oracle's copy: the same algorithm in the same order,
    both without contraction, so the same bits, on random systems, far-from-origin ones and every adversarial neighbour set"""
    rng = np.random.default_rng(1)
    cases = [(rng.uniform(-50, 50, (5, 3)), -np.ones(5)) for _ in range(200)]
    cases += [(rng.uniform(-0.5, 0.5, (5, 3)) + rng.uniform(-700, 700, 3), -np.ones(5)) for _ in range(200)]
    _, adv = _adversarial_neighbour_sets(oracle)
    assert len(adv) > 100
    for A, b in cases + adv:
        x = np.zeros(3)
        dm.dm_colpiv_qr(_d(np.ascontiguousarray(A.reshape(-1))), _d(b.copy()), _d(x))
        assert x.tobytes() == oracle.colpiv_qr_solve(A, b).tobytes(), (A, b)


def test_eigen_sym3_device_copy_equals_oracle_copy(dm, oracle):
    """the device's 3x3 symmetric eigensolver (k_backend_edge's line fit, the Horizon extractor's patches) and the oracle's copy:
    the same bits, eigenvector signs included, on random matrices and on every adversarial edge scatter"""
    rng = np.random.default_rng(2)
    mats = []
    for k in range(300):
        B = rng.normal(size=(3, 3)) * 10.0 ** rng.integers(-3, 3)
        A = B @ B.T
        mats.append(np.array([A[0, 0], A[1, 0], A[2, 0], A[1, 1], A[2, 1], A[2, 2]]))
    adv, _ = _adversarial_neighbour_sets(oracle)
    assert len(adv) > 100
    for k, a in enumerate(mats + adv):
        ev = np.zeros(3); vec = np.zeros(9)
        dm.dm_eigen_sym3(_d(a), _d(ev), _d(vec))
        ev_o, vec_o = oracle.eigen_sym3(_full3(a))
        assert ev.tobytes() == ev_o.tobytes() and vec.tobytes() == np.ascontiguousarray(vec_o).reshape(-1).tobytes(), a
        if k < len(mats):
            np.testing.assert_allclose(ev, np.linalg.eigvalsh(_full3(a)), rtol=1e-10, atol=1e-12 * np.abs(a).max())


def test_solve6_and_pose_plus(dm):
    rng = np.random.default_rng(3)
    iu = np.triu_indices(6)
    for _ in range(200):
        J = rng.normal(size=(40, 6)) * rng.uniform(0.1, 10, 6)
        H = J.T @ J; g = rng.normal(size=6)
        x = np.zeros(6)
        assert dm.dm_solve6(_d(np.ascontiguousarray(H[iu])), _d(g), _d(x)) == 1
        np.testing.assert_allclose(x, np.linalg.solve(H, g), rtol=1e-9, atol=1e-12)
    z = np.zeros(21); x = np.zeros(6)
    assert dm.dm_solve6(_d(z), _d(np.ones(6)), _d(x)) == 0                         # zero pivot reported, no NaN accepted
    from test_oracle_cpu import ceres_plus
    for scale in (1e-9, 1e-3, 0.1, 0.24, 0.26, 1.5):                               # both sides of the Taylor / sincos switch at 0.25
        for _ in range(20):
            p = rng.normal(size=7); p[:4] /= np.linalg.norm(p[:4])
            d = rng.normal(size=6) * scale
            out = np.zeros(7)
            dm.dm_pose_plus(_d(p), _d(d), _d(out))
            np.testing.assert_allclose(out, ceres_plus(p, d), rtol=0, atol=2e-15)
    out = np.zeros(7); p = np.array([1.0, 0, 0, 0, 1, 2, 3])
    dm.dm_pose_plus(_d(p), _d(np.zeros(6)), _d(out))
    assert np.array_equal(out, p)


def test_qrot_matches_eigen_formula(dm):
    rng = np.random.default_rng(4)
    for _ in range(100):
        q = rng.normal(size=4); v = rng.normal(size=3) * 50
        out = np.zeros(3)
        dm.dm_qrot(_d(q), _d(v), _d(out))
        uv = 2.0 * np.cross(q[1:], v)
        np.testing.assert_allclose(out, v + q[0] * uv + np.cross(q[1:], uv), rtol=0, atol=1e-12)


def _upper21(H):
    return np.array([H[a, b] for a in range(6) for b in range(a, 6)], np.float64)


def test_gn_safe_step_device_copy(dm):
    """dev_math.cuh::gn_safe_step (the step every GN pass takes on the device) against NumPy: the plain solution on a well-posed
    system, the Levenberg-damped solution when a pivot falls below 1e-10 * max diag, the 0.35 rad / 5 m trust region, and a refusal
    on a zero or non-finite system (ADVICE r1: an undamped step diverges on one-wall geometry)."""
    rng = np.random.default_rng(3)
    d = np.zeros(6)
    for _ in range(200):                                   # well-posed: J^T J of 400 random rows
        J = rng.normal(size=(400, 6)) * rng.uniform(0.2, 3.0, 6)
        H = J.T @ J; g = J.T @ (rng.normal(size=400) * 0.01)
        assert dm.dm_gn_safe_step(_d(_upper21(H)), _d(-g), _d(d)) == 1
        want = np.linalg.solve(H, -g)
        assert np.allclose(d, want, rtol=1e-9, atol=1e-14)
    for _ in range(100):                                   # rank 5 (one unobservable direction): damped system
        J = rng.normal(size=(300, 6)); v = rng.normal(size=6); v /= np.linalg.norm(v)
        J = J - np.outer(J @ v, v)
        H = J.T @ J; g = J.T @ (rng.normal(size=300) * 0.01)
        assert dm.dm_gn_safe_step(_d(_upper21(H)), _d(-g), _d(d)) == 1
        lam = 1e-6 * H.diagonal().max()
        want = np.linalg.solve(H + lam * np.eye(6), -g)
        assert np.allclose(d, want, rtol=1e-6, atol=1e-10)
        assert abs(d @ v) < 1e-3 * max(np.linalg.norm(d), 1e-12) + 1e-9          # the unobservable direction is (nearly) left alone
    for _ in range(100):                                   # trust region: direction kept, norms clipped
        J = rng.normal(size=(50, 6)) * 1e-3
        H = J.T @ J; g = rng.normal(size=6) * rng.choice([1e-3, 1.0, 50.0])
        assert dm.dm_gn_safe_step(_d(_upper21(H)), _d(-g), _d(d)) == 1
        rot, tr = np.linalg.norm(d[:3]), np.linalg.norm(d[3:])
        assert rot <= 0.35 * (1 + 1e-12) and tr <= 5.0 * (1 + 1e-12)
        full = np.linalg.solve(H, -g)
        if np.linalg.norm(full[:3]) > 0.35 or np.linalg.norm(full[3:]) > 5.0:
            c = d @ full / (np.linalg.norm(d) * np.linalg.norm(full))
            assert c > 1 - 1e-6 and (abs(rot - 0.35) < 1e-9 or abs(tr - 5.0) < 1e-9)
    assert dm.dm_gn_safe_step(_d(np.zeros(21)), _d(np.ones(6)), _d(d)) == 0
    bad = _upper21(np.eye(6)); bad[0] = np.nan
    assert dm.dm_gn_safe_step(_d(bad), _d(np.ones(6)), _d(d)) == 0


def _f(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _gate_numpy(nv, m, s, plane_thres, w_gate):
    """L/src/LidarOdometry.cpp:376-405 restated in the reference's widths: fp64 normal and distances, the query's range in fp32,
    pd and the weight narrowed to fp32.  Returns (ok, normalised nv, pl, weight)."""
    f64, f32 = np.float64, np.float32
    n0, n1, n2_ = f64(nv[0]), f64(nv[1]), f64(nv[2])
    n2 = n0 * n0 + n1 * n1 + n2_ * n2_
    nn = np.sqrt(n2)
    inv = f64(1.0) / nn
    if n2 > 0:
        n0, n1, n2_ = n0 / nn, n1 / nn, n2_ / nn
    valid = not any(abs(n0 * f64(p[0]) + n1 * f64(p[1]) + n2_ * f64(p[2]) + inv) > plane_thres for p in m)
    sx, sy, sz = (f32(v) for v in s)
    nvn = np.array([n0, n1, n2_])
    if not valid:
        return False, nvn, None, None
    pd = f32(((n0 * f64(sx) + n1 * f64(sy)) + n2_ * f64(sz)) + inv)
    rng = np.sqrt(np.sqrt((sx * sx + sy * sy) + sz * sz))
    assert rng.dtype == np.float32
    w = f32(f64(1.0) - (f64(0.9) * f64(abs(pd))) / f64(rng))
    if not f64(w) > w_gate:
        return False, nvn, None, None
    pl = np.array([f32(f64(w) * n0), f32(f64(w) * n1), f32(f64(w) * n2_), f32(f64(w) * inv)], np.float32)
    return True, nvn, pl, w


def _gate_max_dist(nv, m):
    """the largest neighbour distance of the plane gate, as _gate_numpy computes it"""
    f64 = np.float64
    n0, n1, n2_ = (f64(v) for v in nv)
    nn = np.sqrt(n0 * n0 + n1 * n1 + n2_ * n2_)
    inv = f64(1.0) / nn
    n0, n1, n2_ = n0 / nn, n1 / nn, n2_ / nn
    return max(abs(n0 * f64(p[0]) + n1 * f64(p[1]) + n2_ * f64(p[2]) + inv) for p in m)


def test_plane_gate_bit_for_bit_against_numpy(dm):
    """dev_math.cuh::plane_gate (the gates of the GN pass and of the backend's surf search) against a NumPy restatement of
    L:376-405 in the reference's fp32/fp64 widths, bit for bit: flag, normalised normal, weighted plane and weight — on random
    neighbourhoods and on ones exactly at plane_thres and at w_gate, where one ulp decides."""
    rng = np.random.default_rng(5)
    n_ok = n_edge = 0
    for k in range(600):
        c = rng.uniform(-150, 150, 3); c[2] = rng.uniform(-3, 3)
        nrm = rng.normal(size=3); nrm /= np.linalg.norm(nrm)
        P = c + rng.uniform(-0.5, 0.5, (5, 3))
        P -= np.outer((P - c) @ nrm, nrm) * (1.0 - 10.0 ** rng.uniform(-4, -0.5))
        m = np.ones((5, 4), np.float32); m[:, :3] = P
        s = (c + nrm * rng.uniform(-0.4, 0.4) + rng.uniform(-0.3, 0.3, 3)).astype(np.float32)
        nv0 = np.zeros(3)
        dm.dm_plane_fit5(_f(m), _d(nv0))
        dmax = _gate_max_dist(nv0, m[:, :3])
        thr = [0.06, 0.2, float(dmax), float(np.nextafter(dmax, 0.0))]         # on the threshold: kept; one ulp below: refused
        for plane_thres in thr:
            ok_r, nvn_r, pl_r, w_r = _gate_numpy(nv0, m[:, :3], s, plane_thres, 0.1)
            gates = [0.1, 0.5]
            if ok_r:
                gates += [float(w_r), float(np.nextafter(np.float64(w_r), -np.inf))]  # weight == w_gate: refused; one ulp below: kept
            for w_gate in gates:
                ok_r, nvn_r, pl_r, w_r = _gate_numpy(nv0, m[:, :3], s, plane_thres, w_gate)
                for refuse in (0, 1):
                    nv = nv0.copy(); pl = np.full(4, -7.0, np.float32); w = np.full(1, -7.0, np.float32)
                    ok = dm.dm_plane_gate(_d(nv), _f(m), _f(s), plane_thres, w_gate, refuse, _f(pl), _f(w))
                    assert nv.tobytes() == nvn_r.tobytes()
                    assert ok == (ok_r and not refuse)
                    if ok:
                        assert pl.tobytes() == pl_r.tobytes() and w[0].tobytes() == np.float32(w_r).tobytes()
                        n_ok += 1
                        n_edge += plane_thres == dmax or w_gate != float(w_r) and w_gate not in (0.1, 0.5)
                    else:
                        assert (pl == -7.0).all() and w[0] == -7.0                  # a refused plane leaves the outputs alone
    assert n_ok > 500 and n_edge > 100


def _qrot_np(q, v):
    """Eigen's quaternion * vector on rows of v (fp64)"""
    qv = np.broadcast_to(np.asarray(q[1:], np.float64), v.shape)
    uv = 2.0 * np.cross(qv, v)
    return v + q[0] * uv + np.cross(qv, uv)


def _unit_pose(rng):
    p = np.concatenate([rng.normal(size=4), rng.uniform(-20, 20, 3)])
    p[:4] /= np.linalg.norm(p[:4])
    return p


def test_plane_rows_huber_fold_match_oracle_normal_equations(dm, oracle):
    """plane_row + huber_correct + add_row29 (the scan-to-map rows of the GN pass and of the LM solve) against the oracle's
    normal equations on random correspondences, residuals on both sides of the Huber threshold, at the tolerance the device's
    sums are held to."""
    rng = np.random.default_rng(6)
    for trial in range(6):
        n = 3000
        pose = _unit_pose(rng)
        feats = np.ones((n, 4), np.float32); feats[:, :3] = rng.uniform(-60, 60, (n, 3))
        pw = _qrot_np(pose[:4], feats[:, :3].astype(np.float64)) + pose[4:]
        nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        d = -(nrm * pw).sum(1) + rng.uniform(-0.3, 0.3, n)
        w = rng.uniform(0.3, 1.0, n)
        plane = np.concatenate([nrm * w[:, None], (d * w)[:, None]], 1).astype(np.float32)
        valid = (rng.uniform(size=n) < 0.8).astype(np.uint8)
        out = np.zeros(29)
        dm.dm_plane_neq(feats.ctypes.data, n, valid.ctypes.data, plane.ctypes.data, _d(pose), 0.1, _d(out))
        ref = oracle.normal_equations(feats, valid, plane, pose, 0.1)
        assert out[28] == ref[28] == valid.sum()
        np.testing.assert_allclose(out, ref, rtol=1e-9, atol=1e-9)


def test_cauchy_fold_matches_oracle_backend_blocks(dm, oracle):
    """cauchy_correct + add_row29 (k_backend_block's loss and fold) on LidarPlaneNormFactor and LidarEdgeFactor rows built here
    from their closed forms, against the oracle's backend blocks at the tolerances of the device's backend blocks."""
    rng = np.random.default_rng(7)
    for trial in range(4):
        n = 2000
        pose = _unit_pose(rng)
        q_lb = rng.normal(size=4); q_lb /= np.linalg.norm(q_lb); t_lb = rng.uniform(-0.2, 0.2, 3)
        feats = np.ones((n, 4), np.float32); feats[:, :3] = rng.uniform(-60, 60, (n, 3))
        valid = (rng.uniform(size=n) < 0.8).astype(np.uint8)
        sel = valid.astype(bool)
        cp = feats[:, :3].astype(np.float64)
        # surf: r = score (n~ . p_w + d~), p_w = q (q_lb^-1 (p - t_lb)) + t, g = score n~
        pbody = _qrot_np(np.array([q_lb[0], -q_lb[1], -q_lb[2], -q_lb[3]]), cp - t_lb)
        rp = _qrot_np(pose[:4], pbody)
        nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        d = -(nrm * (rp + pose[4:])).sum(1) + rng.uniform(-3.0, 3.0, n)
        w = rng.uniform(0.3, 1.0, n)
        plane = np.concatenate([nrm * w[:, None], (d * w)[:, None]], 1).astype(np.float32)
        score = rng.uniform(0.2, 1.5, n)
        pl64 = plane.astype(np.float64)
        r = score * ((pl64[:, :3] * (rp + pose[4:])).sum(1) + pl64[:, 3])
        g = score[:, None] * pl64[:, :3]
        J = np.concatenate([g, 2.0 * np.cross(rp, g)], 1)
        out = np.zeros(29)
        dm.dm_cauchy_fold(_d(np.ascontiguousarray(J[sel])), _d(np.ascontiguousarray(r[sel])), int(sel.sum()), 1.0, _d(out))
        ref = oracle.backend_surf_block(feats, valid, plane, score, pose, q_lb, t_lb, 1.0)
        assert out[28] == ref[28] == sel.sum()
        np.testing.assert_allclose(out, ref, rtol=1e-9, atol=1e-9 * np.abs(ref[:21]).max())
        # edge: r = s |u x v| / |a-b|, u = p_w - a, v = p_w - b, g = s ((a-b) x (u x v)^) / |a-b|
        s_weight = 0.6
        rp = _qrot_np(pose[:4], cp)
        lp = rp + pose[4:]
        u = rng.normal(size=(n, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
        c = lp + rng.uniform(-2.0, 2.0, (n, 3))
        pa = (c + 0.1 * u).astype(np.float32); pb = (c - 0.1 * u).astype(np.float32)
        A, B = pa.astype(np.float64), pb.astype(np.float64)
        nu = np.cross(lp - A, lp - B); de = A - B
        nn_, dn = np.linalg.norm(nu, axis=1), np.linalg.norm(de, axis=1)
        r = nn_ / dn * s_weight
        g = (s_weight / (dn * nn_))[:, None] * np.cross(de, nu)
        J = np.concatenate([g, 2.0 * np.cross(rp, g)], 1)
        dm.dm_cauchy_fold(_d(np.ascontiguousarray(J[sel])), _d(np.ascontiguousarray(r[sel])), int(sel.sum()), 1.0, _d(out))
        ref = oracle.backend_edge_block(feats, valid, pa, pb, s_weight, pose, 1.0)
        assert out[28] == ref[28] == sel.sum()
        np.testing.assert_allclose(out, ref, rtol=1e-8, atol=1e-9 * np.abs(ref[:21]).max())


def test_qslerp_branches_match_oracle(dm, oracle):
    """dev_math.cuh::qslerp_x (the de-skew's slerp from Identity, Eigen's Quaterniond::slerp) against the oracle's copy on every
    branch: the linear one (|d| >= 1 - DBL_EPSILON, non-unit q included), d < 0 (s1 negated), t < 0 (a negative intensity's
    extrapolation) and t > 1.  Compiled for the host, acos / sin are glibc's on both sides: bit for bit."""
    eps = np.finfo(np.float64).eps
    rng = np.random.default_rng(9)
    qs = [np.array([1.0, 0, 0, 0]), np.array([1.0 - eps / 2, 1e-9, -2e-9, 3e-9]), np.array([1.0 - eps, 0, 1e-9, 0]),
          np.array([1.0 - 2 * eps, 3e-8, 0, 0]), np.array([-1.0, 0, 0, 0]), np.array([-(1.0 - eps / 2), 1e-9, 0, 0])]
    for _ in range(20):
        q = rng.normal(size=4); q /= np.linalg.norm(q)
        qs += [q, -q, q * 1.3, q * 0.7]
    ts = [0.0, 1.0, 0.5, 1e-300, -0.5, -9.99, -1e-6, 1.5, 7.0, 0.999999]
    hit = set()
    out = np.zeros(4)
    for q in qs:
        d = q[0]
        for t in ts:
            dm.dm_qslerp_identity(_d(np.ascontiguousarray(q)), t, _d(out))
            ref = oracle.slerp_identity(q, t)
            assert out.tobytes() == ref.tobytes(), (q, t, out, ref)
            hit.add(("linear" if abs(d) >= 1.0 - eps else "acos", d < 0, t < 0, t > 1))
            if abs(d) >= 1.0 - eps:                      # the linear branch in closed form
                s1 = -t if d < 0 else t
                np.testing.assert_array_equal(out, [(1.0 - t) + s1 * q[0], s1 * q[1], s1 * q[2], s1 * q[3]])
    for branch in ("linear", "acos"):
        for neg in (False, True):
            assert (branch, neg, True, False) in hit and (branch, neg, False, True) in hit, (branch, neg)


def test_scan_id_of_is_x86_truncation(dm):
    """pcl_xform.h::scan_id_of: int(float) as x86-64's cvttss2si gives it, INT_MIN for NaN, +-inf and |x| >= 2^31"""
    f = np.float32
    vals = [0.0, 0.999, 5.09, -0.5, -0.999, -1.0, -1.5, 2147483520.0, -2147483648.0]
    for v in vals:
        assert dm.dm_scan_id_of(float(f(v))) == int(f(v)), v
    for v in (np.nan, np.inf, -np.inf, 3e9, -3e9, 2147483648.0, -2147483904.0, 1e38):
        assert dm.dm_scan_id_of(float(f(v))) == -2147483648, v
