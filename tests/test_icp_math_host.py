"""CPU tier for the ICP arithmetic: liliom_b200/csrc/icp_math.h compiled for the host (tests/icp_math_host.cpp), the same source
k_icp_persistent runs.  The 3x3 SVD against numpy.linalg.svd, one Umeyama step from the 17 sums against NumPy's closed form,
PCL's convergence rule against a Python restatement on inputs placed on each threshold, and the whole loop composed from the
header (brute-force 1-NN in the kernel's candidate order) against a NumPy restatement of PCL's loop."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(ROOT)
SO = os.path.join(ROOT, "build", "libicp_math_host.so")
GO, CONVERGED, STUCK = 0, 1, 2


@pytest.fixture(scope="module")
def im():
    src = os.path.join(ROOT, "tests", "icp_math_host.cpp")
    deps = [src] + [os.path.join(ROOT, "liliom_b200", "csrc", h) for h in ("icp_math.h", "pcl_xform.h", "vg_box.h")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(p) for p in deps):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-ffp-contract=off", "-shared", "-o", SO, src], check=True)
    L = C.CDLL(SO)
    dp = np.ctypeslib.ndpointer(np.float64, flags="C")
    fp = np.ctypeslib.ndpointer(np.float32, flags="C")
    L.im_svd3.argtypes = [dp, dp, dp, dp]
    L.im_det3.argtypes = [dp]
    L.im_det3.restype = C.c_double
    L.im_umeyama.argtypes = [dp, dp, dp]
    L.im_converged.argtypes = [C.c_int, C.c_int, dp, dp, C.c_double, C.c_double, C.c_double, C.c_double]
    L.im_step.argtypes = [dp, C.POINTER(C.c_double), C.POINTER(C.c_int), dp, C.c_int, C.c_double, C.c_double]
    L.im_icp.argtypes = [fp, C.c_int, fp, C.c_int, C.c_double, C.c_int, C.c_double, C.c_double, dp, C.POINTER(C.c_double),
                         C.POINTER(C.c_int), C.POINTER(C.c_int)]
    return L


def svd3(im, A):
    A = np.ascontiguousarray(A, np.float64)
    U, s, V = np.zeros((3, 3)), np.zeros(3), np.zeros((3, 3))
    im.im_svd3(A, U, s, V)
    return U, s, V


def rot(axis, ang):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def svd_inputs():
    rng = np.random.default_rng(3)
    out = [("random", rng.normal(size=(3, 3))) for _ in range(40)]
    out += [("random-scaled", rng.normal(size=(3, 3)) * 10.0 ** rng.uniform(-6, 6)) for _ in range(20)]
    for _ in range(8):
        u, v = rng.normal(size=3), rng.normal(size=3)
        out.append(("rank1", np.outer(u, v)))
        Q1, Q2 = rot(rng.normal(size=3), rng.uniform(0, 3)), rot(rng.normal(size=3), rng.uniform(0, 3))
        out.append(("rank2", Q1 @ np.diag([3.0, 0.7, 0.0]) @ Q2.T))
        out.append(("repeated", Q1 @ np.diag([2.0, 2.0, 0.5]) @ Q2.T))
        out.append(("repeated3", Q1 @ np.diag([1.5, 1.5, 1.5]) @ Q2.T))
        out.append(("negdet", Q1 @ np.diag([4.0, 1.0, 0.25]) @ Q2.T @ np.diag([1.0, 1.0, -1.0])))
    out.append(("diag", np.diag([0.0, 5.0, 2.0])))
    out.append(("identity", np.eye(3)))
    return out


@pytest.mark.parametrize("kind,A", svd_inputs(), ids=lambda x: x if isinstance(x, str) else "")
def test_svd3_against_numpy(im, kind, A):
    U, s, V = svd3(im, A)
    scale = max(np.abs(A).max(), 1e-300)
    assert np.abs(U @ np.diag(s) @ V.T - A).max() <= 1e-13 * scale * 3
    np.testing.assert_allclose(np.sort(s)[::-1], np.linalg.svd(A, compute_uv=False), rtol=0, atol=1e-13 * scale * 3)
    assert (s >= 0).all()
    np.testing.assert_allclose(V.T @ V, np.eye(3), rtol=0, atol=1e-13)
    np.testing.assert_allclose(U.T @ U, np.eye(3), rtol=0, atol=1e-12)
    if kind == "negdet":
        assert im.im_det3(np.ascontiguousarray(U)) * im.im_det3(np.ascontiguousarray(V)) < 0


def test_svd3_zero_matrix(im):
    """no direction to complete from: zero singular values, V = I, U = 0 (U S V^T is still the input)"""
    U, s, V = svd3(im, np.zeros((3, 3)))
    assert (s == 0).all() and np.array_equal(V, np.eye(3)) and not U.any()


def test_det3(im):
    rng = np.random.default_rng(9)
    for _ in range(50):
        M = rng.normal(size=(3, 3))
        assert abs(im.im_det3(M) - np.linalg.det(M)) < 1e-13 * max(1.0, abs(np.linalg.det(M)))


def sums_of(P, Q, d2=None):
    """the 17 sums of the kernel's pass: sum p, sum q, sum p q^T (row = p), sum d2, count"""
    d2 = ((P - Q) ** 2).sum(1) if d2 is None else d2
    return np.ascontiguousarray(np.concatenate([P.sum(0), Q.sum(0), (P[:, :, None] * Q[:, None, :]).sum(0).reshape(9), [d2.sum(), len(P)]]))


def np_umeyama(P, Q):
    """_icp_numpy's closed form (tests/test_gpu_widen.py)"""
    mp, mq = P.mean(0), Q.mean(0)
    S = (Q - mq).T @ (P - mp) / len(P)
    U, D, Vt = np.linalg.svd(S)
    sg = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        sg[2] = -1
    R = U @ np.diag(sg) @ Vt
    return R, mq - R @ mp


@pytest.mark.parametrize("case", ["rigid", "noisy", "reflection", "far"])
def test_umeyama_step_against_numpy(im, case):
    rng = np.random.default_rng({"rigid": 1, "noisy": 2, "reflection": 3, "far": 4}[case])
    P = rng.normal(size=(500, 3)) * np.array([4.0, 2.0, 0.7])
    R0, t0 = rot([0.2, -0.4, 1.0], 0.3), np.array([0.5, -1.2, 0.3])
    if case == "far":
        P += np.array([40.0, -25.0, 3.0])
    Q = P @ R0.T + t0
    if case == "noisy":
        Q += rng.normal(0, 0.05, Q.shape)
    if case == "reflection":
        Q = Q @ np.diag([1.0, 1.0, -1.0])          # no rotation reaches it: the sign fix on the smallest singular value
    R, t = np.zeros((3, 3)), np.zeros(3)
    im.im_umeyama(sums_of(P, Q), R, t)
    Rn, tn = np_umeyama(P, Q)
    np.testing.assert_allclose(R, Rn, rtol=0, atol=1e-12)
    np.testing.assert_allclose(t, tn, rtol=0, atol=1e-12 * max(1.0, np.abs(P).max()))
    np.testing.assert_allclose(R @ R.T, np.eye(3), rtol=0, atol=1e-13)
    assert abs(np.linalg.det(R) - 1.0) < 1e-13
    if case in ("rigid", "far"):
        np.testing.assert_allclose(R, R0, rtol=0, atol=1e-12)


def py_converged(it, max_iter, R, t, mse, prev, trans_eps, fit_eps):
    """DefaultConvergenceCriteria as icp_math.h states it, in the same fp64 operation order"""
    if it >= max_iter:
        return True
    cos_angle = 0.5 * (((R[0, 0] + R[1, 1]) + R[2, 2]) - 1.0)
    tr2 = (t[0] * t[0] + t[1] * t[1]) + t[2] * t[2]
    if cos_angle >= 1.0 - trans_eps and tr2 <= trans_eps:
        return True
    if abs(mse - prev) / prev < fit_eps:
        return True
    return abs(mse - prev) < 1e-12


def around(x, k=3):
    """x and its k nearest doubles on either side"""
    out = [x]
    lo = hi = x
    for _ in range(k):
        lo, hi = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
        out += [lo, hi]
    return out


def check_rule(im, it, max_iter, R, t, mse, prev, te, fe):
    R = np.ascontiguousarray(R, np.float64); t = np.ascontiguousarray(t, np.float64)
    got = bool(im.im_converged(it, max_iter, R, t, mse, prev, te, fe))
    assert got == py_converged(it, max_iter, R, t, mse, prev, te, fe), (it, max_iter, R, t, mse, prev, te, fe)
    return got


def test_convergence_iteration_cap(im):
    far_R, far_t = rot([0, 0, 1], 0.3), np.array([1.0, 0, 0])
    seen = {check_rule(im, it, 10, far_R, far_t, 1.0, 2.0, 1e-6, 1e-6) for it in (8, 9, 10, 11)}
    assert seen == {False, True}


def test_convergence_rotation_and_translation(im):
    te = 1e-6
    seen = set()
    for ang in (np.arccos(1.0 - te) * f for f in (0.999, 0.99999, 1.0, 1.00001, 1.001)):       # cosine on 1 - eps
        for tt in around(np.sqrt(te)):                                                          # |t|^2 on eps
            seen.add(check_rule(im, 1, 100, rot([0.3, 0.1, 1.0], ang), np.array([tt, 0.0, 0.0]), 1.0, 2.0, te, 1e-9))
            seen.add(check_rule(im, 1, 100, np.eye(3), np.array([tt, 0.0, 0.0]), 1.0, 2.0, te, 1e-9))
    for ts in around(te):
        R = np.eye(3)
        seen.add(check_rule(im, 1, 100, R, np.array([np.sqrt(ts / 3)] * 3), 1.0, 2.0, te, 1e-9))
    assert seen == {False, True}


def test_convergence_relative_and_absolute_mse(im):
    far_R, far_t = rot([0, 0, 1], 0.3), np.array([1.0, 0, 0])
    seen_rel, seen_abs = set(), set()
    for prev in (1.0, 0.37, 12.5):
        fe = 1e-6
        for mse in around(prev * (1.0 - fe), 4) + around(prev * (1.0 + fe), 4):     # relative change on fit_eps
            seen_rel.add(check_rule(im, 1, 100, far_R, far_t, mse, prev, 1e-6, fe))
        for d in around(1e-12, 4):                                                    # absolute change on 1e-12 (relative off)
            seen_abs.add(check_rule(im, 1, 100, far_R, far_t, prev + d, prev, 1e-6, 0.0))
            seen_abs.add(check_rule(im, 1, 100, far_R, far_t, prev - d, prev, 1e-6, 0.0))
    assert seen_rel == {False, True} and seen_abs == {False, True}
    # the first iteration compares against DBL_MAX: no relative or absolute verdict
    assert not check_rule(im, 1, 100, far_R, far_t, 0.5, np.finfo(np.float64).max, 1e-6, 1e-6)


def test_step_needs_three_correspondences(im):
    rng = np.random.default_rng(5)
    P = rng.normal(size=(3, 3)); Q = P + 0.1
    for n, want in ((2, STUCK), (3, GO)):
        s = sums_of(P[:n], Q[:n]) if n == 3 else sums_of(P[:2], Q[:2])
        F = np.ascontiguousarray(np.eye(4)); prev = C.c_double(np.finfo(np.float64).max); it = C.c_int(0)
        assert im.im_step(F, C.byref(prev), C.byref(it), s, 100, 1e-6, 1e-6) == want
        assert it.value == (0 if want == STUCK else 1)
        assert np.array_equal(F, np.eye(4)) == (want == STUCK)


def np_icp(src, tgt, max_corr=30.0, max_iter=100, trans_eps=1e-6, fit_eps=1e-6):
    """PCL's loop in NumPy with a brute-force 1-NN in the kernel's order (fp32 squared distance, then the index)"""
    s = src[:, :3]
    tq = tgt[:, :3]

    def nn(F):
        p = [((F[r, 0] * s[:, 0].astype(np.float64) + F[r, 1] * s[:, 1]) + F[r, 2] * s[:, 2]) + F[r, 3] for r in range(3)]
        p = np.stack(p, 1)
        pf = p.astype(np.float32)
        d = pf[:, None, :] - tq[None, :, :]
        d2 = (d[:, :, 0] * d[:, :, 0] + d[:, :, 1] * d[:, :, 1]) + d[:, :, 2] * d[:, :, 2]
        j = np.argmin(d2, 1)
        return p, j, d2[np.arange(len(p)), j]

    F = np.eye(4)
    prev, it, conv = np.finfo(np.float64).max, 0, False
    while True:
        p, j, d2 = nn(F)
        keep = d2 <= np.float32(max_corr * max_corr)
        if keep.sum() < 3:
            break
        R, t = np_umeyama(p[keep], tq[j[keep]].astype(np.float64))
        Ti = np.eye(4); Ti[:3, :3] = R; Ti[:3, 3] = t
        F = Ti @ F
        it += 1
        mse = float(d2[keep].astype(np.float64).mean())
        if py_converged(it, max_iter, R, t, mse, prev, trans_eps, fit_eps):
            conv = True
            break
        prev = mse
    _, _, d2 = nn(F)
    return F, float(d2.astype(np.float64).mean()), conv, it


def host_icp(im, src, tgt, **kw):
    args = dict(max_corr=30.0, max_iter=100, trans_eps=1e-6, fit_eps=1e-6)
    args.update(kw)
    T = np.zeros(16); fit = C.c_double(); conv = C.c_int(); it = C.c_int()
    im.im_icp(np.ascontiguousarray(src, np.float32), len(src), np.ascontiguousarray(tgt, np.float32), len(tgt), args["max_corr"],
              args["max_iter"], args["trans_eps"], args["fit_eps"], T, C.byref(fit), C.byref(conv), C.byref(it))
    return T.reshape(4, 4), fit.value, bool(conv.value), it.value


@pytest.mark.parametrize("seed", range(4))
def test_whole_loop_against_numpy(im, seed):
    rng = np.random.default_rng(100 + seed)
    # a small structured scene: three planes and a pole, the source seen from a frame off by a few degrees / decimetres
    n = 600
    pts = np.concatenate([
        np.c_[rng.uniform(-8, 8, n), rng.uniform(-8, 8, n), np.zeros(n)],
        np.c_[np.full(n, 6.0), rng.uniform(-8, 8, n), rng.uniform(0, 4, n)],
        np.c_[rng.uniform(-8, 8, n), np.full(n, -5.0), rng.uniform(0, 4, n)],
        np.c_[np.full(n // 4, -2.0) + rng.normal(0, 0.05, n // 4), np.full(n // 4, 1.0), rng.uniform(0, 5, n // 4)]])
    tgt = np.ones((len(pts), 4), np.float32); tgt[:, :3] = pts + rng.normal(0, 0.01, pts.shape)
    R0, t0 = rot([0.1, -0.2, 1.0], np.deg2rad(2.0 + seed)), np.array([0.3, -0.2, 0.05 * seed])
    pick = rng.permutation(len(pts))[:700]
    src = np.ones((700, 4), np.float32); src[:, :3] = (pts[pick] - t0) @ R0 + rng.normal(0, 0.01, (700, 3))
    kw = dict(max_corr=30.0 if seed < 2 else 1.5, max_iter=100 if seed != 3 else 4)
    T, fit, conv, it = host_icp(im, src, tgt, **kw)
    Tn, fitn, convn, itn = np_icp(src, tgt, kw["max_corr"], kw["max_iter"])
    assert (conv, it) == (convn, itn) and it >= 3
    np.testing.assert_allclose(T, Tn, rtol=0, atol=1e-9)
    assert abs(fit - fitn) <= 1e-9 * max(1.0, fitn)
    if seed != 3:
        assert np.abs(T[:3, :3] - R0).max() < 5e-3 and np.abs(T[:3, 3] - t0).max() < 0.05


def test_whole_loop_without_correspondences(im):
    rng = np.random.default_rng(7)
    tgt = np.ones((200, 4), np.float32); tgt[:, :3] = rng.uniform(-5, 5, (200, 3))
    far = tgt.copy(); far[:, 0] += 100.0
    T, fit, conv, it = host_icp(im, far, tgt, max_corr=5.0)
    assert not conv and it == 0 and np.array_equal(T, np.eye(4))
    T, fit, conv, it = host_icp(im, far[:0], tgt)
    assert not conv and it == 0 and np.array_equal(T, np.eye(4)) and fit == 0.0
