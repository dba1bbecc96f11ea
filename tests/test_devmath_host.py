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


def test_colpiv_qr_device_copy_equals_oracle_copy(dm, oracle):
    rng = np.random.default_rng(1)
    for _ in range(200):
        A = rng.uniform(-50, 50, (5, 3)); b = -np.ones(5)
        x = np.zeros(3)
        dm.dm_colpiv_qr(_d(np.ascontiguousarray(A.reshape(-1))), _d(b), _d(x))
        np.testing.assert_allclose(x, oracle.colpiv_qr_solve(A, b), rtol=1e-12, atol=1e-14)


def test_eigen_sym3_device_copy_equals_oracle_copy(dm, oracle):
    rng = np.random.default_rng(2)
    for k in range(300):
        B = rng.normal(size=(3, 3)) * 10.0 ** rng.integers(-3, 3)
        A = B @ B.T
        a = np.array([A[0, 0], A[1, 0], A[2, 0], A[1, 1], A[2, 1], A[2, 2]])
        ev = np.zeros(3); vec = np.zeros(9)
        dm.dm_eigen_sym3(_d(a), _d(ev), _d(vec))
        ev_o, vec_o = oracle.eigen_sym3(A)
        # two copies of the same algorithm (Eigen's tridiagonal QL): identical eigenvalues, eigenvectors up to sign
        np.testing.assert_allclose(ev, ev_o, rtol=1e-13, atol=1e-300)
        V = vec.reshape(3, 3)
        for c in range(3):
            assert min(np.abs(V[:, c] - vec_o[:, c]).max(), np.abs(V[:, c] + vec_o[:, c]).max()) < 1e-9
        np.testing.assert_allclose(ev, np.linalg.eigvalsh(A), rtol=1e-10, atol=1e-12 * np.abs(A).max())


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
