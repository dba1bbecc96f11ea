"""CPU tier for the sliding-window bookkeeping of the backend LiDAR rows: liliom_b200/csrc/bk_window.h compiled for the host
(tests/bk_window_host.cpp).  The query -> keyframe lookup (empty keyframes included) and the three weight formulas of the
reference (L/src/BackendFusion.cpp:1581, R/src/BackendFusion.cpp:843, :861) against NumPy restatements at the reference's widths."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "build", "libbk_window_host.so")


@pytest.fixture(scope="module")
def bw():
    src = os.path.join(ROOT, "tests", "bk_window_host.cpp")
    deps = [src, os.path.join(ROOT, "liliom_b200", "csrc", "bk_window.h")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(p) for p in deps):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-ffp-contract=off", "-shared", "-o", SO, src], check=True)
    L = C.CDLL(SO)
    L.bw_find.argtypes = [C.POINTER(C.c_longlong), C.c_int, C.c_longlong]
    L.bw_find.restype = C.c_int
    L.bw_edge_weight.argtypes = [C.c_int, C.c_double, C.c_int]
    L.bw_edge_weight.restype = C.c_double
    L.bw_surf_score.argtypes = [C.c_int, C.c_double, C.c_int]
    L.bw_surf_score.restype = C.c_double
    return L


@pytest.mark.parametrize("counts", [[5], [0], [3, 0, 4], [0, 0, 7, 0], [1] * 16, [0, 2, 0, 2, 0], [1000, 1, 0, 65]])
def test_query_to_keyframe_lookup(bw, counts):
    start = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    sp = start.ctypes.data_as(C.POINTER(C.c_longlong))
    k = len(counts)
    owner = np.repeat(np.arange(k), counts)          # the keyframe each concatenated query belongs to
    for qi in range(int(start[-1])):
        assert bw.bw_find(sp, k, qi) == owner[qi], (counts, qi)
    for qi in (-1, int(start[-1]), int(start[-1]) + 5):
        assert bw.bw_find(sp, k, qi) == -1
    assert bw.bw_find(sp, 0, 0) == -1


def test_weights_at_the_reference_widths(bw):
    rng = np.random.default_rng(3)
    for lc in (1.0, 7.5, 15.0, 20.0, 0.1, 1.0 / 3.0, 123.456789):
        # L:1581: pt.intensity = lidar_const (a float field), handed to the factor as a double
        assert bw.bw_edge_weight(0, lc, 17) == float(np.float32(lc))
        for n in (1, 3, 7, 97, 1000, 4093):
            # R:843: intensity * 200 / vec_edge_res_cnt -> float * int, float / int: all float
            want = float(np.float32(np.float32(np.float32(lc) * np.float32(200)) / np.float32(n)))
            assert bw.bw_edge_weight(1, lc, n) == want, (lc, n)
    for score in list(rng.uniform(0.0, 30.0, 50)) + [0.0, 1e-300, 7.5 * 0.731]:
        assert bw.bw_surf_score(0, score, 9) == score
        for n in (1, 3, 51, 1499):
            # R:861: vec_surf_scores[idVec][i] * 1000 / vec_surf_res_cnt[idVec] in double
            assert bw.bw_surf_score(1, score, n) == (np.float64(score) * 1000.0) / np.float64(n)
