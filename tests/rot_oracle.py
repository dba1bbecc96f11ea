"""ctypes loader for tests/rot_oracle.cpp, the CPU oracle of the ROT extractor with the driver's ring ids (LILIOM_RING_FIELD)
and relTime from the driver's per-point time field (LILIOM_TIME_FIELD) — TEST INFRASTRUCTURE (the product never imports this).
Built on first use into build/ with the oracle library's flags and linked against oracle/liboracle.so (its VoxelGrid)."""
from __future__ import annotations

import ctypes as C

import numpy as np

import host_build
import oracle_lib

PT32 = oracle_lib.PT32

_lib = None


def lib():
    global _lib
    if _lib is None:
        oracle_lib.build()
        d = oracle_lib.ORACLE_DIR
        oracle_lib.lib()                      # liboracle.so loaded first (its VoxelGrid)
        L = host_build.load("rot_oracle", ["tests/rot_oracle.cpp"],
                            ["-O3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-Wextra", "-I", d],
                            deps=[oracle_lib.SO, f"{d}/oracle_math.h", f"{d}/oracle_api.h"], link=[oracle_lib.SO, f"-Wl,-rpath,{d}"])
        vp, dp, ip = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)
        L.orc_extract_rot_timed.argtypes = [vp, vp, vp, C.c_int, dp, dp, C.c_int, C.c_int, vp, ip, vp, ip, vp, ip, vp, vp]
        L.orc_rot_scan_ids.argtypes = [vp, C.c_int, C.c_int, vp]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _d(a):
    return np.ascontiguousarray(a, np.float64).ctypes.data_as(C.POINTER(C.c_double))


def extract_rot(pts, q_imu, q_lb, line_num, ds_rate, rings=None, times=None):
    """(rc, surf, edge, cutted, labels, curvatures).  rings: None = scanID from the elevation tables (line_num 16 / 32 / 64), else
    scanID = rings[i], kept iff 0 <= ring < line_num (1..128).  times: None = relTime from the azimuth rule, else relTime over the
    times of the surviving points, non-finite times dropped."""
    pts = np.ascontiguousarray(pts, dtype=PT32); n = len(pts)
    q, ql = np.asarray(q_imu, np.float64), np.asarray(q_lb, np.float64)
    r = None if rings is None else np.ascontiguousarray(rings, np.int32)
    t = None if times is None else np.ascontiguousarray(times, np.float64)
    assert (r is None or len(r) == n) and (t is None or len(t) == n)
    surf = np.zeros(max(n, 1), PT32); edge = np.zeros(max(n, 1), PT32); cut = np.zeros(max(n, 1), PT32)
    lab = np.zeros(max(n, 1), np.int32); cur = np.zeros(max(n, 1), np.float32)
    ns, ne, nc = C.c_int(), C.c_int(), C.c_int()
    rc = lib().orc_extract_rot_timed(_p(pts), _p(r), _p(t), n, _d(q), _d(ql), line_num, ds_rate, _p(surf), C.byref(ns), _p(edge),
                                     C.byref(ne), _p(cut), C.byref(nc), _p(lab), _p(cur))
    return rc, surf[:ns.value], edge[:ne.value], cut[:nc.value], lab[:nc.value], cur[:nc.value]


def scan_ids(pts, line_num) -> np.ndarray:
    """The elevation tables' verdict per input point: its scanID, or -1 where the point is dropped (removed or a table miss)."""
    pts = np.ascontiguousarray(pts, dtype=PT32)
    ids = np.zeros(max(len(pts), 1), np.int32)
    assert lib().orc_rot_scan_ids(_p(pts), len(pts), line_num, _p(ids)) == 0
    return ids[:len(pts)]
