"""ctypes loader for tests/rot_time_oracle.cpp, the CPU oracle of the ROT extractor with relTime from the driver's per-point
time field (LILIOM_TIME_FIELD) — TEST INFRASTRUCTURE (the product never imports this).  Built on first use into build/ with the
oracle library's flags and linked against oracle/liboracle.so (its VoxelGrid)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "rot_time_oracle.cpp")
SO = os.path.join(ROOT, "build", "librot_time_oracle.so")
PT32 = oracle_lib.PT32

_lib = None


def lib():
    global _lib
    if _lib is None:
        oracle_lib.build()
        deps = [SRC, oracle_lib.SO, os.path.join(oracle_lib.ORACLE_DIR, "oracle_math.h"), os.path.join(oracle_lib.ORACLE_DIR, "oracle_api.h")]
        if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(p) for p in deps):
            os.makedirs(os.path.dirname(SO), exist_ok=True)
            gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
            tmp = f"{SO}.{os.getpid()}"
            subprocess.run([gxx, "-O3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-Wextra", "-shared", "-I", oracle_lib.ORACLE_DIR,
                            "-o", tmp, SRC, oracle_lib.SO, f"-Wl,-rpath,{oracle_lib.ORACLE_DIR}"], check=True)
            os.replace(tmp, SO)
        oracle_lib.lib()                      # liboracle.so loaded first (its VoxelGrid)
        L = C.CDLL(SO)
        vp, dp, ip = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)
        L.orc_extract_rot_timed.argtypes = [vp, vp, vp, C.c_int, dp, dp, C.c_int, C.c_int, vp, ip, vp, ip, vp, ip, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _d(a):
    return np.ascontiguousarray(a, np.float64).ctypes.data_as(C.POINTER(C.c_double))


def extract_rot_timed(pts, rings, times, q_imu, q_lb=(1.0, 0, 0, 0), line_num=128, ds_rate=4):
    """(rc, surf, edge, cutted, labels, curvatures) with optional rings (None: the elevation tables) and optional per-point times
    (None: the azimuth rule; else relTime over the times of the surviving points, non-finite times dropped)."""
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
