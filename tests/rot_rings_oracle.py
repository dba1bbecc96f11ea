"""ctypes loader for tests/rot_rings_oracle.cpp, the CPU oracle of the ROT extractor with the driver's ring ids (LILIOM_RING_FIELD)
— TEST INFRASTRUCTURE (the product never imports this).  Built on first use into build/ with the oracle library's flags and
linked against oracle/liboracle.so (its VoxelGrid)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "rot_rings_oracle.cpp")
SO = os.path.join(ROOT, "build", "librot_rings_oracle.so")
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
        L.orc_extract_rot_rings.argtypes = [vp, vp, C.c_int, dp, dp, C.c_int, C.c_int, vp, ip, vp, ip, vp, ip, vp, vp]
        L.orc_extract_rot_tables.argtypes = [vp, C.c_int, dp, dp, C.c_int, C.c_int, vp, ip, vp, ip, vp, ip, vp, vp]
        L.orc_rot_scan_ids.argtypes = [vp, C.c_int, C.c_int, vp]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _d(a):
    return np.ascontiguousarray(a, np.float64).ctypes.data_as(C.POINTER(C.c_double))


def _run(fn, pts, args):
    pts = np.ascontiguousarray(pts, dtype=PT32); n = len(pts)
    surf = np.zeros(max(n, 1), PT32); edge = np.zeros(max(n, 1), PT32); cut = np.zeros(max(n, 1), PT32)
    lab = np.zeros(max(n, 1), np.int32); cur = np.zeros(max(n, 1), np.float32)
    ns, ne, nc = C.c_int(), C.c_int(), C.c_int()
    rc = fn(*args(pts, n), _p(surf), C.byref(ns), _p(edge), C.byref(ne), _p(cut), C.byref(nc), _p(lab), _p(cur))
    return rc, surf[:ns.value], edge[:ne.value], cut[:nc.value], lab[:nc.value], cur[:nc.value]


def extract_rot_rings(pts, rings, q_imu, q_lb=(1.0, 0, 0, 0), line_num=128, ds_rate=4):
    """(rc, surf, edge, cutted, labels, curvatures) with scanID = rings[i] (kept iff 0 <= ring < line_num)."""
    q, ql = np.asarray(q_imu, np.float64), np.asarray(q_lb, np.float64)
    r = np.ascontiguousarray(rings, np.int32)
    assert len(r) == len(pts)
    return _run(lib().orc_extract_rot_rings, pts, lambda p, n: (_p(p), _p(r), n, _d(q), _d(ql), line_num, ds_rate))


def extract_rot_tables(pts, q_imu, q_lb=(1.0, 0, 0, 0), line_num=64, ds_rate=4):
    """The same function with the elevation tables (must equal oracle_lib.extract_rot)."""
    q, ql = np.asarray(q_imu, np.float64), np.asarray(q_lb, np.float64)
    return _run(lib().orc_extract_rot_tables, pts, lambda p, n: (_p(p), n, _d(q), _d(ql), line_num, ds_rate))


def rot_scan_ids(pts, line_num=64) -> np.ndarray:
    """The elevation tables' verdict per input point: its scanID, or -1 where the point is dropped (removed or a table miss)."""
    pts = np.ascontiguousarray(pts, dtype=PT32)
    ids = np.zeros(max(len(pts), 1), np.int32)
    assert lib().orc_rot_scan_ids(_p(pts), len(pts), line_num, _p(ids)) == 0
    return ids[:len(pts)]
