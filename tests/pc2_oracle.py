"""ctypes loader for tests/pc2_oracle.cpp, the CPU restatement of pcl::fromROSMsg(PointCloud2 -> PointXYZI) — TEST
INFRASTRUCTURE (the product never imports this).  Built on first use into build/ like the other host harnesses."""
from __future__ import annotations

import ctypes as C

import numpy as np

import host_build

PT32 = np.dtype([("x", "f4"), ("y", "f4"), ("z", "f4"), ("w", "f4"), ("intensity", "f4"), ("p0", "f4"), ("p1", "f4"), ("p2", "f4")])


class Field(C.Structure):
    _fields_ = [("name", C.c_char * 16), ("offset", C.c_uint), ("datatype", C.c_ubyte), ("count", C.c_uint)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = host_build.load("pc2_oracle", ["tests/pc2_oracle.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall", "-Wextra"])
        L.orc_pc2_to_pt32.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.POINTER(Field), C.c_int, C.c_void_p]
        L.orc_pc2_to_pt32.restype = C.c_int
        _lib = L
    return _lib


def pc2_to_pt32(msg) -> np.ndarray:
    """msg: liliom_b200.PC2 (payload bytes + header + field tuples).  Returns the decoded PointXYZI cloud."""
    f = (Field * max(len(msg.fields), 1))()
    for i, (name, off, dt, cnt) in enumerate(msg.fields):
        f[i].name = name.encode()[:15]; f[i].offset = off; f[i].datatype = dt; f[i].count = cnt
    n = msg.width * msg.height
    out = np.zeros(max(n, 1), PT32)
    data = np.ascontiguousarray(msg.data)
    got = lib().orc_pc2_to_pt32(data.ctypes.data_as(C.c_void_p), msg.height, msg.width, msg.point_step, msg.row_step, f, len(msg.fields),
                                out.ctypes.data_as(C.c_void_p))
    assert got == n, got
    return out[:n]
