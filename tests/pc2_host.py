"""ctypes loader for tests/pc2_host.cpp, the host build of liliom_b200/csrc/pc2_fields.h — TEST INFRASTRUCTURE (the product never
imports this).  Shared by the CPU tests of the point fields, the `ring` field and the time field."""
from __future__ import annotations

import ctypes as C

import numpy as np

import host_build

_lib = None


def lib():
    global _lib
    if _lib is None:
        from liliom_b200 import _lib as abi
        L = host_build.load("pc2_host", ["tests/pc2_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall", "-Wextra"],
                            deps=["liliom_b200/csrc/pc2_fields.h", "include/liliom.h"])
        msg = C.POINTER(abi.Pc2Msg)
        L.ph_match.argtypes = [msg, C.POINTER(C.c_int)]
        L.ph_match.restype = C.c_int
        L.ph_match_sources.argtypes = [msg, C.c_int, C.c_char_p, C.POINTER(C.c_int)]
        L.ph_match_sources.restype = C.c_int
        L.ph_decode_rings.argtypes = [msg, C.c_void_p]
        L.ph_decode_times.argtypes = [msg, C.c_char_p, C.c_void_p]
        L.ph_rel_times.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_void_p]
        L.ph_rel_times.restype = None
        _lib = L
    return _lib


def match_sources(ph, fields, point_step, want_ring=False, time_name=None, width=10):
    """(rc, {src x, y, z, intensity, n, ring_src, ring_bytes, time_src, time_type}) of ph_match_sources on a one-row message with
    these fields and a zero payload; the output starts at -7 so that an untouched output is visible."""
    from liliom_b200 import PC2
    msg = PC2(np.zeros(max(width * point_step, 1), np.uint8), 1, width, point_step, width * point_step, fields)
    m, _keep = msg.c_msg()
    out = (C.c_int * 9)(*([-7] * 9))
    rc = ph.ph_match_sources(C.byref(m), int(want_ring), None if time_name is None else time_name.encode(), out)
    return rc, tuple(out)
