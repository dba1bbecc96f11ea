"""Builds the host-compiled test libraries (the CPU builds of the library's headers and the CPU oracles beside the tests) —
TEST INFRASTRUCTURE (the product never imports this)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load(name, srcs, flags, deps=(), link=()):
    """build/lib<name>.so compiled by g++ from `srcs` with `flags` (then `link`: libraries, rpath), rebuilt when any source or
    any of `deps` (the headers and libraries it compiles against) is newer; paths are relative to the repository root.  Written
    through a temporary file and os.replace, so that a test process running beside this one never loads a half-written library.
    Returns the loaded ctypes.CDLL."""
    srcs = [os.path.join(ROOT, p) for p in srcs]
    so = os.path.join(ROOT, "build", f"lib{name}.so")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(os.path.join(ROOT, p)) for p in [*srcs, *deps]):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        tmp = f"{so}.{os.getpid()}"
        subprocess.run([gxx, *flags, "-shared", "-o", tmp, *srcs, *link], check=True)
        os.replace(tmp, so)
    return C.CDLL(so)
