"""CPU tier for the ownership of the context's device buffers: liliom_b200/csrc/ctx.cuh compiled for the host (tests/ctx_host.cpp)
and linked against the CUDA runtime.  DevBuf, MapIndex and Frame are move-only with nothrow moves (static_asserts), a moved-from
DevBuf is empty, an empty one is destroyed without a CUDA call, and the map FIFO's recycling of the popped frame's buffer frees
nothing."""
import ctypes as C
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "build", "libctx_host.so")
CUDA = "/usr/local/cuda"


@pytest.fixture(scope="module")
def ctxh():
    src = os.path.join(ROOT, "tests", "ctx_host.cpp")
    hdrs = [os.path.join(ROOT, "liliom_b200", "csrc", h) for h in ("ctx.cuh", "vg_box.h")] + [os.path.join(ROOT, "include", "liliom.h")]
    lib64 = os.path.join(CUDA, "lib64")
    if not os.path.exists(os.path.join(CUDA, "include", "cuda_runtime.h")):
        pytest.skip("CUDA headers not found")
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(p) for p in [src] + hdrs):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-self-move", "-I", os.path.join(CUDA, "include"),
                        "-shared", "-o", SO, src, "-L", lib64, "-Wl,-rpath," + lib64, "-lcudart"], check=True)
    L = C.CDLL(SO)
    L.ctx_host_run.restype = C.c_int
    return L


def test_device_buffers_are_owned_and_moved_never_copied(ctxh):
    assert ctxh.ctx_host_run() == 0
