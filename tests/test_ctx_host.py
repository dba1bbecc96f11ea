"""CPU tier for the ownership of the context's device buffers: liliom_b200/csrc/ctx.cuh compiled for the host (tests/ctx_host.cpp)
and linked against the CUDA runtime.  DevBuf, MapIndex and Frame are move-only with nothrow moves (static_asserts), a moved-from
DevBuf is empty, an empty one is destroyed without a CUDA call, and the map FIFO's recycling of the popped frame's buffer frees
nothing."""
import ctypes as C
import os

import pytest

import host_build

CUDA = "/usr/local/cuda"


@pytest.fixture(scope="module")
def ctxh():
    lib64 = os.path.join(CUDA, "lib64")
    if not os.path.exists(os.path.join(CUDA, "include", "cuda_runtime.h")):
        pytest.skip("CUDA headers not found")
    L = host_build.load("ctx_host", ["tests/ctx_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-self-move", "-I", os.path.join(CUDA, "include")],
                        deps=["liliom_b200/csrc/ctx.cuh", "liliom_b200/csrc/batch.h", "liliom_b200/csrc/vg_box.h", "include/liliom.h"],
                        link=["-L", lib64, "-Wl,-rpath," + lib64, "-lcudart"])
    L.ctx_host_run.restype = C.c_int
    return L


def test_device_buffers_are_owned_and_moved_never_copied(ctxh):
    assert ctxh.ctx_host_run() == 0
