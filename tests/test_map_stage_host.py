"""CPU tier for the block geometry of the batched map update (liliom_b200/csrc/map_stage.h, compiled for the host by
tests/map_stage_host.cpp): a stage's blocks per session, and the walk from a block of the shared grid to its session."""
import ctypes as C
import random

import pytest

import host_build


@pytest.fixture(scope="module")
def ms():
    L = host_build.load("map_stage_host", ["tests/map_stage_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall"],
                        deps=["liliom_b200/csrc/map_stage.h"])
    L.ms_session_of.argtypes = [C.c_int, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int)]
    return L


def _walk(ms, blocks, b):
    arr = (C.c_int * len(blocks))(*blocks)
    place = C.c_int()
    return ms.ms_session_of(len(blocks), arr, b, C.byref(place)), place.value


def test_stage_blocks_cover_every_item_once(ms):
    for threads in (32, 128, 256):
        for items in (0, 1, threads - 1, threads, threads + 1, 5 * threads, 5 * threads + 7, (1 << 24) - 1):
            b = ms.ms_stage_blocks(items, threads)
            assert b * threads >= items and (b - 1) * threads < items, (items, threads, b)
    assert ms.ms_stage_blocks(0, 256) == 0              # an empty frame or map takes part in no launch of that stage
    assert ms.ms_stage_blocks(0 + 1, 256) == 1          # mark / heads run E + 1 threads: the scan sentinel of an empty entry array


def test_box_blocks_are_the_solo_grid(ms):
    for sm in (1, 108, 132):
        for n in (0, 1, 256, 257, 256 * 8 * sm - 1, 256 * 8 * sm, 256 * 8 * sm + 1, 10_000_000):
            want = min((n + 255) // 256, sm * 8)
            assert ms.ms_box_blocks(n, sm) == want, (n, sm)


def test_every_block_finds_its_session_and_place(ms):
    rng = random.Random(5)
    cases = [[1], [7], [1, 1], [3, 1, 5], [1] * 32, [2, 0, 3], [0, 4], [4, 0], [0, 0, 2, 0, 1]]
    cases += [[rng.choice((0, 1, 1, 2, 9, 40)) for _ in range(rng.randint(1, 32))] for _ in range(200)]
    for blocks in cases:
        if sum(blocks) == 0:
            continue
        want = [(s, p) for s, n in enumerate(blocks) for p in range(n)]
        got = [_walk(ms, blocks, b) for b in range(sum(blocks))]
        assert got == want, blocks


def test_one_session_owns_the_whole_grid(ms):
    for b in range(9):
        assert _walk(ms, [9], b) == (0, b)
