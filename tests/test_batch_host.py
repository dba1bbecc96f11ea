"""CPU tier for the launches several sessions share (liliom_b200/csrc/batch.h, compiled for the host by tests/batch_host.cpp):
a stage's blocks per session, the lookup from a block of the shared grid to its session in the table's prefix offsets, and the
first-fit packing of cooperative launches."""
import ctypes as C
import random

import pytest

import host_build


@pytest.fixture(scope="module")
def ms():
    L = host_build.load("batch_host", ["tests/batch_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall"],
                        deps=["liliom_b200/csrc/batch.h"])
    ip = C.POINTER(C.c_int)
    L.bh_session_of.argtypes = [C.c_int, ip, C.c_int, ip]
    L.bh_session_of1.argtypes = [C.c_int, ip, C.c_int, ip]
    L.bh_pack.argtypes = [C.c_int, ip, ip, C.c_int, C.c_int, ip, ip, ip, ip, ip, ip]
    L.bh_pack.restype = C.c_int
    L.bh_batch_max.restype = C.c_int
    return L


def _walk(ms, blocks, b, one_entry=False):
    arr = (C.c_int * len(blocks))(*blocks)
    place = C.c_int()
    lookup = ms.bh_session_of1 if one_entry else ms.bh_session_of
    return lookup(len(blocks), arr, b, C.byref(place)), place.value


def _pack(ms, items, occ, sm, maxper):
    B = len(items)
    flat = (C.c_int * max(3 * B, 1))(*[v for it in items for v in it])
    o = (C.c_int * len(occ))(*occ)
    kind, grid, count, sess, solo = [(C.c_int * max(B, 1))() for _ in range(5)]
    n_solo = C.c_int()
    n = ms.bh_pack(B, flat, o, sm, maxper, kind, grid, count, sess, solo, C.byref(n_solo))
    launches, k = [], 0
    for l in range(n):
        launches.append((kind[l], grid[l], list(sess[k:k + count[l]])))
        k += count[l]
    return launches, list(solo[:n_solo.value])


def test_stage_blocks_cover_every_item_once(ms):
    for threads in (32, 128, 256):
        for items in (0, 1, threads - 1, threads, threads + 1, 5 * threads, 5 * threads + 7, (1 << 24) - 1):
            b = ms.bh_stage_blocks(items, threads)
            assert b * threads >= items and (b - 1) * threads < items, (items, threads, b)
    assert ms.bh_stage_blocks(0, 256) == 0              # an empty frame or map takes part in no launch of that stage
    assert ms.bh_stage_blocks(0 + 1, 256) == 1          # mark / heads run E + 1 threads: the scan sentinel of an empty entry array


def test_box_blocks_are_the_solo_grid(ms):
    for sm in (1, 108, 132):
        for n in (0, 1, 256, 257, 256 * 8 * sm - 1, 256 * 8 * sm, 256 * 8 * sm + 1, 10_000_000):
            want = min((n + 255) // 256, sm * 8)
            assert ms.bh_box_blocks(n, sm) == want, (n, sm)


def test_every_block_finds_its_session_and_place(ms):
    assert ms.bh_batch_max() == 32
    rng = random.Random(5)
    cases = [[1], [7], [1, 1], [3, 1, 5], [1] * 32, [2, 0, 3], [0, 4], [4, 0], [0, 0, 2, 0, 1]]
    cases += [[rng.choice((0, 1, 1, 2, 9, 40)) for _ in range(rng.randint(1, 32))] for _ in range(200)]
    for blocks in cases:
        if sum(blocks) == 0:
            continue
        want = [(s, p) for s, n in enumerate(blocks) for p in range(n)]
        for one_entry in ((False, True) if len(blocks) == 1 else (False,)):    # a one-session launch carries a one-entry table
            got = [_walk(ms, blocks, b, one_entry) for b in range(sum(blocks))]
            assert got == want, (blocks, one_entry)


def test_one_session_owns_the_whole_grid(ms):
    for one_entry in (False, True):
        for b in range(9):
            assert _walk(ms, [9], b, one_entry) == (0, b)


def test_horizon_sessions_four_per_launch(ms):
    """The Horizon batch: one kind, 83 blocks per session.  At k_hz_batch's bound of three blocks per SM on 132 SMs, four
    sessions share a launch (4 * 83 = 332 <= 396 < 5 * 83); at two blocks per SM, three."""
    items = [(83, 0, 1)] * 9
    launches, solo = _pack(ms, items, [3], 132, 32)
    assert solo == [] and launches == [(0, 332, [0, 1, 2, 3]), (0, 332, [4, 5, 6, 7]), (0, 83, [8])]
    launches, solo = _pack(ms, items, [2], 132, 32)
    assert solo == [] and [ss for _, _, ss in launches] == [[0, 1, 2], [3, 4, 5], [6, 7, 8]]
    launches, solo = _pack(ms, items[:2], [0], 132, 32)          # not resident at all: every session on its solo path
    assert launches == [] and solo == [0, 1]
