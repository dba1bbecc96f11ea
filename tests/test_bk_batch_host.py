"""CPU tier for the layout of the batched backend window calls (liliom_b200/csrc/bk_batch.h, compiled for the host by
tests/bk_batch_host.cpp): every session's range of a concatenated table, each block segment's place in it, and the launches that
cover the sessions past 32."""
import ctypes as C
import random

import pytest

import host_build


@pytest.fixture(scope="module")
def bb():
    L = host_build.load("bk_batch_host", ["tests/bk_batch_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall"],
                        deps=["liliom_b200/csrc/bk_batch.h", "liliom_b200/csrc/batch.h", "liliom_b200/csrc/bk_window.h"])
    ip = C.POINTER(C.c_int)
    L.bb_offsets.argtypes = [C.c_int, ip, ip]
    L.bb_offsets.restype = None
    L.bb_segment.argtypes = [C.c_int, ip, C.c_int, C.c_int, C.c_int]
    L.bb_launches.argtypes = [C.c_int, ip, ip]
    L.bb_region.argtypes = [C.c_longlong, C.c_longlong]
    L.bb_region.restype = C.c_longlong
    return L


def _arr(v):
    return (C.c_int * max(len(v), 1))(*v)


def _offsets(bb, count):
    off = (C.c_int * (len(count) + 1))()
    bb.bb_offsets(len(count), _arr(count), off)
    return list(off)


def _launches(bb, count):
    out = (C.c_int * (4 * (len(count) // 32 + 2)))()
    n = bb.bb_launches(len(count), _arr(count), out)
    return [tuple(out[4 * l:4 * l + 4]) for l in range(n)]


def test_constants(bb):
    assert bb.bb_batch_max() == 32 and bb.bb_win_max() == 16 and bb.bb_cnt_ints() == 32


def test_offsets_are_the_prefix_sums(bb):
    rng = random.Random(3)
    for count in ([], [0], [2], [2, 32, 0, 6], [rng.randint(0, 32) for _ in range(70)]):
        off = _offsets(bb, count)
        assert off[0] == 0 and len(off) == len(count) + 1
        assert all(off[m + 1] - off[m] == count[m] for m in range(len(count)))


def test_every_segment_has_one_place(bb):
    """Session m's segment 2 i + kind (keyframe i, 0 edge / 1 surf): the places of all sessions tile the table exactly once, in
    session order, as the solo call orders its own 2 k segments."""
    rng = random.Random(7)
    for k in ([1], [16], [3, 1, 16, 2], [rng.randint(1, 16) for _ in range(34)]):
        ka = _arr(k)
        places = [bb.bb_segment(len(k), ka, m, i, kind) for m in range(len(k)) for i in range(k[m]) for kind in (0, 1)]
        assert places == list(range(2 * sum(k)))


@pytest.mark.parametrize("B", [1, 2, 8, 31, 32, 33, 34, 64, 65, 100])
def test_launches_chunk_at_32_sessions(bb, B):
    rng = random.Random(B)
    count = [2 * rng.randint(1, 16) for _ in range(B)]
    off = _offsets(bb, count)
    L = _launches(bb, count)
    assert len(L) == (B + 31) // 32
    first = 0
    for f, n, item0, items in L:
        assert f == first and 1 <= n <= 32 and item0 == off[f] and items == off[f + n] - off[f]
        assert items <= 32 * 32          # at most 1024 segments: the launch's grid.y
        first += n
    assert first == B
    assert _launches(bb, []) == []


def test_regions_are_aligned_and_large_enough(bb):
    for n in (0, 1, 2, 31, 32, 1000):
        for size in (1, 4, 8, 29 * 8, 1176):
            r = bb.bb_region(n, size)
            assert r % 256 == 0 and r >= n * size and r - n * size < 256
