"""CPU tier for the packing of a batched scan-to-map step (s2m_batch_pack, liliom_b200/csrc/s2m_plan.h, compiled for the host
by tests/s2m_batch_host.cpp): which sessions share a cooperative launch of k_gn_batch and which keep their solo path."""
import ctypes as C
import itertools
import random

import pytest

import host_build

GN = 1
KIND = {(1, 0): 0, (2, 0): 1, (4, 0): 2, (8, 0): 3, (16, 0): 4, (16, 1): 5}


@pytest.fixture(scope="module")
def sb():
    L = host_build.load("s2m_batch_host", ["tests/s2m_batch_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall"],
                        deps=["liliom_b200/csrc/s2m_plan.h", "include/liliom.h"])
    ip = C.POINTER(C.c_int)
    L.sb_pack.argtypes = [C.c_int, ip, ip, C.c_int, C.c_int, ip, ip, ip, ip, ip, ip]
    L.sb_pack.restype = C.c_int
    L.sb_batch_max.restype = C.c_int
    sp = host_build.load("s2m_plan_host", ["tests/s2m_plan_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall"],
                         deps=["liliom_b200/csrc/s2m_plan.h", "include/liliom.h"])
    sp.sp_plan.argtypes = [C.c_int] * 12 + [C.POINTER(C.c_longlong)]
    sp.sp_plan.restype = None
    return L, sp


def _pack(L, plans, occ, sm, maxper):
    B = len(plans)
    flat = (C.c_int * max(4 * B, 1))(*[v for p in plans for v in p])
    o = (C.c_int * 6)(*occ)
    kind, grid, count, sess, solo = [(C.c_int * max(B, 1))() for _ in range(5)]
    n_solo = C.c_int()
    n = L.sb_pack(B, flat, o, sm, maxper, kind, grid, count, sess, solo, C.byref(n_solo))
    launches, k = [], 0
    for l in range(n):
        launches.append((kind[l], grid[l], list(sess[k:k + count[l]])))
        k += count[l]
    return launches, list(solo[:n_solo.value])


def _check(plans, occ, sm, maxper, launches, solo):
    seen = [s for _, _, ss in launches for s in ss]
    assert sorted(seen + solo) == list(range(len(plans)))          # every session exactly once
    for i in solo:
        lanes, tma, grid, pers = plans[i]
        assert not pers or grid > occ[KIND[(lanes, tma)]] * sm      # only non-persistent (or never resident) sessions go solo
    for kind, grid, ss in launches:
        assert 1 <= len(ss) <= maxper and ss == sorted(ss)
        assert all(plans[s][3] and KIND[(plans[s][0], plans[s][1])] == kind for s in ss)   # one instantiation per launch
        assert grid == sum(plans[s][2] for s in ss) <= occ[kind] * sm                   # co-resident


def test_batch_max(sb):
    assert sb[0].sb_batch_max() == 32


def test_headline_sessions_one_per_launch(sb):
    """At one block per SM the headline scan (88 blocks of 132) cannot share a cooperative launch with another."""
    L, _ = sb
    plans = [(16, 0, 88, 1)] * 4
    launches, solo = _pack(L, plans, [1] * 6, 132, 32)
    assert solo == [] and [ss for _, _, ss in launches] == [[0], [1], [2], [3]]


def test_small_sessions_share_launches(sb):
    L, _ = sb
    plans = [(16, 0, 10, 1)] * 40                    # 13 fit one launch by grid, 32 by the table
    launches, solo = _pack(L, plans, [1] * 6, 132, 32)
    assert solo == [] and [len(ss) for _, _, ss in launches] == [13, 13, 13, 1]
    launches, _ = _pack(L, plans, [4] * 6, 132, 32)       # with four resident blocks per SM the table is the limit
    assert [len(ss) for _, _, ss in launches] == [32, 8]
    _check(plans, [4] * 6, 132, 32, launches, [])


def test_mixed_kinds_and_solo(sb):
    L, _ = sb
    plans = [(16, 0, 40, 1), (8, 0, 97, 1), (1, 0, 264, 0), (16, 0, 60, 1), (16, 1, 30, 1), (8, 0, 20, 1), (2, 0, 118, 1), (16, 0, 88, 0)]
    occ = [1] * 6
    launches, solo = _pack(L, plans, occ, 132, 32)
    assert solo == [2, 7]
    assert [(k, ss) for k, _, ss in launches] == [(4, [0, 3]), (3, [1, 5]), (5, [4]), (1, [6])]
    _check(plans, occ, 132, 32, launches, solo)
    launches, solo = _pack(L, plans, [0, 1, 1, 1, 1, 1], 132, 32)    # an instantiation that cannot be resident at all
    _check(plans, [0, 1, 1, 1, 1, 1], 132, 32, launches, solo)


def test_random_invariants(sb):
    L, _ = sb
    rnd = random.Random(3)
    shapes = list(KIND)
    for _ in range(400):
        B = rnd.randint(1, 70)
        sm = rnd.choice((16, 84, 132))
        occ = [rnd.choice((1, 1, 2, 3)) for _ in range(6)]
        maxper = rnd.choice((1, 2, 5, 32))
        plans = []
        for _ in range(B):
            lanes, tma = rnd.choice(shapes)
            pers = rnd.random() < 0.8
            plans.append((lanes, tma, rnd.randint(1, sm if pers else 2 * sm), int(pers)))
        launches, solo = _pack(L, plans, occ, sm, maxper)
        _check(plans, occ, sm, maxper, launches, solo)


def test_solo_plan_unchanged_by_batching(sb):
    """The batch takes each session's solo plan as it is: packing only reads it, so the launch of a session has the grid and
    shape its solo call would have (the plans below are s2m_plan's own)."""
    L, sp = sb
    for n, n_last, dev in itertools.product((40, 200, 1400, 3100, 15000, 60000), (0, 1400), (0, 1)):
        out = (C.c_longlong * 8)()
        sp.sp_plan(n, n_last, dev, 132, GN, 10, 0, 1, 0, 0, 0, 0, out)
        n_est, lanes, rounds, per_task, grid, pers, tma, dyn = tuple(out)
        plans = [(lanes, tma, grid, pers)]
        launches, solo = _pack(L, plans, [1] * 6, 132, 32)
        if pers:
            assert launches == [(KIND[(lanes, tma)], grid, [0])] and solo == []
        else:
            assert launches == [] and solo == [0]
