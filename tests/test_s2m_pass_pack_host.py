"""CPU tier for the launches of a batched scan-to-map step with per-session iteration counts (s2m_pass_pack and s2m_gn_groups,
liliom_b200/csrc/s2m_plan.h, compiled for the host by tests/s2m_pass_host.cpp): which sessions share each Ceres-mode pass's
k_knn_plane_batch and k_lm_solve_batch launches, and how GN-mode sessions of different counts are grouped."""
import ctypes as C
import random

import pytest

import host_build
from test_s2m_batch_host import _pack

LANES = (1, 2, 4, 8, 16)


@pytest.fixture(scope="module")
def libs():
    flags = ["-O2", "-std=c++17", "-fPIC", "-Wall"]
    deps = ["liliom_b200/csrc/s2m_plan.h", "include/liliom.h"]
    sp = host_build.load("s2m_pass_host", ["tests/s2m_pass_host.cpp"], flags, deps=deps)
    ip = C.POINTER(C.c_int)
    sp.sp_pass_pack.argtypes = [C.c_int, ip, ip, C.c_int, ip, C.c_int]
    sp.sp_pass_pack.restype = C.c_int
    sp.sp_gn_groups.argtypes = [C.c_int, ip, ip, ip, C.c_int, C.c_int, ip, C.c_int]
    sp.sp_gn_groups.restype = C.c_int
    sb = host_build.load("s2m_batch_host", ["tests/s2m_batch_host.cpp"], flags, deps=deps)
    sb.sb_pack.argtypes = [C.c_int, ip, ip, C.c_int, C.c_int, ip, ip, ip, ip, ip, ip]
    sb.sb_pack.restype = C.c_int
    return sp, sb


def _ints(v):
    return (C.c_int * max(len(v), 1))(*v)


class _Stream:
    def __init__(self, buf, n):
        self.v, self.k = list(buf[:n]), 0

    def get(self):
        self.k += 1
        return self.v[self.k - 1]

    def list(self):
        n = self.get()
        return [self.get() for _ in range(n)]


def _pass_pack(sp, plans, iters, maxper):
    cap = 64 + 8 * len(plans) * (max(iters, default=0) + 1) * 2
    out = (C.c_int * cap)()
    n = sp.sp_pass_pack(len(plans), _ints([v for p in plans for v in p]), _ints(iters), maxper, out, cap)
    assert n >= 0
    s = _Stream(out, n)
    passes = []
    for _ in range(s.get()):
        knn = [(s.get(), s.list()) for _ in range(s.get())]
        lm = [s.list() for _ in range(s.get())]
        passes.append((knn, lm))
    return passes


def _gn_groups(sp, plans, iters, occ, sm, maxper):
    cap = 64 + 16 * len(plans)
    out = (C.c_int * cap)()
    n = sp.sp_gn_groups(len(plans), _ints([v for p in plans for v in p]), _ints(iters), _ints(occ), sm, maxper, out, cap)
    assert n >= 0
    s = _Stream(out, n)
    groups = []
    for _ in range(s.get()):
        it = s.get()
        launches = [(s.get(), s.get(), s.list()) for _ in range(s.get())]
        groups.append((it, launches, s.list()))
    return groups


def _check_passes(plans, iters, maxper, passes):
    assert len(passes) == max(iters, default=0)
    for it, (knn, lm) in enumerate(passes):
        live = [j for j in range(len(plans)) if iters[j] > it]
        seen = [s for _, ss in knn for s in ss]
        assert sorted(seen) == live                                  # every iterating session in exactly one knn launch
        assert sorted(s for ss in lm for s in ss) == live            # ... and in the pass's LM launches, once
        assert [s for ss in lm for s in ss] == live                  # LM launches in call order
        for lanes, ss in knn:
            assert 1 <= len(ss) <= maxper and ss == sorted(ss)       # at most max_per_launch, in call order
            assert all(plans[s][0] == lanes for s in ss)             # one lane count per launch
        for ss in lm:
            assert 1 <= len(ss) <= maxper
        order = []                                                   # lane groups in the order of their first session
        for j in live:
            if plans[j][0] not in order:
                order.append(plans[j][0])
        assert [l for l, _ in knn] == sorted((l for l, _ in knn), key=order.index)


def test_reference_counts(libs):
    """The reference's counts in one call: 8 outer iterations for a session without two saved poses, then scan_match_cnt."""
    sp, _ = libs
    plans = [(16, 0, 88, 0), (8, 0, 97, 0), (1, 0, 264, 0), (16, 0, 40, 0)]
    iters = [8, 1, 2, 0]
    passes = _pass_pack(sp, plans, iters, 32)
    _check_passes(plans, iters, 32, passes)
    assert passes[0] == ([(16, [0]), (8, [1]), (1, [2])], [[0, 1, 2]])
    assert passes[1] == ([(16, [0]), (1, [2])], [[0, 2]])
    assert all(p == ([(16, [0])], [[0]]) for p in passes[2:])


def test_no_iterations(libs):
    sp, _ = libs
    assert _pass_pack(sp, [(16, 0, 10, 0)] * 3, [0, 0, 0], 32) == []


def test_more_sessions_than_one_table(libs):
    sp, _ = libs
    plans = [(16, 0, 5, 0)] * 40 + [(8, 0, 12, 0)] * 3
    iters = [2] * 43
    passes = _pass_pack(sp, plans, iters, 32)
    _check_passes(plans, iters, 32, passes)
    for knn, lm in passes:
        assert [(l, len(ss)) for l, ss in knn] == [(16, 32), (16, 8), (8, 3)]
        assert [len(ss) for ss in lm] == [32, 11]


def test_random_pass_invariants(libs):
    sp, _ = libs
    rnd = random.Random(7)
    for _ in range(300):
        B = rnd.randint(1, 80)
        maxper = rnd.choice((1, 3, 32))
        plans = [(rnd.choice(LANES), 0, rnd.randint(1, 264), 0) for _ in range(B)]
        iters = [rnd.choice((0, 1, 2, 8, rnd.randint(0, 12))) for _ in range(B)]
        _check_passes(plans, iters, maxper, _pass_pack(sp, plans, iters, maxper))


def test_gn_groups_equal_counts_is_one_pack(libs):
    """With one count for every session the grouping is s2m_batch_pack's output, unchanged."""
    sp, sb = libs
    rnd = random.Random(5)
    shapes = [(1, 0), (2, 0), (4, 0), (8, 0), (16, 0), (16, 1)]
    for _ in range(200):
        B = rnd.randint(1, 60)
        sm = rnd.choice((16, 132))
        occ = [rnd.choice((0, 1, 2)) for _ in range(6)]
        maxper = rnd.choice((1, 4, 32))
        plans = []
        for _ in range(B):
            lanes, tma = rnd.choice(shapes)
            pers = rnd.random() < 0.8
            plans.append((lanes, tma, rnd.randint(1, sm if pers else 2 * sm), int(pers)))
        it = rnd.choice((1, 10))
        groups = _gn_groups(sp, plans, [it] * B, occ, sm, maxper)
        launches, solo = _pack(sb, plans, occ, sm, maxper)
        assert groups == [(it, launches, solo)]


def test_gn_groups_by_count(libs):
    sp, sb = libs
    rnd = random.Random(9)
    for _ in range(200):
        B = rnd.randint(1, 50)
        sm, occ, maxper = 132, [1] * 6, rnd.choice((2, 32))
        plans = [(rnd.choice((8, 16)), 0, rnd.randint(1, 132), 1) for _ in range(B)]
        iters = [rnd.choice((0, 1, 2, 8)) for _ in range(B)]
        groups = _gn_groups(sp, plans, iters, occ, sm, maxper)
        firsts = []
        for j, n in enumerate(iters):
            if n not in [iters[f] for f in firsts]:
                firsts.append(j)
        assert [g[0] for g in groups] == [iters[f] for f in firsts]          # one group per count, in first-session order
        allseen = []
        for it, launches, solo in groups:
            members = [j for j in range(B) if iters[j] == it]
            sub = [plans[j] for j in members]
            sl, ss = _pack(sb, sub, occ, sm, maxper)                        # each group: s2m_batch_pack of its sessions
            assert launches == [(k, g, [members[s] for s in x]) for k, g, x in sl]
            assert solo == [members[s] for s in ss]
            allseen += [s for _, _, x in launches for s in x] + solo
        assert sorted(allseen) == list(range(B))
