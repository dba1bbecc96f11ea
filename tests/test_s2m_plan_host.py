"""CPU tier for the LAUNCH PLAN of the scan-to-map call: liliom_b200/csrc/s2m_plan.h compiled for the host (tests/s2m_plan_host.cpp).
Which kernel shape runs for a given query count, SM count, mode and rank set is decided there; the table pins the decisions the
library makes today (measured shapes, DESIGN.md §3), the invariants what every plan must satisfy for its kernels to be valid."""
import ctypes as C
import itertools

import pytest

import host_build

GN, CERES = 1, 0

# (n, n_last, dev_count, sm_count, mode, iters, want_corr, nranks, peer, force_lanes, force_rounds, knn_tma)
#   -> (n_est, lanes, rounds, per_task, grid, persistent, tma, dyn_smem)
TABLE = [
    ((1400, 0, 0, 132, GN, 10, 0, 1, 0, 0, 0, 0), (1400, 16, 1, 2, 88, 1, 0, 0)),          # headline scan
    ((3100, 0, 0, 132, GN, 10, 0, 1, 0, 0, 0, 0), (3100, 8, 1, 4, 97, 1, 0, 0)),           # configs[2]: the 8-lane override
    ((15000, 0, 0, 132, GN, 10, 0, 1, 0, 0, 0, 0), (15000, 2, 1, 16, 118, 1, 0, 0)),       # dense probe
    ((130000, 0, 0, 132, GN, 10, 0, 1, 0, 0, 0, 0), (130000, 1, 1, 32, 264, 0, 0, 32768)),  # streamed set: per-pass, one thread per query
    ((14400, 0, 1, 132, GN, 10, 0, 1, 0, 0, 0, 0), (14400, 2, 1, 16, 141, 0, 0, 0)),       # first call, device-side count: upper bound
    ((14400, 1400, 1, 132, GN, 10, 0, 1, 0, 0, 0, 0), (1400, 16, 1, 2, 110, 1, 0, 0)),     # second call: predicted from the first
    ((1400, 0, 0, 132, GN, 0, 1, 1, 0, 0, 0, 0), (1400, 16, 1, 2, 88, 0, 0, 0)),           # want_corr
    ((3100, 0, 0, 132, GN, 0, 1, 1, 0, 0, 0, 0), (3100, 16, 1, 2, 194, 0, 0, 0)),          # want_corr: no 8-lane override
    ((1400, 0, 0, 132, CERES, 10, 0, 1, 0, 0, 0, 0), (1400, 16, 1, 2, 88, 0, 0, 0)),       # CERES
    ((1400, 0, 0, 132, GN, 10, 0, 2, 0, 0, 0, 0), (1400, 16, 1, 2, 88, 0, 0, 0)),          # two ranks, NCCL + k_gn_update
    ((1400, 0, 0, 132, GN, 10, 0, 2, 1, 0, 0, 0), (1400, 16, 1, 2, 88, 1, 0, 0)),          # two ranks, fused exchange
    ((1400, 0, 0, 132, GN, 10, 0, 1, 0, 4, 2, 0), (1400, 4, 2, 16, 11, 1, 0, 0)),          # forced lanes and rounds
    ((1400, 0, 0, 132, GN, 10, 0, 1, 0, 1, 3, 0), (1400, 1, 1, 32, 6, 1, 0, 32768)),       # forced rounds clamped to 32 queries per task
    ((1400, 0, 0, 132, GN, 10, 0, 1, 0, 0, 0, 1), (1400, 16, 1, 2, 88, 1, 1, 57856)),      # TMA staging
    ((3100, 0, 0, 132, GN, 10, 0, 1, 0, 0, 0, 1), (3100, 8, 1, 4, 97, 1, 0, 0)),           # TMA switch, 8-lane shape: not staged
    ((1400, 0, 0, 16, GN, 10, 0, 1, 0, 0, 0, 0), (1400, 2, 1, 16, 11, 1, 0, 0)),           # 16 SMs
    ((1400, 0, 0, 132, GN, 0, 0, 1, 0, 0, 0, 0), (1400, 16, 1, 2, 88, 0, 0, 0)),           # no iterations
]


@pytest.fixture(scope="module")
def sp():
    L = host_build.load("s2m_plan_host", ["tests/s2m_plan_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall"],
                        deps=["liliom_b200/csrc/s2m_plan.h", "liliom_b200/csrc/batch.h", "include/liliom.h"])
    L.sp_plan.argtypes = [C.c_int] * 12 + [C.POINTER(C.c_longlong)]
    L.sp_plan.restype = None
    return L


def _plan(sp, args):
    out = (C.c_longlong * 8)()
    sp.sp_plan(*args, out)
    return tuple(out)


@pytest.mark.parametrize("args,want", TABLE)
def test_plan_table(sp, args, want):
    assert _plan(sp, args) == want


def test_plan_invariants(sp):
    for n, n_last, dev, sm, mode, iters, corr, ranks, fl, tma in itertools.product(
            (0, 1, 40, 1400, 1900, 3100, 3800, 8000, 15000, 40000, 130000), (0, 1400, 50000), (0, 1), (16, 84, 132), (GN, CERES),
            (0, 1, 10), (0, 1), ((1, 0), (2, 0), (2, 1)), ((0, 0), (16, 1), (8, 3), (1, 2)), (0, 1)):
        nranks, peer = ranks
        args = (n, n_last, dev, sm, mode, iters, corr, nranks, peer, fl[0], fl[1], tma)
        n_est, lanes, rounds, per_task, grid, persistent, staged, dyn = _plan(sp, args)
        assert lanes in (1, 2, 4, 8, 16) and rounds >= 1 and per_task == (32 // lanes) * rounds <= 32, args
        assert 1 <= grid <= 2 * sm, args
        if persistent:
            assert grid <= sm and mode == GN and iters > 0 and not corr and (nranks == 1 or peer), args
        if staged:
            assert lanes == 16 and persistent and tma, args
        assert (dyn > 0) == (lanes == 1 or bool(staged)), args
