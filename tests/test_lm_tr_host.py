"""CPU tier of the LM's trust-region state machine (liliom_b200/csrc/lm_tr.cuh), compiled for the host (tests/lm_tr_host.cpp)
and driven with the sums tests/lm_reference.py computes on the correspondences of every adversarial LM world
(tests/lm_adversarial.py), for max_num_iter 0, 1, 2 and 15.

The collective LM of a sharded context runs the machine in a fixed number of rounds, 1 + max(0, max_num_iter), with no-op rounds
after the stop; the single-GPU kernel runs it in its own loop until the stop.  Given the same sums, both drivers must ask for the
same evaluations and land on the same iterate, iteration count, stop and stats row, bit for bit, and the fixed driver must be
done by its last round.  Every closed decision and every stop must agree with lm_reference (follow along the machine's iterates,
which are the results of the same solve capped at 0, 1, 2, ... iterations)."""
import ctypes as C
import os

import numpy as np
import pytest

import host_build
import lm_adversarial as LA
import lm_reference as LR

STOPS = {1: "no_correspondences", 2: "iteration_cap", 3: "gradient", 4: "radius_floor", 5: "five_invalid", 6: "parameter",
         7: "function"}                              # lm_tr.cuh::LmStop
CAPS = (0, 1, 2, 15)
CAP_LOG = 64
EVAL = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.POINTER(C.c_double))


class Result(C.Structure):
    _fields_ = [("pose", C.c_double * 7), ("stats", C.c_double * 40), ("iteration", C.c_int), ("done", C.c_int),
                ("n_eval", C.c_int), ("rounds", C.c_int)]


@pytest.fixture(scope="module")
def tr():
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("CUDA headers not found")
    L = host_build.load("lm_tr_host", ["tests/lm_tr_host.cpp"],
                        ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-D_GNU_SOURCE", "-Wno-attributes", "-I", cuda_inc],
                        deps=[f"liliom_b200/csrc/{h}" for h in ("lm_tr.cuh", "dev_math.cuh", "pcl_xform.h", "vg_box.h")])
    dp = C.POINTER(C.c_double)
    L.lmtr_loop.argtypes = [dp, C.c_int, dp, EVAL, dp, C.c_int, C.POINTER(Result)]
    L.lmtr_loop.restype = None
    L.lmtr_rounds.argtypes = [dp, C.c_int, C.c_int, dp, EVAL, dp, C.c_int, C.POINTER(Result)]
    L.lmtr_rounds.restype = None
    return L


@pytest.fixture(scope="module")
def worlds(oracle):
    """builder name -> (feats, valid, plane, guess): the correspondences the oracle finds at each world's guess."""
    out = {}
    for fn, _, _, _ in LA.WORLDS.values():
        if fn.__name__ in out:
            continue
        m, q, g = fn()
        _, v, pl, _, _ = oracle.find_surf_corr(oracle.KdTree(m), q, g)
        out[fn.__name__] = (q, v, pl, g)
    return out


def _drive(tr, which, P, start, mni, rounds=-1):
    x0 = np.ascontiguousarray(start, np.float64)
    neq0 = np.ascontiguousarray(P.at(x0)["S"], np.float64)
    log = np.zeros((CAP_LOG, 7))
    dp = C.POINTER(C.c_double)

    def ev(x, out):
        S = P.at(np.ctypeslib.as_array(x, (7,)).copy())["S"]
        for k in range(29):
            out[k] = float(S[k])
    cb = EVAL(ev)
    r = Result()
    args = (x0.ctypes.data_as(dp), mni) + ((rounds,) if which == "rounds" else ()) + \
        (neq0.ctypes.data_as(dp), cb, log.ctypes.data_as(dp), CAP_LOG, C.byref(r))
    getattr(tr, f"lmtr_{which}")(*args)
    return r, log[:min(r.n_eval, CAP_LOG)].copy()


def _same(a, b):
    ra, la = a
    rb, lb = b
    return (bytes(ra.pose) == bytes(rb.pose) and bytes(ra.stats) == bytes(rb.stats) and ra.iteration == rb.iteration
            and ra.done == rb.done and ra.n_eval == rb.n_eval and la.tobytes() == lb.tobytes())


CASES = [(n, mni) for n in dict.fromkeys(fn.__name__ for fn, _, _, _ in LA.WORLDS.values()) for mni in CAPS]


@pytest.mark.parametrize("world,mni", CASES, ids=[f"{n}-{m}" for n, m in CASES])
def test_fixed_rounds_equal_the_loop(tr, worlds, world, mni):
    feats, v, pl, g = worlds[world]
    P = LR.Problem(feats, v, pl)
    loop = _drive(tr, "loop", P, g, mni)
    fixed = _drive(tr, "rounds", P, g, mni)
    r = fixed[0]
    assert r.rounds == 1 + mni
    assert r.done in STOPS, f"{world} max_num_iter {mni}: not done after {r.rounds} rounds"
    assert _same(loop, fixed), (f"{world} max_num_iter {mni}: loop {loop[0].iteration} iterations, {STOPS.get(loop[0].done)}; "
                                f"rounds {r.iteration}, {STOPS.get(r.done)}")
    assert r.n_eval <= 1 + mni
    # rounds past the bound change nothing: the machine is done and the driver only writes zeros
    assert _same(_drive(tr, "rounds", P, g, mni, rounds=mni + 4), fixed)
    # the stats row: the linearisation sums, the iteration count, the pose
    st = np.array(r.stats)
    S0 = P.at(np.asarray(g, np.float64))["S"]
    assert st[1] == r.iteration and np.array_equal(st[30:37], np.array(r.pose))
    assert np.array_equal(st[3:30], S0[:27]) and st[2] == S0[27] and st[0] == S0[28]


@pytest.mark.parametrize("world,mni", CASES, ids=[f"{n}-{m}" for n, m in CASES])
def test_decisions_and_stop_agree_with_the_reference(tr, worlds, world, mni):
    """lm_reference.follow along the machine's own iterates (the fixed-round solve capped at j = 0 .. its count + 1): every closed
    decision the same, every accepted step within its one-step bound, the stop at the same iteration and for the same reason."""
    feats, v, pl, g = worlds[world]
    P = LR.Problem(feats, v, pl)
    full, _ = _drive(tr, "rounds", P, g, mni)
    its = [np.asarray(g, np.float64)]
    for j in range(1, min(full.iteration + 1, mni) + 1):
        rj, _ = _drive(tr, "rounds", P, g, j)
        assert rj.iteration == min(j, full.iteration), (world, j, rj.iteration, full.iteration)
        its.append(np.array(rj.pose))
    t = LR.follow(feats, v, pl, g, its, full.iteration, mni)
    assert t["stop"] == STOPS[full.done], (world, mni, t["stop"], STOPS[full.done])
    ref = LR.run(feats, v, pl, g, mni)
    if not any(rec["open"] for rec in ref["records"]):
        assert (ref["iters"], ref["stop"]) == (full.iteration, STOPS[full.done]), (world, mni, ref["iters"], ref["stop"])
