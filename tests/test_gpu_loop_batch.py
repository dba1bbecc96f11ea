"""GPU tier for the batched loop closure (liliom_loop_align_batch): B sessions' loop closures in one call against the same
sessions' solo liliom_loop_align calls, bit for bit.  Twin context sets hold the same keyframe stores; set A is driven solo, set B
batched, and every result, status, counter and later solo call is compared on bytes.  Covered: B = 1, 2, 8, 32 and 34 (two
table launches) with 48- and 32-byte sessions mixed and per-session settings; sessions of 1 iteration beside sessions that run
to max_iter; a 300k-point source that fills a co-resident grid by itself; a session whose voxel index wraps (wide keys); empty
and out-of-reach sessions; per-session errors; whole-call refusals; caller streams; and the context's
resident state."""
import ctypes as C
import os

import numpy as np
import pytest

from test_gpu_loop_closure import N_HIST, REVISIT, NO_EDGE, _backend_session, _bytes, _drifted

pytestmark = pytest.mark.gpu

B_MAX = 34
PARAMS = [dict(leaf=0.4), dict(leaf=0.6, max_corr_dist=2.0, max_iter=3), dict(leaf=0.4, max_iter=1),
          dict(leaf=0.5, max_corr_dist=5.0, trans_eps=1e-8, fit_eps=1e-9)]


def _stride(i):
    return 48 if i % 2 == 0 else 32


_SEQS = {}


def _seq(stride, seed):
    from liliom_b200 import synth
    if (stride, seed) not in _SEQS:
        seq = synth.make_keyframe_sequence(N_HIST, stride=stride, seed=seed, revisit=1)
        e5, s5, p5 = seq[5]
        seq.append((e5[:0], s5, p5))             # NO_EDGE: a keyframe stored with an empty edge cloud
        _SEQS[(stride, seed)] = seq
    return _SEQS[(stride, seed)]


def _store(stride, seed, env=None):
    """a context holding the keyframe sequence (stride, seed); env: LILIOM_* variables set while it is created"""
    import liliom_b200 as L
    variant = 0 if stride == 48 else 1
    old = {k: os.environ.get(k) for k in (env or {})}
    try:
        os.environ.update(env or {})
        c = L.Context(variant=variant)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    bp = L.backend_default_params(variant)
    seq = _seq(stride, seed)
    for i, (e, s, _) in enumerate(seq):
        assert c.kf_add(bp, e, s, download=False)[0] == i
    return c, [p for _, _, p in seq]


def _spec(i, poses):
    """session i's lists and settings: test_gpu_loop_closure.py's four shapes and a drifted revisit, cycling with PARAMS"""
    hist = list(range(N_HIST))
    shape = i % 5
    if shape == 0:
        si, ti = [REVISIT], hist
    elif shape == 1:
        si, ti = [3, 3], [0, 1, 1, 2, 2, 2, 4]
    elif shape == 2:
        si, ti = [NO_EDGE], [4, NO_EDGE, 6, 7]
    elif shape == 3:
        si, ti = hist, [REVISIT]
    else:
        si, ti = [REVISIT], hist
    sp, tp = [poses[k] for k in si], [poses[k] for k in ti]
    if shape == 4:
        sp = [_drifted(poses[REVISIT], 2.0, [0.1, -0.1, 1.0], np.array([0.4, -0.25, 0.15]))[0]]
    return dict(si=si, sp=sp, ti=ti, tp=tp, prm=dict(PARAMS[i % len(PARAMS)]))


def _solo(c, s):
    import liliom_b200 as L
    try:
        return c.loop_align(s["si"], s["sp"], s["ti"], s["tp"], **s["prm"]), 0
    except L.LiliomError as e:
        return None, e.code


def _batch(cs, specs):
    import liliom_b200 as L
    return L.loop_align_batch(cs, [s["si"] for s in specs], [s["sp"] for s in specs], [s["ti"] for s in specs],
                              [s["tp"] for s in specs], [s["prm"] for s in specs])


def _counts(c):
    k = c.counters()
    return (k.launches, k.lib_launches)


def _same(a, b, what):
    assert _bytes(a[0]) == _bytes(b[0]), what
    assert np.float64(a[1]).tobytes() == np.float64(b[1]).tobytes(), what
    assert tuple(a[2:]) == tuple(b[2:]), (what, a[1:], b[1:])


def _compare(A, Bc, specs, label):
    """solo calls on A, one batched call on B: results, statuses and counters equal; returns the solo results"""
    want = [_solo(c, s) for c, s in zip(A, specs)]
    got, status = _batch(Bc, specs)
    for i, (w, rc) in enumerate(want):
        assert status[i] == rc, (label, i, status[i], rc)
        if rc == 0:
            _same(got[i], w, f"{label} session {i}")
        assert _counts(A[i]) == _counts(Bc[i]), (label, i, _counts(A[i]), _counts(Bc[i]))
    return want


def _again(A, Bc, specs, label):
    """one more solo call on both sets gives the same bits (the state each call left is the same)"""
    for i, (a, b, s) in enumerate(zip(A, Bc, specs)):
        ra, rca = _solo(a, s)
        rb, rcb = _solo(b, s)
        assert rca == rcb, (label, i)
        if rca == 0:
            _same(ra, rb, f"{label} again {i}")
        assert _counts(a) == _counts(b), (label, i)


@pytest.fixture(scope="module")
def pool():
    """B_MAX twin sessions: A[i] and B[i] hold the same store (layout _stride(i), one of four seeds)"""
    A, Bc, poses = [], [], []
    for i in range(B_MAX):
        a, p = _store(_stride(i), 7 + i % 4)
        b, _ = _store(_stride(i), 7 + i % 4)
        A.append(a); Bc.append(b); poses.append(p)
    yield A, Bc, poses
    for c in A + Bc:
        c.close()


@pytest.mark.parametrize("B", [1, 2, 8, 32, 34])
def test_batch_matches_solo(pool, B):
    A, Bc, poses = pool
    specs = [_spec(i + B, poses[i]) for i in range(B)]
    want = _compare(A[:B], Bc[:B], specs, f"B={B}")
    assert all(rc == 0 for _, rc in want)
    its = [w[0][3] for w in want]
    if B >= 8:
        assert 1 in its and max(its) > 3, its          # 1-iteration sessions shared launches with longer ones
    _again(A[:B], Bc[:B], specs, f"B={B}")


def _big_store(stride, rng):
    """a store whose keyframe 0 holds a 300k-point cloud (kept whole by a fine surf leaf) and keyframe 1 a 30k-point part of it"""
    import liliom_b200 as L
    variant = 0 if stride == 48 else 1
    c = L.Context(variant=variant)
    bp = L.backend_default_params(variant)
    bp.surf_leaf = 0.02
    xyz = np.column_stack([rng.uniform(-30, 30, 300_000), rng.uniform(-30, 30, 300_000), rng.uniform(-2, 2, 300_000)])
    xyz[:, 2] += 0.3 * np.sin(xyz[:, 0] / 3.0) * np.cos(xyz[:, 1] / 4.0)
    cloud = np.zeros(len(xyz), c.dtype)
    cloud["x"], cloud["y"], cloud["z"] = xyz.astype(np.float32).T
    part = cloud[rng.permutation(len(cloud))[:30_000]]
    for s in (cloud, part):
        c.kf_add(bp, cloud[:0], s, download=False)
    return c


def _wide_store(stride):
    """a store whose keyframe 0 spans the wrap box of tests/vg_adversarial.py at leaf 0.001 (2 km of y): its VoxelGrid needs wide keys"""
    import liliom_b200 as L
    import vg_adversarial as V
    variant = 0 if stride == 48 else 1
    c = L.Context(variant=variant)
    bp = L.backend_default_params(variant)
    bp.surf_leaf = 0.001
    w = V.wrap_order(leaf=0.001)
    w = w if stride == 48 else V.to32(w)
    c.kf_add(bp, w[:0], np.ascontiguousarray(w, c.dtype), download=False)
    return c


IDENT = np.array([1.0, 0, 0, 0, 0, 0, 0])


def _special_sessions(stride_of):
    """ordinary, 300k-point source, wide keys, empty source, empty target, out of reach, four erroring sessions, ordinary"""
    rng = np.random.default_rng(5)
    cs, specs = [], []
    c, poses = _store(stride_of(0), 11)
    hist, hp = list(range(N_HIST)), [poses[k] for k in range(N_HIST)]
    cs.append(c); specs.append(dict(si=[REVISIT], sp=[poses[REVISIT]], ti=hist, tp=hp, prm=dict(leaf=0.4)))
    cs.append(_big_store(stride_of(1), rng))
    drift = _drifted(IDENT, 1.0, [0.2, 0.1, 1.0], np.array([0.2, -0.1, 0.05]))[0]
    specs.append(dict(si=[0], sp=[drift], ti=[1], tp=[IDENT], prm=dict(leaf=0.02, max_corr_dist=1.0, max_iter=12)))
    cs.append(_wide_store(stride_of(2)))
    specs.append(dict(si=[0], sp=[IDENT], ti=[0], tp=[IDENT], prm=dict(leaf=0.001, max_iter=5)))
    far = poses[REVISIT].copy(); far[4] += 500.0
    for k, s in enumerate([dict(si=[], sp=[], ti=hist[:10], tp=hp[:10], prm=dict(leaf=0.4)),
                           dict(si=[REVISIT], sp=[poses[REVISIT]], ti=[], tp=[], prm=dict(leaf=0.4)),
                           dict(si=[REVISIT], sp=[far], ti=hist[:10], tp=hp[:10], prm=dict(leaf=0.4, max_corr_dist=5.0)),
                           dict(si=[REVISIT + 100], sp=[poses[0]], ti=hist, tp=hp, prm=dict(leaf=0.4)),
                           dict(si=[REVISIT], sp=[poses[0]], ti=[0, -1], tp=[poses[0]] * 2, prm=dict(leaf=0.4)),
                           dict(si=[REVISIT], sp=[poses[0]], ti=hist, tp=hp, prm=dict(leaf=0.0)),
                           dict(si=[REVISIT], sp=[poses[0]], ti=hist, tp=hp, prm=dict(leaf=0.4, max_iter=0)),
                           dict(si=[1, 2], sp=[poses[1], poses[2]], ti=hist, tp=hp, prm=dict(leaf=0.6, max_corr_dist=2.0, max_iter=3))]):
        c, _ = _store(stride_of(3 + k), 11 + k % 2)
        cs.append(c); specs.append(s)
    return cs, specs


def test_large_wide_empty_and_erroring_sessions_beside_ordinary_ones():
    import liliom_b200 as L
    stride_of = lambda i: 48 if i % 3 != 1 else 32                       # noqa: E731
    A, specs = _special_sessions(stride_of)
    Bc, _ = _special_sessions(stride_of)
    try:
        want = _compare(A, Bc, specs, "special")
        rcs = [rc for _, rc in want]
        assert rcs[:6] == [0] * 6 and rcs[6:10] == [L._binding.E_ARG] * 4 and rcs[10] == 0, rcs
        assert want[1][0][4] > 250_000 and want[1][0][2], want[1][0][1:]          # the big source converged
        for k in (3, 4, 5):
            T, fit, conv, it, ns, nt = want[k][0]
            assert not conv and it == 0 and np.array_equal(T, np.eye(4)), k
        _again(A, Bc, specs, "special")
    finally:
        for c in A + Bc:
            c.close()


def test_caller_streams():
    """two sessions on caller streams (ctxs[0] among them)"""
    import torch
    A, Bc, poses = [], [], []
    for i in range(5):
        a, p = _store(_stride(i), 7 + i % 3)
        b, _ = _store(_stride(i), 7 + i % 3)
        A.append(a); Bc.append(b); poses.append(p)
    try:
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        Bc[0].set_stream(streams[0].cuda_stream); Bc[3].set_stream(streams[1].cuda_stream)
        specs = [_spec(i, poses[i]) for i in range(5)]
        _compare(A, Bc, specs, "streams")
        _again(A, Bc, specs, "streams")
    finally:
        for c in A + Bc:
            c.close()


def test_whole_call_refusals_change_nothing(pool):
    import liliom_b200 as L
    A, Bc, poses = pool
    cs = Bc[:2]
    specs = [_spec(i, poses[i]) for i in range(2)]
    before = [_counts(c) for c in cs]
    for bad in ([cs[0], cs[0]], [cs[0], None]):
        with pytest.raises(L.LiliomError) as e:
            _batch(bad, specs)
        assert e.value.code == L._binding.E_ARG
    lib = L._binding.lib()
    vp = C.c_void_p
    h = (vp * 2)(cs[0]._h, cs[1]._h)
    ip, dp = C.POINTER(C.c_int), C.POINTER(C.c_double)
    ids = [np.array(s["si"], np.int32) for s in specs]
    pz = [np.ascontiguousarray(s["sp"], np.float64).reshape(-1) for s in specs]
    I = (ip * 2)(*[a.ctypes.data_as(ip) for a in ids])
    P = (dp * 2)(*[a.ctypes.data_as(dp) for a in pz])
    k = (C.c_int * 2)(*[len(a) for a in ids])
    prm = (L.LoopParams * 2)(L.LoopParams(0.4, 30.0, 100, 1e-6, 1e-6), L.LoopParams(0.4, 30.0, 100, 1e-6, 1e-6))
    res = (L.LoopResult * 2)()
    st = (C.c_int * 2)()
    calls = [lib.liliom_loop_align_batch(h, 0, I, P, k, I, P, k, prm, res, st),
             lib.liliom_loop_align_batch(h, -1, I, P, k, I, P, k, prm, res, st),
             lib.liliom_loop_align_batch(None, 2, I, P, k, I, P, k, prm, res, st),
             lib.liliom_loop_align_batch(h, 2, None, P, k, I, P, k, prm, res, st),
             lib.liliom_loop_align_batch(h, 2, I, None, k, I, P, k, prm, res, st),
             lib.liliom_loop_align_batch(h, 2, I, P, None, I, P, k, prm, res, st),
             lib.liliom_loop_align_batch(h, 2, I, P, k, None, P, k, prm, res, st),
             lib.liliom_loop_align_batch(h, 2, I, P, k, I, None, k, prm, res, st),
             lib.liliom_loop_align_batch(h, 2, I, P, k, I, P, None, prm, res, st),
             lib.liliom_loop_align_batch(h, 2, I, P, k, I, P, k, None, res, st),
             lib.liliom_loop_align_batch(h, 2, I, P, k, I, P, k, prm, None, st),
             lib.liliom_loop_align_batch(h, 2, I, P, k, I, P, k, prm, res, None)]
    assert calls == [L._binding.E_ARG] * len(calls), calls
    assert [_counts(c) for c in cs] == before
    # a NULL list with k > 0 and a negative k are that session's error; the other session runs
    k_bad = (C.c_int * 2)(-1, len(ids[1]))
    assert lib.liliom_loop_align_batch(h, 2, I, P, k_bad, I, P, k, prm, res, st) == 0
    assert list(st) == [L._binding.E_ARG, 0]
    I_null = (ip * 2)(ip(), ids[1].ctypes.data_as(ip))
    assert lib.liliom_loop_align_batch(h, 2, I_null, P, k, I, P, k, prm, res, st) == 0
    assert list(st) == [L._binding.E_ARG, 0]
    # the solo twin of session 1 made the same two calls: keep the sets in step for the other tests of the module
    for _ in range(2):
        a = A[1]
        a.loop_align(specs[1]["si"], specs[1]["sp"], specs[1]["si"], specs[1]["sp"], 0.4)
    assert _counts(A[0]) == _counts(cs[0]) and _counts(A[1]) == _counts(cs[1])


@pytest.mark.parametrize("stride", [48, 32])
def test_batched_loop_closure_leaves_the_resident_state_alone(stride):
    import liliom_b200 as L
    variant = 0 if stride == 48 else 1
    seq = _seq(stride, 7)
    poses = [p for _, _, p in seq]

    def fill(c, bp):
        for e, s, _ in seq:
            c.kf_add(bp, e, s, download=False)
        return seq[20][0]

    res = {}

    def call(c):
        other, _ = _store(stride, 8)
        try:
            hist = list(range(N_HIST))
            out, status = L.loop_align_batch([c, other], [[REVISIT]] * 2, [[poses[REVISIT]]] * 2, [hist] * 2,
                                             [[poses[i] for i in hist]] * 2, [dict(leaf=0.4)] * 2)
            res["r"], res["status"] = out[0], list(status)
        finally:
            other.close()
        with pytest.raises(L.LiliomError) as e:              # the batch, as the solo call, leaves no resident scan behind
            c.map_update_resident(IDENT)
        res["map_update"] = e.value.code

    with_call = _backend_session(variant, poses, fill, call)
    without = _backend_session(variant, poses, fill, None)
    assert res["status"] == [0, 0] and res["r"][2] and res["r"][3] >= 1
    assert res["map_update"] == L._binding.E_ARG
    for k in without:
        assert _bytes(with_call[k]) == _bytes(without[k]), k


def test_icp_bits_do_not_depend_on_the_grid():
    """sessions whose batched ICP gets fewer blocks than its solo grid (LILIOM_TEST_ICP_BLOCKS, read at create) beside ordinary
    ones: each block then deals several virtual blocks, and every result equals the solo call's (solo grid) bit for bit"""
    hist = list(range(N_HIST))
    A, Bc, specs = [], [], []
    for i, cap in enumerate([0, 1, 0, 3, 0, 7, 0]):
        a, poses = _store(_stride(i), 7 + i % 3)
        b, _ = _store(_stride(i), 7 + i % 3, env={"LILIOM_TEST_ICP_BLOCKS": str(cap)} if cap else None)
        A.append(a); Bc.append(b)
        hp = [poses[k] for k in hist]
        if cap:                                   # the 41 history keyframes onto the revisit: tens of virtual blocks
            specs.append(dict(si=hist, sp=hp, ti=[REVISIT], tp=[poses[REVISIT]], prm=dict(leaf=0.4)))
        else:
            specs.append(_spec(i, poses))
    try:
        want = _compare(A, Bc, specs, "grid")
        for i, cap in enumerate([0, 1, 0, 3, 0, 7, 0]):
            if cap:
                n_src, it = want[i][0][4], want[i][0][3]
                assert (n_src + 255) // 256 > cap and it >= 2, (n_src, it)
        _again(A, Bc, specs, "grid")
    finally:
        for c in A + Bc:
            c.close()
