"""The keyframe hand-off of many sessions in one call (liliom_undistort_resident_batch, liliom_kf_add_resident_batch) against
each session's solo calls (liliom_undistort_resident, liliom_kf_add_resident), byte for byte.

Every case builds a pool of sessions (a source context that extracts and a backend context that stores) twice: one pool goes
through the batched calls, its twin through the solo calls, on the same sweeps.  Compared: statuses, liliom_last_error, ids,
counts, launches and lib_launches, the de-skewed resident clouds, and the stores, read back as they are (liliom_global_map at a
leaf PCL declines) and through liliom_bmap_build, liliom_backend_window_correspond and liliom_loop_align, which pins the ids and
the arena offsets."""
import ctypes as C
import os

import numpy as np
import pytest

import history_ops as H

pytestmark = pytest.mark.gpu

IDENT7 = np.array([1.0, 0, 0, 0, 0, 0, 0])
IDENT_Q = (1.0, 0.0, 0.0, 0.0)
TINY_LEAF = 1e-4          # PCL declines every keyframe-sized cloud at this leaf: the output is the stored cloud
N_SWEEPS = 3


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def _L():
    import liliom_b200 as L
    return L


def _ctx(variant, **kw):
    L = _L()
    p = L.default_params(variant)
    for k, v in kw.items():
        setattr(p, k, v)
    return L.Context(p)


def _last_error(c):
    return _L()._binding.lib().liliom_last_error(c._h).decode()


def _cnt(c):
    k = c.counters()
    return k.launches, k.lib_launches


@pytest.fixture(scope="module")
def sweeps():
    """N_SWEEPS Horizon sweeps and N_SWEEPS 64-line sweeps along a short path"""
    from liliom_b200 import synth
    T0 = synth.default_true_pose()
    out = {0: [], 1: []}
    for k in range(N_SWEEPS):
        T = np.array(T0); T[4] += 0.6 * k; T[5] += 0.12 * k
        pts, q = synth.make_horizon_sweep(T, seed=1 + k)
        out[0].append(dict(pts=pts, q=q))
        pts, q = synth.make_hdl64_sweep(T, seed=2 + k, steps=1200)
        out[1].append(dict(pts=pts, q=q))
    return out


def _extract(c, variant, sw):
    """upload_scan + extract_resident: a Horizon extraction's sizes stay on the device, a ROT one's come back to the host"""
    c.upload_scan(sw["pts"])
    n = c.extract_resident(sw["q"])
    assert (n == (-1, -1, -1)) == (variant == 0), n


def _motion(i, t):
    """publishCloudLast's arguments of session i at tick t: a translation of its own, the identity rotation the reference passes
    for every third session and a small rotation of its own for the others"""
    from liliom_b200 import synth
    trans = (0.22 + 0.013 * i, -0.07 + 0.004 * t, 0.011 * (i % 4))
    quat = IDENT_Q if i % 3 == 0 else tuple(synth.q_from_axis_angle([0.3, -0.2, 1.0 + 0.1 * i], 0.004 * (1 + i % 5)))
    return trans, quat


class Sess:
    """one session: its source `odo`, its backend `bk`, its variant and backend parameters"""

    def __init__(self, variant, bp=None):
        self.variant = variant
        self.odo = _ctx(variant)
        self.bk = _ctx(variant)
        self.bp = bp if bp is not None else _L().backend_default_params(variant)

    def close(self):
        for c in {id(self.odo): self.odo, id(self.bk): self.bk}.values():
            c.close()


def _store_state(bk, bp):
    """everything observable about a store: every keyframe's stored clouds, the local map of all of them, the window search of the
    last three and one loop closure"""
    L = _L()
    n = bk.kf_count()
    out = [n]
    for i in range(n):
        for kind in (L.KF_SURF, L.KF_FULL):
            out.append(_bytes(bk.global_map(kind, [i], [IDENT7], TINY_LEAF)))
    if n:
        ids = list(range(n))
        poses = [IDENT7 + np.array([0, 0, 0, 0, 0.6 * i, 0.12 * i, 0]) for i in ids]
        out.append(bk.bmap_build(bp, ids, poses))
        out += [_bytes(bk.bmap_download(0)), _bytes(bk.bmap_download(1))]
        w = ids[-3:]
        out.append(repr(bk.backend_window_correspond(bp, w, poses[-len(w):])))
    if n >= 2:
        la = bk.loop_align([n - 1], [IDENT7 + np.array([0, 0, 0, 0, 0.6 * n, 0.12 * n, 0])], list(range(n - 1)),
                           [IDENT7 + np.array([0, 0, 0, 0, 0.6 * i, 0.12 * i, 0]) for i in range(n - 1)], 0.4, max_iter=20)
        out += [_bytes(la[0]), repr(la[1:])]
    return out


def _feats(c):
    L = _L()
    try:
        return [_bytes(x) for x in c.features_download()]
    except L.LiliomError as e:
        return e.code


def _deskew_batch(S, t):
    L = _L()
    mot = [_motion(i, t) for i in range(len(S))]
    status = L.undistort_resident_batch([s.odo for s in S], [m[0] for m in mot], [m[1] for m in mot])
    return list(status)


def _deskew_solo(S, t):
    return [(s.odo.undistort_resident(*_motion(i, t)) or 0) for i, s in enumerate(S)]


def _store_batch(S, srcs=None):
    L = _L()
    srcs = [s.odo for s in S] if srcs is None else srcs
    ids, counts, status = L.kf_add_resident_batch([s.bk for s in S], [s.bp for s in S], srcs)
    return [(int(st), int(k), tuple(int(x) for x in n)) if st == 0 else (int(st), _last_error(s.bk))
            for s, st, k, n in zip(S, status, ids, counts)]


def _store_solo(S, srcs=None, order=None):
    L = _L()
    srcs = [s.odo for s in S] if srcs is None else srcs
    out = [None] * len(S)
    for i in (range(len(S)) if order is None else order):
        s = S[i]
        kid, ne, ns, nf = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        rc = L._binding.lib().liliom_kf_add_resident(s.bk._h, C.byref(s.bp), srcs[i]._h if srcs[i] is not None else None, C.byref(kid),
                                                     C.byref(ne), C.byref(ns), C.byref(nf))
        out[i] = (0, kid.value, (ne.value, ns.value, nf.value)) if rc == 0 else (rc, _last_error(s.bk))
    return out


def _reset(S):
    for s in S:
        s.odo.counters(reset=True)
        s.bk.counters(reset=True)


def _all_counts(S):
    return [(_cnt(s.odo), _cnt(s.bk)) for s in S]


def _tick(A, Bp, sweeps, t, oracle=None):
    """one fleet tick on both pools: extraction (untimed, identical), then the hand-off batched on A and solo on Bp; compares
    everything the two calls return and leave"""
    for P in (A, Bp):
        for i, s in enumerate(P):
            _extract(s.odo, s.variant, sweeps[s.variant][(i + t) % N_SWEEPS])
    before = [s.odo.features_download() for s in A] if oracle is not None else None
    _reset(A); _reset(Bp)
    assert _deskew_batch(A, t) == _deskew_solo(Bp, t) == [0] * len(A)
    assert [_feats(s.odo) for s in A] == [_feats(s.odo) for s in Bp], t
    if oracle is not None:
        for i, s in enumerate(A):
            for b, a in zip(before[i], s.odo.features_download()):
                assert _bytes(a) == _bytes(oracle.undistort(b, *_motion(i, t))), (i, t)
    ra, rb = _store_batch(A), _store_solo(Bp)
    assert ra == rb, (t, ra, rb)
    assert _all_counts(A) == _all_counts(Bp), t
    return ra


def _pool(variants):
    return [Sess(v) for v in variants]


def _close(*pools):
    for P in pools:
        for s in P:
            s.close()


# ---------------------------------------------------------------- 1. B and packing
@pytest.mark.parametrize("B", [1, 2, 3, 8, 32, 33])
def test_batch_equals_solo(sweeps, oracle, B):
    """B sessions mixing Horizon / variant 0 and HDL-64E / variant 1, each with its own motion: two ticks batched = solo, the
    de-skew = the oracle's undistortion; then every store reads back the same through the backend's calls"""
    variants = [i % 2 for i in range(B)] if B > 1 else [0]
    A, Bp = _pool(variants), _pool(variants)
    try:
        for t in range(2):
            r = _tick(A, Bp, sweeps, t, oracle if t == 0 else None)
            assert [x[1] for x in r] == [t] * B and all(min(x[2]) > 0 for x in r), r
        for a, b in zip(A, Bp):
            assert _store_state(a.bk, a.bp) == _store_state(b.bk, b.bp)
    finally:
        _close(A, Bp)


def test_deskew_empty_and_erroring_sessions(sweeps):
    """a Horizon session without edge points, an empty sweep (no launch, as in its solo call) and a context with nothing resident
    (its status) beside ordinary sessions"""
    L = _L()
    pools = []
    for _ in range(2):
        cs = [_ctx(0), _ctx(0, edge_thres=1e30), _ctx(1), _ctx(0), _ctx(1)]
        _extract(cs[0], 0, sweeps[0][0])
        _extract(cs[1], 0, sweeps[0][1])
        cs[2].upload_scan(sweeps[1][0]["pts"][:0])
        cs[2].extract_resident(sweeps[1][0]["q"])
        _extract(cs[4], 1, sweeps[1][1])                          # cs[3]: nothing resident
        for c in cs:
            c.counters(reset=True)
        pools.append(cs)
    A, Bp = pools
    try:
        mot = [_motion(i, 0) for i in range(len(A))]
        st = list(L.undistort_resident_batch(A, [m[0] for m in mot], [m[1] for m in mot]))
        sb = []
        for c, m in zip(Bp, mot):
            try:
                c.undistort_resident(*m)
                sb.append(0)
            except L.LiliomError as e:
                sb.append(e.code)
        assert st == sb == [0, 0, 0, L._binding.E_ARG, 0], (st, sb)
        assert [_feats(c) for c in A] == [_feats(c) for c in Bp]
        assert [_last_error(c) for c in A] == [_last_error(c) for c in Bp]
        assert [_cnt(c) for c in A] == [_cnt(c) for c in Bp] and [_cnt(c)[0] for c in A] == [1, 1, 0, 0, 1]
        assert len(A[1].features_download()[1]) == 0 and [len(x) for x in A[2].features_download()] == [0, 0, 0]
    finally:
        for c in A + Bp:
            c.close()


# ---------------------------------------------------------------- 2. special sessions beside ordinary ones
def _loopback_ctx(variant, group):
    """rank 0 of a two-rank loopback group (the single-GPU stand-in for a communicator, see test_gpu_sharded.py)"""
    os.environ["LILIOM_TEST_LOOPBACK"] = f"{group}:0/2"
    try:
        return _ctx(variant)
    finally:
        os.environ.pop("LILIOM_TEST_LOOPBACK", None)


def _wide_sweep():
    """a Horizon sweep whose cut cloud spans the wrap box of tests/vg_adversarial.py at leaf 0.001: the full cloud's VoxelGrid
    (variant 1, surf_leaf 0.001) needs wide keys"""
    import vg_adversarial as V
    w = V.wrap_order(leaf=0.001)
    pts = np.zeros(len(w), _L().PT48)
    for f in pts.dtype.names:
        if f in w.dtype.names:
            pts[f] = w[f]
    return pts


def _special_pool(sweeps, group):
    """ordinary Horizon, growing arenas, wide keys, empty sweep, one session per per-session error, ordinary ROT.  Returns the
    sessions and their tick-1 sources (the error cases' own)"""
    L = _L()
    S, srcs = [], []
    S.append(Sess(0)); srcs.append(None)                           # ordinary
    S.append(Sess(0)); srcs.append(None)                           # its full arena grows, with a copy, inside the tick-1 call
    wide_bp = L.backend_default_params(1)
    wide_bp.surf_leaf = 0.001
    S.append(Sess(0, wide_bp)); srcs.append("wide")
    S.append(Sess(1)); srcs.append("empty")
    S.append(Sess(0)); srcs.append(_ctx(0))                        # nothing resident on the source
    bad = L.backend_default_params(0)
    bad.edge_leaf = 0.0
    S.append(Sess(0)); srcs.append("bad_bp")
    S.append(Sess(0)); srcs.append("rot")                          # strides differ
    S.append(Sess(0)); srcs.append(_loopback_ctx(0, group))        # a source with a communicator
    S.append(Sess(1)); srcs.append("null")
    S.append(Sess(1)); srcs.append(None)                           # ordinary
    return S, srcs, bad


def test_special_sessions_beside_ordinary_ones(sweeps):
    L = _L()
    pools = [_special_pool(sweeps, g) for g in ("kfhb_a", "kfhb_b")]
    try:
        for S, _, _ in pools:                                       # tick 0: one keyframe each, by the solo calls
            for i, s in enumerate(S):
                _extract(s.odo, s.variant, sweeps[s.variant][i % N_SWEEPS])
            assert all(r[0] == 0 for r in _store_solo(S))
        for S, srcs, bad in pools:                                  # tick 1: the special sources and parameters
            for i, s in enumerate(S):
                if srcs[i] == "wide":
                    s.odo.extract_horizon(_wide_sweep(), IDENT_Q)
                elif srcs[i] == "empty":
                    s.odo.upload_scan(sweeps[1][0]["pts"][:0])
                    s.odo.extract_resident(sweeps[1][0]["q"])
                    assert [len(x) for x in s.odo.features_download()] == [0, 0, 0]
                elif srcs[i] is None or srcs[i] == "bad_bp":
                    _extract(s.odo, s.variant, sweeps[s.variant][(i + 1) % N_SWEEPS])
                elif srcs[i] == "rot":
                    srcs[i] = _ctx(1)
                    _extract(srcs[i], 1, sweeps[1][0])
            for i, s in enumerate(S):
                if srcs[i] == "bad_bp":
                    s.bp = bad
            srcs[:] = [s.odo if x in (None, "wide", "empty", "bad_bp") else (None if x == "null" else x) for s, x in zip(S, srcs)]
        (A, sa, _), (Bp, sb, _) = pools
        st0 = [_store_state(s.bk, L.backend_default_params(s.variant)) for s in A]
        feats0 = [_feats(x) if x is not None else None for x in sa]
        _reset(A); _reset(Bp)
        ra, rb = _store_batch(A, sa), _store_solo(Bp, sb)
        assert ra == rb, (ra, rb)
        assert _all_counts(A) == _all_counts(Bp)
        codes = [r[0] for r in ra]
        assert codes == [0, 0, 0, 0] + [L._binding.E_ARG] * 5 + [0], codes
        assert ra[3][1:] == (1, (0, 0, 0))                          # the empty sweep stores an empty keyframe
        nf0, nf1 = _store_solo_counts(Bp[1])
        assert 1.5 * nf0 * 48 >= 2 ** 20 and nf0 + nf1 > 1.5 * nf0, (nf0, nf1)    # tick 1 outgrew the arena tick 0 sized
        # the wide session's full cloud spans the wrap box at its leaf, and its store took the wide keys: one 32-bit chain per filtered
        # cloud with points (6 launches, a sort and a scan), then 6 launches, a sort and a scan more for each cloud redone wide
        import vg_adversarial as V
        wide_feats = sa[2].features_download()
        V.check_wrap_box(wide_feats[2], 0.001)
        k = sum(1 for x in wide_feats if len(x) > 0)
        launches, lib = _cnt(A[2].bk)
        redone = launches // 6 - k
        assert launches % 6 == 0 and redone >= 1 and lib == 2 * (k + redone), (launches, lib, k)
        for i, (a, b) in enumerate(zip(A, Bp)):
            bp = L.backend_default_params(a.variant)
            sa_ = _store_state(a.bk, bp)
            assert sa_ == _store_state(b.bk, bp), i
            if codes[i] != 0:                                      # an erroring session keeps its count and store
                assert a.bk.kf_count() == 1 and sa_ == st0[i], i
        assert [_feats(x) if x is not None else None for x in sa] == feats0     # no source changed
    finally:
        for S, srcs, _ in pools:
            for x in srcs:
                if x is not None and all(x is not s.odo for s in S):
                    x.close()
            _close(S)


def _store_solo_counts(s):
    """the full-cloud points of keyframes 0 and 1 of session s's store"""
    L = _L()
    return tuple(len(s.bk.global_map(L.KF_FULL, [k], [IDENT7], TINY_LEAF)) for k in (0, 1))


# ---------------------------------------------------------------- 3. aliasing: a backend as its own or another's source
def _alias_pool(v0, v):
    """s0 stores from its own backend; s1 from s2's backend; s2 and s3 from one shared source X"""
    S = [Sess(v0), Sess(v), Sess(v), Sess(v)]
    X = S[2].odo
    S[3].odo.close()
    S[3].odo = X
    srcs = [S[0].bk, S[2].bk, X, X]
    extractors = [(S[0].bk, v0), (S[2].bk, v), (X, v)]
    return S, srcs, extractors


@pytest.mark.parametrize("v0,v", [(0, 1), (1, 0)])
def test_aliased_sources_equal_solo_in_either_order(sweeps, v0, v):
    pools = [_alias_pool(v0, v) for _ in range(3)]               # batched, solo in session order, solo in reverse order
    try:
        for t in range(2):
            for S, srcs, ex in pools:
                for k, (c, var) in enumerate(ex):
                    _extract(c, var, sweeps[var][(k + t) % N_SWEEPS])
            feats = [[_feats(c) for c, _ in ex] for _, _, ex in pools]
            assert feats[0] == feats[1] == feats[2]
            for S, _, _ in pools:
                _reset(S)
            (A, sa, exa), (F, sf, _), (R, sr, _) = pools
            L = _L()
            st = L.undistort_resident_batch([c for c, _ in exa], [_motion(k, t)[0] for k in range(3)], [_motion(k, t)[1] for k in range(3)])
            assert list(st) == [0, 0, 0]
            for _, _, ex in pools[1:]:
                for k, (c, _) in enumerate(ex):
                    c.undistort_resident(*_motion(k, t))
            deskewed = [[_feats(c) for c, _ in ex] for _, _, ex in pools]
            assert deskewed[0] == deskewed[1] == deskewed[2] and deskewed[0] != feats[0]
            ra, rf, rr = _store_batch(A, sa), _store_solo(F, sf), _store_solo(R, sr, order=[3, 2, 1, 0])
            assert ra == rf == rr and all(r[:2] == (0, t) for r in ra), (ra, rf, rr)
            assert [[_feats(c) for c, _ in ex] for _, _, ex in pools] == deskewed          # the store reads its sources only
            counts = [[_cnt(c) for s in S for c in (s.odo, s.bk)] for S, _, _ in pools]
            assert counts[0] == counts[1] == counts[2]
        states = [[_store_state(s.bk, s.bp) for s in S] for S, _, _ in pools]
        assert states[0] == states[1] == states[2]
    finally:
        for S, _, _ in pools:
            S[3].odo = None
            for s in S:
                s.bk.close()
                if s.odo is not None and s.odo is not s.bk:
                    s.odo.close()


# ---------------------------------------------------------------- 4. caller streams
def test_caller_streams(sweeps):
    """caller streams (liliom_set_stream) on some backends and some sources, against the solo calls on the contexts' own streams"""
    import torch
    variants = [0, 1, 0, 1, 1]
    A, Bp = _pool(variants), _pool(variants)
    streams = [torch.cuda.Stream() for _ in range(4)]
    try:
        A[1].bk.set_stream(streams[0].cuda_stream)
        A[2].bk.set_stream(streams[1].cuda_stream)
        A[0].odo.set_stream(streams[2].cuda_stream)
        A[1].odo.set_stream(streams[3].cuda_stream)
        A[3].odo.set_stream(streams[3].cuda_stream)
        for t in range(2):
            _tick(A, Bp, sweeps, t)
        for s in A:
            s.odo.set_stream(None)
            s.bk.set_stream(None)
        for a, b in zip(A, Bp):
            assert _store_state(a.bk, a.bp) == _store_state(b.bk, b.bp)
    finally:
        _close(A, Bp)


# ---------------------------------------------------------------- 5. whole-call refusals change nothing
def _raw_kf(bks, bps, srcs, B=None, null=()):
    L = _L()
    B = len(bks) if B is None else B
    ids, st = np.full(max(B, 1), -7, np.int32), np.full(max(B, 1), -99, np.int32)
    a = dict(ctxs=L._binding._handles(bks), bps=(L.BackendParams * max(len(bps), 1))(*bps), srcs=L._binding._handles(srcs),
             kf_id=ids.ctypes.data_as(C.POINTER(C.c_int)), status=st.ctypes.data_as(C.POINTER(C.c_int)))
    for n in null:
        a[n] = None
    rc = L._binding.lib().liliom_kf_add_resident_batch(a["ctxs"], B, a["bps"], a["srcs"], a["kf_id"], None, None, None, a["status"])
    return rc, list(ids), list(st)


def _raw_undistort(cs, B=None, null=()):
    L = _L()
    B = len(cs) if B is None else B
    st = np.full(max(B, 1), -99, np.int32)
    t = np.zeros(3 * max(B, 1)) + 0.2
    q = np.tile(np.array(IDENT_Q), max(B, 1))
    a = dict(ctxs=L._binding._handles(cs), trans=t.ctypes.data_as(C.POINTER(C.c_double)), quat=q.ctypes.data_as(C.POINTER(C.c_double)),
             status=st.ctypes.data_as(C.POINTER(C.c_int)))
    for n in null:
        a[n] = None
    rc = L._binding.lib().liliom_undistort_resident_batch(a["ctxs"], B, a["trans"], a["quat"], a["status"])
    return rc, [0] * 3, list(st)


def test_whole_call_refusals_change_nothing(sweeps):
    L = _L()
    E_ARG = L._binding.E_ARG
    S = _pool([0, 1])
    lb = _loopback_ctx(1, "kfhb_refuse")
    try:
        for i, s in enumerate(S):
            _extract(s.odo, s.variant, sweeps[s.variant][i])
        assert all(r[0] == 0 for r in _store_solo(S))
        for i, s in enumerate(S):
            _extract(s.odo, s.variant, sweeps[s.variant][i + 1])
        bks, bps, odos = [s.bk for s in S], [s.bp for s in S], [s.odo for s in S]
        everyone = bks + odos + [lb]

        def state():
            return ([c.kf_count() for c in bks], [_feats(c) for c in odos], [_cnt(c) for c in everyone])

        cases = [
            ("kf: B = 0", lambda: _raw_kf(bks, bps, odos, B=0)),
            ("kf: B < 0", lambda: _raw_kf(bks, bps, odos, B=-1)),
            *[(f"kf: NULL {n}", lambda n=n: _raw_kf(bks, bps, odos, null=(n,))) for n in ("ctxs", "bps", "srcs", "kf_id", "status")],
            ("kf: NULL backend", lambda: _raw_kf([bks[0], None], bps, odos)),
            ("kf: repeated backend", lambda: _raw_kf([bks[0], bks[0]], [bps[0], bps[0]], odos[:1] * 2)),
            ("kf: backend with a communicator", lambda: _raw_kf([bks[1], lb], [bps[1], bps[1]], [odos[1], odos[1]])),
            ("undistort: B = 0", lambda: _raw_undistort(odos, B=0)),
            *[(f"undistort: NULL {n}", lambda n=n: _raw_undistort(odos, null=(n,))) for n in ("ctxs", "trans", "quat", "status")],
            ("undistort: NULL context", lambda: _raw_undistort([odos[0], None])),
            ("undistort: repeated context", lambda: _raw_undistort([odos[0], odos[0]])),
            ("undistort: context with a communicator", lambda: _raw_undistort([odos[0], lb])),
        ]
        for what, call in cases:
            s0 = state()
            rc, ids, st = call()
            assert rc == E_ARG, what
            assert all(x == -99 for x in st) and all(x in (-7, 0) for x in ids), what     # no output written
            assert state() == s0, what
        assert [r[1] for r in _store_batch(S)] == [1, 1]           # the stores still take keyframes
    finally:
        lb.close()
        _close(S)


# ---------------------------------------------------------------- 6. after a call history
@pytest.mark.parametrize("kind", ["48", "32"])
def test_after_a_call_history(sweeps, kind):
    """a seeded history of tests/history_ops.py's operations on a source and a backend; then both batched calls (beside a fresh
    session) give what they give on fresh contexts"""
    L = _L()
    variant = H.KINDS[kind]["variant"]
    ops = H.ops_of(kind)
    rng = np.random.default_rng(20261019 + variant)
    hist = [_ctx(variant), _ctx(variant)]                          # source, backend
    fresh = [_ctx(variant), _ctx(variant)]
    helpers = [Sess(1 - variant), Sess(1 - variant)]
    try:
        for c in hist:
            for k in rng.permutation(len(ops))[:14]:
                op = ops[k]
                x = "large" if "large" in op.inputs else next(iter(op.inputs))
                op.inputs[x](c)
        out = []
        for (src, bk), helper in zip((hist, fresh), helpers):
            bk.kf_clear()
            if variant == 1:
                src.set_ring_source(L.RING_ELEVATION)
                src.set_time_source(L.TIME_AZIMUTH)
            _extract(src, variant, sweeps[variant][0])
            _extract(helper.odo, helper.variant, sweeps[helper.variant][1])
            for c in (src, bk):
                c.counters(reset=True)
            t, q = _motion(1, 0)
            st = L.undistort_resident_batch([helper.odo, src], [(0.1, 0.2, 0.0), t], [IDENT_Q, q])
            r = [list(st), _feats(src), _cnt(src)]
            bp = L.backend_default_params(variant)
            ids, counts, st = L.kf_add_resident_batch([bk, helper.bk], [bp, helper.bp], [src, helper.odo])
            r += [list(st), list(ids), counts.tolist(), _cnt(bk), _store_state(bk, bp)]
            out.append(r)
        assert out[0] == out[1]
    finally:
        for c in hist + fresh:
            c.close()
        _close(helpers)
