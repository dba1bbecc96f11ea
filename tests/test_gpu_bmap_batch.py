"""The backend local map of many sessions in one call (liliom_bmap_build_batch) against each session's solo liliom_bmap_build,
byte for byte.

Every case builds a pool of sessions twice, each session a backend context with a keyframe store of its own: one pool goes
through the batched call, its twin through the solo calls, with the same lists and poses.  Compared: statuses, liliom_last_error,
counts, launches and lib_launches, both downloaded layers, and what the layers give every later search: the correspondences of
liliom_backend_window_correspond and the blocks of liliom_backend_window_blocks on each pool."""
import ctypes as C
import os

import numpy as np
import pytest

import history_ops as H

pytestmark = pytest.mark.gpu

N_KF = 12
IDENT7 = np.array([1.0, 0, 0, 0, 0, 0, 0])


def _L():
    import liliom_b200 as L
    return L


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def _last_error(c):
    return _L()._binding.lib().liliom_last_error(c._h).decode()


def _cnt(c):
    k = c.counters()
    return k.launches, k.lib_launches


def _nudge(pose, k):
    """a small, deterministic pose change: the pose an optimiser left the keyframe at on tick k"""
    from liliom_b200 import synth
    dq = synth.q_from_axis_angle([1, -1, 2], np.deg2rad(0.15 * k))
    return np.concatenate([synth.qmul(pose[:4], dq), pose[4:] + 0.01 * k * np.array([1.0, -0.5, 0.25])])


def _cat(parts, dtype):
    parts = [p for p in parts if len(p)]
    return np.concatenate(parts) if parts else np.zeros(0, dtype)


@pytest.fixture(scope="module")
def seqs():
    from liliom_b200 import synth
    return {0: synth.make_keyframe_sequence(N_KF, stride=48, seed=7), 1: synth.make_keyframe_sequence(N_KF, stride=32, seed=8)}


class Sess:
    """one session: a backend context, its variant and parameters, and its store (the stored (edge, surf) clouds and the poses
    the keyframes were taken at)"""

    def __init__(self, variant, bp=None):
        L = _L()
        self.variant = variant
        self.c = L.Context(L.default_params(variant))
        self.bp = bp if bp is not None else L.backend_default_params(variant)
        self.kfs, self.poses = [], []

    def add(self, e, s, pose, bp=None):
        kid, eds, sds = self.c.kf_add(self.bp if bp is None else bp, e, s)
        assert kid == len(self.kfs)
        self.kfs.append((eds, sds))
        self.poses.append(np.asarray(pose, np.float64))

    def store(self, seq, first, n):
        """n keyframes of the sequence from `first` on (wrapping): a store of the session's own"""
        for j in range(n):
            e, s, p = seq[(first + j) % len(seq)][:3]
            self.add(e, s, p)

    def close(self):
        self.c.close()


def _pool(seqs, variants):
    P = [Sess(v) for v in variants]
    for i, s in enumerate(P):
        s.store(seqs[s.variant], 3 * i, 6 + i % 5)
    return P


def _close(*pools):
    for P in pools:
        for s in P:
            s.close()


def _lists(S, t, small=False):
    """tick t's list of every session: unsorted ids with repeats (k = 0 for every seventh session), each keyframe's pose nudged by
    session and tick; small=True lists at most two keyframes"""
    out = []
    for i, s in enumerate(S):
        rng = np.random.default_rng(1000 * i + t)
        n = len(s.kfs)
        k = 0 if i % 7 == 3 else int(rng.integers(1, 3 if small else 2 * n + 1))
        ids = rng.integers(0, n, k).astype(np.int32)
        poses = np.array([_nudge(s.poses[j], 1 + i % 4 + t) for j in ids]).reshape(-1, 7)
        out.append((ids, poses, k))
    return out


def _ptr(a, ctype):
    return a.ctypes.data_as(C.POINTER(ctype)) if a is not None else None


def _batch(S, lists, bps=None):
    """one liliom_bmap_build_batch call; lists: per session (ids or None, poses or None, k).  Returns per session (status,
    counts or None, last_error)"""
    L = _L()
    B = len(S)
    bps = [s.bp for s in S] if bps is None else bps
    P_i, P_d = C.POINTER(C.c_int), C.POINTER(C.c_double)
    ids = (P_i * B)(*[_ptr(x[0], C.c_int) if x[0] is not None else P_i() for x in lists])
    k = np.array([x[2] for x in lists], np.int32)
    ne, ns, st = np.full(B, -7, np.int32), np.full(B, -7, np.int32), np.full(B, -99, np.int32)
    keep = [np.ascontiguousarray(x[1]).reshape(-1) if x[1] is not None else None for x in lists]
    poses = (P_d * B)(*[_ptr(a, C.c_double) if a is not None else P_d() for a in keep])
    rc = L._binding.lib().liliom_bmap_build_batch(L._binding._handles([s.c for s in S]), B, (L.BackendParams * B)(*bps), ids, poses,
                                                  _ptr(k, C.c_int), _ptr(ne, C.c_int), _ptr(ns, C.c_int), _ptr(st, C.c_int))
    assert rc == 0
    return [(int(st[i]), (int(ne[i]), int(ns[i])) if st[i] == 0 else None, _last_error(s.c)) for i, s in enumerate(S)]


def _solo(S, lists, bps=None):
    L = _L()
    bps = [s.bp for s in S] if bps is None else bps
    out = []
    for s, bp, (ids, poses, k) in zip(S, bps, lists):
        ne, ns = C.c_int(-7), C.c_int(-7)
        p = np.ascontiguousarray(poses).reshape(-1) if poses is not None else None
        rc = L._binding.lib().liliom_bmap_build(s.c._h, C.byref(bp), _ptr(ids, C.c_int), _ptr(p, C.c_double), k, C.byref(ne), C.byref(ns))
        out.append((rc, (ne.value, ns.value) if rc == 0 else None, _last_error(s.c)))
    return out


def _layers(c):
    L = _L()
    out = []
    for layer in (0, 1):
        try:
            out.append(_bytes(c.bmap_download(layer)))
        except L.LiliomError as e:
            out.append(e.code)
    return out


def _searches(s):
    """what the layers give the window searches: the correspondences of the last three stored keyframes at their poses, every
    resident correspondence, and the blocks at those poses and at nudged ones"""
    L = _L()
    n = len(s.kfs)
    win = list(range(max(0, n - 3), n))
    poses = [s.poses[i] for i in win]
    try:
        ne, ns = s.c.backend_window_correspond(s.bp, win, poses)
    except L.LiliomError as e:
        return [e.code]
    out = [ne.tolist(), ns.tolist()]
    for slot in range(len(win)):
        out += [_bytes(x) for kind in (0, 1) for x in s.c.backend_window_corr(slot, kind)]
    for k in (0, 2):
        out.append(_bytes(s.c.backend_window_blocks(np.array([_nudge(p, k) for p in poses]))))
    return out


def _reset(S):
    for s in S:
        s.c.counters(reset=True)


def _call_both(A, Bp, lists, bps=None, searches=True):
    """the batch on A, the solo calls on Bp: everything they return and leave is the same"""
    _reset(A); _reset(Bp)
    ra, rb = _batch(A, lists, bps), _solo(Bp, lists, bps)
    assert ra == rb, (ra, rb)
    assert [_cnt(s.c) for s in A] == [_cnt(s.c) for s in Bp]
    assert [_layers(s.c) for s in A] == [_layers(s.c) for s in Bp]
    if searches:
        for i, (a, b) in enumerate(zip(A, Bp)):
            assert _searches(a) == _searches(b), i
    return ra


def _oracle_layers(O, s, ids, poses):
    dtype = s.c.dtype
    E = _cat([O.transform_cloud(s.kfs[i][0], p) for i, p in zip(ids, poses)], dtype)
    S_ = _cat([O.transform_cloud(s.kfs[i][1], p) for i, p in zip(ids, poses)], dtype)
    return [_bytes(O.voxelgrid(E, s.bp.edge_leaf)), _bytes(O.voxelgrid(S_, s.bp.surf_leaf))]


# ---------------------------------------------------------------- 1. B, mixed layouts, repeated calls
@pytest.mark.parametrize("B", [1, 2, 5, 33])
def test_batch_equals_solo(seqs, oracle, B):
    """B Horizon / variant 0 and ROT / variant 1 sessions mixed, each with its own store, list and poses: large lists, then small
    lists, then large again; one session of each layout against the oracle composition"""
    variants = [i % 2 for i in range(B)] if B > 1 else [0]
    A, Bp = _pool(seqs, variants), _pool(seqs, variants)
    try:
        for t, small in enumerate([False, True, False]):
            lists = _lists(A, t, small)
            r = _call_both(A, Bp, lists, searches=(t != 1 or B <= 5))
            assert all(x[0] == 0 for x in r), r
            assert all((x[1][1] > 0) if lists[i][2] > 0 else x[1] == (0, 0) for i, x in enumerate(r)), r
            if t == 0:
                for v in set(variants):
                    i = next(i for i, s in enumerate(A) if s.variant == v and lists[i][2] > 0)
                    ids, poses, _ = lists[i]
                    assert _layers(A[i].c) == _oracle_layers(oracle, A[i], ids, poses), (v, i)
    finally:
        _close(A, Bp)


# ---------------------------------------------------------------- 2. empty layers
def test_empty_layers(seqs):
    """keyframes without edge points, without surf points, k = 0, beside ordinary sessions; mixed layouts"""
    pools = []
    for _ in range(2):
        P = [Sess(0), Sess(1), Sess(0), Sess(1), Sess(0)]
        for i, s in enumerate(P):
            seq = seqs[s.variant]
            for j in range(4):
                e, sf, p = seq[(i + j) % N_KF][:3]
                if i in (1, 2):
                    e = e[:0]                                       # no edge points
                if i == 3:
                    sf = sf[:0]                                     # no surf points
                s.add(e, sf, p)
        pools.append(P)
    A, Bp = pools
    try:
        lists = _lists(A, 0)
        lists[3] = (np.array([2, 0, 2], np.int32), np.array([_nudge(A[3].poses[j], 1) for j in (2, 0, 2)]), 3)
        lists[2] = (np.zeros(0, np.int32), np.zeros((0, 7)), 0)
        lists[4] = (np.zeros(0, np.int32), None, 0)                  # k = 0 takes a NULL list
        r = _call_both(A, Bp, lists)
        assert [x[0] for x in r] == [0] * 5
        assert r[1][1][0] == 0 < r[1][1][1] and r[3][1][1] == 0 < r[3][1][0] and r[2][1] == r[4][1] == (0, 0), r
    finally:
        _close(A, Bp)


# ---------------------------------------------------------------- 3. every per-session error beside good sessions
def _error_pools(seqs):
    L = _L()
    pools = []
    for _ in range(2):
        P = _pool(seqs, [0, 1, 0, 1, 0, 1, 0, 1, 0])
        # session 6: a surf-only keyframe far away: the surf layer's cell grid needs more than 2^29 cells (LILIOM_E_GRID after
        # the edge grid is built); session 7: an edge-only keyframe far away: the edge layer's grid fails before the surf box
        for i, keep in ((6, 1), (7, 0)):
            s = P[i]
            e, sf, p = seqs[s.variant][0][:3]
            far = np.array(p); far[4] += 3.0e4; far[5] += 3.0e4
            s.add(e if keep == 0 else e[:0], sf if keep == 1 else sf[:0], far)
        pools.append(P)
    bad = L.backend_default_params(0)
    bad.edge_leaf = 0.0
    return pools, bad


def test_per_session_errors_beside_good_sessions(seqs):
    L = _L()
    (A, Bp), bad = _error_pools(seqs)
    try:
        first = _lists(A, 0)
        _call_both(A, Bp, first, searches=False)                     # every session has layers: an unknown id keeps them
        before = [_layers(s.c) for s in A]
        lists = _lists(A, 1)
        lists[1] = (np.array([0, len(A[1].kfs)], np.int32), np.tile(IDENT7, (2, 1)), 2)        # unknown id
        lists[2] = (None, np.tile(IDENT7, (1, 1)), 1)                                          # NULL id list
        lists[3] = (np.array([0], np.int32), None, 1)                                          # NULL pose list
        lists[4] = (np.array([0], np.int32), np.tile(IDENT7, (1, 1)), -1)                      # k < 0
        for i in (6, 7):                                             # the far keyframe beside the first one
            n = len(A[i].kfs)
            lists[i] = (np.array([0, n - 1], np.int32), np.array([A[i].poses[0], A[i].poses[n - 1]]), 2)
        bps = [s.bp for s in A]
        bps[5] = bad                                                  # an invalid bp
        r = _call_both(A, Bp, lists, bps, searches=False)
        E_ARG, E_GRID = L._binding.E_ARG, L._binding.E_GRID
        assert [x[0] for x in r] == [0, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_GRID, E_GRID, 0], r
        assert "unknown keyframe id" in r[1][2] and "2^29" in r[6][2] and "2^29" in r[7][2], r
        # refused before anything changes: the previous layers stay downloadable; the grid errors come after the VoxelGrids
        assert [_layers(s.c) for s in A[1:6]] == before[1:6]
        assert [_layers(s.c) for s in A[6:8]] == [[L._binding.E_NOMAP] * 2] * 2
        for i, (a, b) in enumerate(zip(A, Bp)):
            assert _searches(a) == _searches(b), i
        _call_both(A, Bp, _lists(A, 2))                              # and every session builds again
    finally:
        _close(A, Bp)


# ---------------------------------------------------------------- 4. wide keys
def _wide_session():
    """a keyframe whose edge cloud is the wrap box of tests/vg_adversarial.py at leaf 0.2 (hundreds of kilometres of y), stored
    as received (a store leaf PCL declines): the local map's edge VoxelGrid at edge_leaf 0.2 needs wide keys"""
    import vg_adversarial as V
    L = _L()
    s = Sess(0)
    w = np.ascontiguousarray(V.wrap_order(leaf=0.2), s.c.dtype)
    store_bp = L.backend_default_params(0)
    store_bp.edge_leaf = 1e-4
    s.add(w, w[:0], IDENT7, store_bp)
    return s


def test_wide_keys_session(seqs):
    """a wide-keys session beside ordinary ones finishes on its solo path inside the call, with its solo call's counters"""
    import vg_adversarial as V
    pools = []
    for _ in range(2):
        P = _pool(seqs, [0, 1, 0])
        P.insert(1, _wide_session())
        pools.append(P)
    A, Bp = pools
    try:
        lists = _lists(A, 0)
        lists[1] = (np.array([0], np.int32), np.tile(IDENT7, (1, 1)), 1)
        r = _call_both(A, Bp, lists)
        assert [x[0] for x in r] == [0] * 4
        V.check_wrap_box(A[1].kfs[0][0], 0.2)                        # the stored cloud spans the wrap box at edge_leaf
        # gather, the edge chain at 32-bit keys and again wide (6 launches, a sort and a scan each), the edge grid's box and cell
        # grid (5 launches, a sort and a scan); the surf layer is empty
        assert _cnt(A[1].c) == (18, 6), _cnt(A[1].c)
    finally:
        _close(A, Bp)


# ---------------------------------------------------------------- 5. resident state on the context survives
def test_resident_scan_and_window_survive(seqs):
    """a resident odometry scan and a resident window: after the batch, liliom_map_update_resident and liliom_backend_window_blocks
    give what they give after the solo call"""
    from liliom_b200 import synth
    T0 = synth.default_true_pose()
    sws = []
    for k in range(2):
        T = np.array(T0); T[4] += 0.6 * k
        pts, q = synth.make_horizon_sweep(T, seed=1 + k)
        sws.append((pts, q, T, synth.perturbed_pose(T)))
    pools = []
    for _ in range(2):
        P = _pool(seqs, [0, 1, 0])
        s = P[0]
        for k, (pts, q, T, guess) in enumerate(sws):                 # scan 0 builds the odometry map, scan 1 stays resident
            s.c.upload_scan(pts)
            s.c.extract_resident(q)
            try:
                s.c.odometry_resident(guess, 4)
            except _L().LiliomError as e:
                assert k == 0 and e.code == _L()._binding.E_NOMAP
            if k == 0:
                s.c.map_update_resident(T)
        for t in P:                                                  # a resident window on every session
            t.c.bmap_build(t.bp, list(range(len(t.kfs))), t.poses)
            n = len(t.kfs)
            t.c.backend_window_correspond(t.bp, list(range(n - 3, n)), t.poses[n - 3:])
        pools.append(P)
    A, Bp = pools
    try:
        _call_both(A, Bp, _lists(A, 0), searches=False)
        for a, b in zip(A, Bp):                                      # the window the earlier correspond call left
            n = len(a.kfs)
            bodies = np.array([_nudge(p, 1) for p in a.poses[n - 3:]])
            assert _bytes(a.c.backend_window_blocks(bodies)) == _bytes(b.c.backend_window_blocks(bodies))
        ma, mb = A[0].c.map_update_resident(sws[1][2]), Bp[0].c.map_update_resident(sws[1][2])
        assert ma == mb and ma > 0
        assert A[0].c.map_download().tobytes() == Bp[0].c.map_download().tobytes()
        assert A[0].c.map_download_cloud().tobytes() == Bp[0].c.map_download_cloud().tobytes()
    finally:
        _close(A, Bp)


# ---------------------------------------------------------------- 6. caller streams
def test_caller_streams(seqs):
    import torch
    variants = [0, 1, 0, 1, 1]
    A, Bp = _pool(seqs, variants), _pool(seqs, variants)
    streams = [torch.cuda.Stream() for _ in range(2)]
    try:
        A[1].c.set_stream(streams[0].cuda_stream)
        A[2].c.set_stream(streams[1].cuda_stream)
        A[4].c.set_stream(streams[1].cuda_stream)
        for t in range(2):
            _call_both(A, Bp, _lists(A, t))
    finally:
        for s in A:
            s.c.set_stream(None)
        _close(A, Bp)


# ---------------------------------------------------------------- 7. whole-call refusals change nothing
def _loopback_ctx(variant, group):
    """rank 0 of a two-rank loopback group (the single-GPU stand-in for a communicator, see test_gpu_sharded.py)"""
    os.environ["LILIOM_TEST_LOOPBACK"] = f"{group}:0/2"
    try:
        return _L().Context(_L().default_params(variant))
    finally:
        os.environ.pop("LILIOM_TEST_LOOPBACK", None)


def _raw(cs, bps, lists, B=None, null=()):
    L = _L()
    B = len(cs) if B is None else B
    n = max(len(cs), 1)
    P_i, P_d = C.POINTER(C.c_int), C.POINTER(C.c_double)
    keep = [np.ascontiguousarray(x[1]).reshape(-1) for x in lists]
    a = dict(ctxs=L._binding._handles(cs), bps=(L.BackendParams * n)(*bps), kf_ids=(P_i * n)(*[_ptr(x[0], C.c_int) for x in lists]),
             poses7=(P_d * n)(*[_ptr(p, C.c_double) for p in keep]))
    k = np.array([x[2] for x in lists], np.int32)
    a["k"] = _ptr(k, C.c_int)
    st = np.full(n, -99, np.int32)
    ne = np.full(n, -7, np.int32)
    a["status"] = _ptr(st, C.c_int)
    for m in null:
        a[m] = None
    rc = L._binding.lib().liliom_bmap_build_batch(a["ctxs"], B, a["bps"], a["kf_ids"], a["poses7"], a["k"], _ptr(ne, C.c_int), None,
                                                  a["status"])
    return rc, list(st), list(ne)


def test_whole_call_refusals_change_nothing(seqs):
    L = _L()
    S = _pool(seqs, [0, 1])
    lb = _loopback_ctx(1, "bmapb_refuse")
    try:
        lists = _lists(S, 0)
        assert [x[0] for x in _batch(S, lists)] == [0, 0]
        cs, bps = [s.c for s in S], [s.bp for s in S]
        everyone = cs + [lb]

        def state():
            return [_layers(c) for c in cs], [_cnt(c) for c in everyone], [_last_error(c) for c in cs]

        other = _lists(S, 1)
        cases = [
            ("B = 0", lambda: _raw(cs, bps, other, B=0)),
            ("B < 0", lambda: _raw(cs, bps, other, B=-1)),
            *[(f"NULL {n}", lambda n=n: _raw(cs, bps, other, null=(n,))) for n in ("ctxs", "bps", "kf_ids", "poses7", "k", "status")],
            ("NULL context", lambda: _raw([cs[0], None], bps, other)),
            ("repeated context", lambda: _raw([cs[0], cs[0]], [bps[0], bps[0]], [other[0], other[0]])),
            ("context with a communicator", lambda: _raw([cs[1], lb], [bps[1], bps[1]], [other[1], (np.zeros(0, np.int32), np.zeros((0, 7)), 0)])),
        ]
        for what, call in cases:
            s0 = state()
            rc, st, ne = call()
            assert rc == L._binding.E_ARG, what
            assert all(x == -99 for x in st) and all(x == -7 for x in ne), what        # no output written
            assert state() == s0, what
        assert [x[0] for x in _batch(S, other)] == [0, 0]            # the contexts still build
    finally:
        lb.close()
        _close(S)


# ---------------------------------------------------------------- 8. after a call history
@pytest.mark.parametrize("kind", ["48", "32"])
def test_after_a_call_history(seqs, kind):
    """a seeded history of tests/history_ops.py's operations on a backend; then the batch (beside a fresh session of the other
    layout) gives what it gives on a fresh context"""
    variant = H.KINDS[kind]["variant"]
    ops = H.ops_of(kind)
    rng = np.random.default_rng(20261020 + variant)
    hist, fresh = Sess(variant), Sess(variant)
    helpers = [Sess(1 - variant), Sess(1 - variant)]
    try:
        for k in rng.permutation(len(ops))[:14]:
            op = ops[k]
            x = "large" if "large" in op.inputs else next(iter(op.inputs))
            op.inputs[x](hist.c)
        out = []
        for s, helper in zip((hist, fresh), helpers):
            s.c.kf_clear()
            s.kfs, s.poses = [], []
            s.store(seqs[variant], 2, 7)
            helper.store(seqs[1 - variant], 5, 6)
            lists = _lists([s, helper], 3)
            _reset([s, helper])
            r = _batch([s, helper], lists)
            # liliom_last_error is only written by a failing call: the history's own message stays behind a successful one
            out.append([[x[:2] for x in r], _cnt(s.c), _layers(s.c), _searches(s)])
        assert out[0] == out[1]
    finally:
        _close([hist, fresh], helpers)
