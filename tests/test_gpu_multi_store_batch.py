"""The backend local map over keyframes of several stores, solo and batched (liliom_bmap_build_multi, _batch_multi), and the batched
multi-store loop closure (liliom_loop_align_batch_multi).

The solo call's contract is the merged store: a context D whose store replays every store's kf_add calls gives, through
liliom_bmap_build with the mapped list, the same counts, layers and window bytes; with every entry naming the caller, it is
liliom_bmap_build.  The batches' contract is the solo multi call: a batched pool against a twin pool of solo calls, byte for byte
(status, liliom_last_error, counts or loop results, layers, window bytes, launches and lib_launches).  Every world has a prior
store per point layout shared by all sessions of that layout, sessions listing their own keyframes beside it, and sessions that
list another session's caller as a store.  A store on another device is refused by the same check as the solo multi calls; it is
not exercised here, since it needs two devices."""
import ctypes as C
import os

import numpy as np
import pytest

import history_ops as H
from test_gpu_multi_store import IDENT, _b, _nudge, _resident

pytestmark = pytest.mark.gpu

N_KF = 16
N_PRIOR = 8
LOOP = dict(leaf=0.4, max_corr_dist=2.0, max_iter=40, trans_eps=1e-8, fit_eps=1e-8)


def _L():
    import liliom_b200 as L
    return L


def _err(c):
    return _L()._binding.lib().liliom_last_error(c._h).decode()


def _cnt(c):
    k = c.counters()
    return k.launches, k.lib_launches


def _layers(c):
    out = []
    for layer in (0, 1):
        try:
            out.append(_b(c.bmap_download(layer)))
        except _L().LiliomError as e:
            out.append(e.code)
    return out


def _searches(c, bp, ids, poses):
    """what the layers give the window searches of c's keyframes ids at poses: the counts, every correspondence, the blocks"""
    L = _L()
    try:
        ne, ns = c.backend_window_correspond(bp, ids, poses)
    except L.LiliomError as e:
        return [e.code]
    out = [ne.tolist(), ns.tolist()]
    for slot in range(len(ids)):
        out += [_b(x) for kind in (0, 1) for x in c.backend_window_corr(slot, kind)]
    for k in (0, 2):
        out.append(_b(c.backend_window_blocks(np.array([_nudge(p, k) for p in poses]))))
    return out


@pytest.fixture(scope="module")
def seqs():
    from liliom_b200 import synth
    return {0: synth.make_keyframe_sequence(N_KF, stride=48, seed=17), 1: synth.make_keyframe_sequence(N_KF, stride=32, seed=18)}


# ---------------------------------------------------------------- the merged store, self-reference, the oracle
class Merged:
    """three stores of different sizes, their stored clouds kept, and D replaying every store's kf_add, store after store"""

    def __init__(self, variant, sizes=(5, 7, 4), seeds=(3, 4, 5)):
        L = _L()
        from liliom_b200 import synth
        self.bp = L.backend_default_params(variant)
        self.stores = [L.Context(L.default_params(variant)) for _ in sizes]
        self.D = L.Context(L.default_params(variant))
        self.kfs, self.base = [], []
        for s, (n, seed) in enumerate(zip(sizes, seeds)):
            self.base.append(self.D.kf_count())
            kf = []
            for e, sf, p in synth.make_keyframe_sequence(n, stride=48 if variant == 0 else 32, seed=seed):
                _, eds, sds = self.stores[s].kf_add(self.bp, e, sf)
                self.D.kf_add(self.bp, e, sf, download=False)
                kf.append((eds, sds, p))
            self.kfs.append(kf)

    def d(self, entries):
        return [self.base[s] + i for s, i in entries]

    def close(self):
        for c in self.stores + [self.D]:
            c.close()


@pytest.fixture(scope="module", params=[0, 1], ids=["horizon_v0", "rot_v1"])
def merged(request):
    m = Merged(request.param)
    yield m
    m.close()


LISTS = ([(0, 1), (1, 0), (2, 3), (0, 1), (1, 6), (2, 3), (1, 2)],        # interleaved, repeated
         [(1, i) for i in range(7)] + [(0, i) for i in range(0, 5, 2)] + [(2, 0)],
         [(2, 1)], [])


def test_bmap_multi_equals_the_merged_store(merged, oracle):
    m = merged
    c = m.stores[1]
    win = [4, 5, 6]                                      # the caller's own window keyframes
    for entries in LISTS:
        poses = [_nudge(m.kfs[s][i][2], j) for j, (s, i) in enumerate(entries)]
        got = c.bmap_build_multi(m.bp, [m.stores[s] for s, _ in entries], [i for _, i in entries], poses)
        want = m.D.bmap_build(m.bp, m.d(entries), poses)
        assert got == want and _layers(c) == _layers(m.D), entries
        wp = [m.kfs[1][i][2] for i in win]
        assert _searches(c, m.bp, win, wp) == _searches(m.D, m.bp, m.d([(1, i) for i in win]), wp), entries
        if entries:
            dt = c.dtype
            cat = lambda l: np.concatenate([oracle.transform_cloud(m.kfs[s][i][l], p) for (s, i), p in zip(entries, poses)
                                            if len(m.kfs[s][i][l])] or [np.zeros(0, dt)])
            assert _layers(c) == [_b(oracle.voxelgrid(cat(0), m.bp.edge_leaf)), _b(oracle.voxelgrid(cat(1), m.bp.surf_leaf))]
    assert got == (0, 0)


def test_self_reference_is_bmap_build(merged):
    m = merged
    c = m.stores[1]
    ids = [0, 3, 3, 6, 1, 5]
    poses = [_nudge(m.kfs[1][i][2], j) for j, i in enumerate(ids)]
    c.counters(reset=True)
    a = c.bmap_build_multi(m.bp, [c] * len(ids), ids, poses)
    ca, la = _cnt(c), _layers(c)
    sa = _searches(c, m.bp, [4, 5, 6], [m.kfs[1][i][2] for i in (4, 5, 6)])
    c.counters(reset=True)
    b = c.bmap_build(m.bp, ids, poses)
    assert (a, ca, la) == (b, _cnt(c), _layers(c))
    assert sa == _searches(c, m.bp, [4, 5, 6], [m.kfs[1][i][2] for i in (4, 5, 6)])


# ---------------------------------------------------------------- tracking in a prior map
def test_a_restarted_session_tracks_in_its_prior_map():
    """Two runs of one seeded world whose start frames are 2 deg / 0.5 m apart.  loop_align_multi recovers the offset; a local map
    of the prior store's keyframes alone, placed by the recovered transform, gives the new session's keyframes window surf
    correspondences, and their blocks cost less at the recovered pose than at the offset one."""
    L = _L()
    from liliom_b200 import synth
    old = synth.make_keyframe_sequence(8, stride=48, seed=21)
    new = synth.make_keyframe_sequence(8, stride=48, seed=22)
    bp = L.backend_default_params(0)
    bp.q_lb[:] = [1.0, 0.0, 0.0, 0.0]                   # lidar = body: the window's poses are the keyframes' own
    bp.t_lb[:] = [0.0, 0.0, 0.0]
    A, B = L.Context(variant=0), L.Context(variant=0)
    try:
        for e, s, _ in old:
            A.kf_add(bp, e, s, download=False)
        for e, s, _ in new:
            B.kf_add(bp, e, s, download=False)
        T_off = np.concatenate([synth.q_from_axis_angle([0.2, -0.1, 1.0], np.deg2rad(2.0)), [0.35, -0.35, 0.1]])
        q_inv = T_off[:4] * np.array([1.0, -1.0, -1.0, -1.0])

        def compose(q, t, p):                           # (q, t) * p
            return np.concatenate([synth.qmul(q, p[:4]), synth.qrot(q, p[4:]) + t])
        in_new = lambda p: compose(q_inv, -synth.qrot(q_inv, T_off[4:]), p)
        tgt = [3, 4, 5, 6, 7]
        T, fit, conv, it, ns, nt = B.loop_align_multi([B], [5], [in_new(new[5][2])], [A] * len(tgt), tgt, [old[i][2] for i in tgt], 0.4,
                                                      max_corr_dist=2.0, max_iter=100)
        assert conv and np.linalg.norm(T[:3, 3] - T_off[4:]) < 0.05
        qT, tT = np.array(_quat(T[:3, :3])), T[:3, 3]
        qTi = qT * np.array([1.0, -1.0, -1.0, -1.0])
        # the prior keyframes in the new session's frame: T^-1 * pose
        placed = [compose(qTi, -synth.qrot(qTi, tT), old[i][2]) for i in range(8)]
        ne_map, ns_map = B.bmap_build_multi(bp, [A] * 8, list(range(8)), placed)
        assert ne_map > 0 and ns_map > 50
        win = [4, 5, 6]
        here = [in_new(new[i][2]) for i in win]
        ne, ns = B.backend_window_correspond(bp, win, here)
        assert (ns > 0).all(), ns
        good = B.backend_window_blocks(np.array(here))
        off = B.backend_window_blocks(np.array([compose(qT, tT, p) for p in here]))
        assert good[:, 1, 27].sum() < off[:, 1, 27].sum(), (good[:, 1, 27], off[:, 1, 27])
    finally:
        A.close()
        B.close()


def _quat(R):
    """wxyz of a rotation matrix (trace > 0 here: small rotations)"""
    w = np.sqrt(max(0.0, 1.0 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    return w, (R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w)


# ---------------------------------------------------------------- batched pools against solo twins
class World:
    """one pool: a prior store per layout (N_PRIOR keyframes) shared by every session of that layout, and sessions, each a backend
    context with a store of its own"""

    def __init__(self, seqs, variants, extra=None):
        L = _L()
        self.seqs, self.variants = seqs, list(variants)
        self.bp = [L.backend_default_params(v) for v in variants]
        self.prior = {v: L.Context(L.default_params(v)) for v in (0, 1)}
        for v, c in self.prior.items():
            for e, s, _ in seqs[v][:N_PRIOR]:
                c.kf_add(L.backend_default_params(v), e, s, download=False)
        self.S = [L.Context(L.default_params(v)) for v in variants]
        self.own = []
        for i, (c, v) in enumerate(zip(self.S, variants)):
            poses = []
            for j in range(4 + i % 3):
                e, s, p = seqs[v][(N_PRIOR + 2 * i + j) % N_KF]
                c.kf_add(self.bp[i], e, s, download=False)
                poses.append(p)
            self.own.append(poses)
        self.extra = extra(self) if extra else {}

    def resolve(self, i, ent):
        """(store, id, pose) of session i's entry: ("o", j) its own keyframe j, ("p", j) the prior store's, ("s", m, j) session m's"""
        if ent[0] == "o":
            return self.S[i], ent[1], self.own[i][ent[1]]
        if ent[0] == "p":
            return self.prior[self.variants[i]], ent[1], self.seqs[self.variants[i]][ent[1]][2]
        return self.S[ent[1]], ent[2], self.own[ent[1]][ent[2]]

    def entries(self, i, t, small=False):
        rng = np.random.default_rng(1000 * i + t)
        if i % 7 == 3:
            return []
        n = len(self.own[i])
        ents = [("o", int(j)) for j in rng.integers(0, n, 1 if small else 3)]
        ents += [("p", int(j)) for j in rng.integers(0, N_PRIOR, 1 if small else 4)]
        same = [m for m in range(len(self.S)) if m != i and self.variants[m] == self.variants[i]]
        if same and i % 2 == 0:
            m = same[int(rng.integers(len(same)))]
            ents.append(("s", m, int(rng.integers(0, len(self.own[m])))))
        return [ents[j] for j in rng.permutation(len(ents))]

    def lists(self, ents_of, t):
        """per session (stores, ids, poses) of the entries, poses nudged by session, tick and place"""
        out = []
        for i, ents in enumerate(ents_of):
            r = [self.resolve(i, e) for e in ents]
            out.append(([x[0] for x in r], np.array([x[1] for x in r], np.int32),
                        np.array([_nudge(x[2], 1 + (i + t + j) % 5) for j, x in enumerate(r)]).reshape(-1, 7)))
        return out

    def window(self, i):
        n = len(self.own[i])
        return list(range(n - 3, n)), self.own[i][n - 3:]

    def close(self):
        for c in self.S + list(self.prior.values()) + [c for c in self.extra.values() if hasattr(c, "close")]:
            c.close()


def _handles(cs):
    return (C.c_void_p * max(len(cs), 1))(*[None if c is None else c._h for c in cs])


def _bmap_solo(W, lists, bps=None):
    L = _L()
    out = []
    for i, (st, ids, poses) in enumerate(lists):
        bp = (bps or W.bp)[i]
        ne, ns = C.c_int(-7), C.c_int(-7)
        p = np.ascontiguousarray(poses).reshape(-1)
        rc = L._binding.lib().liliom_bmap_build_multi(W.S[i]._h, C.byref(bp), None if st is None else _handles(st),
                                                      ids.ctypes.data_as(C.POINTER(C.c_int)), p.ctypes.data_as(C.POINTER(C.c_double)),
                                                      len(ids), C.byref(ne), C.byref(ns))
        out.append((rc, (ne.value, ns.value) if rc == 0 else None, _err(W.S[i])))
    return out


def _bmap_batch(W, lists, bps=None, k=None):
    L = _L()
    B = len(W.S)
    P_i, P_d, P_v = C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.c_void_p)
    keep = [None if st is None else _handles(st) for st, _, _ in lists]
    stores = (P_v * B)(*[P_v() if h is None else C.cast(h, P_v) for h in keep])
    ids = (P_i * B)(*[P_i() if x[1] is None else x[1].ctypes.data_as(P_i) for x in lists])
    pk = [None if x[2] is None else np.ascontiguousarray(x[2]).reshape(-1) for x in lists]
    poses = (P_d * B)(*[P_d() if p is None else p.ctypes.data_as(P_d) for p in pk])
    ks = np.array(k if k is not None else [len(x[1]) for x in lists], np.int32)
    ne, ns, st = np.full(B, -7, np.int32), np.full(B, -7, np.int32), np.full(B, -99, np.int32)
    rc = L._binding.lib().liliom_bmap_build_batch_multi(_handles(W.S), B, (L.BackendParams * B)(*(bps or W.bp)), stores, ids, poses,
                                                        ks.ctypes.data_as(P_i), ne.ctypes.data_as(P_i), ns.ctypes.data_as(P_i),
                                                        st.ctypes.data_as(P_i))
    assert rc == 0
    return [(int(st[i]), (int(ne[i]), int(ns[i])) if st[i] == 0 else None, _err(c)) for i, c in enumerate(W.S)]


def _state(W):
    return [(_cnt(c), _layers(c)) for c in W.S]


def _bmap_both(A, Bw, la, lb, bps=(None, None), searches=True):
    for W in (A, Bw):
        for c in W.S:
            c.counters(reset=True)
    ra, rb = _bmap_batch(A, la, bps[0]), _bmap_solo(Bw, lb, bps[1])
    assert ra == rb, (ra, rb)
    assert _state(A) == _state(Bw)
    if searches:
        for i in range(len(A.S)):
            wa, wb = A.window(i), Bw.window(i)
            assert _searches(A.S[i], A.bp[i], *wa) == _searches(Bw.S[i], Bw.bp[i], *wb), i
    return ra


def _loop_lists(W, t):
    """session i aligns its latest keyframe (nudged) to the prior store's keyframes and its own earlier ones; every seventh session
    lists its own store only"""
    src, tgt = [], []
    for i in range(len(W.S)):
        n = len(W.own[i])
        src.append([("o", n - 1)])
        rng = np.random.default_rng(7 * i + t)
        own_only = i % 7 == 5
        tgt.append([("o", j) for j in range(n - 1)] + ([] if own_only else [("p", int(j)) for j in rng.integers(0, N_PRIOR, 3)]))
    return W.lists(src, t), W.lists(tgt, t + 1)


def _loop_solo(W, src, tgt, prm):
    L = _L()
    out = []
    for i, ((ss, si, sp), (ts, ti, tp)) in enumerate(zip(src, tgt)):
        T = np.zeros(16)
        f, cv, it, ns, nt = C.c_double(), C.c_int(), C.c_int(), C.c_int(), C.c_int()
        P_i, P_d = C.POINTER(C.c_int), C.POINTER(C.c_double)
        spf, tpf = np.ascontiguousarray(sp).reshape(-1), np.ascontiguousarray(tp).reshape(-1)
        p = prm[i]
        rc = L._binding.lib().liliom_loop_align_multi(W.S[i]._h, None if ss is None else _handles(ss), si.ctypes.data_as(P_i),
                                                      spf.ctypes.data_as(P_d), len(si), None if ts is None else _handles(ts),
                                                      ti.ctypes.data_as(P_i), tpf.ctypes.data_as(P_d), len(ti), p["leaf"], p["max_corr_dist"],
                                                      p["max_iter"], p["trans_eps"], p["fit_eps"], T.ctypes.data_as(P_d), C.byref(f),
                                                      C.byref(cv), C.byref(it), C.byref(ns), C.byref(nt))
        out.append((rc, (_b(T), f.value, cv.value, it.value, ns.value, nt.value) if rc == 0 else None, _err(W.S[i])))
    return out


def _loop_batch(W, src, tgt, prm):
    L = _L()
    B = len(W.S)
    P_i, P_d, P_v = C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.c_void_p)
    keep = [[None if x[0] is None else _handles(x[0]) for x in l] for l in (src, tgt)]
    st = [(P_v * B)(*[P_v() if h is None else C.cast(h, P_v) for h in k]) for k in keep]
    flat = [[np.ascontiguousarray(x[2]).reshape(-1) for x in l] for l in (src, tgt)]
    ids = [(P_i * B)(*[x[1].ctypes.data_as(P_i) for x in l]) for l in (src, tgt)]
    poses = [(P_d * B)(*[p.ctypes.data_as(P_d) for p in f]) for f in flat]
    ks = [np.array([len(x[1]) for x in l], np.int32) for l in (src, tgt)]
    prms = (L.LoopParams * B)(*[L.LoopParams(**p) for p in prm])
    res = (L.LoopResult * B)()
    status = np.full(B, -99, np.int32)
    rc = L._binding.lib().liliom_loop_align_batch_multi(_handles(W.S), B, st[0], ids[0], poses[0], ks[0].ctypes.data_as(P_i), st[1], ids[1],
                                                        poses[1], ks[1].ctypes.data_as(P_i), prms, res, status.ctypes.data_as(P_i))
    assert rc == 0
    out = []
    for i, r in enumerate(res):
        T = np.array(r.T16[:], np.float64)
        out.append((int(status[i]), (_b(T), r.fitness, r.converged, r.iters, r.n_src, r.n_tgt) if status[i] == 0 else None, _err(W.S[i])))
    return out


def _loop_both(A, Bw, t, prm=None, edit=None):
    sa, ta = _loop_lists(A, t)
    sb, tb = _loop_lists(Bw, t)
    prm = prm or [dict(LOOP) for _ in A.S]
    if edit:
        edit(A, sa, ta)
        edit(Bw, sb, tb)
    for W in (A, Bw):
        for c in W.S:
            c.counters(reset=True)
    ra, rb = _loop_batch(A, sa, ta, prm), _loop_solo(Bw, sb, tb, prm)
    assert ra == rb, [(i, x, y) for i, (x, y) in enumerate(zip(ra, rb)) if x != y]
    assert [_cnt(c) for c in A.S] == [_cnt(c) for c in Bw.S]
    return ra


def _twins(seqs, variants, extra=None):
    return World(seqs, variants, extra), World(seqs, variants, extra)


@pytest.mark.parametrize("B", [1, 2, 5, 33])
def test_batches_equal_solo_multi_calls(seqs, B):
    """Horizon / variant 0 and ROT / variant 1 sessions mixed, each listing its own keyframes, the shared prior store of its layout
    and another session's store: large lists, small lists, large again; then the loop closures"""
    variants = [i % 2 for i in range(B)] if B > 1 else [0]
    A, Bw = _twins(seqs, variants)
    try:
        for t, small in enumerate([False, True, False]):
            ents = [A.entries(i, t, small) for i in range(B)]
            r = _bmap_both(A, Bw, A.lists(ents, t), Bw.lists(ents, t), searches=(t != 1 or B <= 5))
            assert all(x[0] == 0 for x in r) and all(x[1][1] > 0 for i, x in enumerate(r) if ents[i]), r
        for t in range(2):
            r = _loop_both(A, Bw, t)
            assert all(x[0] == 0 and x[1][4] > 0 and x[1][5] > 0 for x in r), r
    finally:
        A.close()
        Bw.close()


def test_own_store_only_equals_the_single_store_batches(seqs):
    """every session listing only its own store: bmap_build_batch_multi is bmap_build_batch, loop_align_batch_multi is
    loop_align_batch"""
    L = _L()
    A, Bw = _twins(seqs, [0, 1, 1, 0, 1])
    try:
        ents = [[("o", j) for j in (2, 0, 1, 2)] for _ in A.S]
        la, lb = A.lists(ents, 0), Bw.lists(ents, 0)
        for W in (A, Bw):
            for c in W.S:
                c.counters(reset=True)
        ra = _bmap_batch(A, la)
        cnt, st = L.bmap_build_batch(Bw.S, Bw.bp, [x[1] for x in lb], [x[2] for x in lb])
        assert [x[0] for x in ra] == list(st) == [0] * 5 and [x[1] for x in ra] == [tuple(x) for x in cnt.tolist()]
        assert _state(A) == _state(Bw)
        n = [len(o) for o in A.own]
        sa = A.lists([[("o", n[i] - 1)] for i in range(5)], 0)
        ta = A.lists([[("o", j) for j in range(n[i] - 1)] for i in range(5)], 1)
        ra = _loop_batch(A, sa, ta, [dict(LOOP)] * 5)
        rb, st = L.loop_align_batch(Bw.S, [x[1] for x in sa], [x[2] for x in sa], [x[1] for x in ta], [x[2] for x in ta], [dict(LOOP)] * 5)
        assert [x[0] for x in ra] == list(st) == [0] * 5
        assert [x[1] for x in ra] == [(_b(T), f, int(cv), it, ns, nt) for T, f, cv, it, ns, nt in rb]
        assert [_cnt(c) for c in A.S] == [_cnt(c) for c in Bw.S]
    finally:
        A.close()
        Bw.close()


# ---------------------------------------------------------------- per-session errors beside good sessions
def _loopback_ctx(variant, group):
    os.environ["LILIOM_TEST_LOOPBACK"] = f"{group}:0/2"
    try:
        return _L().Context(_L().default_params(variant))
    finally:
        os.environ.pop("LILIOM_TEST_LOOPBACK", None)


def _far_stores(W):
    """stores holding one keyframe far away: its surf (far_s) or edge (far_e) layer needs more than 2^29 cells"""
    L = _L()
    out = {}
    for name, keep in (("far_s", 1), ("far_e", 0)):
        c = L.Context(L.default_params(0))
        e, sf, p = W.seqs[0][0]
        c.kf_add(L.backend_default_params(0), e if keep == 0 else e[:0], sf if keep == 1 else sf[:0], download=False)
        far = np.array(p); far[4] += 3.0e4; far[5] += 3.0e4
        out[name], out[name + "_pose"] = c, far
    out["other"] = L.Context(L.default_params(1))       # another point_stride
    out["other"].kf_add(L.backend_default_params(1), W.seqs[1][0][0], W.seqs[1][0][1], download=False)
    return out


def test_per_session_errors_beside_good_sessions(seqs):
    L = _L()
    variants = [0, 0, 0, 0, 0, 0, 0, 0, 0, 1]
    A, Bw = _twins(seqs, variants, _far_stores)
    lbs = [_loopback_ctx(0, f"msb_err_{n}") for n in range(2)]
    try:
        ents = [A.entries(i, 0) or [("o", 0)] for i in range(10)]
        _bmap_both(A, Bw, A.lists(ents, 0), Bw.lists(ents, 0), searches=False)       # every session has layers
        before = _state(A)

        def broken(W, lb):
            ls = W.lists(ents, 1)
            x = W.extra
            ls[1] = (None, ls[1][1], ls[1][2])                                         # NULL store list
            ls[2] = ([None] + ls[2][0][1:], ls[2][1], ls[2][2])                        # a NULL store
            ls[3] = ([x["other"]] + ls[3][0][1:], ls[3][1], ls[3][2])                  # a store of the other stride
            ls[4] = ([lb] + ls[4][0][1:], ls[4][1], ls[4][2])                          # a store with a communicator
            ls[5] = (ls[5][0], np.array([99] + list(ls[5][1][1:]), np.int32), ls[5][2])       # an unknown id
            for i, name in ((7, "far_s"), (8, "far_e")):                                # LILIOM_E_GRID on the surf / edge layer
                ls[i] = (ls[i][0] + [x[name]], np.append(ls[i][1], 0).astype(np.int32), np.vstack([ls[i][2], x[name + "_pose"]]))
            return ls
        la, lb = broken(A, lbs[0]), broken(Bw, lbs[1])
        bad = L.backend_default_params(0)
        bad.edge_leaf = 0.0
        bps_a, bps_b = list(A.bp), list(Bw.bp)
        bps_a[6] = bps_b[6] = bad                                                      # an invalid bp
        # k < 0 beside: the solo call sees k = -1 through its pose count
        r = _bmap_both(A, Bw, la, lb, (bps_a, bps_b), searches=False)
        E_ARG, E_GRID = L._binding.E_ARG, L._binding.E_GRID
        assert [x[0] for x in r] == [0, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, E_GRID, E_GRID, 0], r
        assert "store of entry 0 is NULL" in r[2][2] and "point_stride" in r[3][2] and "communicator" in r[4][2]
        assert "unknown keyframe id 99" in r[5][2] and "2^29" in r[7][2] and "2^29" in r[8][2], r
        assert [s[1] for s in _state(A)[1:7]] == [s[1] for s in before[1:7]]           # refused: the previous layers stay
        # k < 0
        ks = [len(x[1]) for x in la]
        ks[0] = -1
        ra = _bmap_batch(A, la, bps_a, k=ks)
        assert ra[0][0] == E_ARG and ra[9][0] == 0
        # the loop closure's session errors beside good sessions
        def edit(W, src, tgt, lb=None):
            x = W.extra
            src[1] = (None, src[1][1], src[1][2])
            tgt[2] = ([x["other"]] + tgt[2][0][1:], tgt[2][1], tgt[2][2])
            tgt[3] = (tgt[3][0], np.array([77] + list(tgt[3][1][1:]), np.int32), tgt[3][2])
            tgt[4] = ([lbs[0] if W is A else lbs[1]] + tgt[4][0][1:], tgt[4][1], tgt[4][2])
        prm = [dict(LOOP) for _ in range(10)]
        prm[5]["leaf"] = 0.0
        r = _loop_both(A, Bw, 2, prm, edit)
        assert [x[0] for x in r] == [0, E_ARG, E_ARG, E_ARG, E_ARG, E_ARG, 0, 0, 0, 0], r
        _bmap_both(A, Bw, A.lists(ents, 3), Bw.lists(ents, 3))                          # and every session builds again
    finally:
        for c in lbs:
            c.close()
        A.close()
        Bw.close()


# ---------------------------------------------------------------- wide keys
def _wide_store(W):
    """a store whose keyframe's edge cloud is the wrap box of tests/vg_adversarial.py at leaf 0.2, stored as received"""
    import vg_adversarial as V
    L = _L()
    c = L.Context(L.default_params(0))
    w = np.ascontiguousarray(V.wrap_order(leaf=0.2), c.dtype)
    bp = L.backend_default_params(0)
    bp.edge_leaf = 1e-4
    c.kf_add(bp, w, w[:0], download=False)
    return {"wide": c}


def test_wide_keys_session(seqs):
    A, Bw = _twins(seqs, [0, 0, 1], _wide_store)
    try:
        ents = [A.entries(i, 0) for i in range(3)]
        la, lb = A.lists(ents, 0), Bw.lists(ents, 0)
        for l, W in ((la, A), (lb, Bw)):                  # session 1's local map: the wide store's keyframe alone
            l[1] = ([W.extra["wide"]], np.array([0], np.int32), np.array([IDENT]))
        r = _bmap_both(A, Bw, la, lb)
        assert [x[0] for x in r] == [0, 0, 0]
        # its solo multi call's counters: the gather, the edge chain at 32-bit keys and again wide (6 launches, a sort and a scan
        # each), the edge grid's box and cell grid (5 launches, a sort and a scan); the surf layer is empty
        assert _cnt(A.S[1]) == (18, 6), _cnt(A.S[1])
    finally:
        A.close()
        Bw.close()


# ---------------------------------------------------------------- stores untouched, streams, whole-call refusals, history
def _store_state(st):
    """a store's keyframes: the count and every stored cloud (declined-leaf global map of surf, kf_cloud of edge + surf)"""
    L = _L()
    k = st.kf_count()
    return k, _b(st.global_map(L.KF_SURF, list(range(k)), [IDENT] * k, 1e-4)), _b(st.kf_cloud(list(range(k)), [IDENT] * k, 1e-4))


def test_stores_untouched_and_caller_streams(seqs):
    """every store's keyframes, a store's resident window and a store's resident odometry scan survive both batches; callers and
    the prior stores on streams of their own"""
    import torch
    L = _L()
    A, Bw = _twins(seqs, [0, 1, 0, 1, 0])
    streams = [torch.cuda.Stream() for _ in range(3)]
    try:
        stores = list(A.prior.values()) + A.S
        snaps = [_store_state(s) for s in stores]
        # a resident window on the ROT prior store and a resident scan on the Horizon prior store, and the same on their twins
        bp1 = L.backend_default_params(1)
        wpose = [seqs[1][i][2] for i in range(3)]
        for W in (A, Bw):
            W.prior[1].bmap_build(bp1, [0, 1, 2, 3], [seqs[1][i][2] for i in range(4)])
            W.prior[1].backend_window_correspond(bp1, [0, 1, 2], wpose)
            _resident(W.prior[0], 4)
        A.S[1].set_stream(streams[0].cuda_stream)
        A.S[2].set_stream(streams[1].cuda_stream)
        A.prior[0].set_stream(streams[2].cuda_stream)
        A.prior[1].set_stream(streams[1].cuda_stream)
        ents = [A.entries(i, 0) for i in range(5)]
        _bmap_both(A, Bw, A.lists(ents, 0), Bw.lists(ents, 0), searches=False)
        _loop_both(A, Bw, 0)
        ma, mb = A.prior[0].map_update_resident(IDENT), Bw.prior[0].map_update_resident(IDENT)
        assert ma == mb and ma > 0 and A.prior[0].map_download().tobytes() == Bw.prior[0].map_download().tobytes()
        bodies = np.array([_nudge(p, 1) for p in wpose])
        assert _b(A.prior[1].backend_window_blocks(bodies)) == _b(Bw.prior[1].backend_window_blocks(bodies))
        assert _layers(A.prior[1]) == _layers(Bw.prior[1])
        assert [_store_state(s) for s in stores] == snaps
    finally:
        for c in A.S + list(A.prior.values()):
            c.set_stream(None)
        A.close()
        Bw.close()


def test_whole_call_refusals_change_nothing(seqs):
    L = _L()
    W = World(seqs, [0, 1])
    lb = _loopback_ctx(1, "msb_refuse")
    try:
        ents = [W.entries(i, 0) for i in range(2)]
        ls = W.lists(ents, 0)
        assert [x[0] for x in _bmap_batch(W, ls)] == [0, 0]
        cs = W.S
        P_i, P_d, P_v = C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.c_void_p)
        keep = [_handles(x[0]) for x in ls]
        stores = (P_v * 2)(*[C.cast(h, P_v) for h in keep])
        ids = (P_i * 2)(*[x[1].ctypes.data_as(P_i) for x in ls])
        pk = [np.ascontiguousarray(x[2]).reshape(-1) for x in ls]
        poses = (P_d * 2)(*[p.ctypes.data_as(P_d) for p in pk])
        k = np.array([len(x[1]) for x in ls], np.int32)
        bps = (L.BackendParams * 2)(*W.bp)
        st = np.full(2, -99, np.int32)

        def call(ctxs, B=2, st_arr=stores):
            return L._binding.lib().liliom_bmap_build_batch_multi(_handles(ctxs), B, bps, st_arr, ids, poses, k.ctypes.data_as(P_i), None,
                                                                  None, st.ctypes.data_as(P_i))

        def loop_call(ctxs, s_arr=stores):
            res = (L.LoopResult * 2)()
            prm = (L.LoopParams * 2)(*[L.LoopParams(**LOOP)] * 2)
            return L._binding.lib().liliom_loop_align_batch_multi(_handles(ctxs), 2, s_arr, ids, poses, k.ctypes.data_as(P_i), stores, ids,
                                                                  poses, k.ctypes.data_as(P_i), prm, res, st.ctypes.data_as(P_i))
        state = lambda: (_state(W), [_err(c) for c in cs], _cnt(lb))
        s0 = state()
        for what, rc in [("B = 0", call(cs, B=0)), ("NULL stores", call(cs, st_arr=None)), ("repeated", call([cs[0], cs[0]])),
                         ("NULL context", call([cs[0], None])), ("communicator", call([cs[0], lb])),
                         ("loop NULL stores", loop_call(cs, s_arr=None)), ("loop repeated", loop_call([cs[1], cs[1]]))]:
            assert rc == L._binding.E_ARG, what
            assert (st == -99).all() and state() == s0, what
    finally:
        lb.close()
        W.close()


@pytest.mark.parametrize("kind", ["48", "32"])
def test_after_a_call_history(seqs, kind):
    """a seeded history of tests/history_ops.py's operations on a caller; then both batches give it a fresh caller's bytes"""
    L = _L()
    variant = H.KINDS[kind]["variant"]
    ops = H.ops_of(kind)
    rng = np.random.default_rng(20261018 + variant)
    W = World(seqs, [variant, 1 - variant])
    fresh = L.Context(L.default_params(variant))
    hist = H.make_ctx(kind)
    try:
        for k in rng.permutation(len(ops))[:14]:
            op = ops[k]
            x = "large" if "large" in op.inputs else next(iter(op.inputs))
            op.inputs[x](hist)
        ents = [[("p", 1), ("s", 0, 2), ("p", 5), ("p", 1)], W.entries(1, 0)]
        ls = W.lists(ents, 0)
        out = []
        for c in (hist, fresh):
            c.counters(reset=True)
            r, st = L.bmap_build_batch_multi([c, W.S[1]], W.bp, [x[0] for x in ls], [x[1] for x in ls], [x[2] for x in ls])
            res, st2 = L.loop_align_batch_multi([c, W.S[1]], [[W.S[0]], [W.S[1]]], [[3], [1]], [W.own[0][3:4], W.own[1][1:2]],
                                                [[W.prior[variant]] * 3, [W.S[1]]], [[0, 1, 2], [0]],
                                                [[W.seqs[variant][i][2] for i in range(3)], W.own[1][:1]], [LOOP, LOOP])
            out.append([r[0].tolist(), int(st[0]), _layers(c), _b(res[0][0]), res[0][1:], int(st2[0]), _cnt(c)])
        assert out[0] == out[1]
    finally:
        hist.close()
        fresh.close()
        W.close()
