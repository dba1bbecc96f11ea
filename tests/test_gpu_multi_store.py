"""GPU tests of the calls over keyframes of several stores (liliom_global_map_multi, liliom_loop_align_multi).  Their contract is
the merged store: a context D whose store holds the same clouds (the same kf_add / kf_add_full calls replayed) gives, for the
mapped list, the same bytes through liliom_global_map / liliom_loop_align; with every entry naming the calling context, the
single-store call's bytes.  Also: the oracle's voxelgrid(concat(transform_cloud(...))), a relocalisation between two sessions of
one world, stores left byte-identical, refused calls that change nothing, an at-size fleet, and long call histories."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

IDENT = np.array([1.0, 0, 0, 0, 0, 0, 0])
TINY_LEAF = 1e-4          # PCL declines every keyframe-sized cloud at this leaf: the output is the transformed input
LOOP = dict(max_corr_dist=2.0, max_iter=60, trans_eps=1e-8, fit_eps=1e-8)


def _b(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def _nudge(pose, k):
    from liliom_b200 import synth
    dq = synth.q_from_axis_angle([1, -1, 2], np.deg2rad(0.15 * k))
    return np.concatenate([synth.qmul(pose[:4], dq), pose[4:] + 0.01 * k * np.array([1.0, -0.5, 0.25])])


class Fleet:
    """S stores built from seeded keyframe sequences (edge, surf and full clouds), and D: one context that replays every store's
    adds, store after store.  Entry (s, i) is keyframe i of store s, keyframe base[s] + i of D."""

    def __init__(self, stride, n_kf=6, seeds=(3, 4, 5), extra=None):
        import liliom_b200 as L
        from liliom_b200 import synth
        self.variant = 0 if stride == 48 else 1
        self.bp = L.backend_default_params(self.variant)
        self.seqs = [synth.make_keyframe_sequence(n_kf, stride=stride, seed=s, full=True) for s in seeds]
        self.stores = [L.Context(variant=self.variant) for _ in seeds]
        self.D = L.Context(variant=self.variant)
        self.full = [[] for _ in seeds]          # the stored full clouds (variant 1: VoxelGrid(surf_leaf) of the received ones)
        self.surf = [[] for _ in seeds]
        self.base = []
        for s, seq in enumerate(self.seqs):
            self.base.append(self.D.kf_count())
            for e, sf, _, f in seq:
                self.add(s, e, sf, f)
        if extra is not None:                    # one more keyframe in store 0 (and D, behind everything)
            self.extra_d = self.D.kf_count()
            self.add(0, *extra)

    def add(self, s, edge, surf, full):
        for c in (self.stores[s], self.D):
            kid, _, so = c.kf_add(self.bp, edge, surf)
            m = c.kf_add_full(self.bp, kid, full)
        self.surf[s].append(so)
        self.full[s].append(full if self.variant == 0 else None)
        return kid, m

    def d(self, entries):
        return [self.extra_d if (s, i) == (0, len(self.seqs[0])) else self.base[s] + i for s, i in entries]

    def ctxs(self, entries):
        return [self.stores[s] for s, _ in entries]

    def pose(self, s, i):
        return self.seqs[s][min(i, len(self.seqs[s]) - 1)][2]

    def close(self):
        for c in self.stores + [self.D]:
            c.close()


def _raw_gmap(c, kind, stores, ids, poses, leaf, pre7s=None, out=None, cap=0, null_stores=False):
    import liliom_b200 as L
    k = len(ids)
    ids = np.ascontiguousarray(ids, np.int32)
    p = np.ascontiguousarray(np.asarray(poses, np.float64).reshape(-1, 7)) if k else np.zeros((1, 7))
    pre = None if pre7s is None else np.ascontiguousarray(np.asarray(pre7s, np.float64).reshape(-1, 7))
    st = None if null_stores else (C.c_void_p * max(k, 1))(*[None if x is None else x._h for x in stores])
    n = C.c_int(-7)
    rc = L._binding.lib().liliom_global_map_multi(c._h, kind, st, ids.ctypes.data_as(C.POINTER(C.c_int)), p.ctypes.data_as(C.POINTER(C.c_double)),
                                                  k, None if pre is None else pre.ctypes.data_as(C.POINTER(C.c_double)), leaf,
                                                  None if out is None else out.ctypes.data_as(C.c_void_p), cap, C.byref(n))
    return rc, n.value


def _oracle_map(O, clouds, poses, leaf, dtype, pres=None):
    parts = []
    for j, (cl, p) in enumerate(zip(clouds, poses)):
        x = cl if pres is None else O.transform_cloud(cl, pres[j])
        if len(x):
            parts.append(O.transform_cloud(x, p))
    cat = np.concatenate(parts) if parts else np.zeros(0, dtype)
    return O.voxelgrid(cat, leaf), cat


@pytest.fixture(scope="module", params=[48, 32])
def fleet(request):
    f = Fleet(request.param)
    yield f
    f.close()


LISTS = ([(0, 1), (1, 0), (2, 3), (0, 1), (1, 5), (2, 3)],                 # interleaved, repeated
         [(2, i) for i in range(6)] + [(0, i) for i in range(0, 6, 2)],
         [(1, 4)])


@pytest.mark.parametrize("kind_name", ["FULL", "SURF"])
def test_global_map_equals_the_merged_store(fleet, kind_name, oracle):
    import liliom_b200 as L
    kind = getattr(L, f"KF_{kind_name}")
    c = fleet.stores[1]
    tbl = np.concatenate([np.array(fleet.bp.q_lb[:]), np.array(fleet.bp.t_lb[:])])
    for entries in LISTS:
        poses = [_nudge(fleet.pose(s, i), j) for j, (s, i) in enumerate(entries)]
        clouds = [(fleet.full if kind == L.KF_FULL else fleet.surf)[s][i] for s, i in entries]
        for leaf in (0.3, 0.4, TINY_LEAF):
            for pre in (None, tbl):
                got = c.global_map_multi(kind, fleet.ctxs(entries), [i for _, i in entries], poses, leaf, pre7s=pre)
                want = fleet.D.global_map(kind, fleet.d(entries), poses, leaf, pre7=pre)
                assert len(got) > 0 and _b(got) == _b(want), (entries, leaf, pre is None)
                if clouds[0] is not None:
                    o, cat = _oracle_map(oracle, clouds, poses, leaf, c.dtype, None if pre is None else [pre] * len(entries))
                    assert _b(got) == _b(cat if leaf == TINY_LEAF else o)
        # per-entry pre7s (each robot its own Tbl): the oracle, entry by entry
        pres = [tbl if s == 0 else np.concatenate([tbl[:4], tbl[4:] + 0.01 * s]) for s, _ in entries]
        got = c.global_map_multi(kind, fleet.ctxs(entries), [i for _, i in entries], poses, 0.3, pre7s=pres)
        if clouds[0] is not None:
            assert _b(got) == _b(_oracle_map(oracle, clouds, poses, 0.3, c.dtype, pres)[0])
        if len(set(s for s, _ in entries)) == 1:       # one robot: the single-store call with its Tbl
            assert _b(got) == _b(fleet.D.global_map(kind, fleet.d(entries), poses, 0.3, pre7=pres[0]))
    assert len(c.global_map_multi(kind, [], [], [], 0.3)) == 0


def test_size_query_capacity_and_edge_lists(fleet, oracle):
    import liliom_b200 as L
    c = fleet.stores[0]
    entries = LISTS[0]
    ids = [i for _, i in entries]
    poses = [fleet.pose(s, i) for s, i in entries]
    want = fleet.D.global_map(L.KF_FULL, fleet.d(entries), poses, 0.4)
    rc, n = _raw_gmap(c, L.KF_FULL, fleet.ctxs(entries), ids, poses, 0.4)
    assert (rc, n) == (L._binding.OK, len(want))
    out = np.zeros(len(want), c.dtype)
    assert _raw_gmap(c, L.KF_FULL, fleet.ctxs(entries), ids, poses, 0.4, out=out, cap=len(want) - 1)[0] == L._binding.E_CAPACITY
    assert _raw_gmap(c, L.KF_FULL, fleet.ctxs(entries), ids, poses, 0.4, out=out, cap=len(want)) == (L._binding.OK, len(want))
    assert _b(out) == _b(want)
    assert _raw_gmap(c, L.KF_FULL, [], [], [], 0.4) == (L._binding.OK, 0)


@pytest.mark.parametrize("stride", [48, 32])
def test_all_non_finite_keyframe_and_wrapping_index(stride, oracle):
    """a keyframe whose full cloud is all NaN and the wrap box of tests/vg_adversarial.py split over two stores: the voxel index
    wraps (wide keys) across the stores"""
    import liliom_b200 as L
    import vg_adversarial as V
    from liliom_b200 import synth
    seq = synth.make_keyframe_sequence(2, stride=stride, seed=9, full=True)
    bad = seq[0][3].copy()
    bad["x"][:] = np.nan
    w = V.wrap_order(leaf=0.4)
    w = np.ascontiguousarray(w if stride == 48 else V.to32(w))
    h = len(w) // 2
    f = Fleet(stride, n_kf=2, seeds=(9, 10), extra=(seq[0][0], seq[0][1], bad))
    bp0 = L.backend_default_params(0)                    # both layouts store the wrap cloud as received
    kid = {}
    for s, part in ((0, w[:h]), (1, w[h:])):
        for c in (f.stores[s], f.D):
            k, _, _ = c.kf_add(f.bp, part[:0], part[:0], download=False)
            c.kf_add_full(bp0, k, part)
            kid[(s, c is f.D)] = k
    try:
        c = f.stores[0]
        got = c.global_map_multi(L.KF_FULL, [f.stores[0], f.stores[1]], [kid[(0, False)], kid[(1, False)]], [IDENT, IDENT], 0.4)
        want = f.D.global_map(L.KF_FULL, [kid[(0, True)], kid[(1, True)]], [IDENT, IDENT], 0.4)
        assert len(got) > 0 and _b(got) == _b(want) and _b(got) == _b(oracle.voxelgrid(oracle.transform_cloud(w, IDENT), 0.4))
        e = [(0, 2), (1, 1)]                             # the all-NaN keyframe and an ordinary one
        got = c.global_map_multi(L.KF_FULL, f.ctxs(e), [2, 1], [IDENT, f.pose(1, 1)], 0.3)
        assert _b(got) == _b(f.D.global_map(L.KF_FULL, f.d(e), [IDENT, f.pose(1, 1)], 0.3))
        assert len(c.global_map_multi(L.KF_FULL, [c], [2], [IDENT], 0.3)) == 0
    finally:
        f.close()


def test_self_reference_is_the_single_store_call(fleet):
    import liliom_b200 as L
    c = fleet.stores[2]
    ids = [0, 3, 3, 5, 1]
    poses = [_nudge(fleet.pose(2, i), j) for j, i in enumerate(ids)]
    for kind in (L.KF_FULL, L.KF_SURF):
        for leaf in (0.3, TINY_LEAF):
            assert _b(c.global_map_multi(kind, [c] * 5, ids, poses, leaf)) == _b(c.global_map(kind, ids, poses, leaf))
    a = c.loop_align_multi([c], [5], [fleet.pose(2, 5)], [c] * 3, [1, 2, 3], [fleet.pose(2, i) for i in (1, 2, 3)], 0.4, **LOOP)
    b = c.loop_align(*([5], [fleet.pose(2, 5)], [1, 2, 3], [fleet.pose(2, i) for i in (1, 2, 3)]), 0.4, **LOOP)
    assert _b(a[0]) == _b(b[0]) and a[1:] == b[1:]


def test_loop_align_equals_the_merged_store(fleet):
    for src, tgt in (([(0, 5)], [(1, 3), (0, 4), (2, 4), (1, 4)]), ([(2, 1), (0, 1)], [(0, 0), (1, 1), (0, 2)])):
        sp = [_nudge(fleet.pose(s, i), 1) for s, i in src]
        tp = [fleet.pose(s, i) for s, i in tgt]
        for leaf in (0.3, 0.4):
            a = fleet.stores[0].loop_align_multi(fleet.ctxs(src), [i for _, i in src], sp, fleet.ctxs(tgt), [i for _, i in tgt], tp, leaf, **LOOP)
            b = fleet.D.loop_align(fleet.d(src), sp, fleet.d(tgt), tp, leaf, **LOOP)
            assert _b(a[0]) == _b(b[0]) and a[1:] == b[1:], (src, leaf)
            assert a[4] > 0 and a[5] > 0


def test_restarted_session_recovers_the_offset():
    """Two sessions of one seeded world whose start frames are 2 deg / 0.5 m apart.  The new session lists the old store's poses
    in its own frame (here: the old frame taken as its own, the offset unknown) and aligns its latest keyframe to them: the ICP
    returns the offset between the frames."""
    import liliom_b200 as L
    from liliom_b200 import synth
    old = synth.make_keyframe_sequence(8, stride=48, seed=21)
    new = synth.make_keyframe_sequence(8, stride=48, seed=22)
    bp = L.backend_default_params(0)
    A, B = L.Context(variant=0), L.Context(variant=0)
    try:
        for e, s, _ in old:
            A.kf_add(bp, e, s, download=False)
        for e, s, _ in new:
            B.kf_add(bp, e, s, download=False)
        T_off = np.concatenate([synth.q_from_axis_angle([0.2, -0.1, 1.0], np.deg2rad(2.0)), [0.35, -0.35, 0.1]])   # 0.5 m
        q_inv = T_off[:4] * np.array([1.0, -1.0, -1.0, -1.0])

        def in_new(p):              # T_off^-1 * p
            t = synth._rotate_many(np.broadcast_to(q_inv, (1, 4)), (p[4:] - T_off[4:])[None])[0]
            return np.concatenate([synth.qmul(q_inv, p[:4]), t])
        j = 5
        src_pose = in_new(new[j][2])                      # the new session's own estimate of its keyframe j
        tgt = [3, 4, 5, 6, 7]
        tp = [old[i][2] for i in tgt]                     # the old store's poses, taken as they are
        T, fit, conv, it, ns, nt = A.loop_align_multi([B], [j], [src_pose], [A] * len(tgt), tgt, tp, 0.4, max_corr_dist=2.0, max_iter=100)
        D = L.Context(variant=0)
        for e, s, _ in old + [new[j]]:
            D.kf_add(bp, e, s, download=False)
        want = D.loop_align([8], [src_pose], tgt, tp, 0.4, max_corr_dist=2.0, max_iter=100)
        D.close()
        assert _b(T) == _b(want[0]) and (fit, conv, it, ns, nt) == want[1:]
        w, x, y, z = T_off[:4]
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
        ang = np.degrees(np.arccos(np.clip((np.trace(T[:3, :3] @ R.T) - 1) / 2, -1, 1)))
        assert conv and ns > 0 and nt > 0
        assert np.linalg.norm(T[:3, 3] - T_off[4:]) < 0.05 and ang < 0.2, (T, ang)
    finally:
        A.close()
        B.close()


# ------------------------------------------------------------------------------------------ stores untouched, refused calls
def _snapshot(st, n_full=5):
    """everything a store holds that a multi call must not change: its keyframe count, every stored cloud (declined-leaf global
    maps; the first n_full keyframes have full clouds), its local map, its resident features"""
    import liliom_b200 as L
    k = st.kf_count()
    ids = list(range(k))
    snap = dict(n=k, full=_b(st.global_map(L.KF_FULL, ids[:n_full], [IDENT] * n_full, TINY_LEAF)),
                surf=_b(st.global_map(L.KF_SURF, ids, [IDENT] * k, TINY_LEAF)),
                cloud=_b(st.kf_cloud(ids, [IDENT] * k, TINY_LEAF)), bmap=[_b(st.bmap_download(l)) for l in (0, 1)])
    snap["feats"] = [_b(x) for x in st.features_download()]
    return snap


def _resident(st, i):
    """a resident scan (an odometry call) and resident features (an extraction) on st"""
    from liliom_b200 import synth
    m, _ = synth.make_map(30_000, seed=i)
    st.map_set_points(m)
    T = synth.default_true_pose()
    pts, q = synth.make_horizon_sweep(T, seed=40 + i)
    surf, _, _ = st.extract_horizon(pts, q)
    st.odometry(surf, synth.perturbed_pose(T), 4)
    st.extract_horizon(pts, q)


def test_stores_untouched_and_refusals_change_nothing():
    import liliom_b200 as L
    f = Fleet(48, n_kf=5, seeds=(31, 32, 33))
    other = L.Context(variant=1)                         # another point_stride
    try:
        for i, st in enumerate(f.stores):
            st.bmap_build(f.bp, [0, 1, 2], [f.pose(i, k) for k in range(3)])
        c = L.Context(variant=0)                         # the caller: its own store empty, a resident scan
        for i, st in enumerate(f.stores + [c]):
            _resident(st, i)
        kid, _, _ = f.stores[2].kf_add(f.bp, f.seqs[2][0][0], f.seqs[2][0][1], download=False)     # no full cloud
        snaps = [_snapshot(st) for st in f.stores]
        e = [(0, 1), (1, 0), (2, 3), (0, 1), (1, 4), (2, 3)]              # interleaved, repeated; ids of 5-keyframe stores
        ids, poses = [i for _, i in e], [f.pose(s, i) for s, i in e]
        T = C.c_double * 16
        refused = [
            ("NULL stores", lambda: _raw_gmap(c, L.KF_FULL, None, ids, poses, 0.3, null_stores=True)[0], L._binding.E_ARG),
            ("NULL store", lambda: _raw_gmap(c, L.KF_FULL, [None] + f.ctxs(e)[1:], ids, poses, 0.3)[0], L._binding.E_ARG),
            ("stride", lambda: _raw_gmap(c, L.KF_FULL, [other] + f.ctxs(e)[1:], ids, poses, 0.3)[0], L._binding.E_ARG),
            ("unknown id", lambda: _raw_gmap(c, L.KF_FULL, f.ctxs(e), [99] + ids[1:], poses, 0.3)[0], L._binding.E_ARG),
            ("negative id", lambda: _raw_gmap(c, L.KF_FULL, f.ctxs(e), [-1] + ids[1:], poses, 0.3)[0], L._binding.E_ARG),
            ("no full cloud", lambda: _raw_gmap(c, L.KF_FULL, [f.stores[2]], [kid], [IDENT], 0.3)[0], L._binding.E_ARG),
            ("leaf", lambda: _raw_gmap(c, L.KF_FULL, f.ctxs(e), ids, poses, 0.0)[0], L._binding.E_ARG),
            ("kind", lambda: _raw_gmap(c, 2, f.ctxs(e), ids, poses, 0.3)[0], L._binding.E_ARG),
        ]
        reps = (1 << 31) // len(f.full[0][0]) + 1
        refused.append(("2^31 points", lambda: _raw_gmap(c, L.KF_FULL, [f.stores[0]] * reps, np.zeros(reps, np.int32),
                                                         np.tile(IDENT, (reps, 1)), 0.3)[0], L._binding.E_CAPACITY))

        def loop_rc(ss, si, ts, ti, leaf=0.4, max_iter=10):
            k, m = len(si), len(ti)
            arr = lambda xs: None if xs is None else (C.c_void_p * max(len(xs), 1))(*[None if x is None else x._h for x in xs])
            ia = lambda v: np.ascontiguousarray(v, np.int32)
            sp, tp = np.tile(IDENT, (max(k, 1), 1)), np.tile(IDENT, (max(m, 1), 1))
            out = [T(), C.c_double(), C.c_int(), C.c_int(), C.c_int(), C.c_int()]
            a, b = ia(si), ia(ti)
            return L._binding.lib().liliom_loop_align_multi(
                c._h, arr(ss), a.ctypes.data_as(C.POINTER(C.c_int)), sp.ctypes.data_as(C.POINTER(C.c_double)), k, arr(ts),
                b.ctypes.data_as(C.POINTER(C.c_int)), tp.ctypes.data_as(C.POINTER(C.c_double)), m, leaf, 2.0, max_iter, 1e-6, 1e-6,
                out[0], C.byref(out[1]), C.byref(out[2]), C.byref(out[3]), C.byref(out[4]), C.byref(out[5]))
        s0, s1 = f.stores[0], f.stores[1]
        refused += [
            ("loop NULL src stores", lambda: loop_rc(None, [0], [s1], [1]), L._binding.E_ARG),
            ("loop NULL tgt store", lambda: loop_rc([s0], [0], [None], [1]), L._binding.E_ARG),
            ("loop stride", lambda: loop_rc([other], [0], [s1], [1]), L._binding.E_ARG),
            ("loop unknown id", lambda: loop_rc([s0], [0], [s1], [50]), L._binding.E_ARG),
            ("loop leaf", lambda: loop_rc([s0], [0], [s1], [1], leaf=0.0), L._binding.E_ARG),
            ("loop max_iter", lambda: loop_rc([s0], [0], [s1], [1], max_iter=0), L._binding.E_ARG),
        ]
        for what, call, rc in refused:
            assert call() == rc, what
            c.map_update_resident(IDENT)                 # c's resident scan stays
        assert [_snapshot(st) for st in f.stores] == snaps
        # the calls that run: each store byte-identical before and after every one
        snaps = [_snapshot(st) for st in f.stores]
        c.global_map_multi(L.KF_FULL, f.ctxs(e), ids, poses, 0.3)
        assert [_snapshot(st) for st in f.stores] == snaps
        c.global_map_multi(L.KF_SURF, f.ctxs(e), ids, poses, TINY_LEAF)
        assert [_snapshot(st) for st in f.stores] == snaps
        c.loop_align_multi([s0], [4], [f.pose(0, 4)], [s1, s0], [3, 3], [f.pose(1, 3), f.pose(0, 3)], 0.4, **LOOP)
        assert [_snapshot(st) for st in f.stores] == snaps
        # c's resident scan is gone, as after the single-store calls; every store's own scan is still there
        with pytest.raises(L.LiliomError):
            c.map_update_resident(IDENT)
        for st in f.stores:                              # (a snapshot would overwrite the store's own scan)
            _resident(st, 9)
        f.stores[1].global_map_multi(L.KF_FULL, f.ctxs(e), ids, poses, 0.3)
        for st in (f.stores[0], f.stores[2]):
            st.map_update_resident(IDENT)
        with pytest.raises(L.LiliomError):
            f.stores[1].map_update_resident(IDENT)      # the caller, as after liliom_global_map on it
        f.D.global_map(L.KF_FULL, [0], [IDENT], 0.3)
        with pytest.raises(L.LiliomError):
            f.D.map_update_resident(IDENT)
    finally:
        other.close()
        f.close()


# ------------------------------------------------------------------------------------------ at size
def test_at_size_four_stores_against_the_merged_store():
    """four stores of 500 keyframes of ~20k full points each (~40 M points), an interleaved list of all of them, against D"""
    import liliom_b200 as L
    from liliom_b200 import synth
    sweeps = [kf[3] for kf in synth.make_keyframe_sequence(12, stride=48, seed=3, full=True)]
    T0 = synth.default_true_pose()
    bp = L.backend_default_params(0)
    stores = [L.Context(variant=0) for _ in range(4)]
    D = L.Context(variant=0)
    empty = sweeps[0][:0]
    n_kf = 500
    try:
        for s, st in enumerate(stores):
            for i in range(n_kf):
                for c in (st, D):
                    kid, _, _ = c.kf_add(bp, empty, empty, download=False)
                    c.kf_add_full(bp, kid, sweeps[(s * 7 + i) % len(sweeps)])
        entries = [(s, i) for i in range(n_kf) for s in range(4)]
        poses = []
        for j, (s, i) in enumerate(entries):
            q = synth.qmul(synth.q_from_axis_angle([0, 0, 1], np.deg2rad(1.0 * i + 90 * s)), T0[:4])
            poses.append(np.concatenate([q, T0[4:] + np.array([1.5 * i, 40.0 * s, 0.0])]))
        N = sum(len(sweeps[(s * 7 + i) % len(sweeps)]) for s, i in entries)
        assert N > 38_000_000
        ctxs = [stores[s] for s, _ in entries]
        ids = [i for _, i in entries]
        dids = [s * n_kf + i for s, i in entries]
        for leaf in (0.5, 0.2):
            got = stores[0].global_map_multi(L.KF_FULL, ctxs, ids, poses, leaf)
            want = D.global_map(L.KF_FULL, dids, poses, leaf)
            assert 0 < len(got) < N and _b(got) == _b(want), leaf
            del got, want
    finally:
        for c in stores + [D]:
            c.close()


# ------------------------------------------------------------------------------------------ fresh context
@pytest.mark.parametrize("kind", ["48", "32"])
def test_after_call_histories_each_call_gives_a_fresh_contexts_bytes(kind):
    """a context that has served every operation of tests/history_ops.py (large, refused and empty inputs) gives, as the caller
    of both multi calls, a fresh context's bytes"""
    import history_ops as H
    import liliom_b200 as L
    f = Fleet(48 if kind == "48" else 32, n_kf=4, seeds=(41, 42))
    A = H.make_ctx(kind)
    try:
        for op in H.ops_of(kind):
            for x in ("large", "refused", "empty"):
                if x in op.inputs:
                    op.inputs[x](A)
        e = [(1, 2), (0, 0), (1, 3), (0, 3), (1, 2)]
        ids, poses = [i for _, i in e], [_nudge(f.pose(s, i), j) for j, (s, i) in enumerate(e)]

        def calls(c):
            out = [_b(c.global_map_multi(k, f.ctxs(e), ids, poses, leaf)) for k in (L.KF_FULL, L.KF_SURF) for leaf in (0.3, TINY_LEAF)]
            a = c.loop_align_multi(f.ctxs(e[:1]), ids[:1], poses[:1], f.ctxs(e[1:]), ids[1:], poses[1:], 0.4, **LOOP)
            return out + [_b(a[0]), a[1:]]
        got = calls(A)
        B = H.make_ctx(kind)
        try:
            assert got == calls(B)
        finally:
            B.close()
    finally:
        A.close()
        f.close()
