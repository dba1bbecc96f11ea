"""GPU checks of the batched backend window calls (liliom_backend_window_correspond_batch / liliom_backend_window_blocks_batch):
byte for byte against twin contexts driven by the solo calls (status, counts, liliom_last_error, every slot's resident
correspondences, the blocks, the launch counters, the window left resident), an oracle anchor, every per-session error inside a
batch of healthy sessions, solo and batched calls mixed in every order, empty keyframes, whole-call refusals, caller streams, and
a fleet loop over several keyframes."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NKF = 12            # keyframes per stream
BODY_SETS = 3       # body poses the blocks are evaluated at


@pytest.fixture(scope="module")
def seqs():
    from liliom_b200 import synth
    return {48: synth.make_keyframe_sequence(NKF, stride=48, seed=7), 32: synth.make_keyframe_sequence(NKF, stride=32, seed=5)}


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def _nudge(pose, k):
    from liliom_b200 import synth
    dq = synth.q_from_axis_angle([1, -1, 2], np.deg2rad(0.15 * k))
    return np.concatenate([synth.qmul(pose[:4], dq), pose[4:] + 0.01 * k * np.array([1.0, -0.5, 0.25])])


def _body(pose_l, bp):
    from liliom_b200 import synth
    q = synth.qmul(pose_l[:4], np.array(bp.q_lb[:]))
    return np.concatenate([q / np.linalg.norm(q), pose_l[4:] + synth.qrot(pose_l[:4], np.array(bp.t_lb[:]))])


def _last_error(c):
    import liliom_b200 as L
    return L._binding.lib().liliom_last_error(c._h).decode()


def _launches(c):
    return c.counters().launches


def _try(f):
    import liliom_b200 as L
    try:
        return 0, f()
    except L.LiliomError as e:
        return e.code, None


class Sess:
    """One session's settings: its stream (stride), parameters, local map and window.  s seeds every choice."""

    def __init__(self, seqs, s, k=None, stride=None):
        import liliom_b200 as L
        self.stride = stride or (48 if s % 3 != 1 else 32)
        self.variant = 0 if self.stride == 48 else 1
        self.seq = seqs[self.stride]
        bp = L.backend_default_params(self.variant)
        bp.cauchy_b = bp.cauchy_b * (1.0 + 0.05 * (s % 4))
        bp.lidar_const = bp.lidar_const * (1.0 + 0.1 * (s % 5))
        bp.surf_dist_thres = bp.surf_dist_thres * (1.0 + 0.02 * (s % 3))
        self.bp = bp
        self.k = k if k is not None else 1 + (5 * s + 2) % 16
        lo = s % 5
        self.map_ids = list(range(lo, min(lo + 6, NKF)))
        self.map_poses = [_nudge(self.seq[i][2], s % 3) for i in self.map_ids]
        self.win = [(self.map_ids[-1] - j) % NKF for j in range(self.k)][::-1]
        self.poses_l = [_nudge(self.seq[i][2], 1 + s % 2) for i in self.win]
        self.bodies = [[_nudge(_body(p, bp), j) for p in self.poses_l] for j in range(BODY_SETS)]

    def make(self, store=True, build=True):
        """A context with the stream stored and (build) the local map built."""
        import liliom_b200 as L
        c = L.Context(variant=self.variant)
        if store:
            for e, s, _ in self.seq:
                c.kf_add(self.bp, e, s, download=False)
        if build:
            c.bmap_build(self.bp, self.map_ids, self.map_poses)
        return c


def _corr_state(c, k):
    """Every slot's resident correspondences of both kinds (the solo test hook)."""
    return [tuple(_bytes(x) for x in c.backend_window_corr(slot, kind)) for slot in range(k) for kind in (0, 1)]


def _fleet(seqs, B, **kw):
    S = [Sess(seqs, s, **kw) for s in range(B)]
    return S, [s.make() for s in S], [s.make() for s in S]


def _solo_correspond(c, ss):
    return _try(lambda: c.backend_window_correspond(ss.bp, ss.win, ss.poses_l))


def _batch_correspond(cs, S):
    import liliom_b200 as L
    return L.backend_window_correspond_batch(cs, [s.bp for s in S], [s.win for s in S], [s.poses_l for s in S])


def _assert_same_window(a, b, ss, what):
    """The same window resident in the solo twin a and the batched context b: corr of every slot and the blocks."""
    assert _corr_state(a, ss.k) == _corr_state(b, ss.k), what
    for body in ss.bodies[:1]:
        ra, rb = _try(lambda: a.backend_window_blocks(body)), _try(lambda: b.backend_window_blocks(body))
        assert ra[0] == rb[0] == 0 and _bytes(ra[1]) == _bytes(rb[1]), what


def _close(*groups):
    for g in groups:
        for c in g:
            if c is not None:
                c.close()


# ---------------------------------------------------------------- 1. batch against solo
@pytest.mark.parametrize("B", [1, 2, 8, 32, 34])
def test_batch_matches_solo(seqs, B):
    import liliom_b200 as L
    S, A, Bc = _fleet(seqs, B)
    assert {s.variant for s in S} == ({0} if B == 1 else {0, 1})
    if B >= 16:
        assert {s.k for s in S} == set(range(1, 17))
    la0, lb0 = [_launches(c) for c in A], [_launches(c) for c in Bc]
    solo = [_solo_correspond(A[i], S[i]) for i in range(B)]
    got, status = _batch_correspond(Bc, S)
    for i in range(B):
        assert status[i] == solo[i][0] == 0, (i, status[i], solo[i][0])
        ne, ns = solo[i][1]
        assert _bytes(got[i][0]) == _bytes(ne) and _bytes(got[i][1]) == _bytes(ns), i
        assert ne.sum() > 0 and ns.sum() > 0, (i, ne, ns)
        assert _corr_state(A[i], S[i].k) == _corr_state(Bc[i], S[i].k), i
        assert _launches(A[i]) - la0[i] == _launches(Bc[i]) - lb0[i] == 3, i
    for j in range(BODY_SETS):
        la0, lb0 = [_launches(c) for c in A], [_launches(c) for c in Bc]
        want = [A[i].backend_window_blocks(S[i].bodies[j]) for i in range(B)]
        out, status = L.backend_window_blocks_batch(Bc, [s.bodies[j] for s in S])
        for i in range(B):
            assert status[i] == 0 and out[i].shape == (S[i].k, 2, 29) and _bytes(out[i]) == _bytes(want[i]), (j, i)
            assert _launches(A[i]) - la0[i] == _launches(Bc[i]) - lb0[i] == 2, (j, i)
    _close(A, Bc)


# ---------------------------------------------------------------- 2. oracle anchor
@pytest.mark.parametrize("stride", [48, 32])
def test_batched_window_against_oracle(oracle, seqs, stride):
    """The batched results of a few sessions pass test_gpu_backend_window.py's oracle check (the window correspondences against
    the oracle's search on the layers, the blocks against its reductions)."""
    import liliom_b200 as L
    import test_gpu_backend_window as W
    S = [Sess(seqs, s, k=3, stride=stride) for s in range(3)]
    cs = [L.Context(variant=s.variant) for s in S]
    kfs = [W._store(c, s.bp, s.seq) for c, s in zip(cs, S)]
    for c, s in zip(cs, S):
        c.bmap_build(s.bp, s.map_ids, s.map_poses)
    got, status = _batch_correspond(cs, S)
    assert list(status) == [0, 0, 0]
    blocks, status = L.backend_window_blocks_batch(cs, [s.bodies[0] for s in S])
    assert list(status) == [0, 0, 0]
    for c, s, kf, (ne, ns), blk in zip(cs, S, kfs, got, blocks):
        layers = (c.bmap_download(0), c.bmap_download(1))
        state = _corr_state(c, s.k)
        # W._check_window runs the solo window calls on c, whose results must equal the batched ones already resident
        cne, cns = W._check_window(c, oracle, s.bp, kf, s.win, s.poses_l, layers, [s.bodies[0]])
        assert _bytes(cne) == _bytes(ne) and _bytes(cns) == _bytes(ns) and _corr_state(c, s.k) == state
        assert _bytes(c.backend_window_blocks(s.bodies[0])) == _bytes(blk)
    _close(cs)


# ---------------------------------------------------------------- 3. per-session errors
def _raw_correspond(cs, S, ids, ks, prefill):
    """The batched call through ctypes with count arrays pre-filled with `prefill` (to see the partial zeroing)."""
    import liliom_b200 as L
    B = len(cs)
    h = (C.c_void_p * B)(*[c._h for c in cs])
    bps = (L.BackendParams * B)(*[s.bp for s in S])
    idarr = [np.ascontiguousarray(x, np.int32) if x is not None else None for x in ids]
    parr = [np.ascontiguousarray(np.array(s.poses_l).reshape(-1), np.float64) for s in S]
    P = C.POINTER(C.c_int)
    D = C.POINTER(C.c_double)
    ne = [np.full(16, prefill, np.int32) for _ in range(B)]
    ns = [np.full(16, prefill, np.int32) for _ in range(B)]
    status = np.full(B, 12345, np.int32)
    k = np.array(ks, np.int32)
    rc = L._binding.lib().liliom_backend_window_correspond_batch(
        h, B, bps, (P * B)(*[x.ctypes.data_as(P) if x is not None else P() for x in idarr]), (D * B)(*[x.ctypes.data_as(D) for x in parr]),
        k.ctypes.data_as(P), (P * B)(*[x.ctypes.data_as(P) for x in ne]), (P * B)(*[x.ctypes.data_as(P) for x in ns]), status.ctypes.data_as(P))
    return rc, ne, ns, status


def _raw_solo(c, ss, ids, k, prefill):
    import liliom_b200 as L
    P = C.POINTER(C.c_int)
    ne = np.full(16, prefill, np.int32); ns = np.full(16, prefill, np.int32)
    idarr = np.ascontiguousarray(ids, np.int32) if ids is not None else None
    p = np.ascontiguousarray(np.array(ss.poses_l).reshape(-1), np.float64)
    rc = L._binding.lib().liliom_backend_window_correspond(c._h, C.byref(ss.bp), idarr.ctypes.data_as(P) if idarr is not None else None,
                                                          p.ctypes.data_as(C.POINTER(C.c_double)), k, ne.ctypes.data_as(P), ns.ctypes.data_as(P))
    return rc, ne, ns


def test_per_session_errors_inside_a_batch(seqs):
    """Healthy sessions around each error: every session's status, counts (pre-filled, to see the partial zeroing), last_error,
    launches, and whether a following solo blocks call succeeds, and with which bits, equal its solo twin's."""
    import liliom_b200 as L
    E_ARG, E_NOMAP, E_FEWMAP = -1, L._binding.E_NOMAP, L._binding.E_FEWMAP
    S = [Sess(seqs, s, k=4) for s in range(10)]
    S[4] = Sess(seqs, 4, k=4, stride=32)         # the variant-0-on-a-32-byte-context case
    A = [s.make(build=(i not in (5, 6))) for i, s in enumerate(S)]
    Bc = [s.make(build=(i not in (5, 6))) for i, s in enumerate(S)]
    for c in (A[6], Bc[6]):
        c.bmap_build(S[6].bp, [], [])            # empty layers: the :933 gate
    # a window resident everywhere it can be, so that the errors' effect on it shows
    for i in range(len(S)):
        if i in (5, 6):
            continue
        assert _solo_correspond(A[i], S[i])[0] == 0 and _solo_correspond(Bc[i], S[i])[0] == 0
    ids = [s.win for s in S]
    ks = [s.k for s in S]
    ids[1] = [S[1].win[0], S[1].win[1], 10_000, S[1].win[3]]          # unknown id: counts zeroed up to it
    ks[2] = 0                                                            # k out of range
    ks[3] = 17; ids[3] = (S[3].win * 5)[:17]
    S[4].bp.variant = 0                                                  # variant 0 on a 32-byte context
    S[7].bp.kd_max_radius = 100.0                                        # over the surf layer's cell
    ids[8] = None                                                        # a NULL per-session pointer
    la, lb = [_launches(c) for c in A], [_launches(c) for c in Bc]
    rc, ne, ns, status = _raw_correspond(Bc, S, ids, ks, -7)
    assert rc == 0
    want = {1: E_ARG, 2: E_ARG, 3: E_ARG, 4: E_ARG, 5: E_NOMAP, 6: E_FEWMAP, 7: E_ARG, 8: E_ARG}
    for i in range(len(S)):
        src, sne, sns = _raw_solo(A[i], S[i], ids[i], ks[i], -7)
        assert status[i] == src == want.get(i, 0), (i, status[i], src)
        assert _bytes(ne[i]) == _bytes(sne) and _bytes(ns[i]) == _bytes(sns), i
        assert _last_error(A[i]) == _last_error(Bc[i]), i
        assert _launches(A[i]) - la[i] == _launches(Bc[i]) - lb[i] == (3 if src == 0 else 0), i
    assert list(ne[1][:4]) == [0, 0, 0, -7] and list(ns[1][:4]) == [0, 0, 0, -7]
    assert "unknown keyframe id" in _last_error(Bc[1]) and "48-byte" in _last_error(Bc[4]) and "kd_max_radius" in _last_error(Bc[7])
    # the resident window afterwards: argument errors before the window is dropped keep it; NOMAP, FEWMAP and the cell check drop it
    for i in range(len(S)):
        body = S[i].bodies[1]
        ra, rb = _try(lambda: A[i].backend_window_blocks(body)), _try(lambda: Bc[i].backend_window_blocks(body))
        assert ra[0] == rb[0] == (E_ARG if i in (5, 6, 7) else 0), (i, ra[0], rb[0])
        if ra[0] == 0:
            assert _bytes(ra[1]) == _bytes(rb[1]), i
    # a blocks call whose k does not match, among healthy ones
    bodies = [s.bodies[2] for s in S]
    bodies[0] = bodies[0][:3]
    la, lb = [_launches(c) for c in A], [_launches(c) for c in Bc]
    out, status = L.backend_window_blocks_batch(Bc, bodies)
    for i in range(len(S)):
        ra = _try(lambda: A[i].backend_window_blocks(bodies[i]))
        assert status[i] == ra[0], (i, status[i], ra[0])
        assert _last_error(A[i]) == _last_error(Bc[i]), i
        assert _launches(A[i]) - la[i] == _launches(Bc[i]) - lb[i], i
        if ra[0] == 0:
            assert _bytes(out[i]) == _bytes(ra[1]), i
    assert status[0] == E_ARG and "the k of the window" in _last_error(Bc[0])
    _close(A, Bc)


# ---------------------------------------------------------------- 4. mixing orders
def test_solo_and_batched_calls_mix_and_leave_the_rest_alone(seqs):
    import liliom_b200 as L
    S, A, Bc = _fleet(seqs, 4)
    m, _ = __import__("liliom_b200.synth", fromlist=["make_map"]).make_map(20_000)
    single = []
    for i, c in enumerate(Bc):            # an odometry map and single-keyframe correspondences, resident before the window calls
        c.map_set_points(m)
        e = S[i].seq[0][0]
        c.correspond_edge(e, S[i].seq[0][2], S[i].variant)
        single.append((c.map_download().tobytes(), c.kf_count(), _bytes(c.kf_cloud([0, 3], [S[i].seq[0][2]] * 2, 0.2)),
                       _bytes(c.backend_edge_block(S[i].bodies[0][0], 1.5, S[i].bp.cauchy_b))))
    # batched correspond, then solo blocks and corr
    for i in range(4):
        _solo_correspond(A[i], S[i])
    _batch_correspond(Bc, S)
    for i in range(4):
        _assert_same_window(A[i], Bc[i], S[i], ("batched correspond, solo blocks", i))
    # solo correspond with a new window, then batched blocks
    S2 = [Sess(seqs, s + 1, k=S[s].k + 1) for s in range(4)]
    for i in range(4):
        S2[i].bp = S[i].bp; S2[i].seq = S[i].seq; S2[i].variant = S[i].variant
        S2[i].bodies = [[_nudge(_body(p, S[i].bp), j) for p in S2[i].poses_l] for j in range(BODY_SETS)]
        assert _solo_correspond(A[i], S2[i])[0] == 0 and _solo_correspond(Bc[i], S2[i])[0] == 0
    out, status = L.backend_window_blocks_batch(Bc, [s.bodies[1] for s in S2])
    for i in range(4):
        assert status[i] == 0 and _bytes(out[i]) == _bytes(A[i].backend_window_blocks(S2[i].bodies[1])), i
    # batched correspond, batched blocks, then a solo correspond of the first window and the batched blocks again
    _batch_correspond(Bc, S)
    for i in range(4):
        _solo_correspond(A[i], S[i])
    out, status = L.backend_window_blocks_batch(Bc, [s.bodies[2] for s in S])
    for i in range(4):
        assert _bytes(out[i]) == _bytes(A[i].backend_window_blocks(S[i].bodies[2])), i
    for i, c in enumerate(Bc):            # the odometry map, the keyframe store and the single-keyframe correspondences are intact
        e = S[i].seq[0][0]
        now = (c.map_download().tobytes(), c.kf_count(), _bytes(c.kf_cloud([0, 3], [S[i].seq[0][2]] * 2, 0.2)),
               _bytes(c.backend_edge_block(S[i].bodies[0][0], 1.5, S[i].bp.cauchy_b)))
        assert now == single[i], i
    _close(A, Bc)


# ---------------------------------------------------------------- 5. empty keyframes, no edge queries
def test_empty_keyframes_and_windows_without_edge_queries(seqs):
    import liliom_b200 as L
    S = [Sess(seqs, s, k=3) for s in range(4)]
    A, Bc = [], []
    for s in S:
        for group in (A, Bc):
            c = s.make()
            e, sf, _ = s.seq[0]
            c.kf_add(s.bp, e[:0], sf, download=False)        # id NKF: no edge points
            c.kf_add(s.bp, e[:0], sf[:0], download=False)    # id NKF + 1: empty
            c.kf_add(s.bp, e, sf[:0], download=False)        # id NKF + 2: no surf points
            group.append(c)
    S[0].win = [NKF, NKF, NKF]                   # no edge query in the whole window
    S[1].win = [NKF + 1, NKF + 1, NKF + 1]       # no query at all
    S[2].win = [NKF + 2, NKF + 1, NKF]           # one kind per keyframe
    S[3].win = [NKF + 1, 2, NKF + 2]
    la, lb = [_launches(c) for c in A], [_launches(c) for c in Bc]
    solo = [_solo_correspond(A[i], S[i]) for i in range(4)]
    got, status = _batch_correspond(Bc, S)
    for i in range(4):
        assert status[i] == solo[i][0] == 0
        assert _bytes(got[i][0]) == _bytes(solo[i][1][0]) and _bytes(got[i][1]) == _bytes(solo[i][1][1]), i
        assert _launches(A[i]) - la[i] == _launches(Bc[i]) - lb[i], i
        assert _corr_state(A[i], 3) == _corr_state(Bc[i], 3), i
    assert _launches(Bc[0]) - lb[0] == 2 and _launches(Bc[1]) - lb[1] == 1      # no edge launch; no search launch at all
    la, lb = [_launches(c) for c in A], [_launches(c) for c in Bc]
    out, status = L.backend_window_blocks_batch(Bc, [s.bodies[0] for s in S])
    for i in range(4):
        assert status[i] == 0 and _bytes(out[i]) == _bytes(A[i].backend_window_blocks(S[i].bodies[0])), i
        assert _launches(A[i]) - la[i] == _launches(Bc[i]) - lb[i] == 2, i
    assert not out[1].any()
    _close(A, Bc)


# ---------------------------------------------------------------- 6. whole-call refusals
def test_whole_call_refusals_change_nothing(seqs):
    import liliom_b200 as L
    S, A, Bc = _fleet(seqs, 2)
    for i in range(2):
        _solo_correspond(Bc[i], S[i])
    peer = S[0].make(build=True)
    peer.comm_peer_attach([peer.comm_peer_export()], 0)          # a fused-exchange context: the communicator rule
    before = [(_launches(c), _corr_state(c, s.k), _bytes(c.backend_window_blocks(s.bodies[0]))) for c, s in zip(Bc, S)]
    refused = [([], []), ([Bc[0], None], S), ([Bc[0], Bc[0]], [S[0], S[0]]), ([Bc[0], peer], [S[0], S[0]])]
    lib = L._binding.lib()
    for cs, ss in refused:
        with pytest.raises(L.LiliomError) as e:
            _batch_correspond(cs, ss)
        assert e.value.code == -1
        with pytest.raises(L.LiliomError) as e:
            L.backend_window_blocks_batch(cs, [s.bodies[0] for s in ss])
        assert e.value.code == -1
    h = (C.c_void_p * 2)(Bc[0]._h, Bc[1]._h)
    status = (C.c_int * 2)(7, 7)
    assert lib.liliom_backend_window_correspond_batch(h, 2, None, None, None, None, None, None, status) == -1
    assert lib.liliom_backend_window_blocks_batch(h, 2, None, None, None, status) == -1
    assert lib.liliom_backend_window_blocks_batch(h, 0, None, None, None, status) == -1
    assert list(status) == [7, 7]
    after = [(_launches(c), _corr_state(c, s.k), _bytes(c.backend_window_blocks(s.bodies[0]))) for c, s in zip(Bc, S)]
    assert [(x[0] + 2, x[1], x[2]) for x in before] == after      # only the two blocks calls of `after` itself
    _close(A, Bc, [peer])


# ---------------------------------------------------------------- 7. caller streams
def test_sessions_on_their_own_streams(seqs):
    import torch
    import liliom_b200 as L
    S, A, Bc = _fleet(seqs, 5)
    streams = [torch.cuda.Stream() for _ in range(3)]
    Bc[0].set_stream(streams[0].cuda_stream)      # ctxs[0] on a caller stream: the shared launches run there
    Bc[2].set_stream(streams[1].cuda_stream)
    Bc[3].set_stream(streams[2].cuda_stream)
    for i in (0, 2, 3):
        Bc[i].bmap_build(S[i].bp, S[i].map_ids, S[i].map_poses)      # fresh work queued on the caller stream right before
    solo = [_solo_correspond(A[i], S[i]) for i in range(5)]
    got, status = _batch_correspond(Bc, S)
    for i in range(5):
        assert status[i] == 0 and _bytes(got[i][0]) == _bytes(solo[i][1][0]) and _bytes(got[i][1]) == _bytes(solo[i][1][1]), i
    for j in range(BODY_SETS):
        out, status = L.backend_window_blocks_batch(Bc, [s.bodies[j] for s in S])
        for i in range(5):
            assert status[i] == 0 and _bytes(out[i]) == _bytes(A[i].backend_window_blocks(S[i].bodies[j])), (j, i)
    for i in range(5):
        assert _corr_state(A[i], S[i].k) == _corr_state(Bc[i], S[i].k), i
    torch.cuda.synchronize()
    _close(A, Bc)


# ---------------------------------------------------------------- 8. fleet loop
def test_fleet_loop_equals_solo_loop(seqs):
    """Per keyframe: kf_add, bmap_build over the last keyframes, one batched correspond of the newest window, 16 batched blocks
    calls at LM trial poses; the same loop through the solo calls gives the same bits."""
    import liliom_b200 as L
    B = 6
    S = [Sess(seqs, s) for s in range(B)]
    A = [L.Context(variant=s.variant) for s in S]
    Bc = [L.Context(variant=s.variant) for s in S]
    for j, step in enumerate(range(NKF)):
        for group in (A, Bc):
            for c, s in zip(group, S):
                e, sf, _ = s.seq[step]
                c.kf_add(s.bp, e, sf, download=False)
                ids = list(range(max(0, step - 4), step + 1))
                c.bmap_build(s.bp, ids, [_nudge(s.seq[i][2], 1) for i in ids])
        if step < 3:
            continue
        live = [i for i in range(B) if (step + i) % 3 != 0]            # sessions without a new keyframe this step stay out
        win = list(range(step - 2, step + 1))
        for i in live:
            S[i].win = win; S[i].k = 3
            S[i].poses_l = [_nudge(S[i].seq[w][2], 2) for w in win]
        solo = [_solo_correspond(A[i], S[i]) for i in live]
        got, status = _batch_correspond([Bc[i] for i in live], [S[i] for i in live])
        for m, i in enumerate(live):
            assert status[m] == solo[m][0] == 0
            assert _bytes(got[m][0]) == _bytes(solo[m][1][0]) and _bytes(got[m][1]) == _bytes(solo[m][1][1]), (step, i)
        for it in range(16):
            still = [i for i in live if it < 16 - (i % 4)]                # sessions whose LM stopped early stay out
            bodies = [[_nudge(_body(p, S[i].bp), it) for p in S[i].poses_l] for i in still]
            out, status = L.backend_window_blocks_batch([Bc[i] for i in still], bodies)
            for m, i in enumerate(still):
                assert status[m] == 0 and _bytes(out[m]) == _bytes(A[i].backend_window_blocks(bodies[m])), (step, it, i)
    for i in range(B):
        assert _launches(A[i]) == _launches(Bc[i]), i
    _close(A, Bc)
