"""Batched driver-message ingest (liliom_convert_batch) against solo liliom_convert_livox / liliom_convert_pc2 calls, bit for bit.

Twin context sets get the same parameters and sources; set A converts with solo calls, set B with one batch call.  Per session
the status, the count n, the downloaded bytes, liliom_last_error and the launch counters must be equal, and so must the state
the call leaves: one liliom_extract_resident on both sets afterwards reads the resident sweep and its ring / time side channels
(status, counts, the three resident clouds, the ROT labels and curvatures)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ID = (1.0, 0.0, 0.0, 0.0)
Q_LB = np.array([0.999, 0.01, -0.02, 0.03]) / np.linalg.norm([0.999, 0.01, -0.02, 0.03])
LAYOUTS = ["velodyne22", "pcl32", "ouster48", "organised_nan", "hesai26"]
STEPS128 = 1024
UNSET = -9


def _lib():
    import liliom_b200 as L
    return L._binding.lib()


class Pc2M:
    """A PointCloud2 message as the C call takes it (a Pc2Msg, possibly altered after c_msg) and its point count."""

    def __init__(self, cm, keep, n):
        self.cm, self.keep, self.n = cm, keep, n

    @classmethod
    def of(cls, msg):
        cm, keep = msg.c_msg()
        return cls(cm, (msg, keep), msg.width * msg.height)

    def wire(self):
        import liliom_b200 as L
        w = L.WireMsg()
        w.kind, w.pc2 = L.WIRE_PC2, C.pointer(self.cm)
        return w

    def solo(self, c, out, cap):
        n = C.c_int(UNSET)
        rc = _lib().liliom_convert_pc2(c._h, C.byref(self.cm), out, cap, C.byref(n))
        return rc, n.value


class LivoxM:
    """Livox CustomPoint records (LIVOX20, or raw bytes with a stride)."""

    def __init__(self, arr, stride=None, kind=None):
        import liliom_b200 as L
        self.arr, self.n, self.stride = L.Context._livox(arr, stride)
        self.kind = L.WIRE_LIVOX if kind is None else kind

    def wire(self):
        import liliom_b200 as L
        w = L.WireMsg()
        w.kind, w.n, w.stride = self.kind, self.n, self.stride
        w.custom_pts = self.arr.ctypes.data if self.arr.size else None
        return w

    def solo(self, c, out, cap):
        import liliom_b200 as L
        if self.kind != L.WIRE_LIVOX:                                          # no solo call takes an unknown kind
            return L._binding.E_ARG, UNSET
        rc = _lib().liliom_convert_livox(c._h, self.arr.ctypes.data if self.arr.size else None, self.n, self.stride, out, cap)
        return rc, (self.n if rc == 0 else UNSET)


def livox_records(pts, seed=0, t_end=100_000_000):
    """A Horizon sweep (PT48, intensity = line + 0.1 * relative time) as the Livox driver's CustomPoint records: in time order,
    offset_time in ns with the last record at t_end."""
    import liliom_b200 as L
    rng = np.random.default_rng(seed)
    pts = pts[np.isfinite(pts["intensity"]) & (pts["intensity"] >= 0) & (pts["intensity"] < 6)]
    frac = (pts["intensity"] - np.floor(pts["intensity"])).astype(np.float64)
    order = np.argsort(frac, kind="stable")
    pts, frac = pts[order], frac[order]
    r = np.zeros(len(pts), L.LIVOX20)
    off = np.minimum(np.round(frac / 0.1 * t_end), t_end).astype(np.uint32)
    off[-1] = t_end
    r["offset_time"] = off
    r["x"], r["y"], r["z"] = pts["x"], pts["y"], pts["z"]
    r["reflectivity"] = rng.integers(0, 256, len(pts))
    r["tag"] = 0x10
    r["line"] = np.floor(pts["intensity"]).astype(np.uint8)
    return r


def stride19(rec):
    return np.ascontiguousarray(rec).view(np.uint8).reshape(len(rec), 20)[:, :19].copy().reshape(-1)


class S:
    """One session: its context's settings and the q_imu its extraction takes."""

    def __init__(self, variant, q=ID, line_num=None, ring_field=False, time_name=None, ds_rate=None):
        self.variant, self.q = variant, np.asarray(q, np.float64)
        self.line_num, self.ring_field, self.time_name, self.ds_rate = line_num, ring_field, time_name, ds_rate

    def make(self):
        import liliom_b200 as L
        p = L.default_params(self.variant)
        if self.line_num is not None:
            p.line_num = self.line_num
        if self.ds_rate is not None:
            p.ds_rate = self.ds_rate
        c = L.Context(p)
        if self.ring_field:
            c.set_ring_source(L.RING_FIELD)
        if self.time_name:
            c.set_time_source(L.TIME_FIELD, self.time_name)
        return c


@pytest.fixture(scope="module")
def world(world_small):
    from liliom_b200 import synth
    T = world_small["T"]
    hz = []
    for k in range(3):
        Tk = np.array(T); Tk[4] += 0.5 * k
        pts, q = synth.make_horizon_sweep(Tk, seed=31 + k)
        hz.append((livox_records(pts, seed=k), q))
    pts, q_hdl, ring, step = synth.make_hdl64_sweep(T, grid=True)
    pc2 = {lay: synth.encode_pc2(pts, ring, step, lay) for lay in LAYOUTS}
    small, q_small, ring_s, step_s = synth.make_hdl64_sweep(T, seed=5, steps=400, grid=True)
    small_pc2 = synth.encode_pc2(small, ring_s, step_s, "velodyne22", steps=400)
    p128, q128, r128, s128 = synth.make_spinning_sweep(T, synth.uniform_elevations(128), STEPS128, omega=(0.1, -0.05, 1.5))
    msg128 = synth.encode_pc2(p128, r128, s128, "velodyne22", steps=STEPS128, lines=128, t0=0.37)
    return dict(m=world_small["map"], T=T, hz=hz, pc2=pc2, q_hdl=q_hdl, small=small_pc2, q_small=q_small, msg128=msg128, q128=q128)


def _state(c, s):
    """What the resident sweep gives a later liliom_extract_resident: (status, counts, clouds, labels / curvatures)."""
    import liliom_b200 as L
    try:
        counts = c.extract_resident(s.q, Q_LB)
    except L.LiliomError as e:
        return (e.code,)
    clouds = [a.tobytes() for a in c.features_download()]
    out = (0, counts, clouds)
    if s.variant == 1:
        lab, cur = c.extract_rot_labels(len(c.features_download()[2]))
        out += (lab.tobytes(), cur.tobytes())
    return out


def _counters(c):
    k = c.counters()
    return (k.launches, k.lib_launches)


def _last_error(c):
    return _lib().liliom_last_error(c._h)


def _bufs(sessions, msgs, caps, null_out):
    bufs = []
    for i, (s, m) in enumerate(zip(sessions, msgs)):
        stride = 48 if s.variant == 0 else 32
        bufs.append(None if i in null_out else np.full(max(caps[i], 1) * stride, 0x5C, np.uint8))
    return bufs


def batch_call(cs, msgs, bufs, caps, out_array=True, cap_array=True):
    """liliom_convert_batch on the contexts cs; returns (rc, n, status) with n starting at UNSET."""
    import liliom_b200 as L
    B = len(cs)
    arr = (L.WireMsg * max(B, 1))(*[m.wire() for m in msgs])
    handles = (C.c_void_p * max(B, 1))(*[c._h for c in cs])
    outs = (C.c_void_p * max(B, 1))(*[b.ctypes.data if b is not None else None for b in bufs]) if out_array else None
    cap_arr = np.array(list(caps) + [0], np.int32)
    n = np.full(max(B, 1), UNSET, np.int32)
    status = np.full(max(B, 1), 77, np.int32)
    ip = C.POINTER(C.c_int)
    rc = _lib().liliom_convert_batch(handles, B, arr, outs, cap_arr.ctypes.data_as(ip) if cap_array else None, n.ctypes.data_as(ip),
                                     status.ctypes.data_as(ip))
    return rc, n[:B], status[:B]


def run_twins(sessions, msgs, caps=None, null_out=(), A_=None, B_=None, out_array=True, check_state=True):
    """Solo converts on set A, one batch call on set B; compares every session.  Returns (A, B, status)."""
    A_ = A_ if A_ is not None else [s.make() for s in sessions]
    B_ = B_ if B_ is not None else [s.make() for s in sessions]
    caps = list(caps) if caps is not None else [m.n for m in msgs]
    bufs_a = _bufs(sessions, msgs, caps, null_out)
    bufs_b = _bufs(sessions, msgs, caps, null_out)
    solo = []
    for i, (c, m) in enumerate(zip(A_, msgs)):
        o = bufs_a[i] if out_array else None
        solo.append(m.solo(c, o.ctypes.data if o is not None else None, caps[i] if out_array else 0))
    rc, n, status = batch_call(B_, msgs, bufs_b, caps, out_array=out_array)
    assert rc == 0
    for i in range(len(sessions)):
        assert (solo[i][0], solo[i][1]) == (status[i], n[i]), (i, solo[i], status[i], n[i])
        if bufs_a[i] is not None:
            assert bufs_a[i].tobytes() == bufs_b[i].tobytes(), (i, "download")
        assert _counters(A_[i]) == _counters(B_[i]), (i, _counters(A_[i]), _counters(B_[i]))
        assert _last_error(A_[i]) == _last_error(B_[i]), i
    if check_state:
        for i, s in enumerate(sessions):
            assert _state(A_[i], s) == _state(B_[i], s), (i, "resident sweep")
            assert _counters(A_[i]) == _counters(B_[i]), i
    return A_, B_, status


def close(*sets):
    for cs in sets:
        for c in cs:
            c.close()


def mixed(world):
    """Horizon sessions at stride 20 and 19 beside ROT sessions of every layout and of both ring and time sources."""
    sessions, msgs = [], []
    for k, (rec, q) in enumerate(world["hz"]):
        sessions.append(S(0, q))
        msgs.append(LivoxM(rec) if k != 1 else LivoxM(stride19(rec), 19))
    for lay in LAYOUTS:
        sessions.append(S(1, world["q_hdl"]))
        msgs.append(Pc2M.of(world["pc2"][lay]))
    sessions.append(S(1, world["q_hdl"], ring_field=True))                   # 64 rings from the `ring` field (u16)
    msgs.append(Pc2M.of(world["pc2"]["pcl32"]))
    sessions.append(S(1, world["q_hdl"], ring_field=True, time_name="t"))    # u8 ring, u32 time
    msgs.append(Pc2M.of(world["pc2"]["ouster48"]))
    sessions.append(S(1, world["q_hdl"], time_name="timestamp"))             # f64 time, elevation rings
    msgs.append(Pc2M.of(world["pc2"]["hesai26"]))
    sessions.append(S(1, world["q128"], line_num=128, ring_field=True, time_name="time"))
    msgs.append(Pc2M.of(world["msg128"]))
    return sessions, msgs


def test_mixed_sessions_every_layout_and_source(world):
    sessions, msgs = mixed(world)
    A_, B_, status = run_twins(sessions, msgs)
    assert (status == 0).all()
    # a second call reuses every buffer
    order = list(reversed(range(len(sessions))))
    run_twins([sessions[i] for i in order], [msgs[i] for i in order], A_=[A_[i] for i in order], B_=[B_[i] for i in order])
    close(A_, B_)


@pytest.mark.parametrize("B", [1, 2, 8, 32, 34])
def test_session_counts(world, B):
    """B sessions of each kind; 34 of a kind take two launches of that kind."""
    rec, q = world["hz"][0]
    sessions, msgs = [], []
    for k in range(B):
        sessions += [S(0, q), S(1, world["q_small"])]
        msgs += [LivoxM(rec if k % 2 == 0 else stride19(rec), None if k % 2 == 0 else 19), Pc2M.of(world["small"])]
    if B == 1:
        sessions, msgs = sessions[:1], msgs[:1]
    A_, B_, status = run_twins(sessions, msgs, check_state=B <= 8)
    assert (status == 0).all()
    if B > 8:
        for i in (0, 1, len(sessions) - 2, len(sessions) - 1):
            assert _state(A_[i], sessions[i]) == _state(B_[i], sessions[i]), i
    close(A_, B_)


def test_empty_messages(world):
    import liliom_b200 as L
    m = world["pc2"]["velodyne22"]
    sessions, msgs = mixed(world)
    for h, w in ((1, 0), (0, m.width), (0, 0)):
        sessions.append(S(1, world["q_hdl"]))
        msgs.append(Pc2M.of(L.PC2(np.zeros(0, np.uint8), h, w, m.point_step, w * m.point_step, m.fields)))
    sessions.append(S(1, world["q_hdl"], ring_field=True, time_name="time"))
    msgs.append(Pc2M.of(L.PC2(np.zeros(0, np.uint8), 1, 0, m.point_step, 0, m.fields)))
    sessions.append(S(0))
    msgs.append(LivoxM(np.zeros(0, L.LIVOX20)))
    sessions.append(S(0))
    msgs.append(LivoxM(np.zeros(0, np.uint8), 19))
    A_, B_, status = run_twins(sessions, msgs)
    assert (status == 0).all()
    # every session empty: no launch at all
    k = len(sessions) - 6
    A2, B2, _ = run_twins(sessions[k:], msgs[k:], A_=A_[k:], B_=B_[k:])
    close(A_, B_)


def _bad_pc2(m):
    """Header variants of a valid message that liliom_convert_pc2 refuses (tests/test_gpu_pc2.py's list)."""
    import liliom_b200 as L
    out = []

    def variant(**kw):
        a = dict(data=m.data, height=m.height, width=m.width, point_step=m.point_step, row_step=m.row_step, fields=m.fields,
                 is_bigendian=m.is_bigendian)
        raw = kw.pop("raw", None)
        a.update(kw)
        msg = L.PC2(**a)
        cm, keep = msg.c_msg()
        if raw:
            raw(cm)
        out.append(Pc2M(cm, (msg, keep), msg.width * msg.height))

    variant(point_step=0)
    variant(row_step=m.width * m.point_step - 1)
    variant(fields=[(n, m.point_step - 2 if n == "intensity" else o, d, c) for n, o, d, c in m.fields])
    variant(is_bigendian=True)
    variant(raw=lambda cm: setattr(cm, "data", None))
    variant(raw=lambda cm: setattr(cm, "fields", C.POINTER(L._binding.Pc2Field)()))
    variant(raw=lambda cm: setattr(cm, "n_fields", -1))
    variant(raw=lambda cm: (setattr(cm, "height", 2), setattr(cm, "width", 1 << 30), setattr(cm, "point_step", 1),
                            setattr(cm, "row_step", 1 << 30), setattr(cm, "n_fields", 0)))
    return out


def test_refused_sessions_beside_good_ones(world):
    """Every refusal of the solo calls and a kind that does not fit the context, each beside good sessions: the refused session
    keeps the sweep it had (liliom_extract_resident afterwards), the others convert."""
    import liliom_b200 as L
    rec, q = world["hz"][0]
    good_pc2 = Pc2M.of(world["pc2"]["velodyne22"])
    bad = [(S(1, world["q_hdl"]), b) for b in _bad_pc2(world["pc2"]["velodyne22"])]
    bad += [(S(1, world["q_hdl"]), LivoxM(rec)),                                   # LIVOX on a 32-byte context
            (S(0, q), good_pc2),                                                 # PC2 on a 48-byte context
            (S(0, q), LivoxM(rec, kind=7)),                                      # unknown kind
            (S(0, q), LivoxM(stride19(rec)[:-3], 17)),                           # bad stride
            (S(0, q), LivoxM(np.ascontiguousarray(rec).view(np.uint8).reshape(-1)[:0], 20)),
            (S(1, world["q_hdl"], ring_field=True), Pc2M.of(world["pc2"]["organised_nan"])),   # no ring field
            (S(1, world["q_hdl"], time_name="time"), Pc2M.of(world["pc2"]["pcl32"]))]          # no time field
    bad[-3][1].arr = np.zeros(0, np.uint8)
    bad[-3][1].n = 5                                                             # NULL payload, 5 points
    for sb, mb in bad:
        sessions = [S(0, q), sb, S(1, world["q_hdl"])]
        msgs = [LivoxM(rec), mb, good_pc2]
        A_, B_ = [s.make() for s in sessions], [s.make() for s in sessions]
        prior = LivoxM(world["hz"][1][0]) if sb.variant == 0 else Pc2M.of(world["small"])
        for c in (A_[1], B_[1]):
            assert prior.solo(c, None, 0)[0] == 0                                # a sweep resident before the call
        _, _, status = run_twins(sessions, msgs, A_=A_, B_=B_)
        assert status[0] == 0 and status[2] == 0 and status[1] == L._binding.E_ARG, status
        kept = _state(B_[1], sb)
        assert kept[0] == 0 and len(kept[2][2]) > 0                              # the earlier sweep is still resident
        close(A_, B_)


def test_capacity_and_null_out_entries(world):
    sessions, msgs = mixed(world)
    caps = [m.n for m in msgs]
    caps[0] -= 1                     # Livox: E_CAPACITY, n not written
    caps[3] -= 1                     # PC2: E_CAPACITY, n = the message's points
    caps[5] = 0
    A_, B_, status = run_twins(sessions, msgs, caps=caps, null_out={1, 4, 6})
    assert status[0] == status[3] == status[5] == -4 and status[1] == status[4] == status[6] == 0
    close(A_, B_)
    # a NULL out array: no download, and cap is not read
    A_, B_, status = run_twins(sessions, msgs, out_array=False)
    assert (status == 0).all()
    close(A_, B_)
    # a NULL cap array with an out array: capacity 0 for every session with an out entry
    A_ = [s.make() for s in sessions]
    B_ = [s.make() for s in sessions]
    bufs = _bufs(sessions, msgs, [m.n for m in msgs], set(range(1, len(msgs))))
    rc, n, status = batch_call(B_, msgs, bufs, [0] * len(msgs), cap_array=False)
    assert rc == 0 and status[0] == -4 and (status[1:] == 0).all()
    close(A_, B_)


def test_caller_streams(world):
    import torch
    sessions, msgs = mixed(world)
    streams = [torch.cuda.Stream() for _ in range(3)]
    A_, B_ = [s.make() for s in sessions], [s.make() for s in sessions]
    for cs in (A_, B_):
        for k, i in enumerate((0, 4, 5, 8)):
            cs[i].set_stream(streams[k % 3].cuda_stream)        # two sessions share a stream; ctxs[0] has a caller stream
    run_twins(sessions, msgs, A_=A_, B_=B_)
    for cs in (A_, B_):
        for c in cs:
            c.set_stream(None)
    close(A_, B_)


def test_whole_call_refusals(world):
    import liliom_b200 as L
    rec, q = world["hz"][0]
    sessions = [S(0, q), S(1, world["q_hdl"])]
    msgs = [LivoxM(rec), Pc2M.of(world["small"])]
    cs = [s.make() for s in sessions]
    before = [_counters(c) for c in cs]
    arr = (L.WireMsg * 2)(*[m.wire() for m in msgs])
    ip = C.POINTER(C.c_int)
    n = np.full(2, UNSET, np.int32)
    status = np.full(2, 77, np.int32)
    h = lambda *xs: (C.c_void_p * len(xs))(*xs)
    lib = _lib()
    args = lambda handles, B=2, a=arr, nn=n.ctypes.data_as(ip), st=status.ctypes.data_as(ip): (handles, B, a, None, None, nn, st)
    assert lib.liliom_convert_batch(*args(h(cs[0]._h, cs[1]._h), B=0)) == L._binding.E_ARG
    assert lib.liliom_convert_batch(*args(None)) == L._binding.E_ARG
    assert lib.liliom_convert_batch(*args(h(cs[0]._h, cs[1]._h), a=None)) == L._binding.E_ARG
    assert lib.liliom_convert_batch(*args(h(cs[0]._h, cs[1]._h), nn=None)) == L._binding.E_ARG
    assert lib.liliom_convert_batch(*args(h(cs[0]._h, cs[1]._h), st=None)) == L._binding.E_ARG
    assert lib.liliom_convert_batch(*args(h(cs[0]._h, cs[0]._h))) == L._binding.E_ARG
    assert lib.liliom_convert_batch(*args(h(cs[0]._h, None))) == L._binding.E_ARG
    assert (n == UNSET).all() and (status == 77).all()
    assert [_counters(c) for c in cs] == before
    fresh = [s.make() for s in sessions]
    for c, f, s in zip(cs, fresh, sessions):
        assert _state(c, s) == _state(f, s)                         # nothing resident
    close(cs, fresh)


def _features(c, variant):
    out = [a.tobytes() for a in c.features_download()]
    if variant == 1:
        lab, cur = c.extract_rot_labels(len(c.features_download()[2]))
        out += [lab.tobytes(), cur.tobytes()]
    return out


def test_extract_resident_batch_after_the_batch(world):
    """convert batch + extract batch against solo convert + solo extract: clouds, ROT labels and curvatures"""
    import liliom_b200 as L
    sessions, msgs = mixed(world)
    A_, B_ = [s.make() for s in sessions], [s.make() for s in sessions]
    solo = []
    for c, s, m in zip(A_, sessions, msgs):
        assert m.solo(c, None, 0)[0] == 0
        solo.append(c.extract_resident(s.q, Q_LB))
    n, status = L.convert_batch(B_, [m.keep[0] if isinstance(m, Pc2M) else (m.arr, m.stride) for m in msgs])
    assert (status == 0).all() and list(n) == [m.n for m in msgs]
    counts, st = L.extract_resident_batch(B_, np.stack([s.q for s in sessions]), np.stack([Q_LB] * len(sessions)))
    assert (st == 0).all()
    for i, s in enumerate(sessions):
        assert tuple(solo[i]) == tuple(int(x) for x in counts[i]), i
        assert _features(A_[i], s.variant) == _features(B_[i], s.variant), i
        assert _counters(A_[i]) == _counters(B_[i]), i
    close(A_, B_)


def test_binding_downloads(world):
    import liliom_b200 as L
    rec, q = world["hz"][2]
    msg = world["pc2"]["ouster48"]
    cs = [L.Context(variant=0), L.Context(variant=1)]
    clouds, status = L.convert_batch(cs, [rec, msg], download=True)
    assert (status == 0).all()
    ref = [L.Context(variant=0), L.Context(variant=1)]
    assert clouds[0].tobytes() == ref[0].convert_livox(rec).tobytes()
    assert clouds[1].tobytes() == ref[1].convert_pc2(msg).tobytes()
    close(cs, ref)


@pytest.mark.parametrize("mode", ["gn", "ceres"])
def test_fleet_loop(world, mode):
    """convert batch -> extract batch -> odometry batch -> map update batch over 20 scans, against the same steps in solo
    calls: poses, statuses, map sizes and the final maps"""
    import liliom_b200 as L
    from liliom_b200 import synth
    md = L.MODE_GN if mode == "gn" else L.MODE_CERES
    hz, pc2 = world["hz"], [world["pc2"]["velodyne22"], world["pc2"]["hesai26"], world["small"]]
    sessions = [S(0, hz[0][1]), S(0, hz[1][1]), S(1, world["q_hdl"]), S(1, world["q_hdl"], time_name="timestamp")]
    A_, B_ = [s.make() for s in sessions], [s.make() for s in sessions]
    guess = synth.perturbed_pose(world["T"])
    for c in A_ + B_:
        c.map_set_points(world["m"])
    pa = [np.array(guess) for _ in sessions]
    pb = np.stack([np.array(guess) for _ in sessions])
    for step in range(20):
        msgs, qs = [], []
        for i, s in enumerate(sessions):
            if s.variant == 0:
                rec, q = hz[(step + i) % 3]
                msgs.append(rec if step % 2 else (stride19(rec), 19))
            else:
                msgs.append(pc2[(step + i) % 2] if i == 2 else pc2[1])
                q = world["q_hdl"]
            qs.append(q)
        sa, ma = [], []
        for i, c in enumerate(A_):
            m = msgs[i]
            if isinstance(m, L.PC2):
                c.convert_pc2(m, download=False)
            else:
                c.convert_livox(*(m if isinstance(m, tuple) else (m, None)), download=False)
            c.extract_resident(qs[i], Q_LB)
            try:
                pa[i], _, _ = c.odometry_resident(pa[i], 4, 15, md)
                sa.append(0)
                ma.append(c.map_update_resident(pa[i]))
            except L.LiliomError as e:
                sa.append(e.code)
                ma.append(None)
        n, st = L.convert_batch(B_, msgs)
        assert (st == 0).all()
        _, st = L.extract_resident_batch(B_, np.stack(qs), np.stack([Q_LB] * len(sessions)))
        assert (st == 0).all()
        pb, st, _, _ = L.odometry_resident_batch_ex(B_, pb, 4, 15, md)
        assert list(st) == sa, (step, list(st), sa)
        ok = [i for i in range(len(sessions)) if st[i] == 0]
        nm, st2 = L.map_update_batch([B_[i] for i in ok], pb[ok])
        assert (st2 == 0).all()
        for k, i in enumerate(ok):
            assert pa[i].tobytes() == pb[i].tobytes(), (step, i)
            assert ma[i] == nm[k], (step, i)
    for a, b in zip(A_, B_):
        assert a.map_download_cloud().tobytes() == b.map_download_cloud().tobytes()
        assert _counters(a) == _counters(b)
    close(A_, B_)
