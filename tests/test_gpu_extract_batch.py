"""Batched extraction (liliom_extract_resident_batch) against solo liliom_extract_resident calls, bit for bit.

Twin context sets get the same parameters and resident sweeps; set A extracts with solo calls, set B with one batch call per
step.  Per session the status, the counts, the bytes of the three resident clouds (liliom_features_download), the ROT labels
and curvatures, and the launch counters must be equal; one solo odometry_resident on both sets afterwards checks the state the
batch left in every context (pose, status, stats and DS bytes)."""
import ctypes as C
import os

import numpy as np
import pytest

import rot_adversarial as A

pytestmark = pytest.mark.gpu

ID = (1.0, 0.0, 0.0, 0.0)
Q_LB = np.array([0.999, 0.01, -0.02, 0.03]) / np.linalg.norm([0.999, 0.01, -0.02, 0.03])
STEPS128 = 1024


def _ctx(variant, line_num=None, ds_rate=None, env=(), ring_field=False, time_name=None):
    import liliom_b200 as L
    p = L.default_params(variant)
    if line_num is not None:
        p.line_num = line_num
    if ds_rate is not None:
        p.ds_rate = ds_rate
    old = {k: os.environ.get(k) for k in ("LILIOM_ROT_SLOW_WALK", "LILIOM_HZ_CHAIN")}
    for k in old:
        os.environ.pop(k, None)
    os.environ.update(dict(env))                           # read at liliom_create
    try:
        c = L.Context(p)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    if ring_field:
        c.set_ring_source(L.RING_FIELD)
    if time_name is not None:
        c.set_time_source(L.TIME_FIELD, time_name)
    return c


class Session:
    """One session: how to make its context, how to make its sweep resident, and its q_imu / q_lb."""

    def __init__(self, variant, load, q_imu=ID, q_lb=ID, **kw):
        self.variant, self.load, self.kw = variant, load, kw
        self.q_imu, self.q_lb = np.asarray(q_imu, np.float64), np.asarray(q_lb, np.float64)

    def make(self):
        return _ctx(self.variant, **self.kw)


def upload(pts):
    return lambda c: c.upload_scan(pts)


def pc2(msg):
    return lambda c: c.convert_pc2(msg, download=False)


def rot_session(sw, **kw):
    return Session(1, upload(sw["pts"]), sw["q_imu"], sw["q_lb"], line_num=sw["line_num"], ds_rate=sw["ds_rate"], **kw)


def _features(c):
    import liliom_b200 as L
    try:
        return 0, [a.copy() for a in c.features_download()]
    except L.LiliomError as e:
        return e.code, None


def _labels(c, n):
    lab, cur = c.extract_rot_labels(n)
    return lab.tobytes(), cur.tobytes()


def _counters(c):
    k = c.counters()
    return (k.launches, k.lib_launches)


def _solo(c, s, use_q_lb):
    import liliom_b200 as L
    try:
        return 0, c.extract_resident(s.q_imu, s.q_lb if use_q_lb else ID)
    except L.LiliomError as e:
        return e.code, (0, 0, 0)


def _check_session(i, a, b, variant):
    ra, fa = _features(a)
    rb, fb = _features(b)
    assert ra == rb, (i, ra, rb)
    n = 0
    if fa is not None:
        for k, what in enumerate(("surf", "edge", "cut")):
            assert len(fa[k]) == len(fb[k]), (i, what, len(fa[k]), len(fb[k]))
            assert fa[k].tobytes() == fb[k].tobytes(), (i, what)
        n = len(fa[2])
    if variant == 1:
        assert _labels(a, n) == _labels(b, n), (i, "labels / curvature")
    assert _counters(a) == _counters(b), (i, _counters(a), _counters(b))


def run_twins(sessions, steps=1, use_q_lb=True, setup=None, after=None):
    """Extract every step's sweeps solo on set A and batched on set B, compare each session; returns (A, B)."""
    import liliom_b200 as L
    A_, B_ = [s.make() for s in sessions], [s.make() for s in sessions]
    if setup:
        setup(A_, B_)
    for step in range(steps):
        for cs in (A_, B_):
            for c, s in zip(cs, sessions):
                (s.load[step] if isinstance(s.load, list) else s.load)(c)
        solo = [_solo(c, s, use_q_lb) for c, s in zip(A_, sessions)]
        q_imu = np.stack([s.q_imu for s in sessions])
        q_lb = np.stack([s.q_lb for s in sessions]) if use_q_lb else None
        counts, status = L.extract_resident_batch(B_, q_imu, q_lb)
        for i, s in enumerate(sessions):
            assert solo[i][0] == status[i], (step, i, solo[i][0], status[i])
            assert tuple(solo[i][1]) == tuple(int(x) for x in counts[i]), (step, i, solo[i][1], counts[i])
            _check_session(i, A_[i], B_[i], s.variant)
        if after:
            after(step, solo, status)
    return A_, B_


def check_state(A_, B_, m):
    """One solo odometry_resident on every context of both sets: the state the extraction left must give the same bits."""
    import liliom_b200 as L
    from liliom_b200 import synth
    guess = synth.perturbed_pose(synth.default_true_pose())
    for i, (a, b) in enumerate(zip(A_, B_)):
        out = []
        for c in (a, b):
            c.map_set_points(m)
            try:
                pose, st, ds = c.odometry_resident(guess, 4, mode=L.MODE_GN, want_ds=True, cap=400000, want_stats=True)
                out.append((0, pose.tobytes(), [bytes(memoryview(x)) for x in st], ds.tobytes()))
            except L.LiliomError as e:
                out.append((e.code,))
        assert out[0] == out[1], i


def close(*sets):
    for cs in sets:
        for c in cs:
            c.close()


@pytest.fixture(scope="module")
def world(world_small):
    from liliom_b200 import synth
    T = world_small["T"]
    hz = []
    for k in range(3):
        Tk = np.array(T); Tk[4] += 0.6 * k
        hz.append(synth.make_horizon_sweep(Tk, seed=11 + k))
    hdl = [synth.make_hdl64_sweep(T, seed=21 + k) for k in range(2)]
    pts, q, ring, step = synth.make_spinning_sweep(T, synth.uniform_elevations(128), STEPS128, omega=(0.1, -0.05, 1.5))
    msg = synth.encode_pc2(pts, ring, step, "velodyne22", steps=STEPS128, lines=128, t0=0.37)
    return dict(m=world_small["map"], hz=hz, hdl=hdl, msg128=msg, q128=q)


def test_headline_horizon_and_rot(world):
    """Headline sweeps of both variants in one call, two steps (the second reuses every buffer and barrier word)."""
    sessions = [Session(0, [upload(world["hz"][k][0]), upload(world["hz"][(k + 1) % 3][0])], world["hz"][k][1]) for k in range(3)]
    sessions += [Session(1, [upload(world["hdl"][k][0]), upload(world["hdl"][1 - k][0])], world["hdl"][k][1], Q_LB) for k in range(2)]
    A_, B_ = run_twins(sessions, steps=2)
    check_state(A_, B_, world["m"])
    close(A_, B_)


@pytest.mark.parametrize("B", [1, 2, 3, 8])
def test_session_counts(world, B):
    sessions = [Session(1, upload(world["hdl"][k % 2][0]), world["hdl"][k % 2][1], Q_LB) if k % 3 != 2 else
                Session(0, upload(world["hz"][k % 3][0]), world["hz"][k % 3][1]) for k in range(B)]
    A_, B_ = run_twins(sessions)
    check_state(A_, B_, world["m"])
    close(A_, B_)


def test_q_lb_null_is_identity(world):
    sessions = [Session(1, upload(world["hdl"][k][0]), world["hdl"][k][1], Q_LB) for k in range(2)]
    A_, B_ = run_twins(sessions, use_q_lb=False)
    close(A_, B_)


@pytest.mark.parametrize("line_num", [16, 32, 64])
def test_rot_tables(line_num):
    """The elevation tables at every ds_rate, all in one call."""
    sessions = []
    for ds in (1, 2, 3, 4):
        sw = dict(A.tables_sweep(line_num, 1)); sw["ds_rate"] = ds
        sessions.append(rot_session(sw))
    A_, B_ = run_twins(sessions)
    close(A_, B_)


def test_more_than_one_table():
    """33 ROT sessions: the rings go in two shared launches."""
    sws = [dict(A.tables_sweep(16, 1)) for _ in range(33)]
    for k, sw in enumerate(sws):
        sw["ds_rate"] = 1 + k % 4
    A_, B_ = run_twins([rot_session(sw) for sw in sws])
    close(A_, B_)


def test_ring_and_time_fields(world):
    """128 rings from the ring field and relTime from the time field, both decoded by liliom_convert_pc2."""
    msg, q = world["msg128"], world["q128"]
    sessions = [Session(1, pc2(msg), q, Q_LB, line_num=128, ds_rate=ds, ring_field=True) for ds in (1, 2)]
    sessions.append(Session(1, pc2(msg), q, Q_LB, line_num=128, ds_rate=1, ring_field=True, time_name="time"))
    sessions.append(Session(1, pc2(msg), q, Q_LB, line_num=64, ds_rate=4, time_name="time"))
    A_, B_ = run_twins(sessions)
    check_state(A_, B_, world["m"])
    close(A_, B_)


@pytest.mark.parametrize("slow", [False, True], ids=["mask_walk", "slow_walk"])
def test_rot_adversarial(slow):
    """Every adversarial ROT sweep (more than 32 of them, so two shared launches), on both ring walks."""
    env = {"LILIOM_ROT_SLOW_WALK": "1"} if slow else {}
    sessions = [rot_session(sw, env=env) for _, sw in A.all_sweeps()]
    assert len(sessions) > 32
    A_, B_ = run_twins(sessions)
    close(A_, B_)


def test_horizon_shared_launches(world):
    """Seven Horizon sessions share cooperative k_hz_batch launches at 83 blocks per session, where each solo k_hz_coop launch
    has one block per SM: equal bytes show that a session's output does not depend on its grid.  Four steps walk every
    session's barrier words through their whole rotation."""
    hz = world["hz"]
    sessions = [Session(0, [upload(hz[(k + t) % 3][0]) for t in range(4)], hz[k % 3][1]) for k in range(7)]
    A_, B_ = run_twins(sessions, steps=4)
    check_state(A_, B_, world["m"])
    close(A_, B_)


def test_horizon_adversarial():
    import hz_adversarial as H
    sws = [sw for _, sw in H.all_sweeps()]
    sessions = [Session(0, upload(sw["pts"]), sw["q"]) for sw in sws]
    sessions += [Session(0, upload(sw["pts"]), sw["q"], env={"LILIOM_HZ_CHAIN": "1"}) for sw in sws[:2]]
    A_, B_ = run_twins(sessions)
    close(A_, B_)


def test_mixed_with_empty_sweeps_and_chain(world):
    """Empty sweeps of both variants, a LILIOM_HZ_CHAIN context, a slow-walk ROT context and headline sessions in one call."""
    from liliom_b200 import PT32, PT48
    sessions = [Session(0, upload(np.zeros(0, PT48))), Session(1, upload(np.zeros(0, PT32))),
                Session(0, upload(world["hz"][0][0]), world["hz"][0][1], env={"LILIOM_HZ_CHAIN": "1"}),
                Session(1, upload(world["hdl"][0][0]), world["hdl"][0][1], Q_LB, env={"LILIOM_ROT_SLOW_WALK": "1"}),
                Session(0, upload(world["hz"][1][0]), world["hz"][1][1]),
                Session(1, upload(world["hdl"][1][0]), world["hdl"][1][1], Q_LB)]
    A_, B_ = run_twins(sessions)
    check_state(A_, B_, world["m"])
    close(A_, B_)


def test_per_session_errors(world):
    """A ring above 16384 points (LILIOM_E_CAPACITY), then a good sweep on the same context; a missing ring side channel
    (LILIOM_E_ARG); a bad line_num (LILIOM_E_LINES).  The other sessions run and match their solo calls."""
    import liliom_b200 as L
    big = A.cap_sweep(16385)
    good = dict(A.tables_sweep(16, 1))
    hdl = world["hdl"][0]
    sessions = [Session(1, [upload(big["pts"]), upload(good["pts"])], big["q_imu"], big["q_lb"], line_num=16, ds_rate=1),
                Session(1, upload(hdl[0]), hdl[1], Q_LB),
                Session(1, upload(hdl[0]), hdl[1], Q_LB, line_num=64, ring_field=True),      # no ring ids with upload_scan
                Session(1, upload(hdl[0]), hdl[1], Q_LB, line_num=20),                      # not a table
                Session(0, upload(world["hz"][0][0]), world["hz"][0][1])]
    seen = []

    def after(step, solo, status):
        seen.append([int(x) for x in status])

    A_, B_ = run_twins(sessions, steps=2, after=after)
    assert seen[0] == [L._binding.E_CAPACITY, 0, L._binding.E_ARG, L._binding.E_LINES, 0], seen[0]
    assert seen[1] == [0, 0, L._binding.E_ARG, L._binding.E_LINES, 0], seen[1]
    check_state(A_, B_, world["m"])
    close(A_, B_)


def test_whole_call_refusals(world):
    """Refused calls change nothing: counts, statuses, resident clouds and counters of every context stay as they were."""
    import liliom_b200 as L
    lib = L._binding.lib()
    cs = [_ctx(1), _ctx(0)]
    cs[0].upload_scan(world["hdl"][0][0]); cs[0].extract_resident(world["hdl"][0][1], Q_LB)
    cs[1].upload_scan(world["hz"][0][0]); cs[1].extract_resident(world["hz"][0][1])
    before = [(_features(c)[1], _counters(c)) for c in cs]
    cs[0].upload_scan(world["hdl"][1][0]); cs[1].upload_scan(world["hz"][1][0])
    q = np.tile(np.asarray(ID, np.float64), (3, 1)).reshape(-1)
    ip = C.POINTER(C.c_int)
    outs = [np.full(3, 7, np.int32) for _ in range(4)]
    dp = q.ctypes.data_as(C.POINTER(C.c_double))

    def call(handles, B, qi=dp, arrays=None):
        arr = (C.c_void_p * max(len(handles), 1))(*handles)
        a = arrays if arrays is not None else [o.ctypes.data_as(ip) for o in outs]
        return lib.liliom_extract_resident_batch(arr, B, qi, None, *a)

    h0, h1 = cs[0]._h, cs[1]._h
    refusals = [call([h0, h1], 0), call([h0, None], 2), call([h0, h0], 2), call([h0, h1], 2, qi=None),
                lib.liliom_extract_resident_batch(None, 2, dp, None, *[o.ctypes.data_as(ip) for o in outs])]
    for k in range(4):
        arrays = [o.ctypes.data_as(ip) for o in outs]
        arrays[k] = None
        refusals.append(call([h0, h1], 2, arrays=arrays))
    assert all(r == L._binding.E_ARG for r in refusals), refusals
    assert all((o == 7).all() for o in outs)
    after = [(_features(c)[1], _counters(c)) for c in cs]
    for (fb, kb), (fa, ka) in zip(before, after):
        assert kb == ka
        assert all(x.tobytes() == y.tobytes() for x, y in zip(fb, fa))
    close(cs)


def test_features_download_capacity(world):
    """A cloud larger than its buffer: LILIOM_E_CAPACITY with the counts written (the size a retry needs) and nothing copied."""
    import liliom_b200 as L
    lib = L._binding.lib()
    for variant, (pts, q) in ((0, world["hz"][0]), (1, world["hdl"][0])):
        c = _ctx(variant)
        c.upload_scan(pts)
        L.extract_resident_batch([c], np.asarray([q]))
        surf, edge, cut = c.features_download()
        buf = np.full(len(surf), 0x5A, np.uint8)
        n = [C.c_int(-9) for _ in range(3)]
        rc = lib.liliom_features_download(c._h, buf.ctypes.data_as(C.c_void_p), 1, C.byref(n[0]), None, 0, C.byref(n[1]), None, 0,
                                          C.byref(n[2]))
        assert rc == L._binding.E_CAPACITY
        assert [x.value for x in n] == [len(surf), len(edge), len(cut)]
        assert (buf == 0x5A).all()
        c.close()


def test_batch_argument_shapes(world):
    import liliom_b200 as L
    cs = [_ctx(1), _ctx(1)]
    with pytest.raises(ValueError):
        L.extract_resident_batch(cs, np.zeros((1, 4)))
    with pytest.raises(ValueError):
        L.extract_resident_batch(cs, np.tile(ID, (2, 1)), np.zeros(4))
    close(cs)


def test_caller_streams(world):
    """Sessions on caller streams (liliom_set_stream): ctxs[0] and one other on one stream, one on another, one on its own."""
    import torch
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()

    def setup(A_, B_):
        for cs in (A_, B_):
            cs[0].set_stream(s1.cuda_stream); cs[1].set_stream(s2.cuda_stream); cs[2].set_stream(s1.cuda_stream)

    sessions = [Session(1, upload(world["hdl"][0][0]), world["hdl"][0][1], Q_LB), Session(0, upload(world["hz"][0][0]), world["hz"][0][1]),
                Session(1, upload(world["hdl"][1][0]), world["hdl"][1][1], Q_LB), Session(0, upload(world["hz"][1][0]), world["hz"][1][1])]
    A_, B_ = run_twins(sessions, setup=setup)
    check_state(A_, B_, world["m"])
    for cs in (A_, B_):
        for c in cs:
            c.set_stream(None)
    close(A_, B_)


@pytest.mark.parametrize("mode", ["gn", "ceres"])
def test_end_to_end(world, mode):
    """extract_resident_batch then odometry_resident_batch_ex gives the bits of solo extraction then solo odometry."""
    import liliom_b200 as L
    from liliom_b200 import synth
    md = L.MODE_GN if mode == "gn" else L.MODE_CERES
    guess = synth.perturbed_pose(synth.default_true_pose())
    sessions = [Session(0, upload(world["hz"][k][0]), world["hz"][k][1]) for k in range(2)]
    sessions += [Session(1, upload(world["hdl"][k][0]), world["hdl"][k][1], Q_LB) for k in range(2)]
    A_, B_ = [s.make() for s in sessions], [s.make() for s in sessions]
    for cs in (A_, B_):
        for c, s in zip(cs, sessions):
            c.map_set_points(world["m"])
            s.load(c)
    solo = []
    for c, s in zip(A_, sessions):
        c.extract_resident(s.q_imu, s.q_lb)
        try:
            pose, st, ds = c.odometry_resident(guess, 4, max_num_iter=15, mode=md, want_ds=True, cap=65536, want_stats=True)
            solo.append((0, pose.tobytes(), ds.tobytes()))
        except L.LiliomError as e:
            solo.append((e.code,))
    counts, status = L.extract_resident_batch(B_, np.stack([s.q_imu for s in sessions]), np.stack([s.q_lb for s in sessions]))
    assert (status == 0).all()
    P, st, _, ds = L.odometry_resident_batch_ex(B_, [guess] * len(B_), 4, 15, md, want_ds=True)
    for i in range(len(sessions)):
        got = (0, P[i].tobytes(), ds[i].tobytes()) if st[i] == 0 else (int(st[i]),)
        assert got == solo[i], i
    close(A_, B_)
