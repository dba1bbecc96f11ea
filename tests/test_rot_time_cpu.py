"""CPU tier for the ROT extractor's time source LILIOM_TIME_FIELD (relTime from the driver's per-point PointCloud2 time field):
  - the time field rules of liliom_b200/csrc/pc2_fields.h compiled for the host (tests/pc2_host.cpp): matching, refusals,
    the per-point read against a NumPy structured-dtype decode on every layout, and the relTime expression;
  - the timed oracle (tests/rot_oracle.cpp): without times it is the untimed oracle (orc_extract_rot) byte for byte, and its
    intensity column is a NumPy restatement of the rule (span 0 and non-finite times included);
  - on a fast-turning ring-major (ouster48) sweep the timed de-skew lands every cutted point where it was at the sweep start,
    which the azimuth rule does not."""
import ctypes as C

import numpy as np
import pytest

import pc2_host
import rot_oracle as RT

F32, F64, U8, U16, I32, U32 = 7, 8, 2, 4, 5, 6
E_ARG = -1
Q_LB = np.array([0.999, 0.01, -0.02, 0.03]) / np.linalg.norm([0.999, 0.01, -0.02, 0.03])
STEPS = 1024
FAST_OMEGA = (0.1, -0.05, 1.5)            # rad/s: a vehicle turning fast, pitching and rolling a little


def _same(a, b):
    assert len(a) == len(b), (len(a), len(b))
    assert a.tobytes() == b.tobytes()


@pytest.fixture(scope="module")
def pth():
    return pc2_host.lib()


@pytest.fixture(scope="module")
def sweep128():
    from liliom_b200 import synth
    return synth.make_spinning_sweep(synth.default_true_pose(), synth.uniform_elevations(128), STEPS)


XYZI = [("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("intensity", 12, F32, 1)]


def _match(pth, fields, point_step, name="time", want_ring=False, width=10):
    return pc2_host.match_sources(pth, fields, point_step, want_ring=want_ring, time_name=name, width=width)


def test_each_time_datatype_matches(pth):
    base = (0, 4, 8, 12, 10, -1, 0)
    assert _match(pth, XYZI + [("time", 16, F32, 1)], 20) == (0, base + (16, F32))
    assert _match(pth, XYZI + [("t", 16, U32, 1)], 20, name="t") == (0, base + (16, U32))
    assert _match(pth, XYZI + [("timestamp", 16, F64, 1)], 24, name="timestamp") == (0, base + (16, F64))
    assert _match(pth, XYZI + [("time", 17, F64, 0)], 25) == (0, base + (17, F64))            # count 0 counts as 1, any offset
    # the ring and the time are matched independently
    assert _match(pth, XYZI + [("ring", 16, U16, 1), ("time", 18, F32, 1)], 22, want_ring=True) == (0, (0, 4, 8, 12, 10, 16, 2, 18, F32))
    # a 15-character name is the longest that can match
    assert _match(pth, XYZI + [("a" * 15, 16, F32, 1)], 20, name="a" * 15) == (0, base + (16, F32))


def test_first_matching_time_wins_and_other_datatypes_are_skipped(pth):
    base = (0, 4, 8, 12, 10, -1, 0)
    fields = XYZI + [("time", 16, U16, 1), ("time", 18, I32, 1), ("time", 22, U8, 1), ("time", 24, F32, 2), ("time", 28, U32, 1),
                     ("time", 32, F64, 1)]
    assert _match(pth, fields, 40) == (0, base + (28, U32))
    assert _match(pth, XYZI + [("time", 16, F64, 1), ("time", 24, F32, 1)], 28) == (0, base + (16, F64))
    assert _match(pth, XYZI + [("times", 16, F32, 1), ("Time", 20, F32, 1), ("time", 24, F32, 1)], 28) == (0, base + (24, F32))


def test_missing_count2_or_overrunning_time_is_refused(pth):
    bad = (E_ARG, (-7,) * 9)
    assert _match(pth, XYZI, 16) == bad                                             # no field of that name
    assert _match(pth, XYZI + [("time", 16, F32, 2)], 24) == bad                   # count 2 only
    assert _match(pth, XYZI + [("time", 16, U16, 1)], 18) == bad                   # no accepted datatype
    assert _match(pth, XYZI + [("time", 16, F32, 1)], 19) == bad                   # 4 bytes past point_step
    assert _match(pth, XYZI + [("time", 16, F64, 1)], 23) == bad                   # 8 bytes past point_step
    assert _match(pth, XYZI + [("t", 16, U32, 1)], 20, name="time") == bad          # another name
    # an overrunning field of a skipped datatype is never read: the first accepted match is taken
    assert _match(pth, XYZI + [("time", 16, U16, 8), ("time", 16, F32, 1)], 20) == (0, (0, 4, 8, 12, 10, -1, 0, 16, F32))


def test_without_the_time_source_the_field_is_not_looked_at(pth):
    assert _match(pth, XYZI, 16, name=None) == (0, (0, 4, 8, 12, 10, -1, 0, -1, 0))
    assert _match(pth, XYZI + [("time", 16, F64, 1)], 17, name=None) == (0, (0, 4, 8, 12, 10, -1, 0, -1, 0))


def _numpy_times(msg, name):
    """The time field of every point, row-major, decoded with a NumPy structured dtype (rows stripped of any padding)."""
    from liliom_b200 import synth
    f = [x for x in msg.fields if x[0] == name][0]
    dt = np.dtype({"names": [name], "formats": [synth._PC2_NP[f[2]]], "offsets": [f[1]], "itemsize": msg.point_step})
    rows = np.ascontiguousarray(msg.data.reshape(msg.height, msg.row_step)[:, :msg.width * msg.point_step]).reshape(-1)
    return rows.view(dt)[name].astype(np.float64)


@pytest.mark.parametrize("t0", [0.0, 0.25])
@pytest.mark.parametrize("layout", ["velodyne22", "ouster48", "hesai26"])
def test_host_time_decode_equals_numpy(pth, sweep128, layout, t0):
    from liliom_b200 import synth
    pts, _q, ring, step = sweep128
    name = synth.PC2_TIME_FIELDS[layout]
    msg = synth.encode_pc2(pts, ring, step, layout, steps=STEPS, lines=128, t0=t0)
    m, _keep = msg.c_msg()
    n = msg.width * msg.height
    got = np.full(n, -1.0)
    assert pth.ph_decode_times(C.byref(m), name.encode(), got.ctypes.data_as(C.c_void_p)) == n
    want = _numpy_times(msg, name)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    if layout == "hesai26":                          # 26-byte points: most FLOAT64 stamps are unaligned
        assert msg.point_step == 26 and got.min() >= synth.HESAI_EPOCH
        np.testing.assert_allclose(got - synth.HESAI_EPOCH - t0, step * (0.1 / STEPS), atol=1e-6)
    idx = np.arange(len(pts)) if msg.height == 1 else ring * msg.width + step
    t_start = {"velodyne22": np.float32(t0), "ouster48": round(t0 * 1e9), "hesai26": synth.HESAI_EPOCH + t0}[layout]
    assert got[idx].min() == t_start


def test_without_an_offset_the_existing_layouts_keep_their_times(sweep128):
    """t0 = 0 (the default): velodyne22 `time` and ouster48 `t` are the values those layouts always carried."""
    from liliom_b200 import synth
    pts, _q, ring, step = sweep128
    v = synth.encode_pc2(pts, ring, step, "velodyne22", steps=STEPS, lines=128)
    assert np.array_equal(_numpy_times(v, "time"), (step * (0.1 / STEPS)).astype(np.float32).astype(np.float64))
    o = synth.encode_pc2(pts, ring, step, "ouster48", steps=STEPS, lines=128)
    assert np.array_equal(_numpy_times(o, "t")[ring * STEPS + step], (step * (100_000_000 // STEPS)).astype(np.float64))


def _np_rel(t, t_min, t_max):
    span = t_max - t_min
    return np.zeros(len(t), np.float32) if span == 0 else ((t - t_min) / span).astype(np.float32)


def test_rel_time_expression(pth):
    rng = np.random.default_rng(5)
    for t in (rng.uniform(0, 0.1, 1000), 1.7e9 + rng.uniform(0, 0.1, 1000), rng.integers(0, 100_000_000, 1000).astype(np.float64),
              np.full(10, 3.25)):
        got = np.zeros(len(t), np.float32)
        pth.ph_rel_times(t.ctypes.data_as(C.c_void_p), len(t), t.min(), t.max(), got.ctypes.data_as(C.c_void_p))
        want = _np_rel(t, t.min(), t.max())
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        assert got.min() == 0.0 and got.max() == (1.0 if t.max() > t.min() else 0.0)


# ---------------------------------------------------------------- the oracle's timed mode
@pytest.fixture(scope="module")
def hdl():
    from liliom_b200 import synth
    return synth.make_hdl64_sweep(synth.default_true_pose(), grid=True)


def test_timed_oracle_without_times_is_the_untimed_oracle(oracle, hdl, sweep128):
    pts, q, ring, _step = sweep128
    hp, hq, _hr, _hs = hdl
    ids = RT.scan_ids(hp, 64)
    rings = np.where(ids < 0, 65535, ids)                   # the tables' verdicts as the ring field
    for ds_rate in (1, 4):
        want = oracle.extract_rot(hp, hq, Q_LB, 64, ds_rate)
        got = RT.extract_rot(hp, hq, Q_LB, 64, ds_rate, rings=rings, times=None)
        assert got[0] == want[0] == 0
        for g, w in zip(got[1:], want[1:]):
            _same(g, w)
    want = oracle.extract_rot(hp, hq, Q_LB, 64, 2)
    got = RT.extract_rot(hp, hq, Q_LB, 64, 2, rings=None, times=None)
    assert got[0] == want[0] == 0
    for g, w in zip(got[1:], want[1:]):
        _same(g, w)
    assert RT.extract_rot(hp[:100], hq, Q_LB, 40, 1)[0] == -2      # the tables know 16 / 32 / 64 only
    assert RT.extract_rot(pts[:100], q, Q_LB, 129, 1, rings=ring[:100])[0] == -2


def _np_intensity(pts, ring, times, line_num):
    """NumPy restatement of the rule: (cutted order, intensity) from the points, their rings and their times."""
    x, y, z = (pts[f].astype(np.float32) for f in ("x", "y", "z"))
    with np.errstate(invalid="ignore", over="ignore"):
        keep = np.isfinite(x) & np.isfinite(y) & np.isfinite(z) & ~((x * x + y * y + z * z) < np.float32(9.0)) & np.isfinite(times)
    t = times[keep]
    rel = _np_rel(times, t.min(), t.max())
    idx = np.flatnonzero(keep & (ring >= 0) & (ring < line_num))
    order = idx[np.argsort(ring[idx], kind="stable")]
    inten = (ring[order].astype(np.float64) + 0.1 * rel[order].astype(np.float64)).astype(np.float32)
    return order, inten


def _times_of(step, kind):
    t = 0.25 + step * (0.1 / STEPS)
    if kind == "equal":
        return np.full(len(step), 7.0)
    if kind == "nonfinite":
        t = t.copy()
        t[::97] = np.nan; t[5::389] = np.inf; t[11::1013] = -np.inf
        t[np.argmin(t)] = np.nan                         # the earliest return leaves t_min: the span shrinks
    return t


@pytest.mark.parametrize("kind", ["plain", "equal", "nonfinite"])
@pytest.mark.parametrize("line_num", [128, 40])
def test_timed_oracle_intensity_is_the_rule(sweep128, kind, line_num):
    pts, q, ring, step = sweep128
    times = _times_of(step, kind)
    rc, surf, edge, cut, lab, cur = RT.extract_rot(pts, q, Q_LB, line_num, 1, rings=ring, times=times)
    assert rc == 0
    order, inten = _np_intensity(pts, ring, times, line_num)
    assert len(cut) == len(order)
    assert np.array_equal(cut["intensity"].view(np.uint32), inten.view(np.uint32))
    if kind == "equal":
        assert np.array_equal(cut["intensity"], ring[order].astype(np.float32))
    if kind == "nonfinite":
        assert (~np.isfinite(times)).sum() > 1000 and not np.isin(np.flatnonzero(~np.isfinite(times)), order).any()
    assert len(edge) > 50 and len(surf) > 1000


# ---------------------------------------------------------------- the de-skew lands the points where they were
def _decode_organised(msg, name):
    import pc2_oracle
    from liliom_b200 import synth
    f = [x for x in msg.fields if x[0] == "ring"][0]
    dt = np.dtype({"names": ["ring"], "formats": [synth._PC2_NP[f[2]]], "offsets": [f[1]], "itemsize": msg.point_step})
    return pc2_oracle.pc2_to_pt32(msg), msg.data.view(dt)["ring"].astype(np.int64), _numpy_times(msg, name)


def _ground_truth(cloud, step, q_imu):
    """Each raw return rotated to the sweep start by the synth's own slerp at its firing fraction step / STEPS: d_start * r."""
    from liliom_b200 import synth
    p = np.stack([cloud[f].astype(np.float64) for f in ("x", "y", "z")], 1)
    return synth._rotate_many(synth._slerp_from_identity(np.asarray(q_imu, float), step / float(STEPS)), p)


def deskew_errors(timed):
    """(|cutted - truth| / range per cutted point, bound factor angle(qIMU) / (STEPS - 1)) on the fast-turn ouster48 sweep."""
    from liliom_b200 import synth
    pts, q, ring, step = synth.make_spinning_sweep(synth.default_true_pose(), synth.uniform_elevations(128), STEPS, omega=FAST_OMEGA)
    q = q / np.linalg.norm(q)        # a unit rotation: the de-skew rotates by it as given (a non-unit one also scales the point)
    msg = synth.encode_pc2(pts, ring, step, "ouster48", steps=STEPS, lines=128, t0=0.5)
    cloud, rings, times = _decode_organised(msg, "t")
    ident = (1.0, 0.0, 0.0, 0.0)
    rc, _s, _e, cut, _l, _c = RT.extract_rot(cloud, q, ident, 128, 1, rings=rings, times=times if timed else None)
    assert rc == 0
    order, _ = _np_intensity(cloud, rings, times, 128)
    assert len(order) == len(cut) and len(cut) > 80_000
    truth = _ground_truth(cloud[order], order % msg.width, q)
    got = np.stack([cut[f].astype(np.float64) for f in ("x", "y", "z")], 1)
    rng_m = np.linalg.norm(truth, axis=1)
    angle = 2.0 * np.arccos(min(1.0, abs(q[0])))
    return np.linalg.norm(got - truth, axis=1) / rng_m, angle / (STEPS - 1)


def test_time_field_deskew_lands_the_points_where_they_were():
    err, per_step = deskew_errors(timed=True)
    assert per_step > 1e-4                                          # ~0.15 rad over the sweep
    assert (err <= per_step + 1e-5).all(), (err.max(), per_step)


def test_azimuth_rule_misses_on_a_ring_major_cloud():
    err, per_step = deskew_errors(timed=False)
    miss = err > per_step + 1e-5
    assert miss.mean() > 0.9, miss.mean()           # 99.9 % of the returns on this sweep, median error 2.3 % of the range
