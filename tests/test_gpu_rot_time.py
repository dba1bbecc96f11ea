"""GPU tier for the ROT extractor's time source LILIOM_TIME_FIELD (liliom_set_time_source): relTime from the driver's per-point
PointCloud2 time field instead of the azimuth rule.
  - bit-exact against the timed CPU oracle: the 128 x 1024 sweep as velodyne22 (`time`), ouster48 (`t`) and hesai26
    (`timestamp`) with the ring field, the HDL-64E sweep in ouster48 with the elevation tables, NaN times and equal times;
  - refused calls leave the outputs untouched; the resident pipeline and its invalidation rules; the node mirror;
  - a fast-turning ring-major sweep through scan-to-map end to end."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

Q_LB = np.array([0.999, 0.01, -0.02, 0.03]) / np.linalg.norm([0.999, 0.01, -0.02, 0.03])
F = ["x", "y", "z", "intensity"]
STEPS128 = 1024
FAST_OMEGA = (0.1, -0.05, 1.5)
T0 = {"velodyne22": 0.37, "ouster48": 0.5, "hesai26": 0.0}      # the first return is not at t = 0


def _fields_equal(a, b):
    assert len(a) == len(b), (len(a), len(b))
    for f in F:
        assert np.array_equal(a[f].view(np.uint32), b[f].view(np.uint32)), f


def _same(a, b):
    assert len(a) == len(b), (len(a), len(b))
    assert a.tobytes() == b.tobytes()


def _ctx(line_num, ds_rate, ring_field, time_name):
    import liliom_b200 as L
    p = L.default_params(1)
    p.line_num = line_num; p.ds_rate = ds_rate
    c = L.Context(p)
    if ring_field:
        c.set_ring_source(L.RING_FIELD)
    if time_name is not None:
        c.set_time_source(L.TIME_FIELD, time_name)
    return c


def _field_view(msg, name):
    from liliom_b200 import synth
    f = [x for x in msg.fields if x[0] == name][0]
    assert msg.row_step == msg.width * msg.point_step
    return msg.data.view(np.dtype({"names": [name], "formats": [synth._PC2_NP[f[2]]], "offsets": [f[1]], "itemsize": msg.point_step}))[name]


def _decode(msg, name):
    """(PointXYZI cloud, rings, times) of every point, row-major: the CPU fromROSMsg and NumPy structured-dtype decodes."""
    import pc2_oracle
    return pc2_oracle.pc2_to_pt32(msg), _field_view(msg, "ring").astype(np.int64), _field_view(msg, name).astype(np.float64)


def _with_times(msg, name, values):
    """A copy of msg whose time field holds `values` (one per point, row-major)."""
    import liliom_b200 as L
    data = msg.data.copy()
    m = L.PC2(data, msg.height, msg.width, msg.point_step, msg.row_step, msg.fields)
    v = _field_view(m, name)
    v[...] = np.asarray(values).astype(v.dtype)
    return m


def _extract(c, msg, q):
    surf, edge, cut = c.extract_rot_pc2(msg, q, Q_LB)
    lab, cur = c.extract_rot_labels(len(cut))
    return [a.copy() for a in (surf, edge, cut, lab, cur)]


def _check_against_oracle(c, msg, q, rings, times, cloud, line_num, ds_rate):
    import rot_time_oracle as RT
    surf, edge, cut, lab, cur = _extract(c, msg, q)
    rc, surf_o, edge_o, cut_o, lab_o, cur_o = RT.extract_rot_timed(cloud, rings, times, q, Q_LB, line_num, ds_rate)
    assert rc == 0
    _fields_equal(cut, cut_o); _fields_equal(edge, edge_o); _fields_equal(surf, surf_o)
    assert np.array_equal(lab, lab_o) and np.array_equal(cur.view(np.uint32), cur_o.view(np.uint32))
    assert len(edge) > 50 and len(surf) > 1000
    return cut


@pytest.fixture(scope="module")
def s128(world_small):
    from liliom_b200 import synth
    pts, q, ring, step = synth.make_spinning_sweep(world_small["T"], synth.uniform_elevations(128), STEPS128, omega=FAST_OMEGA)
    msgs = {lay: synth.encode_pc2(pts, ring, step, lay, steps=STEPS128, lines=128, t0=T0[lay]) for lay in T0}
    return pts, q, ring, step, msgs


@pytest.mark.parametrize("ds_rate", [1, 2, 4])
@pytest.mark.parametrize("layout", ["velodyne22", "ouster48", "hesai26"])
def test_time_field_against_the_oracle(s128, layout, ds_rate):
    from liliom_b200 import synth
    pts, q, ring, step, msgs = s128
    msg = msgs[layout]
    name = synth.PC2_TIME_FIELDS[layout]
    cloud, rings, times = _decode(msg, name)
    c = _ctx(128, ds_rate, True, name)
    cut = _check_against_oracle(c, msg, q, rings, times, cloud, 128, ds_rate)
    frac = cut["intensity"] - np.floor(cut["intensity"])
    assert frac.min() == 0.0 and frac.max() > 0.0999           # relTime spans [0, 1]
    c.close()


@pytest.mark.parametrize("ds_rate", [1, 2, 4])
def test_hdl64_ouster48_with_the_elevation_tables(world_small, ds_rate):
    from liliom_b200 import synth
    pts, q, ring, step = synth.make_hdl64_sweep(world_small["T"], grid=True)
    msg = synth.encode_pc2(pts, ring, step, "ouster48", t0=0.125)
    cloud, _rings, times = _decode(msg, "t")
    c = _ctx(64, ds_rate, False, "t")
    _check_against_oracle(c, msg, q, None, times, cloud, 64, ds_rate)
    c.close()


@pytest.mark.parametrize("layout", ["velodyne22", "hesai26"])
def test_nan_times_are_dropped(s128, layout):
    from liliom_b200 import synth
    pts, q, ring, step, msgs = s128
    name = synth.PC2_TIME_FIELDS[layout]
    _, _, t = _decode(msgs[layout], name)
    t = t.copy()
    t[::97] = np.nan; t[5::389] = np.inf; t[11::1013] = -np.inf
    t[np.argmin(t)] = np.nan
    msg = _with_times(msgs[layout], name, t)
    cloud, rings, times = _decode(msg, name)
    assert (~np.isfinite(times)).sum() > 1000
    for ds_rate in (1, 4):
        c = _ctx(128, ds_rate, True, name)
        _check_against_oracle(c, msg, q, rings, times, cloud, 128, ds_rate)
        c.close()


@pytest.mark.parametrize("layout", ["ouster48", "hesai26"])
def test_equal_times(s128, layout):
    from liliom_b200 import synth
    pts, q, ring, step, msgs = s128
    name = synth.PC2_TIME_FIELDS[layout]
    msg = _with_times(msgs[layout], name, np.full(msgs[layout].width * msgs[layout].height, 12345))
    cloud, rings, times = _decode(msg, name)
    for ds_rate in (1, 4):
        c = _ctx(128, ds_rate, True, name)
        cut = _check_against_oracle(c, msg, q, rings, times, cloud, 128, ds_rate)
        assert np.array_equal(cut["intensity"], np.floor(cut["intensity"]))      # relTime 0 everywhere
        c.close()


def _call_rot_pc2(c, cm, q, n):
    """liliom_extract_rot_pc2 into 0x5C-filled buffers with counts preset to -3: (rc, untouched)."""
    import liliom_b200 as L
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    ql = np.asarray(Q_LB, np.float64); q = np.asarray(q, np.float64)
    bufs = [np.full(n * 32, 0x5C, np.uint8) for _ in range(3)]
    cnt = [C.c_int(-3) for _ in range(3)]
    rc = L._binding.lib().liliom_extract_rot_pc2(c._h, C.byref(cm), dp(q), dp(ql), bufs[0].ctypes.data_as(C.c_void_p), n, C.byref(cnt[0]),
                                                 bufs[1].ctypes.data_as(C.c_void_p), n, C.byref(cnt[1]),
                                                 bufs[2].ctypes.data_as(C.c_void_p), n, C.byref(cnt[2]))
    return rc, all((b == 0x5C).all() for b in bufs) and all(x.value == -3 for x in cnt)


def test_refusals_leave_the_outputs_untouched(s128):
    import liliom_b200 as L
    E = L._binding
    lib = E.lib()
    pts, q, ring, step, msgs = s128
    m = msgs["velodyne22"]
    n = m.width
    c = _ctx(128, 4, True, "time")
    want = _extract(c, m, q)
    re = lambda fn: [(f[0],) + fn(f) if f[0] == "time" else f for f in m.fields]
    bad_msgs = {"no time field": [f for f in m.fields if f[0] != "time"],
                "UINT16 time": re(lambda f: (f[1], 4, f[3])),
                "count 2": re(lambda f: (f[1], f[2], 2)),
                "overrun": re(lambda f: (m.point_step - 2, f[2], f[3]))}
    for what, fields in bad_msgs.items():
        bad = L.PC2(m.data, m.height, m.width, m.point_step, m.row_step, fields)
        cm, _keep = bad.c_msg()
        rc, untouched = _call_rot_pc2(c, cm, q, n)
        assert rc == E.E_ARG and untouched, what
        conv = np.full(n * 32, 0x5C, np.uint8); k = C.c_int(-3)
        assert lib.liliom_convert_pc2(c._h, C.byref(cm), conv.ctypes.data_as(C.c_void_p), n, C.byref(k)) == E.E_ARG, what
        assert (conv == 0x5C).all() and k.value == -3, what
        # the same message is fine for the azimuth rule, which does not read the time
        ca = _ctx(128, 4, True, None)
        assert ca.convert_pc2(bad, download=False) == n
        ca.close()
    # names: NULL, 16 characters; another source; a 48-byte context
    for bad_name in (None, "a" * 16):
        assert lib.liliom_set_time_source(c._h, E.TIME_FIELD, None if bad_name is None else bad_name.encode()) == E.E_ARG
    for bad_src in (-1, 2):
        assert lib.liliom_set_time_source(c._h, bad_src, b"time") == E.E_ARG
    c48 = L.Context(variant=0)
    assert lib.liliom_set_time_source(c48._h, E.TIME_FIELD, b"time") == E.E_ARG
    c48.set_time_source(L.TIME_AZIMUTH)
    c48.close()
    # the refused calls left the setting as it was
    for g, w in zip(_extract(c, m, q), want):
        _same(g, w)
    # host 32-byte points carry no time (also with the elevation tables)
    ct = _ctx(64, 4, False, "time")
    for cc in (c, ct):
        with pytest.raises(L.LiliomError) as e:
            cc.extract_rot(pts, q, Q_LB)
        assert e.value.code == E.E_ARG
    ct.close()
    # no times resident after upload_scan or any set_time_source call; convert_pc2 in FIELD mode makes them resident
    c.upload_scan(pts)
    with pytest.raises(L.LiliomError) as e:
        c.extract_resident(q, Q_LB)
    assert e.value.code == E.E_ARG
    assert c.convert_pc2(m, download=False) == n
    assert c.extract_resident(q, Q_LB)[0] == len(want[0])
    c.set_time_source(L.TIME_FIELD, "time")
    with pytest.raises(L.LiliomError) as e:
        c.extract_resident(q, Q_LB)
    assert e.value.code == E.E_ARG
    # decoded under the azimuth rule: no times resident for a later switch to the field
    c.set_time_source(L.TIME_AZIMUTH)
    assert c.convert_pc2(m, download=False) == n
    c.set_time_source(L.TIME_FIELD, "time")
    with pytest.raises(L.LiliomError) as e:
        c.extract_resident(q, Q_LB)
    assert e.value.code == E.E_ARG
    # the context still gives the same clouds
    for g, w in zip(_extract(c, m, q), want):
        _same(g, w)
    c.close()


def test_azimuth_default_is_unchanged(s128):
    """A context that set the field and went back to TIME_AZIMUTH gives a fresh context's bytes."""
    import liliom_b200 as L
    pts, q, ring, step, msgs = s128
    for layout in ("velodyne22", "ouster48"):
        a, b = _ctx(128, 4, True, None), _ctx(128, 4, True, "time")
        b.set_time_source(L.TIME_AZIMUTH, None)
        for x, y in zip(_extract(a, msgs[layout], q), _extract(b, msgs[layout], q)):
            _same(x, y)
        a.close(); b.close()


@pytest.mark.parametrize("layout", ["velodyne22", "ouster48", "hesai26"])
def test_resident_pipeline_matches_the_host_path(s128, world_small, layout):
    """convert_pc2 -> extract_resident -> odometry_resident gives the pose of extract_rot_pc2 -> odometry (host surf cloud)."""
    import liliom_b200 as L
    from liliom_b200 import synth
    pts, q, ring, step, msgs = s128
    msg = msgs[layout]
    n = msg.width * msg.height
    out = []
    for resident in (True, False):
        c = _ctx(128, 4, True, synth.PC2_TIME_FIELDS[layout])
        c.map_set_points(world_small["map"])
        if resident:
            assert c.convert_pc2(msg, download=False) == n
            ns, _, _ = c.extract_resident(q, Q_LB)
            assert ns > 1000
            pose, _, ds = c.odometry_resident(world_small["guess"], 4, mode=L.MODE_GN, want_ds=True, cap=n, want_stats=False)
        else:
            surf, _, _ = c.extract_rot_pc2(msg, q, Q_LB)
            pose, _, ds = c.odometry(surf, world_small["guess"], 4, mode=L.MODE_GN, want_stats=False)
        out.append((pose.copy(), ds.tobytes()))
        c.close()
    assert out[0][0].tobytes() == out[1][0].tobytes() and out[0][1] == out[1][1] and len(out[0][1]) > 0


def test_preprocessing_node_on_a_time_field_context(world_small):
    """liliom_pre_cloud_pc2 on a time-field context returns liliom_extract_rot_pc2's clouds for the message it processed."""
    import liliom_b200 as L
    from liliom_b200 import synth
    seq = {}
    for k in range(5):
        pts, _, ring, step = synth.make_spinning_sweep(world_small["T"], synth.uniform_elevations(128), STEPS128, seed=60 + k)
        seq[round(0.1 * k, 6)] = synth.encode_pc2(pts, ring, step, "ouster48", steps=STEPS128, lines=128, t0=0.1 * k)
    ca, cb = _ctx(128, 4, True, "t"), _ctx(128, 4, True, "t")
    node = L.PreprocessingNode(ca, q_lb=Q_LB)
    t_imu = 0.0
    got = 0
    for stamp, msg in seq.items():
        while t_imu < stamp + 0.1501:
            node.imu(t_imu, (0.02 * np.sin(3 * t_imu), -0.01, 0.2 + 0.05 * np.cos(2 * t_imu)))
            t_imu += 0.005
        a = node.cloud_pc2(stamp, msg)
        if a is None:
            continue
        got += 1
        want = cb.extract_rot_pc2(seq[round(a[0], 6)], a[4], Q_LB)
        for x, y in zip(a[1:4], want):
            _same(x, y)
        assert len(a[1]) > 1000
    assert got == 3
    node.close(); ca.close(); cb.close()


def _rot_angle(qa, qb):
    qa = qa / np.linalg.norm(qa); qb = qb / np.linalg.norm(qb)
    return 2.0 * np.arccos(min(1.0, abs(float(np.dot(qa, qb)))))


def test_fast_turn_ring_major_sweep_scan_to_map_end_to_end(oracle):
    """The fast-turn ouster48 sweep through the time-field extractor and liliom_odometry (GN, 10 iterations) against a 2 M-point
    map: the oracle's pose on the oracle's clouds within 1e-4 m / 1e-4 rad.  Each mode's distance from the true pose is printed."""
    import liliom_b200 as L
    import rot_time_oracle as RT
    from liliom_b200 import synth
    m, _ = synth.make_map(2_000_000)
    T = synth.default_true_pose()
    pts, q, ring, step = synth.make_spinning_sweep(T, synth.uniform_elevations(128), STEPS128, omega=FAST_OMEGA)
    msg = synth.encode_pc2(pts, ring, step, "ouster48", steps=STEPS128, lines=128, t0=0.5)
    cloud, rings, times = _decode(msg, "t")
    guess = synth.perturbed_pose(T)
    ident = (1.0, 0, 0, 0)
    report = {}
    for name in ("t", None):
        c = _ctx(128, 4, True, name)
        c.map_set_points(m)
        surf, edge, cut = c.extract_rot_pc2(msg, q, ident)
        rc, surf_o, edge_o, cut_o, _, _ = RT.extract_rot_timed(cloud, rings, times if name else None, q, ident, 128, 4)
        assert rc == 0
        _fields_equal(surf, surf_o); _fields_equal(edge, edge_o); _fields_equal(cut, cut_o)
        ds_o = oracle.voxelgrid(surf_o, 0.4)
        pose, _, ds = c.odometry(surf, guess, 10, mode=L.MODE_GN)
        _fields_equal(ds, ds_o)
        rc, pose_o, _ = oracle.scan_to_map_gn(oracle.KdTree(m), ds_o, guess, 10, 8)
        if name:
            assert np.linalg.norm(pose[4:] - pose_o[4:]) < 1e-4, (pose, pose_o)
            assert _rot_angle(pose[:4], pose_o[:4]) < 1e-4, (pose, pose_o)
        report["time field" if name else "azimuth rule"] = (float(np.linalg.norm(pose[4:] - T[4:])), _rot_angle(pose[:4], T[:4]))
        c.close()
    for k, (dt, dr) in report.items():
        print(f"[fast-turn ouster48, {k}] distance from the true pose: {dt * 100:.2f} cm, {np.degrees(dr):.4f} deg")
