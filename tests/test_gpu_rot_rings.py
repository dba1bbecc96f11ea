"""GPU tier for the ROT extractor's ring source LILIOM_RING_FIELD (liliom_set_ring_source): scanID from the driver's
PointCloud2 `ring` field, for spinning LiDARs of any beam layout up to 128 rings.
  - table identity: with the elevation tables' own verdicts in the ring field, FIELD mode gives ELEVATION mode's bytes;
  - a 128-ring Ouster-like sweep (packed and organised, u8 and u16 rings) against the CPU oracle, and line_num 40 on it;
  - refused calls leave the outputs untouched; the resident pipeline, the node mirror and scan-to-map end to end."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

Q_LB = np.array([0.999, 0.01, -0.02, 0.03]) / np.linalg.norm([0.999, 0.01, -0.02, 0.03])
F = ["x", "y", "z", "intensity"]
SUBSAMPLE = {16: 3, 32: 2, 64: 1}
STEPS128 = 1024


def _fields_equal(a, b):
    assert len(a) == len(b), (len(a), len(b))
    for f in F:
        assert np.array_equal(a[f].view(np.uint32), b[f].view(np.uint32)), f


def _same(a, b):
    assert len(a) == len(b), (len(a), len(b))
    assert a.tobytes() == b.tobytes()


def _ctx(line_num, ds_rate, field):
    import liliom_b200 as L
    p = L.default_params(1)
    p.line_num = line_num; p.ds_rate = ds_rate
    c = L.Context(p)
    if field:
        c.set_ring_source(L.RING_FIELD)
    return c


def _ring_field(msg):
    return [f for f in msg.fields if f[0] == "ring"][0]


def _ring_dtype(msg):
    from liliom_b200 import synth
    f = _ring_field(msg)
    return np.dtype({"names": ["ring"], "formats": [synth._PC2_NP[f[2]]], "offsets": [f[1]], "itemsize": msg.point_step})


def _decode_rings(msg):
    """The ring field of every point, row-major (NumPy structured dtype; the synthetic layouts have no row padding)."""
    assert msg.row_step == msg.width * msg.point_step
    return msg.data.view(_ring_dtype(msg))["ring"].astype(np.int64)


def _set_rings(msg, values):
    """A copy of msg whose ring field holds `values` (one per point, row-major); -1 becomes the type's maximum (out of range)."""
    import liliom_b200 as L
    assert msg.row_step == msg.width * msg.point_step
    data = msg.data.copy()
    rec = data.view(_ring_dtype(msg))
    top = np.iinfo(rec["ring"].dtype).max
    rec["ring"] = np.where(np.asarray(values) < 0, top, values).astype(rec["ring"].dtype)
    return L.PC2(data, msg.height, msg.width, msg.point_step, msg.row_step, msg.fields)


def _extract(c, msg, q):
    surf, edge, cut = c.extract_rot_pc2(msg, q, Q_LB)
    lab, cur = c.extract_rot_labels(len(cut))
    return [a.copy() for a in (surf, edge, cut, lab, cur)]


@pytest.fixture(scope="module")
def hdl(world_small):
    from liliom_b200 import synth
    pts, q, ring, step = synth.make_hdl64_sweep(world_small["T"], grid=True)
    return pts, q, ring, step


@pytest.fixture(scope="module")
def s128(world_small):
    from liliom_b200 import synth
    pts, q, ring, step = synth.make_spinning_sweep(world_small["T"], synth.uniform_elevations(128), STEPS128)
    msgs = {lay: synth.encode_pc2(pts, ring, step, lay, steps=STEPS128, lines=128) for lay in ("velodyne22", "pcl32", "ouster48")}
    return pts, q, ring, step, msgs


@pytest.mark.parametrize("layout", ["velodyne22", "pcl32", "ouster48"])
@pytest.mark.parametrize("lines", [16, 32, 64])
def test_table_identity_on_the_device(hdl, layout, lines):
    import pc2_oracle
    import rot_oracle as R
    from liliom_b200 import synth
    pts, q, ring, step = hdl
    k = SUBSAMPLE[lines]
    msg = synth.encode_pc2(pts[::k].copy(), ring[::k], step[::k], layout)
    msg = _set_rings(msg, R.scan_ids(pc2_oracle.pc2_to_pt32(msg), lines))
    for ds_rate in (1, 2, 4):
        ce, cf = _ctx(lines, ds_rate, False), _ctx(lines, ds_rate, True)
        want = _extract(ce, msg, q)
        got = _extract(cf, msg, q)
        for g, w in zip(got, want):
            _same(g, w)
        assert len(want[1]) > 10 and len(want[0]) > 100, (lines, ds_rate)
        ce.close(); cf.close()


@pytest.mark.parametrize("ds_rate", [1, 2, 4])
@pytest.mark.parametrize("layout", ["velodyne22", "pcl32", "ouster48"])
def test_128_rings_against_the_oracle(s128, layout, ds_rate):
    import pc2_oracle
    import rot_oracle as R
    pts, q, ring, step, msgs = s128
    msg = msgs[layout]
    cloud = pc2_oracle.pc2_to_pt32(msg)
    rings = _decode_rings(msg)
    for line_num in (128, 40):
        c = _ctx(line_num, ds_rate, True)
        surf, edge, cut, lab, cur = _extract(c, msg, q)
        rc, surf_o, edge_o, cut_o, lab_o, cur_o = R.extract_rot(cloud, q, Q_LB, line_num, ds_rate, rings=rings)
        assert rc == 0
        _fields_equal(cut, cut_o); _fields_equal(edge, edge_o); _fields_equal(surf, surf_o)
        assert np.array_equal(lab, lab_o) and np.array_equal(cur.view(np.uint32), cur_o.view(np.uint32))
        assert cut["intensity"].astype(np.int32).max() == line_num - 1
        if line_num == 128:
            assert len(edge) > 50 and len(surf) > 1000
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
    c = _ctx(128, 4, True)
    want = _extract(c, m, q)
    no_ring = L.PC2(m.data, m.height, m.width, m.point_step, m.row_step, [f for f in m.fields if f[0] != "ring"])
    f32_ring = L.PC2(m.data, m.height, m.width, m.point_step, m.row_step,
                     [(f[0], f[1], 7 if f[0] == "ring" else f[2], f[3]) for f in m.fields])
    for what, bad in (("no ring field", no_ring), ("FLOAT32 ring", f32_ring)):
        cm, _keep = bad.c_msg()
        rc, untouched = _call_rot_pc2(c, cm, q, n)
        assert rc == E.E_ARG and untouched, what
        conv = np.full(n * 32, 0x5C, np.uint8); k = C.c_int(-3)
        assert lib.liliom_convert_pc2(c._h, C.byref(cm), conv.ctypes.data_as(C.c_void_p), n, C.byref(k)) == E.E_ARG, what
        assert (conv == 0x5C).all() and k.value == -3, what
        # the same message is fine for the elevation tables, which do not read the ring
        ce = _ctx(64, 4, False)
        assert ce.convert_pc2(bad, download=False) == n
        ce.close()
    for lines in (0, 129):
        cl = _ctx(lines, 4, True)
        cm, _keep = m.c_msg()
        rc, untouched = _call_rot_pc2(cl, cm, q, n)
        assert rc == E.E_LINES and untouched, lines
        cl.close()
    # host 32-byte points carry no ring
    with pytest.raises(L.LiliomError) as e:
        c.extract_rot(pts, q, Q_LB)
    assert e.value.code == E.E_ARG
    # no ring ids resident after upload_scan or a change of the source; convert_pc2 in FIELD mode makes them resident
    c.upload_scan(pts)
    with pytest.raises(L.LiliomError) as e:
        c.extract_resident(q, Q_LB)
    assert e.value.code == E.E_ARG
    assert c.convert_pc2(m, download=False) == n
    assert c.extract_resident(q, Q_LB)[0] == len(want[0])
    c.set_ring_source(L.RING_ELEVATION); c.set_ring_source(L.RING_FIELD)
    with pytest.raises(L.LiliomError) as e:
        c.extract_resident(q, Q_LB)
    assert e.value.code == E.E_ARG
    # the context still gives the same clouds
    for g, w in zip(_extract(c, m, q), want):
        _same(g, w)
    # the source setting itself
    for bad_src in (-1, 2):
        with pytest.raises(L.LiliomError) as e:
            c.set_ring_source(bad_src)
        assert e.value.code == E.E_ARG
    c48 = L.Context(variant=0)
    with pytest.raises(L.LiliomError) as e:
        c48.set_ring_source(L.RING_FIELD)
    assert e.value.code == E.E_ARG
    c48.set_ring_source(L.RING_ELEVATION)
    c48.close(); c.close()


@pytest.mark.parametrize("layout", ["velodyne22", "ouster48"])
def test_resident_pipeline_matches_the_host_path(s128, world_small, layout):
    """convert_pc2 -> extract_resident -> odometry_resident gives the pose of extract_rot_pc2 -> odometry (host surf cloud), each
    on a fresh context so that both solves take the same launch shape."""
    import liliom_b200 as L
    pts, q, ring, step, msgs = s128
    msg = msgs[layout]
    n = msg.width * msg.height
    out = []
    for resident in (True, False):
        c = _ctx(128, 4, True)
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


def test_preprocessing_node_on_a_field_context(world_small):
    """liliom_pre_cloud_pc2 on a FIELD context returns liliom_extract_rot_pc2's clouds for the message it processed."""
    import liliom_b200 as L
    from liliom_b200 import synth
    seq = {}
    for k in range(5):
        pts, _, ring, step = synth.make_spinning_sweep(world_small["T"], synth.uniform_elevations(128), STEPS128, seed=60 + k)
        seq[round(0.1 * k, 6)] = synth.encode_pc2(pts, ring, step, ("velodyne22", "ouster48")[k % 2], steps=STEPS128, lines=128)
    ca, cb = _ctx(128, 4, True), _ctx(128, 4, True)
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


def test_128_beam_sweep_scan_to_map_end_to_end(oracle):
    """The 128-beam sweep through the FIELD extractor and liliom_odometry (GN, 10 iterations) against a 2 M-point map, within
    the tolerance the 64-beam sweep's end-to-end test uses."""
    import liliom_b200 as L
    import pc2_oracle
    import rot_oracle as R
    from liliom_b200 import synth
    m, _ = synth.make_map(2_000_000)
    T = synth.default_true_pose()
    pts, q, ring, step = synth.make_spinning_sweep(T, synth.uniform_elevations(128), STEPS128)
    msg = synth.encode_pc2(pts, ring, step, "velodyne22", steps=STEPS128, lines=128)
    guess = synth.perturbed_pose(T)
    c = _ctx(128, 4, True)
    c.map_set_points(m)
    surf, edge, cut = c.extract_rot_pc2(msg, q, (1.0, 0, 0, 0))
    rc, surf_o, edge_o, cut_o, _, _ = R.extract_rot(pc2_oracle.pc2_to_pt32(msg), q, (1.0, 0, 0, 0), 128, 4, rings=ring)
    _fields_equal(surf, surf_o); _fields_equal(edge, edge_o); _fields_equal(cut, cut_o)
    ds_o = oracle.voxelgrid(surf_o, 0.4)
    pose, _, ds = c.odometry(surf, guess, 10, mode=L.MODE_GN)
    _fields_equal(ds, ds_o)
    rc, pose_o, _ = oracle.scan_to_map_gn(oracle.KdTree(m), ds_o, guess, 10, 8)
    assert np.linalg.norm(pose[4:] - pose_o[4:]) < 1e-4, (pose, pose_o)
    qa = pose[:4] / np.linalg.norm(pose[:4]); qb = pose_o[:4] / np.linalg.norm(pose_o[:4])
    assert 2.0 * np.arccos(min(1.0, abs(float(np.dot(qa, qb))))) < 1e-4, (pose, pose_o)
    c.close()
