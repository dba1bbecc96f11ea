"""GPU tier for the PointCloud2 ingest of the ROT package (SURVEY §8 f3): pcl::fromROSMsg on the device (liliom_convert_pc2,
liliom_extract_rot_pc2, liliom_pre_cloud_pc2) on the 130k-point HDL sweep encoded in four driver layouts, against the CPU
decode (tests/pc2_oracle.cpp), the 32-byte host path and the CPU oracle of the extractor."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LAYOUTS = ["velodyne22", "pcl32", "ouster48", "organised_nan"]
Q_LB = np.array([0.999, 0.01, -0.02, 0.03]) / np.linalg.norm([0.999, 0.01, -0.02, 0.03])
F = ["x", "y", "z", "intensity"]


def _fields_equal(a, b):
    assert len(a) == len(b), (len(a), len(b))
    for f in F:
        assert np.array_equal(a[f].view(np.uint32), b[f].view(np.uint32)), f


@pytest.fixture(scope="module")
def msgs(world_small):
    from liliom_b200 import synth
    pts, q, ring, step = synth.make_hdl64_sweep(world_small["T"], grid=True)
    assert pts.tobytes() == world_small["hdl"].tobytes() and np.array_equal(q, world_small["q_hdl"])
    return {lay: synth.encode_pc2(pts, ring, step, lay) for lay in LAYOUTS}


@pytest.fixture(scope="module")
def ctxs():
    import liliom_b200 as L
    out = {}
    for ds in (1, 4):
        p = L.default_params(1)
        p.ds_rate = ds
        out[ds] = L.Context(p)
    yield out
    for c in out.values():
        c.close()


@pytest.mark.parametrize("layout", LAYOUTS)
def test_convert_pc2_equals_cpu_decode(ctxs, msgs, layout):
    import pc2_oracle
    msg = msgs[layout]
    ref = pc2_oracle.pc2_to_pt32(msg)
    got = ctxs[4].convert_pc2(msg)
    assert len(got) == msg.width * msg.height and got.tobytes() == ref.tobytes()


@pytest.mark.parametrize("ds_rate", [1, 4])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_extract_rot_pc2_equals_host_path_and_oracle(ctxs, msgs, oracle, world_small, layout, ds_rate):
    import pc2_oracle
    c = ctxs[ds_rate]
    msg = msgs[layout]
    cloud = pc2_oracle.pc2_to_pt32(msg)
    q = world_small["q_hdl"]
    surf_h, edge_h, cut_h = c.extract_rot(cloud, q, Q_LB)
    lab_h, cur_h = c.extract_rot_labels(len(cut_h))
    surf, edge, cut = c.extract_rot_pc2(msg, q, Q_LB)
    lab, cur = c.extract_rot_labels(len(cut))
    for got, ref in ((surf, surf_h), (edge, edge_h), (cut, cut_h)):
        assert len(got) == len(ref) and got.tobytes() == ref.tobytes()
    assert lab.tobytes() == lab_h.tobytes() and cur.tobytes() == cur_h.tobytes()
    rc, surf_o, edge_o, cut_o, lab_o, cur_o = oracle.extract_rot(cloud, q, Q_LB, 64, ds_rate)
    _fields_equal(cut, cut_o); _fields_equal(edge, edge_o); _fields_equal(surf, surf_o)
    assert np.array_equal(lab, lab_o) and np.array_equal(cur.view(np.uint32), cur_o.view(np.uint32))
    assert len(edge) > 50 and len(surf) > 1000


def test_empty_messages(ctxs, msgs, world_small):
    import liliom_b200 as L
    c = ctxs[4]
    for lay in LAYOUTS:
        m = msgs[lay]
        for h, w in ((1, 0), (0, m.width), (0, 0)):
            e = L.PC2(np.zeros(0, np.uint8), h, w, m.point_step, w * m.point_step, m.fields)
            assert len(c.convert_pc2(e)) == 0 and c.convert_pc2(e, download=False) == 0
            surf, edge, cut = c.extract_rot_pc2(e, world_small["q_hdl"], Q_LB)
            assert len(surf) == len(edge) == len(cut) == 0


def _bad_messages(m):
    """Header variants of a valid message that must be refused: (what, msg, keep-alive)."""
    import liliom_b200 as L
    out = []

    def variant(what, **kw):
        a = dict(data=m.data, height=m.height, width=m.width, point_step=m.point_step, row_step=m.row_step, fields=m.fields,
                 is_bigendian=m.is_bigendian)
        raw = kw.pop("raw", None)
        a.update(kw)
        msg = L.PC2(**a)
        cm, keep = msg.c_msg()
        if raw:
            raw(cm)
        out.append((what, cm, keep))

    variant("point_step 0", point_step=0)
    variant("short row_step", row_step=m.width * m.point_step - 1)
    variant("field past point_step", fields=[(n, m.point_step - 2 if n == "intensity" else o, d, c) for n, o, d, c in m.fields])
    variant("big-endian", is_bigendian=True)
    variant("null data", raw=lambda cm: setattr(cm, "data", None))
    variant("null fields", raw=lambda cm: setattr(cm, "fields", C.POINTER(L._binding.Pc2Field)()))
    variant("negative n_fields", raw=lambda cm: setattr(cm, "n_fields", -1))
    variant("2^31 points", raw=lambda cm: (setattr(cm, "height", 2), setattr(cm, "width", 1 << 30), setattr(cm, "point_step", 1),
                                           setattr(cm, "row_step", 1 << 30), setattr(cm, "n_fields", 0)))
    return out


def test_rejected_messages_change_nothing(ctxs, msgs, world_small):
    import liliom_b200 as L
    lib = L._binding.lib()
    c = ctxs[4]
    m = msgs["velodyne22"]
    q = np.asarray(world_small["q_hdl"], np.float64); ql = np.asarray(Q_LB, np.float64)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    want = c.extract_rot_pc2(m, q, Q_LB)
    want = [w.copy() for w in want]
    n = m.width
    for what, cm, _keep in _bad_messages(m):
        bufs = [np.full(n * 32, 0x5C, np.uint8) for _ in range(3)]
        cnt = [C.c_int(-3) for _ in range(3)]
        rc = lib.liliom_extract_rot_pc2(c._h, C.byref(cm), dp(q), dp(ql), bufs[0].ctypes.data_as(C.c_void_p), n, C.byref(cnt[0]),
                                        bufs[1].ctypes.data_as(C.c_void_p), n, C.byref(cnt[1]), bufs[2].ctypes.data_as(C.c_void_p), n,
                                        C.byref(cnt[2]))
        assert rc == L._binding.E_ARG, what
        assert all((b == 0x5C).all() for b in bufs) and all(x.value == -3 for x in cnt), what
        conv = np.full(n * 32, 0x5C, np.uint8); k = C.c_int(-3)
        assert lib.liliom_convert_pc2(c._h, C.byref(cm), conv.ctypes.data_as(C.c_void_p), n, C.byref(k)) == L._binding.E_ARG, what
        assert (conv == 0x5C).all() and k.value == -3, what
        got = c.extract_rot_pc2(m, q, Q_LB)                 # the context is still usable and gives the same clouds
        for g, w in zip(got, want):
            assert g.tobytes() == w.tobytes(), what
    # a caller buffer one point short: E_CAPACITY, the size reported, nothing written
    cm, _keep = m.c_msg()
    conv = np.full((n - 1) * 32, 0x5C, np.uint8); k = C.c_int(-3)
    assert lib.liliom_convert_pc2(c._h, C.byref(cm), conv.ctypes.data_as(C.c_void_p), n - 1, C.byref(k)) == L._binding.E_CAPACITY
    assert (conv == 0x5C).all() and k.value == n
    # a 48-byte (Horizon) context has no PointCloud2 ingest
    c48 = L.Context(variant=0)
    with pytest.raises(L.LiliomError) as e:
        c48.convert_pc2(m)
    assert e.value.code == L._binding.E_ARG
    with pytest.raises(L.LiliomError) as e:
        c48.extract_rot_pc2(m, q, Q_LB)
    assert e.value.code == L._binding.E_ARG
    c48.close()


@pytest.mark.parametrize("layout", ["velodyne22", "ouster48"])
def test_resident_pipeline_matches_host_pt32(msgs, world_small, layout):
    """convert_pc2(download=False) -> extract_resident -> odometry_resident gives the pose of upload_scan(decoded cloud) -> the
    same two calls (each on a fresh context, so that both solves take the same launch shape)."""
    import liliom_b200 as L
    import pc2_oracle
    msg = msgs[layout]
    poses = []
    for via_pc2 in (True, False):
        c = L.Context(variant=1)
        c.map_set_points(world_small["map"])
        if via_pc2:
            assert c.convert_pc2(msg, download=False) == msg.width * msg.height
        else:
            c.upload_scan(pc2_oracle.pc2_to_pt32(msg))
        c.extract_resident(world_small["q_hdl"], Q_LB)
        pose, _, ds = c.odometry_resident(world_small["guess"], 4, mode=L.MODE_GN, want_ds=True, cap=msg.width * msg.height,
                                          want_stats=False)
        poses.append((pose.copy(), ds.tobytes()))
        c.close()
    assert poses[0][0].tobytes() == poses[1][0].tobytes() and poses[0][1] == poses[1][1]
    assert len(poses[0][1]) > 0


def test_preprocessing_node_pc2_sequence(world_small):
    """liliom_pre_cloud_pc2 on six driver messages (every layout, a refused message in between) against liliom_pre_cloud fed
    the decoded clouds: same processed scans, stamps, q_iMU and clouds."""
    import liliom_b200 as L
    import pc2_oracle
    from liliom_b200 import synth
    T = world_small["T"]
    seq = []
    for k in range(6):
        pts, _, ring, step = synth.make_hdl64_sweep(T, seed=60 + k, grid=True)
        seq.append(synth.encode_pc2(pts, ring, step, LAYOUTS[k % 4]))
    ca, cb = L.Context(variant=1), L.Context(variant=1)
    na, nb = L.PreprocessingNode(ca, q_lb=Q_LB), L.PreprocessingNode(cb, q_lb=Q_LB)
    t_imu = 0.0
    got, want = [], []
    for k, msg in enumerate(seq):
        stamp = 0.1 * k
        while t_imu < stamp + 0.1501:
            g = (0.02 * np.sin(3 * t_imu), -0.01, 0.2 + 0.05 * np.cos(2 * t_imu))
            na.imu(t_imu, g); nb.imu(t_imu, g)
            t_imu += 0.005
        if k == 3:                                        # refused: not queued, the sequence continues as if it had not come
            bad = L.PC2(msg.data, msg.height, msg.width, msg.point_step, msg.row_step, msg.fields, is_bigendian=True)
            with pytest.raises(L.LiliomError) as e:
                na.cloud_pc2(stamp - 0.05, bad)
            assert e.value.code == L._binding.E_ARG
        a = na.cloud_pc2(stamp, msg)
        b = nb.cloud(stamp, pc2_oracle.pc2_to_pt32(msg))
        assert (a is None) == (b is None)
        if a is not None:
            got.append(a); want.append(b)
    assert len(got) == 4
    for a, b in zip(got, want):
        assert a[0] == b[0]
        np.testing.assert_array_equal(a[4], b[4])
        for x, y in zip(a[1:4], b[1:4]):
            assert len(x) == len(y) and x.tobytes() == y.tobytes()
        assert len(a[1]) > 1000
    c48 = L.Context(variant=0)
    n48 = L.PreprocessingNode(c48)
    with pytest.raises(L.LiliomError):
        n48.cloud_pc2(0.0, seq[0])
    for n in (na, nb, n48):
        n.close()
    for c in (ca, cb, c48):
        c.close()
