"""CPU tier for the ROT extractor's ring source LILIOM_RING_FIELD (the driver's PointCloud2 `ring` field as scanID):
  - the oracle with given rings (tests/rot_rings_oracle.cpp) is the reference's cloudHandler with ONE substitution: fed the
    elevation tables' own verdicts it reproduces orc_extract_rot in every output, labels and curvatures included;
  - on a 128-ring sweep every cutted point sits in its input ring, rings keep arrival order, rings >= line_num are absent;
  - the `ring` field rules of liliom_b200/csrc/pc2_fields.h compiled for the host (tests/pc2_ring_host.cpp): matching, refusals
    and the per-point read against a NumPy structured-dtype decode."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "build", "libpc2_ring_host.so")
F32, F64, U8, U16, I16, U32 = 7, 8, 2, 4, 3, 6
E_ARG = -1
Q_LB = np.array([0.999, 0.01, -0.02, 0.03]) / np.linalg.norm([0.999, 0.01, -0.02, 0.03])
SUBSAMPLE = {16: 3, 32: 2, 64: 1}        # the 16 / 32-line sweeps the existing ROT tests use: the HDL sweep thinned


def _same(a, b):
    assert len(a) == len(b), (len(a), len(b))
    assert a.tobytes() == b.tobytes()


@pytest.fixture(scope="module")
def hdl():
    from liliom_b200 import synth
    pts, q = synth.make_hdl64_sweep(synth.default_true_pose())
    return pts, q


@pytest.fixture(scope="module")
def sweep128():
    from liliom_b200 import synth
    pts, q, ring, step = synth.make_spinning_sweep(synth.default_true_pose(), synth.uniform_elevations(128), 1024)
    return pts, q, ring, step


def test_table_mode_of_the_restated_body_equals_the_oracle(oracle, hdl):
    import rot_rings_oracle as R
    pts, q = hdl
    for lines in (16, 64):
        p = pts[::SUBSAMPLE[lines]].copy()
        want = oracle.extract_rot(p, q, Q_LB, lines, 1)
        got = R.extract_rot_tables(p, q, Q_LB, lines, 1)
        assert got[0] == want[0] == 0
        for g, w in zip(got[1:], want[1:]):
            _same(g, w)


@pytest.mark.parametrize("ds_rate", [1, 2, 4])
@pytest.mark.parametrize("lines", [16, 32, 64])
def test_table_identity(oracle, hdl, lines, ds_rate):
    """scanID from the field, with the field holding the tables' verdicts (dropped points out of range) == the tables."""
    import rot_rings_oracle as R
    pts, q = hdl
    p = pts[::SUBSAMPLE[lines]].copy()
    p["x"][::501] = np.nan                                   # removeNaN
    p["z"][7::613] *= 1e-3; p["x"][7::613] *= 1e-3; p["y"][7::613] *= 1e-3   # removeClosedPointCloud(3.0)
    ids = R.rot_scan_ids(p, lines)
    assert (ids == -1).any() and (ids >= 0).sum() > 0.5 * len(p)
    rings = np.where(ids < 0, 65535, ids)
    want = oracle.extract_rot(p, q, Q_LB, lines, ds_rate)
    got = R.extract_rot_rings(p, rings, q, Q_LB, lines, ds_rate)
    assert got[0] == want[0] == 0
    for g, w in zip(got[1:], want[1:]):
        _same(g, w)
    assert len(want[2]) > 20 and len(want[1]) > 200


def _bucket(pts, ring, line_num):
    """NumPy restatement of the ring concatenation (:371, :378-382): the surviving points grouped by ring in arrival order."""
    x, y, z = (pts[f].astype(np.float32) for f in ("x", "y", "z"))
    finite = np.isfinite(x) & np.isfinite(y) & np.isfinite(z)
    with np.errstate(invalid="ignore"):
        near = (x * x + y * y + z * z) < np.float32(9.0)
    keep = finite & ~near & (ring >= 0) & (ring < line_num)
    idx = np.flatnonzero(keep)
    return idx[np.argsort(ring[idx], kind="stable")]


@pytest.mark.parametrize("line_num", [128, 40])
def test_bucket_semantics_on_128_rings(sweep128, line_num):
    import rot_rings_oracle as R
    pts, _q, ring, _step = sweep128
    assert ring.max() == 127 and len(pts) > 80_000
    ident = (1.0, 0.0, 0.0, 0.0)                    # no de-skew: the cutted cloud carries the input coordinates
    rc, surf, edge, cut, lab, cur = R.extract_rot_rings(pts, ring, ident, ident, line_num, 1)
    assert rc == 0
    order = _bucket(pts, ring, line_num)
    assert len(cut) == len(order)
    assert np.array_equal(cut["intensity"].astype(np.int32), ring[order])       # intensity = ring + 0.1 * relTime
    assert ((cut["intensity"] - ring[order]) <= np.float32(0.1) + 1e-6).all()
    for f in ("x", "y", "z"):
        assert np.array_equal(cut[f].view(np.uint32), pts[f][order].view(np.uint32)), f
    assert cut["intensity"].astype(np.int32).max() == line_num - 1
    assert len(edge) > 50 and len(surf) > 1000
    if line_num < 128:
        assert (ring >= line_num).sum() > 10_000


def test_ring_limits_of_the_oracle(sweep128):
    import rot_rings_oracle as R
    pts, q, ring, _ = sweep128
    assert R.extract_rot_rings(pts[:100], ring[:100], q, Q_LB, 0, 1)[0] == -2
    assert R.extract_rot_rings(pts[:100], ring[:100], q, Q_LB, 129, 1)[0] == -2
    assert R.extract_rot_rings(pts[:100], ring[:100], q, Q_LB, 1, 1)[0] == 0


# ---------------------------------------------------------------- the `ring` field of pc2_fields.h compiled for the host
@pytest.fixture(scope="module")
def prh():
    src = os.path.join(ROOT, "tests", "pc2_ring_host.cpp")
    deps = [src, os.path.join(ROOT, "liliom_b200", "csrc", "pc2_fields.h"), os.path.join(ROOT, "include", "liliom.h")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(p) for p in deps):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        tmp = f"{SO}.{os.getpid()}"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wextra", "-shared", "-o", tmp, src], check=True)
        os.replace(tmp, SO)
    from liliom_b200 import _lib
    L = C.CDLL(SO)
    L.prh_match.argtypes = [C.POINTER(_lib.Pc2Msg), C.c_int, C.POINTER(C.c_int)]
    L.prh_decode_rings.argtypes = [C.POINTER(_lib.Pc2Msg), C.c_void_p]
    return L


XYZI = [("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("intensity", 12, F32, 1)]


def _match(prh, fields, point_step, want_ring=True, width=10):
    from liliom_b200 import PC2
    msg = PC2(np.zeros(max(width * point_step, 1), np.uint8), 1, width, point_step, width * point_step, fields)
    m, _keep = msg.c_msg()
    out = (C.c_int * 7)(*([-7] * 7))
    rc = prh.prh_match(C.byref(m), int(want_ring), out)
    return rc, tuple(out)


def test_uint8_and_uint16_rings_match(prh):
    assert _match(prh, XYZI + [("ring", 16, U16, 1)], 18) == (0, (0, 4, 8, 12, 10, 16, 2))
    assert _match(prh, XYZI + [("ring", 17, U8, 1)], 18) == (0, (0, 4, 8, 12, 10, 17, 1))
    assert _match(prh, XYZI + [("ring", 16, U16, 0)], 18) == (0, (0, 4, 8, 12, 10, 16, 2))    # count 0 counts as 1


def test_first_matching_ring_wins_and_other_datatypes_are_skipped(prh):
    fields = XYZI + [("ring", 16, F32, 1), ("ring", 20, I16, 1), ("ring", 22, U32, 1), ("ring", 26, U16, 2), ("ring", 28, U8, 1),
                     ("ring", 30, U16, 1)]
    assert _match(prh, fields, 32) == (0, (0, 4, 8, 12, 10, 28, 1))
    assert _match(prh, XYZI + [("ring", 16, U16, 1), ("ring", 18, U8, 1)], 20) == (0, (0, 4, 8, 12, 10, 16, 2))
    assert _match(prh, XYZI + [("rings", 16, U16, 1), ("Ring", 18, U16, 1), ("ring", 20, U8, 1)], 21) == (0, (0, 4, 8, 12, 10, 20, 1))


def test_missing_or_overrunning_ring_is_refused(prh):
    assert _match(prh, XYZI, 16) == (E_ARG, (-7,) * 7)
    assert _match(prh, XYZI + [("ring", 16, F32, 1)], 20) == (E_ARG, (-7,) * 7)          # no UINT8 / UINT16 ring
    assert _match(prh, XYZI + [("ring", 16, U16, 1)], 17) == (E_ARG, (-7,) * 7)          # 2 bytes past point_step
    assert _match(prh, XYZI + [("ring", 16, U8, 1)], 16) == (E_ARG, (-7,) * 7)
    # an overrunning ring of another datatype is never read: the first fitting match is taken
    assert _match(prh, XYZI + [("ring", 16, F64, 1), ("ring", 16, U8, 1)], 17) == (0, (0, 4, 8, 12, 10, 16, 1))


def test_without_the_ring_source_the_ring_is_not_looked_at(prh):
    """ELEVATION mode: the match is the one it always was (the ring field is ignored, even when it could not be read)."""
    assert _match(prh, XYZI, 16, want_ring=False) == (0, (0, 4, 8, 12, 10, -1, 0))
    assert _match(prh, XYZI + [("ring", 16, U16, 1)], 17, want_ring=False) == (0, (0, 4, 8, 12, 10, -1, 0))


@pytest.mark.parametrize("layout", ["velodyne22", "pcl32", "ouster48"])
def test_host_ring_decode_equals_numpy(prh, sweep128, layout):
    from liliom_b200 import synth
    pts, _q, ring, step = sweep128
    msg = synth.encode_pc2(pts, ring, step, layout, steps=1024, lines=128)
    m, _keep = msg.c_msg()
    n = msg.width * msg.height
    got = np.full(n, 0xFFFF, np.uint16)
    assert prh.prh_decode_rings(C.byref(m), got.ctypes.data_as(C.c_void_p)) == n
    f = [x for x in msg.fields if x[0] == "ring"][0]
    dt = np.dtype({"names": ["ring"], "formats": [synth._PC2_NP[f[2]]], "offsets": [f[1]], "itemsize": msg.point_step})
    rows = np.ascontiguousarray(msg.data.reshape(msg.height, msg.row_step)[:, :msg.width * msg.point_step]).reshape(-1)
    want = rows.view(dt)["ring"].astype(np.uint16)
    assert np.array_equal(got, want)
    if msg.height == 1:
        assert np.array_equal(got, ring)
    else:
        assert np.array_equal(got[ring * msg.width + step], ring)
