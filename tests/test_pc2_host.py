"""CPU tier for the PointCloud2 ingest (SURVEY §8 f3, ROT package): the field matching and message validation of
liliom_b200/csrc/pc2_fields.h compiled for the host (tests/pc2_host.cpp), the CPU restatement of pcl::fromROSMsg
(tests/pc2_oracle.cpp) against a NumPy structured-dtype decode on the synthetic driver layouts, and the publishing-side table
that now comes from the same header."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "build", "libpc2_host.so")
F32, F64, U8, U16 = 7, 8, 2, 4
E_ARG = -1


@pytest.fixture(scope="module")
def ph():
    src = os.path.join(ROOT, "tests", "pc2_host.cpp")
    deps = [src, os.path.join(ROOT, "liliom_b200", "csrc", "pc2_fields.h"), os.path.join(ROOT, "include", "liliom.h")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(p) for p in deps):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wextra", "-shared", "-o", SO, src], check=True)
    from liliom_b200 import _lib
    L = C.CDLL(SO)
    L.ph_match.argtypes = [C.POINTER(_lib.Pc2Msg), C.POINTER(C.c_int)]
    L.ph_match.restype = C.c_int
    return L


def _match(ph, fields, point_step, width=10, height=1, row_step=None, is_bigendian=False, data=True, raw_fields=None):
    """(rc, (src x, y, z, intensity, n)); the output array starts at -7 so that an untouched output is visible."""
    from liliom_b200 import PC2
    row_step = width * point_step if row_step is None else row_step
    msg = PC2(np.zeros(max(height * row_step, 1), np.uint8), height, width, point_step, row_step, fields, is_bigendian)
    m, keep = msg.c_msg()
    if not data:
        m.data = None
    if raw_fields is not None:
        m.fields, m.n_fields = raw_fields
    out = (C.c_int * 5)(*([-7] * 5))
    rc = ph.ph_match(C.byref(m), out)
    return rc, tuple(out)


XYZI = [("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("intensity", 12, F32, 1)]


def test_plain_layout(ph):
    assert _match(ph, XYZI, 16) == (0, (0, 4, 8, 12, 10))


def test_fields_listed_out_of_offset_order(ph):
    fields = [("intensity", 16, F32, 1), ("ring", 20, U16, 1), ("z", 8, F32, 1), ("x", 0, F32, 1), ("y", 4, F32, 1)]
    assert _match(ph, fields, 32) == (0, (0, 4, 8, 16, 10))


def test_float64_x_before_the_float32_one(ph):
    fields = [("x", 0, F64, 1), ("x", 8, F32, 1), ("y", 12, F32, 1), ("z", 16, F32, 1), ("intensity", 20, F32, 1)]
    assert _match(ph, fields, 24) == (0, (8, 12, 16, 20, 10))


def test_first_matching_field_wins(ph):
    fields = XYZI + [("x", 16, F32, 1)]
    assert _match(ph, fields, 20) == (0, (0, 4, 8, 12, 10))


def test_count_zero_matches_and_count_two_does_not(ph):
    fields = [("x", 0, F32, 0), ("y", 4, F32, 2), ("z", 12, F32, 1), ("intensity", 16, F32, 1)]
    assert _match(ph, fields, 20) == (0, (0, -1, 12, 16, 10))
    # a count-2 field is skipped, a later count-1 field of the same name is taken
    assert _match(ph, fields + [("y", 20, F32, 1)], 24) == (0, (0, 20, 12, 16, 10))


def test_uint8_intensity_is_unmapped(ph):
    fields = XYZI[:3] + [("intensity", 12, U8, 1)]
    assert _match(ph, fields, 13) == (0, (0, 4, 8, -1, 10))


def test_missing_intensity_is_unmapped(ph):
    assert _match(ph, XYZI[:3], 12) == (0, (0, 4, 8, -1, 10))
    assert _match(ph, [], 12) == (0, (-1, -1, -1, -1, 10))


def test_names_compare_whole(ph):
    fields = [("xx", 0, F32, 1), ("X", 4, F32, 1), ("y", 8, F32, 1), ("z", 12, F32, 1), ("intensity_", 16, F32, 1)]
    assert _match(ph, fields, 20) == (0, (-1, 8, 12, -1, 10))


def test_name_without_terminator_matches_nothing(ph):
    from liliom_b200 import _lib
    f = (_lib.Pc2Field * 2)()
    C.memmove(C.addressof(f[0]), b"x" + b"\0" * 15, 16); f[0].offset = 0; f[0].datatype = F32; f[0].count = 1
    C.memmove(C.addressof(f[1]), b"x" * 16, 16); f[1].offset = 4; f[1].datatype = F32; f[1].count = 1
    assert _match(ph, XYZI, 16, raw_fields=(f, 2)) == (0, (0, -1, -1, -1, 10))
    f2 = (_lib.Pc2Field * 1)()
    C.memmove(C.addressof(f2[0]), b"x" * 16, 16); f2[0].datatype = F32; f2[0].count = 1
    assert _match(ph, XYZI, 16, raw_fields=(f2, 1)) == (0, (-1, -1, -1, -1, 10))


def test_packed_22_byte_velodyne(ph):
    fields = XYZI + [("ring", 16, U16, 1), ("time", 18, F32, 1)]
    assert _match(ph, fields, 22) == (0, (0, 4, 8, 12, 10))


def test_mapped_field_past_point_step_is_rejected(ph):
    assert _match(ph, XYZI, 15)[0] == E_ARG
    assert _match(ph, XYZI[:3] + [("intensity", 13, F32, 1)], 16) == (E_ARG, (-7,) * 5)
    # the same overrun on a field that does not match is not an error (it is never read)
    assert _match(ph, XYZI[:3] + [("intensity", 14, U8, 1), ("intensity", 15, F64, 1)], 15) == (0, (0, 4, 8, -1, 10))


def test_row_step(ph):
    assert _match(ph, XYZI, 16, width=10, height=3, row_step=159) == (E_ARG, (-7,) * 5)
    assert _match(ph, XYZI, 16, width=10, height=3, row_step=160) == (0, (0, 4, 8, 12, 30))
    assert _match(ph, XYZI, 16, width=10, height=3, row_step=200) == (0, (0, 4, 8, 12, 30))


def test_is_bigendian_is_rejected(ph):
    assert _match(ph, XYZI, 16, is_bigendian=True) == (E_ARG, (-7,) * 5)


def test_other_rejections(ph):
    assert _match(ph, XYZI, 0, row_step=0)[0] == E_ARG                              # point_step 0
    assert _match(ph, XYZI, 16, data=False)[0] == E_ARG                             # null payload
    assert _match(ph, XYZI, 16, raw_fields=(None, 4))[0] == E_ARG                   # null fields, n_fields > 0
    assert _match(ph, XYZI, 16, raw_fields=(None, -1))[0] == E_ARG                  # n_fields < 0
    assert ph.ph_match(None, (C.c_int * 5)()) == E_ARG                              # null msg


def test_point_count_limit(ph):
    from liliom_b200 import _lib
    buf = C.create_string_buffer(1)                                                 # never read: only the header is checked
    m = _lib.Pc2Msg(C.cast(buf, C.c_void_p), 2, 1 << 30, 1, 1 << 30, None, 0, 0)  # 2^31 points
    out = (C.c_int * 5)()
    assert ph.ph_match(C.byref(m), out) == E_ARG
    m.height = 1; m.width = (1 << 31) - 1; m.row_step = (1 << 31) - 1
    assert ph.ph_match(C.byref(m), out) == 0 and out[4] == (1 << 31) - 1


def test_empty_sweep_is_valid(ph):
    assert _match(ph, XYZI, 16, width=0) == (0, (0, 4, 8, 12, 0))
    assert _match(ph, XYZI, 16, width=0, data=False) == (0, (0, 4, 8, 12, 0))      # an empty msg.data may have no storage
    assert _match(ph, XYZI, 16, width=5, height=0, data=False) == (0, (0, 4, 8, 12, 0))


# ---------------------------------------------------------------- the CPU decode against NumPy
def _np_decode(msg):
    """pcl::fromROSMsg restated with NumPy structured dtypes: per PointXYZI field the first FLOAT32 field of that name with
    count 0 or 1, read through a dtype with that one field at its offset and itemsize = point_step, row by row."""
    from liliom_b200 import PT32
    n = msg.width * msg.height
    out = np.zeros(n, PT32)
    out["w"] = 1.0
    rows = np.ascontiguousarray(msg.data.reshape(msg.height, msg.row_step)[:, :msg.width * msg.point_step]).reshape(-1)
    for name in ("x", "y", "z", "intensity"):
        hit = [f for f in msg.fields if f[0] == name and f[2] == F32 and f[3] in (0, 1)]
        if hit:
            dt = np.dtype({"names": [name], "formats": ["<f4"], "offsets": [hit[0][1]], "itemsize": msg.point_step})
            out[name] = rows.view(dt)[name]
    return out


@pytest.fixture(scope="module")
def hdl_grid():
    from liliom_b200 import synth
    pts, _, ring, step = synth.make_hdl64_sweep(synth.default_true_pose(), grid=True)
    return pts, ring, step


@pytest.mark.parametrize("layout", ["velodyne22", "pcl32", "ouster48", "organised_nan"])
def test_oracle_decode_equals_numpy(hdl_grid, layout):
    import pc2_oracle
    from liliom_b200 import synth
    pts, ring, step = hdl_grid
    msg = synth.encode_pc2(pts, ring, step, layout)
    got = pc2_oracle.pc2_to_pt32(msg)
    want = _np_decode(msg)
    assert len(got) == msg.width * msg.height and got.tobytes() == want.tobytes()
    # every return of the sweep is in the message with its coordinates
    if msg.height == 1:
        assert got.tobytes() == pts.tobytes()
    else:
        at = got[ring * msg.width + step]
        for f in ("x", "y", "z", "intensity"):
            assert at[f].tobytes() == pts[f].tobytes()


def test_oracle_decode_unmapped_and_mixed_fields():
    import pc2_oracle
    from liliom_b200 import PC2
    rng = np.random.default_rng(3)
    data = rng.integers(0, 256, size=3 * 70, dtype=np.uint8)                        # 3 rows of 5 points x 13 B + 5 B padding
    fields = [("x", 0, F64, 1), ("x", 1, F32, 1), ("y", 5, F32, 0), ("intensity", 9, U8, 1), ("z", 9, F32, 2)]
    msg = PC2(data, 3, 5, 13, 70, fields)
    got = pc2_oracle.pc2_to_pt32(msg)
    assert got.tobytes() == _np_decode(msg).tobytes()
    assert (got["z"] == 0).all() and (got["intensity"] == 0).all() and (got["w"] == 1).all()


def test_publishing_table_unchanged():
    """liliom_pc2_layout reads the same header's tables: PCL's PointXYZINormal / PointXYZI field lists."""
    import liliom_b200 as L
    assert L.pc2_layout(48) == ([("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("normal_x", 16, 7, 1), ("normal_y", 20, 7, 1),
                                 ("normal_z", 24, 7, 1), ("intensity", 32, 7, 1), ("curvature", 36, 7, 1)], 48)
    assert L.pc2_layout(32) == ([("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("intensity", 16, 7, 1)], 32)
