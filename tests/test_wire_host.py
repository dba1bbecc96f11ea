"""CPU tier for the driver-message decode (SURVEY §8 f3) that liliom_convert_livox, liliom_convert_pc2 and liliom_convert_batch
run on the device: liliom_b200/csrc/wire_decode.h compiled for the host (tests/wire_host.cpp), byte for byte against the CPU
oracles: FormatConvert (oracle_lib.convert_livox) for Livox CustomPoint records at stride 19 and 20, and pcl::fromROSMsg
(tests/pc2_oracle.py) for PointCloud2 messages, with the ring and time side channels against the fields as NumPy reads them."""
import ctypes as C

import numpy as np
import pytest

import host_build
import hz_adversarial as H

F32, F64, U8, U16, U32 = 7, 8, 2, 4, 6
NP = {F32: "<f4", F64: "<f8", U8: "u1", U16: "<u2", U32: "<u4"}
STEPS = 512


@pytest.fixture(scope="module")
def wh():
    from liliom_b200 import _lib as abi
    L = host_build.load("wire_host", ["tests/wire_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall", "-Wextra", "-ffp-contract=off"],
                        deps=["liliom_b200/csrc/wire_decode.h", "liliom_b200/csrc/pc2_fields.h", "liliom_b200/csrc/pcl_xform.h",
                              "liliom_b200/csrc/vg_box.h", "include/liliom.h"])
    L.wh_livox.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.wh_livox.restype = None
    L.wh_pc2.argtypes = [C.POINTER(abi.Pc2Msg), C.c_int, C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.wh_pc2.restype = C.c_int
    return L


def _livox(wh, a, stride):
    from liliom_b200 import PT48
    a = np.ascontiguousarray(a)
    n = a.size * a.dtype.itemsize // stride
    out = np.zeros(max(n, 1), PT48)
    out.view(np.uint8)[:] = 0x5C                            # every byte must be written
    wh.wh_livox(a.ctypes.data_as(C.c_void_p), n, stride, out.ctypes.data_as(C.c_void_p))
    return out[:n]


def _stride19(rec):
    return np.ascontiguousarray(rec).view(np.uint8).reshape(len(rec), 20)[:, :19].copy().reshape(-1)


LIVOX_CASES = H.livox_messages()


@pytest.mark.parametrize("case", [c[0] for c in LIVOX_CASES])
def test_livox_records_equal_format_convert(wh, case):
    import oracle_lib as O
    _, rec, stride = next(c for c in LIVOX_CASES if c[0] == case)
    ref = O.convert_livox(np.ascontiguousarray(rec).view(np.uint8).reshape(-1), stride)
    got = _livox(wh, rec, stride)
    assert len(got) == len(ref) and len(got) > 0
    assert got.tobytes() == ref.tobytes()
    if stride == 20:                                        # the same records without the trailing pad byte
        raw = _stride19(rec)
        assert _livox(wh, raw, 19).tobytes() == O.convert_livox(raw, 19).tobytes() == ref.tobytes()


def _decode(wh, msg, want_ring=False, time_name=None):
    """(rc or n, PT32 cloud, rings, times) of wh_pc2; outputs start at a non-zero pattern so that an unwritten byte shows."""
    from liliom_b200 import PT32
    n = msg.width * msg.height
    out = np.zeros(max(n, 1), PT32)
    out.view(np.uint8)[:] = 0x5C
    rings = np.full(max(n, 1), 0xBEEF, np.uint16)
    times = np.full(max(n, 1), -7.5)
    cm, _keep = msg.c_msg()
    got = wh.wh_pc2(C.byref(cm), int(want_ring), time_name.encode() if time_name else None, out.ctypes.data_as(C.c_void_p),
                    rings.ctypes.data_as(C.c_void_p), times.ctypes.data_as(C.c_void_p))
    return got, out[:max(got, 0)], rings[:max(got, 0)], times[:max(got, 0)]


def _field(msg, off, dt):
    """Field `off` of every point, row-major, as NumPy reads it from the payload (rows of row_step bytes)."""
    size = np.dtype(dt).itemsize
    rows = msg.data.reshape(msg.height, msg.row_step)[:, :msg.width * msg.point_step]
    pts = rows.reshape(msg.height * msg.width, msg.point_step)
    return np.ascontiguousarray(pts[:, off:off + size]).view(dt).reshape(-1)


@pytest.fixture(scope="module")
def sweep():
    from liliom_b200 import synth
    T = synth.default_true_pose()
    pts, _q, ring, step = synth.make_hdl64_sweep(T, steps=STEPS, grid=True)
    return pts, ring, step


LAYOUTS = ["velodyne22", "pcl32", "ouster48", "organised_nan", "hesai26"]


@pytest.mark.parametrize("layout", LAYOUTS)
def test_pc2_layouts_equal_from_ros_msg(wh, sweep, layout):
    import pc2_oracle
    from liliom_b200 import synth
    pts, ring, step = sweep
    msg = synth.encode_pc2(pts, ring, step, layout, steps=STEPS)
    ref = pc2_oracle.pc2_to_pt32(msg)
    n, got, _, _ = _decode(wh, msg)
    assert n == msg.width * msg.height > 0
    assert got.tobytes() == ref.tobytes()
    fields = {f[0]: f for f in msg.fields}
    if "ring" in fields:
        _, off, dt, _ = fields["ring"]
        n, got2, rings, _ = _decode(wh, msg, want_ring=True)
        assert got2.tobytes() == ref.tobytes()
        want = _field(msg, off, NP[dt]).astype(np.uint16)
        assert np.array_equal(rings, want) and want.max() > 0
    name = synth.PC2_TIME_FIELDS.get(layout)
    if name:
        _, off, dt, _ = fields[name]
        n, got3, _, times = _decode(wh, msg, time_name=name)
        assert got3.tobytes() == ref.tobytes()
        want = _field(msg, off, NP[dt]).astype(np.float64)
        assert np.array_equal(times.view(np.uint64), want.view(np.uint64)) and np.ptp(want) > 0


def _random_msg(fields, point_step, width=37, height=3, pad=5, seed=0):
    """A message whose every payload byte is random, so that each mapped field reads distinct bits."""
    from liliom_b200 import PC2
    rng = np.random.default_rng(seed)
    row_step = width * point_step + pad
    data = rng.integers(0, 256, height * row_step, dtype=np.uint8)
    return PC2(data, height, width, point_step, row_step, fields)


XYZI = [("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("intensity", 12, F32, 1)]
# the field-matching cases of tests/test_pc2_host.py, each decoded from a random payload
MATCH_CASES = {
    "plain": (XYZI, 16),
    "out_of_offset_order": ([("intensity", 16, F32, 1), ("ring", 20, U16, 1), ("z", 8, F32, 1), ("x", 0, F32, 1), ("y", 4, F32, 1)], 32),
    "float64_x_first": ([("x", 0, F64, 1), ("x", 8, F32, 1), ("y", 12, F32, 1), ("z", 16, F32, 1), ("intensity", 20, F32, 1)], 24),
    "first_match_wins": (XYZI + [("x", 16, F32, 1)], 20),
    "count_zero_and_two": ([("x", 0, F32, 0), ("y", 4, F32, 2), ("z", 12, F32, 1), ("intensity", 16, F32, 1), ("y", 20, F32, 1)], 24),
    "uint8_intensity": (XYZI[:3] + [("intensity", 12, U8, 1)], 13),
    "missing_intensity": (XYZI[:3], 12),
    "no_fields": ([], 12),
    "names_compare_whole": ([("xx", 0, F32, 1), ("X", 4, F32, 1), ("y", 8, F32, 1), ("z", 12, F32, 1), ("intensity_", 16, F32, 1)], 20),
    "odd_offsets": ([("x", 1, F32, 1), ("y", 6, F32, 1), ("z", 11, F32, 1), ("intensity", 15, F32, 1)], 19),
}


@pytest.mark.parametrize("case", sorted(MATCH_CASES))
def test_pc2_field_matching_cases_equal_from_ros_msg(wh, case):
    import pc2_oracle
    fields, step = MATCH_CASES[case]
    msg = _random_msg(fields, step, seed=len(case))
    n, got, _, _ = _decode(wh, msg)
    assert n == msg.width * msg.height
    assert got.tobytes() == pc2_oracle.pc2_to_pt32(msg).tobytes()


@pytest.mark.parametrize("ring_type", [U8, U16])
@pytest.mark.parametrize("time_type", [F32, F64, U32])
def test_pc2_side_channels_at_unaligned_offsets(wh, ring_type, time_type):
    """ring and time at odd offsets of a packed point, every type: the values NumPy reads from the payload"""
    import pc2_oracle
    tbytes = 8 if time_type == F64 else 4
    fields = XYZI + [("ring", 17, ring_type, 1), ("t", 19, time_type, 1)]
    msg = _random_msg(fields, 19 + tbytes + 1, seed=ring_type * 10 + time_type)
    n, got, rings, times = _decode(wh, msg, want_ring=True, time_name="t")
    assert n == msg.width * msg.height
    assert got.tobytes() == pc2_oracle.pc2_to_pt32(msg).tobytes()
    assert np.array_equal(rings, _field(msg, 17, NP[ring_type]).astype(np.uint16))
    with np.errstate(invalid="ignore"):                     # random float32 payloads hold signalling NaNs
        want = _field(msg, 19, NP[time_type]).astype(np.float64)
    same = (times.view(np.uint64) == want.view(np.uint64)) | (np.isnan(times) & np.isnan(want))
    assert same.all()


def test_refused_messages_decode_nothing(wh, sweep):
    from liliom_b200 import synth
    pts, ring, step = sweep
    msg = synth.encode_pc2(pts, ring, step, "pcl32", steps=STEPS)
    assert _decode(wh, msg, time_name="time")[0] == -1       # no time field in this layout
    bad = _random_msg(XYZI, 16)
    bad.point_step = 0
    assert _decode(wh, bad)[0] == -1
