"""CPU tier for the keyframe image (liliom_kf_export / liliom_kf_import): liliom_b200/csrc/kf_image.h compiled for the host
(tests/kf_image_host.cpp) against the NumPy restatement of the format (tests/kf_image_reference.py): the encoder, both checksums
and the size on random images of both point strides, and every check in its order on named malformed images."""
import ctypes as C

import numpy as np
import pytest

import host_build
import kf_image_reference as R

STRIDES = (48, 32)


@pytest.fixture(scope="module")
def ki():
    L = host_build.load("kf_image_host", ["tests/kf_image_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall"],
                        deps=["liliom_b200/csrc/kf_image.h", "liliom_b200/csrc/vg_box.h"])
    u8 = C.c_char_p
    L.kih_term.argtypes = [C.c_ulonglong, C.c_ulonglong]; L.kih_term.restype = C.c_ulonglong
    L.kih_sum.argtypes = [u8, C.c_longlong, C.c_ulonglong]; L.kih_sum.restype = C.c_ulonglong
    L.kih_check_name.argtypes = [C.c_int]; L.kih_check_name.restype = C.c_char_p
    L.kih_size.argtypes = [C.c_int, C.c_longlong, C.c_longlong, C.c_longlong]; L.kih_size.restype = C.c_longlong
    L.kih_check.argtypes = [u8, C.c_longlong, C.c_int, C.POINTER(C.c_int)]; L.kih_check.restype = C.c_int
    L.kih_check_all.argtypes = [u8, C.c_longlong, C.c_int]; L.kih_check_all.restype = C.c_int
    L.kih_encode.argtypes = [C.c_int, C.c_int, C.c_uint, C.POINTER(C.c_int), u8, C.c_longlong, u8, C.c_longlong, C.c_char_p]
    return L


def check_all(ki, img, stride):
    """the name of the first failed check (R.CHECKS), or None"""
    e = ki.kih_check_all(img, len(img), stride)
    return None if e == 0 else R.CHECKS[e - 1]


def encode(ki, stride, records, a, f, flags):
    counts = (C.c_int * max(3 * len(records), 1))(*[x for r in records for x in r])
    out = C.create_string_buffer(R.size(stride, records))
    ki.kih_encode(stride, len(records), flags, counts, a, len(a), f, len(f), out)
    return out.raw


def test_check_names_follow_the_order(ki):
    names = [ki.kih_check_name(e).decode() for e in range(1, len(R.CHECKS) + 1)]
    for want, got in zip(R.CHECKS, names):
        assert want in got, (want, got)


def test_term_and_sum_agree_with_numpy(ki):
    rng = np.random.default_rng(1)
    words = rng.integers(0, 2**63, 257, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, 257, dtype=np.uint64)
    words[:4] = [0, 2**64 - 1, 1, 0x9E3779B97F4A7C15]
    buf = words.astype("<u8").tobytes()
    for j0 in (0, 1, 8, 2**40 + 3):
        assert ki.kih_sum(buf, len(words), j0) == R.checksum(buf, j0)
        assert ki.kih_term(int(words[5]), j0) == R.checksum(words[5:6].astype("<u8").tobytes(), j0)
    assert ki.kih_sum(b"", 0, 0) == 0 == R.checksum(b"")


def test_the_sum_is_keyed_by_position(ki):
    w = np.arange(1, 9, dtype="<u8").tobytes()
    swapped = w[8:16] + w[:8] + w[16:]
    assert R.checksum(w) != R.checksum(swapped)
    assert R.checksum(w[:56]) != R.checksum(w)
    # order-independent: the sum of two halves, each keyed by its own position, is the whole
    assert (R.checksum(w[:24]) + R.checksum(w[24:], 3)) % 2**64 == R.checksum(w)


@pytest.mark.parametrize("stride", STRIDES)
@pytest.mark.parametrize("full", [True, False])
def test_encode_and_decode_agree_with_numpy(ki, stride, full):
    rng = np.random.default_rng(stride + full)
    for k in (0, 1, 2, 7, 33):
        img, records = R.random_image(rng, stride, k, full)
        d = R.decode(img)
        got = encode(ki, stride, records, d["a"], d["f"], R.FLAG_FULL if full else 0)
        assert got == img, (k, full)
        assert len(img) == ki.kih_size(stride, k, int(d["header"]["n_scan"]), int(d["header"]["n_full"])) == R.size(stride, records)
        kk = C.c_int(-1)
        assert ki.kih_check(img, len(img), stride, C.byref(kk)) == 0 and kk.value == k
        assert check_all(ki, img, stride) is None
        h = d["header"]
        assert bytes(h["magic"]) == R.MAGIC and h["version"] == 1 and h["stride"] == stride and h["k"] == k
        assert int(h["points_sum"]) == R.checksum(d["a"] + d["f"])
        assert int(h["table_sum"]) == R.table_sum(img[:R.HEADER], img[R.HEADER:R.HEADER + R.RECORD * k])
        for (ne, ns, nf), (e, s, f) in zip(records, d["kfs"]):
            assert len(e) == ne * stride and len(s) == ns * stride
            assert (f is None) == (nf < 0) and (f is None or len(f) == nf * stride)
            if not full:
                assert nf == -1


def _fixture_image(stride):
    rng = np.random.default_rng(7)
    records = [(3, 5, 4), (0, 2, -1), (6, 6, 0), (2, 0, 9)]
    a = rng.integers(0, 256, stride * sum(e + s for e, s, _ in records), dtype=np.uint8).tobytes()
    f = rng.integers(0, 256, stride * sum(max(x, 0) for _, _, x in records), dtype=np.uint8).tobytes()
    return R.encode(stride, records, a, f)


@pytest.mark.parametrize("stride", STRIDES)
def test_every_malformed_image_fails_its_check(ki, stride):
    img = _fixture_image(stride)
    assert check_all(ki, img, stride) is None
    cases = R.malformed(img, stride)
    seen = set()
    for name, bad, want in cases:
        got = check_all(ki, bad, stride)
        assert got == want, (name, got, want)
        if want != "points":                  # the library's host checks refuse it before any upload
            assert ki.kih_check(bad, len(bad), stride, None) == R.CHECKS.index(want) + 1, name
        else:                                 # ... or only the points checksum, which the device sums, catches it
            assert ki.kih_check(bad, len(bad), stride, None) == 0, name
        seen.add(want)
    assert seen == set(R.CHECKS)
    names = [n for n, _, _ in cases]
    assert {"one_byte_short", "one_byte_more", "n_full_minus_2", "swapped_point_words", "totals_disagree",
            "flipped_first_word_of_A", "flipped_last_word_of_A", "flipped_first_word_of_F", "flipped_last_word_of_F"} <= set(names)
    assert sum(n.startswith("truncated_at_") for n in names) >= 10 + 1 + 4


def test_empty_image_and_a_full_flag_without_full_clouds(ki):
    for stride in STRIDES:
        img = R.encode(stride, [], b"", b"")
        assert len(img) == 64 and check_all(ki, img, stride) is None
        img = R.encode(stride, [(0, 0, -1), (0, 0, 0)], b"", b"")
        assert check_all(ki, img, stride) is None
        # without the full flag a record with a full cloud (even an empty one) is refused
        img = R.encode(stride, [(0, 0, 0)], b"", b"", flags=0)
        assert check_all(ki, img, stride) == "counts"
