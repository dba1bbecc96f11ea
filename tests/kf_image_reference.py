"""TEST INFRASTRUCTURE: the keyframe image (liliom_kf_export / liliom_kf_import) restated in NumPy from its format text, not from
liliom_b200/csrc/kf_image.h: an encoder, a decoder, both checksums, random images, and named malformed images with the check
that refuses each.

Format: little-endian.  A 64-byte header (magic b"LILIKF01", u32 version 1, u32 point_stride, i32 k, u32 flags, u64 edge+surf
points, u64 full points, u64 table checksum, u64 points checksum, u64 reserved 0), k 16-byte records (i32 n_edge, n_surf,
n_full (-1: no full cloud), reserved 0), section A (each keyframe's edge points then its surf points, in table order), section F
(the full clouds).  Size = 64 + 16 k + stride * (sum E + sum S + sum F).
Checksum: h = sum_j splitmix64_finaliser(w_j ^ j * 0x9E3779B97F4A7C15) mod 2^64 over u64 words; the points checksum over the
words of A then F (j from the start of A), the table checksum over the header with both checksum fields zero, then the table."""
from __future__ import annotations

import numpy as np

MAGIC = b"LILIKF01"
VERSION = 1
FLAG_FULL = 1
HEADER, RECORD = 64, 16
GOLDEN = np.uint64(0x9E3779B97F4A7C15)
HDR = np.dtype([("magic", "S8"), ("version", "<u4"), ("stride", "<u4"), ("k", "<i4"), ("flags", "<u4"), ("n_scan", "<u8"),
                ("n_full", "<u8"), ("table_sum", "<u8"), ("points_sum", "<u8"), ("reserved", "<u8")])
REC = np.dtype([("n_edge", "<i4"), ("n_surf", "<i4"), ("n_full", "<i4"), ("reserved", "<i4")])
assert HDR.itemsize == HEADER and REC.itemsize == RECORD

# the checks in the order they are made (their names as liliom_last_error gives them follow "keyframe image: ")
CHECKS = ["magic", "version", "stride", "flags", "counts", "totals", "length", "table", "points"]


def checksum(buf, j0: int = 0) -> int:
    """sum_j mix(w_j ^ (j0 + j) * golden) mod 2^64 over the little-endian u64 words of buf (any bytes-like object; summed in
    chunks, so that an image of gigabytes needs no copy of itself)"""
    mv = memoryview(buf).cast("B")
    chunk = 1 << 23                      # words
    total = 0
    for w0 in range(0, len(mv) // 8, chunk):
        w = np.frombuffer(mv[8 * w0:8 * (w0 + chunk)], "<u8").astype(np.uint64)
        j = np.arange(j0 + w0, j0 + w0 + len(w), dtype=np.uint64)
        with np.errstate(over="ignore"):
            z = w ^ (j * GOLDEN)
            z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
            z = z ^ (z >> np.uint64(31))
        total = (total + int(z.sum(dtype=np.uint64))) % 2**64
    return total


def table_sum(header: bytes, table: bytes) -> int:
    h = np.frombuffer(header, HDR).copy()
    h["table_sum"] = 0
    h["points_sum"] = 0
    return (checksum(h.tobytes()) + checksum(table, HEADER // 8)) % 2**64


def encode(stride: int, records, a: bytes, f: bytes, flags: int = FLAG_FULL) -> bytes:
    """records: (n_edge, n_surf, n_full) per keyframe; a, f: the bytes of sections A and F"""
    rec = np.zeros(len(records), REC)
    for i, (ne, ns, nf) in enumerate(records):
        rec[i] = (ne, ns, nf, 0)
    h = np.zeros(1, HDR)
    h["magic"] = MAGIC; h["version"] = VERSION; h["stride"] = stride; h["k"] = len(records); h["flags"] = flags
    h["n_scan"] = sum(ne + ns for ne, ns, _ in records)
    h["n_full"] = sum(max(nf, 0) for _, _, nf in records)
    h["points_sum"] = checksum(a + f)
    h["table_sum"] = table_sum(h.tobytes(), rec.tobytes())
    return h.tobytes() + rec.tobytes() + a + f


def decode(img: bytes) -> dict:
    """The header, the records, and per keyframe its edge, surf and full bytes (None: no full cloud)"""
    h = np.frombuffer(img[:HEADER], HDR)[0]
    k, s = int(h["k"]), int(h["stride"])
    rec = np.frombuffer(img[HEADER:HEADER + RECORD * k], REC)
    a0 = HEADER + RECORD * k
    f0 = a0 + s * int(h["n_scan"])
    kfs, pa, pf = [], a0, f0
    for r in rec:
        ne, ns, nf = int(r["n_edge"]), int(r["n_surf"]), int(r["n_full"])
        e = img[pa:pa + s * ne]; pa += s * ne
        su = img[pa:pa + s * ns]; pa += s * ns
        fu = None
        if nf >= 0:
            fu = img[pf:pf + s * nf]; pf += s * nf
        kfs.append((e, su, fu))
    return dict(header=h, records=rec, kfs=kfs, a=img[a0:f0], f=img[f0:])


def size(stride: int, records) -> int:
    return HEADER + RECORD * len(records) + stride * sum(ne + ns + max(nf, 0) for ne, ns, nf in records)


def random_image(rng, stride: int, k: int, full: bool = True):
    """An image of k keyframes with random counts (empty clouds and keyframes without a full cloud among them) and random point
    bytes (NaN payloads, -0 and any padding included).  Returns (image, records)."""
    records = []
    for _ in range(k):
        ne = int(rng.choice([0, 1, int(rng.integers(2, 40))]))
        ns = int(rng.choice([0, 1, int(rng.integers(2, 60))]))
        nf = int(rng.choice([-1, 0, int(rng.integers(1, 80))])) if full else -1
        records.append((ne, ns, nf))
    n_a = sum(ne + ns for ne, ns, _ in records)
    n_f = sum(max(nf, 0) for _, _, nf in records)
    a = rng.integers(0, 256, n_a * stride, dtype=np.uint8).tobytes()
    f = rng.integers(0, 256, n_f * stride, dtype=np.uint8).tobytes()
    return encode(stride, records, a, f, FLAG_FULL if full else 0), records


def _set(img: bytes, off: int, fmt: str, value) -> bytes:
    b = bytearray(img)
    b[off:off + np.dtype(fmt).itemsize] = np.array([value], fmt).tobytes()
    return bytes(b)


def _flip(img: bytes, off: int, bit: int = 0) -> bytes:
    b = bytearray(img)
    b[off] ^= 1 << bit
    return bytes(b)


def _resum(img: bytes) -> bytes:
    """the table checksum made right again after a header or table edit (so that an earlier check is the one that fails)"""
    k = int(np.frombuffer(img[:HEADER], HDR)[0]["k"])
    return _set(img, 40, "<u8", table_sum(img[:HEADER], img[HEADER:HEADER + RECORD * k]))


def malformed(img: bytes, stride: int):
    """Named malformed variants of a valid image of point_stride `stride` whose table holds at least one keyframe with points
    in A and one with a full cloud (and two different edge and surf counts in one record): (name, bytes, the failing check)."""
    d = decode(img)
    k = int(d["header"]["k"])
    rec = d["records"]
    a0 = HEADER + RECORD * k
    f0 = a0 + stride * int(d["header"]["n_scan"])
    end = len(img)
    out = []
    # truncations: at every header field, at every record, at every keyframe's clouds in A and F, one byte short; one byte more
    cuts = {0, 8, 12, 16, 20, 24, 32, 40, 48, 56, HEADER} | {HEADER + RECORD * i for i in range(k)}
    pa, pf = a0, f0
    for r in rec:
        cuts |= {pa, pa + stride * int(r["n_edge"])}
        pa += stride * (int(r["n_edge"]) + int(r["n_surf"]))
        cuts.add(pf)
        pf += stride * max(int(r["n_full"]), 0)
    for c in sorted(x for x in cuts if x < end):
        out.append((f"truncated_at_{c}", img[:c], "length"))
    out.append(("one_byte_short", img[:-1], "length"))
    out.append(("one_byte_more", img + b"\0", "length"))
    # the header
    out.append(("bad_magic", _flip(img, 3), "magic"))
    out.append(("bad_version", _set(img, 8, "<u4", 2), "version"))
    out.append(("header_reserved", _resum(_set(img, 56, "<u8", 1)), "version"))
    out.append(("wrong_stride", _set(img, 12, "<u4", 80 - stride), "stride"))
    out.append(("unknown_flag", _set(img, 20, "<u4", 3), "flags"))
    out.append(("flipped_header_n_scan", _flip(img, 24), "totals"))
    out.append(("flipped_header_table_sum", _flip(img, 40, 5), "table"))
    out.append(("flipped_header_points_sum", _flip(img, 48, 7), "points"))
    out.append(("totals_disagree", _resum(_set(img, 32, "<u8", int(d["header"]["n_full"]) + 1)), "totals"))
    # the table
    i_full = next(i for i, r in enumerate(rec) if int(r["n_full"]) >= 0)
    out.append(("n_full_minus_2", _resum(_set(img, HEADER + RECORD * i_full + 8, "<i4", -2)), "counts"))
    out.append(("negative_n_edge", _flip(img, HEADER + 3, 7), "counts"))
    out.append(("record_reserved", _resum(_set(img, HEADER + 12, "<i4", 1)), "counts"))
    out.append(("flipped_table_bit", _flip(img, HEADER), "totals"))
    i_swap = next(i for i, r in enumerate(rec) if int(r["n_edge"]) != int(r["n_surf"]))
    t = bytearray(img)
    o = HEADER + RECORD * i_swap
    t[o:o + 4], t[o + 4:o + 8] = img[o + 4:o + 8], img[o:o + 4]
    out.append(("swapped_table_words", bytes(t), "table"))
    # the points: only the points checksum catches these
    for name, lo, hi in (("A", a0, f0), ("F", f0, end)):
        if hi > lo:
            out.append((f"flipped_first_word_of_{name}", _flip(img, lo, 2), "points"))
            out.append((f"flipped_last_word_of_{name}", _flip(img, hi - 8, 6), "points"))
    t = bytearray(img)
    w0, w1 = a0, a0 + 8
    if img[w0:w0 + 8] != img[w1:w1 + 8]:
        t[w0:w0 + 8], t[w1:w1 + 8] = img[w1:w1 + 8], img[w0:w0 + 8]
        out.append(("swapped_point_words", bytes(t), "points"))
    return out
