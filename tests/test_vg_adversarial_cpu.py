"""CPU tier of the adversarial VoxelGrid cases (tests/vg_adversarial.py): the oracle's VoxelGrid against a second NumPy
restatement of pcl::VoxelGrid (the int index wrapping modulo 2^32 included), the host composition of the sort chain from
liliom_b200/csrc/vg_box.h against the oracle byte for byte, and the header's wrap predicate against NumPy on boxes whose
divisions multiply to 2^32 - 1, 2^32 and 2^32 + 1."""
import ctypes as C

import numpy as np
import pytest

import host_build
import vg_adversarial as V

F = np.float32
CASES = V.cases()
IDS = [c.name for c in CASES]


@pytest.fixture(scope="module")
def vb():
    L = host_build.load("vg_box_host", ["tests/vg_box_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall", "-ffp-contract=off"],
                        deps=["liliom_b200/csrc/vg_box.h"])
    fp, ip = np.ctypeslib.ndpointer(np.float32, flags="C"), np.ctypeslib.ndpointer(np.int32, flags="C")
    L.vb_voxelgrid.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, fp]
    L.vb_voxelgrid.restype = C.c_int
    L.vb_wraps.argtypes = [ip, C.c_float]
    L.vb_wraps.restype = C.c_int
    L.vb_key_bits.argtypes = [ip, C.c_float]
    L.vb_key_bits.restype = C.c_int
    L.vb_chain_key_bits.argtypes = [ip, C.c_float]
    L.vb_chain_key_bits.restype = C.c_int
    return L


def fsum(v):
    """left-to-right float32 sum from +0.0 (so that -0.0 members sum to +0.0, as an accumulator started at 0 gives)"""
    return np.cumsum(np.r_[F(0), v].astype(F), dtype=F)[-1]


def np_voxelgrid(c, leaf):
    """pcl::VoxelGrid restated in NumPy float32: PCL's overflow test (output = input), the wrapped uint32 index, members in
    input order (the oracle's stable sort), sequential float32 sums, pcl::CentroidPoint's output point"""
    p = V.params(c, leaf)
    if p is None:
        return c[:0]
    overflow, min_b, div_b, _, _ = p
    if overflow:
        return c.copy()
    fin = np.flatnonzero(V.finite_mask(c))
    idx = V.index(c[fin], leaf, min_b, div_b)
    order = np.argsort(idx, kind="stable")
    idx, members = idx[order], fin[order]
    starts = np.flatnonzero(np.r_[True, idx[1:] != idx[:-1]])
    ends = np.r_[starts[1:], len(idx)]
    out = np.zeros(len(starts), c.dtype)
    has_n = "nx" in c.dtype.names
    fields = ["x", "y", "z", "intensity"] + (["curvature"] if has_n else [])
    for o, (a, b) in enumerate(zip(starts, ends)):
        m = c[members[a:b]]
        cnt = F(b - a)
        for f in fields:
            out[f][o] = fsum(m[f]) / cnt
        out["w"][o] = 1.0
        if has_n:
            s = [fsum(m[g]) for g in ("nx", "ny", "nz")]
            n2 = F(F(F(s[0] * s[0]) + F(s[1] * s[1])) + F(s[2] * s[2]))
            if n2 > 0:
                nn = np.sqrt(n2, dtype=F)
                s = [F(v / nn) for v in s]
            out["nx"][o], out["ny"][o], out["nz"][o] = s
    return out


def host_voxelgrid(vb, pts, leaf):
    pts = np.ascontiguousarray(pts)
    out = np.zeros(max(len(pts), 1), pts.dtype)
    xyz = np.zeros((max(len(pts), 1), 3), np.float32)
    m = vb.vb_voxelgrid(pts.ctypes.data, len(pts), pts.dtype.itemsize, leaf, out.ctypes.data, xyz)
    assert m >= 0
    return out[:m]


def test_cases_cover_the_issue():
    names = set(IDS)
    for want in ("wrap_collide", "wrap_order", "sentinel", "overflow_below", "overflow_above", "heavy", "payload", "empty",
                 "size_ncap", "size_ncap1", "far_cluster", "huge_extent", "key_limit_out_x"):
        assert want in names


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_oracle_matches_numpy_restatement(oracle, case):
    for stride in (48, 32):
        pts = case.layout(stride)
        want = np_voxelgrid(pts, case.leaf)
        got = oracle.voxelgrid(pts, case.leaf)
        assert len(got) == len(want), case.name
        assert got.tobytes() == want.tobytes(), case.name


def test_wrap_cases_differ_from_absolute_cells(oracle):
    """the wrap cases are what their notes say: a collision merges two cells, the sentinel point is output last"""
    by = {c.name: c for c in CASES}
    wc = by["wrap_collide"].pt48
    assert len(oracle.voxelgrid(wc, 0.4)) == len(np.unique(V.cells(wc, 0.4), axis=0)) - 1
    st = by["sentinel"].pt48
    out = oracle.voxelgrid(st, 0.4)
    hit = np.flatnonzero(V.finite_mask(st))
    hit = hit[V.index(st[hit], 0.4, V.WRAP_MIN, [2, V.WRAP_DY + 1, V.WRAP_DZ + 1]) == 2**32 - 1]
    assert len(hit) == 1 and out[-1]["x"] == st[hit[0]]["x"] and out[-1]["y"] == st[hit[0]]["y"]


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_host_sort_chain_matches_oracle(vb, oracle, case):
    for stride in (48, 32):
        pts = case.layout(stride)
        want = oracle.voxelgrid(pts, case.leaf)
        got = host_voxelgrid(vb, pts, case.leaf)
        assert len(got) == len(want), case.name
        assert got.tobytes() == want.tobytes(), case.name


def test_sentinel_on_both_sides(vb, oracle):
    """non-finite points only before, only after, or on neither side of the point at index 2^32 - 1"""
    for first, after in ((True, False), (False, True), (False, False)):
        pts = V.sentinel(nan_first=first, nan_after=after)
        for c in (pts, V.to32(pts)):
            assert host_voxelgrid(vb, c, 0.4).tobytes() == oracle.voxelgrid(c, 0.4).tobytes()


def _box(lo, hi):
    enc = lambda f: np.where(f.view(np.int32) >= 0, f.view(np.int32), f.view(np.int32) ^ np.int32(0x7FFFFFFF))
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    return np.concatenate([enc(lo), enc(hi), [2]]).astype(np.int32)


@pytest.mark.parametrize("divs", [(65535, 65537, 1), (2048, 2048, 1024), (641, 6700417, 1), (2, 2097150, 1025), (2, 2097151, 1024),
                                  (1, 65536, 65535), (1, 1, 1)])
def test_wrap_predicate_around_2_pow_32(vb, divs):
    """boxes at leaf 1 (exact arithmetic) whose divisions multiply to 2^32 - 1, 2^32, 2^32 + 1 and neighbours: the header's
    predicate against NumPy, and the sort chain's key width: the wide keys exactly where PCL filters a wrapping box"""
    leaf = 1.0
    lo = np.array([-(d // 2) + 0.5 for d in divs], np.float32)
    hi = np.array([-(d // 2) + d - 1 + 0.5 for d in divs], np.float32)
    c = np.zeros(2, V.PT48)
    c["x"], c["y"], c["z"] = np.stack([lo, hi]).T
    overflow, _, div_b, _, _ = V.params(c, leaf)
    assert tuple(div_b) == divs
    box = _box(lo, hi)
    want = V.wraps(div_b)
    assert want == (np.prod(divs, dtype=object) >= 2**32)
    assert vb.vb_wraps(box, leaf) == int(want)
    bits = vb.vb_chain_key_bits(box, leaf)
    assert bits == (33 if want and not overflow else vb.vb_key_bits(box, leaf))
    assert vb.vb_key_bits(box, leaf) <= 32


def test_wrap_box_takes_wide_keys(vb):
    """the wrap cases' box passes PCL's test and wraps: the sort chain's keys are the wide ones"""
    for name in ("wrap_collide", "wrap_order", "sentinel"):
        c = next(k for k in CASES if k.name == name).pt48
        fin = c[V.finite_mask(c)]
        xyz = np.stack([fin["x"], fin["y"], fin["z"]], 1)
        box = _box(xyz.min(0), xyz.max(0))
        box[6] = len(fin)
        assert vb.vb_wraps(box, 0.4) == 1 and vb.vb_chain_key_bits(box, 0.4) == 33, name
