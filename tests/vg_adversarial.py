"""Named adversarial clouds for every VoxelGrid path (the sort chain, k_vg_coop, the incremental map, the global map's table
filter): CPU only, deterministic.  Each case is one cloud in both PCL layouts (PT48, PT32) with its leaf and a note on the path
it targets.  NumPy restatements of PCL's box parameters and voxel index (voxel_grid.hpp, x86-64 conversions, the int index
wrapping modulo 2^32) live here too, so that the generators can check that each cloud lands where its note says."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

F = np.float32
INT_MAX = 2**31 - 1
KEY_LIM = 2**20                     # vg_abs_key: |cell coordinate| < 2^20
VGC_NCAP = 32768                    # k_vg_coop's size limit
VGC_VCAP = 256                      # members per voxel k_vg_coop orders in shared memory

PT48 = np.dtype([("x", "f4"), ("y", "f4"), ("z", "f4"), ("w", "f4"), ("nx", "f4"), ("ny", "f4"), ("nz", "f4"), ("nw", "f4"),
                 ("intensity", "f4"), ("curvature", "f4"), ("p0", "f4"), ("p1", "f4")])
PT32 = np.dtype([("x", "f4"), ("y", "f4"), ("z", "f4"), ("w", "f4"), ("intensity", "f4"), ("p0", "f4"), ("p1", "f4"), ("p2", "f4")])


@dataclass
class Case:
    name: str
    pt48: np.ndarray
    pt32: np.ndarray
    leaf: float
    note: str
    abs_key_ok: bool = True        # an absolute-key path (k_vg_coop, the incremental map) may serve it

    def layout(self, stride):
        return self.pt48 if stride == 48 else self.pt32


# ---- NumPy restatement of PCL's parameters and index (x86-64 float -> int conversions, int arithmetic wrapping)

def x86_int(v):
    """int(float32) as x86-64 converts it: truncation, INT_MIN for NaN, inf and everything outside int range"""
    v = float(F(v))
    return int(v) if -2.0**31 <= v < 2.0**31 else -(2**31)


def x86_int64(v):
    v = float(F(v))
    return int(v) if -2.0**63 <= v < 2.0**63 else -(2**63)


def wrap32(v):
    return (int(v) + 2**31) % 2**32 - 2**31


def wrap64(v):
    return (int(v) + 2**63) % 2**64 - 2**63


def finite_mask(c):
    return np.isfinite(c["x"]) & np.isfinite(c["y"]) & np.isfinite(c["z"])


def params(c, leaf):
    """(overflow, min_b, div_b, n_finite) of voxel_grid.hpp's applyFilter for cloud c; None when no point is finite"""
    inv = F(1) / F(leaf)
    fin = finite_mask(c)
    if not fin.any():
        return None
    lo = [F(c[a][fin].min()) for a in "xyz"]
    hi = [F(c[a][fin].max()) for a in "xyz"]
    d = [wrap64(x86_int64(F(F(hi[k] - lo[k]) * inv)) + 1) for k in range(3)]
    overflow = wrap64(wrap64(d[0] * d[1]) * d[2]) > INT_MAX
    min_b = [x86_int(np.floor(F(lo[k] * inv))) for k in range(3)]
    max_b = [x86_int(np.floor(F(hi[k] * inv))) for k in range(3)]
    div_b = [wrap32(max_b[k] - min_b[k] + 1) for k in range(3)]
    return overflow, min_b, div_b, int(fin.sum()), d


def wraps(div_b):
    """the divisions' product, each read as an unsigned count (0: 2^32), reaches 2^32: PCL's int index wraps"""
    prod = 1
    for d in div_b:
        prod *= (d % 2**32) or 2**32
    return prod >= 2**32


def index(c, leaf, min_b, div_b):
    """PCL's voxel index of every point of c (uint32, the int idx wrapped modulo 2^32; meaningless for non-finite points)"""
    inv = F(1) / F(leaf)
    mul = [1, div_b[0], wrap32(div_b[0] * div_b[1])]
    out = np.zeros(len(c), np.uint64)
    for i in range(len(c)):
        idx = 0
        for k, a in enumerate("xyz"):
            ik = x86_int(F(np.floor(F(F(c[a][i]) * inv)) - F(min_b[k])))
            idx += ik * mul[k]
        out[i] = idx % 2**32
    return out


def cells(c, leaf):
    """absolute cell coordinates floor(p / leaf) of every point (float32 arithmetic), int64"""
    inv = F(1) / F(leaf)
    return np.stack([np.floor(c[a].astype(F) * inv).astype(np.float64) for a in "xyz"], 1).astype(np.int64)


# ---- building blocks

def _cloud(xyz, rng, w=1.0):
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    c = np.zeros(len(xyz), PT48)
    c["x"], c["y"], c["z"] = xyz.T
    c["w"] = w
    c["intensity"] = rng.uniform(0, 100, len(c)).astype(F)
    c["curvature"] = rng.uniform(0, 10, len(c)).astype(F)
    for f in ("nx", "ny", "nz"):
        c[f] = rng.uniform(-1, 1, len(c)).astype(F)
    return c


def to32(c):
    out = np.zeros(len(c), PT32)
    for f in PT32.names:
        if f in c.dtype.names:
            out[f] = c[f]
    return out


def _case(name, c, leaf, note, abs_key_ok=True):
    c = np.ascontiguousarray(c, PT48)
    return Case(name, c, to32(c), float(leaf), note, abs_key_ok)


def in_cell(cell, frac, leaf):
    """float32 coordinate at fraction frac of cell `cell` (along one axis)"""
    return F((float(cell) + float(frac)) * float(leaf))


# ---- the wrap box: d = (1, Dy, Dz) passes PCL's test, div_b = (2, Dy + 1, Dz + 1) has a product >= 2^32

WRAP_DY, WRAP_DZ = 2097149, 1024
WRAP_MIN = (-3, -(KEY_LIM - 1), -512)          # min_b; every cell coordinate stays inside (-2^20, 2^20)


def wrap_corners(leaf):
    """two points spanning the wrap box: x over a cell face (d = 1, div_b = 2), y and z over Dy + 1 and Dz + 1 cells with
    extents that truncate to Dy - 1 and Dz - 1 leaves"""
    ax, ay, az = WRAP_MIN
    lo = [in_cell(ax, 0.7, leaf), in_cell(ay, 0.7, leaf), in_cell(az, 0.7, leaf)]
    hi = [in_cell(ax + 1, 0.3, leaf), in_cell(ay + WRAP_DY, 0.3, leaf), in_cell(az + WRAP_DZ, 0.3, leaf)]
    return np.array([lo, hi], np.float32)


def wrap_point(rel, leaf, frac=0.5):
    """a point in the wrap box's relative cell rel (x, y, z); frac keeps it inside the box's partial end cells"""
    out = []
    for k, r in enumerate(rel):
        f = frac
        if r == 0:
            f = max(f, 0.75)
        top = (1, WRAP_DY, WRAP_DZ)[k]
        if r == top:
            f = min(f, 0.25)
        out.append(in_cell(WRAP_MIN[k] + r, f, leaf))
    return out


def wrap_rel_index(rel):
    dx, dy = 2, WRAP_DY + 1
    return (rel[0] + rel[1] * dx + rel[2] * dx * dy) % 2**32


def check_wrap_box(c, leaf):
    p = params(c, leaf)
    assert p is not None
    overflow, min_b, div_b, _, d = p
    assert not overflow and d == [1, WRAP_DY, WRAP_DZ] and div_b == [2, WRAP_DY + 1, WRAP_DZ + 1], (d, div_b)
    assert list(min_b) == list(WRAP_MIN) and wraps(div_b)
    return min_b, div_b


def wrap_collide(leaf=0.4, seed=0):
    """two distinct cells sharing PCL index (div_b[0] * div_b[1] * 1024 = 2^32 - 4096 makes rel (0, j - 2048, 0) and (0, j, 1024)
    collide), each with two members, among other points"""
    rng = np.random.default_rng(seed)
    pts = list(wrap_corners(leaf))
    j = 4548
    a, b = (0, j - 2048, 0), (0, j, WRAP_DZ)
    assert wrap_rel_index(a) == wrap_rel_index(b)
    for rel in (a, b, a, b):
        pts.append(wrap_point(rel, leaf, frac=rng.uniform(0.3, 0.7)))
    for _ in range(40):
        pts.append(wrap_point((int(rng.integers(0, 2)), int(rng.integers(0, WRAP_DY + 1)), int(rng.integers(0, WRAP_DZ + 1))), leaf))
    c = _cloud(pts, rng)
    c = c[rng.permutation(len(c))]
    check_wrap_box(c, leaf)
    return c


def wrap_order(leaf=0.4, seed=1):
    """wrapped indices without a collision: cells of high z (index past 2^32, wrapped to small values) and low z, so PCL's
    order differs from absolute-key order"""
    rng = np.random.default_rng(seed)
    pts = list(wrap_corners(leaf))
    rels = [(0, 100, WRAP_DZ), (1, 5000, WRAP_DZ), (0, 7, 0), (1, 3, 1), (0, 900000, 1000), (1, 2000000, 3), (0, 10, 1023)]
    for rel in rels:
        for _ in range(2):
            pts.append(wrap_point(rel, leaf, frac=rng.uniform(0.35, 0.65)))
    c = _cloud(pts, rng)
    c = c[rng.permutation(len(c))]
    min_b, div_b = check_wrap_box(c, leaf)
    idx = index(c, leaf, min_b, div_b)
    assert len(np.unique(idx)) == len(np.unique(cells(c, leaf), axis=0))      # no two cells share an index
    key = cells(c, leaf)
    absorder = np.lexsort((key[:, 0], key[:, 1], key[:, 2]))
    assert not np.array_equal(np.argsort(idx, kind="stable"), absorder)
    return c


SENTINEL_REL = (1, 2047, WRAP_DZ)              # 1 + 2047 * 2 + 1024 * 2 * 2097150 = 2^32 - 1


def sentinel(leaf=0.4, seed=2, nan_first=True, nan_after=True):
    """a finite point at PCL index 2^32 - 1 (the sort chain's 32-bit sentinel for non-finite points), with non-finite points
    before and after it in the input"""
    rng = np.random.default_rng(seed)
    assert wrap_rel_index(SENTINEL_REL) == 2**32 - 1
    pts = [wrap_point((0, 3, 5), leaf)]
    bad = []
    if nan_first:
        bad.append(len(pts)); pts.append([np.nan, 1.0, 2.0])
        bad.append(len(pts)); pts.append([1.0, np.inf, 2.0])
    pts.append(wrap_point(SENTINEL_REL, leaf))
    hit = len(pts) - 1
    if nan_after:
        bad.append(len(pts)); pts.append([1.0, 2.0, -np.inf])
    pts += list(wrap_corners(leaf))
    for _ in range(20):
        pts.append(wrap_point((int(rng.integers(0, 2)), int(rng.integers(0, WRAP_DY + 1)), int(rng.integers(0, WRAP_DZ + 1))), leaf))
    c = _cloud(pts, rng)
    min_b, div_b = check_wrap_box(c, leaf)
    assert index(c[hit:hit + 1], leaf, min_b, div_b)[0] == 2**32 - 1
    assert not finite_mask(c[bad]).any()
    return c


def faces(leaf, seed=3):
    """coordinates at k*leaf and one float32 ulp either side, negative ones, -0.0 and denormals; at leaves whose inverse is
    inexact floor(p * inv) is not round(p / leaf)"""
    rng = np.random.default_rng(seed)
    vals = []
    for k in range(-25, 26):
        v = F(k * leaf)
        vals += [np.nextafter(v, F(-np.inf)), v, np.nextafter(v, F(np.inf))]
    vals += [F(-0.0), F(0.0), F(1e-45), F(-1e-45), F(1.2e-38), F(-1.2e-38)]
    vals = np.array(vals, np.float32)
    n = 1500
    xyz = np.stack([rng.choice(vals, n), rng.choice(vals, n), rng.choice(vals, n)], 1)
    xyz[:len(vals), 0] = vals                      # every value at least once on x
    c = _cloud(xyz, rng)
    inv = F(1) / F(leaf)
    fl = np.floor(c["x"] * inv)
    rd = np.round(c["x"].astype(np.float64) / leaf)
    assert (fl != rd).any()
    return c


def _extent_for(d, leaf):
    """float32 extent e with trunc(e / leaf) + 1 = d in PCL's float32 arithmetic"""
    inv = F(1) / F(leaf)
    d_of = lambda e: int(np.trunc(F(e * inv))) + 1
    e = F((d - 0.5) * leaf)
    while d_of(e) > d:
        e = np.nextafter(e, F(-np.inf))
    while d_of(e) < d:
        e = np.nextafter(e, F(np.inf))
    assert d_of(e) == d
    return e


def overflow_edge(leaf, above, seed=4):
    """dx*dy*dz around INT_MAX: 2^31 - 2 (INT_MAX is prime: the closest product below it) is filtered, 2^31 = INT_MAX + 1 is
    PCL's overflow and the output is the input"""
    rng = np.random.default_rng(seed)
    d = (65536, 32768, 1) if above else (49981, 42966, 1)
    lo = np.array([0.05 * leaf, -3.3, 0.0], np.float32)
    hi = np.array([lo[k] + _extent_for(d[k], leaf) for k in range(3)], np.float32)
    hi = np.array([F(lo[k] + _extent_for(d[k], leaf)) for k in range(3)], np.float32)
    inner = lo + rng.uniform(0, 1, (200, 3)).astype(np.float32) * (hi - lo)
    c = _cloud(np.concatenate([[lo, hi], inner]), rng)
    p = params(c, leaf)
    prod = p[4][0] * p[4][1] * p[4][2]
    assert prod == (2**31 if above else 2**31 - 2) and p[0] == above, (p[4], prod)
    return c


def key_limit(leaf, inside, axis, seed=5):
    """cells at -(2^20 - 1) and 2^20 - 1 on one axis (the absolute key's last cells), or at -2^20 and 2^20 (the first it cannot
    hold: k_vg_coop declines, the incremental map falls back to the sort chain); one axis at a time, since two such spans are
    PCL's overflow"""
    rng = np.random.default_rng(seed + axis)
    lim = KEY_LIM - 1 if inside else KEY_LIM
    pts = []
    for s in (-1, 1):
        for _ in range(3):
            p = [in_cell(int(rng.integers(-3, 3)), rng.uniform(0.3, 0.7), leaf) for _ in range(3)]
            p[axis] = in_cell(s * lim, rng.uniform(0.3, 0.7), leaf)
            pts.append(p)
    pts += [[in_cell(int(rng.integers(-3, 3)), rng.uniform(0.3, 0.7), leaf) for _ in range(3)] for _ in range(60)]
    c = _cloud(pts, rng)
    k = cells(c, leaf)
    assert k[:, axis].min() == -lim and k[:, axis].max() == lim
    p = params(c, leaf)
    assert not p[0] and not wraps(p[2])             # PCL filters it, the index does not wrap
    return c


def out_of_range(leaf, seed=6):
    """box bounds whose cells leave int range (x86 sends them to INT_MIN), and a ~1e38 extent whose int64 product of d wraps
    past PCL's test"""
    rng = np.random.default_rng(seed)
    k = np.arange(90)
    far = np.stack([1.5e9 + 128.0 * (k // 30), 0.5 + (k % 30) * 0.125, np.zeros(90)], 1)
    huge = np.stack([np.where(k == 3, 1e38, k * 0.3), k * 0.1, np.zeros(90)], 1)
    return _cloud(far, rng), _cloud(huge, rng)


def heavy(leaf, seed=7):
    """voxels of 255, 256 and 257 members (VGC_VCAP) spread over the input; member payloads 1e8, 1, -1e8 in turn, so a sum in
    any other order than the input's shows in the bits"""
    rng = np.random.default_rng(seed)
    counts = (VGC_VCAP - 1, VGC_VCAP, VGC_VCAP + 1, 3, 1)
    cell = np.array([[3 * v - 4, v % 2, -v] for v in range(len(counts))])
    member = np.repeat(np.arange(len(counts)), counts)
    xyz = (cell[member] + rng.uniform(0.2, 0.8, (len(member), 3))) * leaf
    c = _cloud(xyz, rng)
    pat = np.array([1e8, 1.0, -1e8, 3.0, -1.0], np.float32)
    j = np.arange(len(c))
    c["intensity"] = pat[j % 5] * F(1.5) ** (j % 7)
    c["curvature"] = pat[(j + 2) % 5]
    c["nx"] = pat[(j + 1) % 5]
    return c[rng.permutation(len(c))]


def payload(leaf, seed=8):
    """finite xyz with NaN intensity or normal fields (the sums carry them), and voxels whose normals sum to exactly zero"""
    rng = np.random.default_rng(seed)
    xyz = (np.repeat(np.arange(12), 4)[:, None] * np.array([1, 0, 2]) + rng.uniform(0.2, 0.8, (48, 3))) * leaf
    c = _cloud(xyz, rng)
    c["intensity"][[1, 9]] = np.nan
    c["nx"][[13]] = np.nan
    c["curvature"][[17]] = np.inf
    for v in range(6, 12):                         # voxels 6..11: members in pairs n, -n
        a, b, e, f = 4 * v, 4 * v + 1, 4 * v + 2, 4 * v + 3
        for g in ("nx", "ny", "nz"):
            c[g][b] = -c[g][a]; c[g][f] = -c[g][e]
    return c


def trivial(leaf, seed=9):
    rng = np.random.default_rng(seed)
    same = _cloud(np.tile([[1.25, -2.5, 0.75]], (50, 1)), rng)
    single = _cloud([[0.3, 0.2, -0.1]], rng)
    bad = _cloud([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [np.nan, np.nan, np.nan]], rng)
    empty = _cloud(np.zeros((0, 3)), rng)
    return same, single, bad, empty


def sized(n, leaf, seed=10):
    """n points over ~2k voxels with a few non-finite ones: at VGC_NCAP the cooperative filter's size, one more the sort chain"""
    rng = np.random.default_rng(seed + n)
    xyz = rng.uniform(-6, 6, (n, 3)) * np.array([1.0, 1.0, 0.3])
    c = _cloud(xyz, rng)
    c["x"][rng.choice(n, 7, replace=False)] = np.nan
    return c


def cases():
    """every named case (CPU-sized: the largest holds 32769 points)"""
    out = []
    for leaf in (0.1, 0.3, 0.6):
        out.append(_case(f"faces_{leaf}", faces(leaf), leaf, "cell faces, -0.0, denormals: floor(p * inv) at every boundary"))
    out.append(_case("overflow_below", overflow_edge(0.4, False), 0.4, "dx*dy*dz = 2^31 - 2: filtered"))
    out.append(_case("overflow_above", overflow_edge(0.4, True), 0.4, "dx*dy*dz = 2^31: PCL copies the input"))
    out.append(_case("wrap_collide", wrap_collide(), 0.4, "index wraps: two cells share one index and merge", False))
    out.append(_case("wrap_order", wrap_order(), 0.4, "index wraps: PCL's order is not absolute-key order", False))
    out.append(_case("sentinel", sentinel(), 0.4, "a finite point at index 2^32 - 1, non-finite points before and after", False))
    for axis in range(3):
        out.append(_case(f"key_limit_in_{'xyz'[axis]}", key_limit(0.4, True, axis), 0.4,
                         "cells at +-(2^20 - 1): the absolute key's last cells"))
        out.append(_case(f"key_limit_out_{'xyz'[axis]}", key_limit(0.4, False, axis), 0.4,
                         "cells at +-2^20: absolute keys cannot hold them", False))
    far, huge = out_of_range(0.6)
    out.append(_case("far_cluster", far, 0.6, "box bound cells out of int range: x86 INT_MIN indices", False))
    out.append(_case("huge_extent", huge, 0.6, "~1e38 extent: the int64 d product wraps past PCL's test", False))
    out.append(_case("heavy", heavy(0.4), 0.4, "255 / 256 / 257 members: k_vg_coop's bucket size, order-sensitive sums"))
    out.append(_case("payload", payload(0.4), 0.4, "NaN / inf payload fields, normals summing to zero"))
    same, single, bad, empty = trivial(0.4)
    out.append(_case("identical", same, 0.4, "all points identical: one voxel"))
    out.append(_case("single", single, 0.4, "one point"))
    out.append(_case("all_nonfinite", bad, 0.4, "no finite point: empty output"))
    out.append(_case("empty", empty, 0.4, "no point"))
    out.append(_case("size_ncap", sized(VGC_NCAP, 0.4), 0.4, "n = VGC_NCAP: the cooperative filter's largest cloud"))
    out.append(_case("size_ncap1", sized(VGC_NCAP + 1, 0.4), 0.4, "n = VGC_NCAP + 1: the sort chain"))
    return out
