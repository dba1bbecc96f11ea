"""CPU tier for the VoxelGrid arithmetic: liliom_b200/csrc/vg_box.h compiled for the host (tests/vg_box_host.cpp).  The
ordered-int encoding, the box of a cloud, PCL's VoxelGrid parameters (pcl::getMinMax3D and the leaf division of
voxel_grid.hpp), the sort chain's key width and the absolute 21-bit voxel key against NumPy float32 restatements, at the
leaves the reference uses (0.2, 0.4, 0.6); and the whole sort chain and the ROT extractor's per-ring filter composed from the
header (voxel index, heads, member walk, pcl::CentroidPoint writer) against the oracle's VoxelGrid, byte for byte."""
import ctypes as C

import numpy as np
import pytest

import host_build

INT_MAX = 2**31 - 1
LEAVES = (0.2, 0.4, 0.6)
F = np.float32


@pytest.fixture(scope="module")
def vb():
    L = host_build.load("vg_box_host", ["tests/vg_box_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall", "-ffp-contract=off"],
                        deps=["liliom_b200/csrc/vg_box.h"])
    fp, ip = np.ctypeslib.ndpointer(np.float32, flags="C"), np.ctypeslib.ndpointer(np.int32, flags="C")
    L.vb_f2ord.argtypes = [fp, ip, C.c_int]
    L.vb_ord2f.argtypes = [ip, fp, C.c_int]
    L.vb_box_of.argtypes = [fp, C.c_int, ip]
    L.vb_params.argtypes = [ip, C.c_float, ip, C.POINTER(C.c_float)]
    L.vb_key_bits.argtypes = [ip, C.c_float]
    L.vb_key_bits.restype = C.c_int
    L.vb_abs_key.argtypes = [C.c_float, C.c_float, C.c_float, C.c_float, C.POINTER(C.c_ulonglong)]
    L.vb_abs_key.restype = C.c_int
    L.vb_voxelgrid.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, fp]
    L.vb_voxelgrid.restype = C.c_int
    L.vb_voxelgrid_rings.argtypes = [C.c_void_p, ip, C.c_int, C.c_float, C.c_void_p, fp]
    L.vb_voxelgrid_rings.restype = C.c_int
    return L


def f2ord(vb, f):
    f = np.ascontiguousarray(f, np.float32)
    out = np.empty(f.shape, np.int32)
    vb.vb_f2ord(f, out, f.size)
    return out


def ord2f(vb, i):
    i = np.ascontiguousarray(i, np.int32)
    out = np.empty(i.shape, np.float32)
    vb.vb_ord2f(i, out, i.size)
    return out


def np_encode(f):
    """float32 -> ordered int32: i >= 0 ? i : i ^ 0x7fffffff"""
    i = np.asarray(f, np.float32).view(np.int32)
    return np.where(i >= 0, i, i ^ np.int32(0x7FFFFFFF)).astype(np.int32)


def np_box(pts):
    """pcl::getMinMax3D over the finite points, in the 7-int layout: min xyz, max xyz (encoded), finite count"""
    pts = np.asarray(pts, np.float32).reshape(-1, 3)
    fin = pts[np.isfinite(pts).all(axis=1)]
    if len(fin) == 0:
        return np.array([INT_MAX] * 3 + [-INT_MAX - 1] * 3 + [0], np.int32)
    return np.concatenate([np_encode(fin.min(axis=0)), np_encode(fin.max(axis=0)), [len(fin)]]).astype(np.int32)


def np_params(lo, hi, n_finite, leaf):
    """voxel_grid.hpp applyFilter in float32: inverse_leaf_size_, min_b_, div_b_, divb_mul_ and the dx*dy*dz > INT_MAX test"""
    inv = F(1) / F(leaf)
    if n_finite == 0:
        min_b, div_b, overflow = [0, 0, 0], [1, 1, 1], 0
    else:
        d = [int(np.trunc(F(F(hi[k]) - F(lo[k])) * inv)) + 1 for k in range(3)]
        min_b = [int(np.floor(F(lo[k]) * inv)) for k in range(3)]
        div_b = [int(np.floor(F(hi[k]) * inv)) - min_b[k] + 1 for k in range(3)]
        overflow = int(d[0] * d[1] * d[2] > INT_MAX)
    mul = [1, div_b[0], int(np.int64(div_b[0] * div_b[1]).astype(np.int32))]
    return inv, min_b, div_b, mul, overflow


def np_key_bits(lo, hi, n_finite, leaf):
    """the sort chain's key width: fewest bits (>= 8) with all-ones free; 32 for an empty box, PCL's overflow, >= 2^31 voxels"""
    if n_finite <= 0:
        return 32
    _, _, div_b, _, overflow = np_params(lo, hi, n_finite, leaf)
    cells = div_b[0] * div_b[1] * div_b[2]
    if overflow or not 0 < cells < 2**31:
        return 32
    return max(8, cells.bit_length())


def call_params(vb, box, leaf):
    out = np.zeros(12, np.int32)
    inv = C.c_float()
    vb.vb_params(np.ascontiguousarray(box, np.int32), leaf, out, C.byref(inv))
    return F(inv.value), list(out[0:3]), list(out[3:6]), list(out[6:9]), int(out[9]), int(out[10]), int(out[11])


def box_of_extent(lo, hi):
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    return np_box(np.stack([lo, hi])), lo, hi


def test_encoding_round_trip_and_order(vb):
    fmax, tiny = np.finfo(np.float32).max, np.finfo(np.float32).tiny
    special = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, tiny, -tiny, 1.0, -1.0, fmax, -fmax, np.inf, -np.inf], np.float32)
    rng = np.random.default_rng(11)
    bits = rng.integers(0, 2**32, 200_000, dtype=np.uint64).astype(np.uint32)
    vals = np.concatenate([special, bits.view(np.float32)])
    enc = f2ord(vb, vals)
    assert np.array_equal(enc, np_encode(vals))
    assert np.array_equal(ord2f(vb, enc).view(np.uint32), vals.view(np.uint32))             # round trip, NaN payloads included
    fin = vals[~np.isnan(vals)]
    order = np.lexsort((~np.signbit(fin), fin))                                              # float order, -0 before +0
    e = f2ord(vb, fin[order])
    assert (np.diff(e.astype(np.int64)) >= 0).all()
    assert ((np.diff(e.astype(np.int64)) > 0) == (np.diff(fin[order].view(np.uint32).astype(np.int64)) != 0)).all()
    assert f2ord(vb, np.float32(-0.0)) < f2ord(vb, np.float32(0.0))
    nans = np.array([0x7FC00000, 0x7F800001, 0x7FFFFFFF, 0xFFC00000, 0xFF800001, 0xFFFFFFFF], np.uint32).view(np.float32)
    en = f2ord(vb, nans)
    lo_f, hi_f = f2ord(vb, np.float32(-np.inf)), f2ord(vb, np.float32(np.inf))
    assert ((en > hi_f) | (en < lo_f)).all()
    assert (en[np.signbit(nans)] < lo_f).all() and (en[~np.signbit(nans)] > hi_f).all()


@pytest.mark.parametrize("seed", range(4))
def test_box_of_a_cloud(vb, seed):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-300.0, 300.0, (1001, 3)).astype(np.float32)
    pts[rng.integers(0, len(pts), 40), rng.integers(0, 3, 40)] = rng.choice(np.array([np.nan, np.inf, -np.inf], np.float32), 40)
    pts[5] = [-0.0, 0.0, -0.0]
    box = np.zeros(7, np.int32)
    vb.vb_box_of(np.ascontiguousarray(pts), len(pts), box)
    assert np.array_equal(box, np_box(pts))
    vb.vb_box_of(np.full((3, 3), np.nan, np.float32), 3, box)
    assert np.array_equal(box, np_box(np.zeros((0, 3))))                                    # no finite point: the empty box


def check_params(vb, box, lo, hi, leaf):
    got = call_params(vb, box, leaf)
    inv, min_b, div_b, mul, overflow = np_params(lo, hi, int(box[6]), leaf)
    assert got[0] == inv
    assert (got[1], got[2], got[3], got[4], got[5], got[6]) == (min_b, div_b, mul, overflow, int(box[6]), 0), (lo, hi, leaf)
    assert vb.vb_key_bits(np.ascontiguousarray(box, np.int32), leaf) == np_key_bits(lo, hi, int(box[6]), leaf), (lo, hi, leaf)
    return overflow


@pytest.mark.parametrize("leaf", LEAVES)
def test_params_random_and_empty_boxes(vb, leaf):
    rng = np.random.default_rng(int(leaf * 10))
    for scale in (1.0, 50.0, 1e3, 1e5):
        for _ in range(200):
            pts = (rng.uniform(-1.0, 1.0, (8, 3)) * scale + rng.uniform(-scale, scale, 3)).astype(np.float32)
            box = np_box(pts)
            check_params(vb, box, ord2f(vb, box[0:3]), ord2f(vb, box[3:6]), leaf)
    for pts in ([[-0.3, -7.9, -0.01]], [[-0.0, 0.0, -0.0]], [[-1.2, -1.2, -1.2], [-0.6, -0.6, -0.6]]):    # negative / single-point boxes
        box = np_box(pts)
        check_params(vb, box, ord2f(vb, box[0:3]), ord2f(vb, box[3:6]), leaf)
    empty = np_box(np.zeros((0, 3)))
    assert check_params(vb, empty, [0, 0, 0], [0, 0, 0], leaf) == 0
    assert vb.vb_key_bits(empty, leaf) == 32


@pytest.mark.parametrize("leaf", LEAVES + (1.0,))
def test_params_on_both_sides_of_the_overflow_boundary(vb, leaf):
    """dx*dy*dz just below and just above INT_MAX: PCL copies the input above it, and the sort chain then takes 32-bit keys"""
    inv = F(1) / F(leaf)
    d_of = lambda ext: int(np.trunc(F(ext) * inv)) + 1
    seen = set()
    # (voxel coordinates stay below 2^31: beyond it float -> int conversion differs between the device and the host)
    for dy, dz in ((1024, 1024), (3000, 77), (2, 3), (46341, 46340)):
        target = INT_MAX // (dy * dz)                                     # dx with dx*dy*dz <= INT_MAX < (dx+1)*dy*dz
        for want in (target, target + 1):
            ext = {}
            for k, d in (("x", want), ("y", dy), ("z", dz)):
                e = F((d - 0.5) * float(leaf))
                while d_of(e) > d:
                    e = np.nextafter(e, F(-np.inf))
                while d_of(e) < d:
                    e = np.nextafter(e, F(np.inf))
                ext[k] = e
            for org in ((0.0, 0.0, 0.0), (-3.1, 0.0, 17.3), (-40000.7, -20000.1, -5.55)):
                lo = np.array(org, np.float32)
                hi = (lo + np.array([ext["x"], ext["y"], ext["z"]], np.float32)).astype(np.float32)
                box, lo, hi = box_of_extent(lo, hi)
                seen.add(check_params(vb, box, lo, hi, leaf))
    assert seen == {0, 1}


def test_key_bits_widths(vb):
    """8-bit floor, each power of two, and the 32-bit cases of the rule"""
    for leaf in LEAVES:
        for cells_x in (1, 200, 255, 256, 257, 4095, 4096, 70000, 2**20, 2**22):
            lo = np.array([0.05 * leaf, 0.05 * leaf, 0.05 * leaf], np.float32)
            hi = np.array([F((cells_x - 0.5) * leaf), lo[1], lo[2]], np.float32)
            box, lo, hi = box_of_extent(lo, hi)
            got = vb.vb_key_bits(box, leaf)
            assert got == np_key_bits(lo, hi, 2, leaf)
            assert 8 <= got <= 32
    box, lo, hi = box_of_extent([0, 0, 0], [2000.0, 2000.0, 2000.0])    # PCL's overflow at 0.2: 10^4^3 voxels
    assert np_params(lo, hi, 2, 0.2)[4] == 1 and vb.vb_key_bits(box, 0.2) == 32


@pytest.mark.parametrize("leaf", LEAVES)
def test_absolute_key_and_its_limit(vb, leaf):
    inv = F(1) / F(leaf)
    lim = 2**20
    rng = np.random.default_rng(int(leaf * 100))
    pts = rng.uniform(-(lim + 50) * leaf, (lim + 50) * leaf, (4000, 3)).astype(np.float32)
    edge = np.array([-lim, -lim + 1, lim - 1, lim, 0], np.float64)
    near = np.concatenate([edge * leaf, edge * leaf + 1e-3, edge * leaf - 1e-3]).astype(np.float32)
    pts = np.concatenate([pts, np.stack([near, np.roll(near, 3), np.roll(near, 7)], axis=1),
                          np.array([[-0.0, 0.0, -1e-30], [0.1, -0.1, 0.0]], np.float32)])
    key = C.c_ulonglong()
    n_ok = 0
    for p in pts:
        f = [int(np.floor(F(p[k]) * inv)) for k in range(3)]
        ok = all(abs(v) < lim for v in f)
        key.value = 0xDEADBEEF
        assert vb.vb_abs_key(float(p[0]), float(p[1]), float(p[2]), float(inv), C.byref(key)) == int(ok), p
        if ok:
            n_ok += 1
            assert key.value == ((f[2] + lim) << 42) | ((f[1] + lim) << 21) | (f[0] + lim), p
        else:
            assert key.value == 0xDEADBEEF                                # untouched
    assert 0 < n_ok < len(pts)


# ---- the centroid: sort chain and per-ring filter composed from the header, against the oracle

def host_voxelgrid(vb, pts, leaf, ring=None):
    """(output cloud, the centroids' xyz returned by the writer); ring: per-point ring ids -> the per-ring batch of 32-byte points"""
    pts = np.ascontiguousarray(pts)
    out = np.zeros(max(len(pts), 1), pts.dtype)
    xyz = np.zeros((max(len(pts), 1), 3), np.float32)
    if ring is None:
        m = vb.vb_voxelgrid(pts.ctypes.data, len(pts), pts.dtype.itemsize, leaf, out.ctypes.data, xyz)
    else:
        m = vb.vb_voxelgrid_rings(pts.ctypes.data, np.ascontiguousarray(ring, np.int32), len(pts), leaf, out.ctypes.data, xyz)
    assert m >= 0
    return out[:m], xyz[:m]


def check_voxelgrid(vb, want, pts, leaf, ring=None):
    got, xyz = host_voxelgrid(vb, pts, leaf, ring)
    assert len(got) == len(want)
    assert got.tobytes() == want.tobytes()
    assert np.array_equal(xyz.view(np.uint32), np.stack([got["x"], got["y"], got["z"]], 1).view(np.uint32))
    return got


def as_layout(pts, dt):
    """the cloud in the other PCL layout: the fields both have copied, the others zero"""
    out = np.zeros(len(pts), dt)
    for f in dt.names:
        if f in pts.dtype.names:
            out[f] = pts[f]
    return out


@pytest.mark.parametrize("leaf", LEAVES)
@pytest.mark.parametrize("sweep", ["hz", "hdl"])
def test_sort_chain_matches_oracle_on_sweeps(vb, oracle, world_small, sweep, leaf):
    for dt in (oracle.PT48, oracle.PT32):
        pts = as_layout(world_small[sweep], dt)
        got = check_voxelgrid(vb, oracle.voxelgrid(pts, leaf), pts, leaf)
        assert 0 < len(got) < len(pts)


def test_sort_chain_matches_oracle_on_adversarial_inputs(vb, oracle):
    """points exactly on voxel faces, duplicates, non-finite points, a single point, an empty cloud"""
    rng = np.random.default_rng(8)
    for dt, leaf in ((oracle.PT48, 0.4), (oracle.PT32, 0.6), (oracle.PT48, 0.25), (oracle.PT32, 0.2)):
        n = 3000
        c = np.zeros(n, dt)
        xyz = rng.uniform(-7, 7, (n, 3)).astype(np.float32)
        xyz[:300] = np.round(xyz[:300] / np.float32(leaf)) * np.float32(leaf)
        xyz[300:400] = xyz[:100]
        c["x"], c["y"], c["z"] = xyz.T
        c["intensity"] = rng.uniform(0, 50, n).astype(np.float32)
        if dt is oracle.PT48:
            c["curvature"] = rng.uniform(0, 25, n).astype(np.float32)
            for f in ("nx", "ny", "nz"):
                c[f] = rng.uniform(-1, 1, n).astype(np.float32)
        bad = rng.choice(n, 40, replace=False)
        c["x"][bad[:15]] = np.nan; c["y"][bad[15:30]] = np.inf; c["z"][bad[30:]] = -np.inf
        check_voxelgrid(vb, oracle.voxelgrid(c, leaf), c, leaf)
        check_voxelgrid(vb, oracle.voxelgrid(c[bad], leaf), c[bad], leaf)                        # no finite point: nothing out
    for dt in (oracle.PT48, oracle.PT32):
        one = np.zeros(1, dt); one["x"] = 1.5; one["intensity"] = 3
        assert len(check_voxelgrid(vb, oracle.voxelgrid(one, 0.4), one, 0.4)) == 1
        assert len(check_voxelgrid(vb, oracle.voxelgrid(one[:0], 0.4), one[:0], 0.4)) == 0


def cloud_of_voxels(dt, counts, leaf, rng):
    """len(counts) voxels with counts[k] members each, in a shuffled input order; members well inside their voxel, voxel k is
    output k"""
    cells = np.array([[3 * k - 11, (k * 5) % 4, 2 * k - 3] for k in range(len(counts))], np.float64)
    member = np.repeat(np.arange(len(counts)), counts)
    pos = (cells[member] + rng.uniform(0.1, 0.9, (len(member), 3))) * leaf
    c = np.zeros(len(member), dt)
    c["x"], c["y"], c["z"] = pos.astype(np.float32).T
    c["intensity"] = rng.uniform(0, 100, len(c)).astype(np.float32)
    if "nx" in dt.names:
        c["curvature"] = rng.uniform(0, 10, len(c)).astype(np.float32)
        for f in ("nx", "ny", "nz"):
            c[f] = rng.uniform(-1, 1, len(c)).astype(np.float32)
    perm = rng.permutation(len(c))
    return c[perm], member[perm]


@pytest.mark.parametrize("leaf", LEAVES)
def test_walk_across_batches_of_eight(vb, oracle, leaf):
    """voxels of 1, 7, 8, 9, 16, 17 and 300 members: the walk fetches 8 entries at a time and stops inside or at a batch's end"""
    counts = (1, 7, 8, 9, 16, 17, 300)
    rng = np.random.default_rng(int(leaf * 10) + 3)
    for dt in (oracle.PT48, oracle.PT32):
        c, _ = cloud_of_voxels(dt, counts, leaf, rng)
        assert len(check_voxelgrid(vb, oracle.voxelgrid(c, leaf), c, leaf)) == len(counts)


def test_normals_summing_to_zero_stay_zero(vb, oracle):
    """pcl::CentroidPoint normalises the normal sum only when its squared norm is > 0: a zero sum is written as it is"""
    rng = np.random.default_rng(5)
    counts = (2, 4, 10, 3, 16)
    c, member = cloud_of_voxels(oracle.PT48, counts, 0.4, rng)
    for k in (0, 1, 2, 4):                          # members in pairs n, -n (in input order): the fp32 sum is exactly zero
        idx = np.flatnonzero(member == k)
        for a, b in zip(idx[0::2], idx[1::2]):
            for f in ("nx", "ny", "nz"):
                c[f][b] = -c[f][a]
    c["nx"][member == 4] = c["ny"][member == 4] = c["nz"][member == 4] = 0.0
    got = check_voxelgrid(vb, oracle.voxelgrid(c, 0.4), c, 0.4)
    n = np.stack([got["nx"], got["ny"], got["nz"]], 1)
    assert (n[[0, 1, 2, 4]] == 0).all()
    np.testing.assert_allclose(np.linalg.norm(n[3]), 1.0, rtol=1e-6)


@pytest.mark.parametrize("leaf", LEAVES)
def test_per_ring_batch_matches_oracle_ring_by_ring(vb, oracle, world_small, leaf):
    """the ROT extractor's batch: ring << 32 | voxel index keys over all rings at once = the oracle's VoxelGrid of every ring's
    points, rings in ascending order; one ring in PCL's overflow case keeps its points, one point per voxel"""
    rng = np.random.default_rng(int(leaf * 10) + 7)
    pts = world_small["hdl"]
    pts = pts[np.isfinite(pts["x"]) & np.isfinite(pts["y"]) & np.isfinite(pts["z"])][::3]
    ring = rng.integers(0, 64, len(pts)).astype(np.int32)
    far = np.zeros(5, pts.dtype)
    far["x"], far["y"], far["z"] = ([-5000.0, 5000.0, 0.0, 1.0, 2.5], [-5000.0, 5000.0, 3.0, 1.0, 0.5], [-5000.0, 5000.0, -1.0, 2.0, 0.0])
    far["w"] = 1.0
    far["intensity"] = [1.0, 2.0, 3.0, 4.0, 5.0]
    pts = np.concatenate([pts, far])
    ring = np.concatenate([ring, np.full(5, 64, np.int32)])
    want = np.concatenate([oracle.voxelgrid(pts[ring == r], leaf) for r in range(65)])
    got = check_voxelgrid(vb, want, pts, leaf, ring)
    assert np.array_equal(got[-5:], far)


def _x86_int(v):
    """int(float) as x86-64 converts it: truncation, INT_MIN out of range or not finite"""
    v = float(np.float32(v))
    return int(v) if -2.0 ** 31 <= v < 2.0 ** 31 else -(2 ** 31)


@pytest.mark.parametrize("leaf", [0.6, 0.4])
def test_params_and_sort_chain_on_out_of_range_boxes(vb, oracle, leaf):
    """boxes whose cells leave int range: a tight far cluster (every x index INT_MIN, as PCL's x86 build computes it), a cluster
    far on the negative side, and a box spanning ~1e38 (d out of int64 range).  min_b follows x86's conversion, the box is
    flagged (bail) and the sort chain's key width is 32; the host sort chain equals the oracle's VoxelGrid on each."""
    clouds = {}
    k = np.arange(90)
    clouds["far_x"] = np.stack([1.5e9 + 128.0 * (k // 30), 0.5 + (k % 30) * 0.125, np.zeros(90)], 1)
    clouds["far_neg_y"] = np.stack([0.5 + (k % 30) * 0.125, -1.6e9 - 256.0 * (k // 30), np.ones(90)], 1)
    clouds["huge"] = np.stack([np.where(k == 3, 1e38, k * 0.3), k * 0.1, np.zeros(90)], 1)
    for name, xyz in clouds.items():
        xyz = xyz.astype(np.float32)
        box = np_box(xyz)
        inv, min_b, div_b, mul, overflow, n_finite, bail = call_params(vb, box, leaf)
        lo, hi = xyz.min(0), xyz.max(0)
        assert min_b == [_x86_int(np.floor(F(lo[j]) * inv)) for j in range(3)], name
        assert bail == 1 and vb.vb_key_bits(np.ascontiguousarray(box, np.int32), leaf) == 32, name
        for dt in (oracle.PT48, oracle.PT32):
            c = np.zeros(len(xyz), dt)
            c["x"], c["y"], c["z"] = xyz.T
            c["intensity"] = (k % 5).astype(np.float32)
            got = check_voxelgrid(vb, oracle.voxelgrid(c, leaf), c, leaf)
            if name == "far_x":
                assert len(got) < 30 * 3                   # voxels that differ only in x merge
    # in range: no flag
    box = np_box(np.array([[1.0, 2.0, 3.0], [5.0, -4.0, 2.0]], np.float32))
    assert call_params(vb, box, 0.4)[6] == 0
