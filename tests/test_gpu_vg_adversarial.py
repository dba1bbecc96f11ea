"""Every device VoxelGrid path against the oracle's pcl::VoxelGrid, byte for byte, on the adversarial cases of
tests/vg_adversarial.py: liliom_voxelgrid (k_vg_coop where it applies, and the sort chain on the case padded past its size
limit), the odometry's scan filter (24-bit key speculation and its redo), the local map (incremental update and push + rebuild,
solo and batched), and the backend's keyframe filters (kf_add's layers, kf_add_full and the global map's table filter).

The wrap cases (PCL's int index wrapping modulo 2^32: two cells sharing an index, an order that is not the cells' order, a
finite point at the non-finite sentinel's index) must not be served by the absolute-key paths; the map cases are the same boxes
at a 1 cm leaf (~21 km by 10 m), so that the 1 m search grid stays small."""
import ctypes as C

import numpy as np
import pytest

import vg_adversarial as V

pytestmark = pytest.mark.gpu

IDENT = np.array([1.0, 0, 0, 0, 0, 0, 0])
CASES = V.cases()
IDS = [c.name for c in CASES]
MAP_LEAF = 0.01


@pytest.fixture(scope="module")
def ctxs():
    import liliom_b200 as L
    cs = {48: L.Context(variant=0), 32: L.Context(variant=1)}
    yield cs
    for c in cs.values():
        c.close()


def _ctx(stride, **kw):
    import liliom_b200 as L
    p = L.default_params(0 if stride == 48 else 1)
    for k, v in kw.items():
        setattr(p, k, v)
    return L.Context(p)


def _nan_canonical(a):
    """the cloud's words with every NaN written as 0x7fffffff.  A NaN payload field (the "payload" case) sums to a NaN on both
    sides, but the device's float arithmetic returns the canonical NaN where x86 propagates the operand's bits: only NaN-ness
    is compared there, every other bit exactly."""
    u = np.ascontiguousarray(a).view(np.uint32).copy()
    u[((u & 0x7F800000) == 0x7F800000) & ((u & 0x007FFFFF) != 0)] = 0x7FFFFFFF
    return u.tobytes()


def _same(got, want, what):
    assert len(got) == len(want), what
    assert _nan_canonical(got) == _nan_canonical(want), what


# ---- liliom_voxelgrid

@pytest.mark.parametrize("stride", [48, 32])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_voxelgrid_at_size_and_padded(ctxs, oracle, case, stride):
    c = ctxs[stride]
    pts = case.layout(stride)
    c.counters(reset=True)
    got = c.voxelgrid(pts, case.leaf)
    launches = c.counters().launches
    _same(got, oracle.voxelgrid(pts, case.leaf), case.name)
    if 0 < len(pts) <= V.VGC_NCAP and not case.abs_key_ok:
        assert launches > 1, f"{case.name}: served by k_vg_coop"
    if len(pts) == 0:
        return
    reps = -(-(V.VGC_NCAP + 1) // len(pts))
    padded = np.concatenate([pts] * max(reps, 1) if len(pts) > V.VGC_NCAP else [pts] * (reps + 1))
    assert len(padded) > V.VGC_NCAP
    _same(c.voxelgrid(padded, case.leaf), oracle.voxelgrid(padded, case.leaf), case.name + " padded")


# ---- the odometry's scan filter

ODO_CASES = ("wrap_collide", "wrap_order", "sentinel", "key_limit_out_y", "key_limit_in_z", "heavy", "faces_0.3", "payload",
             "overflow_above", "size_ncap", "size_ncap1")


@pytest.mark.parametrize("stride", [48, 32])
@pytest.mark.parametrize("name", ODO_CASES)
def test_odometry_scan_filter(oracle, name, stride):
    """the DS cloud of liliom_odometry (k_vg_coop, or the sort chain with 24-bit keys, redone on a miss) at leaf_scan = the
    case's leaf, on a small installed map"""
    case = next(k for k in CASES if k.name == name)
    c = _ctx(stride, leaf_scan=case.leaf, max_scan_points=max(65536, len(case.pt48)))
    try:
        rng = np.random.default_rng(3)
        m = np.c_[rng.uniform(-5, 5, (400, 3)), np.ones(400)].astype(np.float32)
        c.map_set_points(m)
        pts = case.layout(stride)
        _, _, ds = c.odometry(pts, IDENT, 1, want_stats=False)
        _same(ds, oracle.voxelgrid(pts, case.leaf), name)
    finally:
        c.close()


# ---- the local map

def map_cases():
    """(name, frames) at MAP_LEAF: wrap and sentinel clouds split over three frames, and a stream whose FIFO union enters the
    wrap regime and leaves it again while no frame alone is in it"""
    out = {}
    for name, cloud in (("wrap_collide", V.wrap_collide(MAP_LEAF)), ("wrap_order", V.wrap_order(MAP_LEAF)),
                        ("sentinel", V.sentinel(MAP_LEAF))):
        out[name] = np.array_split(cloud, 3)
    rng = np.random.default_rng(11)
    lo, hi = V.wrap_corners(MAP_LEAF)
    P = lambda rel: V.wrap_point(rel, MAP_LEAF, frac=rng.uniform(0.35, 0.65))
    f1 = [lo] + [P((int(rng.integers(0, 2)), int(rng.integers(0, 100)), int(rng.integers(0, 6)))) for _ in range(30)] + [P((0, 2500, 0))] * 2
    f2 = [P((int(rng.integers(0, 2)), V.WRAP_DY - int(rng.integers(0, 100)), int(rng.integers(0, 6)))) for _ in range(30)]
    f2 += [[np.nan, 0.0, 0.0]]
    f3 = [hi, P((0, 4548, V.WRAP_DZ)), P((0, 4548, V.WRAP_DZ)), V.wrap_point(V.SENTINEL_REL, MAP_LEAF)]
    f3 += [P((int(rng.integers(0, 2)), 4000 + int(rng.integers(0, 100)), V.WRAP_DZ - int(rng.integers(0, 3)))) for _ in range(20)]
    small = lambda: [P((int(rng.integers(0, 2)), 10 + int(rng.integers(0, 50)), 3 + int(rng.integers(0, 4)))) for _ in range(25)]
    frames = [V._cloud(f, rng) for f in (f1, f2, f3, small(), small(), small())]
    for k in range(3):
        assert not V.wraps(V.params(frames[k], MAP_LEAF)[2])
    assert V.wraps(V.params(np.concatenate(frames[:3]), MAP_LEAF)[2])
    out["fifo_union"] = frames
    return out


MAP_CASES = map_cases()
FIFO = 3


def _frames(frames, stride):
    return [f if stride == 48 else V.to32(f) for f in frames]


def _want(oracle, frames, k):
    live = frames[max(0, k + 1 - FIFO):k + 1]
    return oracle.voxelgrid(np.concatenate([oracle.transform_cloud(f, IDENT) for f in live]), MAP_LEAF)


@pytest.mark.parametrize("stride", [48, 32])
@pytest.mark.parametrize("name", list(MAP_CASES))
def test_local_map_update_and_rebuild(oracle, name, stride):
    frames = _frames(MAP_CASES[name], stride)
    inc = _ctx(stride, leaf_map=MAP_LEAF, max_map_frames=FIFO)
    reb = _ctx(stride, leaf_map=MAP_LEAF, max_map_frames=FIFO)
    try:
        for k, f in enumerate(frames):
            want = _want(oracle, frames, k)
            n = inc.map_update(f, IDENT)
            _same(inc.map_download_cloud(), want, f"{name}: map_update after frame {k}")
            assert n == len(want)
            reb.map_push_frame(f, IDENT)
            assert reb.map_rebuild() == len(want)
            _same(reb.map_download_cloud(), want, f"{name}: map_rebuild after frame {k}")
    finally:
        inc.close(); reb.close()


def _odo_leave_ds(c, pts):
    """liliom_odometry with leaf_scan = 0: the scan itself is left on the device as the step's down-sampled cloud (whatever the
    step returns: the map may not be ready yet)"""
    import liliom_b200 as L
    lib = L._binding.lib()
    pts = np.ascontiguousarray(pts, c.dtype)
    pose = np.array(IDENT)
    ds = np.zeros(max(len(pts), 1), c.dtype)
    nds = C.c_int()
    rc = lib.liliom_odometry(c._h, pts.ctypes.data_as(C.c_void_p), len(pts), pose.ctypes.data_as(C.POINTER(C.c_double)), 1, 15,
                             L.MODE_GN, None, ds.ctypes.data_as(C.c_void_p), len(ds), C.byref(nds))
    B = L._binding
    assert rc in (B.OK, B.E_NOMAP, B.E_FEWMAP)
    assert nds.value == len(pts)


@pytest.mark.parametrize("stride", [48, 32])
def test_map_update_batch_next_to_ordinary_sessions(oracle, stride):
    """liliom_map_update_batch over sessions carrying the wrap and sentinel streams beside an ordinary one: each session equals
    its solo liliom_map_update_resident and the oracle after every step"""
    names = ["fifo_union", "sentinel", "wrap_collide"]
    rng = np.random.default_rng(5)
    ordinary = [V._cloud(rng.uniform(-3, 3, (300, 3)), rng) for _ in range(6)]
    streams = [_frames(MAP_CASES[n], stride) for n in names] + [_frames(ordinary, stride)]
    mk = lambda: _ctx(stride, leaf_map=MAP_LEAF, leaf_scan=0.0, max_map_frames=FIFO)
    solo = [mk() for _ in streams]
    bat = [mk() for _ in streams]
    import liliom_b200 as L
    try:
        for k in range(max(len(s) for s in streams)):
            live = [i for i, s in enumerate(streams) if k < len(s)]
            for i in live:
                _odo_leave_ds(solo[i], streams[i][k])
                _odo_leave_ds(bat[i], streams[i][k])
            n_b, status = L.map_update_batch([bat[i] for i in live], np.tile(IDENT, (len(live), 1)))
            assert (status == L._binding.OK).all()
            for j, i in enumerate(live):
                n_s = solo[i].map_update_resident(IDENT)
                want = _want(oracle, streams[i], k)
                got_s, got_b = solo[i].map_download_cloud(), bat[i].map_download_cloud()
                what = f"session {i} step {k}"
                _same(got_s, want, what + " solo")
                _same(got_b, want, what + " batch")
                assert n_s == n_b[j] == len(want)
    finally:
        for c in solo + bat:
            c.close()


# ---- the backend's keyframe filters

KF_CASES = ("wrap_collide", "wrap_order", "sentinel", "faces_0.6", "heavy", "payload", "overflow_above", "far_cluster", "huge_extent")


@pytest.mark.parametrize("stride", [48, 32])
@pytest.mark.parametrize("name", KF_CASES)
def test_keyframe_layers_and_global_map(oracle, name, stride):
    """kf_add's edge and surf layers (the sort chain at edge_leaf / surf_leaf), and the global map's table filter over the case
    split into two keyframes' full clouds"""
    import liliom_b200 as L
    case = next(k for k in CASES if k.name == name)
    pts = case.layout(stride)
    c = _ctx(stride)
    try:
        bp = L.backend_default_params(0)
        bp.edge_leaf = bp.surf_leaf = case.leaf
        halves = np.array_split(pts, 2)
        ids = []
        for h in halves:
            kid, e, s = c.kf_add(bp, h, pts)
            _same(e, oracle.voxelgrid(h, case.leaf), f"{name}: kf_add edge layer")
            _same(s, oracle.voxelgrid(pts, case.leaf), f"{name}: kf_add surf layer")
            assert c.kf_add_full(bp, kid, h) == len(h)
            ids.append(kid)
        poses = np.tile(IDENT, (2, 1))
        want = oracle.voxelgrid(np.concatenate([oracle.transform_cloud(h, IDENT) for h in halves]), case.leaf)
        _same(c.global_map(L.KF_FULL, ids, poses, case.leaf), want, f"{name}: global map")
    finally:
        c.close()
