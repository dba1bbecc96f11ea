"""CPU tier for the global map's table filter (liliom_global_map): liliom_b200/csrc/kf_table.h compiled for the host with
vg_box.h and pcl_xform.h (tests/gmap_host.cpp) and composed as the device composes it (box of the transformed rows, voxel keys,
stable sort, heads, vg_walk through the transforming loader, the centroid writer; PCL's declined case gathers), against the
oracle's voxelgrid(concat(transform_cloud(...))) byte for byte: both point layouts, with and without the pre-transform of
save_pcd, lists that repeat keyframes, empty clouds, non-finite points, and boxes on both sides of PCL's overflow test.  The same
build composes the multi-store global map (liliom_global_map_multi): rows that each name an arena of their own (one arena per
store) must give, byte for byte, what rows over one arena holding the same clouds give (the merged store), and the oracle's
composition: both point layouts, per-entry pre-transforms, interleaved and repeated lists, non-finite points, and PCL's declined
case."""
import ctypes as C

import numpy as np
import pytest

import host_build

T_BL = np.array([0.7071, 0.0, 0.0, 0.7071, -0.18, 0.0, -0.095])      # R/config/config_fr_iosb.yaml ql2b_*, tl2b_* (not quite unit)


@pytest.fixture(scope="module")
def gm():
    L = host_build.load("gmap_host", ["tests/gmap_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall", "-ffp-contract=off"],
                        deps=[f"liliom_b200/csrc/{h}" for h in ("kf_table.h", "pcl_xform.h", "vg_box.h")])
    vp, llp, ip, dp = C.c_void_p, np.ctypeslib.ndpointer(np.int64, flags="C"), np.ctypeslib.ndpointer(np.int32, flags="C"), C.c_void_p
    L.gm_global_map.argtypes = [vp, C.c_int, llp, ip, C.c_int, dp, dp, C.c_float, vp, C.POINTER(C.c_int)]
    L.gm_global_map.restype = C.c_longlong
    L.gm_rows_of.argtypes = [ip, C.c_int, llp, C.c_int, ip]
    L.gm_rows_of.restype = None
    for f in (L.gmm_single, L.gmm_multi):
        f.argtypes = [C.POINTER(vp), C.c_int, llp, ip, C.c_int, vp, vp, C.c_float, vp, C.POINTER(C.c_int)]
        f.restype = C.c_longlong
    return L


@pytest.fixture(scope="module")
def seqs():
    from liliom_b200 import synth
    return {s: synth.make_keyframe_sequence(10, stride=s, seed=5, full=True) for s in (48, 32)}


def host_global_map(gm, clouds, ids, poses, leaf, pre7=None):
    """the store holds `clouds` back to back in reverse order (offsets that are not the list order); returns (map, declined)"""
    dt = clouds[0].dtype
    order = list(range(len(clouds)))[::-1]
    arena = np.concatenate([clouds[i] for i in order]) if clouds else np.zeros(0, dt)
    start = {}
    off = 0
    for i in order:
        start[i] = off
        off += len(clouds[i])
    src = np.array([start[i] for i in ids], np.int64)
    n = np.array([len(clouds[i]) for i in ids], np.int32)
    total = int(n.sum())
    out = np.zeros(max(total, 1), dt)
    p = np.ascontiguousarray(np.asarray(poses, np.float64).reshape(-1, 7)) if len(ids) else np.zeros((1, 7))
    pre = None if pre7 is None else np.ascontiguousarray(pre7, np.float64)
    declined = C.c_int()
    arena = np.ascontiguousarray(arena) if len(arena) else np.zeros(1, dt)
    m = gm.gm_global_map(arena.ctypes.data, dt.itemsize, src, n, len(ids), p.ctypes.data, None if pre is None else pre.ctypes.data,
                         leaf, out.ctypes.data, C.byref(declined))
    assert m >= 0
    return out[:m], declined.value


def oracle_global_map(O, clouds, ids, poses, leaf, pre7=None):
    dt = clouds[0].dtype
    parts = []
    for i, p in zip(ids, poses):
        c = clouds[i] if pre7 is None else O.transform_cloud(clouds[i], pre7)
        parts.append(O.transform_cloud(c, p))
    parts = [x for x in parts if len(x)]
    cat = np.concatenate(parts) if parts else np.zeros(0, dt)
    return O.voxelgrid(cat, leaf), cat


def nudge(pose, k):
    from liliom_b200 import synth
    dq = synth.q_from_axis_angle([1, -1, 2], np.deg2rad(0.2 * k))
    return np.concatenate([synth.qmul(pose[:4], dq), pose[4:] + 0.01 * k * np.array([1.0, -0.5, 0.25])])


def check(gm, O, clouds, ids, poses, leaf, pre7=None, declined=False):
    got, dec = host_global_map(gm, clouds, ids, poses, leaf, pre7)
    want, cat = oracle_global_map(O, clouds, ids, poses, leaf, pre7)
    assert dec == int(declined), (leaf, dec)
    assert len(got) == len(want) and got.tobytes() == want.tobytes(), (leaf, len(got), len(want))
    if declined:
        assert got.tobytes() == cat.tobytes()             # PCL publishes the transformed concatenation itself
    return got


@pytest.mark.parametrize("stride", [48, 32])
@pytest.mark.parametrize("leaf", [0.3, 0.2])
def test_full_clouds_match_oracle_composition(gm, oracle, seqs, stride, leaf):
    seq = seqs[stride]
    full = [kf[3] for kf in seq]
    assert min(len(f) for f in full) > 10_000
    for ids in (list(range(0, 10, 2)), list(range(0, 10, 7)), [9, 1, 4]):
        poses = [nudge(seq[i][2], j) for j, i in enumerate(ids)]
        got = check(gm, oracle, full, ids, poses, leaf)
        assert 1000 < len(got) < sum(len(full[i]) for i in ids)


@pytest.mark.parametrize("stride", [48, 32])
def test_surf_clouds_with_pre_transform(gm, oracle, seqs, stride):
    """save_pcd: every surf frame through Tbl and then through its pose, the intermediate cloud in fp32"""
    seq = seqs[stride]
    surf = [kf[1] for kf in seq]
    ids = list(range(10))
    poses = [kf[2] for kf in seq]
    assert len(check(gm, oracle, surf, ids, poses, 0.2, pre7=T_BL)) > 500


@pytest.mark.parametrize("stride", [48, 32])
def test_repeated_keyframes_empty_and_non_finite_clouds(gm, oracle, seqs, stride):
    seq = seqs[stride]
    clouds = [kf[3][::4] for kf in seq[:5]]
    bad = clouds[2].copy()
    bad["x"][::9] = np.nan
    bad["y"][4::13] = np.inf
    bad["z"][7::17] = -np.inf
    clouds = clouds + [clouds[0][:0], bad, clouds[1][:1]]
    poses = [kf[2] for kf in seq]
    for ids in ([0, 0, 1, 0], [5, 3, 5, 6, 7, 6], [5], [6], [6, 6, 6]):
        ps = [nudge(poses[i % 5], j) for j, i in enumerate(ids)]
        for pre in (None, T_BL):
            check(gm, oracle, clouds, ids, ps, 0.3, pre7=pre)
    allbad = bad[~(np.isfinite(bad["x"]) & np.isfinite(bad["y"]) & np.isfinite(bad["z"]))]
    got = check(gm, oracle, clouds + [allbad], [8, 5], [poses[0], poses[1]], 0.3)
    assert len(got) == 0                                   # no finite point: nothing out
    assert len(check(gm, oracle, clouds, [], [], 0.3)) == 0


@pytest.mark.parametrize("stride", [48, 32])
def test_both_sides_of_the_overflow_test(gm, oracle, seqs, stride):
    """a small enough leaf makes dx*dy*dz exceed INT_MAX: PCL declines and the output is the transformed concatenation,
    non-finite points included"""
    seq = seqs[stride]
    clouds = [kf[3][::3].copy() for kf in seq]
    clouds[4]["x"][::11] = np.nan
    ids = list(range(0, 10, 3)) + [4]
    poses = [nudge(seq[i][2], j) for j, i in enumerate(ids)]
    from test_vg_box_host import np_params
    for leaf, declined in ((0.05, False), (0.004, True), (0.3, False)):
        _, cat = oracle_global_map(oracle, clouds, ids, poses, leaf)
        xyz = np.stack([cat["x"], cat["y"], cat["z"]], 1)
        xyz = xyz[np.isfinite(xyz).all(axis=1)]
        assert np_params(xyz.min(axis=0), xyz.max(axis=0), len(xyz), leaf)[4] == int(declined)    # PCL's test on this box
        check(gm, oracle, clouds, ids, poses, leaf, declined=declined)


def test_row_search(gm):
    n = np.array([5, 0, 3, 0, 0, 1, 7], np.int32)
    starts = np.cumsum(np.concatenate([[0], n[n > 0]]))[:-1]
    idx = np.arange(int(n.sum()), dtype=np.int64)
    row = np.zeros(len(idx), np.int32)
    gm.gm_rows_of(n, len(n), idx, len(idx), row)
    assert np.array_equal(row, np.searchsorted(starts, idx, side="right") - 1)


# ---------------------------------------------------------------- several stores: one arena per store against the merged store
@pytest.fixture(scope="module")
def stores():
    """three sessions' full clouds: store s holds the sweeps of a keyframe sequence of its own seed"""
    from liliom_b200 import synth
    return {st: [synth.make_keyframe_sequence(4, stride=st, seed=11 + s, full=True) for s in range(3)] for st in (48, 32)}


def _arena(clouds):
    """clouds back to back in reverse order (offsets that are not the list order): (arena, start of each cloud)"""
    order = list(range(len(clouds)))[::-1]
    start, off = {}, 0
    for i in order:
        start[i] = off
        off += len(clouds[i])
    arena = np.ascontiguousarray(np.concatenate([clouds[i] for i in order]))
    return arena, start


def _call(f, arenas, src, n, poses, pre7s, leaf, dt):
    k = len(n)
    total = int(np.sum(n)) if k else 0
    out = np.zeros(max(total, 1), dt)
    p = np.ascontiguousarray(np.asarray(poses, np.float64).reshape(-1, 7)) if k else np.zeros((1, 7))
    pre = None if pre7s is None else np.ascontiguousarray(np.asarray(pre7s, np.float64).reshape(-1, 7))
    ptrs = (C.c_void_p * max(len(arenas), 1))(*[a.ctypes.data for a in arenas])
    declined = C.c_int()
    m = f(ptrs, dt.itemsize, np.ascontiguousarray(src, np.int64), np.ascontiguousarray(n, np.int32), k, p.ctypes.data,
          None if pre is None else pre.ctypes.data, leaf, out.ctypes.data, C.byref(declined))
    assert m >= 0
    return out[:m], declined.value


def check_stores(gm, O, clouds_of, entries, poses, leaf, pre7s=None, declined=False):
    """entries: (store, keyframe) pairs; clouds_of[s][i] is keyframe i's cloud in store s"""
    dt = clouds_of[0][0].dtype
    # the stores: one arena each
    per = [_arena(cl) for cl in clouds_of]
    arenas_m = [per[s][0] for s, _ in entries]
    src_m = [per[s][1][i] for s, i in entries]
    n = [len(clouds_of[s][i]) for s, i in entries]
    got_m, dec_m = _call(gm.gmm_multi, arenas_m, src_m, n, poses, pre7s, leaf, dt)
    # the merged store D: every store's clouds in one arena
    flat = [(s, i) for s in range(len(clouds_of)) for i in range(len(clouds_of[s]))]
    arena_d, start_d = _arena([clouds_of[s][i] for s, i in flat])
    src_d = [start_d[flat.index(e)] for e in entries]
    got_d, dec_d = _call(gm.gmm_single, [arena_d], src_d, n, poses, pre7s, leaf, dt)
    assert dec_m == dec_d == int(declined)
    assert got_m.tobytes() == got_d.tobytes(), (leaf, len(got_m), len(got_d))
    # the oracle: per-entry pre-transforms composed one entry at a time
    pres = [None] * len(entries) if pre7s is None else list(np.asarray(pre7s, np.float64).reshape(-1, 7))
    parts = []
    for (s, i), p, pre in zip(entries, poses, pres):
        c = clouds_of[s][i] if pre is None else O.transform_cloud(clouds_of[s][i], pre)
        if len(c):
            parts.append(O.transform_cloud(c, p))
    cat = np.concatenate(parts) if parts else np.zeros(0, dt)
    want = cat if declined else O.voxelgrid(cat, leaf)
    assert got_m.tobytes() == want.tobytes()
    return got_m


@pytest.mark.parametrize("stride", [48, 32])
def test_rows_of_several_arenas_match_the_merged_store(gm, oracle, stores, stride):
    seqs = stores[stride]
    full = [[kf[3][::2] for kf in seq] for seq in seqs]
    entries = [(0, 1), (2, 0), (1, 3), (0, 1), (2, 2), (1, 0)]          # interleaved, one keyframe repeated
    poses = [nudge(seqs[s][i][2], j) for j, (s, i) in enumerate(entries)]
    for leaf in (0.3, 0.4):
        got = check_stores(gm, oracle, full, entries, poses, leaf)
        assert 500 < len(got) < sum(len(full[s][i]) for s, i in entries)


@pytest.mark.parametrize("stride", [48, 32])
def test_per_entry_pre_transforms(gm, oracle, stores, stride):
    """save_pcd over several robots: each entry through its own robot's Tbl, then its pose"""
    from liliom_b200 import synth
    seqs = stores[stride]
    surf = [[kf[1] for kf in seq] for seq in seqs]
    entries = [(s, i) for i in range(4) for s in range(3)]
    poses = [seqs[s][i][2] for s, i in entries]
    tbls = [T_BL, np.array([1.0, 0, 0, 0, 0.1, -0.02, 0.3]),
            np.concatenate([synth.q_from_axis_angle([0, 1, 0], np.deg2rad(3.0)), [0.05, 0.0, -0.1]])]
    pre7s = [tbls[s] for s, _ in entries]
    assert len(check_stores(gm, oracle, surf, entries, poses, 0.2, pre7s=pre7s)) > 300
    # the same pre for every entry: the single-store call's shared pre7
    assert len(check_stores(gm, oracle, surf, entries, poses, 0.2, pre7s=[T_BL] * len(entries))) > 300


@pytest.mark.parametrize("stride", [48, 32])
def test_non_finite_empty_and_declined(gm, oracle, stores, stride):
    seqs = stores[stride]
    clouds = [[kf[3][::5].copy() for kf in seq] for seq in seqs]
    clouds[1][2]["x"][::7] = np.nan
    clouds[2][1]["z"][3::11] = np.inf
    clouds[0][3] = clouds[0][3][:0]                                       # an empty stored cloud
    entries = [(1, 2), (0, 3), (2, 1), (1, 2)]
    poses = [nudge(seqs[s][i][2], j) for j, (s, i) in enumerate(entries)]
    check_stores(gm, oracle, clouds, entries, poses, 0.3)
    check_stores(gm, oracle, clouds, entries, poses, 0.004, declined=True)      # PCL declines: the transformed concatenation
    assert len(check_stores(gm, oracle, clouds, [], [], 0.3)) == 0
