"""CPU tier for the global map's table filter (liliom_global_map): liliom_b200/csrc/kf_table.h compiled for the host with
vg_box.h and pcl_xform.h (tests/gmap_host.cpp) and composed as the device composes it (box of the transformed rows, voxel keys,
stable sort, heads, vg_walk through the transforming loader, the centroid writer; PCL's declined case gathers), against the
oracle's voxelgrid(concat(transform_cloud(...))) byte for byte: both point layouts, with and without the pre-transform of
save_pcd, lists that repeat keyframes, empty clouds, non-finite points, and boxes on both sides of PCL's overflow test."""
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
