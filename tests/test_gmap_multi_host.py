"""CPU tier for the multi-store global map (liliom_global_map_multi): kf_table.h's two row types compiled for the host
(tests/gmap_multi_host.cpp) and composed as the device composes them.  Rows that each name an arena of their own (KfRowM, one
arena per store) must give, byte for byte, what rows over one arena holding the same clouds give (KfRow, the merged store),
and the oracle's voxelgrid(concat(transform_cloud(...))): both point layouts, per-entry pre-transforms, interleaved and repeated
lists, non-finite points, and PCL's declined case."""
import ctypes as C

import numpy as np
import pytest

import host_build
from test_gmap_host import T_BL, nudge, oracle_global_map


@pytest.fixture(scope="module")
def gmm():
    L = host_build.load("gmap_multi_host", ["tests/gmap_multi_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall", "-ffp-contract=off"],
                        deps=[f"liliom_b200/csrc/{h}" for h in ("kf_table.h", "pcl_xform.h", "vg_box.h")])
    vp, llp, ip = C.c_void_p, np.ctypeslib.ndpointer(np.int64, flags="C"), np.ctypeslib.ndpointer(np.int32, flags="C")
    for f in (L.gmm_single, L.gmm_multi):
        f.argtypes = [C.POINTER(vp), C.c_int, llp, ip, C.c_int, vp, vp, C.c_float, vp, C.POINTER(C.c_int)]
        f.restype = C.c_longlong
    return L


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


def check(gmm, O, clouds_of, entries, poses, leaf, pre7s=None, declined=False):
    """entries: (store, keyframe) pairs; clouds_of[s][i] is keyframe i's cloud in store s"""
    dt = clouds_of[0][0].dtype
    # the stores: one arena each
    per = [_arena(cl) for cl in clouds_of]
    arenas_m = [per[s][0] for s, _ in entries]
    src_m = [per[s][1][i] for s, i in entries]
    n = [len(clouds_of[s][i]) for s, i in entries]
    got_m, dec_m = _call(gmm.gmm_multi, arenas_m, src_m, n, poses, pre7s, leaf, dt)
    # the merged store D: every store's clouds in one arena
    flat = [(s, i) for s in range(len(clouds_of)) for i in range(len(clouds_of[s]))]
    arena_d, start_d = _arena([clouds_of[s][i] for s, i in flat])
    src_d = [start_d[flat.index(e)] for e in entries]
    got_d, dec_d = _call(gmm.gmm_single, [arena_d], src_d, n, poses, pre7s, leaf, dt)
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
def test_rows_of_several_arenas_match_the_merged_store(gmm, oracle, stores, stride):
    seqs = stores[stride]
    full = [[kf[3][::2] for kf in seq] for seq in seqs]
    entries = [(0, 1), (2, 0), (1, 3), (0, 1), (2, 2), (1, 0)]          # interleaved, one keyframe repeated
    poses = [nudge(seqs[s][i][2], j) for j, (s, i) in enumerate(entries)]
    for leaf in (0.3, 0.4):
        got = check(gmm, oracle, full, entries, poses, leaf)
        assert 500 < len(got) < sum(len(full[s][i]) for s, i in entries)


@pytest.mark.parametrize("stride", [48, 32])
def test_per_entry_pre_transforms(gmm, oracle, stores, stride):
    """save_pcd over several robots: each entry through its own robot's Tbl, then its pose"""
    from liliom_b200 import synth
    seqs = stores[stride]
    surf = [[kf[1] for kf in seq] for seq in seqs]
    entries = [(s, i) for i in range(4) for s in range(3)]
    poses = [seqs[s][i][2] for s, i in entries]
    tbls = [T_BL, np.array([1.0, 0, 0, 0, 0.1, -0.02, 0.3]),
            np.concatenate([synth.q_from_axis_angle([0, 1, 0], np.deg2rad(3.0)), [0.05, 0.0, -0.1]])]
    pre7s = [tbls[s] for s, _ in entries]
    assert len(check(gmm, oracle, surf, entries, poses, 0.2, pre7s=pre7s)) > 300
    # the same pre for every entry: the single-store call's shared pre7
    assert len(check(gmm, oracle, surf, entries, poses, 0.2, pre7s=[T_BL] * len(entries))) > 300


@pytest.mark.parametrize("stride", [48, 32])
def test_non_finite_empty_and_declined(gmm, oracle, stores, stride):
    seqs = stores[stride]
    clouds = [[kf[3][::5].copy() for kf in seq] for seq in seqs]
    clouds[1][2]["x"][::7] = np.nan
    clouds[2][1]["z"][3::11] = np.inf
    clouds[0][3] = clouds[0][3][:0]                                       # an empty stored cloud
    entries = [(1, 2), (0, 3), (2, 1), (1, 2)]
    poses = [nudge(seqs[s][i][2], j) for j, (s, i) in enumerate(entries)]
    check(gmm, oracle, clouds, entries, poses, 0.3)
    check(gmm, oracle, clouds, entries, poses, 0.004, declined=True)      # PCL declines: the transformed concatenation
    assert len(check(gmm, oracle, clouds, [], [], 0.3)) == 0
