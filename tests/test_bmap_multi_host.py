"""CPU tier for the multi-store backend local map (liliom_bmap_build_multi and its batch): the local map's table builder
(kf_table.h's kf_bmap_rows) compiled for the host for both row types (tests/bmap_multi_host.cpp) and composed as the device
composes it.  Rows that each name the arena of their entry's store (KfRowM) must give, byte for byte, the rows and the
edge-then-surf concatenation that KfRow rows over one merged arena holding the same clouds give; each layer's VoxelGrid must be
the oracle's voxelgrid(concat(transform_cloud(...))).  Both point layouts, interleaved and repeated lists, stores of different
sizes, and keyframes whose edge or surf cloud is empty."""
import ctypes as C

import numpy as np
import pytest

import host_build
from test_gmap_host import nudge


@pytest.fixture(scope="module")
def bm():
    L = host_build.load("bmap_multi_host", ["tests/bmap_multi_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall", "-ffp-contract=off"],
                        deps=[f"liliom_b200/csrc/{h}" for h in ("kf_table.h", "pcl_xform.h", "vg_box.h")])
    vp, llp, ip = C.c_void_p, np.ctypeslib.ndpointer(np.int64, flags="C"), np.ctypeslib.ndpointer(np.int32, flags="C")
    for f in (L.bm_gather_single, L.bm_gather_multi):
        f.argtypes = [C.POINTER(vp), C.c_int, llp, llp, ip, ip, C.c_int, vp, vp, llp, C.POINTER(C.c_longlong), llp]
        f.restype = C.c_int
    L.bm_voxelgrid.argtypes = [vp, C.c_longlong, C.c_int, C.c_float, vp]
    L.bm_voxelgrid.restype = C.c_longlong
    return L


@pytest.fixture(scope="module")
def stores():
    """three sessions' (edge, surf, pose) keyframes, stores of 3, 6 and 4 keyframes, for each point layout"""
    from liliom_b200 import synth
    return {st: [synth.make_keyframe_sequence(n, stride=st, seed=21 + s)[:n] for s, n in enumerate((3, 6, 4))] for st in (48, 32)}


def _arena(kfs):
    """a store's arena: each keyframe's edge points then its surf points, keyframes back to back in reverse order (offsets that
    are not the list order).  Returns (arena, edge_off, surf_off) per keyframe."""
    parts, eo, so, off = [], {}, {}, 0
    for i in reversed(range(len(kfs))):
        e, s = kfs[i][0], kfs[i][1]
        eo[i], so[i] = off, off + len(e)
        off += len(e) + len(s)
        parts += [e, s]
    dt = kfs[0][0].dtype
    arena = np.ascontiguousarray(np.concatenate([p for p in parts if len(p)] or [np.zeros(1, dt)]))
    return arena, eo, so


def _gather(f, arenas, eo, so, ne, ns, poses, dt):
    k = len(ne)
    E, S = int(np.sum(ne)) if k else 0, int(np.sum(ns)) if k else 0
    out = np.zeros(max(E + S, 1), dt)
    p = np.ascontiguousarray(np.asarray(poses, np.float64).reshape(-1, 7)) if k else np.zeros((1, 7))
    ptrs = (C.c_void_p * max(len(arenas), 1))(*[a.ctypes.data for a in arenas])
    n = np.zeros(2, np.int64)
    largest = C.c_longlong(-1)
    rows = np.zeros(3 * max(2 * k, 1), np.int64)
    r = f(ptrs, dt.itemsize, np.ascontiguousarray(eo, np.int64), np.ascontiguousarray(so, np.int64), np.ascontiguousarray(ne, np.int32),
          np.ascontiguousarray(ns, np.int32), k, p.ctypes.data, out.ctypes.data, n, C.byref(largest), rows)
    return out[:E + S], tuple(n), largest.value, rows[:3 * r].reshape(-1, 3)


def _vg(bm, pts, leaf):
    out = np.zeros(max(len(pts), 1), pts.dtype)
    m = bm.bm_voxelgrid(pts.ctypes.data if len(pts) else None, len(pts), pts.dtype.itemsize, leaf, out.ctypes.data)
    assert m >= 0
    return out[:m]


def _cat(parts, dt):
    parts = [p for p in parts if len(p)]
    return np.concatenate(parts) if parts else np.zeros(0, dt)


def check(bm, O, kfs_of, entries, poses, leaves=(0.2, 0.4)):
    """entries: (store, keyframe) pairs; kfs_of[s][i] = (edge, surf, ...) of keyframe i of store s"""
    dt = kfs_of[0][0][0].dtype
    ne = [len(kfs_of[s][i][0]) for s, i in entries]
    ns = [len(kfs_of[s][i][1]) for s, i in entries]
    # the stores: one arena each
    per = [_arena(kfs) for kfs in kfs_of]
    got = _gather(bm.bm_gather_multi, [per[s][0] for s, _ in entries], [per[s][1][i] for s, i in entries],
                  [per[s][2][i] for s, i in entries], ne, ns, poses, dt)
    # the merged store D: every store's keyframes in one arena
    flat = [(s, i) for s in range(len(kfs_of)) for i in range(len(kfs_of[s]))]
    arena_d, eo_d, so_d = _arena([kfs_of[s][i] for s, i in flat])
    want = _gather(bm.bm_gather_single, [arena_d], [eo_d[flat.index(e)] for e in entries], [so_d[flat.index(e)] for e in entries],
                   ne, ns, poses, dt)
    assert got[0].tobytes() == want[0].tobytes()
    assert got[1:3] == want[1:3] and np.array_equal(got[3][:, :2], want[3][:, :2])
    E, S = got[1]
    assert (E, S) == (sum(ne), sum(ns)) and got[2] == max([max(a, b) for a, b in zip(ne, ns)] or [0])
    # the rows, entry by entry in list order: its edge row (destinations from 0), then its surf row (from E); an empty cloud has none
    rows, de, ds = [], 0, E
    for a, b in zip(ne, ns):
        rows += ([(de, a)] if a else []) + ([(ds, b)] if b else [])
        de, ds = de + a, ds + b
    assert [tuple(r) for r in got[3][:, :2].tolist()] == rows
    # each layer: the oracle's composition
    edge = _cat([O.transform_cloud(kfs_of[s][i][0], p) for (s, i), p in zip(entries, poses)], dt)
    surf = _cat([O.transform_cloud(kfs_of[s][i][1], p) for (s, i), p in zip(entries, poses)], dt)
    assert got[0][:E].tobytes() == edge.tobytes() and got[0][E:].tobytes() == surf.tobytes()
    for leaf in leaves:
        for lo, hi, cat in ((0, E, edge), (E, E + S, surf)):
            vg = _vg(bm, np.ascontiguousarray(got[0][lo:hi]), leaf)
            assert vg.tobytes() == O.voxelgrid(cat, leaf).tobytes(), leaf
    return got


@pytest.mark.parametrize("stride", [48, 32])
def test_rows_of_several_stores_match_the_merged_store(bm, oracle, stores, stride):
    kfs = stores[stride]
    for entries in ([(0, 1), (1, 4), (2, 0), (0, 1), (1, 5), (2, 3), (1, 0)],         # interleaved, one keyframe repeated
                    [(1, i) for i in range(6)] + [(0, 2), (2, 2), (2, 2)],
                    [(2, 1)]):
        poses = [nudge(kfs[s][i][2], j) for j, (s, i) in enumerate(entries)]
        got = check(bm, oracle, kfs, entries, poses)
        assert got[1][0] > 0 and got[1][1] > 0


@pytest.mark.parametrize("stride", [48, 32])
def test_empty_edge_or_surf_clouds_and_empty_lists(bm, oracle, stores, stride):
    kfs = [[list(kf) for kf in seq] for seq in stores[stride]]
    kfs[0][1][0] = kfs[0][1][0][:0]                    # no edge points
    kfs[1][3][1] = kfs[1][3][1][:0]                    # no surf points
    kfs[2][2][0] = kfs[2][2][0][:0]                    # neither
    kfs[2][2][1] = kfs[2][2][1][:0]
    entries = [(0, 1), (2, 2), (1, 3), (0, 0), (2, 2), (1, 3)]
    poses = [nudge(kfs[s][i][2], j) for j, (s, i) in enumerate(entries)]
    check(bm, oracle, kfs, entries, poses)
    check(bm, oracle, kfs, [(2, 2)], [kfs[2][2][2]])   # both layers empty
    check(bm, oracle, kfs, [(0, 1), (0, 1)], [kfs[0][1][2]] * 2)        # no edge layer
    assert check(bm, oracle, kfs, [], [])[1] == (0, 0)
