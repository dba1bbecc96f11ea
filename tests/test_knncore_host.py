"""CPU tier for the PRUNED SEARCH of the scan-to-map kernels: liliom_b200/csrc/knn_core.cuh compiled for the host
(tests/knncore_host.cpp) and compared, key for key, with an exhaustive search over the whole map.  What must hold (DESIGN.md §3.1):
the running threshold, the cell lower bounds, the trimming of runs, the per-thread run list, the per-lane rows and butterfly merge
of the 2/4/8/16-lane shape and a tightened start threshold (temporal coherence) never change the five smallest (fp32 distance,
index) keys inside the gate; the coherence bound of the GN passes (coherence_tau) keeps every point of the previous set; a query with fewer than five points inside the gate keeps exactly those; points outside the 3x3x3
cell block are never inside the gate; every lane of a group ends with the merged set.  The plain reference the GPU tier compares
the device with (tests/knn_reference.py) is itself checked here against the host build."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "build", "libknncore_host.so")
F = np.float32
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


@pytest.fixture(scope="module")
def kc():
    src = os.path.join(ROOT, "tests", "knncore_host.cpp")
    hdrs = [os.path.join(ROOT, "liliom_b200", "csrc", h) for h in ("knn_core.cuh", "dev_math.cuh", "ctx.cuh")]
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("CUDA headers not found")
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(p) for p in [src] + hdrs):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++20", "-pthread", "-fPIC", "-ffp-contract=off", "-frounding-math", "-D_GNU_SOURCE", "-Wno-attributes", "-Wno-unknown-pragmas",
                        "-I", cuda_inc, "-shared", "-o", SO, src], check=True)
    L = C.CDLL(SO)
    L.kc_gate_tau.argtypes = [C.c_double]; L.kc_gate_tau.restype = C.c_float
    L.kc_thread_knn5.argtypes = [C.c_float, C.c_float, C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_int), C.c_float,
                                 C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_float, C.POINTER(C.c_uint64)]
    L.kc_thread_knn5.restype = C.c_uint64
    L.kc_group_knn5.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p]
    L.kc_group_knn5.restype = C.c_int
    L.kc_coherence_tau.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p]
    L.kc_coherence_tau.restype = None
    L.kc_owner_of.argtypes = [C.c_float, C.c_float, C.c_float, C.c_int, C.c_float]; L.kc_owner_of.restype = C.c_int
    return L


def _grid(pts, cell=1.0):
    """The cell grid of grid_build (liliom_b200/csrc/grid_knn.cu): cells floor(p / cell), x fastest, dense cell_start."""
    inv = F(1.0 / cell)
    c = np.floor(pts * inv).astype(np.int64)
    org = c.min(0); dim = c.max(0) - org + 1
    rel = c - org
    key = (rel[:, 2] * dim[1] + rel[:, 1]) * dim[0] + rel[:, 0]
    order = np.argsort(key, kind="stable")
    ms = np.zeros((len(pts), 4), F)
    ms[:, :3] = pts[order]
    ms[:, 3] = order.astype(np.int32).view(F)                      # w = index into the un-sorted map
    ncells = int(dim.prod())
    cell_start = np.searchsorted(key[order], np.arange(ncells + 1)).astype(np.int32)
    return ms, cell_start, org.astype(np.int32), dim.astype(np.int32), inv


def _exhaustive(q, pts, tau):
    """Five smallest (bits(d) << 32 | index) keys with d <= tau; d = ((dx*dx) + dy*dy) + dz*dz in fp32, dx = q - p (FLANN L2_Simple)."""
    d = pts.astype(F)
    dx = F(q[0]) - d[:, 0]; dy = F(q[1]) - d[:, 1]; dz = F(q[2]) - d[:, 2]
    dist = (dx * dx + dy * dy) + dz * dz
    assert dist.dtype == F
    keep = np.nonzero(dist <= tau)[0]
    keys = (dist[keep].view(np.uint32).astype(np.uint64) << np.uint64(32)) | keep.astype(np.uint64)
    keys.sort()
    out = np.full(5, EMPTY, np.uint64)
    out[: min(5, len(keys))] = keys[:5]
    return out, dist


def _search(kc, q, grid, tau):
    ms, cs, org, dim, inv = grid
    out = np.zeros(5, np.uint64)
    cand = kc.kc_thread_knn5(F(q[0]), F(q[1]), F(q[2]), ms.ctypes.data_as(C.POINTER(C.c_float)), cs.ctypes.data_as(C.POINTER(C.c_int)), inv,
                             org.ctypes.data_as(C.POINTER(C.c_int)), dim.ctypes.data_as(C.POINTER(C.c_int)), F(tau),
                             out.ctypes.data_as(C.POINTER(C.c_uint64)))
    return out, int(cand)


def _group_search(kc, lanes, queries, grid, taus):
    """kc_group_knn5: (keys [n, 5], every lane holds the merged set [n], examined candidates [n])."""
    ms, cs, org, dim, inv = grid
    q3 = np.ascontiguousarray(np.asarray(queries, F)[:, :3])
    taus = np.ascontiguousarray(np.broadcast_to(np.asarray(taus, F), (len(q3),)))
    out = np.zeros((len(q3), 5), np.uint64); agree = np.zeros(len(q3), np.int32); cand = np.zeros(len(q3), np.uint64)
    rc = kc.kc_group_knn5(lanes, len(q3), q3.ctypes.data, ms.ctypes.data, cs.ctypes.data, inv, org.ctypes.data, dim.ctypes.data,
                          taus.ctypes.data, out.ctypes.data, agree.ctypes.data, cand.ctypes.data)
    assert rc == 0
    return out, agree.astype(bool), cand


SEEDED = [(0, 3.0), (1, 12.0), (2, 40.0), (3, 0.6)]


def _seeded_world(seed, density):
    """Uniform points at `density` per cubic metre with adversarial structure: exact duplicates (index tie-break), points on cell
    faces, a lattice with equal distances; queries inside and outside the grid, on cell corners and equidistant from lattice points."""
    rng = np.random.default_rng(seed)
    ext = np.array([9.0, 7.0, 4.0])
    m = int(density * ext.prod())
    pts = (rng.uniform(-0.5, 0.5, (m, 3)) * ext + np.array([100.3, -40.7, 2.2])).astype(F)
    pts[: m // 20] = pts[m // 20: 2 * (m // 20)]
    pts[-(m // 25):] = np.round(pts[-(m // 25):])
    lat = np.stack(np.meshgrid(np.arange(-2, 3), np.arange(-2, 3), np.arange(-1, 2), indexing="ij"), -1).reshape(-1, 3) * 0.25
    pts = np.concatenate([pts, (lat + np.array([100.0, -41.0, 2.0])).astype(F)])
    queries = np.concatenate([
        (rng.uniform(-0.55, 0.55, (400, 3)) * ext + np.array([100.3, -40.7, 2.2])),     # some outside the grid
        np.round(rng.uniform(-0.5, 0.5, (60, 3)) * ext + np.array([100.3, -40.7, 2.2])),  # on cell corners
        lat[:40] + np.array([100.0, -41.0, 2.0]) + 0.125,                                  # equidistant from lattice points
    ]).astype(F)
    return pts, queries


def _coherence_thresholds(want, gate):
    """For every query with five keys: start thresholds >= its true fifth distance (the fifth itself, one float above, and a loose
    bound below the gate).  Returns (query rows, thresholds)."""
    rows, taus = [], []
    for i, w in enumerate(want):
        if w[4] == EMPTY:
            continue
        d5 = F(np.uint32(w[4] >> np.uint64(32)).view(F))
        for t in (d5, np.nextafter(d5, F(2.0)), F(min(float(d5) * 1.5 + 1e-3, float(gate)))):
            rows.append(i); taus.append(t)
    return np.array(rows, np.int64), np.array(taus, F)


@pytest.mark.parametrize("seed,density", SEEDED)
def test_pruned_search_equals_exhaustive_search(kc, seed, density):
    pts, queries = _seeded_world(seed, density)
    grid = _grid(pts)
    gate = kc.kc_gate_tau(1.0)
    assert gate < 1.0 and np.nextafter(F(gate), F(2.0)) >= 1.0
    examined = []
    n_full = 0
    for q in queries:
        want, dist = _exhaustive(q, pts, gate)
        got, cand = _search(kc, q, grid, gate)
        assert np.array_equal(got, want), (q, got, want)
        examined.append(cand)
        if want[4] != EMPTY:
            n_full += 1
            # temporal coherence: any start threshold >= the true fifth distance gives the same five keys and examines no more
            d5 = F(np.uint32(want[4] >> np.uint64(32)).view(F))
            for t in (d5, np.nextafter(d5, F(2.0)), F(min(float(d5) * 1.5 + 1e-3, float(gate)))):
                got2, cand2 = _search(kc, q, grid, t)
                assert np.array_equal(got2, want), (q, t)
                assert cand2 <= cand
        # exactness of the 3x3x3 block: nothing outside it is inside the gate
        c = np.floor(pts).astype(np.int64); cq = np.floor(q).astype(np.int64)
        outside = (np.abs(c - cq) > 1).any(1)
        assert not (dist[outside] <= gate).any()
    assert n_full > 50 or density < 1.0
    # the pruning prunes: on dense maps most of the block is never fetched
    if density >= 12.0:
        block = np.array([((np.abs(np.floor(pts).astype(np.int64) - np.floor(q).astype(np.int64)) <= 1).all(1)).sum() for q in queries[:100]])
        assert np.mean(examined[:100]) < 0.8 * np.mean(block)


@pytest.mark.parametrize("lanes", [2, 4, 8, 16])
@pytest.mark.parametrize("seed,density", SEEDED)
def test_group_search_equals_exhaustive_search(kc, seed, density, lanes):
    """group_knn5<lanes> (each lane ranks rows sub, sub + lanes, ... into a private top-5 with its own running threshold, then five
    butterfly rounds merge them) against the exhaustive search, key for key, with the gate and with coherence start thresholds."""
    pts, queries = _seeded_world(seed, density)
    grid = _grid(pts)
    gate = F(kc.kc_gate_tau(1.0))
    want = np.stack([_exhaustive(q, pts, gate)[0] for q in queries])
    got, agree, cand = _group_search(kc, lanes, queries, grid, gate)
    bad = np.nonzero((got != want).any(1))[0]
    assert len(bad) == 0, (lanes, queries[bad[:3]], got[bad[:3]], want[bad[:3]])
    assert agree.all(), np.nonzero(~agree)[0][:5]
    assert (want[:, 4] != EMPTY).sum() > 50 or density < 1.0
    if density < 12.0:                                        # empty and partial sets occur
        assert (want[:, 0] == EMPTY).any() and ((want[:, 0] != EMPTY) & (want[:, 4] == EMPTY)).any()
    rows, taus = _coherence_thresholds(want, gate)
    got2, agree2, cand2 = _group_search(kc, lanes, queries[rows], grid, taus)
    assert np.array_equal(got2, want[rows]) and agree2.all(), lanes
    assert (cand2 <= cand[rows]).all()                       # a tighter start examines no more


def _coherence_tau(kc, old, d5, new, gate):
    st = np.ascontiguousarray(np.concatenate([np.asarray(old, F), np.asarray(d5, F)[:, None]], 1))
    s3 = np.ascontiguousarray(np.asarray(new, F))
    out = np.zeros(len(s3), F)
    kc.kc_coherence_tau(len(s3), st.ctypes.data, s3.ctypes.data, F(gate), out.ctypes.data)
    return out


def test_coherence_bound_covers_the_previous_neighbours(kc):
    """coherence_tau (the start threshold of every GN pass after the first) must keep every map point that lay within the previous
    fifth distance d5 at the previous position p': its fp32 distance from the new position p may not exceed the bound.  The tight
    case is a move straight away from the point (|p - n| = |p' - n| + |p - p'| in exact arithmetic): there only the upward roundings
    and the relative margin separate the bound from the candidate's own rounded distance.  Points at 0.05 - 0.99 m, moves from
    1e-9 to 1e-2 m, map coordinates up to 200 m; plus oblique moves, no move, a point on the previous position, and no previous
    set (d5 beyond the gate, +inf, NaN)."""
    import knn_reference as R
    gate = F(kc.kc_gate_tau(1.0))
    rng = np.random.default_rng(17)
    n_pts = 200_000
    pt = rng.uniform(-200, 200, (n_pts, 3)).astype(F)
    u = rng.normal(size=(n_pts, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    r0 = rng.uniform(0.05, 0.99, (n_pts, 1))
    step = 10.0 ** rng.uniform(-9, -2, (n_pts, 1))
    old = (pt + r0 * u).astype(F)
    away = (old + step * u).astype(F)                                          # straight away from the point
    w = rng.normal(size=(n_pts, 3)); w /= np.linalg.norm(w, axis=1, keepdims=True)
    oblique = (old + step * 10.0 * w).astype(F)
    for new, tight in ((away, True), (oblique, False), (old, False)):
        d5 = R.fp32_sqdist(old, pt)
        tau = _coherence_tau(kc, old, d5, new, gate)
        dn = R.fp32_sqdist(new, pt)
        inside = dn <= gate
        bad = np.nonzero(inside & (dn > tau))[0]
        assert len(bad) == 0, (len(bad), old[bad[:3]], new[bad[:3]], pt[bad[:3]], d5[bad[:3]], dn[bad[:3]], tau[bad[:3]])
        assert (tau <= gate).all() and (tau >= d5).all()
        if tight:
            # the moves do press against the margin: the closest cases keep less than 0.1 % more than the margin's 1e-5
            free = tau < gate
            slack = (tau[free].astype(np.float64) - dn[free]) / dn[free]
            assert slack.min() < 1.001e-5, slack.min()
    # the previous position itself (d5 = 0) and a point right there after a move
    z = np.zeros(n_pts, F)
    assert (_coherence_tau(kc, old, z, old, gate) == 0).all()
    tau = _coherence_tau(kc, old, z, away, gate)
    assert (R.fp32_sqdist(away, old) <= tau).all()
    # nothing to exploit: the full gate
    for d in (np.nextafter(gate, F(2)), F(np.inf), F(np.nan)):
        assert (_coherence_tau(kc, old[:100], np.full(100, d, F), away[:100], gate) == gate).all()


def test_reference_equals_host_search(kc):
    """The kd-tree reference of the GPU tier (tests/knn_reference.py, no cell grid) against the one-thread search compiled for the
    host and the exhaustive search, on the seeded worlds and on the adversarial map of the GPU tier."""
    import knn_reference as R
    gate = F(kc.kc_gate_tau(1.0))
    assert R.gate_tau(1.0) == gate
    worlds = [_seeded_world(s, d) for s, d in SEEDED]
    m, qs, _ = R.adversarial_world(0)
    worlds.append((m[:, :3], qs[:, :3]))
    for pts, queries in worlds:
        idx, sqd, keys = R.reference_knn5(queries, pts, gate)
        grid = _grid(pts)
        for i, q in enumerate(queries):
            assert np.array_equal(keys[i], _search(kc, q, grid, gate)[0]), (q, keys[i])
            assert np.array_equal(keys[i], _exhaustive(q, pts, gate)[0]), q
        full = idx[:, 4] >= 0
        assert np.array_equal(sqd[full].view(np.uint32), (keys[full] >> np.uint64(32)).astype(np.uint32))
        assert ((idx < 0) == (keys == EMPTY)).all()


@pytest.mark.parametrize("lanes", [1, 2, 4, 8, 16])
def test_search_on_adversarial_world(kc, lanes):
    """Every shape on the adversarial map of the GPU tier: a point seven times, cell corners, an equidistant lattice, an 80-point
    clump in one cell, sparse queries with 0 - 4 neighbours, map points exactly on the gate (d == tau0, kept) and one float beyond
    it (d == 1.0f, dropped), queries outside the grid on all six sides; and the coherence property on all of it."""
    import knn_reference as R
    m, qs, notes = R.adversarial_world(0)
    pts = m[:, :3]
    gate = F(kc.kc_gate_tau(1.0))
    _, _, want = R.reference_knn5(qs, pts, gate)
    grid = _grid(pts)
    # the map really has the structure the cases are about
    d5 = (want[:, 4] >> np.uint64(32)).astype(np.uint32).view(F)
    s0, s1 = notes["sparse"]
    nfound = (want[s0:s1] != EMPTY).sum(1)
    assert set(nfound.tolist()) == {0, 1, 2, 3, 4, 5}
    assert (d5[s0:s1] == gate).sum() >= 3                                     # fifth neighbour exactly on the gate
    assert (want[notes["duplicates"][0]] >> np.uint64(32) == 0).all()      # five of the seven copies, at distance 0
    o0, o1 = notes["outside"]
    assert (want[o0:o1, 0] == EMPTY).any() and (want[o0:o1, 0] != EMPTY).any()
    if lanes == 1:
        got = np.stack([_search(kc, q, grid, gate)[0] for q in qs])
        agree = np.ones(len(qs), bool)
    else:
        got, agree, cand = _group_search(kc, lanes, qs, grid, gate)
    bad = np.nonzero((got != want).any(1))[0]
    assert len(bad) == 0, (lanes, bad[:5], got[bad[:3]], want[bad[:3]])
    assert agree.all()
    rows, taus = _coherence_thresholds(want, gate)
    if lanes == 1:
        got2 = np.stack([_search(kc, qs[r], grid, t)[0] for r, t in zip(rows, taus)])
    else:
        got2, agree2, _ = _group_search(kc, lanes, qs[rows], grid, taus)
        assert agree2.all()
    assert np.array_equal(got2, want[rows])


def test_partition_rule_mirror_equals_the_device_function(kc):
    """liliom_b200/sharding.py::owner_of (what the gloo tests and the bench's shard report use) against knn_core.cuh::owner_of compiled
    for the host: same rank for points on both sides of cube faces, negative coordinates, the half-cube z shift, every rank count."""
    from liliom_b200 import sharding
    rng = np.random.default_rng(11)
    pts = np.concatenate([
        rng.uniform(-700, 700, (3000, 3)),
        np.round(rng.uniform(-40, 40, (600, 3))) * 16.0 + rng.choice([-1e-3, 0.0, 1e-3], (600, 3)),          # on / beside 16 m faces
        np.round(rng.uniform(-10, 10, (600, 3))) * 64.0 + np.array([0.0, 0.0, 32.0]) + rng.choice([-1e-3, 0.0, 1e-3], (600, 3)),
    ]).astype(F)
    for block in (16, 64):
        for nranks in (1, 2, 3, 4, 8, 16):
            want = sharding.owner_of(pts, nranks, block)
            got = np.array([kc.kc_owner_of(F(p[0]), F(p[1]), F(p[2]), nranks, F(1.0 / block)) for p in pts], np.int32)
            assert np.array_equal(got, want), (block, nranks)
            assert got.min() >= 0 and got.max() < nranks
            if nranks > 1:
                share = np.bincount(got[:3000], minlength=nranks) / 3000.0
                assert share.max() < 2.2 / nranks                                   # the linear hash spreads a 1.4 km stretch evenly
