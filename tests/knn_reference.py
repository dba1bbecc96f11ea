"""TEST INFRASTRUCTURE: a plain reference of the scan-to-map 5-NN search and an adversarial map to run it on.

reference_knn5 is what liliom_b200/csrc/knn_core.cuh must compute, written without the cell grid: candidates come from a kd-tree
ball slightly larger than the gate (fp64, scipy), their distances are FLANN's fp32 expression ((dx*dx) + dy*dy) + dz*dz, a
candidate is kept when d <= tau0 (the largest float below the gate, knn_gate_tau), and the five smallest (distance bits, map index)
keys are the answer.  The CPU tier checks it against the host build of the search; the GPU tier checks the device against it."""
import numpy as np
from scipy.spatial import cKDTree

F = np.float32


def gate_tau(max_sqd=1.0):
    """Largest float t with (double)t < max_sqd (knn_gate_tau)."""
    t = F(max_sqd)
    while float(t) >= max_sqd:
        t = np.nextafter(t, F(-np.inf))
    while float(np.nextafter(t, F(np.inf))) < max_sqd:
        t = np.nextafter(t, F(np.inf))
    return t


def fp32_sqdist(q, p):
    """FLANN L2_Simple<float>: ((dx*dx) + dy*dy) + dz*dz in fp32, dx = q - p, no contraction."""
    q = np.asarray(q, F); p = np.asarray(p, F)
    dx = q[..., 0] - p[..., 0]; dy = q[..., 1] - p[..., 1]; dz = q[..., 2] - p[..., 2]
    d = (dx * dx + dy * dy) + dz * dz
    assert d.dtype == F
    return d


def reference_knn5(queries, pts, tau0):
    """(idx, sqd, keys) of the five nearest map points inside d <= tau0 for every query; empty slots: index -1, key ~0."""
    q = np.ascontiguousarray(np.asarray(queries, F)[:, :3])
    p = np.ascontiguousarray(np.asarray(pts, F)[:, :3])
    n = len(q)
    r = float(np.sqrt(float(tau0))) * (1.0 + 1e-5) + 1e-6        # fp32 rounding moves a distance by a few 1e-7 relative
    lists = cKDTree(p.astype(np.float64)).query_ball_point(q.astype(np.float64), r)
    cnt = np.fromiter((len(c) for c in lists), np.int64, n)
    qi = np.repeat(np.arange(n), cnt)
    pi = np.fromiter((j for c in lists for j in c), np.int64, int(cnt.sum()))
    d = fp32_sqdist(q[qi], p[pi])
    keep = d <= F(tau0)
    qi, pi, d = qi[keep], pi[keep], d[keep]
    keys = (d.view(np.uint32).astype(np.uint64) << np.uint64(32)) | pi.astype(np.uint64)
    order = np.lexsort((keys, qi))
    qi, keys = qi[order], keys[order]
    first = np.searchsorted(qi, np.arange(n))
    rank = np.arange(len(qi)) - first[qi]
    top = rank < 5
    out = np.full((n, 5), np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64)
    out[qi[top], rank[top]] = keys[top]
    empty = out == np.uint64(0xFFFFFFFFFFFFFFFF)
    idx = np.where(empty, -1, (out & np.uint64(0xFFFFFFFF)).astype(np.int64)).astype(np.int32)
    sqd = (out >> np.uint64(32)).astype(np.uint32).view(F)
    return idx, sqd, out


def _point_at(q, target, direction, rng):
    """A map point p near q + sqrt(target) * direction whose fp32 distance to q is exactly `target`: search the neighbouring floats of
    every coordinate."""
    q = np.asarray(q, F)
    c0 = (q.astype(np.float64) + np.sqrt(float(target)) * np.asarray(direction, np.float64)).astype(F)
    axes = []
    for k in range(3):
        vals = [c0[k]]
        u = c0[k]; v = c0[k]
        for _ in range(24):
            u = np.nextafter(u, F(np.inf)); v = np.nextafter(v, F(-np.inf))
            vals += [u, v]
        axes.append(np.array(vals, F))
    X, Y, Z = np.meshgrid(*axes, indexing="ij")
    cand = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1)
    hit = np.nonzero(fp32_sqdist(q, cand) == F(target))[0]
    if len(hit) == 0:
        return None
    return cand[hit[rng.integers(len(hit))]]


def adversarial_world(seed=0):
    """A map (m x 4, w = 1) and queries (n x 4) where the search goes wrong if anything is off by one.  Returns (map, queries, notes):
    notes names index ranges of the queries and the points that sit exactly on the gate."""
    rng = np.random.default_rng(seed)
    tau0 = gate_tau(1.0)
    parts, queries, notes = [], [], {}

    def add_q(name, q):
        q = np.asarray(q, F).reshape(-1, 3)
        s = sum(len(x) for x in queries)
        queries.append(q)
        notes[name] = (s, s + len(q))

    # a dense region on the integer lattice of 1 m cells: random points, some of them rounded onto cell corners and faces
    lo = np.array([20.0, -8.0, 1.0])
    ext = np.array([10.0, 8.0, 4.0])
    base = (lo + rng.uniform(0, 1, (int(4.0 * ext.prod()), 3)) * ext).astype(F)
    base[: len(base) // 8] = np.round(base[: len(base) // 8])
    base[len(base) // 8: len(base) // 6, :2] = np.round(base[len(base) // 8: len(base) // 6, :2])
    parts.append(base)
    add_q("dense", (lo + rng.uniform(0, 1, (400, 3)) * ext).astype(F))
    add_q("corners", np.round(lo + rng.uniform(0, 1, (60, 3)) * ext).astype(F))
    # one point seven times: the fifth slot is an index tie among equal distances
    dup = np.array([23.3, -4.6, 2.7], F)
    parts.append(np.repeat(dup[None], 7, 0))
    add_q("duplicates", np.concatenate([dup[None], dup + rng.uniform(-0.2, 0.2, (20, 3)).astype(F)]))
    # an equidistant lattice (0.25 m) with queries at the centres of its cubes
    lat = np.stack(np.meshgrid(np.arange(-2, 3), np.arange(-2, 3), np.arange(-1, 2), indexing="ij"), -1).reshape(-1, 3) * 0.25
    lat_o = np.array([26.0, -3.0, 3.0])
    parts.append((lat + lat_o).astype(F))
    add_q("lattice", (lat[:40] + lat_o + 0.125).astype(F))
    # a clump of 80 points in one cell: a three-cell run far longer than a staging tile, several register batches per lane
    clump_c = np.array([28.0, -6.0, 2.0])
    parts.append((clump_c + rng.uniform(0.05, 0.95, (80, 3))).astype(F))
    add_q("clump", (clump_c + rng.uniform(-0.3, 1.3, (40, 3))).astype(F))
    # a sparse region: queries 4 m apart with 0 .. 4 neighbours at 0.3 - 0.9 m, and queries whose fifth candidate sits exactly on the
    # gate (d == tau0: inside) or one float beyond it (d == 1.0f: outside)
    gate_pts = []
    sq = []
    k = 0
    for nn in range(5):
        for rep in range(4):
            q = np.array([40.0 + 4.0 * k + 0.37, -6.0 + 4.0 * (rep % 2) + 0.21, 2.0 + 2.0 * (rep // 2) + 0.43], F)
            k += 1
            dirs = rng.normal(size=(nn, 3)); dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
            parts.append((q + dirs * rng.uniform(0.3, 0.9, (nn, 1))).astype(F))
            sq.append(q)
    sparse_q = np.array(sq, F)
    for j, (nn, targets) in enumerate([(4, (tau0,)), (4, (F(1.0),)), (4, (tau0, F(1.0))), (3, (tau0, F(1.0))), (4, (tau0, tau0)),
                                        (2, (tau0,)), (5, (tau0,)), (4, (np.nextafter(tau0, F(0)), F(1.0)))]):
        q = np.array([40.0 + 4.0 * (k + j) + 0.61, 6.0 + 0.17 * j, 3.0 + 0.29], F)
        dirs = rng.normal(size=(nn, 3)); dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
        parts.append((q + dirs * rng.uniform(0.3, 0.9, (nn, 1))).astype(F))
        for t in targets:
            p = None
            while p is None:                 # a direction along one axis leaves few distinct sums: try another
                d = rng.normal(size=3); d /= np.linalg.norm(d)
                p = _point_at(q, t, d, rng)
            assert fp32_sqdist(q, p) == t
            gate_pts.append(p)
        sparse_q = np.concatenate([sparse_q, q[None]])
    parts.append(np.array(gate_pts, F))
    add_q("sparse", sparse_q)
    pts = np.concatenate(parts).astype(F)
    # outside the grid box on all six sides: just beyond each face (neighbours across it) and far away
    bmin, bmax = pts.min(0), pts.max(0)
    outs = []
    for ax in range(3):
        for side, b in ((-1, bmin), (1, bmax)):
            for off in (0.3, 0.9, 50.0, 4000.0):
                q = pts[rng.integers(len(pts))].copy()
                q[ax] = b[ax] + side * off
                outs.append(q)
    add_q("outside", np.array(outs, F))
    m = np.ones((len(pts), 4), F)
    m[:, :3] = pts
    qs = np.ones((sum(len(x) for x in queries), 4), F)
    qs[:, :3] = np.concatenate(queries)
    notes["tau0"] = tau0
    return m, qs, notes
