"""TEST INFRASTRUCTURE: adversarial partitions of the sharded map (knn_core.cuh owner_of / shard_keep, map.cu's shard filters).

A sharded context answers a query only on the rank that owns the cube its transformed position falls in, from that rank's shard
of the map: the points whose +-halo box touches a cube the rank owns.  With a halo of at least the search radius every neighbour
of an owned query is local, so the shard's 5-NN equals the whole map's.  That claim is about fp32 floors at cube faces and fp32
squared distances at the gate, so every world here is built at the faces of one corner where cubes meet:

* queries exactly on an x, y or z face (z faces lie at 16k - 8 for 16 m cubes: the cubes are shifted by half an edge in z) and
  one fp32 ulp either side, and 27 queries at the corner where eight cubes meet;
* per face query, four neighbours on its own side and a fifth across the face whose fp32 squared distance
  ((dx*dx) + dy*dy) + dz*dz is the largest float below 1.0 (the gate accepts it: "tight in") or exactly 1.0 (rejected: "tight
  out"), tuned along an axis where the coordinate is small enough to reach those values; or two neighbours at one exact
  distance on either side of the face ("tie"), so the index tie-break must agree between the shard and the whole map;
* the same at |x|, |y| ~ 1e4 and 1e5 m, where an fp32 ulp is a millimetre or more, and at negative coordinates;
* for map maintenance, frames whose points lie at the push halo (search radius + one voxel diagonal + 0.05, in fp32 as map.cu
  sums it) from a face and one ulp inside and outside it, with 0.4 m voxels straddling that boundary.

The pose of every search is the identity, so a query's transformed position is the query itself, bit for bit."""
from __future__ import annotations

import numpy as np

from knn_reference import fp32_sqdist, gate_tau

F = np.float32
BLOCKS = (8, 16, 64, 256)
RANKS = (2, 3, 4, 8)
BASES = ((0.0, 0.0), (1e4, 1e4), (-1e4, 1e5), (1e5, -1e5), (-1e5, -1e4))
TAU0 = gate_tau(1.0)                       # largest float below the gate 1.0
GATE_HALO = 1.0                            # gate_cell(1.0): the halo of the installed / filtered map
LEAF = F(0.4)
PUSH_HALO = F(F(F(1.0) + F(F(1.7320508) * LEAF)) + F(0.05))     # map.cu's frame halo, summed in fp32 as the device sums it


def corner(block, base):
    """(X, Y, Z): x and y faces nearest the base, the z face below z = 0 (cubes shifted by half an edge in z)"""
    return np.array([round(base[0] / block) * block, round(base[1] / block) * block, -block / 2], F)


def ulp_step(v, s):
    v = F(v)
    return v if s == 0 else np.nextafter(v, F(np.inf) if s > 0 else F(-np.inf))


def _tune(q, p, f, kind, span=96):
    """p with p[f] moved (by up to `span` ulps from the exact solution) so that the fp32 squared distance to q is the largest
    float below 1.0 (kind "in") or the smallest float >= 1.0 ("out"); the other coordinates of p are kept"""
    p = np.array(p, F)
    d_other = float(np.sum((q.astype(np.float64) - p.astype(np.float64)) ** 2) - (float(q[f]) - float(p[f])) ** 2)
    sgn = 1.0 if p[f] >= q[f] else -1.0
    p[f] = F(float(q[f]) + sgn * np.sqrt(max(0.0, 1.0 - d_other)))
    cand = np.repeat(p[None], 2 * span + 1, 0)
    v = p[f]
    lo = [v]
    for _ in range(span):
        lo.append(np.nextafter(lo[-1], F(-np.inf)))
    hi = [v]
    for _ in range(span):
        hi.append(np.nextafter(hi[-1], F(np.inf)))
    cand[:, f] = np.array(lo[::-1] + hi[1:], F)
    d = fp32_sqdist(q[None], cand)
    ok = d <= TAU0 if kind == "in" else d >= F(1.0)
    j = np.flatnonzero(ok)
    j = j[np.argmax(d[j])] if kind == "in" else j[np.argmin(d[j])]
    return cand[j], d[j]


def _equidistant(q, pa, a, v, span=16):
    """pa moved to p[a] near v (within `span` ulps) at exactly pa's fp32 squared distance from q"""
    want = fp32_sqdist(q, pa)
    for k in range(span + 1):
        for sgn in (1, -1):
            c = np.array(pa, F)
            c[a] = v
            for _ in range(k):
                c[a] = np.nextafter(c[a], F(np.inf) if sgn > 0 else F(-np.inf))
            if fp32_sqdist(q, c) == want:
                return c
    raise AssertionError("no equidistant point")


def world(block, base, seed=0):
    """dict(map = float32 [M, 4] (w = 1), queries = float32 [Q, 4], kind = per query "in" / "out" / "tie" / "corner",
    d5 = per query the fp32 squared distance of the tuned neighbour across the face (nan: none), across = index of that
    neighbour in map (-1: none), corner)"""
    rng = np.random.default_rng(seed)
    C = corner(block, base)
    pts, qs, kinds, d5s, across = [], [], [], [], []
    offs = [o for o in (2.5, 5.0, 7.5, 10.0) if o <= block - 1.5]     # 2.5 m apart, and clear of the corner's cloud
    offs = [s * o for o in offs for s in (1, -1)]
    for a in range(3):
        f = 2 if a < 2 else 0                     # the tuning axis: z near 0 for x / y faces, x for z faces
        t = 3 - a - f                             # the plane of a query's neighbours: p[t] = q[t]
        slots = [(o, z) for o in offs for z in (0.3125, -1.6875, 2.3125)] if a < 2 else [(o1, o2) for o1 in offs for o2 in offs]
        assert len(slots) >= 9
        rng.shuffle(slots)
        k = 0
        for s in (-1, 0, 1):
            for kind in ("in", "out", "tie"):
                o1, o2 = slots[k % len(slots)]; k += 1
                q = C.copy()
                q[a] = ulp_step(C[a], s)
                if a < 2:
                    q[1 - a] = F(C[1 - a] + o1); q[2] = F(o2)
                else:
                    q[0] = F(C[0] + o1); q[1] = F(C[1] + o2)
                side = 1.0 if q[a] >= C[a] else -1.0          # q's own side of the face (a point on the face owns the cube above)
                ea = np.zeros(3); ea[a] = 1.0
                ef = np.zeros(3); ef[f] = 1.0
                near = [0.2 * side * ea, 0.3 * ef, -0.35 * ef, 0.25 * side * ea + 0.2 * ef]
                mine = [np.array(q + v, F) for v in near]
                for m in mine:
                    m[t] = q[t]
                if kind == "tie":
                    # two neighbours at one exact distance, one on each side of the face: the fifth and sixth by (distance, index)
                    pa = np.array(q, F); pa[a] = F(float(q[a]) - side * 0.75)
                    pb = _equidistant(q, pa, a, F(float(q[a]) + side * 0.75))
                    pair = [pa, pb] if rng.integers(0, 2) else [pb, pa]
                    across.append(len(pts) + 4 + (0 if pair[0] is pa else 1))
                    d5s.append(float(fp32_sqdist(q, pa)))
                    block_pts = mine + pair
                else:
                    p0 = np.array(q + (-side * 0.6) * ea + 0.8 * ef, F)
                    p0[t] = q[t]
                    p5, d5 = _tune(q, p0, f, kind)
                    across.append(len(pts) + 4)
                    d5s.append(float(d5))
                    block_pts = mine + [p5]
                order = rng.permutation(len(block_pts))            # the across-face neighbour at varying ranks of the map order
                inv = np.argsort(order)
                across[-1] = len(pts) + int(inv[across[-1] - len(pts)])
                pts.extend(block_pts[i] for i in order)
                qs.append(q); kinds.append(kind)
    # the corner: 27 queries within one ulp of the point where eight cubes meet, over a cloud around it
    cloud = C + rng.uniform(-0.9, 0.9, (60, 3))
    pts.extend(np.array(p, F) for p in cloud)
    for sx in (-1, 0, 1):
        for sy in (-1, 0, 1):
            for sz in (-1, 0, 1):
                qs.append(np.array([ulp_step(C[0], sx), ulp_step(C[1], sy), ulp_step(C[2], sz)], F))
                kinds.append("corner"); d5s.append(np.nan); across.append(-1)
    m = np.ones((len(pts), 4), F); m[:, :3] = np.array(pts, F)
    qq = np.ones((len(qs), 4), F); qq[:, :3] = np.array(qs, F)
    return dict(map=m, queries=qq, kind=np.array(kinds), d5=np.array(d5s), across=np.array(across), corner=C)


def worlds():
    """every (block, base) world, named"""
    return [(f"b{b}_{'n' if bx < 0 else 'p'}{abs(int(bx))}_{'n' if by < 0 else 'p'}{abs(int(by))}", b, (bx, by))
            for b in BLOCKS for bx, by in BASES]


def halo_frame(block, base, seed=0):
    """[K, 3] float32 points of one map frame (world frame: pushed at the identity pose) at the push halo of the faces of the
    corner: p[a] = face -+ PUSH_HALO and one ulp either side, each with partners 0.1 - 0.3 m further in and out, so 0.4 m voxels
    straddle the boundary where the frame's shard filter cuts"""
    rng = np.random.default_rng(seed)
    C = corner(block, base)
    out = []
    for a in range(3):
        for sign in (-1.0, 1.0):
            edge = F(C[a] + F(sign) * PUSH_HALO)
            for s in (-1, 0, 1):
                for _ in range(4):
                    p = C + rng.uniform(-3.0, 3.0, 3)
                    if a < 2:
                        p[2] = rng.uniform(-2.0, 2.0)
                    p = np.array(p, F)
                    p[a] = ulp_step(edge, s)
                    out.append(p.copy())
                    for dd in (0.1, -0.1, 0.3, -0.3):
                        r = p.copy(); r[a] = F(float(p[a]) + dd)
                        out.append(r)
    out.extend(np.array(C + rng.uniform(-2.5, 2.5, (80, 3)), F))
    return np.array(out, F)
