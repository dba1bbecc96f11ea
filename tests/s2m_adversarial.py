"""TEST INFRASTRUCTURE: adversarial worlds for the plane stage of the scan-to-map search (phase B of grid_knn.cu:
dev_math.cuh::plane_fit_gate).

s2m_world(name) returns the map (m x 4 fp32, installed with liliom_map_set_points), the body-frame queries (n x 4 fp32), the pose
that takes them into the map, `notes` (case name -> query indices) and `sets` (query -> the map indices built as its neighbours).
Every case sits at its own site, 4 m from every other, so its 5-NN set is exactly the points built for it.  A site is chosen in
the body frame and sent through the oracle's transform; the neighbours are placed around the transformed query.  The plane and
weight gates are reached by bisecting one float with the oracle deciding, so each pair sits one step either side of its gate.

Worlds: "near" (a 180-degree yaw and a dyadic translation: the transform is exact) and "far" (an oblique rotation, a translation
of hundreds of metres), the poses of tests/bk_adversarial.py."""
import numpy as np

import bk_adversarial as BK
import oracle_lib as O

F = np.float32
WORLDS = ("near", "far")
# the degenerate sets: the fast fit declines them, so the exact path (the oracle's QR) decides them and their planes must be the
# oracle's bits.  (A gate pair's sides are one fp32 step of one neighbour apart, which can leave a case outside the guard band; the
# tests compare plane bits on every case the host build of plane_fit_gate sends to the exact path.)
EXACT = ("coincident", "two_points", "collinear_axis", "collinear_oblique", "lattice_axis", "lattice_tilted", "origin_plane",
         "plane_1e-2", "plane_1e-4")


def _oracle_valid(pts, f, pose):
    m = np.ones((len(pts), 4), F); m[:, :3] = pts
    _, v, _, _, _ = O.find_surf_corr(O.KdTree(m), np.array([[f[0], f[1], f[2], 1.0]], F), pose)
    return int(v[0])


class _Builder:
    def __init__(self, world, seed):
        self.pose = BK.pose_of(world)
        self.rng = np.random.default_rng(seed)
        self.map, self.q, self.sets, self.notes = [], [], [], {}
        self.site = 0
        self.nmap = 0

    def next_site(self):
        k = self.site
        self.site += 1
        f = np.array([-40.0, -12.0, -6.0]) + np.array([4.0 * (k % 20), 4.0 * ((k // 20) % 6), 4.0 * (k // 120)])
        f = (f + self.rng.uniform(0.1, 0.3, 3)).astype(F)
        return f, BK.world_of(self.pose, f)

    def add(self, name, fs, pts):
        fs = np.asarray(fs, F).reshape(-1, 3)
        pts = np.asarray(pts, F).reshape(-1, 3)
        s = len(self.q)
        self.notes.setdefault(name, []).extend(range(s, s + len(fs)))
        ids = np.arange(self.nmap, self.nmap + len(pts))
        self.nmap += len(pts)
        self.map.append(pts)
        for f in fs:
            self.q.append(f)
            self.sets.append(ids)

    def done(self):
        m = np.ones((self.nmap, 4), F); m[:, :3] = np.concatenate(self.map)
        q = np.ones((len(self.q), 4), F); q[:, :3] = np.array(self.q)
        return m, q, {k: np.array(v) for k, v in self.notes.items()}, self.sets


def _axis_lattice(s, ax):
    e = [np.eye(3)[(ax + 1) % 3], np.eye(3)[(ax + 2) % 3]]
    offs = ((0, 0), (0.25, 0), (0, 0.25), (-0.25, 0.125), (0.125, -0.25))
    return np.array([s + a * e[0] + b * e[1] for a, b in offs], np.float64).astype(F)


def _cases(B, near):
    rng = B.rng
    pose = B.pose
    R = BK._rot(pose)
    # the plane gate: the innermost point of a plane moved along the normal until the oracle refuses, bisected to one step
    for k in range(12):
        f, s = B.next_site()
        n = BK._unit(rng)
        base = BK._plane_pts(s, n, rng, r=0.35, k=5)

        def make(t, base=base, n=n):
            p = base.copy(); p[0] = (base[0].astype(np.float64) + t * n).astype(F)
            return p
        a, b = BK._bisect(lambda p, f=f: _oracle_valid(p, f, pose), 0.0, 0.3, make)
        if k % 2 == 0:
            B.add("plane_keep", [f], a)            # one step inside the gate
        else:
            B.add("plane_refuse", [f], b)          # one step outside it
    # degenerate sets the fast fit declines: coincident, two points repeated, collinear (axis and oblique), fp32 lattices
    for _ in range(2):
        f, s = B.next_site()
        B.add("coincident", [f], np.repeat((s + F(0.2) * BK._unit(rng).astype(F))[None], 5, 0))
        f, s = B.next_site()
        p, q = s + F(0.25) * BK._unit(rng).astype(F), s - F(0.125) * BK._unit(rng).astype(F)
        B.add("two_points", [f], np.array([p, p, p, q, q], F))
    for ax in range(3):
        f, s = B.next_site()
        d = np.zeros(3); d[ax] = 0.125
        B.add("collinear_axis", [f], np.array([s + k * d for k in (-2, -1, 0, 1, 2)], np.float64).astype(F))
        f, s = B.next_site()
        B.add("lattice_axis", [f], _axis_lattice(s, ax))
    for sgn in ((1, 1, 1), (1, -1, 0.5)):
        f, s = B.next_site()
        d = np.array(sgn, np.float64) * 0.125
        B.add("collinear_oblique", [f], np.array([s + k * d for k in (-2, -1, 0, 1, 2)], np.float64).astype(F))
        f, s = B.next_site()
        e1, e2 = np.array([0.25, 0.0, 0.125]), np.array([0.0, 0.25, -0.0625])
        offs = ((0, 0), (1, 0), (0, 1), (-1, 0.5), (0.5, -1))
        B.add("lattice_tilted", [f], np.array([s + a * e1 + b * e2 for a, b in offs], np.float64).astype(F))
    # planes z = 0 (through the world origin: A n = -1 has no exact solution), z = 1e-2 and z = 1e-4, the query moved onto them
    for name, z in (("origin_plane", 0.0), ("plane_1e-2", 1e-2), ("plane_1e-4", 1e-4)):
        f, s = B.next_site()
        tgt = s.astype(np.float64).copy(); tgt[2] = z
        f = (f.astype(np.float64) + R.T @ (tgt - s)).astype(F)
        s = BK.world_of(pose, f)
        offs = ((0, 0), (0.25, 0), (0, 0.25), (-0.25, 0.125), (0.125, -0.25))
        B.add(name, [f], np.array([(s[0] + a, s[1] + b, F(z)) for a, b in offs], F))
    # sub-millimetre patches (far out in the far world): scatter pivots near the fast fit's 1e-9 tr decline threshold
    for k in range(4):
        f, s = B.next_site()
        B.add("submm", [f], BK._plane_pts(s, BK._unit(rng), rng, r=5e-4 * (k + 1), k=5, noise=1e-7 * 10 ** k))
    if near:
        # the weight gate near the map origin: the query moves along the plane normal until the oracle refuses; and a query at
        # the world origin itself (rng = 0: w is -inf) on the same neighbours
        s0 = np.array([0.0625, -0.03125, 0.09375])
        f = (R.T @ (s0 - pose[4:])).astype(F)
        s = BK.world_of(pose, f)
        n = np.array([0.6, 0.64, 0.48])
        pts = BK._plane_pts(s, n, rng, r=0.25, k=5)
        dirb = R.T @ n

        def make(t):
            return (f.astype(np.float64) + t * dirb).astype(F)
        a, b = BK._bisect(lambda g: _oracle_valid(pts, g, pose), 0.0, 0.9, make)
        fo = (R.T @ (-pose[4:])).astype(F)
        assert np.array_equal(BK.world_of(pose, fo), np.zeros(3, F))
        B.add("w_keep", [a], pts)
        B.notes.setdefault("w_refuse", []).append(len(B.q)); B.q.append(b); B.sets.append(B.sets[-1])
        B.notes.setdefault("origin_query", []).append(len(B.q)); B.q.append(fo); B.sets.append(B.sets[-1])
    else:
        # a query hundreds of metres out is every far case; one more near a kilometre (inside the dense cell grid's extent)
        f = (np.array([800.0, 500.0, 60.0]) + rng.uniform(0.1, 0.3, 3)).astype(F)
        s = BK.world_of(pose, f)
        B.add("huge_range", [f], BK._plane_pts(s, BK._unit(rng), rng, r=0.4, k=5, noise=0.01))
    # ordinary noisy planes
    for _ in range(8):
        f, s = B.next_site()
        B.add("noisy_plane", [f], BK._plane_pts(s, BK._unit(rng), rng, r=0.4, k=5, noise=0.02))


_CACHE = {}


def s2m_world(world="far", seed=0):
    """dict(pose, map (m x 4 f32), feats (n x 4 f32, body frame), notes, sets)"""
    if world not in _CACHE:
        B = _Builder(world, seed)
        _cases(B, world == "near")
        m, q, notes, sets = B.done()
        _CACHE[world] = dict(pose=BK.pose_of(world), map=m, feats=q, notes=notes, sets=sets)
    return _CACHE[world]
