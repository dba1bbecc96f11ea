"""TEST INFRASTRUCTURE: adversarial keyframe maps for the backend's correspondence searches (liliom_b200/csrc/backend_corr.cu).

backend_world(name) returns an edge layer, a surf layer (PT48, the reflectivity in `curvature`), body-frame edge and surf queries
(PT48, the query reflectivity in `curvature`), the lidar pose that takes them into the map, and `notes`: case name -> the
indices of its queries, per kind.  Every case sits at its own site, 4 m from every other, so its 5-NN set is exactly the points built for
it.  A site is chosen in the body frame and sent through the oracle's transform first; the map points are then placed around the
transformed query, so that its fp32 distances, collinearities and symmetries are exact where a case needs them.  Cases on a
threshold that no closed form reaches (variant 1's line distance, the plane and weight gates) are found by bisecting one float
with the oracle deciding, so each of them sits one ulp from the other side.

Worlds: "near" (a 180-degree yaw and a dyadic translation: q * p + t is exact, so a query on a line stays on it in fp64 as well)
and "far" (an oblique rotation, a translation of hundreds of metres)."""
import numpy as np

import knn_reference as KR
import oracle_lib as O
from liliom_b200._lib import PT48

F = np.float32
# the thresholds every case is built against: the backend defaults of both variants (liliom_backend_default_params)
SURF_DIST_THRES = 0.12
W_GATE = {0: 0.2, 1: 0.3}
LIDAR_CONST = {0: 20.0, 1: 7.5}
REFLECT_THRES = 2.0          # a dyadic value the reflectivity sums below hit exactly (the default 15.0 is not special)
KD_RADII = (1.0, 0.49)       # the default surf gate and a non-default one (0.49 <= the 1 m cell^2 of the map grid)
WORLDS = ("near", "far")

POSES = {
    "near": np.array([0.0, 0.0, 0.0, 1.0, 3.25, -1.5, 0.75]),
    "far": None,
}


def _far_pose():
    ax = np.array([0.3, -0.5, 0.8]); ax /= np.linalg.norm(ax)
    h = np.deg2rad(37.0) / 2
    return np.concatenate([[np.cos(h)], np.sin(h) * ax, [612.3, -437.9, 28.4]])


def pose_of(world):
    return POSES[world] if world == "near" else _far_pose()


def _pt48(xyz, refl=0.0):
    a = np.zeros(len(xyz), PT48)
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    a["x"], a["y"], a["z"], a["w"] = xyz[:, 0], xyz[:, 1], xyz[:, 2], 1.0
    a["curvature"] = refl
    return a


def world_of(pose, f):
    """the fp32 map-frame point the searches transform body point f to (the oracle's xform)"""
    return np.array([tuple(p)[:3] for p in O.transform_cloud(_pt48([f]), pose)], F)[0]


def f4(pts):
    out = np.ones((len(pts), 4), F)
    out[:, 0], out[:, 1], out[:, 2] = pts["x"], pts["y"], pts["z"]
    return out


# five distinct integer offsets (x_i, y_i) with sum x = sum y = sum xy = 0 and sum x^2 = 30 = 3 sum y^2: centred at the query,
# their scatter is diag(30, 10, 0) h^2 in the (e1, e2) frame, so ev2 = 3 ev1 in exact arithmetic
P31_X = np.array([3.0, 3.0, -2.0, -2.0, -2.0])
P31_Y = np.array([2.0, -2.0, 1.0, -1.0, 0.0])


class _Builder:
    def __init__(self, world, kind, seed):
        self.pose = pose_of(world)
        self.rng = np.random.default_rng(seed)
        self.kind = kind
        self.map, self.refl, self.q, self.qrefl, self.notes = [], [], [], [], {}
        self.site = 0
        self.near = world == "near"
        self.off = np.array([-40.0, -12.0, -6.0])

    def next_site(self):
        k = self.site
        self.site += 1
        f = self.off + np.array([4.0 * (k % 20), 4.0 * ((k // 20) % 6), 4.0 * (k // 120)]) + self.rng.uniform(0.1, 0.3, 3)
        f = f.astype(F)
        return f, world_of(self.pose, f)

    def add(self, name, fs, pts, qrefl=10.0, refl=None):
        fs = np.asarray(fs, F).reshape(-1, 3)
        pts = np.asarray(pts, F).reshape(-1, 3)
        if refl is None:       # distinct reflectivity differences: finite weights, a sum below REFLECT_THRES
            refl = np.float32(qrefl) + np.arange(1, len(pts) + 1, dtype=F) * F(0.125)
        s = sum(len(x) for x in self.q)
        self.notes.setdefault(name, []).extend(range(s, s + len(fs)))
        self.q.append(fs)
        self.qrefl.append(np.broadcast_to(np.asarray(qrefl, F), (len(fs),)).copy())
        self.map.append(pts)
        self.refl.append(np.asarray(refl, F).reshape(-1))

    def done(self):
        m = _pt48(np.concatenate(self.map), 0.0)
        m["curvature"] = np.concatenate(self.refl)
        q = _pt48(np.concatenate(self.q))
        q["curvature"] = np.concatenate(self.qrefl)
        return m, q, {k: np.array(v) for k, v in self.notes.items()}


def _perp(u, rng):
    v = np.cross(u, rng.normal(size=3))
    return v / np.linalg.norm(v)


def _unit(rng):
    u = rng.normal(size=3)
    return u / np.linalg.norm(u)


def _dyadic(v, bits=10):
    return np.round(np.asarray(v, np.float64) * (1 << bits)) / (1 << bits)


def _bisect(decide, lo, hi, make):
    """decide(make(t)) differs at t = lo and t = hi: shrink [lo, hi] until make(lo) and make(hi) are neighbouring floats (or equal
    bits on all but one float step).  Returns (make(lo), make(hi))."""
    dlo = decide(make(lo))
    assert dlo != decide(make(hi))
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        a, b, m = make(lo), make(hi), make(mid)
        if m.tobytes() in (a.tobytes(), b.tobytes()):
            break
        if decide(m) == dlo:
            lo = mid
        else:
            hi = mid
    return make(lo), make(hi)


def _oracle_edge(pts, f, pose, variant):
    tree = O.KdTree(np.concatenate([np.asarray(pts, F), np.ones((len(pts), 1), F)], 1))
    v, _, _ = O.correspond_edge(tree, _pt48([f]), pose, variant)
    return int(v[0])


def _oracle_surf(pts, refl, f, qrefl, pose, variant, kd=1.0):
    m = np.concatenate([np.asarray(pts, F), np.ones((len(pts), 1), F)], 1)
    tree = O.KdTree(m)
    extra = dict(map_refl=np.asarray(refl, F), feat_refl=np.array([qrefl], F), reflect_thres=REFLECT_THRES) if variant == 0 else {}
    v, _, _ = O.correspond_surf_backend(tree, _pt48([f]), pose, kd, SURF_DIST_THRES, W_GATE[variant], LIDAR_CONST[variant], **extra)
    return int(v[0])


def _line(s, u, ts, rng, noise=0.0):
    return np.array([s + t * u + (rng.normal(size=3) * noise if noise else 0) for t in ts], np.float64).astype(F)


def _edge_cases(B):
    rng = B.rng
    tau = KR.gate_tau(1.0)
    one = F(1.0)
    inner = (-0.45, -0.2, 0.15, 0.4)

    def gate(name, targets, n_in=4):
        f, s = B.next_site()
        u = _unit(rng)
        pts = list(_line(s, u, inner[:n_in], rng, 1e-3))
        for t in targets:
            p = None
            while p is None:
                d = u + 0.05 * _unit(rng)
                p = KR._point_at(s, t, d / np.linalg.norm(d), rng)
            pts.append(p)
        B.add(name, [f], pts)

    for _ in range(2):
        gate("gate_tau0", (tau,))             # fifth at d == tau0: inside
        gate("gate_one", (one,))              # fifth at d == 1.0f: outside
        gate("gate_tau0_one", (tau, one))
        gate("gate_tie", (tau, tau))          # two fifth candidates at the same distance: the index decides
        gate("gate_three", (one, one), 3)     # fewer than five inside
        gate("gate_below", (np.nextafter(tau, F(0)), one))
    # seven copies of one point: all eigenvalues 0 (rejected), the fifth slot an index tie
    for _ in range(2):
        f, s = B.next_site()
        B.add("duplicates", [f], np.repeat((s + F(0.2) * _unit(rng).astype(F))[None], 7, 0))
    # exactly collinear: along an axis through the query (the query on the line: zero cross product) and along a diagonal
    for ax in range(3):
        f, s = B.next_site()
        d = np.zeros(3); d[ax] = 0.125
        B.add("collinear_axis", [f], np.array([s + k * d for k in (-2, -1, 0, 1, 2)], np.float64).astype(F))
    for sgn in ((1, 1, 1), (1, -1, 1), (-1, 1, 1)):
        f, s = B.next_site()
        d = np.array(sgn, np.float64) * 0.125
        base = s + np.array([0.25, -0.125, 0.0625])
        B.add("collinear_diag", [f], np.array([base + k * d for k in (-2, -1, 0, 1, 2)], np.float64).astype(F))
    # the 3:1 boundary: an integer pattern with ev2 = 3 ev1 exactly, on axis pairs and on diagonal pairs, then ratio sweeps
    x, y = P31_X, P31_Y
    frames = [(np.array([1.0, 0, 0]), np.array([0, 1.0, 0])), (np.array([0, 0, 1.0]), np.array([1.0, 0, 0])),
              (np.array([1.0, 1.0, 0]), np.array([1.0, -1.0, 0])), (np.array([0, 1.0, 1.0]), np.array([0, 1.0, -1.0]))]
    h = 0.0625
    for e1, e2 in frames:
        for k in (0, -8, -4, -2, -1, 1, 2, 4, 8):
            f, s = B.next_site()
            sc = 1.0 + k * 2.0 ** -14
            pts = np.array([s + h * (xi * e1 + sc * yi * e2) for xi, yi in zip(x, y)], np.float64).astype(F)
            B.add("ratio3" if k == 0 else "ratio3_sweep", [f], pts)
    # sets symmetric about the query: the eigenvector's sign is decided by rounding alone
    for j in range(8):
        f, s = B.next_site()
        u = _unit(rng); v = _perp(u, rng)
        d1 = _dyadic(0.35 * u); d2 = _dyadic((0.04 if j % 2 == 0 else 0.3) * v)
        B.add("symmetric", [f], np.array([s + d1, s - d1, s + d2, s - d2, s], np.float64).astype(F))
    # variant 1's distance: a line 0.1 m from the query, the query moved along the normal until dist < 0.1 flips
    Rt = _rot(B.pose).T
    for j in range(4):
        f, s = B.next_site()
        u = _unit(rng); n = _perp(u, rng)
        pts = _line(s - 0.1 * n, u, (-0.3, -0.15, 0.0, 0.15, 0.3), rng)
        dirb = Rt @ n

        def make(t, f=f, dirb=dirb):
            return (f.astype(np.float64) + t * dirb).astype(F)
        a, b = _bisect(lambda g, pts=pts: _oracle_edge(pts, g, B.pose, 1), -0.02, 0.02, make)
        B.add("var1_dist", [a, b, make(-0.02), make(0.02)], pts)


def _rot(pose):
    w, x, y, z = pose[:4]
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _plane_pts(s, n, rng, r=0.4, k=5, noise=0.0):
    u = _perp(n, rng); v = np.cross(n, u)
    ang = np.linspace(0, 2 * np.pi, k, endpoint=False) + rng.uniform(0, 1)
    rad = r * np.linspace(0.5, 1.0, k)
    return np.array([s + a * np.cos(t) * u + a * np.sin(t) * v + n * (rng.normal() * noise) for a, t in zip(rad, ang)],
                    np.float64).astype(F)


# four fp32 reflectivity differences whose sum is 2 - 2^-50 exactly; a fifth of 2^-50, 1.5 2^-50 or 0.75 2^-50 makes the sum
# REFLECT_THRES = 2, one double ulp above it or one below it.  Every partial sum is a multiple of 2^-52 below 2 (exact in any order).
_SUM4 = [1.0, 1.0 - 2.0 ** -24, 2.0 ** -24 - 2.0 ** -47, 2.0 ** -47 - 2.0 ** -50]
assert all(float(np.float32(v)) == v for v in _SUM4 + [2.0 ** -50, 1.5 * 2.0 ** -50, 0.75 * 2.0 ** -50])


def _surf_cases(B):
    rng = B.rng
    # the squared-distance gate at kd = 1.0 and 0.49: four points in a plane through the query, the fifth on the gate
    for kd in KD_RADII:
        tau = KR.gate_tau(kd)
        for name, t in (("gate_tau0", tau), ("gate_above", np.nextafter(tau, F(np.inf)))):
            for _ in range(2):
                f, s = B.next_site()
                n = _unit(rng)
                pts = list(_plane_pts(s, n, rng, r=0.3, k=4))
                p = None
                while p is None:
                    p = KR._point_at(s, t, _perp(n, rng), rng)
                B.add(f"{name}_{kd}", [f], pts + [p])
    # exactly coplanar: axis planes and a dyadic tilted plane; collinear neighbours (rank-deficient QR)
    for ax in range(3):
        f, s = B.next_site()
        e = [np.eye(3)[(ax + 1) % 3], np.eye(3)[(ax + 2) % 3]]
        offs = ((0, 0), (0.25, 0), (0, 0.25), (-0.25, 0.125), (0.125, -0.25))
        B.add("coplanar_axis", [f, (f + F(0.03)).astype(F)], np.array([s + a * e[0] + b * e[1] for a, b in offs], np.float64).astype(F))
    for _ in range(2):
        f, s = B.next_site()
        e1, e2 = np.array([0.25, 0.0, 0.125]), np.array([0.0, 0.25, -0.0625])
        offs = ((0, 0), (1, 0), (0, 1), (-1, 0.5), (0.5, -1))
        B.add("coplanar_tilted", [f], np.array([s + a * e1 + b * e2 for a, b in offs], np.float64).astype(F))
    for ax in range(3):
        f, s = B.next_site()
        d = np.zeros(3); d[ax] = 0.125
        B.add("collinear", [f], np.array([s + k * d for k in (-2, -1, 0, 1, 2)], np.float64).astype(F))
    # neighbours on planes through the origin (z = 0 and x = y): A n = -1 has no exact solution
    for plane in ("z0", "xy"):
        f, s = B.next_site()
        tgt = s.astype(np.float64).copy()
        if plane == "z0":
            tgt[2] = 0.0
        else:
            tgt[0] = tgt[1] = 0.5 * (tgt[0] + tgt[1])
        # move the query onto (near) that plane through the body frame, then put the neighbours on it exactly
        f = (f.astype(np.float64) + _rot(B.pose).T @ (tgt - s)).astype(F)
        s = world_of(B.pose, f)
        offs = ((0, 0), (0.25, 0), (0, 0.25), (-0.25, 0.125), (0.125, -0.25))
        if plane == "z0":
            pts = [(s[0] + a, s[1] + b, 0.0) for a, b in offs]
        else:
            pts = [(s[0] + a, s[0] + a, s[2] + b) for a, b in offs]
        B.add("origin_plane", [f], np.array(pts, np.float64).astype(F))
    # the plane gate: one neighbour's offset from the plane bisected until max distance > surf_dist_thres flips
    for variant in (1, 0):
        for keep in (0, 1):
            for _ in range(2):
                f, s = B.next_site()
                n = _unit(rng)
                base = _plane_pts(s, n, rng, r=0.35, k=5)
                refl = F(10.0) + np.arange(1, 6, dtype=F) * F(0.125)

                def make(t, base=base, n=n):        # the innermost point: a tilt of the plane cannot absorb its offset
                    p = base.copy(); p[0] = (base[0].astype(np.float64) + t * n).astype(F)
                    return p
                a, b = _bisect(lambda p, f=f, refl=refl, variant=variant: _oracle_surf(p, refl, f, 10.0, B.pose, variant),
                               0.0, 0.3, make)
                B.add(f"plane_thres_v{variant}", [f], a if keep == 0 else b, refl=refl)
    # the weight gate, 1 - 0.9 |pd| / |s|^(1/2) > w_gate: with |pd| below the 1 m search gate it can only fail within ~0.1 m of
    # the map origin, so the near world has one site there; the query moves along the plane normal (away from every other
    # site) until the gate flips, for each variant's w_gate
    if B.near:
        R = _rot(B.pose)
        s0 = np.array([0.0625, -0.03125, 0.09375])
        f = (R.T @ (s0 - B.pose[4:])).astype(F)
        s = world_of(B.pose, f)
        n = np.array([0.6, 0.64, 0.48])
        pts = _plane_pts(s, n, rng, r=0.25, k=5)
        refl = F(10.0) + np.arange(1, 6, dtype=F) * F(0.125)
        dirb = R.T @ n
        qs = []
        for variant in (1, 0):
            def make(t, f=f, dirb=dirb):
                return (f.astype(np.float64) + t * dirb).astype(F)
            a, b = _bisect(lambda g, variant=variant: _oracle_surf(pts, refl, g, 10.0, B.pose, variant), 0.0, 0.9, make)
            qs += [a, b]
        B.add("w_gate", qs, pts, refl=refl)
    # reflectivity (variant 0): ties with one and with all five neighbours (infinite weights, a zero sum), sums on REFLECT_THRES
    # and one double ulp either side, NaN on the query and on a map point
    for name, qr, rf in (("refl_tie_one", 12.0, [12.0, 12.125, 12.25, 12.375, 12.5]), ("refl_tie_all", 12.0, [12.0] * 5),
                         ("refl_sum_eq", 0.0, _SUM4 + [2.0 ** -50]),
                         ("refl_sum_above", 0.0, _SUM4 + [1.5 * 2.0 ** -50]),
                         ("refl_sum_below", 0.0, _SUM4 + [0.75 * 2.0 ** -50]),
                         ("refl_nan_query", np.nan, [10.125, 10.25, 10.375, 10.5, 10.625]),
                         ("refl_nan_map", 10.0, [10.125, np.nan, 10.375, 10.5, 10.625])):
        for _ in range(2):
            f, s = B.next_site()
            n = _unit(rng)
            B.add(name, [f], _plane_pts(s, n, rng, r=0.35, k=5), qrefl=qr, refl=np.array(rf, F))
    # ordinary noisy planes, accepted and refused by the plane gate
    for _ in range(6):
        f, s = B.next_site()
        B.add("noisy_plane", [f], _plane_pts(s, _unit(rng), rng, r=0.4, k=6, noise=0.03))


_CACHE = {}


def backend_world(world="far", seed=0):
    """dict(pose, edge_map (m x 4 f32), edge_map48 and surf_map (PT48), edge_q, surf_q (PT48 body frame), edge_notes, surf_notes)"""
    key = (world, seed)
    if key not in _CACHE:
        be = _Builder(world, "edge", seed)
        _edge_cases(be)
        em, eq, en = be.done()
        bs = _Builder(world, "surf", seed + 1)
        _surf_cases(bs)
        sm, sq, sn = bs.done()
        _CACHE[key] = dict(pose=pose_of(world), edge_map=f4(em), edge_map48=em, surf_map=sm, edge_q=eq, surf_q=sq,
                           edge_notes=en, surf_notes=sn)
    return _CACHE[key]
