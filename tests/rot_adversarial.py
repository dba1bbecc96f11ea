"""Adversarial spinning-LiDAR sweeps for the ROT extractor (R/src/Preprocessing.cpp:276-509): seeded, every return placed
directly by (ring, azimuth), each case a named set of input rows or a ring so that a failure names its case.

Layout.  A ring is a sequence of returns at one elevation (the centre of its table bin) and azimuths that decrease with the
sequence, so that -atan2(y, x) grows as the reference's sweep does; the sweep's input order interleaves the rings by azimuth
(column-major, the order a spinning sensor fires in) and keeps each ring's own order.  The default ring content alternates
blocks of three returns at two ranges: every block edge is a break of the suppression (gap > 0.05 m) and a sharp candidate, and
the blocks' inner returns are flat ones.  Special cases are separate rings or single rows:

  * an exact wall: returns on the line x = X, z = 0, y on a 1/32 m grid — every coordinate and every partial sum of the stencil
    exact, so the curvature of an untouched return is exactly 0 and a displaced return sets its neighbours' curvature exactly;
  * the z = 0 plane is elevation 0 for any range: ring 6 of the 64-line table, 8 of the 16-line one; far, huge and exact-line
    rings live there.

A sweep is a dict: pts (PT32), q_imu, q_lb, line_num, ds_rate, cases {name: dict(rows=input rows) or dict(ring=r)}."""
from __future__ import annotations

import math

import numpy as np

import rot_oracle
from oracle_lib import PT32
from rot_restate import F, curvature

ID = (1.0, 0.0, 0.0, 0.0)
A0 = 0.3                                 # azimuth of u = 0: startOri is about -A0
CTR = {16: lambda r: 2.0 * r - 15.0, 32: lambda r: (r + 0.5) * 4.0 / 3.0 - 92.0 / 3.0,
       64: lambda r: 2.0 - r / 3.0 if r <= 32 else -8.83 - (r - 32) / 2.0}


def n_rings(line_num):
    return 51 if line_num == 64 else line_num


def pt(rng_m, az, el_deg):
    el = math.radians(el_deg)
    return (F(rng_m * math.cos(el) * math.cos(az)), F(rng_m * math.cos(el) * math.sin(az)), F(rng_m * math.sin(el)))


def az_of(u):
    return A0 - 2 * math.pi * u


def u_of(x, y):
    """the sequence position of a return by its azimuth"""
    return ((A0 - math.atan2(float(y), float(x))) / (2 * math.pi)) % 1.0


def blocks_ring(line_num, r, n, R, u0=0.0, u1=1.0, block=3, far=1.25):
    """n returns over u in [u0, u1): blocks of `block` returns alternately at R and far * R"""
    out = []
    for k in range(n):
        u = u0 + (u1 - u0) * (k + 0.5) / n
        rr = R * (far if (k // block) % 2 else 1.0)
        out.append((u, pt(rr, az_of(u), CTR[line_num](r))))
    return out


class Sweep:
    def __init__(self, line_num, ds_rate=1, q_imu=ID, q_lb=ID):
        self.line_num, self.ds_rate, self.q_imu, self.q_lb = line_num, ds_rate, q_imu, q_lb
        self.rows = []          # (u, seq, xyz, tag)
        self.cases = {}

    def add(self, seq, tag=None):
        """seq: [(u, xyz)] in ring order; tag: a case name for all of these rows"""
        for u, p in seq:
            self.rows.append((u, len(self.rows), p, tag))

    def ring(self, name, r):
        self.cases[name] = dict(ring=r)

    def build(self):
        order = sorted(range(len(self.rows)), key=lambda i: (self.rows[i][0], self.rows[i][1]))
        pts = np.zeros(len(order), PT32)
        tags = {}
        for k, i in enumerate(order):
            pts[k]["x"], pts[k]["y"], pts[k]["z"] = self.rows[i][2]
            pts[k]["w"] = 1.0
            t = self.rows[i][3]
            if t:
                tags.setdefault(t, []).append(k)
        for t, ks in tags.items():
            self.cases[t] = dict(rows=np.array(ks, np.int64))
        return dict(pts=pts, q_imu=np.asarray(self.q_imu, np.float64), q_lb=np.asarray(self.q_lb, np.float64),
                    line_num=self.line_num, ds_rate=self.ds_rate, cases=dict(self.cases))


def fill(sw, skip=(), n=60, R=12.0, seed=0):
    """every ring not in skip: a dense arc at ~8 m over u in [0.05, 0.17) (flat returns, no breaks) with a step in range in its
    middle, then n returns in blocks over the rest of the turn"""
    rng = np.random.default_rng(seed)
    for r in range(n_rings(sw.line_num)):
        if r in skip:
            continue
        R0 = 8.0 + float(rng.uniform(0, 1))
        arc = blocks_ring(sw.line_num, r, 90, R0, 0.05, 0.17, block=45, far=1.02)
        sw.add(arc + blocks_ring(sw.line_num, r, n + int(rng.integers(0, 8)), R + float(rng.uniform(0, 4)), 0.2, 1.0))


# ---- the tables' bin edges: the two adjacent floats of z where the verdict changes, found by bisection on the oracle
def _ord(f):
    i = np.asarray(f, F).view(np.int32).astype(np.int64)
    return np.where(i >= 0, i, -(i & 0x7fffffff))


def _unord(o):
    o = np.asarray(o, np.int64)
    i = np.where(o >= 0, o, (-o) | 0x80000000).astype(np.uint32)
    return i.view(F)


def bin_edge_pairs(line_num, R=20.0, az=0.0):
    """[(z_below, z_above, verdict_below, verdict_above)] at every change of the table's verdict along elevation -30..25 deg"""
    x, y = F(R * math.cos(az)), F(R * math.sin(az))
    zs = np.array([R * math.tan(math.radians(e)) for e in np.arange(-30.0, 25.0, 0.02)], F)

    def verdict(z):
        p = np.zeros(len(z), PT32); p["x"] = x; p["y"] = y; p["z"] = z
        return rot_oracle.scan_ids(p, line_num)
    v = verdict(zs)
    idx = np.nonzero(v[1:] != v[:-1])[0]
    lo, hi = _ord(zs[idx]), _ord(zs[idx + 1])
    vlo = v[idx]
    for _ in range(40):
        mid = (lo + hi) // 2
        vm = verdict(_unord(mid))
        same = vm == vlo
        lo = np.where(same & (hi - lo > 1), mid, lo); hi = np.where(~same & (hi - lo > 1), mid, hi)
    zl, zh = _unord(lo), _unord(hi)
    return [(x, y, zl[k], zh[k], int(verdict(zl[k:k + 1])[0]), int(verdict(zh[k:k + 1])[0])) for k in range(len(idx))]


def angle_pairs_64(R=20.0):
    """returns whose float elevation is the float either side of 2.0, -8.83 and -24.33 (the 64-line gates)"""
    import rot_restate
    out = []
    for a in (2.0, -8.83, -24.33):
        z0 = F(R * math.tan(math.radians(a)))
        below = above = None
        z = z0
        for _ in range(400):
            z = np.nextafter(z, F(-np.inf))
            if float(rot_restate.elevation(R, 0, z)) < a:
                below = z; break
        z = z0
        for _ in range(400):
            if float(rot_restate.elevation(R, 0, z)) >= a:
                above = z; break
            z = np.nextafter(z, F(np.inf))
        out.append((a, below, above))
    return out


def tables_sweep(line_num, ds_rate):
    sw = Sweep(line_num, ds_rate)
    fill(sw, skip=(2, 3, 4), seed=line_num)
    sw.add(blocks_ring(line_num, 3, 17, 9.0))                 # ring 2 empty; ring 3: 17 returns (scanEnd - scanStart = 6)
    sw.add(blocks_ring(line_num, 4, 16, 9.0))                 # ring 4: 16 (scanEnd - scanStart = 5: skipped)
    sw.ring("ring_17", 3); sw.ring("ring_16", 4); sw.ring("ring_0", 2)
    for (x, y, zl, zh, vl, vh) in bin_edge_pairs(line_num):
        u = u_of(x, y) + 0.25
        sw.add([(u, (x, y, zl)), (u, (x, y, zh))], f"edge_{vl}_{vh}")
    if line_num == 64:
        for a, b, c in angle_pairs_64():
            sw.add([(0.4, (F(20.0), F(0), b)), (0.4, (F(20.0), F(0), c))], f"angle_{a}")
    # r^2 one ulp either side of 9.0f (removeClosedPointCloud), NaN / +-inf coordinates, finite returns whose r^2 overflows
    import hz_adversarial as H
    d = (math.cos(0.5), math.sin(0.5), 0.0)
    for nm, t in (("r2_below9", np.nextafter(F(9.0), F(0))), ("r2_at9", F(9.0)), ("r2_above9", np.nextafter(F(9.0), F(10)))):
        sw.add([(0.3, tuple(H.point_with_sq(t, d)))], nm)
    sw.add([(0.31, (F(np.nan), F(5), F(0))), (0.31, (F(5), F(np.inf), F(0))), (0.31, (F(5), F(0), F(-np.inf)))], "nonfinite_xyz")
    sw.add([(0.6, (F(3e19), F(-2e19), F(0)))], "r2_overflow")
    return sw.build()


# ---- the exact wall (16-line table, z = 0: ring 8)
WALL_X = F(128.0)
WALL_S = F(1.0 / 32.0)


def wall(n, y0, u0, u1):
    ys = [F(y0 - k * WALL_S) for k in range(n)]
    return [[u0 + (u1 - u0) * (k + 0.5) / n, [WALL_X, ys[k], F(0)]] for k in range(n)]


def _set_curv_neighbour(seq, i, target):
    """displace seq[i] in z so that its neighbour i + 1 has curvature `target` exactly (dZ = z_i, dX = dY = 0); the z displacement
    is searched over neighbouring floats, with an x displacement of k * 2^-13 for finer steps"""
    base = [tuple(p) for _, p in seq[i - 6:i + 7]]
    z0 = F(math.sqrt(float(target)))
    for kx in range(0, 64):
        for dz in range(-40, 41):
            z = F(z0)
            for _ in range(abs(dz)):
                z = np.nextafter(z, F(np.inf) if dz > 0 else F(-np.inf))
            P = np.array(base, F)
            P[6, 2] = z
            P[6, 0] = F(WALL_X + F(kx * 2.0 ** -13))
            if curvature(P)[7] == target:
                seq[i][1] = [P[6, 0], P[6, 1], z]
                return
    raise AssertionError(target)


def curv_sweep():
    """ring 8 of the 16-line table is an exact wall with the threshold cases, the other rings are filled"""
    sw = Sweep(16, 1)
    fill(sw, skip=(8,), seed=5)
    seq = wall(660, 10.0, u_of(128, 10.0), u_of(128, -10.6))
    case = {}
    # exact 2.0: the return at 40 moved by (+1, +1) in x and y; its ten neighbours' curvature is 1 + 1
    seq[40][1] = [F(WALL_X + 1), F(seq[40][1][1] + 1), F(0)]
    case["curv_eq2"] = [35, 36, 37, 38, 39, 41, 42, 43, 44, 45]
    for nm, i, t in (("curv_2_up", 100, np.nextafter(F(2), F(3))), ("curv_2_down", 160, np.nextafter(F(2), F(0))),
                     ("curv_01_up", 220, np.nextafter(F(0.1), F(1))), ("curv_01_at", 280, F(0.1)),
                     ("curv_01_down", 340, np.nextafter(F(0.1), F(0)))):
        _set_curv_neighbour(seq, i, t)
        case[nm] = [i + 1]
    # gaps: a pick at i (moved by dz in z: curvature 100 dz^2 ~ 5) whose squared gap to both neighbours, (1/32)^2 + dz^2 in fp32,
    # is 0.05f (the float just above 0.05: a break) or the float below it (no break: the pick marks its neighbours)
    for nm, i, g in (("gap_at", 420, F(0.05)), ("gap_below", 480, np.nextafter(F(0.05), F(0)))):
        s2 = F(WALL_S * WALL_S)
        z = F(math.sqrt(float(g) - float(s2)))
        for _ in range(200):
            gg = F(s2 + F(z * z))
            if gg == g:
                break
            z = np.nextafter(z, F(np.inf) if gg < g else F(-np.inf))
        assert F(s2 + F(z * z)) == g, (nm, g)
        seq[i][1] = [WALL_X, seq[i][1][1], z]
        # i + 6 moved by (+1, +1): i + 1 .. i + 5 become sharp candidates (curvature 2 + dz^2) that only a break keeps pickable
        seq[i + 6][1] = [F(WALL_X + 1), F(seq[i + 6][1][1] + 1), F(0)]
        case[nm] = [i]
    # more than 10 sharp candidates of equal curvature: 12 displaced returns 11 apart on one segment
    for k in range(12):
        i = 560 + 8 * k
        if i >= 655:
            break
        seq[i][1] = [F(WALL_X + 2), seq[i][1][1], F(0)]
    case["sharp_many"] = [560 + 8 * k for k in range(12) if 560 + 8 * k < 655]
    sw.add([(u, tuple(p)) for u, p in seq], "wall")
    s = sw.build()
    rows_of_seq = s["cases"]["wall"]["rows"]       # input rows of the wall in sequence order (ring order is input order)
    for nm, ks in case.items():
        s["cases"][nm] = dict(rows=rows_of_seq[np.array(ks)])
    s["cases"]["wall"]["ring"] = 8
    return s


# ---- azimuth: first and last returns, the latch
def azimuth_sweep(kind):
    sw = Sweep(16, 2)
    fill(sw, seed=7, n=40)
    if kind == "end_sub":           # last return puts endOri - startOri above 3 pi
        sw.add([(-0.01, pt(9.0, math.pi - 0.1, CTR[16](2))), (1.2, pt(9.0, -0.5, CTR[16](2)))], "first_last")
    elif kind == "end_add":         # below pi
        sw.add([(-0.01, pt(9.0, -math.pi + 0.1, CTR[16](2))), (1.2, pt(9.0, 0.5, CTR[16](2)))], "first_last")
    elif kind == "cut_pi_pos":      # first return just either side of the +-pi cut
        sw.add([(-0.02, pt(9.0, math.pi - 1e-6, CTR[16](0)))], "first_last")
    elif kind == "cut_pi_neg":
        sw.add([(-0.02, pt(9.0, -math.pi + 1e-6, CTR[16](0)))], "first_last")
    elif kind == "latch_never":     # every return in the first half turn
        sw = Sweep(16, 1)
        for r in range(16):
            sw.add(blocks_ring(16, r, 40, 10.0 + r, 0.0, 0.45))
    elif kind == "latch_first":     # the first kept return already past startOri + pi: a dropped return (table miss) opens
        sw = Sweep(16, 1)
        sw.add([(-0.2, pt(9.0, A0, 40.0))], "dropped_ahead")          # elevation 40 deg: removed by the table, sets startOri
        sw.add([(-0.1, pt(9.0, A0 - math.pi - 0.3, CTR[16](0)))], "latch_row")
        for r in range(16):
            sw.add(blocks_ring(16, r, 40, 10.0 + r, 0.0, 0.9))
    elif kind == "latch_last":
        sw = Sweep(16, 1)
        for r in range(16):
            sw.add(blocks_ring(16, r, 40, 10.0 + r, 0.0, 0.45))
        sw.add([(2.0, pt(9.0, A0 - math.pi - 0.2, CTR[16](0)))], "latch_row")
    elif kind == "reltime_out":     # returns behind the start and far past the end, negative intensities on ring 0
        sw.add([(0.5, pt(9.0, A0 + 0.4, CTR[16](0))), (0.5, pt(9.0, A0 - 2 * math.pi + 0.8, CTR[16](0))),
                (0.95, pt(9.0, -0.5, CTR[16](0)))], "reltime_out")
    return sw.build()


def latch_ring0_sweep():
    """the latch fires at a ring-0 return whose azimuth does not survive the latched branch's +2 pi / -2 pi round trip: the
    latch index's own branch is visible in its intensity"""
    sw = Sweep(16, 1)
    sw.add([(-1.0, pt(9.0, A0, CTR[16](1)))], "first")                  # startOri = -A0
    for r in range(16):
        sw.add(blocks_ring(16, r, 30, 10.0 + r, 0.0, 0.9))
    for k in range(200):
        a = A0 - math.pi - 1e-3 - k * 1.37e-5
        p = pt(9.0, a, CTR[16](0))
        o = F(-math.atan2(float(p[1]), float(p[0])))
        rt = F(float(F(float(o) + 2 * math.pi)) - 2 * math.pi)
        if rt != o:
            sw.add([(0.5 - 1e-4, p)], "latch_row")
            return sw.build()
    raise AssertionError("no latch azimuth")


# ---- de-skew
def deskew_sweeps(base):
    qs = {"q_nonunit": ((0.9, 0.2, -0.1, 0.05), ID), "q_nan": ((np.nan, 0.1, 0, 0), ID), "q_wneg": ((-0.995, 0.05, 0.08, -0.02), ID),
          "q_lb": ((0.998, 0.01, -0.05, 0.02), (0.9, 0.1, 0.3, -0.2)), "q_slerp_lin": ((1.0, 1e-17, 0.0, 0.0), ID),
          "q_general": ((0.9987, 0.03, -0.02, 0.035), ID)}
    out = []
    for nm, (q, ql) in qs.items():
        s = dict(base); s["q_imu"] = np.asarray(q, np.float64); s["q_lb"] = np.asarray(ql, np.float64); s["cases"] = dict(base["cases"])
        out.append((nm, s))
    return out


def nonunit_near_sweep():
    """a non-unit q_iMU (|q| = 0.2) shrinks returns past 3 m to within 0.5 m: the flat walk's `continue`"""
    sw = Sweep(16, 1, q_imu=(0.2, 0.0, 0.0, 0.0))
    fill(sw, skip=(0,), seed=11, n=40, R=4.0)
    sw.add(blocks_ring(16, 0, 40, 3.05, 0.93, 0.99, block=40), "near")
    return sw.build()


# ---- ring and segment shapes
def shapes_sweep():
    sw = Sweep(64, 1)
    fill(sw, skip=(1, 2, 5, 9, 10, 20, 21), seed=13, n=40)
    sw.add(blocks_ring(64, 1, 1, 9.0)); sw.ring("ring_1", 1)
    sw.add(blocks_ring(64, 2, 11, 9.0)); sw.ring("ring_11", 2)
    sw.add(blocks_ring(64, 5, 12, 9.0)); sw.ring("ring_12", 5)
    sw.add(blocks_ring(64, 20, 6158, 15.0, block=5)); sw.ring("ring_1024_1025", 20)   # scanEnd - scanStart = 6147
    sw.ring("empty_9", 9); sw.ring("empty_10", 10); sw.ring("empty_21", 21)
    return sw.build()


def cap_sweep(n_ring):
    sw = Sweep(16, 1)
    fill(sw, skip=(8,), seed=17, n=30)
    sw.add(blocks_ring(16, 8, n_ring, 25.0, block=7)); sw.ring("big_ring", 8)
    return sw.build()


# ---- per-ring VoxelGrid
def line_ring(n, x0, y0, s, u0=0.3):
    """n returns on z = 0 at (x0 + k s, y0 + k s): exact, collinear, equally spaced, in descending k (so that a filtered ring
    comes out reversed and a passed-through one does not)"""
    return [(u0 + 1e-4 * (n - k), (F(x0 + k * s), F(y0 + k * s), F(0))) for k in range(n)]


def vg_sweep(kind):
    sw = Sweep(64, 1)
    fill(sw, skip=(6,), seed=19, n=50)
    if kind == "overflow":        # 50 less-flat returns spanning d = 46346 cells in x and y: d^2 > INT_MAX, passed through
        seq = line_ring(61, 3000.0, -24000.0, 567.5)
    elif kind == "short":         # d = 46326: d^2 < INT_MAX, filtered
        seq = line_ring(61, 3000.0, -24000.0, 567.25)
    elif kind == "far":           # a tight cluster ~1.5e9 m out: x / leaf beyond 2^31, PCL sends every x index to INT_MIN
        seq = []
        for xr in range(3):
            for k in range(30):
                x, y = F(1.5e9 + 128.0 * xr), F(0.5 + k * 0.125)
                seq.append((u_of(x, y) + 1e-3 * (xr * 30 + k), (x, y, F(0))))
    else:                         # leaf multiples: returns on exact multiples of 0.6 and one ulp below
        seq = []
        for k in range(60):
            xm = F(0.6 * (10 + k // 2))
            x = xm if k % 2 == 0 else np.nextafter(xm, F(0))
            seq.append((u_of(x, F(3.0)) + 1e-4 * k, (x, F(3.0), F(0))))
        seq.sort(key=lambda t: t[0])
    sw.add(seq, f"vg_{kind}")
    sw.ring(f"vg_ring_{kind}", 6)
    return sw.build()


# ---- non-finite curvature
def nonfinite_curv_sweep(kind):
    sw = Sweep(64, 1)
    fill(sw, skip=(6,), seed=23, n=50)
    seq = line_ring(80, 20.0, -40.0, 1.0)
    m = 40
    if kind == "nan":             # 2e38 + 2e38 = inf, then - 10 * 1e38 = -inf: inf + -inf in the stencil
        seq[m + 2] = (seq[m + 2][0], (F(2e38), F(0), F(0)))        # ring order is descending k: 2e38, 2e38, 1e38
        seq[m + 1] = (seq[m + 1][0], (F(2e38), F(0), F(0)))
        seq[m] = (seq[m][0], (F(1e38), F(0), F(0)))
    else:                         # returns ~1e19 out: curvature +inf
        seq[m] = (seq[m][0], (F(1e19), F(0), F(0)))
    sw.add(seq, f"curv_{kind}")
    sw.ring(f"curv_ring_{kind}", 6)
    return sw.build()


def edge_table_sweep():
    """the full edge table of the 64-line tables: all 51 rings they can produce have six segments of sharp-only returns (blocks
    of 2, a break between every block), so each of the 306 segments picks 10 edges"""
    sw = Sweep(64, 1)
    for r in range(51):
        sw.add(blocks_ring(64, r, 6 * 40 + 11, 10.0 + 0.1 * r, block=2, far=1.6))
    return sw.build()


def single_sweep():
    sw = Sweep(64, 1)
    sw.add([(0.1, pt(10.0, 0.0, 0.0))], "single")
    return sw.build()


def dropped_sweep():
    sw = Sweep(32, 1)
    sw.add([(k / 50, pt(2.0, az_of(k / 50), 0.0)) for k in range(50)] + [(0.5, pt(10.0, 0.0, 60.0))], "dropped")
    return sw.build()


def all_sweeps():
    """[(name, sweep)]"""
    out = []
    for ln in (16, 32, 64):
        base = tables_sweep(ln, 1)
        for ds in (1, 2, 3, 4):
            s = dict(base); s["ds_rate"] = ds
            out.append((f"tables{ln}_ds{ds}", s))
    out.append(("curv16", curv_sweep()))
    for k in ("end_sub", "end_add", "cut_pi_pos", "cut_pi_neg", "latch_never", "latch_first", "latch_last", "reltime_out"):
        out.append((f"az_{k}", azimuth_sweep(k)))
    out.append(("latch_ring0", latch_ring0_sweep()))
    out += [(f"deskew_{nm}", s) for nm, s in deskew_sweeps(dict(out[0][1]))]
    out.append(("nonunit_near", nonunit_near_sweep()))
    out.append(("shapes64", shapes_sweep()))
    out.append(("ring16384", cap_sweep(16384)))
    for k in ("overflow", "short", "far", "multiples"):
        out.append((f"vg_{k}", vg_sweep(k)))
    for k in ("nan", "inf"):
        out.append((f"curv_{k}", nonfinite_curv_sweep(k)))
    out.append(("edge_table", edge_table_sweep()))
    out.append(("single", single_sweep()))
    out.append(("dropped", dropped_sweep()))
    return out


def identity_q(sw):
    return np.array_equal(sw["q_imu"], ID) or bool(np.isnan(sw["q_imu"]).any())


def far_cluster(stride):
    """the far cluster alone as a cloud of the given stride (48: PT48, 32: PT32) for liliom_voxelgrid"""
    import oracle_lib
    dt = oracle_lib.PT48 if stride == 48 else PT32
    pts = np.zeros(90, dt)
    k = np.arange(90)
    pts["x"] = (1.5e9 + 128.0 * (k // 30)).astype(F); pts["y"] = (0.5 + (k % 30) * 0.125).astype(F); pts["w"] = 1.0
    pts["intensity"] = (k % 7).astype(F)
    return pts
