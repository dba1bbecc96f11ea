"""Adversarial Livox-Horizon sweeps for the Horizon extractor (L/src/Preprocessing.cpp:225-383): seeded, every return placed
directly on a (line, column) cell, each case a named range of patches so that a failure names its case.

Layout.  The 664 patches (columns 5 + 6p .. 10 + 6p) are grouped in blocks of four: a filler patch, the CASE patch, a filler
patch and an empty separator.  A block's cells lie on a sphere of radius R around the sensor (every depth is R to the last
ulp, so the depth Laplacian of an untouched cell is ~1e-7 and only what a case puts there crosses 0.06), with azimuth
A * (column - case patch centre) and elevation E * (line - 2.5): the case patch and its two window-wide neighbours are mirror
symmetric in azimuth, and the empty separator keeps blocks from seeing each other (an empty neighbour only lowers a
Laplacian).  Columns 0-4 and 3989-3999 lie outside every patch and are filled as well.

A sweep is a dict: pts (PT48, array order = compaction order), q (q_iMU), cases {name: dict(patches=[...]) or
dict(rows=index array)} naming the case patches or the array rows of single returns."""
from __future__ import annotations

import math

import numpy as np

from oracle_lib import LIVOX20, PT48

F = np.float32
N_SCANS, H_SCANS = 6, 4000
T_INTERVAL = 0.1 / (H_SCANS - 1)       # Preprocessing.cpp:239
N_PATCHES = 664
A_STEP, E_STEP = 0.05, 0.05            # rad per column / per line inside a block
POLE = 0.93                            # depth factor of an edge candidate: g1 = 0.07 / 0.93 / 1 ~ 0.075 > 0.06
DBL_EPS = np.finfo(np.float64).eps


def scan_id_of(x) -> int:
    """int(float) as x86-64 converts it (cvttss2si): truncation, INT_MIN for NaN, +-inf and |x| >= 2^31."""
    x = float(np.float32(x))
    if not (-2147483648.0 <= x < 2147483648.0):
        return -2147483648
    return int(x)


def round_half_away(v: float) -> float:
    """std::round"""
    if not math.isfinite(v):
        return v
    r = math.floor(abs(v) + 0.5) if abs(v) - math.floor(abs(v)) >= 0.5 else math.floor(abs(v))
    return math.copysign(r, v)


def col_quotient(inten) -> float:
    """(intensity - scan_id) / t_interval as the reference evaluates it: float - int -> float, widened, / double (:262)"""
    sid = scan_id_of(inten)
    return float(F(F(inten) - F(sid))) / T_INTERVAL


def col_of(inten) -> int | None:
    q = round_half_away(col_quotient(inten))
    return int(q) if math.isfinite(q) else None


def patch_first_col(p: int) -> int:
    return 5 + 6 * p


def patch_of_col(c: int) -> int | None:
    if c < 5 or c > 5 + 6 * N_PATCHES - 1:
        return None
    return (c - 5) // 6


def intensity_of(line: int, col: int) -> np.float32:
    """a float intensity whose scan id is `line` and whose column rounds to `col`"""
    f = F(line + col * T_INTERVAL)
    for _ in range(64):
        c = col_of(f)
        if scan_id_of(f) == line and c == col:
            return f
        f = np.nextafter(f, F(np.inf) if c < col else F(-np.inf))
    raise AssertionError((line, col))


def half_columns(line: int, lo: int, hi: int, k: int = 2):
    """The intensities of `line` whose column quotient comes closest to a half (c + 0.5) from below and from above, over columns
    lo..hi-1: the k closest of each side.  (No float fraction gives an exact half for t_interval = 0.1 / 3999: the quotient is
    rounded to 53 bits, the fraction only has 24.)  Returns [(intensity, quotient)]."""
    below, above = [], []
    for c in range(lo, hi):
        f0 = F(line + (c + 0.5) * T_INTERVAL)
        u = v = f0
        cands = [f0]
        for _ in range(4):
            u = np.nextafter(u, F(np.inf)); v = np.nextafter(v, F(-np.inf)); cands += [u, v]
        for f in cands:
            qv = col_quotient(f)
            if scan_id_of(f) != line:
                continue
            d = qv - (c + 0.5)
            (below if d < 0 else above).append((abs(d), f, qv))
    below.sort(key=lambda t: t[0]); above.sort(key=lambda t: t[0])
    return [(f, qv) for _, f, qv in below[:k] + above[:k]]


def _dir(az, el):
    return np.array([math.cos(el) * math.cos(az), math.cos(el) * math.sin(az), math.sin(el)])


def fp32_sq(p) -> np.float32:
    """x*x + y*y + z*z in fp32, left to right (the gate's `dep` before widening, :259)"""
    x, y, z = (F(v) for v in p)
    return F(F(F(x * x) + F(y * y)) + F(z * z))


def point_with_sq(target: np.float32, direction, span: int = 6):
    """An fp32 point near sqrt(target) * direction whose fp32 squared norm is exactly `target` (neighbouring floats of each
    coordinate searched, as knn_reference._point_at does)."""
    c0 = (math.sqrt(float(target)) * np.asarray(direction, np.float64)).astype(F)
    axes = []
    for k in range(3):
        vals = [c0[k]]
        u = v = c0[k]
        for _ in range(span):
            u = np.nextafter(u, F(np.inf)); v = np.nextafter(v, F(-np.inf))
            vals += [u, v]
        axes.append(np.array(vals, F))
    X, Y, Z = np.meshgrid(*axes, indexing="ij")
    cand = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1)
    sq = ((cand[:, 0] * cand[:, 0]) + (cand[:, 1] * cand[:, 1])) + (cand[:, 2] * cand[:, 2])
    assert sq.dtype == F
    hit = np.nonzero(sq == target)[0]
    assert len(hit), (target, direction)
    p = cand[hit[0]]
    assert fp32_sq(p) == target
    return p


def floats_around(v: float):
    """(largest float < v, smallest float > v, and v itself when it is a float)"""
    f = F(v)
    lo = f if float(f) < v else np.nextafter(f, F(-np.inf))
    hi = f if float(f) > v else np.nextafter(f, F(np.inf))
    return lo, hi


class SweepBuilder:
    def __init__(self, seed: int):
        self.rng = np.random.default_rng(seed)
        self.cells: dict[tuple[int, int], list] = {}     # (line, col) -> [(x, y, z, curvature)], first = time order
        self.extra: list[tuple] = []                     # single returns not tied to a cell: (x, y, z, intensity, curvature, case)
        self.cases: dict[str, dict] = {}
        self.block = 0
        self.shuffled: list[tuple] = []                  # collision returns placed at random positions: (line, col, xyz, curv, case)

    def refl(self):
        return F(0.1 * int(self.rng.integers(10, 201)))

    # -- blocks
    def next_block(self):
        b = self.block
        self.block += 1
        assert 4 * b + 3 < N_PATCHES + 1, "out of patches"
        return 4 * b + 1

    def fill_block(self, case_patch: int, R: float, noise: float = 0.0):
        """filler + case + filler patches on the sphere of radius R (the case patch's cells may be replaced afterwards)"""
        c0 = patch_first_col(case_patch - 1)
        centre = patch_first_col(case_patch) + 2.5
        for c in range(c0, c0 + 18):
            for k in range(N_SCANS):
                self.put(k, c, self.sphere(R * (1.0 + noise * self.rng.normal()), c - centre, k))

    def sphere(self, r, dc, k):
        return (r * _dir(A_STEP * dc, E_STEP * (k - 2.5))).astype(F)

    def put(self, k, c, xyz, curv=None):
        self.cells[(k, c)] = [(np.asarray(xyz, F), self.refl() if curv is None else F(curv))]

    def case(self, name, patch):
        self.cases.setdefault(name, {"patches": []})["patches"].append(patch)

    def centre(self, p):
        return patch_first_col(p) + 2.5

    # -- the sweep
    def build(self, q, extra_first: bool = False):
        rows = []
        for (k, c) in sorted(self.cells, key=lambda kc: (kc[1], kc[0])):            # time order: column outer, line inner
            inten = intensity_of(k, c)
            for xyz, curv in self.cells[(k, c)]:
                rows.append((xyz[0], xyz[1], xyz[2], inten, curv, None))
        for (k, c, xyz, curv, name) in self.shuffled:                                # a cell's later returns anywhere in the array
            pos = int(self.rng.integers(0, len(rows) + 1))
            rows.insert(pos, (xyz[0], xyz[1], xyz[2], intensity_of(k, c), curv, name))
        tail = list(self.extra)
        if extra_first:
            rows = tail + rows
        else:
            rows = rows + tail
        pts = np.zeros(len(rows), PT48)
        for fld, j in (("x", 0), ("y", 1), ("z", 2), ("intensity", 3), ("curvature", 4)):
            pts[fld] = np.array([r[j] for r in rows], F)
        pts["w"] = 1.0
        cases = dict(self.cases)
        names = [r[5] for r in rows]
        for nm in set(n for n in names if n):
            idx = [i for i, n in enumerate(names) if n == nm]
            cases.setdefault(nm, {})["rows"] = np.array(idx)
        return dict(pts=pts, q=np.asarray(q, np.float64), cases=cases)


# ---------------------------------------------------------------------------------------------------------------- the cases
def _patch_cases(B: SweepBuilder):
    rng = B.rng
    R = 10.0
    cells36 = [(k, j) for j in range(6) for k in range(N_SCANS)]
    # cell counts: 36, 25 and 24 valid cells (the missing ones empty or refused by the reflectivity gate)
    for name, keep in (("num36", 36), ("num25", 25), ("num24", 24), ("num25", 25), ("num24", 24)):
        p = B.next_block(); B.fill_block(p, R, noise=2e-4); B.case(name, p)
        c0 = patch_first_col(p)
        drop = rng.permutation(36)[: 36 - keep]
        for t, e in enumerate(drop):
            k, j = cells36[e]
            if t % 2 == 0:
                del B.cells[(k, c0 + j)]
            else:
                xyz, _ = B.cells[(k, c0 + j)][0]
                B.cells[(k, c0 + j)] = [(xyz, F(0.01))]                               # curvature < 0.05: in the cutted cloud, no cell
    # edge candidates: 3 (refused: nedge > 3), 4 and 6 per patch; the same column on every line (a vertical, line-like set)
    for name, lines, j in (("edges3", (0, 1, 2), 2), ("edges4", (0, 1, 2, 3), 2), ("edges6", range(6), 3),
                           ("edges4_hi", (2, 3, 4, 5), 5), ("edges4_hi", (1, 3, 4, 5), 4), ("edges6_hi", range(6), 5),
                           ("edges3_hi", (3, 4, 5), 4)):
        p = B.next_block(); B.fill_block(p, R); B.case(name, p)
        c = patch_first_col(p) + j
        for k in lines:
            B.put(k, c, B.sphere(R * POLE, c - B.centre(p), k))
    # Laplacian ties: poles at j = 0 and j = 5 of every line, mirror images of each other -> equal g1, the first column wins
    for _ in range(2):
        p = B.next_block(); B.fill_block(p, R); B.case("tie", p)
        for j in (0, 5):
            c = patch_first_col(p) + j
            for k in range(N_SCANS):
                B.put(k, c, B.sphere(R * POLE, c - B.centre(p), k))
    # degenerate patches
    p = B.next_block(); B.fill_block(p, R); B.case("coincident", p)
    same = B.sphere(R, 0.0, 2.5)
    for k, j in cells36:
        B.put(k, patch_first_col(p) + j, same)
    p = B.next_block(); B.fill_block(p, R); B.case("collinear", p)
    base = B.sphere(R, 0.0, 2.5)
    for k, j in cells36:
        B.put(k, patch_first_col(p) + j, base + np.array([0.0, 0.0, 0.05 * (6 * j + k - 17.5)], F))
    p = B.next_block(); B.fill_block(p, R); B.case("plane_sym", p)
    for k, j in cells36:                                                                 # x = R, a symmetric 6 x 6 grid in (y, z)
        B.put(k, patch_first_col(p) + j, np.array([R, 0.25 * (j - 2.5), 0.25 * (k - 2.5)], F))
    # gates at their edges: 24 valid cells + the gate cell, so the patch emits iff the gate cell is binned
    lo4, hi4 = np.nextafter(F(4.0), F(0)), np.nextafter(F(4.0), F(np.inf))
    lo4e, hi4e = np.nextafter(F(40000.0), F(0)), np.nextafter(F(40000.0), F(np.inf))
    c_lo, c_hi = floats_around(0.05)
    k_lo, k_hi = floats_around(25.45)
    gates = [("dep_4_below", 2.0, lo4, None, False), ("dep_4_at", 2.0, F(4.0), None, True), ("dep_4_above", 2.0, hi4, None, True),
             ("dep_40000_below", 200.0, lo4e, None, True), ("dep_40000_at", 200.0, F(40000.0), None, True),
             ("dep_40000_above", 200.0, hi4e, None, False),
             ("curv_0.05_below", R, None, c_lo, False), ("curv_0.05_above", R, None, c_hi, True),
             ("curv_25.45_below", R, None, k_lo, True), ("curv_25.45_above", R, None, k_hi, False)]
    for name, r, dep, curv, passes in gates:
        p = B.next_block()
        inside = 1.0 + 5e-4 if r < 100 else 1.0 - 5e-4                                   # every other cell safely inside the range gate
        B.fill_block(p, r * inside); B.case(name, p)
        B.cases[name]["gate_passes"] = passes
        c0 = patch_first_col(p)
        order = rng.permutation(36)
        gk, gj = cells36[order[0]]
        for e in order[1:12]:                                                            # 11 others removed: 24 + the gate cell
            k, j = cells36[e]
            del B.cells[(k, c0 + j)]
        c = c0 + gj
        if dep is not None:
            B.put(gk, c, point_with_sq(dep, _dir(A_STEP * (c - B.centre(p)), E_STEP * (gk - 2.5))))
        else:
            B.put(gk, c, B.sphere(r, c - B.centre(p), gk), curv=curv)
        B.cases[name]["cell"] = (gk, c)
    # cell collisions: 2-5 returns per cell, the later ones anywhere in the array (other block chunks), some refused by a gate
    for _ in range(3):
        p = B.next_block(); B.fill_block(p, R); B.case("collisions", p)
        c0 = patch_first_col(p)
        for e in rng.permutation(36)[:14]:
            k, j = cells36[e]
            c = c0 + j
            for m in range(int(rng.integers(1, 5))):
                xyz = B.sphere(R * (1.0 + 2e-3 * rng.normal()), c - B.centre(p) + 0.3 * rng.normal(), k + 0.3 * rng.normal())
                curv = F(0.01) if m == 0 and rng.uniform() < 0.3 else None
                B.shuffled.append((k, c, xyz, B.refl() if curv is None else curv, "collisions_rows"))
    # column rounding: cells whose quotient is the closest float to a half, on both sides, inside a patch
    p = B.next_block(); B.fill_block(p, R); B.case("col_half", p)
    c0 = patch_first_col(p)
    halves = []
    for k in range(N_SCANS):
        for f, qv in half_columns(k, c0, c0 + 5, k=1):
            c = col_of(f)
            B.cells.pop((k, c), None)                                                    # the half return is the cell's only one
            xyz = B.sphere(R * (1.0 + 1e-3), c - B.centre(p), k)
            B.extra.append((xyz[0], xyz[1], xyz[2], f, B.refl(), "col_half_rows"))
            halves.append((k, qv, c))
    B.cases["col_half"]["halves"] = halves


def _outside_cells(B: SweepBuilder):
    """columns 0-4 and 3989-3999 (outside every patch) and the returns that round to 3999 and 4000"""
    for c in list(range(0, 5)) + list(range(3989, 4000)):
        for k in range(N_SCANS):
            B.put(k, c, B.sphere(10.0, 0.0, k))
    B.cases["outside_cols"] = {"cols": list(range(0, 5)) + list(range(3989, 4000))}
    for k in range(N_SCANS):
        for f in (F(k + 3999 * T_INTERVAL), F(k + 3999.49 * T_INTERVAL), F(k + 3999.51 * T_INTERVAL), F(k + 4000 * T_INTERVAL)):
            xyz = B.sphere(10.0, 0.0, k)
            B.extra.append((xyz[0], xyz[1], xyz[2], f, B.refl(), "col_3999_4000_rows"))


def intensity_edge_rows(B: SweepBuilder):
    """single returns at a finite, well-ranged position with the intensities the extractor must treat like x86 does"""
    vals = []
    for k in range(N_SCANS):
        vals += [F(k + 0.1), np.nextafter(F(k + 0.1), F(np.inf)), F(k + 0.15), F(k + 0.5), F(k + 0.999)]        # ratio clamped to 1
    frac_hi = len(vals)
    neg = [F(-0.5), F(-0.999), F(-1e-6), F(-1.2e-5), F(-1.3e-5), np.nextafter(F(-1.0), F(0))]
    ids = [F(6.02), F(7.0), F(100.05), F(255.09), F(2147483520.0)]
    bad = [F(np.nan), F(np.inf), F(-np.inf), F(3e9), F(-3e9), F(2147483648.0), F(-2147483648.0), F(-2147483904.0)]
    groups = (("intensity_frac_ge_0.1", vals[:frac_hi]), ("intensity_negative", neg), ("intensity_scan_id_6_plus", ids),
              ("intensity_non_finite_or_huge", bad))
    for name, vs in groups:
        for v in vs:
            xyz = B.sphere(12.0 * (1.0 + 0.2 * B.rng.uniform()), 40.0 * B.rng.uniform(-1, 1), 6 * B.rng.uniform())
            B.extra.append((xyz[0], xyz[1], xyz[2], v, B.refl(), name))


def _nonunit(q, s):
    return np.asarray(q, np.float64) * s


Q_ROT = np.array([math.cos(0.01), 0.2 * math.sin(0.01), -0.3 * math.sin(0.01), math.sqrt(0.87) * math.sin(0.01)])


def q_cases():
    """q_iMU of the extra sweeps: (name, q, slerp branch of Identity . q)"""
    e = DBL_EPS
    out = [("q_identity", np.array([1.0, 0.0, 0.0, 0.0])),
           ("q_eps_linear", np.array([1.0 - e / 2, 1e-9, -2e-9, 3e-9])),            # |d| within DBL_EPSILON of 1: linear branch
           ("q_eps_linear_at", np.array([1.0 - e, 1e-9, 0.0, -1e-9])),
           ("q_eps_acos", np.array([1.0 - 2 * e, 3e-8, 0.0, 0.0])),                 # just outside: acos of |d| ~ 1 - 2 eps
           ("q_negative_w", -Q_ROT),                                                 # d < 0: s1 negated
           ("q_nonunit_long", _nonunit(Q_ROT, 1.3)),                                 # |d| > 1: linear branch, not re-normalised
           ("q_nonunit_short", _nonunit(Q_ROT, 0.7)),
           ("q_rot", Q_ROT)]
    return [(n, q, "linear" if abs(q[0]) >= 1.0 - e else "acos") for n, q in out]


def make_cells_sweep(seed: int = 5, q=(1.0, 0.0, 0.0, 0.0)):
    """every patch case, the outside columns and the column-rounding returns; q_iMU = identity by default, so the de-skew moves
    nothing and the gates see the coordinates placed here"""
    B = SweepBuilder(seed)
    _patch_cases(B)
    _outside_cells(B)
    # plain blocks in the remaining patches (generic planes, a little noise)
    while 4 * B.block + 3 < N_PATCHES:
        p = B.next_block(); B.fill_block(p, 10.0 + 20.0 * B.rng.uniform(), noise=3e-4); B.case("plain", p)
    return B.build(q)


def make_q_sweep(name: str, q, seed: int):
    """a plainer sweep (planes, edges, collisions) + every intensity edge, de-skewed by q"""
    B = SweepBuilder(seed)
    _outside_cells(B)
    rng = B.rng
    while 4 * B.block + 3 < N_PATCHES:
        R = 8.0 + 30.0 * rng.uniform()
        p = B.next_block(); B.fill_block(p, R, noise=3e-4); B.case("plain", p)
        if rng.uniform() < 0.3:
            c = patch_first_col(p) + int(rng.integers(0, 6))
            for k in range(N_SCANS):
                B.put(k, c, B.sphere(R * POLE, c - B.centre(p), k))
    intensity_edge_rows(B)
    sw = B.build(q, extra_first=bool(seed % 2))
    sw["name"] = name
    return sw


def all_sweeps():
    """[(name, sweep)]: the cell sweep (q = identity), the same cells de-skewed by a rotation, one sweep per q_iMU case"""
    out = [("cells", make_cells_sweep()), ("cells_rot", make_cells_sweep(q=Q_ROT))]
    for i, (name, q, _) in enumerate(q_cases()):
        out.append((name, make_q_sweep(name, q, seed=100 + i)))
    return out


# ---------------------------------------------------------------------------------------------------------------- Livox
def livox_messages(seed: int = 9):
    """[(name, records LIVOX20 or raw bytes, stride)]: FormatConvert.cpp:11-24 inputs at their edges"""
    rng = np.random.default_rng(seed)
    sw = make_q_sweep("livox", Q_ROT, seed=seed)["pts"]
    sw = sw[np.isfinite(sw["intensity"]) & (sw["intensity"] >= 0) & (sw["intensity"] < 6)]
    n = len(sw)
    t_end = 100_000_000
    frac = (sw["intensity"] - np.floor(sw["intensity"])).astype(np.float64)
    order = np.argsort(frac, kind="stable")
    sw, frac = sw[order], frac[order]

    def rec(off, line, pts):
        r = np.zeros(len(pts), LIVOX20)
        r["offset_time"] = off; r["x"] = pts["x"]; r["y"] = pts["y"]; r["z"] = pts["z"]
        r["reflectivity"] = rng.integers(10, 201, len(pts)); r["line"] = line
        return r

    base_off = np.minimum(np.round(frac / 0.1 * t_end), t_end).astype(np.uint32)
    base_off[-1] = t_end
    line = np.floor(sw["intensity"]).astype(np.uint8)
    normal = rec(base_off, line, sw)
    out = [("normal", normal, 20)]
    m = normal.copy(); m["offset_time"][-1] = 0
    out.append(("last_offset_zero", m, 20))                                # time_end = 0: s = x / 0 = inf, 0 / 0 = NaN
    out.append(("one_point_offset_zero", rec(np.zeros(1, np.uint32), np.zeros(1, np.uint8), sw[:1]), 20))
    out.append(("all_offsets_zero", rec(np.zeros(n, np.uint32), line, sw), 20))
    m = normal.copy(); sel = rng.choice(n - 1, n // 10, replace=False)
    m["offset_time"][sel] = t_end + rng.integers(1, t_end, len(sel)).astype(np.uint32)
    out.append(("offset_beyond_end", m, 20))                               # s > 1: ratio clamped, column >= 4000
    m = normal.copy(); sel = rng.choice(n - 1, n // 10, replace=False)
    m["line"][sel] = rng.integers(6, 256, len(sel))
    out.append(("line_6_255", m, 20))
    raw = np.ascontiguousarray(normal).view(np.uint8).reshape(n, 20)[:, :19].copy().reshape(-1)
    out.append(("stride19", raw, 19))
    return out
