"""The ROT extractor (R/src/Preprocessing.cpp:276-509) restated in Python from the reference source, for the CPU tier's checks of
oracle/oracle_rot.cpp and of the kernels' reformulations — TEST INFRASTRUCTURE:

  * `assign` — removeNaN / removeClosedPointCloud, the elevation tables (16, 32 and 64 lines) through glibc's own atanf / atan2f
    (ctypes: what `using namespace std` makes the reference call for floats), the halfPassed azimuth unwrapping and intensity =
    scanID + 0.1 * relTime, bucketed by ring in input order;
  * `curvature` — the 11-point stencil in the literal left-to-right fp32 order;
  * `walk_sequential` — the greedy walk of one ring (:401-500) line by line;
  * `walk_masks` — the availability-mask walk of k_rot_ring (liliom_b200/csrc/extract_rot.cu, segments up to 1024 points);
  * `restate_cloud` — curvature, labels, edge picks and the per-ring VoxelGrid (oracle_lib.voxelgrid) of a laserCloud.

Curvature order: ascending (curvature, index), a NaN after +inf; a NaN is never a candidate (`> 2.0` and `< 0.1` are false)."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

F = np.float32
_libm = None


def libm():
    global _libm
    if _libm is None:
        L = C.CDLL("libm.so.6")
        L.atanf.restype = C.c_float; L.atanf.argtypes = [C.c_float]
        L.atan2f.restype = C.c_float; L.atan2f.argtypes = [C.c_float, C.c_float]
        _libm = L
    return _libm


def removed(x, y, z) -> bool:
    """removeNaN + removeClosedPointCloud(3.0): r^2 in fp32 (an overflow to inf keeps the point)"""
    x, y, z = F(x), F(y), F(z)
    if not (np.isfinite(x) and np.isfinite(y) and np.isfinite(z)):
        return True
    with np.errstate(over="ignore"):
        return bool(F(F(F(x * x) + F(y * y)) + F(z * z)) < F(9.0))


def elevation(x, y, z) -> np.float32:
    """float angle = atan(pz / sqrt(px*px + py*py)) * 180 / M_PI (:315)"""
    x, y, z = F(x), F(y), F(z)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        rxy = np.sqrt(F(F(x * x) + F(y * y)))
        return F(float(F(F(libm().atanf(F(z / rxy))) * F(180))) / math.pi)


def table_scan_id(x, y, z, line_num) -> int:
    """:315-347, -1 for `count--; continue`"""
    a = elevation(x, y, z)
    if line_num == 16:
        s = int(float(F(F(a + F(15)) / F(2))) + 0.5)
        return s if 0 <= s <= 15 else -1
    if line_num == 32:
        s = int((float(a) + 92.0 / 3.0) * 3.0 / 4.0)
        return s if 0 <= s <= 31 else -1
    if float(a) >= -8.83:
        s = int(float(F(F(2) - a)) * 3.0 + 0.5)
    else:
        s = 32 + int((-8.83 - float(a)) * 2.0 + 0.5)
    if a > F(2) or float(a) < -24.33 or s > 50 or s < 0:
        return -1
    return s


def assign(pts, line_num):
    """:280-372.  Returns dict(order: input row of each laserCloud row, ring, intensity (fp32), kept: input rows that survive the
    removal, start_branch ('sub' / 'add' / None: which endOri correction of :290-294 ran), latch: input row where halfPassed fires
    (None: never), rel: relTime per laserCloud row)."""
    X, Y, Z = pts["x"], pts["y"], pts["z"]
    kept = [i for i in range(len(pts)) if not removed(X[i], Y[i], Z[i])]
    out = dict(order=np.zeros(0, np.int64), ring=np.zeros(0, np.int64), intensity=np.zeros(0, F), kept=kept, start_branch=None,
               latch=None, rel=np.zeros(0, F))
    if not kept:
        return out
    a2 = libm().atan2f
    f0, fl = kept[0], kept[-1]
    startOri = F(-a2(Y[f0], X[f0]))
    endOri = F(float(F(-a2(Y[fl], X[fl]))) + 2 * math.pi)
    if float(F(endOri - startOri)) > 3 * math.pi:
        endOri = F(float(endOri) - 2 * math.pi); out["start_branch"] = "sub"
    elif float(F(endOri - startOri)) < math.pi:
        endOri = F(float(endOri) + 2 * math.pi); out["start_branch"] = "add"
    half = False
    buckets = [[] for _ in range(line_num)]
    for i in kept:
        scan = table_scan_id(X[i], Y[i], Z[i], line_num)
        if scan < 0:
            continue
        ori = F(-a2(Y[i], X[i]))
        if not half:
            if float(ori) < float(startOri) - math.pi / 2:
                ori = F(float(ori) + 2 * math.pi)
            elif float(ori) > float(startOri) + math.pi * 3 / 2:
                ori = F(float(ori) - 2 * math.pi)
            if float(F(ori - startOri)) > math.pi:
                half = True; out["latch"] = i
        else:
            ori = F(float(ori) + 2 * math.pi)
            if float(ori) < float(endOri) - math.pi * 3 / 2:
                ori = F(float(ori) + 2 * math.pi)
            elif float(ori) > float(endOri) + math.pi / 2:
                ori = F(float(ori) - 2 * math.pi)
        rel = F(F(ori - startOri) / F(endOri - startOri))
        buckets[scan].append((i, scan, F(scan + 0.1 * float(rel)), rel))
    rows = [t for b in buckets for t in b]
    out["order"] = np.array([t[0] for t in rows], np.int64)
    out["ring"] = np.array([t[1] for t in rows], np.int64)
    out["intensity"] = np.array([t[2] for t in rows], F)
    out["rel"] = np.array([t[3] for t in rows], F)
    return out


def ring_bounds(ring, line_num):
    """[first, end) row of every ring in a ring-major cloud"""
    rf = np.searchsorted(ring, np.arange(line_num), "left"); re = np.searchsorted(ring, np.arange(line_num), "right")
    return rf, re


def curvature(P):
    """:385-394, fp32 left to right; 0 for the first and last five rows"""
    P = np.asarray(P, F)
    n = len(P)
    c = np.zeros(n, F)
    if n < 11:
        return c
    with np.errstate(over="ignore", invalid="ignore"):
        d = P[0:n - 10].copy()
        for k in range(1, 5):
            d = d + P[k:n - 10 + k]
        d = d - F(10) * P[5:n - 5]
        for k in range(6, 11):
            d = d + P[k:n - 10 + k]
        c[5:n - 5] = F(d[:, 0] * d[:, 0]) + F(d[:, 1] * d[:, 1]) + F(d[:, 2] * d[:, 2])
    return c


def _gap_break(P, a, b):
    with np.errstate(over="ignore", invalid="ignore"):
        d = P[a] - P[b]                                   # float32 arithmetic, ((dx*dx)+dy*dy)+dz*dz
        g = F(F(d[0] * d[0]) + F(d[1] * d[1])) + F(d[2] * d[2])
    return float(F(g)) > 0.05


def _range2(P, k):
    p = P[k]
    with np.errstate(over="ignore", invalid="ignore"):
        return float(F(F(p[0] * p[0]) + F(p[1] * p[1])) + F(p[2] * p[2]))


def segments(rf, re):
    scan_start, scan_end = rf + 5, re - 6            # :379-381
    if scan_end - scan_start < 6:
        return []
    return [(scan_start + (scan_end - scan_start) * j // 6, scan_start + (scan_end - scan_start) * (j + 1) // 6 - 1) for j in range(6)]


def curv_key(c, i):
    """ascending (curvature, index), NaN after +inf"""
    c = float(c)
    return (1, 0.0, i) if math.isnan(c) else (0, c, i)


def walk_sequential(P, curv, rf, re):
    """One ring, the reference loop.  Returns (label[], lessflat[], edge picks per segment)."""
    n = len(P)
    label = np.zeros(n, np.int32); picked = np.zeros(n, np.uint8); lessflat = np.zeros(n, np.uint8)
    edges = []

    def suppress(ind):
        for l in range(1, 6):
            if _gap_break(P, ind + l, ind + l - 1): break
            picked[ind + l] = 1
        for l in range(-1, -6, -1):
            if _gap_break(P, ind + l, ind + l + 1): break
            picked[ind + l] = 1

    for sp, ep in segments(rf, re):
        order = sorted(range(sp, ep + 1), key=lambda i: curv_key(curv[i], i))         # std::stable_sort on curvature: ties stay in index order
        seg_edges = []
        largest = 0
        for ind in reversed(order):
            if picked[ind] == 0 and float(curv[ind]) > 2.0:
                largest += 1
                if largest <= 2: label[ind] = 2; seg_edges.append(ind)
                elif largest <= 10: label[ind] = 1; seg_edges.append(ind)
                else: break
                picked[ind] = 1
                suppress(ind)
        smallest = 0
        for ind in order:
            if _range2(P, ind) < 0.25: continue
            if picked[ind] == 0 and float(curv[ind]) < 0.1:
                label[ind] = -1
                smallest += 1
                if smallest >= 4: break
                picked[ind] = 1
                suppress(ind)
        for k in range(sp, ep + 1):
            if _range2(P, k) < 0.25: continue
            if label[k] <= 0: lessflat[k] = 1
        edges.append(seg_edges)
    return label, lessflat, edges


def walk_masks(P, curv, rf, re):
    """One ring, the kernel's fast path (k_rot_ring, `L <= fast_cap` branch), same outputs."""
    n = len(P)
    label = np.zeros(n, np.int32); lessflat = np.zeros(n, np.uint8)
    picked_ring = np.zeros(re - rf, np.uint8)          # S.picked, ring-local
    edges = []
    for sp, ep in segments(rf, re):
        L = ep - sp + 1
        keys = np.array([(int(np.float32(curv[sp + t]).view(np.uint32)) << 32) | (sp + t) for t in range(L)], np.uint64)
        rank_of = np.empty(L, np.int64)
        rank_of[np.argsort(keys, kind="stable")] = np.arange(L)             # the counting sort: keys are unique
        ind_of_rank = [0] * L
        cls = [0] * L
        for t in range(L):
            r = int(rank_of[t])
            ind_of_rank[r] = t
            cv = float(curv[sp + t]); near = _range2(P, sp + t) < 0.25
            cls[r] = (1 if cv > 2.0 else 0) | (2 if (cv < 0.1 and not near) else 0)
        # window index i <-> global sp - 5 + i; brk[i]: pair (i, i-1)
        brk = [0] * (L + 10)
        for i in range(1, L + 10):
            brk[i] = 1 if _gap_break(P, sp - 5 + i, sp - 5 + i - 1) else 0
        ext = []
        for t in range(L):
            w = t + 5
            nf = 0
            while nf < 5 and not brk[w + nf + 1]: nf += 1
            nb = 0
            while nb < 5 and not brk[w - nb]: nb += 1
            ext.append((nf, nb))
        availS = 0; availF = 0                          # bit r: rank r still available
        for r in range(L):
            un = picked_ring[sp + ind_of_rank[r] - rf] == 0
            if (cls[r] & 1) and un: availS |= 1 << r
            if (cls[r] & 2) and un: availF |= 1 << r

        def mark(t):
            nonlocal availS, availF
            nf, nb = ext[t]
            for q in [t] + [t + l for l in range(1, nf + 1)] + [t - l for l in range(1, nb + 1)]:
                picked_ring[sp + q - rf] = 1
                if 0 <= q < L:
                    availS &= ~(1 << int(rank_of[q])); availF &= ~(1 << int(rank_of[q]))

        seg_edges = []
        largest = 0
        while availS:
            largest += 1
            if largest > 10: break
            t = ind_of_rank[availS.bit_length() - 1]    # highest set bit
            label[sp + t] = 2 if largest <= 2 else 1
            seg_edges.append(sp + t)
            mark(t)
        smallest = 0
        while availF:
            t = ind_of_rank[(availF & -availF).bit_length() - 1]      # lowest set bit
            label[sp + t] = -1
            smallest += 1
            if smallest >= 4: break
            mark(t)
        for k in range(sp, ep + 1):
            if _range2(P, k) < 0.25: continue
            if label[k] <= 0: lessflat[k] = 1
        edges.append(seg_edges)
    return label, lessflat, edges


def restate_cloud(cloud, ring, line_num, ds_rate, walk=walk_sequential):
    """laserCloud (PT32, ring-major) and its ring per row -> (curvature, labels, edge cloud, surf cloud, per-ring edge picks):
    :385-508 with the per-ring VoxelGrid(0.6) of oracle_lib"""
    import oracle_lib
    P = np.stack([cloud["x"], cloud["y"], cloud["z"]], 1).astype(F)
    curv = curvature(P)
    label = np.zeros(len(cloud), np.int32)
    edge_rows, surf = [], []
    rf, re = ring_bounds(ring, line_num)
    picks = {}
    for r in range(line_num):
        if r % ds_rate != 0 or re[r] - rf[r] - 11 < 6:
            continue
        lab, lf, edges = walk(P, curv, int(rf[r]), int(re[r]))
        label[rf[r]:re[r]] = lab[rf[r]:re[r]]
        picks[r] = edges
        for e in edges:
            edge_rows += e
        lf_rows = np.nonzero(lf)[0]
        if len(lf_rows):
            surf.append(oracle_lib.voxelgrid(np.ascontiguousarray(cloud[lf_rows]), 0.6))
    surf = np.concatenate(surf) if surf else np.zeros(0, cloud.dtype)
    return curv, label, np.ascontiguousarray(cloud[np.array(edge_rows, np.int64)]), surf, picks
