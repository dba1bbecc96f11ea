"""TEST INFRASTRUCTURE: a plain reference of the loop-closure ICP (liliom_b200/csrc/icp.cu) and an adversarial world to run it on.

reference_nn1 is the 1-NN k_icp_persistent must find, written without the cell grid: candidates come from a kd-tree in fp64 (the
nearest point, then a ball slightly wider than its distance), they are ranked by the kernel's key (fp32 distance bits << 32 |
target index), and a match is kept when (double)d <= max_corr^2 (PCL's determineCorrespondences).  icp_trace runs PCL's loop pass
by pass on it, with the kernel's own arithmetic from the host build of icp_math.h (tests/icp_math_host.cpp): im_transform (the
contracted source transform), im_sums (the kernel's reduction order) and im_step (SVD, Umeyama, composition, convergence).  The
CPU tier checks both against brute force and NumPy; the GPU tier checks the device against the trace bit for bit."""
import ctypes as C

import numpy as np
from scipy.spatial import cKDTree

import host_build
from knn_reference import _point_at, fp32_sqdist

F32 = np.float32
GO, CONVERGED, STUCK = 0, 1, 2
DBL_MAX = float(np.finfo(np.float64).max)
MAX_CORRS = (0.3, 1.0, 1.7, 30.0)
# the criterion that ended the loop (DefaultConvergenceCriteria's order, then icp.hpp's "fewer than 3 correspondences")
CAP, ROT_TRANS, REL_MSE, ABS_MSE, STUCK_END = "cap", "rotation+translation", "relative mse", "absolute mse", "stuck"

_lib = None


def host_lib():
    """tests/icp_math_host.cpp built for the host (-ffp-contract=off), rebuilt when it or a header it includes is newer"""
    global _lib
    if _lib is not None:
        return _lib
    L = host_build.load("icp_math_host", ["tests/icp_math_host.cpp"], ["-O2", "-std=c++17", "-fPIC", "-Wall", "-ffp-contract=off"],
                        deps=[f"liliom_b200/csrc/{h}" for h in ("icp_math.h", "pcl_xform.h", "vg_box.h")])
    dp = np.ctypeslib.ndpointer(np.float64, flags="C")
    fp = np.ctypeslib.ndpointer(np.float32, flags="C")
    ip = np.ctypeslib.ndpointer(np.int32, flags="C")
    L.im_svd3.argtypes = [dp, dp, dp, dp]
    L.im_det3.argtypes = [dp]
    L.im_det3.restype = C.c_double
    L.im_umeyama.argtypes = [dp, dp, dp]
    L.im_converged.argtypes = [C.c_int, C.c_int, dp, dp, C.c_double, C.c_double, C.c_double, C.c_double]
    L.im_step.argtypes = [dp, C.POINTER(C.c_double), C.POINTER(C.c_int), dp, C.c_int, C.c_double, C.c_double]
    L.im_icp.argtypes = [fp, C.c_int, fp, C.c_int, C.c_double, C.c_int, C.c_double, C.c_double, dp, C.POINTER(C.c_double),
                         C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.im_transform.argtypes = [dp, fp, C.c_int, dp, fp]
    L.im_sums.argtypes = [dp, fp, ip, fp, C.c_int, dp]
    _lib = L
    return L


def as_f4(pts):
    """n x 4 float32 (w = 1) from n x 3 or n x 4 coordinates"""
    pts = np.asarray(pts)
    out = np.ones((len(pts), 4), F32)
    out[:, :3] = pts[:, :3]
    return out


def im_transform(F, src):
    """the kernel's transform of src (n x 4 floats) under F: (px fp64 n x 3, sx fp32 n x 3)"""
    src = np.ascontiguousarray(src, F32)
    px = np.zeros((len(src), 3)); sx = np.zeros((len(src), 3), F32)
    host_lib().im_transform(np.ascontiguousarray(F, np.float64), src, len(src), px, sx)
    return px, sx


def im_sums(px, tgt, nn_idx, nn_d):
    """the 17 sums of one pass in the kernel's reduction order; nn_idx < 0: no correspondence"""
    s = np.zeros(17)
    host_lib().im_sums(np.ascontiguousarray(px, np.float64), np.ascontiguousarray(tgt, F32), np.ascontiguousarray(nn_idx, np.int32),
                       np.ascontiguousarray(nn_d, F32), len(px), s)
    return s


def reference_nn1(sx, tgt, max_corr=None):
    """(idx int32, d fp32, key uint64) of every query's nearest target point in the kernel's ranking: the smallest key
    bits(fp32 distance) << 32 | target index.  With max_corr, a match is kept iff (double)d <= max_corr^2 (idx -1 otherwise; d and
    key still name the nearest point)."""
    q = np.ascontiguousarray(np.asarray(sx, F32)[:, :3])
    p = np.ascontiguousarray(np.asarray(tgt, F32)[:, :3])
    n, k = len(q), min(8, len(p))
    tree = cKDTree(p.astype(np.float64))
    dk, ik = tree.query(q.astype(np.float64), k=k)
    dk, ik = dk.reshape(n, k), ik.reshape(n, k)
    # fp32 rounding moves a squared distance by a few 1e-7 relative: every point whose fp32 distance can tie or beat the nearest's
    # lies in this ball
    r = dk[:, 0] * (1.0 + 1e-5) + 1e-6
    qi = np.repeat(np.arange(n), k)[(dk <= r[:, None]).ravel()]
    pi = ik[dk <= r[:, None]]
    more = np.nonzero(dk[:, -1] <= r)[0] if k < len(p) else np.zeros(0, np.int64)
    if len(more):                                   # the k-NN list may have cut the ball short: take the whole ball
        lists = tree.query_ball_point(q[more].astype(np.float64), r[more])
        keep = ~np.isin(qi, more)
        qi = np.concatenate([qi[keep], np.repeat(more, [len(c) for c in lists])])
        pi = np.concatenate([pi[keep], np.fromiter((j for c in lists for j in c), np.int64)])
    d = fp32_sqdist(q[qi], p[pi])
    keys = (d.view(np.uint32).astype(np.uint64) << np.uint64(32)) | pi.astype(np.uint64)
    best = np.full(n, np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64)
    np.minimum.at(best, qi, keys)
    idx = (best & np.uint64(0xFFFFFFFF)).astype(np.int32)
    dist = (best >> np.uint64(32)).astype(np.uint32).view(F32)
    if max_corr is not None:
        idx = np.where(dist.astype(np.float64) <= float(max_corr) * float(max_corr), idx, -1).astype(np.int32)
    return idx, dist, best


def _criterion(st_it, max_iter, s, prev, trans_eps, fit_eps):
    """which rule of DefaultConvergenceCriteria ended the loop after a step from sums s (the first that holds, in PCL's order)"""
    R, t = np.zeros(9), np.zeros(3)
    host_lib().im_umeyama(s, R, t)
    R = R.reshape(3, 3)
    mse = s[15] / s[16]
    if st_it >= max_iter:
        return CAP
    if 0.5 * (((R[0, 0] + R[1, 1]) + R[2, 2]) - 1.0) >= 1.0 - trans_eps and (t[0] * t[0] + t[1] * t[1]) + t[2] * t[2] <= trans_eps:
        return ROT_TRANS
    if abs(mse - prev) / prev < fit_eps:
        return REL_MSE
    assert abs(mse - prev) < 1e-12
    return ABS_MSE


def icp_trace(src, tgt, max_corr=30.0, max_iter=100, trans_eps=1e-6, fit_eps=1e-6, transform=im_transform, nn=reference_nn1,
              sums=im_sums, fitness_nn=None):
    """PCL's loop pass by pass with the kernel's arithmetic.  Returns a dict: passes (per pass: F after it, the 17 sums, n_corr, mse,
    the correspondence index per source point), end (the criterion that ended the loop), T, fitness (over every source point),
    converged, iters.  transform / nn / sums / fitness_nn replace a stage (the CPU tier plants faults through them)."""
    src = as_f4(src); tgt = as_f4(tgt)
    lib = host_lib()
    F = np.ascontiguousarray(np.eye(4))
    prev, it = C.c_double(DBL_MAX), C.c_int(0)
    passes, end, verdict = [], None, STUCK
    if len(src) == 0 or len(tgt) == 0:
        return dict(passes=passes, end=None, T=F, fitness=0.0, converged=False, iters=0)
    while True:
        px, sx = transform(F, src)
        idx, d, _ = nn(sx, tgt, max_corr)
        s = sums(px, tgt, idx, d)
        prev_before = prev.value
        verdict = lib.im_step(F, C.byref(prev), C.byref(it), s, max_iter, trans_eps, fit_eps)
        passes.append(dict(F=F.copy(), sums=s, n_corr=int((idx >= 0).sum()), mse=s[15] / s[16] if s[16] > 0 else None, idx=idx))
        if verdict == STUCK:
            end = STUCK_END
            break
        if verdict == CONVERGED:
            end = _criterion(it.value, max_iter, s, prev_before, trans_eps, fit_eps)
            break
    px, sx = transform(F, src)
    idx, d, _ = (fitness_nn or nn)(sx, tgt, None)
    s = sums(px, tgt, idx, d)
    fitness = s[15] / s[16] if s[16] > 0 else DBL_MAX
    return dict(passes=passes, end=end, T=F.copy(), fitness=fitness, converged=verdict == CONVERGED, iters=it.value)


def grid_of(tgt, cell):
    """the target's cell grid as grid_build lays it out: (org, dim) per axis"""
    p = np.asarray(tgt, F32)[:, :3]
    inv = F32(1.0 / cell)
    org = np.floor(p.min(0) * inv).astype(np.int64)
    dim = np.floor(p.max(0) * inv).astype(np.int64) - org + 1
    return org, dim


def _rot(axis, ang):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def _transform_splitting_point(F, row, near, rng):
    """a float point near `near` whose row `row` under F lands so close to 0 that the contracted (kernel) and the uncontracted
    (source-order) transform round to different fp32 values: solve the row for its own coordinate, then search the neighbouring floats of all
    three coordinates"""
    c0s = np.asarray(near, F32).copy()
    others = [a for a in range(3) if a != row]
    c0s[row] = F32(-(sum(F[row, a] * float(c0s[a]) for a in others) + F[row, 3]) / F[row, row])
    axes = []
    for c0 in c0s:
        vals = [c0]; u = v = c0
        for _ in range(20):
            u = np.nextafter(u, F32(np.inf)); v = np.nextafter(v, F32(-np.inf))
            vals += [u, v]
        axes.append(np.array(vals, F32))
    X, Y, Z = np.meshgrid(*axes, indexing="ij")
    cand = as_f4(np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1))
    _, sx = im_transform(F, cand)
    c = cand[:, :3].astype(np.float64)
    plain = (((F[:3, 0] * c[:, :1] + F[:3, 1] * c[:, 1:2]) + F[:3, 2] * c[:, 2:3]) + F[:3, 3]).astype(F32)
    hit = np.nonzero(plain[:, row] != sx[:, row])[0]
    return None if len(hit) == 0 else cand[hit[rng.integers(len(hit))], :3]


def adversarial_icp_world(seed=0, cell=1.0, offset=(0.0, 0.0, 0.0)):
    """A target (m x 4) and a source (n x 4) where the shell walk, the cut or the reduction shows any off-by-one, for cells of
    `cell` metres (1.0 and 2.0: knn_max_sqdist 1.0 and 4.0).  Returns (src, tgt, notes); notes names index ranges of the source
    and the gate pairs.  `offset` moves the whole world (e.g. to (5000, -3000, 20) m, where an fp32 step is 0.5 mm)."""
    rng = np.random.default_rng(seed)
    off = np.asarray(offset, np.float64)
    tparts, sparts, notes = [], [], {}

    def add_s(name, pts):
        pts = np.asarray(pts, F32).reshape(-1, 3)
        s0 = sum(len(x) for x in sparts)
        sparts.append(pts)
        notes[name] = (s0, s0 + len(pts))

    # a room with negative coordinates: a floor, two walls, a pole, plus clutter; some points on cell corners and faces
    lo, ext = np.array([-12.0, -9.0, -3.0]), np.array([24.0, 18.0, 6.0])
    n = 700
    room = np.concatenate([
        np.c_[rng.uniform(lo[0], lo[0] + ext[0], n), rng.uniform(lo[1], lo[1] + ext[1], n), np.full(n, lo[2])],
        np.c_[np.full(n, 9.5), rng.uniform(lo[1], lo[1] + ext[1], n), rng.uniform(lo[2], lo[2] + ext[2], n)],
        np.c_[rng.uniform(lo[0], lo[0] + ext[0], n), np.full(n, -7.25), rng.uniform(lo[2], lo[2] + ext[2], n)],
        np.c_[np.full(n // 4, -3.0) + rng.normal(0, 0.05, n // 4), np.full(n // 4, 2.0), rng.uniform(lo[2], 2.0, n // 4)],
        lo + rng.uniform(0, 1, (n, 3)) * ext])
    k8, k6 = len(room) // 8, len(room) // 6
    room[:k8] = np.round(room[:k8] / cell) * cell                                # cell corners
    room[k8:k6, :2] = np.round(room[k8:k6, :2] / cell) * cell                    # cell edges / faces
    room = room + off
    tparts.append(room)
    # the source: most of the room seen from a frame off by 1.5 deg / (0.12, -0.08, 0.03) m, with 5 mm noise
    R0, t0 = _rot([0.2, -0.1, 1.0], np.deg2rad(1.5)), np.array([0.12, -0.08, 0.03])
    pick = rng.permutation(len(room))[:1800]
    add_s("room", (room[pick] - off - t0) @ R0 + off + rng.normal(0, 0.005, (1800, 3)))
    add_s("corners", np.round((lo + rng.uniform(0, 1, (80, 3)) * ext) / cell) * cell + off)
    # duplicates (index ties at distance 0 and beyond) and an equidistant 0.25 m lattice with queries at its cube centres
    dup = np.array([4.3, -2.6, 0.7]) + off
    tparts.append(np.repeat(dup[None], 5, 0))
    add_s("duplicates", np.concatenate([dup[None], dup + rng.uniform(-0.2, 0.2, (10, 3))]))
    lat = np.stack(np.meshgrid(np.arange(-2, 3), np.arange(-2, 3), np.arange(-1, 2), indexing="ij"), -1).reshape(-1, 3) * 0.25
    lat_o = np.array([-6.0, 5.0, 1.0]) + off
    tparts.append(lat + lat_o)
    add_s("lattice", lat[:30] + lat_o + 0.125)
    # a clump of 60 points inside one cell
    clump = (np.floor(np.array([2.3, 6.1, -1.2]) / cell) * cell) + off
    tparts.append(clump + rng.uniform(0.05, 0.95, (60, 3)) * cell)
    add_s("clump", clump + rng.uniform(-0.3, 1.3, (30, 3)) * cell)
    # isolated pairs 4 m apart beyond the room's +x wall: a source point whose only near target point lies at exactly
    # fp32(max_corr^2) (PCL rejects it: max_corr^2 rounds up) or one float below it (kept)
    gate = {}
    k = 0
    for mc in (0.3, 1.7):
        t_at = F32(mc * mc)
        assert float(t_at) > mc * mc
        for name, target in (("at", t_at), ("below", np.nextafter(t_at, F32(0)))):
            for _ in range(3):
                q = (np.array([14.0 + 4.0 * (k % 5), -8.0 + 4.0 * (k // 5), 0.5]) + off + rng.uniform(-0.3, 0.3, 3)).astype(F32)
                k += 1
                p = None
                while p is None:
                    d = rng.normal(size=3); d /= np.linalg.norm(d)
                    p = _point_at(q, target, d, rng)
                assert fp32_sqdist(q, p) == target
                tparts.append(p[None].astype(np.float64))
                s0 = sum(len(x) for x in sparts)
                add_s(f"gate{mc}-{name}-{k}", q[None])
                gate.setdefault((mc, name), []).append(s0)
    notes["gate"] = gate
    tgt = as_f4(np.concatenate(tparts))
    # outside the target's box on all six faces: just beyond (0.3, 0.9 m: neighbours across the face) and far (50, 4000 m: beyond
    # the grid's largest dimension)
    bmin, bmax = tgt[:, :3].min(0), tgt[:, :3].max(0)
    outs = []
    for ax in range(3):
        for side, b in ((-1, bmin), (1, bmax)):
            for d in (0.3, 0.9, 50.0, 4000.0):
                q = tgt[rng.integers(len(tgt)), :3].astype(np.float64)
                q[ax] = b[ax] + side * d
                outs.append(q)
    add_s("outside", outs)
    src = as_f4(np.concatenate(sparts))
    # points whose transform rounds differently when contracted, under the final F of each cut: 60 m beyond the room in -y, so no
    # correspondence pass ever matches them (their F does not depend on them), while the fitness pass does
    split = []
    for mc in MAX_CORRS:
        F = icp_trace(src, tgt, mc)["T"]
        for row in (0, 2):
            p = None
            while p is None:
                p = _transform_splitting_point(F, row, off + np.array([rng.uniform(-5, 5), -70.0, rng.uniform(-1, 1)]), rng)
            split.append(p)
    s0 = len(src)
    src = np.concatenate([src, as_f4(np.array(split))])
    notes["split"] = (s0, len(src))
    return src, tgt, notes
