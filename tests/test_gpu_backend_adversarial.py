"""GPU tier of the backend's adversarial keyframe maps (tests/bk_adversarial.py): k_backend_edge and k_backend_surf against the
oracle bit for bit, through the single-keyframe calls and through a full 16-keyframe window, and k_backend_block's 29 sums against
a long-double restatement of the rows within an error bound derived from the rows themselves.

The one allowance: the reflectivity variant's score is lidar_const * (weight + exp(-sum_w)), and CUDA's fp64 exp is documented
to within 1 ulp while glibc's may round the other way.  One ulp of exp moves weight + exp(-sum_w) by at most one ulp, and the
product with lidar_const (20) then by at most 1.25 ulp before rounding, so that score may differ from the oracle's by up to two
ulps.  Every other output (flags, line ends, planes, the other scores) must be the same bits."""
import numpy as np
import pytest

import bk_adversarial as BK

pytestmark = pytest.mark.gpu

IDENT = np.array([1.0, 0, 0, 0, 0, 0, 0])
K_WIN = 16            # kWinMax
BIG_SLOT = 9          # a keyframe with more than 64 * 256 surf rows: k_backend_block's grid-stride loop
NO_EDGE = (3, 7)      # keyframes without edge rows between non-empty ones (bkw_find crosses empty segments)
NO_SURF = (5, 11)


def _b(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def _score_ok(sc, sc_o, refl):
    if not refl:
        return _b(sc) == _b(sc_o)
    return bool(np.all(np.abs(sc - sc_o) <= 2 * np.spacing(np.abs(sc_o))))


def _oracle_edge(oracle, W, q, variant):
    return oracle.correspond_edge(oracle.KdTree(W["edge_map"]), q, W["pose"], variant)


def _oracle_surf(oracle, W, q, variant, kd):
    extra = dict(map_refl=W["surf_map"]["curvature"], feat_refl=q["curvature"], reflect_thres=BK.REFLECT_THRES) if variant == 0 else {}
    return oracle.correspond_surf_backend(oracle.KdTree(BK.f4(W["surf_map"])), q, W["pose"], kd, BK.SURF_DIST_THRES,
                                          BK.W_GATE[variant], BK.LIDAR_CONST[variant], **extra)


def _surf_call(c, q, pose, variant, kd):
    if variant == 0:
        return c.correspond_surf_refl(q, pose, kd, BK.SURF_DIST_THRES, BK.W_GATE[0], BK.LIDAR_CONST[0], BK.REFLECT_THRES)
    return c.correspond_surf(q, pose, kd, BK.SURF_DIST_THRES, BK.W_GATE[1], BK.LIDAR_CONST[1])


# ---------------------------------------------------------------- the rows of k_backend_block, restated in long double
LD = np.longdouble


def _qrot(q, v):
    w = LD(q[0]); qv = np.array(q[1:], LD)
    uv = 2 * np.cross(np.broadcast_to(qv, v.shape), v)
    return v + w * uv + np.cross(np.broadcast_to(qv, v.shape), uv)


def _rows_edge(feats, valid, pa, pb, s_weight, pose):
    sel = valid.astype(bool)
    p = np.stack([feats["x"], feats["y"], feats["z"]], 1)[sel].astype(LD)
    A, B = pa[sel].astype(LD), pb[sel].astype(LD)
    rp = _qrot(np.asarray(pose[:4], LD), p)
    lp = rp + np.asarray(pose[4:], LD)
    u, v = lp - A, lp - B
    nu = np.cross(u, v); de = A - B
    nn = np.sqrt((nu * nu).sum(1)); dn = np.sqrt((de * de).sum(1))
    s = LD(s_weight)
    r = nn / dn * s
    with np.errstate(divide="ignore", invalid="ignore"):
        g = np.where((nn > 0)[:, None], (s / (dn * nn))[:, None] * np.cross(de, nu), LD(0))
        nl = lambda x: np.sqrt((x * x).sum(1))
        # the rounding of lp (relative to u = lp - a, v = lp - b) is amplified again by the cancellation of u x v: the factors multiply
        kappa = ((nl(lp) + nl(A)) / nl(u) + (nl(lp) + nl(B)) / nl(v)) * (1 + nl(u) * nl(v) / nn) + (nl(A) + nl(B)) / dn
    # a cross product that cancels to (nearly) nothing leaves g's direction to rounding: such a row is only known to have
    # |g| <= s (kappa = inf marks it; _fold bounds it by its largest possible terms)
    kappa = np.where(np.isfinite(kappa) & (kappa < LD(2.0) ** 40), kappa, LD(np.inf))
    g_max = np.full(len(r), s)
    return rp, g, r, kappa, g_max


def _rows_surf(feats, valid, plane, score, pose, q_lb, t_lb):
    sel = valid.astype(bool)
    p = np.stack([feats["x"], feats["y"], feats["z"]], 1)[sel].astype(LD)
    q_lb = np.asarray(q_lb, LD)
    qi = np.array([q_lb[0], -q_lb[1], -q_lb[2], -q_lb[3]]) / (q_lb * q_lb).sum()
    pr = _qrot(qi, p - np.asarray(t_lb, LD))
    rp = _qrot(np.asarray(pose[:4], LD), pr)
    pw = rp + np.asarray(pose[4:], LD)
    pl = plane[sel].astype(LD); sc = score[sel].astype(LD)
    dot = (pl[:, :3] * pw).sum(1) + pl[:, 3]
    r = sc * dot
    g = sc[:, None] * pl[:, :3]
    with np.errstate(divide="ignore", invalid="ignore"):
        kappa = (np.abs(pl[:, :3] * pw).sum(1) + np.abs(pl[:, 3])) / np.abs(dot)
    kappa = np.where(np.isfinite(kappa), kappa, LD(0))
    return rp, g, r, kappa, np.zeros(len(r), LD)


def _terms(J, r, cauchy_b):
    b2 = LD(cauchy_b) ** 2
    ssum = 1 + r * r / b2
    rho0 = b2 * np.log(ssum)
    sr = np.sqrt(np.maximum(LD(np.finfo(np.float64).tiny), 1 / ssum))      # Ceres' max(DBL_MIN, rho')
    J = J * sr[:, None]; r = r * sr
    terms = [J[:, i] * J[:, j] for i in range(6) for j in range(i, 6)] + [J[:, i] * r for i in range(6)] + [rho0 / 2]
    return np.stack(terms, 1) if len(r) else np.zeros((0, 28), LD)


def _fold(rp, g, r, kappa, g_max, cauchy_b):
    """(sums, bound): the 29 sums of the Cauchy-corrected rows and, per sum, the error bound
       2^-53 * (4 (n + 10) sum_i |t_i| + 256 sum_i kappa_i |t_i|)  (+ 8 n b^2 2^-53 for the cost),
    n rows folded in some order, kappa_i the cancellation of the row's own evaluation (0 for an exactly evaluated row); a row
    whose g is left to rounding (kappa = inf) adds its largest possible terms, |g| = g_max, instead"""
    n = len(r)
    ill = ~np.isfinite(kappa)
    T = _terms(np.concatenate([g, 2 * np.cross(rp, g)], 1), r, cauchy_b)
    eps = LD(2.0) ** -53
    sums = np.concatenate([T.sum(0), [LD(n)]])
    k = np.where(ill, LD(0), kappa)
    # per Jacobian entry: the row's own cancellation, plus that of the difference in each component of rp x g
    a = np.abs(np.stack([rp[:, 1] * g[:, 2], rp[:, 2] * g[:, 0], rp[:, 0] * g[:, 1]], 1))
    b = np.abs(np.stack([rp[:, 2] * g[:, 1], rp[:, 0] * g[:, 2], rp[:, 1] * g[:, 0]], 1))
    with np.errstate(divide="ignore", invalid="ignore"):
        kx = np.where(a + b > 0, (a + b) / np.abs(a - b), LD(0))
    kx = np.where(np.isfinite(kx), kx, LD(0))
    kJ = np.concatenate([np.repeat(k[:, None], 3, 1), k[:, None] + kx], 1)
    kT = np.stack([kJ[:, i] + kJ[:, j] for i in range(6) for j in range(i, 6)] + [kJ[:, i] + k for i in range(6)] + [k], 1) \
        if n else np.zeros((0, 28), LD)
    bound = eps * (4 * (n + 10) * np.abs(T).sum(0) + 256 * (kT * np.abs(T)).sum(0))
    if ill.any():
        rpn = np.sqrt((rp[ill] * rp[ill]).sum(1))
        Jmax = np.stack([g_max[ill]] * 3 + [2 * rpn * g_max[ill]] * 3, 1)
        bound += np.abs(_terms(Jmax, np.abs(r[ill]) + g_max[ill], cauchy_b)).sum(0)
    bound[27] += 8 * n * eps * LD(cauchy_b) ** 2
    return sums, np.concatenate([bound, [LD(0)]])


def _check_block(got, sums, bound, what):
    assert got[28] == sums[28], what
    err = np.abs(got[:28].astype(LD) - sums[:28])
    assert (err <= bound[:28]).all(), (what, np.nonzero(err > bound[:28])[0], err, bound)


def _bodies(W):
    """the lidar pose, a pose with an exact rotation (180-degree yaw, dyadic t: rows of queries on their line stay exactly zero),
    and the lidar pose moved by ~4e4 m (residuals ~1e6, Cauchy weights ~1e-12)"""
    far = W["pose"].copy(); far[4:] += (3.0e4, -2.0e4, 1.0e4)
    return [W["pose"], np.array([0.0, 0, 0, 1.0, 3.25, -1.5, 0.75]), far]


Q_LB = np.array([0.9990482, 0.0, 0.0436194, 0.0]); T_LB = np.array([0.05, -0.02, 0.10])


# ---------------------------------------------------------------- single-keyframe calls
@pytest.mark.parametrize("world", BK.WORLDS)
def test_single_keyframe_calls_bit_for_bit(oracle, world):
    import liliom_b200 as L
    W = BK.backend_world(world)
    c = L.Context(variant=0)
    c.map_set_cloud(W["edge_map48"])
    eq = W["edge_q"]
    for variant in (0, 1):
        v, pa, pb = c.correspond_edge(eq, W["pose"], variant)
        v_o, pa_o, pb_o = _oracle_edge(oracle, W, eq, variant)
        bad = np.nonzero((v != v_o) | (pa != pa_o).any(1) | (pb != pb_o).any(1))[0]
        assert len(bad) == 0, (world, variant, {k: np.intersect1d(ix, bad).tolist() for k, ix in W["edge_notes"].items()})
        assert set(v.tolist()) == {0, 1}
        for k, body in enumerate(_bodies(W)):
            got = c.backend_edge_block(body, 0.6, 1.0)
            _check_block(got, *_fold(*_rows_edge(eq, v, pa, pb, 0.6, body), 1.0), (world, variant, "edge", k))
        # the queries exactly on their line have a zero row at the exact pose: r = 0, J = 0, rho = 0, count 1
        if world == "near":
            ix = W["edge_notes"]["collinear_axis"]
            c.correspond_edge(eq[ix], W["pose"], variant)
            got = c.backend_edge_block(_bodies(W)[1], 0.6, 1.0)
            assert got[28] == len(ix) and not got[:28].any(), got
    c.map_set_cloud(W["surf_map"])
    sq = W["surf_q"]
    for variant in (0, 1):
        for kd in BK.KD_RADII:
            v, pl, sc = _surf_call(c, sq, W["pose"], variant, kd)
            v_o, pl_o, sc_o = _oracle_surf(oracle, W, sq, variant, kd)
            bad = np.nonzero((v != v_o) | (pl.view(np.uint32) != pl_o.view(np.uint32)).any(1))[0]
            assert len(bad) == 0, (world, variant, kd, {k: np.intersect1d(ix, bad).tolist() for k, ix in W["surf_notes"].items()})
            assert _score_ok(sc, sc_o, variant == 0), (world, variant, kd, np.nonzero(sc != sc_o))
            for k, body in enumerate(_bodies(W)):
                got = c.backend_surf_block(body, Q_LB, T_LB, 1.0)
                _check_block(got, *_fold(*_rows_surf(sq, v, pl, sc, body, Q_LB, T_LB), 1.0), (world, variant, kd, "surf", k))
    c.close()


# ---------------------------------------------------------------- the window path
def _window_layout(W):
    """the adversarial queries spread round-robin over 16 keyframes: two without edge rows, two without surf rows, and one with
    every surf query repeated past 64 * 256 rows"""
    eq, sq = W["edge_q"], W["surf_q"]
    e_slots = [s for s in range(K_WIN) if s not in NO_EDGE]
    s_slots = [s for s in range(K_WIN) if s not in NO_SURF and s != BIG_SLOT]
    edge = [eq[np.arange(len(eq))[i::len(e_slots)]] if s in e_slots else eq[:0] for s in range(K_WIN)
            for i in [e_slots.index(s) if s in e_slots else 0]]
    surf = []
    for s in range(K_WIN):
        if s == BIG_SLOT:
            surf.append(np.tile(sq, 64 * 256 // len(sq) + 2))
        elif s in s_slots:
            surf.append(sq[np.arange(len(sq))[s_slots.index(s)::len(s_slots)]])
        else:
            surf.append(sq[:0])
    return edge, surf


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("world", BK.WORLDS)
def test_window_equals_single_calls_and_oracle(oracle, world, variant):
    import liliom_b200 as L
    W = BK.backend_world(world)
    bp = L.backend_default_params(variant)
    # PCL declines a VoxelGrid whose voxel count (an int64 product) exceeds INT_MAX: the clouds pass unchanged.  1 mm leaves do
    # that for every cloud here without overflowing the int64 product itself
    bp.edge_leaf = bp.surf_leaf = 1e-3
    bp.reflect_thres = BK.REFLECT_THRES
    assert (bp.surf_dist_thres, bp.w_gate, bp.lidar_const, bp.kd_max_radius) == \
        (BK.SURF_DIST_THRES, BK.W_GATE[variant], BK.LIDAR_CONST[variant], 1.0)
    c = L.Context(variant=0)
    kid, eds, sds = c.kf_add(bp, W["edge_map48"], W["surf_map"])
    assert _b(eds) == _b(W["edge_map48"]) and _b(sds) == _b(W["surf_map"])
    edge, surf = _window_layout(W)
    assert len(surf[BIG_SLOT]) > 64 * 256
    ids = []
    for e, s in zip(edge, surf):
        kid, eds, sds = c.kf_add(bp, e, s)
        assert _b(eds) == _b(e) and _b(sds) == _b(s), kid
        ids.append(kid)
    c.bmap_build(bp, [0], [IDENT])
    assert _b(c.bmap_download(0)) == _b(W["edge_map48"]) and _b(c.bmap_download(1)) == _b(W["surf_map"])
    poses = [W["pose"]] * K_WIN
    ne, ns = c.backend_window_correspond(bp, ids, poses)
    single = L.Context(variant=0)
    n_big = 0
    for slot in range(K_WIN):
        v, pa, pb = c.backend_window_corr(slot, 0)
        assert len(v) == len(edge[slot]) and int(v.sum()) == ne[slot]
        single.map_set_cloud(W["edge_map48"])
        v1, pa1, pb1 = single.correspond_edge(edge[slot], W["pose"], variant)
        v_o, pa_o, pb_o = _oracle_edge(oracle, W, edge[slot], variant)
        assert _b(v) == _b(v1) == _b(v_o) and _b(pa) == _b(pa1) == _b(pa_o) and _b(pb) == _b(pb1) == _b(pb_o), slot
        vs, pl, sc = c.backend_window_corr(slot, 1)
        assert len(vs) == len(surf[slot]) and int(vs.sum()) == ns[slot]
        single.map_set_cloud(W["surf_map"])
        vs1, pl1, sc1 = _surf_call(single, surf[slot], W["pose"], variant, 1.0)
        vs_o, pl_o, sc_o = _oracle_surf(oracle, W, surf[slot], variant, 1.0)
        assert _b(vs) == _b(vs1) == _b(vs_o) and _b(pl) == _b(pl1) == _b(pl_o) and _b(sc) == _b(sc1), slot
        assert _score_ok(sc, sc_o, variant == 0), slot
        n_big += slot == BIG_SLOT and ns[slot] > 64 * 256 // 2
    assert n_big == 1 and (ne[list(NO_EDGE)] == 0).all() and (ns[list(NO_SURF)] == 0).all()
    # the blocks: against the single-keyframe calls bit for bit and against the long-double rows within the bound
    qlb, tlb = np.array(bp.q_lb[:]), np.array(bp.t_lb[:])
    for k, body in enumerate(_bodies(W)):
        got = c.backend_window_blocks([body] * K_WIN)
        for slot in range(K_WIN):
            v, pa, pb = c.backend_window_corr(slot, 0)
            sw = float(np.float32(np.float32(np.float32(bp.lidar_const) * np.float32(200)) / np.float32(ne[slot]))) \
                if variant == 1 else float(np.float32(bp.lidar_const))
            _check_block(got[slot, 0], *_fold(*_rows_edge(edge[slot], v, pa, pb, sw, body), bp.cauchy_b), (world, variant, k, slot, 0))
            vs, pl, sc = c.backend_window_corr(slot, 1)
            scw = sc * 1000.0 / np.float64(ns[slot]) if variant == 1 else sc
            _check_block(got[slot, 1], *_fold(*_rows_surf(surf[slot], vs, pl, scw, body, qlb, tlb), bp.cauchy_b),
                         (world, variant, k, slot, 1))
            if slot in (0, BIG_SLOT, NO_EDGE[0]):
                single.map_set_cloud(W["edge_map48"])
                single.correspond_edge(edge[slot], W["pose"], variant)
                assert _b(single.backend_edge_block(body, sw, bp.cauchy_b)) == _b(got[slot, 0]), slot
                if variant == 0:
                    single.map_set_cloud(W["surf_map"])
                    _surf_call(single, surf[slot], W["pose"], 0, 1.0)
                    assert _b(single.backend_surf_block(body, qlb, tlb, bp.cauchy_b)) == _b(got[slot, 1]), slot
    single.close()
    c.close()
