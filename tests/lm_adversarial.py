"""TEST INFRASTRUCTURE: adversarial correspondence sets for the Ceres-faithful LM (grid_knn.cu::lm_solve_body), each built to
drive one branch or stop of the trust-region loop (tests/lm_reference.py).

The site construction of tests/s2m_adversarial.py: every feature sits at its own site, at least 4 m from every other, among
exactly the five map points built for it, so its 5-NN set, its plane and therefore the LM's input are chosen by construction.
Every guess has w > 0 and every world's trace stays clear of w = 0.  Every world is seeded and built in well under a second.

  zero_residual   axis-aligned walls at power-of-two offsets, features on them in +-p pairs, identity guess: |g| near 1e-13
                  (the fitted normals keep 1e-17 off-axis parts), so the gradient test stops the solve before iteration 1,
                  the pose bit-unchanged
  no_corr         the same map, every feature 2 m off its wall: no correspondence, 0 iterations
  gradient        zero_residual from a 2e-8 m translation: one accepted step leaves |g| below 5e-11, the gradient stop after it
  huber           features 0.5 m either side of parallel planes 3 m apart (Huber's outer region, corrected rows the majority)
                  around zero-residual pairs, from the minimum plus 1e-9 m: the parameter-tolerance stop
  rotation        a 0.56 rad rotation error, six features 15-38 m out: rejected steps, decrease_factor doubling, then acceptances
  ordinary        a well-posed noisy world from a small error: with max_num_iter 0, 1, 2 the iteration cap; uncapped it stops on
                  the function tolerance
  parameter_edge  gradient's offset bisected until the first step's length sits on the parameter tolerance: the one world
                  with an open decision, where a device may take either outcome
  single_wall, corridor   one wall, or two parallel walls and a floor, with 1 cm fit noise: weak in J^T J (cond near 1e6),
                  but the damped system the LM solves has cond 70-90, so the normal equations and QR agree to 1e-15 here;
                  the exactly flat planes of test_reanchor_cpu.PLANE_WORLDS are the rank-deficient cases
No world makes the two model_cost_change formulas disagree in sign.  At a step the gradient test let through (|g| > 1e-10)
the model residuals J s are far above u |r| (residuals are below 1 m, Huber-corrected below sqrt(0.1 m)), so the rounding
of -(J s).(r + J s / 2) stays far below its value; the tests report the gap between the formulas instead.
The radius floor and invalid steps are out of reach (lm_reference's docstring says why); no world pretends otherwise."""
import numpy as np

import lm_reference as LR

F = np.float32
OFFS = ((0.0, 0.0), (0.25, 0.0), (0.0, 0.25), (-0.25, 0.125), (0.125, -0.25))


def _quat(axis, ang):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * axis])


def _inplane(n):
    a = np.eye(3)[int(np.argmin(np.abs(n)))]
    e1 = np.cross(n, a); e1 /= np.linalg.norm(e1)
    return e1, np.cross(n, e1)


def _far_enough(sites, p, d=4.0):
    return all(np.linalg.norm(p - s) >= d for s in sites)


def _exact_sites(signs=(1, -1)):
    """(feature, axis) of zero-residual sites: features ON axis-aligned walls whose coordinate is a power of two, in +-p pairs
    (so the rotation rows cancel exactly in the gradient), every site at least 4 m from every other."""
    out, pos = [], []
    for ax in range(3):
        for c in (8.0, 16.0):
            for i in (-1, 1):
                for j in (-1, 1):
                    p = np.zeros(3)
                    p[ax] = c; p[(ax + 1) % 3] = 4.5 * i + (ax + 1); p[(ax + 2) % 3] = 4.5 * j - (ax + 1) * 0.5
                    if _far_enough(pos, p) and _far_enough(pos, -p):
                        for s in signs:
                            pos.append(s * p); out.append((s * p, ax))
    return out


def _exact_world(feature_shift=0.0):
    m, q = [], []
    for p, ax in _exact_sites():
        e = np.eye(3)
        u, v = e[(ax + 1) % 3], e[(ax + 2) % 3]
        m += [p + a * u + b * v for a, b in OFFS]
        q.append(p + feature_shift * np.sign(p[ax]) * e[ax])
    return m, q


def _pack(m, q):
    mm = np.ones((len(m), 4), F); mm[:, :3] = np.asarray(m, np.float64)
    qq = np.ones((len(q), 4), F); qq[:, :3] = np.asarray(q, np.float64)
    assert np.array_equal(mm[:, :3].astype(np.float64), np.asarray(m)), "map not exact in fp32"
    return mm, qq


def zero_residual():
    m, q = _exact_world()
    mm, qq = _pack(m, q)
    return mm, qq, np.array([1.0, 0, 0, 0, 0, 0, 0])


def no_corr():
    m, q = _exact_world(feature_shift=2.0)
    mm, qq = _pack(m, q)
    return mm, qq, np.array([1.0, 0, 0, 0, 0, 0, 0])


def gradient():
    mm, qq, _ = zero_residual()
    return mm, qq, np.array([1.0, 0, 0, 0, 2e-8, -1.5e-8, 1.25e-8])


def huber():
    """Outer pairs: a feature 0.5 m below its plane and one 4 m further along the normal 0.5 m above its own, planes at -2 and
    1 (weighted residuals near 0.2, twice Huber's 0.1); around them the zero-residual pairs of the inner region.  The guess is
    the minimiser plus 1e-9 m."""
    m, q = _exact_world()
    pos = [np.asarray(x) for x in q] + [-np.asarray(x) for x in q]
    e = np.eye(3)
    for ax in range(3):
        u, v = e[(ax + 1) % 3], e[(ax + 2) % 3]
        for i in range(-3, 4):
            for j in range(-3, 4):
                base = (4.0 * i + 0.5 * ax) * u + (4.0 * j - 0.25 * ax) * v
                f1, f2 = base - 2.5 * e[ax], base + 1.5 * e[ax]
                if not (_far_enough(pos, f1) and _far_enough(pos, f2)) or np.abs(base).max() > 14:
                    continue
                pos += [f1, f2]
                for f, c in ((f1, -2.0), (f2, 1.0)):
                    pl = f.copy(); pl[ax] = c
                    m += [pl + a * u + b * v for a, b in OFFS]
                    q.append(f)
    mm, qq = _pack(m, q)
    x = _minimiser(mm, qq, np.array([1.0, 0, 0, 0, 0, 0, 0]))
    return mm, qq, x + np.array([0, 0, 0, 0, 1e-9, 0, 0])


def parameter_edge():
    """zero_residual from a translation along (2, -1.5, 1.25) bisected until the first step's length sits on the parameter
    tolerance 1e-8 (|x| + 1e-8) to within its rounding bound: a genuinely open decision.  Either outcome is admissible: stop
    with the pose kept (parameter), or accept the step and stop on the gradient.  The offsets stay below 3e-8 m, where every
    plane's weight is 1.0f, so the correspondences do not change with the offset and the decision is continuous in it."""
    import oracle_lib as O
    mm, qq, _ = zero_residual()
    tree = O.KdTree(mm)
    d = np.array([2.0, -1.5, 1.25]); d /= np.linalg.norm(d)

    def margin(a):
        g = np.concatenate([[1.0, 0, 0, 0], a * d])
        _, v, pl, _, _ = O.find_surf_corr(tree, qq, g)
        rec = LR.run(qq, v, pl, g, 1)["records"][0]
        return next(x["margin"] for x in rec["decisions"] if x["name"] == "parameter"), g
    lo, hi = 0.5e-8, 2e-8
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        if mid in (lo, hi):
            break
        if margin(mid)[0] > 0:
            hi = mid
        else:
            lo = mid
    return mm, qq, min((margin(lo), margin(hi)), key=lambda t: abs(t[0]))[1]


def _noisy_world(seed, n_sites, rmin, rmax, guess, planes=None, noise=0.0):
    """Sites 4 m apart at ranges [rmin, rmax]; each feature's plane passes through its true position (identity pose) with a
    random normal (or one of `planes`: (n, c) with n.x = c) and its five points are laid on it around the projection of the
    guess-transformed feature, with `noise` m of normal noise."""
    rng = np.random.default_rng(seed)
    G = LR._rotmat(guess[:4])
    m, q, pos = [], [], []
    tries = 0
    while len(q) < n_sites and tries < 200000:
        tries += 1
        if planes is None:
            d = rng.normal(size=3); d /= np.linalg.norm(d)
            f = d * rng.uniform(rmin, rmax)
            n = rng.normal(size=3); n /= np.linalg.norm(n)
            c = n @ f
        else:
            n, c = planes[len(q) % len(planes)]
            n = np.asarray(n, np.float64)
            e1, e2 = _inplane(n)
            f = c * n + rng.uniform(-rmax, rmax) * e1 + rng.uniform(-rmax, rmax) * e2
            if np.linalg.norm(f) < rmin:
                continue
        gw = G @ f + guess[4:]
        rg = n @ gw - c
        if abs(c) < 0.5 or abs(rg) > 0.5 or 0.9 * abs(rg) / np.sqrt(np.linalg.norm(gw)) > 0.45 or not _far_enough(pos, gw):
            continue
        pos.append(gw)
        e1, e2 = _inplane(n)
        ang = rng.uniform(0, 2 * np.pi)
        e1, e2 = np.cos(ang) * e1 + np.sin(ang) * e2, -np.sin(ang) * e1 + np.cos(ang) * e2
        proj = gw - rg * n
        for a, b in OFFS:
            m.append(proj + 1.2 * a * e1 + 1.2 * b * e2 + rng.normal(0, noise) * n if noise else proj + 1.2 * a * e1 + 1.2 * b * e2)
        q.append(f)
    assert len(q) == n_sites
    mm = np.ones((len(m), 4), F); mm[:, :3] = np.asarray(m)
    qq = np.ones((len(q), 4), F); qq[:, :3] = np.asarray(q)
    return mm, qq, np.asarray(guess, np.float64)


def rotation():
    """A 0.56 rad rotation error and 2 m of translation over six features 15-38 m out: the first GN-like steps overshoot."""
    rng = np.random.default_rng(9)
    ang, ax = rng.uniform(0.3, 0.6), rng.normal(size=3)
    tr = rng.normal(size=3) * rng.uniform(0, 2)
    n_sites, rmax = int(rng.integers(6, 40)), rng.uniform(20, 60)
    return _noisy_world(9, n_sites, 15.0, rmax, np.concatenate([_quat(ax, ang), tr]))


def _minimiser(m, q, x, rounds=20):
    """The minimiser of the frozen problem at the correspondences found from it (Newton on the fsum sums; the weight of each
    plane depends on the pose, so repeated until the pose stops moving)."""
    import oracle_lib as O
    tree = O.KdTree(m)
    for _ in range(rounds):
        _, v, pl, _, _ = O.find_surf_corr(tree, q, x)
        xn = LR.minimiser(LR.Problem(q, v, pl), x)
        done = np.abs(xn - x).max() < 1e-13
        x = xn
        if done:
            break
    return x


def ordinary():
    return _noisy_world(8, 80, 4.0, 25.0, np.concatenate([_quat((1.0, 0.4, -0.2), 0.03), [0.12, -0.08, 0.05]]), noise=0.01)


def single_wall():
    return _noisy_world(9, 60, 2.0, 18.0, np.concatenate([_quat((0.2, 1.0, 0.1), 0.02), [0.05, 0.1, -0.03]]),
                        planes=[((1.0, 0.0, 0.0), 6.0)], noise=0.01)


def corridor():
    return _noisy_world(10, 90, 2.0, 24.0, np.concatenate([_quat((0.1, 0.2, 1.0), 0.02), [0.08, -0.05, 0.04]]),
                        planes=[((0.0, 1.0, 0.0), 2.0), ((0.0, 1.0, 0.0), -2.0), ((0.0, 0.0, 1.0), -1.5)], noise=0.01)


# name -> (builder, max_num_iter, what the reference must show: a stop reason, and branches that must occur)
WORLDS = {
    "zero_residual": (zero_residual, 15, "gradient", ()),
    "no_corr": (no_corr, 15, "no_correspondences", ()),
    "gradient": (gradient, 15, "gradient", ("accepted",)),
    "huber": (huber, 15, "parameter", ()),
    "rotation": (rotation, 15, None, ("rejected", "accepted")),
    "ordinary": (ordinary, 15, "function", ("accepted",)),
    "ordinary_cap0": (ordinary, 0, "iteration_cap", ()),
    "ordinary_cap1": (ordinary, 1, "iteration_cap", ("accepted",)),
    "ordinary_cap2": (ordinary, 2, "iteration_cap", ("accepted",)),
    "parameter_edge": (parameter_edge, 15, None, ()),
    "single_wall": (single_wall, 15, None, ("accepted",)),
    "corridor": (corridor, 15, None, ("accepted",)),
}
WEAK = ("single_wall", "corridor")
