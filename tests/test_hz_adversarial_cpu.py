"""CPU tier of the Horizon extractor's adversarial sweeps (tests/hz_adversarial.py): every named case is hit, read from the
oracle's own outputs, and the oracle agrees with a NumPy restatement of L/src/Preprocessing.cpp:225-383 written from the
reference source (test_oracle_cpu.py::test_horizon_extractor_second_restatement's rules, plus the x86 scan-id rule and the
de-skew) on every sweep.  Only a PCA gate within a derived margin of its threshold may be decided differently by numpy's
eigvalsh; such patches are excluded from the comparison and counted."""
import math

import numpy as np
import pytest

import hz_adversarial as H

F = np.float32


@pytest.fixture(scope="module")
def sweeps():
    return H.all_sweeps()


@pytest.fixture(scope="module")
def outputs(oracle, sweeps):
    return {name: oracle.extract_horizon(sw["pts"], sw["q"]) for name, sw in sweeps}


def _cells(cloud):
    """(line, column) of every point of a published cloud, from its intensity"""
    return [(H.scan_id_of(v), H.col_of(v)) for v in cloud["intensity"]]


def _per_patch(cloud):
    out = {}
    for k, c in _cells(cloud):
        out.setdefault(H.patch_of_col(c), []).append((k, c))
    return out


def _deskew_numpy(pts, q):
    """undistortion (:104-127) in NumPy: slerp(Identity -> q) by min(frac / 0.1, 1), Eigen's q * v, not re-normalised"""
    inten = pts["intensity"]
    line = np.array([H.scan_id_of(v) for v in inten], np.int64)
    ratio = np.minimum((inten - line.astype(F)).astype(np.float64) / 0.1, 1.0)
    d = q[0]
    if abs(d) >= 1.0 - H.DBL_EPS:
        s0, s1 = 1.0 - ratio, ratio
    else:
        th = math.acos(abs(d)); sth = math.sin(th)
        s0 = np.sin((1.0 - ratio) * th) / sth; s1 = np.sin(ratio * th) / sth
    if d < 0:
        s1 = -s1
    qs = np.stack([s0 + s1 * q[0], s1 * q[1], s1 * q[2], s1 * q[3]], 1)
    P = np.stack([pts["x"], pts["y"], pts["z"]], 1).astype(np.float64)
    uv = 2.0 * np.cross(qs[:, 1:], P)
    return (P + qs[:, :1] * uv + np.cross(qs[:, 1:], uv)).astype(F)


def _kept_numpy(pts):
    """removeNaN (:225), removeClosedPointCloud (:72-97), scan_id >= 0 with x86's int(float) (:250-253)"""
    fin = np.isfinite(pts["x"]) & np.isfinite(pts["y"]) & np.isfinite(pts["z"])
    r2 = (pts["x"] * pts["x"] + pts["y"] * pts["y"]) + pts["z"] * pts["z"]
    sid = np.array([H.scan_id_of(v) for v in pts["intensity"]], np.int64)
    return fin & ~(r2 < F(0.1) * F(0.1)) & (sid >= 0)


def _gate_margin(A):
    """0 when the scatter matrix is diagonal (its eigenvalues are its diagonal, exactly, in every solver), else a bound well
    above the difference of two backward-stable 3x3 eigen-solvers"""
    if A[1, 0] == 0 and A[2, 0] == 0 and A[2, 1] == 0:
        return 0.0, np.sort(np.diag(A))
    ev = np.linalg.eigvalsh(A)
    return 1e-9 * max(abs(ev).max(), 1e-300), ev


def restate(cut):
    """binning + patch classifier (:238-383) on the oracle's cutted cloud.  Returns (surf cells, edge cells, excluded patches,
    per-patch detail)"""
    T = H.T_INTERVAL
    mat_idx = -np.ones((H.N_SCANS, H.H_SCANS), np.int64)
    dep = ((cut["x"] * cut["x"] + cut["y"] * cut["y"]) + cut["z"] * cut["z"]).astype(np.float64)
    for i, p in enumerate(cut):
        cv = float(p["curvature"])                                  # widened: a float32 compared with 25.45 would round the threshold
        if dep[i] > 40000.0 or dep[i] < 4.0 or cv < 0.05 or cv > 25.45:
            continue
        sid = H.scan_id_of(p["intensity"])
        c = H.col_of(p["intensity"])
        if c is None or c >= H.H_SCANS or c < 0 or sid >= H.N_SCANS:
            continue
        if mat_idx[sid, c] < 0:
            mat_idx[sid, c] = i
    occ = mat_idx >= 0
    sel = np.where(occ, mat_idx, 0)
    xyz = np.where(occ[..., None], np.stack([cut["x"][sel], cut["y"][sel], cut["z"][sel]], -1), F(0)).astype(F)
    curv = np.where(occ, cut["curvature"][sel], F(0)).astype(F)
    depth = np.sqrt((xyz[..., 0] * xyz[..., 0] + xyz[..., 1] * xyz[..., 1]) + xyz[..., 2] * xyz[..., 2]).astype(np.float64)
    X = xyz.astype(np.float64)
    surf, edge, excluded, detail = [], [], [], {}
    for p, i in enumerate(range(5, H.H_SCANS - 12, 6)):
        cells = [(k, i + j) for j in range(6) for k in range(H.N_SCANS) if curv[k, i + j] > 0]
        g1s = {}
        ids = []
        for k in range(H.N_SCANS):
            max_s, idx = 0.0, i
            for j in range(6):
                if curv[k, i + j] <= 0:
                    continue
                d = depth[k]
                g1 = d[i + j - 4] + d[i + j - 3] + d[i + j - 2] + d[i + j - 1] - 8 * d[i + j] + d[i + j + 1] + d[i + j + 2] + d[i + j + 3] + d[i + j + 4]
                g1 = g1 / (8 * d[i + j] + 1e-3)
                g1s[(k, i + j)] = g1
                if g1 > 0.06 and g1 > max_s:
                    max_s, idx = g1, i + j
            if max_s != 0:
                ids.append((k, idx))
        detail[p] = dict(num=len(cells), ids=ids, g1=g1s)
        if len(cells) < 25:
            continue
        P = np.array([X[c] for c in cells]); ctr = P.sum(0) / len(cells)
        A = (P - ctr).T @ (P - ctr)
        m_s, ev = _gate_margin(A)
        detail[p]["scatter"] = A
        skip = m_s > 0 and abs(ev[0] - 0.2 * ev[1]) <= m_s
        emitted = []
        if len(ids) > 0:
            E = np.array([X[c] for c in ids]); ce = E.sum(0) / len(ids)
            m_e, eve = _gate_margin((E - ce).T @ (E - ce))
            if len(ids) > 3:
                skip |= m_e > 0 and abs(eve[2] - 4.0 * eve[1]) <= m_e
                if eve[2] > 4.0 * eve[1]:
                    emitted = [c for c in ids if not (curv[c] <= 0)]
        if skip:
            excluded.append(p)
            continue
        for c in emitted:
            edge.append(c); curv[c] *= -1
        if ev[0] < 0.2 * ev[1]:
            for j in range(6):
                for k in range(H.N_SCANS):
                    if curv[k, i + j] > 0:
                        surf.append((k, i + j)); curv[k, i + j] *= -1
    return surf, edge, excluded, detail


def test_oracle_matches_numpy_restatement_on_adversarial_sweeps(oracle, sweeps, outputs):
    n_excl = n_patches = 0
    for name, sw in sweeps:
        pts, q = sw["pts"], sw["q"]
        surf_o, edge_o, cut_o = outputs[name]
        keep = _kept_numpy(pts)
        kept = pts[keep]
        assert len(cut_o) == keep.sum(), (name, len(cut_o), keep.sum())
        assert cut_o["intensity"].tobytes() == kept["intensity"].tobytes() and cut_o["curvature"].tobytes() == kept["curvature"].tobytes()
        got = np.stack([cut_o["x"], cut_o["y"], cut_o["z"]], 1)
        want = _deskew_numpy(kept, q)
        ulp = np.spacing(np.maximum(np.abs(got), np.abs(want)))
        assert (np.abs(got - want) <= ulp).all(), (name, int((np.abs(got - want) > ulp).sum()))           # numpy's acos / sin
        if abs(q[0]) >= 1.0 - H.DBL_EPS and not q[1:].any():
            assert got.tobytes() == np.stack([kept["x"], kept["y"], kept["z"]], 1).tobytes(), name         # identity: untouched
        surf, edge, excluded, _ = restate(cut_o)
        n_excl += len(excluded); n_patches += H.N_PATCHES
        ex = set(excluded)
        for sel, out in ((surf, surf_o), (edge, edge_o)):
            cells_o = _cells(out)
            keep_o = [H.patch_of_col(c) not in ex for _, c in cells_o]
            assert [c for c in sel if H.patch_of_col(c[1]) not in ex] == [c for c, k in zip(cells_o, keep_o) if k], name
    print(f"patches excluded for a PCA gate within the margin: {n_excl} of {n_patches}")
    assert n_excl <= n_patches // 100


def test_every_patch_case_is_hit(sweeps, outputs):
    for name in ("cells",):                     # q_iMU = identity: the de-skew leaves the placed geometry as it is
        sw = dict(sweeps)[name]
        surf_o, edge_o, cut_o = outputs[name]
        S, E = _per_patch(surf_o), _per_patch(edge_o)
        cases = sw["cases"]
        ns = lambda p: len(S.get(p, []))          # noqa: E731
        ne = lambda p: len(E.get(p, []))          # noqa: E731
        for p in cases["num36"]["patches"]:
            assert ns(p) == 36 and ne(p) == 0, (name, p)
        for p in cases["num25"]["patches"]:
            assert ns(p) == 25, (name, p)
        for p in cases["num24"]["patches"]:
            assert ns(p) == 0 and ne(p) == 0, (name, p)
        for p in cases["edges3"]["patches"] + cases["edges3_hi"]["patches"]:
            assert ne(p) == 0, (name, p)
        for p in cases["edges4"]["patches"] + cases["edges4_hi"]["patches"]:
            assert ne(p) == 4, (name, p)
        for p in cases["edges6"]["patches"] + cases["edges6_hi"]["patches"]:
            assert ne(p) == 6, (name, p)
        # the high word of the flipped mask: an edge at window index >= 64 (line 4 at j >= 4, line 5) in a surf-accepted patch,
        # which the surf list must then skip
        hi = 0
        for p in cases["edges4_hi"]["patches"] + cases["edges6_hi"]["patches"]:
            if ns(p) > 0:
                wi = [k * 14 + (c - H.patch_first_col(p)) + 4 for k, c in E[p]]
                assert not set(E[p]) & set(S[p])
                hi += any(w >= 64 for w in wi)
        assert hi >= 2, (name, hi)
        for p in cases["tie"]["patches"]:
            assert ne(p) == 6, (name, p)
            if name == "cells":                  # un-rotated mirror images: equal g1, and strict '>' keeps the first of the two maxima
                g1 = restate(cut_o)[3][p]["g1"]
                c0 = H.patch_first_col(p)
                assert all(g1[(k, c0)] == g1[(k, c0 + 5)] > 0.06 for k in range(H.N_SCANS))
                assert all(c == c0 for _, c in E[p]), (name, p, E.get(p))
        for nm in ("coincident", "collinear"):
            for p in cases[nm]["patches"]:
                assert ns(p) == 0 and ne(p) == 0, (name, nm, p)
        for p in cases["plane_sym"]["patches"]:
            assert ns(p) == 36, (name, p)
        for nm, case in cases.items():
            if "gate_passes" in case:
                p = case["patches"][0]
                assert ns(p) == (25 if case["gate_passes"] else 0), (name, nm, ns(p))
        # collisions: a cell's returns sit in different block chunks; some first returns are refused by the reflectivity gate
        rows = cases["collisions_rows"]["rows"]
        key = sw["pts"]["intensity"].view(np.uint32)
        spread = [np.nonzero(key == key[r])[0] for r in rows]
        assert len(rows) > 40 and max(len(s) for s in spread) >= 5 and sum(s.max() - s.min() > 2000 for s in spread) > 10
        assert all(ns(p) > 0 for p in cases["collisions"]["patches"])
        # column rounding at the closest floats to a half, on both sides
        halves = cases["col_half"]["halves"]
        assert any(qv < math.floor(qv) + 0.5 for _, qv, _ in halves) and any(qv > math.floor(qv) + 0.5 for _, qv, _ in halves)
        assert all(c == (math.floor(qv) + (1 if qv - math.floor(qv) >= 0.5 else 0)) for _, qv, c in halves)
        half_set = {(k, c) for k, _, c in halves}
        assert len(half_set & set(_cells(surf_o))) >= 4
        # outside every patch: binned, never published
        cut_cols = {c for _, c in _cells(cut_o)}
        assert set(cases["outside_cols"]["cols"]) <= cut_cols and {3999, 4000} <= cut_cols
        for cloud in (surf_o, edge_o):
            assert all(5 <= c <= 3988 for _, c in _cells(cloud))


def test_every_intensity_and_q_case_is_hit(sweeps, outputs):
    branches = {b for _, _, b in H.q_cases()}
    assert branches == {"linear", "acos"}
    assert any(q[0] < 0 for _, q, _ in H.q_cases()) and any(abs(np.linalg.norm(q) - 1) > 0.1 for _, q, _ in H.q_cases())
    e = H.DBL_EPS
    assert any(1 - e <= abs(q[0]) < 1 for _, q, _ in H.q_cases()) and any(1 - 3 * e < abs(q[0]) < 1 - e for _, q, _ in H.q_cases())
    for name, q, _ in H.q_cases():
        sw = dict(sweeps)[name]
        _, _, cut_o = outputs[name]
        inten = sw["pts"]["intensity"]
        cut_i = cut_o["intensity"]
        c = sw["cases"]
        bad = inten[c["intensity_non_finite_or_huge"]["rows"]]
        assert not np.isin(cut_i.view(np.uint32), bad.view(np.uint32)).any()          # dropped as on x86
        for nm in ("intensity_frac_ge_0.1", "intensity_negative", "intensity_scan_id_6_plus"):
            v = inten[c[nm]["rows"]]
            assert np.isin(v.view(np.uint32), cut_i.view(np.uint32)).all(), (name, nm)    # kept, de-skewed
        neg_cols = [H.col_of(v) for v in inten[c["intensity_negative"]["rows"]]]
        assert 0 in neg_cols and any(x < 0 for x in neg_cols)                             # -0.0 rounds into column 0
        assert any(H.col_quotient(v) / 3999.0 > 1.0 for v in inten[c["intensity_frac_ge_0.1"]["rows"]])


def test_livox_messages_cases(oracle):
    msgs = {n: (a, s) for n, a, s in H.livox_messages()}
    q = H.Q_ROT
    res = {n: oracle.extract_horizon(oracle.convert_livox(a, s if s != 20 else None), q) for n, (a, s) in msgs.items()}
    n = len(msgs["normal"][0])
    assert len(res["normal"][2]) == n and len(res["normal"][0]) > 1000
    for nm in ("last_offset_zero", "one_point_offset_zero", "all_offsets_zero"):
        conv = oracle.convert_livox(msgs[nm][0])
        assert not np.isfinite(conv["intensity"]).all()
        assert len(res[nm][2]) == 0 and len(res[nm][0]) == 0, nm                        # NaN / inf scan ids: every point dropped
    beyond = oracle.convert_livox(msgs["offset_beyond_end"][0])
    assert ((beyond["intensity"] - np.floor(beyond["intensity"])) > 0.1).sum() > 100 and len(res["offset_beyond_end"][2]) == n
    lines = res["line_6_255"][2]["intensity"]
    assert (lines >= 6).sum() > 100
    for a, b in zip(res["stride19"], res["normal"]):
        assert a.tobytes() == b.tobytes()
