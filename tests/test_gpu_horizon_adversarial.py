"""The Horizon extractor on the adversarial sweeps (tests/hz_adversarial.py) against the oracle, on both launch chains (the
single cooperative k_hz_coop and the multi-launch chain a device with fewer than 83 SMs takes, forced by LILIOM_HZ_CHAIN=1):
surf and edge clouds field by field and bit for bit; the cutted cloud bit for bit in intensity and curvature and within one fp32
ulp in x, y, z (the slerp's acos / sin are CUDA's fp64 routines, not glibc's; the count of such flips is printed).  Through
extract_horizon (with and without cut_out, cut_cap below and at least n: the early copy and its capacity refusal),
extract_horizon_livox, and the resident upload_scan + extract_resident + odometry_resident(want_ds=True)."""
import ctypes as C

import numpy as np
import pytest

import hz_adversarial as H

pytestmark = pytest.mark.gpu

F_EXACT = ["nx", "ny", "nz", "intensity", "curvature", "x", "y", "z"]
SENTINEL = 0x7F


def _fields_equal(a, b, fields, what):
    assert len(a) == len(b), (what, len(a), len(b))
    for f in fields:
        fa, fb = a[f].view(np.uint32), b[f].view(np.uint32)
        bad = np.nonzero(fa != fb)[0]
        assert len(bad) == 0, f"{what} field {f}: {len(bad)} of {len(a)} differ, first at {bad[:5]}: {a[f][bad[:5]]} vs {b[f][bad[:5]]}"


def _cut_equal(cut, cut_o, what):
    """intensity / curvature bit for bit, x y z within one fp32 ulp; returns the number of coordinates one ulp off"""
    _fields_equal(cut, cut_o, ["intensity", "curvature", "w", "nx", "ny", "nz"], what)
    flips = 0
    for f in ("x", "y", "z"):
        a, b = cut[f], cut_o[f]
        ulp = np.spacing(np.maximum(np.abs(a), np.abs(b)))
        d = np.abs(a.astype(np.float64) - b.astype(np.float64))
        assert (d <= ulp).all(), f"{what} cut {f}: {int((d > ulp).sum())} coordinates more than one ulp off"
        flips += int((a.view(np.uint32) != b.view(np.uint32)).sum())
    return flips


@pytest.fixture(scope="module")
def sweeps():
    return H.all_sweeps()


@pytest.fixture(scope="module")
def oracle_out(oracle, sweeps):
    return {name: oracle.extract_horizon(sw["pts"], sw["q"]) for name, sw in sweeps}


def _ctx(monkeypatch, chain, leaf_scan=None):
    import liliom_b200 as L
    if chain:
        monkeypatch.setenv("LILIOM_HZ_CHAIN", "1")
    else:
        monkeypatch.delenv("LILIOM_HZ_CHAIN", raising=False)
    p = L.default_params(0)
    if leaf_scan is not None:
        p.leaf_scan = leaf_scan
    c = L.Context(p)
    monkeypatch.delenv("LILIOM_HZ_CHAIN", raising=False)
    return c


def _extract(c, pts, q, cut_cap, livox_stride=None):
    """liliom_extract_horizon(_livox) with a cut buffer of cut_cap slots (None: no cut_out).  Returns (rc, surf, edge, cut, raw cut
    buffer)."""
    import liliom_b200 as L
    from liliom_b200._lib import _dptr, _ptr, lib
    n = len(pts) if livox_stride is None else pts.size * pts.dtype.itemsize // livox_stride
    surf = np.empty(max(n, 1), L.PT48); edge = np.empty(max(n, 1), L.PT48)
    cut = None if cut_cap is None else np.full(max(cut_cap, 1) * 48, SENTINEL, np.uint8).view(L.PT48)
    ns, ne, nc = C.c_int(-5), C.c_int(-5), C.c_int(-5)
    qd = np.asarray(q, np.float64)
    args = (_ptr(surf), len(surf), C.byref(ns), _ptr(edge), len(edge), C.byref(ne), _ptr(cut), 0 if cut is None else cut_cap, C.byref(nc))
    if livox_stride is None:
        rc = lib().liliom_extract_horizon(c._h, _ptr(pts), n, _dptr(qd), *args)
    else:
        rc = lib().liliom_extract_horizon_livox(c._h, _ptr(np.ascontiguousarray(pts)), n, livox_stride, _dptr(qd), *args)
    if rc != 0:
        return rc, None, None, None, cut
    return rc, surf[:ns.value], edge[:ne.value], (None if cut is None else cut[:nc.value]), cut


def _check_all_caps(c, pts, q, ref, what, livox_stride=None):
    """the call with cut_cap >= n (early copy), cut_cap == the oracle's count (< n when returns are dropped), cut_cap one short
    (refused: E_CAPACITY, the caller's buffer untouched) and no cut_out"""
    surf_o, edge_o, cut_o = ref
    n = len(pts) if livox_stride is None else pts.size * pts.dtype.itemsize // livox_stride
    flips = 0
    for cap in (n + 3, len(cut_o), None):
        rc, surf, edge, cut, _ = _extract(c, pts, q, cap, livox_stride)
        assert rc == 0, (what, cap, rc)
        _fields_equal(surf, surf_o, F_EXACT, f"{what} cap={cap} surf")
        _fields_equal(edge, edge_o, F_EXACT, f"{what} cap={cap} edge")
        if cap is not None:
            flips += _cut_equal(cut, cut_o, f"{what} cap={cap}")
    if len(cut_o) > 0:
        rc, _, _, _, buf = _extract(c, pts, q, len(cut_o) - 1, livox_stride)
        assert rc == -4, (what, rc)                                                           # LILIOM_E_CAPACITY
        assert (buf.view(np.uint8) == SENTINEL).all(), what
    return flips


@pytest.mark.parametrize("chain", [False, True], ids=["coop", "chain"])
def test_extract_horizon_adversarial(oracle_out, sweeps, monkeypatch, chain):
    c = _ctx(monkeypatch, chain)
    flips = 0
    try:
        for name, sw in sweeps:
            flips += _check_all_caps(c, sw["pts"], sw["q"], oracle_out[name], f"{name}/{'chain' if chain else 'coop'}")
    finally:
        c.close()
    print(f"cut coordinates one fp32 ulp from the oracle's ({'chain' if chain else 'coop'}): {flips}")


@pytest.mark.parametrize("chain", [False, True], ids=["coop", "chain"])
def test_extract_horizon_livox_adversarial(oracle, monkeypatch, chain):
    c = _ctx(monkeypatch, chain)
    q = H.Q_ROT
    flips = 0
    try:
        for name, msg, stride in H.livox_messages():
            ref = oracle.extract_horizon(oracle.convert_livox(msg, None if stride == 20 else stride), q)
            flips += _check_all_caps(c, msg, q, ref, f"livox {name}/{'chain' if chain else 'coop'}", livox_stride=stride)
    finally:
        c.close()
    print(f"livox cut coordinates one fp32 ulp from the oracle's ({'chain' if chain else 'coop'}): {flips}")


@pytest.mark.parametrize("chain", [False, True], ids=["coop", "chain"])
def test_resident_extract_adversarial(oracle, oracle_out, sweeps, monkeypatch, chain):
    """upload_scan + extract_resident + odometry_resident(want_ds=True): with leaf_scan = 0 the queries are the surf cloud itself
    (its count and its points), with the default 0.4 m leaf the down-sampled cloud is the oracle's VoxelGrid of the oracle's surf"""
    import liliom_b200 as L
    ctx = {leaf: _ctx(monkeypatch, chain, leaf) for leaf in (0.0, None)}
    try:
        for name, sw in sweeps:
            surf_o = oracle_out[name][0]
            m = np.ones((len(surf_o), 4), np.float32)
            m[:, 0], m[:, 1], m[:, 2] = surf_o["x"], surf_o["y"], surf_o["z"]
            for leaf, c in ctx.items():
                c.map_set_points(m)
                c.upload_scan(sw["pts"])
                ns, ne, nc = c.extract_resident(sw["q"])
                _, _, ds = c.odometry_resident((1.0, 0, 0, 0, 0, 0, 0), 1, mode=L.MODE_GN, want_ds=True, cap=len(sw["pts"]),
                                               want_stats=False)
                want = surf_o if leaf == 0.0 else oracle.voxelgrid(surf_o, 0.4)
                _fields_equal(ds, want, F_EXACT, f"resident {name} leaf={leaf} {'chain' if chain else 'coop'}")
    finally:
        for c in ctx.values():
            c.close()
