"""The ROT extractor on the adversarial sweeps (tests/rot_adversarial.py) against the oracle, on both walks of k_rot_ring (the
availability-mask walk for segments up to 1024 points and the general walk, forced for every segment by LILIOM_ROT_SLOW_WALK):

  * extract_rot + extract_rot_labels: with an identity de-skew the cut, edge and surf clouds, labels and curvature bit for bit
    (a NaN curvature as NaN); with a general q_iMU the cut within one fp32 ulp in x, y, z (CUDA's fp64 acos / sin are not
    glibc's; the flips are printed) and its intensity exact, and labels, curvature, edge and surf bit for bit against the
    restatement (tests/rot_restate.py) applied to the device's own cut, rings taken from the oracle;
  * caller capacities at the count and one short (E_CAPACITY, sentinel buffers and preset counts untouched);
  * the PointCloud2 `ring` field holding the tables' verdict (LILIOM_RING_FIELD) gives the table path's bytes;
  * the resident upload_scan + extract_resident + odometry_resident(want_ds=True): surf itself (leaf_scan 0) and its VoxelGrid;
  * a 16385-return ring is refused without touching the outputs, and the next call is right;
  * liliom_voxelgrid on the far cluster, 48- and 32-byte points."""
import ctypes as C

import numpy as np
import pytest

import rot_adversarial as A
import rot_oracle
import rot_restate as RS

pytestmark = pytest.mark.gpu
F = np.float32
SENT = 0x5C
WALKS = pytest.mark.parametrize("slow", [False, True], ids=["default", "slow_walk"])


@pytest.fixture(scope="module")
def sweeps():
    return A.all_sweeps()


@pytest.fixture(scope="module")
def ref(sweeps):
    out = {}
    for nm, s in sweeps:
        rc, surf, edge, cut, lab, cur = rot_oracle.extract_rot(s["pts"], s["q_imu"], s["q_lb"], s["line_num"], s["ds_rate"])
        assert rc == 0
        out[nm] = dict(surf=surf, edge=edge, cut=cut, lab=lab, cur=cur, ring=RS.assign(s["pts"], s["line_num"])["ring"])
    return out


def _ctx(monkeypatch, slow, line_num, ds_rate, leaf_scan=None):
    import liliom_b200 as L
    if slow:
        monkeypatch.setenv("LILIOM_ROT_SLOW_WALK", "1")
    else:
        monkeypatch.delenv("LILIOM_ROT_SLOW_WALK", raising=False)
    p = L.default_params(1)
    p.line_num, p.ds_rate = line_num, ds_rate
    if leaf_scan is not None:
        p.leaf_scan = leaf_scan
    c = L.Context(p)
    monkeypatch.delenv("LILIOM_ROT_SLOW_WALK", raising=False)
    return c


def _bytes_equal(a, b, what):
    assert len(a) == len(b), (what, len(a), len(b))
    if a.tobytes() != b.tobytes():
        diff = np.nonzero((a.view(np.uint32).reshape(len(a), -1) != b.view(np.uint32).reshape(len(b), -1)).any(1))[0]
        raise AssertionError(f"{what}: {len(diff)} of {len(a)} rows differ, first {diff[:5]}: {a[diff[:3]]} vs {b[diff[:3]]}")


def _curv_equal(a, b, what):
    a, b = np.asarray(a, F), np.asarray(b, F)
    ok = (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))
    assert len(a) == len(b) and ok.all(), (what, np.nonzero(~ok)[0][:5])


def _call(c, pts, s, caps):
    """liliom_extract_rot into sentinel-filled buffers of the given capacities (surf, edge, cut) with counts preset to -3"""
    import liliom_b200 as L
    from liliom_b200._lib import _dptr, _ptr, lib
    bufs = [np.full(max(k, 1) * 32, SENT, np.uint8) for k in caps]
    cnt = [C.c_int(-3) for _ in range(3)]
    rc = lib().liliom_extract_rot(c._h, _ptr(np.ascontiguousarray(pts)), len(pts), _dptr(np.asarray(s["q_imu"], np.float64)),
                                  _dptr(np.asarray(s["q_lb"], np.float64)), _ptr(bufs[0]), caps[0], C.byref(cnt[0]),
                                  _ptr(bufs[1]), caps[1], C.byref(cnt[1]), _ptr(bufs[2]), caps[2], C.byref(cnt[2]))
    return rc, [b.view(L.PT32) for b in bufs], [x.value for x in cnt]


def _check_sweep(c, nm, s, r):
    """returns the number of cut coordinates one fp32 ulp from the oracle's"""
    pts = s["pts"]
    surf, edge, cut = c.extract_rot(pts, s["q_imu"], s["q_lb"])
    lab, cur = c.extract_rot_labels(len(cut))
    flips = 0
    if A.identity_q(s):
        _bytes_equal(cut, r["cut"], f"{nm} cut")
        _bytes_equal(edge, r["edge"], f"{nm} edge")
        _bytes_equal(surf, r["surf"], f"{nm} surf")
        assert np.array_equal(lab, r["lab"]), (nm, np.nonzero(lab != r["lab"])[0][:10])
        _curv_equal(cur, r["cur"], nm)
    else:
        assert len(cut) == len(r["cut"]), nm
        assert cut["intensity"].tobytes() == r["cut"]["intensity"].tobytes(), nm
        for f in ("x", "y", "z"):
            a, b = cut[f], r["cut"][f]
            d = np.abs(a.astype(np.float64) - b.astype(np.float64))
            assert (d <= np.spacing(np.maximum(np.abs(a), np.abs(b)))).all(), (nm, f)
            flips += int((a.view(np.uint32) != b.view(np.uint32)).sum())
        curv, label, edge_r, surf_r, _ = RS.restate_cloud(cut, r["ring"], s["line_num"], s["ds_rate"])
        _curv_equal(cur, curv, nm)
        assert np.array_equal(lab, label), (nm, np.nonzero(lab != label)[0][:10])
        _bytes_equal(edge, edge_r, f"{nm} edge (restated on the device's cut)")
        _bytes_equal(surf, surf_r, f"{nm} surf (restated on the device's cut)")
    # capacities: each at the count works; each one short is refused and leaves everything untouched
    ns, ne, nc = len(surf), len(edge), len(cut)
    rc, bufs, cnt = _call(c, pts, s, (ns, ne, nc))
    assert rc == 0 and cnt == [ns, ne, nc], (nm, rc, cnt)
    assert bufs[2][:nc].tobytes() == cut.tobytes(), nm
    for k, n_k in enumerate((ns, ne, nc)):
        if n_k == 0:
            continue
        caps = [ns, ne, nc]; caps[k] -= 1
        rc, bufs, cnt = _call(c, pts, s, caps)
        assert rc == -4, (nm, k, rc)                                                   # LILIOM_E_CAPACITY
        assert cnt == [-3, -3, -3] and all((b.view(np.uint8) == SENT).all() for b in bufs), (nm, k)
    return flips


@WALKS
def test_extract_rot_adversarial(sweeps, ref, monkeypatch, slow):
    flips = 0
    ctxs = {}
    try:
        for nm, s in sweeps:
            key = (s["line_num"], s["ds_rate"])
            if key not in ctxs:
                ctxs[key] = _ctx(monkeypatch, slow, *key)
            flips += _check_sweep(ctxs[key], nm, s, ref[nm])
    finally:
        for c in ctxs.values():
            c.close()
    print(f"cut coordinates one fp32 ulp from the oracle's ({'slow' if slow else 'default'} walk): {flips}")


@WALKS
def test_ring_field_gives_the_table_bytes(sweeps, ref, monkeypatch, slow):
    """the tables' verdict written into a PointCloud2 `ring` field (a miss as ring = line_num) reproduces the table path"""
    import liliom_b200 as L
    from liliom_b200 import synth
    for nm, s in sweeps:
        if s["line_num"] != 64 or not A.identity_q(s) or len(s["pts"]) == 0:
            continue
        ids = rot_oracle.scan_ids(s["pts"], 64)
        ring = np.where(ids < 0, 64, ids)
        msg = synth.encode_pc2(s["pts"], ring, np.zeros(len(ring), np.int64), "pcl32")
        c = _ctx(monkeypatch, slow, 64, s["ds_rate"])
        try:
            c.set_ring_source(L.RING_FIELD)
            surf, edge, cut = c.extract_rot_pc2(msg, s["q_imu"], s["q_lb"])
        finally:
            c.close()
        r = ref[nm]
        _bytes_equal(cut, r["cut"], f"{nm} ring field cut")
        _bytes_equal(edge, r["edge"], f"{nm} ring field edge")
        _bytes_equal(surf, r["surf"], f"{nm} ring field surf")


@WALKS
def test_resident_leg(sweeps, ref, monkeypatch, slow):
    import liliom_b200 as L
    import oracle_lib
    for nm, s in sweeps:
        if not A.identity_q(s) or len(ref[nm]["surf"]) < 10:
            continue
        surf_o = ref[nm]["surf"]
        near = surf_o[(np.abs(surf_o["x"]) < 1e4) & (np.abs(surf_o["y"]) < 1e4) & (np.abs(surf_o["z"]) < 1e4)]    # the map: the surf cloud's near part
        m = np.ones((len(near), 4), np.float32)
        m[:, 0], m[:, 1], m[:, 2] = near["x"], near["y"], near["z"]
        for leaf in (0.0, None):
            c = _ctx(monkeypatch, slow, s["line_num"], s["ds_rate"], leaf)
            try:
                c.map_set_points(m)
                c.upload_scan(s["pts"])
                c.extract_resident(s["q_imu"], s["q_lb"])
                _, _, ds = c.odometry_resident((1.0, 0, 0, 0, 0, 0, 0), 1, mode=L.MODE_GN, want_ds=True, cap=len(s["pts"]),
                                               want_stats=False)
            finally:
                c.close()
            want = surf_o if leaf == 0.0 else oracle_lib.voxelgrid(surf_o, L.default_params(1).leaf_scan)
            _bytes_equal(ds, want, f"resident {nm} leaf={leaf}")


@WALKS
def test_ring_cap_refusal_then_recovery(sweeps, ref, monkeypatch, slow):
    s_big = A.cap_sweep(16385)
    s_ok = dict(sweeps)["ring16384"]
    c = _ctx(monkeypatch, slow, 16, 1)
    try:
        n = len(s_big["pts"])
        rc, bufs, cnt = _call(c, s_big["pts"], s_big, (n, n, n))
        assert rc == -4 and cnt == [-3, -3, -3] and all((b.view(np.uint8) == SENT).all() for b in bufs), rc
        _check_sweep(c, "ring16384 after the refusal", s_ok, ref["ring16384"])
    finally:
        c.close()


@pytest.mark.parametrize("stride", [48, 32])
def test_voxelgrid_far_cluster(stride):
    """PCL's x86 indices: every x index of the far cluster is INT_MIN, voxels that differ only in x merge"""
    import liliom_b200 as L
    import oracle_lib
    pts = A.far_cluster(stride)
    want = oracle_lib.voxelgrid(pts, 0.6)
    assert len(want) == 7                             # 3 x columns x 7 y voxels, merged across x
    c = L.Context(L.default_params(0 if stride == 48 else 1))
    try:
        got = c.voxelgrid(pts, 0.6)
    finally:
        c.close()
    _bytes_equal(got, want, f"far cluster stride {stride}")
