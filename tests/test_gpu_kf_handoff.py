"""The keyframe hand-off from the odometry to the backend on the device: publishCloudLast's de-skew on the resident clouds
(liliom_undistort_resident) and the keyframe store filled from them (liliom_kf_add_resident), against the host chain they replace
(liliom_features_download, liliom_undistort per cloud, liliom_kf_add, liliom_kf_add_full), bit for bit.

Every comparison is of bytes.  The stored clouds are read back four ways: each keyframe's surf and full cloud through
liliom_global_map at a leaf PCL declines (the output is the stored cloud, transformed by the identity), the backend local map
(liliom_bmap_build + liliom_bmap_download), liliom_kf_cloud, and one liliom_loop_align."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

IDENT7 = np.array([1.0, 0, 0, 0, 0, 0, 0])
IDENT_Q = (1.0, 0.0, 0.0, 0.0)
TINY_LEAF = 1e-4          # PCL declines every keyframe-sized cloud at this leaf: the output is the transformed input
N_KF = 8
ITERS = 4


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def _code(f):
    import liliom_b200 as L
    try:
        f()
        return L._binding.OK
    except L.LiliomError as e:
        return e.code


def _ctx(variant, **kw):
    import liliom_b200 as L
    p = L.default_params(variant)
    for k, v in kw.items():
        setattr(p, k, v)
    return L.Context(p)


def _motion(k):
    """publishCloudLast's arguments for keyframe k: the scan's relative translation, the identity rotation"""
    return (0.25 + 0.02 * k, -0.08, 0.015), IDENT_Q


def _livox(pts):
    """Livox CustomMsg records of a Horizon sweep: FormatConvert (L/src/FormatConvert.cpp:14-22) gives them back as the sweep,
    up to float rounding of the time fraction"""
    import liliom_b200 as L
    t_end = 100_000_000
    frac = (pts["intensity"] - np.floor(pts["intensity"])).astype(np.float64) / 0.1
    order = np.argsort(frac, kind="stable")
    p, s = pts[order], frac[order]
    r = np.zeros(len(p), L.LIVOX20)
    off = np.minimum(np.round(s * t_end), t_end).astype(np.uint32)
    off[-1:] = t_end
    r["offset_time"] = off
    r["x"], r["y"], r["z"] = p["x"], p["y"], p["z"]
    r["reflectivity"] = np.clip(np.round(p["curvature"] * 10.0), 0, 255).astype(np.uint8)
    r["line"] = np.floor(p["intensity"]).astype(np.uint8)
    return r


@pytest.fixture(scope="module")
def world():
    """N_KF Horizon sweeps and N_KF 64-line sweeps along a short path through synth's world (the one synth.make_map samples),
    each with its true pose and a perturbed guess."""
    from liliom_b200 import synth
    T0 = synth.default_true_pose()
    out = {0: [], 1: []}
    for k in range(N_KF):
        T = np.array(T0); T[4] += 0.6 * k; T[5] += 0.12 * k
        pts, q = synth.make_horizon_sweep(T, seed=1 + k)
        out[0].append(dict(T=T, guess=synth.perturbed_pose(T), pts=pts, q=q))
        pts, q = synth.make_hdl64_sweep(T, seed=2 + k, steps=1200)
        out[1].append(dict(T=T, guess=synth.perturbed_pose(T), pts=pts, q=q))
    return out


def _extract(c, path, sw, other=None):
    """One extraction of sweep sw on c by `path`; the clouds stay resident"""
    import liliom_b200 as L
    if path == "hz_host":                      # liliom_extract_horizon: the counts come back to the host
        c.extract_horizon(sw["pts"], sw["q"])
    elif path == "hz_livox":                   # liliom_convert_livox + liliom_extract_resident: the counts stay on the device
        c.convert_livox(_livox(sw["pts"]), download=False)
        assert c.extract_resident(sw["q"]) == (-1, -1, -1)
    elif path == "rot_resident":
        c.upload_scan(sw["pts"])
        c.extract_resident(sw["q"])
    elif path == "rot_batch":                  # liliom_extract_resident_batch, beside another session
        c.upload_scan(sw["pts"])
        other.upload_scan(sw["pts"][::2])
        _, status = L.extract_resident_batch([c, other], np.stack([sw["q"], sw["q"]]))
        assert list(status) == [0, 0]
    else:
        raise ValueError(path)


# ---------------------------------------------------------------- 1. the de-skew, every residency path
PATHS = [("hz_host", 0), ("hz_livox", 0), ("rot_resident", 1), ("rot_batch", 1)]


def _deskew_args(motion):
    from liliom_b200 import synth
    if motion == "moving":                                   # a non-zero translation and a non-identity rotation
        return (0.31, -0.12, 0.05), tuple(synth.q_from_axis_angle([0.3, -0.2, 1.0], 0.02))
    return (0.0, 0.0, 0.0), IDENT_Q                          # no motion: the clouds keep their bits


@pytest.mark.parametrize("motion", ["moving", "still"])
@pytest.mark.parametrize("path,variant", PATHS)
def test_undistort_resident_equals_undistort(oracle, world, path, variant, motion):
    """features_download after liliom_undistort_resident = liliom_undistort (and the oracle) of each cloud downloaded before,
    in one launch; a second call de-skews again"""
    t, q = _deskew_args(motion)
    c, ref, other = _ctx(variant), _ctx(variant), _ctx(variant)
    for k in (0, 3):
        _extract(c, path, world[variant][k], other)
        before = c.features_download()
        assert all(len(x) > 0 for x in before), [len(x) for x in before]
        c.counters(reset=True)
        c.undistort_resident(t, q)
        assert c.counters().launches == 1
        after = c.features_download()
        for name, b, a in zip(("surf", "edge", "cut"), before, after):
            assert len(a) == len(b), name
            assert _bytes(a) == _bytes(ref.undistort(b, t, q)), (path, motion, k, name)
            assert _bytes(a) == _bytes(oracle.undistort(b, t, q)), (path, motion, k, name)
            if motion == "still":
                assert _bytes(a) == _bytes(b), name
    c.undistort_resident(t, q)                                      # twice = undistortion twice
    for a, b in zip(c.features_download(), after):
        assert _bytes(a) == _bytes(ref.undistort(b, t, q))
    for x in (c, ref, other):
        x.close()


@pytest.mark.parametrize("path", ["hz_host", "hz_livox"])
def test_undistort_resident_empty_clouds(world, path):
    """an empty edge cloud gets no blocks and the others are de-skewed; an empty sweep launches nothing"""
    t, q = _deskew_args("moving")
    c, ref = _ctx(0, edge_thres=1e30), _ctx(0)                      # no return passes the edge threshold
    _extract(c, path, world[0][1])
    before = c.features_download()
    assert len(before[1]) == 0 and len(before[0]) > 0 and len(before[2]) > 0
    c.counters(reset=True)
    c.undistort_resident(t, q)
    assert c.counters().launches == 1
    for a, b in zip(c.features_download(), before):
        assert _bytes(a) == _bytes(ref.undistort(b, t, q))
    sw = dict(world[0][1], pts=world[0][1]["pts"][:0])
    _extract(c, path, sw)
    assert [len(x) for x in c.features_download()] == [0, 0, 0]
    c.counters(reset=True)
    c.undistort_resident(t, q)
    assert c.counters().launches == 0
    c.close(); ref.close()


# ---------------------------------------------------------------- 2. the odometry's state is left alone
def _odo(c, guess):
    """liliom_odometry_resident with ds_out: (rc, pose, DS cloud)"""
    import liliom_b200 as L
    pose = np.array(guess, dtype=np.float64)
    ds = np.zeros(65536, c.dtype)
    nds = C.c_int()
    rc = L._binding.lib().liliom_odometry_resident(c._h, pose.ctypes.data_as(C.POINTER(C.c_double)), ITERS, 15, L.MODE_GN, None,
                                                   ds.ctypes.data_as(C.c_void_p), len(ds), C.byref(nds))
    return rc, pose, ds[:nds.value].copy()


@pytest.mark.parametrize("variant", [0, 1])
def test_odometry_state_untouched(world, variant):
    """extract -> odometry_resident -> de-skew on keyframes -> map_update_resident: the same poses, down-sampled scans and maps
    as a control context that never de-skews"""
    a, b = _ctx(variant), _ctx(variant)                             # a de-skews on keyframes, b is the control
    for k, sw in enumerate(world[variant][:6]):
        for c in (a, b):
            c.upload_scan(sw["pts"])
            c.extract_resident(sw["q"])
        ra, rb = _odo(a, sw["guess"]), _odo(b, sw["guess"])
        if k % 2 == 0:
            a.undistort_resident(*_motion(k))
        assert ra[0] == rb[0] == (-8 if k == 0 else 0), (k, ra[0], rb[0])
        assert _bytes(ra[1]) == _bytes(rb[1]), (k, "pose")
        assert len(ra[2]) > 0 and _bytes(ra[2]) == _bytes(rb[2]), (k, "DS")
        pose = ra[1] if ra[0] == 0 else sw["T"]
        assert a.map_update_resident(pose) == b.map_update_resident(pose)
        assert _bytes(a.map_download_cloud()) == _bytes(b.map_download_cloud()), k
        assert _bytes(a.map_download()) == _bytes(b.map_download()), k
    # after the map update (which moves a resident Horizon extraction's cut count aside) the de-skew still reads every count
    ref = _ctx(variant)
    before = a.features_download()
    a.undistort_resident(*_motion(9))
    for x, y in zip(a.features_download(), before):
        assert _bytes(x) == _bytes(ref.undistort(y, *_motion(9)))
    for c in (a, b, ref):
        c.close()


# ---------------------------------------------------------------- 3, 4. the store, four ways
def _host_keyframe(bk, bp, odo, motion):
    """the seven-call chain: download, liliom_undistort per cloud, liliom_kf_add, liliom_kf_add_full"""
    surf, edge, cut = odo.features_download()
    if motion is not None:
        surf, edge, cut = (odo.undistort(x, *motion) for x in (surf, edge, cut))
    kid, e_ds, s_ds = bk.kf_add(bp, edge, surf)
    nf = bk.kf_add_full(bp, kid, cut)
    return kid, len(e_ds), len(s_ds), nf


def _resident_keyframe(bk, bp, odo, motion):
    if motion is not None:
        odo.undistort_resident(*motion)
    return bk.kf_add_resident(bp, odo)


def _store(world, variant, deskew, mode):
    """A backend context filled with N_KF keyframes by `mode`: 'host' (the host chain), 'resident' (separate odometry and
    backend contexts), 'same' (one context for both) or 'streams' (separate contexts, each on a caller stream).
    Returns (backend context, per-keyframe results)."""
    import liliom_b200 as L
    bp = L.backend_default_params(variant)
    streams = []
    bk = _ctx(variant)
    odo = bk if mode == "same" else _ctx(variant)
    if mode == "streams":
        import torch
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        odo.set_stream(streams[0].cuda_stream)
        bk.set_stream(streams[1].cuda_stream)
    res = []
    for k, sw in enumerate(world[variant]):
        odo.upload_scan(sw["pts"])
        odo.extract_resident(sw["q"])
        if mode == "same" and k == 0:                               # a down-sampled scan is resident before the hand-off ...
            assert _odo(odo, sw["guess"])[0] == L._binding.E_NOMAP
        motion = _motion(k) if deskew else None
        res.append((_host_keyframe if mode == "host" else _resident_keyframe)(bk, bp, odo, motion))
        if mode == "same" and k == 0:                               # ... and gone after it, as after liliom_kf_add
            assert _code(lambda: bk.map_update_resident(sw["T"])) == L._binding.E_ARG
    if mode != "same":
        odo.set_stream(None)
        odo.close()
    bk.set_stream(None)
    return bk, res


def _same_store(a, b, variant, what):
    import liliom_b200 as L
    bp = L.backend_default_params(variant)
    n = a.kf_count()
    assert n == b.kf_count() == N_KF, what
    for i in range(n):
        for kind in (L.KF_SURF, L.KF_FULL):
            ga, gb = a.global_map(kind, [i], [IDENT7], TINY_LEAF), b.global_map(kind, [i], [IDENT7], TINY_LEAF)
            assert len(ga) > 0 and _bytes(ga) == _bytes(gb), (what, i, kind)
    ids = list(range(n))
    poses = [IDENT7 + np.array([0, 0, 0, 0, 0.6 * i, 0.12 * i, 0]) for i in ids]
    assert a.bmap_build(bp, ids, poses) == b.bmap_build(bp, ids, poses), what
    for layer in (0, 1):
        assert _bytes(a.bmap_download(layer)) == _bytes(b.bmap_download(layer)), (what, "bmap", layer)
    assert _bytes(a.kf_cloud(ids, poses, 0.4)) == _bytes(b.kf_cloud(ids, poses, 0.4)), (what, "kf_cloud")
    la = a.loop_align([n - 1], [poses[-1]], ids[:-1], poses[:-1], 0.4, max_iter=20)
    lb = b.loop_align([n - 1], [poses[-1]], ids[:-1], poses[:-1], 0.4, max_iter=20)
    assert _bytes(la[0]) == _bytes(lb[0]) and la[1:] == lb[1:], (what, "loop", la[1:], lb[1:])


@pytest.fixture(scope="module")
def host_stores(world):
    out = {}
    for variant in (0, 1):
        for deskew in (False, True):
            out[variant, deskew] = _store(world, variant, deskew, "host")
    yield out
    for bk, _ in out.values():
        bk.close()


@pytest.mark.parametrize("deskew", [False, True])
@pytest.mark.parametrize("variant", [0, 1])
def test_store_parity(world, host_stores, variant, deskew):
    """liliom_kf_add_resident over N_KF keyframes stores what the host chain stores: ids, counts and every stored cloud"""
    a, ra = host_stores[variant, deskew]
    b, rb = _store(world, variant, deskew, "resident")
    assert ra == rb and [r[0] for r in rb] == list(range(N_KF))
    assert all(r[1] > 0 and r[2] > 0 and r[3] > 0 for r in rb), rb
    _same_store(a, b, variant, (variant, deskew))
    b.close()


@pytest.mark.parametrize("mode", ["same", "streams"])
@pytest.mark.parametrize("variant", [0, 1])
def test_store_parity_same_context_and_caller_streams(world, host_stores, variant, mode):
    """src == c, and both contexts on caller streams (liliom_set_stream): the bits of the host chain"""
    a, ra = host_stores[variant, True]
    b, rb = _store(world, variant, True, mode)
    assert ra == rb
    _same_store(a, b, variant, (variant, mode))
    b.close()


# ---------------------------------------------------------------- 5. refusals change nothing
def _state(c):
    import liliom_b200 as L
    try:
        return tuple(_bytes(x) for x in c.features_download())
    except L.LiliomError as e:
        return e.code


def _raw_add(c, bp, src, null_id=False):
    import liliom_b200 as L
    kid, ne, ns, nf = C.c_int(-7), C.c_int(-7), C.c_int(-7), C.c_int(-7)
    return L._binding.lib().liliom_kf_add_resident(c._h, C.byref(bp), src._h, None if null_id else C.byref(kid), C.byref(ne),
                                                   C.byref(ns), C.byref(nf))


def _loopback_ctx(variant, group):
    """rank 0 of a two-rank loopback group (the single-GPU stand-in for a communicator, see test_gpu_sharded.py)"""
    os.environ["LILIOM_TEST_LOOPBACK"] = f"{group}:0/2"
    try:
        return _ctx(variant)
    finally:
        os.environ.pop("LILIOM_TEST_LOOPBACK", None)


def test_refusals_change_nothing(world):
    import liliom_b200 as L
    E_ARG = L._binding.E_ARG
    bp0 = L.backend_default_params(0)
    sw0, sw1 = world[0][2], world[1][2]
    bk = _ctx(0)
    good = _ctx(0)
    _extract(good, "hz_livox", sw0)
    assert bk.kf_add_resident(bp0, good)[0] == 0                    # one keyframe stored before the refusals

    fresh = _ctx(0)
    host_feats = _ctx(0)
    _extract(host_feats, "hz_host", sw0)
    surf = host_feats.features_download()[0]
    _code(lambda: host_feats.odometry(surf, sw0["guess"], ITERS))    # the caller's surf features replace the extracted ones
    rot = _ctx(1)
    _extract(rot, "rot_resident", sw1)
    bad_bp = L.backend_default_params(0)
    bad_bp.edge_leaf = 0.0
    lb_src = _loopback_ctx(0, "kfh_src")
    _code(lambda: _extract(lb_src, "hz_host", sw0))                 # refused for its communicator whether or not it extracts
    lb_bk = _loopback_ctx(0, "kfh_bk")

    cases = [
        ("fresh src", bk, lambda: _raw_add(bk, bp0, fresh), fresh),
        ("src after liliom_odometry", bk, lambda: _raw_add(bk, bp0, host_feats), host_feats),
        ("strides differ", bk, lambda: _raw_add(bk, bp0, rot), rot),
        ("invalid bp", bk, lambda: _raw_add(bk, bad_bp, good), good),
        ("NULL kf_id", bk, lambda: _raw_add(bk, bp0, good, null_id=True), good),
        ("src with a communicator", bk, lambda: _raw_add(bk, bp0, lb_src), lb_src),
        ("c with a communicator", lb_bk, lambda: _raw_add(lb_bk, bp0, good), good),
        ("undistort, nothing resident", bk, lambda: L._binding.lib().liliom_undistort_resident(
            fresh._h, np.zeros(3).ctypes.data_as(C.POINTER(C.c_double)), np.array(IDENT_Q).ctypes.data_as(C.POINTER(C.c_double))), fresh),
        ("undistort, NULL trans", bk, lambda: L._binding.lib().liliom_undistort_resident(
            good._h, None, np.array(IDENT_Q).ctypes.data_as(C.POINTER(C.c_double))), good),
    ]
    for what, c, call, src in cases:
        n0, s0, c0 = c.kf_count(), _state(src), _state(c)
        assert call() == E_ARG, what
        assert c.kf_count() == n0, what
        assert _state(src) == s0 and _state(c) == c0, what
    assert _state(fresh) == E_ARG and _state(host_feats) == E_ARG
    assert bk.kf_count() == 1 and bk.kf_add_resident(bp0, good)[0] == 1      # the store still takes keyframes
    for c in (bk, good, fresh, host_feats, rot, lb_src, lb_bk):
        c.close()


# ---------------------------------------------------------------- 6. an empty sweep
@pytest.mark.parametrize("variant", [0, 1])
def test_empty_sweep_stores_an_empty_keyframe(world, variant):
    """all counts 0: a keyframe with no points is stored, as liliom_kf_add / liliom_kf_add_full with n = 0 store it"""
    import liliom_b200 as L
    bp = L.backend_default_params(variant)
    odo, a, b = _ctx(variant), _ctx(variant), _ctx(variant)
    sw = world[variant][0]
    for bk in (a, b):                                               # one keyframe with points first
        odo.upload_scan(sw["pts"]); odo.extract_resident(sw["q"])
        (_host_keyframe if bk is a else _resident_keyframe)(bk, bp, odo, None)
    odo.upload_scan(sw["pts"][:0])
    odo.extract_resident(sw["q"])
    assert [len(x) for x in odo.features_download()] == [0, 0, 0]
    ra = _host_keyframe(a, bp, odo, None)
    rb = _resident_keyframe(b, bp, odo, None)
    assert ra == rb == (1, 0, 0, 0)
    assert a.kf_count() == b.kf_count() == 2
    for kind in (L.KF_SURF, L.KF_FULL):
        assert len(b.global_map(kind, [1], [IDENT7], TINY_LEAF)) == 0
        assert _bytes(a.global_map(kind, [0, 1], [IDENT7, IDENT7], TINY_LEAF)) == _bytes(b.global_map(kind, [0, 1], [IDENT7, IDENT7], TINY_LEAF))
    for c in (odo, a, b):
        c.close()
