"""GPU tier for loop closure from the keyframe store (liliom_loop_align): detectLoopClosure's two clouds and performLoopClosure's
ICP in one call on the backend context.  Bit-identical to liliom_kf_cloud x2 + liliom_icp_align on a second context in both
point layouts; a known drift is undone; the empty and out-of-reach cases and the argument errors; the context's resident state
(odometry map, local map, single-keyframe and window correspondences) is left exactly as it was; and a source larger than one
co-resident grid (the ICP kernel's virtual blocks) against the NumPy restatement of PCL's loop."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_HIST = 41               # his_key_frames_ds at lc_map_width = 20: 2 * 20 + 1 keyframes
LEAF = 0.4                # the loop-closure clouds' VoxelGrid (L/src/BackendFusion.cpp:2494, :2545)
REVISIT = N_HIST          # id of the keyframe that comes back to keyframe 0's pose
NO_EDGE = N_HIST + 1      # id of a keyframe stored with an empty edge cloud


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


@pytest.fixture(scope="module")
def stores():
    """per point layout: (context, backend params, the keyframe poses) with N_HIST + 2 keyframes stored"""
    import liliom_b200 as L
    from liliom_b200 import synth
    out = {}
    for stride, variant in ((48, 0), (32, 1)):
        seq = synth.make_keyframe_sequence(N_HIST, stride=stride, revisit=1)
        e5, s5, p5 = seq[5]
        seq.append((e5[:0], s5, p5))
        bp = L.backend_default_params(variant)
        c = L.Context(variant=variant)
        for i, (e, s, _) in enumerate(seq):
            assert c.kf_add(bp, e, s, download=False)[0] == i
        out[stride] = (c, bp, [p for _, _, p in seq], variant)
    yield out
    for c, _, _, _ in out.values():
        c.close()


def _two_step(c, variant, src_ids, src_poses, tgt_ids, tgt_poses, leaf=LEAF, **kw):
    """the composition liliom_loop_align replaces: both clouds to the host, ICP on a second context"""
    import liliom_b200 as L
    src = c.kf_cloud(src_ids, src_poses, leaf)
    tgt = c.kf_cloud(tgt_ids, tgt_poses, leaf)
    c2 = L.Context(variant=variant)
    try:
        T, fit, conv, it = c2.icp_align(src, tgt, **kw)
    finally:
        c2.close()
    return T, fit, conv, it, len(src), len(tgt)


def _lists():
    hist = list(range(N_HIST))
    return [
        ("1-vs-41", [REVISIT], hist),
        ("repeated-ids", [3, 3], [0, 1, 1, 2, 2, 2, 4]),
        ("empty-edge-cloud", [NO_EDGE], [4, NO_EDGE, 6, 7]),
        ("41-vs-1", hist, [REVISIT]),
    ]


@pytest.mark.parametrize("stride", [48, 32])
def test_loop_align_bit_identical_to_kf_cloud_and_icp_align(stores, stride):
    c, _, poses, variant = stores[stride]
    for name, si, ti in _lists():
        sp, tp = [poses[i] for i in si], [poses[i] for i in ti]
        got = c.loop_align(si, sp, ti, tp, LEAF)
        want = _two_step(c, variant, si, sp, ti, tp)
        T, fit, conv, it, ns, nt = got
        assert ns > 0 and nt > 0, name
        assert (ns, nt) == want[4:], name
        assert _bytes(T) == _bytes(want[0]), name
        assert np.float64(fit).tobytes() == np.float64(want[1]).tobytes(), name
        assert (conv, it) == (want[2], want[3]), name
        assert it >= 1, name
    # other ICP settings go through the same code
    si, ti = [REVISIT], list(range(0, 12))
    sp, tp = [poses[i] for i in si], [poses[i] for i in ti]
    got = c.loop_align(si, sp, ti, tp, 0.6, max_corr_dist=2.0, max_iter=3, trans_eps=1e-8, fit_eps=1e-9)
    want = _two_step(c, variant, si, sp, ti, tp, 0.6, max_corr_dist=2.0, max_iter=3, trans_eps=1e-8, fit_eps=1e-9)
    assert _bytes(got[0]) == _bytes(want[0]) and got[1:] == want[1:] and got[3] == 3


def _drifted(pose, ang_deg, axis, dt):
    from liliom_b200 import synth
    qd = synth.q_from_axis_angle(axis, np.deg2rad(ang_deg))
    Rd = _rotm(qd)
    return np.concatenate([synth.qmul(qd, pose[:4]), Rd @ pose[4:] + dt]), Rd


def _rotm(q):
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


@pytest.mark.parametrize("stride", [48, 32])
def test_loop_align_undoes_a_known_drift(stores, stride):
    """a keyframe listed with a pose off by 2 deg / 0.5 m in the world frame: the alignment is the inverse drift.  Keyframe 0
    itself (its clouds are part of the history cloud): within 0.1 deg / 3 cm, fitness below lc_icp_thres.  The revisit keyframe
    (a new sweep from keyframe 0's pose, so the best fit is not exactly the inverse drift, and PCL's relative-MSE rule ends the
    slow last steps early): within 0.6 deg / 15 cm, i.e. most of the drift undone"""
    c, _, poses, _ = stores[stride]
    dt = np.array([0.4, -0.25, 0.15])
    hist, hp = list(range(N_HIST)), [poses[i] for i in range(N_HIST)]
    for kf, tol_r, tol_t in ((0, 2e-3, 0.03), (REVISIT, 1e-2, 0.15)):
        p_d, Rd = _drifted(poses[kf], 2.0, [0.1, -0.1, 1.0], dt)
        T, fit, conv, it, ns, nt = c.loop_align([kf], [p_d], hist, hp, LEAF)
        assert conv and 1 <= it < 100, kf
        assert np.abs(T[:3, :3] - Rd.T).max() < tol_r, (kf, T)
        assert np.abs(T[:3, 3] - (-Rd.T @ dt)).max() < tol_t, (kf, T)
        assert np.array_equal(T[3], [0, 0, 0, 1])
        if kf == 0:
            assert fit < 0.1, fit                                 # lc_icp_thres (L/config/config_fr_iosb.yaml)


@pytest.mark.parametrize("stride", [48, 32])
def test_loop_align_empty_out_of_reach_and_bad_arguments(stores, stride):
    import liliom_b200 as L
    c, _, poses, _ = stores[stride]
    hist, hp = list(range(10)), [poses[i] for i in range(10)]
    far = poses[REVISIT].copy(); far[4] += 500.0
    T, fit, conv, it, ns, nt = c.loop_align([REVISIT], [far], hist, hp, LEAF, max_corr_dist=5.0)
    assert not conv and it == 0 and np.array_equal(T, np.eye(4)) and ns > 0 and nt > 0
    for si, sp, ti, tp in (([], [], hist, hp), ([REVISIT], [poses[REVISIT]], [], [])):
        T, fit, conv, it, ns, nt = c.loop_align(si, sp, ti, tp, LEAF)
        assert not conv and it == 0 and np.array_equal(T, np.eye(4)) and fit == 0.0
        assert (ns == 0) == (len(si) == 0) and (nt == 0) == (len(ti) == 0)
    before = c.loop_align([REVISIT], [poses[REVISIT]], hist, hp, LEAF)
    n_kf = c.kf_count()
    bad = [dict(si=[REVISIT + 100]), dict(ti=[0, -1]), dict(leaf=0.0), dict(leaf=-0.4), dict(max_corr_dist=0.0),
           dict(max_corr_dist=-1.0), dict(max_iter=0)]
    for b in bad:
        si = b.get("si", [REVISIT]); ti = b.get("ti", hist)
        with pytest.raises(L.LiliomError) as e:
            c.loop_align(si, [poses[0]] * len(si), ti, [poses[0]] * len(ti), b.get("leaf", LEAF),
                         max_corr_dist=b.get("max_corr_dist", 30.0), max_iter=b.get("max_iter", 100))
        assert e.value.code == L._binding.E_ARG, b
    assert c.kf_count() == n_kf
    after = c.loop_align([REVISIT], [poses[REVISIT]], hist, hp, LEAF)
    assert _bytes(after[0]) == _bytes(before[0]) and after[1:] == before[1:]


def _backend_session(variant, seq_poses, fill, call_between):
    """local map, odometry map, a single-keyframe correspondence and resident window correspondences on one context; the
    call (optional) between window_correspond and window_blocks; then everything that reads the resident state"""
    import liliom_b200 as L
    from liliom_b200 import synth
    c = L.Context(variant=variant)
    bp = L.backend_default_params(variant)
    feats = fill(c, bp)
    m, _ = synth.make_map(60_000)
    c.map_set_points(m)
    ve, pa, pb = c.correspond_edge(feats, seq_poses[20], 0)
    c.bmap_build(bp, list(range(10, 30)), [seq_poses[i] for i in range(10, 30)])
    win = [27, 28, 29]
    c.backend_window_correspond(bp, win, [seq_poses[i] for i in win])
    if call_between:
        call_between(c)
    out = {"blocks": c.backend_window_blocks([seq_poses[i] for i in win]), "edge": c.bmap_download(0), "surf": c.bmap_download(1),
           "edge_block": c.backend_edge_block(seq_poses[20], 0.6), "map": c.map_download(), "edge_valid": ve}
    for slot in range(len(win)):
        for kind in (0, 1):
            out[f"win{slot}{kind}"] = np.frombuffer(b"".join(_bytes(a) for a in c.backend_window_corr(slot, kind)), np.uint8)
    c.close()
    return out


@pytest.mark.parametrize("stride", [48, 32])
def test_loop_align_leaves_the_resident_state_alone(stores, stride):
    from liliom_b200 import synth
    _, _, poses, variant = stores[stride]
    seq = synth.make_keyframe_sequence(N_HIST, stride=stride, revisit=1)

    def fill(c, bp):
        for e, s, _ in seq:
            c.kf_add(bp, e, s, download=False)
        return seq[20][0]

    res = {}

    def call(c):
        res["r"] = c.loop_align([REVISIT], [poses[REVISIT]], list(range(N_HIST)), [poses[i] for i in range(N_HIST)], LEAF)

    with_call = _backend_session(variant, poses, fill, call)
    without = _backend_session(variant, poses, fill, None)
    assert res["r"][3] >= 1 and res["r"][2]
    assert with_call["edge_valid"].sum() > 0 and len(with_call["edge"]) > 0 and len(with_call["map"]) > 0
    assert np.abs(with_call["blocks"]).sum() > 0
    for k in without:
        assert _bytes(with_call[k]) == _bytes(without[k]), k


def test_virtual_block_path_against_numpy(oracle, world_small):
    """a 300k-point source: more virtual blocks than co-resident blocks, so blocks take several; the ICP follows the NumPy /
    kd-tree restatement to test_loop_closure_icp's tolerance and is bit-identical between the two entry points' layouts"""
    import liliom_b200 as L
    from test_gpu_widen import _icp_numpy
    rng = np.random.default_rng(12)
    m = world_small["map"]
    near = m[(np.abs(m[:, 0]) < 45) & (np.abs(m[:, 1]) < 45)]
    tgt = near[rng.permutation(len(near))[:30000]].copy()
    ang = np.deg2rad(1.5)
    Rz = np.array([[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1.0]])
    t_true = np.array([0.3, -0.2, 0.05])
    pick = near[rng.integers(0, len(near), 300_000)]
    src = np.ones((len(pick), 4), np.float32)
    src[:, :3] = ((pick[:, :3].astype(np.float64) - t_true) @ Rz + rng.normal(0, 0.02, (len(pick), 3))).astype(np.float32)
    c = L.Context(variant=0)
    T, fit, conv, it = c.icp_align(src, tgt)
    c.close()
    T_o, fit_o, conv_o, it_o = _icp_numpy(oracle, src, tgt)
    assert conv and conv_o and abs(it - it_o) <= 1 and 3 <= it < 100, (it, it_o)
    np.testing.assert_allclose(T, T_o, rtol=0, atol=2e-6 if it == it_o else 2e-4)
    assert abs(fit - fit_o) < 1e-6 * max(1.0, fit_o)
    assert np.abs(T[:3, :3] - Rz).max() < 5e-3 and np.abs(T[:3, 3] - t_true).max() < 0.05
