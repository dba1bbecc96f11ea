"""GPU parity for SURVEY.md §8 (f5): the backend's keyframe store, device-resident local map, window correspondences and blocks,
and the loop-closure clouds, through the C ABI against the oracle composed from existing pieces (voxelgrid, transform_cloud,
KdTree, correspond_edge, correspond_surf_backend, backend_*_block) with the variant weights restated in NumPy."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

WIDTH = 5          # local_map_width of the deque-policy test
WINDOW = 3         # slide_window_width (config_fr_iosb.yaml)


@pytest.fixture(scope="module")
def seq48():
    from liliom_b200 import synth
    return synth.make_keyframe_sequence(16, stride=48)


@pytest.fixture(scope="module")
def seq32():
    from liliom_b200 import synth
    return synth.make_keyframe_sequence(16, stride=32)


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def _f4(cloud):
    out = np.ones((len(cloud), 4), np.float32)
    out[:, 0] = cloud["x"]; out[:, 1] = cloud["y"]; out[:, 2] = cloud["z"]
    return out


def _cat(parts, dtype):
    parts = [p for p in parts if len(p)]
    return np.concatenate(parts) if parts else np.zeros(0, dtype)


def _qmul(a, b):
    from liliom_b200 import synth
    return synth.qmul(a, b)


def _body_from_lidar(pose_l, bp):
    """Inverse of :929-930 (Q2 = Q q_lb^-1, T2 = T - Q2 t_lb): the body pose whose lidar pose is pose_l."""
    from liliom_b200 import synth
    q_lb = np.array(bp.q_lb[:]); t_lb = np.array(bp.t_lb[:])
    q = _qmul(pose_l[:4], q_lb)
    # unit, like every quaternion Ceres' QuaternionParameterization keeps (the closed-form rows assume it; R's q_lb of
    # 0.7071 / 0.7071 is not quite unit)
    return np.concatenate([q / np.linalg.norm(q), pose_l[4:] + synth.qrot(pose_l[:4], t_lb)])


def _nudge(pose, k):
    """A small, deterministic pose change (an optimiser's correction / an LM trial step)."""
    from liliom_b200 import synth
    dq = synth.q_from_axis_angle([1, -1, 2], np.deg2rad(0.15 * k))
    return np.concatenate([_qmul(pose[:4], dq), pose[4:] + 0.01 * k * np.array([1.0, -0.5, 0.25])])


def _oracle_layers(O, kfs, ids, poses, bp, dtype):
    E = _cat([O.transform_cloud(kfs[i][0], p) for i, p in zip(ids, poses)], dtype)
    S = _cat([O.transform_cloud(kfs[i][1], p) for i, p in zip(ids, poses)], dtype)
    return O.voxelgrid(E, bp.edge_leaf), O.voxelgrid(S, bp.surf_leaf)


def _store(c, bp, seq):
    """kf_add every keyframe; returns the stored (edge_ds, surf_ds) per keyframe."""
    kfs = []
    for i, (e, s, _) in enumerate(seq):
        kid, eds, sds = c.kf_add(bp, e, s)
        assert kid == i
        kfs.append((eds, sds))
    return kfs


def _edge_weight(bp, n):
    if bp.variant == 1:
        return float(np.float32(np.float32(np.float32(bp.lidar_const) * np.float32(200)) / np.float32(n)))
    return float(np.float32(bp.lidar_const))


def _check_window(c, O, bp, kfs, win_ids, poses_l, layers, bodies):
    """Window correspondences against the oracle searched on the oracle's layers; blocks against the oracle's reductions."""
    edge_map, surf_map = layers
    te, ts = O.KdTree(_f4(edge_map)), O.KdTree(_f4(surf_map))
    ne, ns = c.backend_window_correspond(bp, win_ids, poses_l)
    for slot, (i, pl) in enumerate(zip(win_ids, poses_l)):
        eds, sds = kfs[i]
        v_o, pa_o, pb_o = O.correspond_edge(te, eds, pl, bp.variant)
        v, pa, pb = c.backend_window_corr(slot, 0)
        assert np.array_equal(v, v_o) and int(v.sum()) == ne[slot]
        both = v == 1
        # line ends as an unordered pair: a = c + 0.1 u, b = c - 0.1 u (:1579-1580) with u an eigenvector, whose sign is not fixed
        # when the 5-NN set is nearly symmetric; LidarEdgeFactor is symmetric in a and b
        swap = np.abs(pa - pa_o).max(1) > np.abs(pa - pb_o).max(1)
        assert swap[both].sum() <= max(3, both.sum() // 50)
        pa_m, pb_m = np.where(swap[:, None], pb_o, pa_o), np.where(swap[:, None], pa_o, pb_o)
        np.testing.assert_allclose(pa[both], pa_m[both], rtol=5e-6, atol=1e-6)
        np.testing.assert_allclose(pb[both], pb_m[both], rtol=5e-6, atol=1e-6)
        refl = dict(map_refl=surf_map["curvature"], feat_refl=sds["curvature"], reflect_thres=bp.reflect_thres) if bp.variant == 0 else {}
        vs_o, pl_o, sc_o = O.correspond_surf_backend(ts, sds, pl, bp.kd_max_radius, bp.surf_dist_thres, bp.w_gate, bp.lidar_const, **refl)
        vs, pls, scs = c.backend_window_corr(slot, 1)
        assert np.array_equal(vs, vs_o) and int(vs.sum()) == ns[slot]
        both = vs == 1
        np.testing.assert_allclose(pls[both], pl_o[both], rtol=5e-6, atol=1e-6)
        np.testing.assert_allclose(scs[both], sc_o[both], rtol=1e-6, atol=1e-9)
    q_lb, t_lb = np.array(bp.q_lb[:]), np.array(bp.t_lb[:])
    for body in bodies:
        got = c.backend_window_blocks(body)
        for slot, i in enumerate(win_ids):
            eds, sds = kfs[i]
            v, pa, pb = c.backend_window_corr(slot, 0)
            ref = O.backend_edge_block(eds, v, pa, pb, _edge_weight(bp, ne[slot]), body[slot], bp.cauchy_b)
            assert got[slot, 0, 28] == ref[28] == ne[slot]
            np.testing.assert_allclose(got[slot, 0], ref, rtol=1e-8, atol=1e-9 * max(np.abs(ref[:21]).max(), 1e-30))
            vs, pls, scs = c.backend_window_corr(slot, 1)
            sc = scs * 1000.0 / np.float64(ns[slot]) if bp.variant == 1 else scs
            ref = O.backend_surf_block(sds, vs, pls, sc, body[slot], q_lb, t_lb, bp.cauchy_b)
            assert got[slot, 1, 28] == ref[28] == ns[slot]
            np.testing.assert_allclose(got[slot, 1], ref, rtol=1e-9, atol=1e-9 * max(np.abs(ref[:21]).max(), 1e-30))
    return ne, ns


# ---------------------------------------------------------------- keyframe store
@pytest.mark.parametrize("stride", [48, 32])
def test_kf_add_matches_voxelgrid_and_survives_regrowth(oracle, seq48, seq32, stride):
    import liliom_b200 as L
    from liliom_b200 import synth
    seq = seq48 if stride == 48 else seq32
    variant = 0 if stride == 48 else 1
    bp = L.backend_default_params(variant)
    c = L.Context(variant=variant)
    kfs = []
    for i, (e, s, _) in enumerate(seq):
        kid, eds, sds = c.kf_add(bp, e, s)
        assert kid == i and c.kf_count() == i + 1
        assert _bytes(eds) == _bytes(oracle.voxelgrid(e, bp.edge_leaf)) and _bytes(sds) == _bytes(oracle.voxelgrid(s, bp.surf_leaf))
        kfs.append((eds, sds))
    # empty clouds and non-finite points
    e, s, _ = seq[0]
    kid, eds, sds = c.kf_add(bp, e[:0], s[:0])
    assert kid == len(seq) and len(eds) == 0 and len(sds) == 0
    bad = s.copy(); bad["x"][::7] = np.nan; bad["z"][3::11] = np.inf
    kid, eds, sds = c.kf_add(bp, e[:0], bad)
    assert len(eds) == 0 and _bytes(sds) == _bytes(oracle.voxelgrid(bad, bp.surf_leaf))
    kfs += [(e[:0], s[:0]), (eds, sds)]
    # a stream long enough for the arena (1 MiB first, then doubling) to grow at least twice; no host download
    more = synth.make_keyframe_sequence(40, stride=stride, seed=11, surf_every=1)
    stored = sum(len(a) + len(b) for a, b in kfs)
    for e, s, _ in more:
        eds, sds = oracle.voxelgrid(e, bp.edge_leaf), oracle.voxelgrid(s, bp.surf_leaf)
        kid, _, _ = c.kf_add(bp, e, s, download=False)
        kfs.append((eds, sds))
        stored += len(eds) + len(sds)
    assert stored * stride > 4 << 20 and c.kf_count() == len(kfs)
    # every earlier keyframe intact: its cloud through kf_cloud at the identity, with a leaf small enough to keep every point
    ident = np.array([1.0, 0, 0, 0, 0, 0, 0])
    for i in list(range(0, len(kfs), 5)) + [len(kfs) - 1]:
        got = c.kf_cloud([i], [ident], 0.001)
        want = oracle.voxelgrid(_cat([oracle.transform_cloud(kfs[i][0], ident), oracle.transform_cloud(kfs[i][1], ident)], c.dtype), 0.001)
        assert _bytes(got) == _bytes(want), i
    c.kf_clear()
    assert c.kf_count() == 0
    with pytest.raises(L.LiliomError):
        c.bmap_build(bp, [0], [ident])
    c.close()


# ---------------------------------------------------------------- local map
@pytest.mark.parametrize("stride", [48, 32])
def test_bmap_build_matches_oracle_composition(oracle, seq48, seq32, stride):
    import liliom_b200 as L
    seq = seq48 if stride == 48 else seq32
    variant = 0 if stride == 48 else 1
    bp = L.backend_default_params(variant)
    c = L.Context(variant=variant)
    kfs = _store(c, bp, seq)
    poses = [p for _, _, p in seq]
    for ids in (list(range(8)), [7, 2, 5, 0, 3, 6, 1, 4], [3]):
        ps = [_nudge(poses[i], j) for j, i in enumerate(ids)]
        ne, ns = c.bmap_build(bp, ids, ps)
        we, ws = _oracle_layers(oracle, kfs, ids, ps, bp, c.dtype)
        assert (ne, ns) == (len(we), len(ws)) and ns > 500 and ne > 50
        assert _bytes(c.bmap_download(0)) == _bytes(we) and _bytes(c.bmap_download(1)) == _bytes(ws)
    # an unknown id: argument error, the previous layers stay
    with pytest.raises(L.LiliomError) as e:
        c.bmap_build(bp, [0, len(kfs)], [poses[0], poses[0]])
    assert e.value.code == L._binding.E_ARG
    assert _bytes(c.bmap_download(0)) == _bytes(we) and _bytes(c.bmap_download(1)) == _bytes(ws)
    # k = 0: empty layers, and the window gate (:933) refuses them
    assert c.bmap_build(bp, [], []) == (0, 0)
    assert len(c.bmap_download(0)) == 0 and len(c.bmap_download(1)) == 0
    with pytest.raises(L.LiliomError) as e:
        c.backend_window_correspond(bp, [0], [poses[0]])
    assert e.value.code == L._binding.E_FEWMAP
    # the odometry map is a separate index: installing it leaves the layers alone
    c.bmap_build(bp, [0, 1], poses[:2])
    e0, s0 = c.bmap_download(0), c.bmap_download(1)
    c.map_set_cloud(s0[:100])
    assert _bytes(c.bmap_download(0)) == _bytes(e0) and _bytes(c.bmap_download(1)) == _bytes(s0) and c.map_size() == 100
    c.close()


def test_kf_cloud_matches_oracle(oracle, seq48):
    import liliom_b200 as L
    bp = L.backend_default_params(0)
    c = L.Context(variant=0)
    kfs = _store(c, bp, seq48)
    ids = [9, 3, 12, 4]
    ps = [_nudge(seq48[i][2], j + 1) for j, i in enumerate(ids)]
    got = c.kf_cloud(ids, ps, 0.4)
    parts = []
    for i, p in zip(ids, ps):       # :2492-2493: edge THEN surf of each keyframe
        parts += [oracle.transform_cloud(kfs[i][0], p), oracle.transform_cloud(kfs[i][1], p)]
    want = oracle.voxelgrid(_cat(parts, c.dtype), 0.4)
    assert len(got) > 1000 and _bytes(got) == _bytes(want)
    assert len(c.kf_cloud([], [], 0.4)) == 0
    c.close()


# ---------------------------------------------------------------- window correspondences and blocks
@pytest.mark.parametrize("stride", [48, 32])
def test_window_against_oracle(oracle, seq48, seq32, stride):
    import liliom_b200 as L
    seq = seq48 if stride == 48 else seq32
    variant = 0 if stride == 48 else 1
    bp = L.backend_default_params(variant)
    c = L.Context(variant=variant)
    kfs = _store(c, bp, seq)
    poses = [p for _, _, p in seq]
    ids = list(range(2, 12))
    ne, ns = c.bmap_build(bp, ids, [poses[i] for i in ids])
    layers = (c.bmap_download(0), c.bmap_download(1))
    win = [9, 10, 11]
    poses_l = [_nudge(poses[i], 1) for i in win]
    bodies = [[_body_from_lidar(p, bp) for p in poses_l], [_nudge(_body_from_lidar(p, bp), 2) for p in poses_l]]
    cne, cns = _check_window(c, oracle, bp, kfs, win, poses_l, layers, bodies)
    assert cne.min() > 30 and cns.min() > 150, (cne, cns)
    # the blocks may be evaluated again and again (LM trial poses, marginalisation): same bits for the same poses
    assert _bytes(c.backend_window_blocks(bodies[0])) == _bytes(c.backend_window_blocks(bodies[0]))
    with pytest.raises(L.LiliomError):
        c.backend_window_blocks(bodies[0][:2])          # not the resident window's k
    c.close()


@pytest.mark.parametrize("variant", [0, 1])
def test_window_blocks_equal_the_single_keyframe_calls(seq48, seq32, variant):
    """bmap_download -> map_set_cloud -> correspond_* -> backend_*_block on the same context gives the same bits per keyframe
    (variant 0 both kinds, variant 1 the edge block: its surf weight has no single-keyframe form)."""
    import liliom_b200 as L
    seq = seq48 if variant == 0 else seq32
    bp = L.backend_default_params(variant)
    c = L.Context(variant=variant)
    kfs = _store(c, bp, seq)
    poses = [p for _, _, p in seq]
    c.bmap_build(bp, list(range(1, 11)), poses[1:11])
    win = [8, 9, 10]
    poses_l = [_nudge(poses[i], 1) for i in win]
    body = [_body_from_lidar(p, bp) for p in poses_l]
    ne, ns = c.backend_window_correspond(bp, win, poses_l)
    got = c.backend_window_blocks(body)
    edge_map, surf_map = c.bmap_download(0), c.bmap_download(1)
    q_lb, t_lb = np.array(bp.q_lb[:]), np.array(bp.t_lb[:])
    for slot, i in enumerate(win):
        eds, sds = kfs[i]
        c.map_set_cloud(edge_map)
        v, _, _ = c.correspond_edge(eds, poses_l[slot], variant)
        assert int(v.sum()) == ne[slot]
        e29 = c.backend_edge_block(body[slot], _edge_weight(bp, ne[slot]), bp.cauchy_b)
        assert _bytes(e29) == _bytes(got[slot, 0]), slot
        if variant == 0:
            c.map_set_cloud(surf_map)
            v, _, _ = c.correspond_surf_refl(sds, poses_l[slot], bp.kd_max_radius, bp.surf_dist_thres, bp.w_gate, bp.lidar_const, bp.reflect_thres)
            assert int(v.sum()) == ns[slot]
            s29 = c.backend_surf_block(body[slot], q_lb, t_lb, bp.cauchy_b)
            assert _bytes(s29) == _bytes(got[slot, 1]), slot
    c.close()


def test_deque_policy_sequence(oracle, seq48):
    """A Python mirror of buildLocalMapWithLandMark's deque (L/src/BackendFusion.cpp:1407-1477) with local_map_width = 5 over the
    16-keyframe stream: rebuild from current poses while fewer than 5 frames are held, then pop_front + push_back of the newest
    (older entries keep the pose they were transformed with), and a clear as correctPoses does after a loop closure (:2181-2182).
    Every step's layers equal the oracle composition; every window's correspondences and blocks match the oracle."""
    import liliom_b200 as L
    bp = L.backend_default_params(0)
    c = L.Context(variant=0)
    poses = [p.copy() for _, _, p in seq48]        # the optimiser's current keyframe poses, corrected a little at every step
    deque = []                                     # (keyframe id, pose it was transformed with)
    kfs = []
    regimes = set()
    for j, (e, s, _) in enumerate(seq48):
        kid, eds, sds = c.kf_add(bp, e, s)
        kfs.append((eds, sds))
        if j == 10:
            deque.clear()                          # correctPoses after a loop closure
            regimes.add("clear")
        if len(deque) < WIDTH:
            deque = [(i, poses[i].copy()) for i in range(max(0, j + 1 - WIDTH), j + 1)]
            regimes.add("rebuild")
        else:
            deque.pop(0)
            deque.append((j, poses[j].copy()))
            regimes.add("push")
        ids = [i for i, _ in deque]
        ps = [p for _, p in deque]
        ne, ns = c.bmap_build(bp, ids, ps)
        layers = _oracle_layers(oracle, kfs, ids, ps, bp, c.dtype)
        assert _bytes(c.bmap_download(0)) == _bytes(layers[0]) and _bytes(c.bmap_download(1)) == _bytes(layers[1]), j
        if j >= WINDOW:
            win = list(range(j - WINDOW, j))       # the reference's idx - 1 over the window
            poses_l = [poses[i] for i in win]
            bodies = [[_body_from_lidar(p, bp) for p in poses_l]]
            _check_window(c, oracle, bp, kfs, win, poses_l, layers, bodies)
        for i in range(max(0, j - WINDOW), j + 1):  # the window solve moves the recent poses
            poses[i] = _nudge(poses[i], 1)
    assert regimes == {"rebuild", "push", "clear"}
    c.close()
