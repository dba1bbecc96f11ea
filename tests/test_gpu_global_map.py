"""GPU parity for the keyframes' full clouds (liliom_kf_add_full) and the global map (liliom_global_map): publishCompleteMap and
save_pcd's map through the C ABI, bit-exact against the oracle composition voxelgrid(concat(transform_cloud(...))) in both
point layouts and both variants; PCL's declined case against the transformed concatenation; the error returns; and an at-size
map whose stored clouds and output both pass 2^31 bytes."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

IDENT = np.array([1.0, 0, 0, 0, 0, 0, 0])
TINY_LEAF = 1e-4          # PCL declines every keyframe-sized cloud at this leaf: the output is the transformed input


@pytest.fixture(scope="module")
def seqs():
    from liliom_b200 import synth
    return {s: synth.make_keyframe_sequence(16, stride=s, full=True) for s in (48, 32)}


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def _nudge(pose, k):
    from liliom_b200 import synth
    dq = synth.q_from_axis_angle([1, -1, 2], np.deg2rad(0.15 * k))
    return np.concatenate([synth.qmul(pose[:4], dq), pose[4:] + 0.01 * k * np.array([1.0, -0.5, 0.25])])


def _oracle_map(O, clouds, ids, poses, leaf, dtype, pre7=None):
    parts = []
    for i, p in zip(ids, poses):
        c = clouds[i] if pre7 is None else O.transform_cloud(clouds[i], pre7)
        if len(c):
            parts.append(O.transform_cloud(c, p))
    cat = np.concatenate(parts) if parts else np.zeros(0, dtype)
    return O.voxelgrid(cat, leaf), cat


def _store(c, bp, seq):
    """kf_add + kf_add_full of every keyframe; returns the stored full clouds as the oracle computes them"""
    import oracle_lib as O
    full = []
    for i, (e, s, _, f) in enumerate(seq):
        kid, _, _ = c.kf_add(bp, e, s, download=False)
        assert kid == i
        want = f if bp.variant == 0 else O.voxelgrid(f, bp.surf_leaf)
        assert c.kf_add_full(bp, kid, f) == len(want)
        full.append(want)
    return full


def _raw_global_map(c, kind, ids, poses, leaf, pre7=None, out=None, cap=0):
    import liliom_b200 as L
    ids = np.ascontiguousarray(ids, np.int32)
    p = np.ascontiguousarray(np.asarray(poses, np.float64).reshape(-1, 7)) if len(ids) else np.zeros((1, 7))
    pre = None if pre7 is None else np.ascontiguousarray(pre7, np.float64)
    n = C.c_int(-7)
    rc = L._binding.lib().liliom_global_map(c._h, kind, ids.ctypes.data_as(C.POINTER(C.c_int)), p.ctypes.data_as(C.POINTER(C.c_double)),
                                            len(ids), None if pre is None else pre.ctypes.data_as(C.POINTER(C.c_double)), leaf,
                                            None if out is None else out.ctypes.data_as(C.c_void_p), cap, C.byref(n))
    return rc, n.value


@pytest.mark.parametrize("stride", [48, 32])
def test_kf_add_full_stores_and_survives_regrowth(oracle, seqs, stride):
    """variant 0 stores the cloud as received, variant 1 VoxelGrid(surf_leaf) of it; 16 clouds of ~1 MB grow the 1 MiB arena
    several times (copying); a second attach is refused and changes nothing; kf_clear drops the full clouds"""
    import liliom_b200 as L
    seq = seqs[stride]
    variant = 0 if stride == 48 else 1
    bp = L.backend_default_params(variant)
    c = L.Context(variant=variant)
    full = _store(c, bp, seq)
    assert sum(len(f) for f in full) * stride > (4 << 20) or variant == 1
    for i in range(len(seq)):                             # each stored cloud, read back through the declined (copying) path
        got = c.global_map(L.KF_FULL, [i], [IDENT], TINY_LEAF)
        assert _bytes(got) == _bytes(oracle.transform_cloud(full[i], IDENT)), i
    before = c.global_map(L.KF_FULL, [3, 5], [seq[3][2], seq[5][2]], 0.3)
    with pytest.raises(L.LiliomError) as e:
        c.kf_add_full(bp, 3, seq[0][3])
    assert e.value.code == L._binding.E_ARG
    assert _bytes(c.global_map(L.KF_FULL, [3, 5], [seq[3][2], seq[5][2]], 0.3)) == _bytes(before)
    with pytest.raises(L.LiliomError) as e:
        c.kf_add_full(bp, len(seq), seq[0][3])          # unknown keyframe
    assert e.value.code == L._binding.E_ARG
    c.kf_clear()
    assert c.kf_count() == 0
    e0, s0, _, f0 = seq[0]
    kid, _, _ = c.kf_add(bp, e0, s0, download=False)
    with pytest.raises(L.LiliomError) as e:
        c.global_map(L.KF_FULL, [kid], [IDENT], 0.3)     # the new keyframe 0 has no full cloud: the old one is gone
    assert e.value.code == L._binding.E_ARG
    assert c.kf_add_full(bp, kid, f0[:0]) == 0           # an empty full cloud is a full cloud
    assert len(c.global_map(L.KF_FULL, [kid], [IDENT], 0.3)) == 0
    c.close()


@pytest.mark.parametrize("stride", [48, 32])
def test_global_map_full_matches_oracle(oracle, seqs, stride):
    import liliom_b200 as L
    seq = seqs[stride]
    variant = 0 if stride == 48 else 1
    bp = L.backend_default_params(variant)
    c = L.Context(variant=variant)
    full = _store(c, bp, seq)
    leaf = 0.3 if variant == 0 else 0.2                   # mapping_ds (L:568) / the hard-coded 0.2 of R:496
    for ids in (list(range(0, 16, 7)), list(range(0, 16, 2)), [4, 4, 9, 4]):
        poses = [_nudge(seq[i][2], j) for j, i in enumerate(ids)]
        got = c.global_map(L.KF_FULL, ids, poses, leaf)
        want, cat = _oracle_map(oracle, full, ids, poses, leaf, c.dtype)
        assert len(want) < len(cat) and _bytes(got) == _bytes(want), ids
    assert len(c.global_map(L.KF_FULL, [], [], leaf)) == 0
    c.close()


@pytest.mark.parametrize("stride", [48, 32])
def test_global_map_surf_with_tbl(oracle, seqs, stride):
    """save_pcd: transform_cloud(transform_cloud(surf, Tbl), pose) of every keyframe, concatenated, filtered"""
    import liliom_b200 as L
    seq = seqs[stride]
    variant = 0 if stride == 48 else 1
    bp = L.backend_default_params(variant)
    c = L.Context(variant=variant)
    surf = [c.kf_add(bp, e, s)[2] for e, s, _, _ in seq]
    tbl = np.concatenate([np.array(bp.q_lb[:]), np.array(bp.t_lb[:])])
    ids = list(range(16))
    poses = [_nudge(seq[i][2], 1) for i in ids]
    for leaf in (0.3, 0.2):
        got = c.global_map(L.KF_SURF, ids, poses, leaf, pre7=tbl)
        want, _ = _oracle_map(oracle, surf, ids, poses, leaf, c.dtype, pre7=tbl)
        assert len(got) > 1000 and _bytes(got) == _bytes(want)
    c.close()


@pytest.mark.parametrize("stride", [48, 32])
def test_declined_map_is_the_transformed_concatenation(oracle, seqs, stride):
    import liliom_b200 as L
    seq = seqs[stride]
    variant = 0 if stride == 48 else 1
    bp = L.backend_default_params(variant)
    c = L.Context(variant=variant)
    full = _store(c, bp, seq)
    ids = [0, 6, 6, 11, 15]
    poses = [_nudge(seq[i][2], j) for j, i in enumerate(ids)]
    got = c.global_map(L.KF_FULL, ids, poses, 0.004)
    want, cat = _oracle_map(oracle, full, ids, poses, 0.004, c.dtype)
    assert len(got) == len(cat) and _bytes(want) == _bytes(cat) and _bytes(got) == _bytes(cat)
    c.close()


def test_error_returns_and_size_query(oracle, seqs):
    import liliom_b200 as L
    seq = seqs[48]
    bp = L.backend_default_params(0)
    c = L.Context(variant=0)
    full = _store(c, bp, seq[:6])
    kid, _, _ = c.kf_add(bp, seq[6][0], seq[6][1], download=False)        # keyframe 6: no full cloud
    ids = [0, 2, 4]
    poses = [seq[i][2] for i in ids]
    ref = c.global_map(L.KF_FULL, ids, poses, 0.3)
    want, _ = _oracle_map(oracle, full, ids, poses, 0.3, c.dtype)
    assert _bytes(ref) == _bytes(want)
    # the size query and the capacity check: test_gpu_abi_contract.py
    for bad_ids in ([0, 99], [0, kid], [-1]):
        rc, n = _raw_global_map(c, L.KF_FULL, bad_ids, [IDENT] * len(bad_ids), 0.3)
        assert (rc, n) == (L._binding.E_ARG, -7), bad_ids
    # 2^31 listed points: one keyframe listed over and over
    reps = (1 << 31) // len(full[0]) + 1
    rc, n = _raw_global_map(c, L.KF_FULL, np.zeros(reps, np.int32), np.tile(IDENT, (reps, 1)), 0.3)
    assert (rc, n) == (L._binding.E_CAPACITY, -7)
    assert _raw_global_map(c, L.KF_FULL, ids, poses, 0.0)[0] == L._binding.E_ARG
    assert _raw_global_map(c, 2, ids, poses, 0.3)[0] == L._binding.E_ARG
    # nothing changed
    assert c.kf_count() == 7 and _bytes(c.global_map(L.KF_FULL, ids, poses, 0.3)) == _bytes(ref)
    c.close()


# ---------------------------------------------------------------- at size: > 2^31 bytes stored and published
def _np_transform(cloud, pose):
    """transformCloud in NumPy float64 with the operation order of pcl_xform.h (NumPy never fuses): xyz, normal, w = 1,
    intensity/curvature copied, padding cleared"""
    q, t = np.asarray(pose[:4], np.float64), np.asarray(pose[4:], np.float64)

    def rot(x, y, z):
        ux, uy, uz = q[2] * z - q[3] * y, q[3] * x - q[1] * z, q[1] * y - q[2] * x
        ux, uy, uz = ux + ux, uy + uy, uz + uz
        cx, cy, cz = q[2] * uz - q[3] * uy, q[3] * ux - q[1] * uz, q[1] * uy - q[2] * ux
        return (x + q[0] * ux) + cx, (y + q[0] * uy) + cy, (z + q[0] * uz) + cz

    out = np.zeros(len(cloud), cloud.dtype)
    x, y, z = rot(cloud["x"].astype(np.float64), cloud["y"].astype(np.float64), cloud["z"].astype(np.float64))
    out["x"], out["y"], out["z"], out["w"] = (x + t[0]).astype(np.float32), (y + t[1]).astype(np.float32), (z + t[2]).astype(np.float32), 1.0
    out["intensity"] = cloud["intensity"]
    if "nx" in cloud.dtype.names:
        nx, ny, nz = rot(cloud["nx"].astype(np.float64), cloud["ny"].astype(np.float64), cloud["nz"].astype(np.float64))
        out["nx"], out["ny"], out["nz"] = nx.astype(np.float32), ny.astype(np.float32), nz.astype(np.float32)
        out["curvature"] = cloud["curvature"]
    return out


def test_at_size_map_past_2_31_bytes(oracle):
    """~46M 48-byte points (2.2 GB) of full clouds, a dozen sweeps reused along a 3.4 km path: PCL declines at a 1 cm leaf and
    the 2.2 GB output is checked keyframe by keyframe against the NumPy transform; at 0.5 m the whole list is filtered and
    checked against the oracle composition."""
    import liliom_b200 as L
    from liliom_b200 import synth
    sweeps = [kf[3] for kf in synth.make_keyframe_sequence(12, stride=48, seed=3, full=True)]
    T0 = synth.default_true_pose()
    n_kf = (46_000_000 + 20_000) // 20_000
    poses = []
    for i in range(n_kf):
        q = synth.qmul(synth.q_from_axis_angle([0, 0, 1], np.deg2rad(2.0 * i)), T0[:4])
        poses.append(np.concatenate([q, T0[4:] + np.array([1.5 * i, 0.35 * np.sin(0.4 * i), 0.0])]))
    bp = L.backend_default_params(0)
    c = L.Context(variant=0)
    empty = sweeps[0][:0]
    for i in range(n_kf):
        kid, _, _ = c.kf_add(bp, empty, empty, download=False)
        c.kf_add_full(bp, kid, sweeps[i % len(sweeps)])
    sizes = np.array([len(sweeps[i % len(sweeps)]) for i in range(n_kf)])
    N = int(sizes.sum())
    assert N * 48 > (1 << 31) and N < (1 << 31)
    ids = list(range(n_kf))
    # np.transform against the oracle's transformCloud first (the NumPy restatement is the yardstick below)
    assert _bytes(_np_transform(sweeps[1], poses[77])) == _bytes(oracle.transform_cloud(sweeps[1], poses[77]))
    got = c.global_map(L.KF_FULL, ids, poses, 0.01)
    assert len(got) == N and got.nbytes > (1 << 31)
    off = 0
    for i in range(n_kf):
        s = sweeps[i % len(sweeps)]
        assert _bytes(got[off:off + len(s)]) == _bytes(_np_transform(s, poses[i])), i
        off += len(s)
    del got
    got = c.global_map(L.KF_FULL, ids, poses, 0.5)
    cat = np.concatenate([oracle.transform_cloud(sweeps[i % len(sweeps)], poses[i]) for i in ids])
    want = oracle.voxelgrid(cat, 0.5)
    del cat
    assert 0 < len(got) < N // 10 and _bytes(got) == _bytes(want)
    c.close()
