"""GPU tier of the sharded map and search, on ONE GPU: n loopback ranks against one ordinary context.

LILIOM_TEST_LOOPBACK=<group>:<rank>/<nranks> makes a context rank `rank` of `nranks` contexts in this process; its all-reduce
meets the other ranks on the host (comm.cu) in place of NCCL, adding the ranks' vectors in rank order.  Each rank is called from
its own Python thread (ctypes releases the GIL), and a rank that is never called makes the others fail with LILIOM_E_NCCL after
LILIOM_TEST_LOOPBACK_MS instead of hanging.  Only host threads wait on each other: the fused peer exchange and the persistent
multi-rank kernel stay out of this tier (loopback contexts refuse liliom_comm_peer_attach), because two cooperative kernels on one
GPU, each waiting on the other's sums, can deadlock.  So every sharded pass here is k_knn_plane, the loopback all-reduce and
k_gn_update on each rank's own stream.

Checked against the single context: the installed shard (bytes and order), every query's correspondence on its owner rank (flag,
plane, neighbours bit for bit), every GN pass re-anchored at the single context's start pose, the maintained map over a 25-scan
stream with frames that straddle the push halo, the "< 10 map points" guard, PCL's declined and wrapping VoxelGrid boxes, and the
refusals of what is single-GPU only."""
import os
import threading
import uuid

import numpy as np
import pytest

import shard_adversarial as S
import vg_adversarial as V
from liliom_b200 import sharding

pytestmark = pytest.mark.gpu

IDENT = np.array([1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0])
WORLDS = S.worlds()


def _params(**kw):
    import liliom_b200 as L
    p = L.default_params(0)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def make_ranks(nranks, block, ms=None, **kw):
    """nranks loopback contexts of one fresh group, shard block `block` metres"""
    import liliom_b200 as L
    group = uuid.uuid4().hex
    out = []
    try:
        for r in range(nranks):
            os.environ["LILIOM_TEST_LOOPBACK"] = f"{group}:{r}/{nranks}"
            if ms is not None:
                os.environ["LILIOM_TEST_LOOPBACK_MS"] = str(ms)
            out.append(L.Context(_params(**kw)))
            out[-1].comm_set_shard_block(block)
    finally:
        os.environ.pop("LILIOM_TEST_LOOPBACK", None)
        os.environ.pop("LILIOM_TEST_LOOPBACK_MS", None)
    return out


def single(**kw):
    import liliom_b200 as L
    return L.Context(_params(**kw))


def close_all(cs):
    for c in cs:
        c.close()


def on_ranks(ctxs, fn, timeout=120.0):
    """fn(rank, ctx) on every rank, each from its own thread; returns the results in rank order (a LiliomError is returned as
    itself, any other exception re-raised).  Every thread is joined: none outlives the call."""
    import liliom_b200 as L
    res = [None] * len(ctxs)

    def run(r):
        try:
            res[r] = fn(r, ctxs[r])
        except L.LiliomError as e:
            res[r] = e
        except BaseException as e:        # noqa: B902 - re-raised below
            res[r] = _Raised(e)
    ts = [threading.Thread(target=run, args=(r,), daemon=True) for r in range(len(ctxs))]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout)
    assert not any(t.is_alive() for t in ts), "a rank did not return within the bound"
    for x in res:
        if isinstance(x, _Raised):
            raise x.e
    return res


class _Raised:
    def __init__(self, e):
        self.e = e


def code(x):
    import liliom_b200 as L
    return x.code if isinstance(x, L.LiliomError) else L._binding.OK


def rc_of(fn):
    import liliom_b200 as L
    try:
        fn()
        return L._binding.OK
    except L.LiliomError as e:
        return e.code


def restrict(m4, nranks, rank, block):
    """the rows of a downloaded map (float4) that rank's shard of it holds (shard_keep at the search radius), in order"""
    return m4[sharding.shard_mask(m4[:, :3], nranks, rank, halo=S.GATE_HALO, block=block)]


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ---- 1 + 2a: the installed map and every query's correspondence, on every adversarial world

@pytest.mark.parametrize("nranks", S.RANKS)
@pytest.mark.parametrize("name,block,base", WORLDS, ids=[w[0] for w in WORLDS])
def test_installed_shard_and_owner_correspondences(name, block, base, nranks):
    w = S.world(block, base)
    m, q = w["map"], w["queries"]
    one = single()
    ranks = make_ranks(nranks, block)
    try:
        one.map_set_points(m)
        full = one.map_download()
        assert np.array_equal(bits(full[:, :3]), bits(m[:, :3]))
        v1, p1, i1, d1, _ = one.find_surf_corr(q, IDENT)
        own = sharding.owner_of(q[:, :3], nranks, block)
        answered = np.zeros(len(q), int)
        for r, c in enumerate(ranks):
            c.map_set_points(m)
            got = c.map_download()
            want = restrict(full, nranks, r, block)
            assert got.tobytes() == want.tobytes(), f"{name} n={nranks} rank {r}: installed shard (x, y, z and w, in order)"
            v, p, i, d, _ = c.find_surf_corr(q, IDENT)
            mine = own == r
            answered += mine
            assert np.array_equal(v[mine], v1[mine]), f"{name} n={nranks} rank {r}: accept flags"
            assert np.array_equal(bits(p[mine]), bits(p1[mine])), f"{name} n={nranks} rank {r}: planes"
            assert np.array_equal(bits(d[mine]), bits(d1[mine])), f"{name} n={nranks} rank {r}: neighbour distances"
            # an installed shard keeps each point's installed index in w, and the search reports neighbours by that index
            assert np.array_equal(i[mine], i1[mine]), f"{name} n={nranks} rank {r}: neighbours"
            nb = i[mine & (v1 == 1)].ravel()
            loc = {int(x): j for j, x in enumerate(got[:, 3].view(np.int32))}
            assert np.array_equal(bits(got[[loc[x] for x in nb]][:, :3]), bits(full[nb][:, :3])), f"{name}: neighbour coordinates"
            assert not v[~mine].any() and (i[~mine] == -1).all(), f"{name} n={nranks} rank {r}: answered a query it does not own"
        assert (answered == 1).all()
        assert v1.sum() >= 15
    finally:
        close_all(ranks + [one])


# ---- 2b: every GN pass of a real scan, re-anchored at the single context's start pose

SEARCH = [(2, 16), (3, 8), (4, 64), (8, 256), (8, 8)]


@pytest.fixture(scope="module")
def scan_world():
    import oracle_lib as O
    from liliom_b200 import synth
    m, _ = synth.make_map(30000)
    T = synth.default_true_pose()
    pts, q = synth.make_horizon_sweep(T, seed=21)
    surf, _, _ = O.extract_horizon(pts, q)
    ds = O.voxelgrid(surf, 0.4)
    feats = np.ones((len(ds), 4), np.float32)
    feats[:, 0] = ds["x"]; feats[:, 1] = ds["y"]; feats[:, 2] = ds["z"]
    return m, feats, synth.perturbed_pose(T)


@pytest.mark.parametrize("nranks,block", SEARCH)
def test_gn_passes_reanchored(scan_world, nranks, block):
    import reanchor as RA
    m, feats, guess = scan_world
    iters = 4
    one = single()
    ranks = make_ranks(nranks, block)
    try:
        one.map_set_points(m)
        for c in ranks:
            c.map_set_points(m)
        _, st = one.scan_to_map(feats, guess, iters)
        starts = RA.start_poses(guess, st)
        for k, start in enumerate(starts):
            # the pass's correspondences: each query on its owner, bit for bit
            v1, p1, _, d1, _ = one.find_surf_corr(feats, start)
            pw = sharding.transform_f32(feats[:, :3], start)
            own = sharding.owner_of(pw, nranks, block)
            for r, c in enumerate(ranks):
                v, p, _, d, _ = c.find_surf_corr(feats, start)
                mine = own == r
                assert np.array_equal(v[mine], v1[mine]) and not v[~mine].any(), f"pass {k} rank {r}: accept flags"
                assert np.array_equal(bits(p[mine]), bits(p1[mine])) and np.array_equal(bits(d[mine]), bits(d1[mine])), f"pass {k} rank {r}"
            # the pass itself: one GN step through the all-reduce on every rank
            res = on_ranks(ranks, lambda r, c: c.scan_to_map(feats, start, 1))
            assert all(code(x) == 0 for x in res), [str(x) for x in res]
            poses = np.array([x[0] for x in res])
            assert all(p.tobytes() == poses[0].tobytes() for p in poses), f"pass {k}: ranks disagree on the pose"
            for pose, sts in res:
                s = sts[0]
                assert s.n_corr == st[k].n_corr, f"pass {k}: {s.n_corr} correspondences, one GPU {st[k].n_corr}"
                np.testing.assert_allclose(RA.sums29(s), RA.sums29(st[k]), rtol=RA.SUMS_RTOL, atol=RA.SUMS_ATOL)
            want, _, d, A = RA.gn_step(RA.sums29(st[k]), start)
            tol = RA.step_tolerance(start, d, A) if A is not None else np.zeros(7)
            dev = np.abs(RA.unify(poses[0]) - RA.unify(np.array(st[k].pose7)))
            assert (dev <= np.maximum(tol, 1e-9)).all(), f"pass {k}: pose {poses[0]} vs one GPU {list(st[k].pose7)} ({dev} > {tol})"
        assert st[0].n_corr > 100
    finally:
        close_all(ranks + [one])


# ---- 3: map maintenance over a 25-scan stream: the FIFO of 20 fills and pops, frames straddle the push halo

MAINT = [(2, 16, (0.0, 0.0)), (3, 8, (1e4, 1e4)), (4, 64, (-1e5, -1e4)), (8, 16, (1e5, -1e5)), (3, 256, (-1e4, 1e5))]


def _pt48(xyz, rng):
    import liliom_b200 as L
    a = np.zeros(len(xyz), L.PT48)
    a["x"], a["y"], a["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    a["w"] = 1.0
    a["intensity"] = rng.uniform(0, 100, len(xyz)).astype(np.float32)
    a["curvature"] = rng.uniform(0, 1, len(xyz)).astype(np.float32)
    return a


@pytest.mark.parametrize("nranks,block,base", MAINT)
def test_map_maintenance_stream(nranks, block, base):
    rng = np.random.default_rng(block + nranks)
    one = single()
    ranks = make_ranks(nranks, block)
    try:
        C = S.corner(block, base)
        for k in range(25):
            if k % 2 == 0:
                frame, pose = S.halo_frame(block, base, seed=k), IDENT      # world frame: the halo exactly where it was built
            else:
                frame = np.array(C + rng.uniform(-4, 4, (600, 3)), np.float32)
                pose = np.array([1.0, 0, 0, 0, 0.013 * k, -0.007 * k, 0.002 * k])
            pts = _pt48(frame, rng)
            n1 = one.map_update(pts, pose)
            res = on_ranks(ranks, lambda r, c: c.map_update(pts, pose))
            assert all(code(x) == 0 for x in res), [str(x) for x in res]
            full = one.map_download()
            assert len(full) == n1
            for r, c in enumerate(ranks):
                got = c.map_download()
                want = restrict(full, nranks, r, block)
                # x, y, z bit for bit and in order (w is an index into each context's own filtered cloud)
                assert got[:, :3].tobytes() == want[:, :3].tobytes(), f"scan {k} rank {r}: {len(got)} voxels, want {len(want)}"
    finally:
        close_all(ranks + [one])


# ---- 4: the "< 10 map points" guard counts the whole map's voxels, each once

def _voxel_map(n_vox, C, rng):
    """n_vox points in distinct 0.4 m voxels within 0.6 m of the corner: in the halo of several ranks' cubes"""
    cells = set()
    out = []
    while len(out) < n_vox:
        p = np.array(C + rng.uniform(-0.6, 0.6, 3), np.float32)
        key = tuple(np.floor(p / np.float32(0.4)).astype(int))
        if key not in cells:
            cells.add(key); out.append(p)
    return np.array(out, np.float32)


@pytest.mark.parametrize("n_vox", [6, 7, 8, 9, 10, 11, 12])
@pytest.mark.parametrize("nranks,block", [(2, 16), (3, 8), (4, 64), (8, 16)])
def test_map_size_guard(nranks, block, n_vox):
    import liliom_b200 as L
    rng = np.random.default_rng(n_vox * 31 + nranks)
    C = S.corner(block, (1e4, -1e4))
    pts = _pt48(_voxel_map(n_vox, C, rng), rng)
    feats = np.ones((40, 4), np.float32)
    feats[:, :3] = C + rng.uniform(-0.5, 0.5, (40, 3))
    one = single()
    ranks = make_ranks(nranks, block)
    try:
        assert one.map_update(pts, IDENT) == n_vox
        on_ranks(ranks, lambda r, c: c.map_update(pts, IDENT))
        want = rc_of(lambda: one.scan_to_map(feats, IDENT, 2))
        assert want == (L._binding.E_FEWMAP if n_vox < 10 else L._binding.OK)
        got = [code(x) for x in on_ranks(ranks, lambda r, c: c.scan_to_map(feats, IDENT, 2))]
        sizes = [c.map_size() for c in ranks]
        assert got == [want] * nranks, f"{n_vox} voxels, shard sizes {sizes}: ranks return {got}, one GPU {want}"
    finally:
        close_all(ranks + [one])


# ---- 5: PCL's declined and wrapping VoxelGrid boxes through a sharded map update

# (Not wrap_collide: there PCL merges two cells kilometres apart into one voxel, which no rank holds both halves of.)
VG_CASES = {"overflow_below": lambda: V.overflow_edge(0.4, False), "overflow_above": lambda: V.overflow_edge(0.4, True),
            "wrap_order": lambda: V.wrap_order(0.4)}


@pytest.mark.parametrize("nranks,block", [(2, 16), (3, 64), (8, 256)])
@pytest.mark.parametrize("name", list(VG_CASES))
def test_voxelgrid_boxes(name, nranks, block):
    cloud = np.ascontiguousarray(VG_CASES[name](), V.PT48)
    finite = np.isfinite(cloud["x"]) & np.isfinite(cloud["y"]) & np.isfinite(cloud["z"])
    cloud = cloud[finite]
    one = single()
    ranks = make_ranks(nranks, block)
    try:
        halves = np.array_split(cloud, 2)           # two frames: the box is the union of the frames' boxes
        for k, f in enumerate(halves):
            one.map_update(f, IDENT)
            res = on_ranks(ranks, lambda r, c: c.map_update(f, IDENT))
            assert all(code(x) == 0 for x in res), [str(x) for x in res]
            full = one.map_download()
            for r, c in enumerate(ranks):
                got = c.map_download()
                want = restrict(full, nranks, r, block)
                assert got[:, :3].tobytes() == want[:, :3].tobytes(), f"{name} frame {k} rank {r}: {len(got)} voxels, want {len(want)}"
    finally:
        close_all(ranks + [one])


# ---- 6: refusals

def test_single_gpu_calls_refuse_sharded_contexts(scan_world):
    import liliom_b200 as L
    B = L._binding
    m, feats, guess = scan_world
    ranks = make_ranks(3, 16)
    try:
        for c in ranks:
            c.map_set_points(m)
        pose_in = np.array(guess)
        res = on_ranks(ranks, lambda r, c: c.scan_to_map(feats, pose_in, 2, mode=L.MODE_CERES))
        assert [code(x) for x in res] == [B.E_ARG] * 3
        assert np.array_equal(pose_in, guess)
        for c in ranks:
            assert rc_of(lambda: c.icp_align(m[:100], m[:200])) == B.E_ARG
            assert rc_of(lambda: c.kf_add(L.backend_default_params(0), np.zeros(10, L.PT48), np.zeros(10, L.PT48))) == B.E_ARG
            assert rc_of(lambda: c.map_download_cloud()) == B.E_ARG
            assert rc_of(lambda: c.map_set_cloud(np.zeros(20, L.PT48))) == B.E_ARG
            assert rc_of(lambda: c.comm_peer_attach([c.comm_peer_export()] * 3, c_rank(ranks, c))) == B.E_ARG
        # the sharded step still runs after the refusals
        res = on_ranks(ranks, lambda r, c: c.scan_to_map(feats, guess, 1))
        assert [code(x) for x in res] == [B.OK] * 3
    finally:
        close_all(ranks)


def c_rank(ranks, c):
    return ranks.index(c)


def test_forgotten_rank_fails_within_the_bound(scan_world):
    import time
    import liliom_b200 as L
    B = L._binding
    m, feats, guess = scan_world
    ranks = make_ranks(3, 16, ms=300)
    try:
        for c in ranks:
            c.map_set_points(m)
        t0 = time.monotonic()
        res = on_ranks(ranks[:2], lambda r, c: c.scan_to_map(feats, guess, 1), timeout=30.0)
        assert [code(x) for x in res] == [B.E_NCCL] * 2 and "did not gather" in str(res[0])
        # all three ranks together still meet
        res = on_ranks(ranks, lambda r, c: c.scan_to_map(feats, guess, 1))
        assert [code(x) for x in res] == [B.OK] * 3
        # the map rebuild's all-reduce (the ranks' maps are then gone: the rebuild reset them before it failed)
        res = on_ranks(ranks[:2], lambda r, c: c.map_update(np.zeros(0, L.PT48), IDENT), timeout=30.0)
        assert [code(x) for x in res] == [B.E_NCCL] * 2
        assert time.monotonic() - t0 < 10.0
    finally:
        close_all(ranks)


def test_malformed_loopback_spec_refuses_the_context():
    import liliom_b200 as L
    for bad in ("g:0/1", "g:2/2", "g:-1/2", ":0/2", "g:0/2x", "g0/2", "g:0/65"):
        os.environ["LILIOM_TEST_LOOPBACK"] = bad
        try:
            with pytest.raises(L.LiliomError) as e:
                L.Context()
            assert e.value.code == L._binding.E_ARG, bad
        finally:
            os.environ.pop("LILIOM_TEST_LOOPBACK", None)
