"""Batched scan-to-map steps (liliom_scan_to_map_resident_batch / liliom_odometry_resident_batch) against solo calls, bit for bit.

Twin context sets get the same maps and inputs; set A steps with solo calls, set B with one batch call per step.  Per session
and step the pose, status, every liliom_iter_stats entry, the DS cloud and the device-side query / candidate counts must be
equal as bytes; after the batched steps one more solo call on both sets checks the state the batch left in every context."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ITERS = 10


@pytest.fixture(scope="module")
def world():
    from liliom_b200 import synth
    big, _ = synth.make_map(1_000_000)
    small, _ = synth.make_map(100_000)
    T0 = synth.default_true_pose()
    sweeps = []
    for k in range(4):
        T = np.array(T0); T[4] += 0.7 * k; T[5] += 0.15 * k
        pts, q = synth.make_horizon_sweep(T, seed=1 + k)
        sweeps.append(dict(T=T, guess=synth.perturbed_pose(T), pts=pts, q=q))
    hdl, q_hdl = synth.make_hdl64_sweep(T0)
    return dict(big=big, small=small, sweeps=sweeps, hdl=hdl, q_hdl=q_hdl, guess=synth.perturbed_pose(T0))


def _ctx(variant=0):
    import liliom_b200 as L
    c = L.Context(variant=variant)
    c.set_kernel_timing(1)                                 # device-side query / candidate counts
    return c


def _stats_bytes(st):
    return None if st is None else [bytes(memoryview(s)) for s in st]


def _counts(c):
    k = c.counters()
    return (k.knn_queries, k.knn_candidates, k.launches)


def _twins(n, variant=0):
    return [_ctx(variant if np.isscalar(variant) else variant[i]) for i in range(n)], \
           [_ctx(variant if np.isscalar(variant) else variant[i]) for i in range(n)]


def _odo_solo(ctxs, poses):
    out = []
    for c, p in zip(ctxs, poses):
        import liliom_b200 as L
        try:
            pose, st, ds = c.odometry_resident(p, ITERS, mode=L.MODE_GN, want_ds=True, cap=65536, want_stats=True)
            rc = 0
        except L.LiliomError as e:
            pose, st, ds, rc = np.array(p, dtype=np.float64), None, None, e.code
        out.append((pose, rc, st, ds))
    return out


def _odo_batch(ctxs, poses):
    import liliom_b200 as L
    P, status, st, ds = L.odometry_resident_batch(ctxs, poses, ITERS, want_stats=True, want_ds=True)
    return [(P[i], int(status[i]), st[i] if status[i] == 0 else None, ds[i] if status[i] == 0 else None) for i in range(len(ctxs))]


def _same(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        assert x[1] == y[1], (what, i, x[1], y[1])
        assert x[0].tobytes() == y[0].tobytes(), (what, i, x[0], y[0])
        if x[1] == 0:
            assert _stats_bytes(x[2]) == _stats_bytes(y[2]), (what, i)
            if x[3] is not None:
                assert len(x[3]) == len(y[3]) and x[3].tobytes() == y[3].tobytes(), (what, i)


def _feed_sweep(ca, cb, sw):
    for c in (ca, cb):
        c.upload_scan(sw["pts"])
        c.extract_resident(sw["q"])


def _check_counters(A, B, what):
    for i, (a, b) in enumerate(zip(A, B)):
        assert _counts(a) == _counts(b), (what, i, _counts(a), _counts(b))


def _close(*sets):
    for s in sets:
        for c in s:
            c.close()


@pytest.mark.parametrize("B", [1, 2, 3, 8])
def test_odometry_batch_matches_solo(world, B):
    """Headline sessions: different sweeps and poses, a shared 1 M-point map and 100 k-point maps, three consecutive steps
    (the second and third size their launch from the previous scan's query count), then a solo step on both sets."""
    A, Bs = _twins(B)
    for i in range(B):
        m = world["big"] if i % 2 == 0 else world["small"]
        A[i].map_set_points(m); Bs[i].map_set_points(m)
    for step in range(3):
        sws = [world["sweeps"][(i + step) % len(world["sweeps"])] for i in range(B)]
        for i in range(B):
            _feed_sweep(A[i], Bs[i], sws[i])
        poses = np.array([s["guess"] for s in sws])
        ra, rb = _odo_solo(A, poses), _odo_batch(Bs, poses)
        _same(ra, rb, f"step {step}")
        assert all(r[1] == 0 for r in rb)
        _check_counters(A, Bs, f"step {step}")
    sw = world["sweeps"][0]
    for i in range(B):
        _feed_sweep(A[i], Bs[i], sw)
    _same(_odo_solo(A, [sw["guess"]] * B), _odo_solo(Bs, [sw["guess"]] * B), "solo after batch")
    _check_counters(A, Bs, "solo after batch")
    _close(A, Bs)


def _ds_clouds(world):
    """The headline Horizon DS cloud (48-byte) and a down-sampled HDL-64E cloud (32-byte), from solo odometry steps."""
    import liliom_b200 as L
    out = {}
    for variant, pts, q in ((0, world["sweeps"][0]["pts"], world["sweeps"][0]["q"]), (1, world["hdl"], world["q_hdl"])):
        c = L.Context(variant=variant)
        c.map_set_points(world["small"])
        c.upload_scan(pts)
        c.extract_resident(q)
        _, _, ds = c.odometry_resident(world["guess"], 1, mode=L.MODE_GN, want_ds=True, cap=len(pts))
        out[variant] = ds.copy()
        c.close()
    return out


def _s2m_solo(ctxs, poses):
    import liliom_b200 as L
    out = []
    for c, p in zip(ctxs, poses):
        try:
            pose, st = c.scan_to_map_resident(p, ITERS, mode=L.MODE_GN, want_stats=True)
            rc = 0
        except L.LiliomError as e:
            pose, st, rc = np.array(p, dtype=np.float64), None, e.code
        out.append((pose, rc, st, None))
    return out


def _s2m_batch(ctxs, poses):
    import liliom_b200 as L
    P, status, st = L.scan_to_map_resident_batch(ctxs, poses, ITERS, want_stats=True)
    return [(P[i], int(status[i]), st[i] if status[i] == 0 else None, None) for i in range(len(ctxs))]


def _run_s2m(A, Bs, feats, poses, steps=2):
    for step in range(steps):
        for i, f in enumerate(feats):
            A[i].upload_feats(f); Bs[i].upload_feats(f)
        ra, rb = _s2m_solo(A, poses), _s2m_batch(Bs, poses)
        _same(ra, rb, f"step {step}")
        _check_counters(A, Bs, f"step {step}")
    return rb


def test_mixed_shapes_one_call(world):
    """A 16-lane Horizon session, an 8-lane HDL-64E session (~3.1k queries), a dense session that is not persistent (its solo
    per-pass path inside the call) and a tiny one, 48-byte and 32-byte contexts together."""
    ds = _ds_clouds(world)
    hz = ds[0]
    hdl = ds[1]
    rng = np.random.default_rng(5)
    dense = world["small"][rng.choice(len(world["small"]), 60000, replace=False)].astype(np.float32)
    variants = [0, 1, 0, 1]
    feats = [hz, hdl, dense, hdl[:200]]
    A, Bs = _twins(4, variants)
    for c in A + Bs:
        c.map_set_points(world["small"])
    poses = [world["guess"]] * 4
    rb = _run_s2m(A, Bs, feats, poses)
    assert all(r[1] == 0 for r in rb)
    _same(_s2m_solo(A, poses), _s2m_solo(Bs, poses), "solo after batch")
    _close(A, Bs)


def test_per_session_errors(world):
    """A session without a map (LILIOM_E_NOMAP) and one with fewer than 10 map points (LILIOM_E_FEWMAP) keep their poses; the
    others run and match their solo calls."""
    A, Bs = _twins(4)
    for i in (0, 3):
        A[i].map_set_points(world["small"]); Bs[i].map_set_points(world["small"])
    A[2].map_set_points(world["small"][:5]); Bs[2].map_set_points(world["small"][:5])
    sws = world["sweeps"]
    for i in range(4):
        _feed_sweep(A[i], Bs[i], sws[i])
    poses = np.array([s["guess"] for s in sws])
    ra, rb = _odo_solo(A, poses), _odo_batch(Bs, poses)
    assert [r[1] for r in rb] == [0, -8, -3, 0]                # LILIOM_E_NOMAP, LILIOM_E_FEWMAP
    assert rb[1][0].tobytes() == poses[1].tobytes() and rb[2][0].tobytes() == poses[2].tobytes()
    _same(ra, rb, "errors")
    _check_counters(A, Bs, "errors")
    _close(A, Bs)


def test_whole_call_refusals_change_nothing(world):
    import liliom_b200 as L
    A, Bs = _twins(2)
    for c in A + Bs:
        c.map_set_points(world["small"])
    sw = world["sweeps"][0]
    for i in range(2):
        _feed_sweep(A[i], Bs[i], sw)
    poses = np.array([sw["guess"]] * 2)
    refused = [[], [Bs[0], None], [Bs[0], Bs[0]]]
    peer = _ctx()
    peer.map_set_points(world["small"])
    peer.comm_peer_attach([peer.comm_peer_export()], 0)
    refused.append([Bs[0], peer])
    comm = _ctx()
    try:
        comm.comm_init(L.comm_get_unique_id(), 1, 0)
        refused.append([Bs[1], comm])
    except Exception:
        pass                                            # no NCCL here: the fused-exchange context covers the communicator rule
    for ctxs in refused:
        with pytest.raises(L.LiliomError) as e:
            L.odometry_resident_batch(ctxs, poses[:len(ctxs)] if ctxs else np.zeros((0, 7)), ITERS)
        assert e.value.code == -1
        with pytest.raises(L.LiliomError) as e:
            L.scan_to_map_resident_batch(ctxs, poses[:len(ctxs)] if ctxs else np.zeros((0, 7)), ITERS)
        assert e.value.code == -1
    import torch
    if torch.cuda.device_count() > 1:
        other = L.Context(variant=0, device=1)
        with pytest.raises(L.LiliomError):
            L.scan_to_map_resident_batch([Bs[0], other], poses, ITERS)
        other.close()
    _same(_odo_solo(A, poses), _odo_solo(Bs, poses), "solo after refusals")
    _check_counters(A, Bs, "solo after refusals")
    _close(A, Bs, [peer, comm])


def _small_sessions(world, n):
    """n sessions of a few hundred queries each (grids of 3-30 blocks): several sessions share each cooperative launch."""
    hz = _ds_clouds(world)[0]
    rng = np.random.default_rng(11)
    feats = [hz[rng.choice(len(hz), int(k), replace=False)] for k in rng.integers(40, 480, n)]
    poses = [world["sweeps"][0]["guess"]] * n
    return feats, poses


def test_more_sessions_than_one_launch(world):
    feats, poses = _small_sessions(world, 40)
    A, Bs = _twins(40)
    for c in A + Bs:
        c.map_set_points(world["small"])
    rb = _run_s2m(A, Bs, feats, poses, steps=3)
    assert all(r[1] == 0 for r in rb)
    _same(_s2m_solo(A, poses), _s2m_solo(Bs, poses), "solo after batch")
    _close(A, Bs)


def test_caller_streams(world):
    """Sessions on caller-owned streams (liliom_set_stream) give the same bits, and the call returns with the work done."""
    import torch
    feats, poses = _small_sessions(world, 6)
    A, Bs = _twins(6)
    for c in A + Bs:
        c.map_set_points(world["small"])
    streams = [torch.cuda.Stream() for _ in range(3)]
    for k, i in enumerate((0, 2, 5)):
        Bs[i].set_stream(streams[k].cuda_stream)
    _run_s2m(A, Bs, feats, poses)
    for s in streams:
        assert s.query()                                   # nothing left pending on the caller's streams
    for c in Bs:
        c.set_stream(None)
    _close(A, Bs)
