"""Batched scan-to-map steps with per-session counts and either mode (liliom_scan_to_map_resident_batch_ex /
liliom_odometry_resident_batch_ex) against solo calls, bit for bit.

Twin context sets get the same maps and inputs; set A steps with solo calls (each with its own match_cnt and max_num_iter), set B
with one _ex call per step.  Per session and step the pose, status, every liliom_iter_stats entry (lm_iters included), the DS
cloud and (knn_queries, knn_candidates, launches) must be equal as bytes; after the batched steps one more solo call on both
sets checks the state the batch left in every context."""
import numpy as np
import pytest

from test_gpu_batch import (_check_counters, _close, _ctx, _ds_clouds, _feed_sweep, _same, _small_sessions, _twins,  # noqa: F401
                            world)

pytestmark = pytest.mark.gpu

CERES, GN = 0, 1


def _vec(v, B):
    return [int(v)] * B if np.isscalar(v) else [int(x) for x in v]


def _odo_solo(ctxs, poses, cnt, mni, mode):
    import liliom_b200 as L
    out = []
    for c, p, n, m in zip(ctxs, poses, _vec(cnt, len(ctxs)), _vec(mni, len(ctxs))):
        try:
            pose, st, ds = c.odometry_resident(p, n, max_num_iter=m, mode=mode, want_ds=True, cap=65536, want_stats=True)
            rc = 0
        except L.LiliomError as e:
            pose, st, ds, rc = np.array(p, dtype=np.float64), None, None, e.code
        out.append((pose, rc, st, ds))
    return out


def _odo_batch(ctxs, poses, cnt, mni, mode):
    import liliom_b200 as L
    P, status, st, ds = L.odometry_resident_batch_ex(ctxs, poses, cnt, mni, mode, want_stats=True, want_ds=True)
    return [(P[i], int(status[i]), st[i] if status[i] == 0 else None, ds[i] if status[i] == 0 else None) for i in range(len(ctxs))]


def _s2m_solo(ctxs, poses, cnt, mni, mode):
    import liliom_b200 as L
    out = []
    for c, p, n, m in zip(ctxs, poses, _vec(cnt, len(ctxs)), _vec(mni, len(ctxs))):
        try:
            pose, st = c.scan_to_map_resident(p, n, max_num_iter=m, mode=mode, want_stats=True)
            rc = 0
        except L.LiliomError as e:
            pose, st, rc = np.array(p, dtype=np.float64), None, e.code
        out.append((pose, rc, st, None))
    return out


def _s2m_batch(ctxs, poses, cnt, mni, mode):
    import liliom_b200 as L
    P, status, st = L.scan_to_map_resident_batch_ex(ctxs, poses, cnt, mni, mode, want_stats=True)
    return [(P[i], int(status[i]), st[i] if status[i] == 0 else None, None) for i in range(len(ctxs))]


def _run_s2m(A, Bs, feats, poses, cnt, mni, mode, steps=2):
    for step in range(steps):
        for i, f in enumerate(feats):
            A[i].upload_feats(f); Bs[i].upload_feats(f)
        ra, rb = _s2m_solo(A, poses, cnt, mni, mode), _s2m_batch(Bs, poses, cnt, mni, mode)
        _same(ra, rb, f"step {step}")
        _check_counters(A, Bs, f"step {step}")
    return rb


def _odo_steps(world, A, Bs, cnt, mni, mode, steps=3):
    B = len(A)
    for step in range(steps):
        sws = [world["sweeps"][(i + step) % len(world["sweeps"])] for i in range(B)]
        for i in range(B):
            _feed_sweep(A[i], Bs[i], sws[i])
        poses = np.array([s["guess"] for s in sws])
        ra, rb = _odo_solo(A, poses, cnt, mni, mode), _odo_batch(Bs, poses, cnt, mni, mode)
        _same(ra, rb, f"step {step}")
        _check_counters(A, Bs, f"step {step}")
        if mode == CERES:
            for i, r in enumerate(rb):
                assert r[1] == 0
                assert [s.lm_iters for s in r[2]] == [s.lm_iters for s in ra[i][2]]
    sw = world["sweeps"][0]
    for i in range(B):
        _feed_sweep(A[i], Bs[i], sw)
    _same(_odo_solo(A, [sw["guess"]] * B, cnt, mni, mode), _odo_solo(Bs, [sw["guess"]] * B, cnt, mni, mode), "solo after batch")
    _check_counters(A, Bs, "solo after batch")


def _maps(world, A, Bs):
    for i in range(len(A)):
        m = world["big"] if i % 2 == 0 else world["small"]
        A[i].map_set_points(m); Bs[i].map_set_points(m)


@pytest.mark.parametrize("B", [1, 2, 3, 8])
def test_ceres_odometry_batch_matches_solo(world, B):
    """Headline Horizon sessions in Ceres mode at the reference's configs (scan_match_cnt 2, max_num_iter 15), on a shared
    1 M-point map and 100 k-point maps, three consecutive steps, then a solo step on both sets."""
    A, Bs = _twins(B)
    _maps(world, A, Bs)
    _odo_steps(world, A, Bs, 2, 15, CERES)
    _close(A, Bs)


def test_ceres_mixed_counts(world):
    """Per-session counts in one call: 8 outer iterations (a session with fewer than two saved poses), 1, 2 and 0 (no kernel),
    and max_num_iter 15, 20, 1."""
    A, Bs = _twins(4)
    _maps(world, A, Bs)
    _odo_steps(world, A, Bs, [8, 1, 2, 0], [15, 20, 1, 15], CERES)
    _close(A, Bs)


def test_ceres_mixed_shapes_one_call(world):
    """A 16-lane Horizon session, an 8-lane HDL-64E session, a dense 60 k-query one-thread-per-query session and a 200-query
    one, 48-byte and 32-byte contexts together, with different counts."""
    ds = _ds_clouds(world)
    rng = np.random.default_rng(5)
    dense = world["small"][rng.choice(len(world["small"]), 60000, replace=False)].astype(np.float32)
    feats = [ds[0], ds[1], dense, ds[1][:200]]
    A, Bs = _twins(4, [0, 1, 0, 1])
    for c in A + Bs:
        c.map_set_points(world["small"])
    poses = [world["guess"]] * 4
    cnt, mni = [2, 8, 1, 2], [15, 20, 1, 15]
    rb = _run_s2m(A, Bs, feats, poses, cnt, mni, CERES)
    assert all(r[1] == 0 for r in rb)
    _same(_s2m_solo(A, poses, cnt, mni, CERES), _s2m_solo(Bs, poses, cnt, mni, CERES), "solo after batch")
    _close(A, Bs)


def test_ceres_more_sessions_than_one_table(world):
    feats, poses = _small_sessions(world, 40)
    cnt = [(1, 2, 8)[i % 3] for i in range(40)]
    A, Bs = _twins(40)
    for c in A + Bs:
        c.map_set_points(world["small"])
    rb = _run_s2m(A, Bs, feats, poses, cnt, 15, CERES, steps=3)
    assert all(r[1] == 0 for r in rb)
    _same(_s2m_solo(A, poses, cnt, 15, CERES), _s2m_solo(Bs, poses, cnt, 15, CERES), "solo after batch")
    _close(A, Bs)


def test_ceres_per_session_errors(world):
    """LILIOM_E_NOMAP and LILIOM_E_FEWMAP sessions keep their poses; the others run and match their solo calls."""
    A, Bs = _twins(4)
    for i in (0, 3):
        A[i].map_set_points(world["small"]); Bs[i].map_set_points(world["small"])
    A[2].map_set_points(world["small"][:5]); Bs[2].map_set_points(world["small"][:5])
    sws = world["sweeps"]
    for i in range(4):
        _feed_sweep(A[i], Bs[i], sws[i])
    poses = np.array([s["guess"] for s in sws])
    cnt = [2, 2, 8, 1]
    ra, rb = _odo_solo(A, poses, cnt, 15, CERES), _odo_batch(Bs, poses, cnt, 15, CERES)
    assert [r[1] for r in rb] == [0, -8, -3, 0]
    assert rb[1][0].tobytes() == poses[1].tobytes() and rb[2][0].tobytes() == poses[2].tobytes()
    _same(ra, rb, "errors")
    _check_counters(A, Bs, "errors")
    _close(A, Bs)


def test_ceres_caller_streams(world):
    import torch
    feats, poses = _small_sessions(world, 6)
    A, Bs = _twins(6)
    for c in A + Bs:
        c.map_set_points(world["small"])
    streams = [torch.cuda.Stream() for _ in range(3)]
    for k, i in enumerate((0, 2, 5)):
        Bs[i].set_stream(streams[k].cuda_stream)
    _run_s2m(A, Bs, feats, poses, [2, 8, 1, 2, 0, 2], 15, CERES)
    for s in streams:
        assert s.query()
    for c in Bs:
        c.set_stream(None)
    _close(A, Bs)


def test_ex_whole_call_refusals_change_nothing(world):
    import liliom_b200 as L
    A, Bs = _twins(2)
    for c in A + Bs:
        c.map_set_points(world["small"])
    sw = world["sweeps"][0]
    for i in range(2):
        _feed_sweep(A[i], Bs[i], sw)
    poses = np.array([sw["guess"]] * 2)
    before = poses.copy()
    refused = [
        ([], [], 15, CERES), ([Bs[0], None], 2, 15, CERES), ([Bs[0], Bs[0]], 2, 15, CERES),   # the existing refusals
        (Bs, None, 15, CERES),                   # NULL match_cnt
        (Bs, [2, -1], 15, CERES),                # a negative match_cnt[i]
        (Bs, 2, 15, 2), (Bs, 2, 15, -1),         # a mode other than CERES / GN
        (Bs, 2, None, CERES),                    # CERES with a NULL max_num_iter
    ]
    for ctxs, cnt, mni, mode in refused:
        P = poses[:len(ctxs)] if ctxs else np.zeros((0, 7))
        with pytest.raises(L.LiliomError) as e:
            L.odometry_resident_batch_ex(ctxs, P, cnt, mni, mode)
        assert e.value.code == -1
        with pytest.raises(L.LiliomError) as e:
            L.scan_to_map_resident_batch_ex(ctxs, P, cnt, mni, mode)
        assert e.value.code == -1
    assert poses.tobytes() == before.tobytes()
    _same(_odo_solo(A, poses, 2, 15, CERES), _odo_solo(Bs, poses, 2, 15, CERES), "solo after refusals")
    _check_counters(A, Bs, "solo after refusals")
    _close(A, Bs)


def test_gn_ex_uniform_matches_batch_call(world):
    """GN mode through _ex with one count (and max_num_iter NULL) gives the bits of liliom_odometry_resident_batch."""
    import liliom_b200 as L
    A, Bs = _twins(3)
    _maps(world, A, Bs)
    for step in range(2):
        sws = [world["sweeps"][(i + step) % len(world["sweeps"])] for i in range(3)]
        for i in range(3):
            _feed_sweep(A[i], Bs[i], sws[i])
        poses = np.array([s["guess"] for s in sws])
        P, status, st, ds = L.odometry_resident_batch(A, poses, 10, want_stats=True, want_ds=True)
        ra = [(P[i], int(status[i]), st[i], ds[i]) for i in range(3)]
        _same(ra, _odo_batch(Bs, poses, 10, None, GN), f"step {step}")
        _check_counters(A, Bs, f"step {step}")
    _close(A, Bs)


def test_gn_ex_mixed_counts_match_solo(world):
    """GN mode with per-session counts: sessions of equal counts share cooperative launches, and every session gets its solo
    call's bits; headline sessions and small ones."""
    A, Bs = _twins(4)
    _maps(world, A, Bs)
    _odo_steps(world, A, Bs, [10, 4, 0, 10], 15, GN, steps=2)
    _close(A, Bs)
    feats, poses = _small_sessions(world, 12)
    cnt = [(1, 4, 10, 0)[i % 4] for i in range(12)]
    A, Bs = _twins(12)
    for c in A + Bs:
        c.map_set_points(world["small"])
    rb = _run_s2m(A, Bs, feats, poses, cnt, 15, GN)
    assert all(r[1] == 0 for r in rb)
    _close(A, Bs)
