"""GPU tier of the collective LM (Ceres mode on a sharded context, liliom_comm_set_ceres), on ONE GPU: loopback ranks
(LILIOM_TEST_LOOPBACK, see test_gpu_sharded.py) against one ordinary context.

Each outer iteration runs k_knn_plane on every rank, the all-reduce of the linearisation sums, 1 + max_num_iter rounds of
[k_lm_eval_part, the all-reduce of its 29 sums, k_lm_advance] and k_lm_end.  The ranks' sums are added in rank order, so every
rank holds the same pose bits, but not one GPU's: each outer iteration is checked against one GPU from the ranks' own start
(n_corr exactly, the sums at reanchor's tolerances), and LM iteration by LM iteration against the oracle's trust-region loop
(reanchor.check_ceres with the ranks' own capped solves), on the scan world of test_gpu_sharded.py and on every adversarial LM
world of lm_adversarial.py.  Then the guards (map size, no map, match_cnt 0, max_num_iter 0, no correspondence), a rank that is
never called, and the odometry calls on the ranks: extract + odometry_resident, a stream with map updates, the LidarOdometry
node."""
import json

import numpy as np
import pytest

import lm_adversarial as LA
import reanchor as RA
from liliom_b200 import sharding
from test_gpu_reanchored import probe_of
from test_gpu_sharded import SEARCH, _pt48, _voxel_map, close_all, code, make_ranks, on_ranks, rc_of, scan_world, single  # noqa: F401
import shard_adversarial as S

pytestmark = pytest.mark.gpu

IDENT = np.array([1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0])
OUTER, LM = 2, 15


def ceres_ranks(nranks, block, ms=None, **kw):
    ranks = make_ranks(nranks, block, ms, **kw)
    for c in ranks:
        c.comm_set_ceres(1)
    return ranks


def _ceres_on(ranks, fn):
    """fn(rank, ctx) -> (pose, stats) on every rank: all succeed and agree bit for bit (pose and every stats row)."""
    res = on_ranks(ranks, fn)
    assert all(code(x) == 0 for x in res), [str(x) for x in res]
    pose0, st0 = res[0][0], res[0][1]
    for r, (pose, st) in enumerate(res):
        assert pose.tobytes() == pose0.tobytes(), f"rank {r} pose {pose} vs rank 0 {pose0}"
        if st is not None:
            assert [bytes(s) for s in st] == [bytes(s) for s in st0], f"rank {r}: stats differ from rank 0's"
    return pose0, st0


def truncated_on(ranks, feats):
    """The ranks' match_cnt = 1 call from `start` capped at j LM iterations (reanchor.check_ceres): (pose, iterations)."""
    import liliom_b200 as L

    def run(start, j):
        pose, st = _ceres_on(ranks, lambda r, c: c.scan_to_map(feats, start, 1, max_num_iter=j, mode=L.MODE_CERES))
        return pose, st[0].lm_iters
    return run


def _pose_close(a, b, tol=1e-4):
    a, b = RA.unify(a), RA.unify(b)
    return np.linalg.norm(a[4:] - b[4:]) < tol and 2 * np.arccos(min(1.0, abs(float(np.dot(a[:4], b[:4]))))) < tol


# ---- the setting

def test_setting_and_default(scan_world):
    import liliom_b200 as L
    B = L._binding
    m, feats, guess = scan_world
    ranks = make_ranks(2, 16)
    one = single()
    try:
        for c in ranks:
            c.map_set_points(m)
        call = lambda r, c: c.scan_to_map(feats, guess, 2, max_num_iter=LM, mode=L.MODE_CERES)  # noqa: E731
        assert [code(x) for x in on_ranks(ranks, call)] == [B.E_ARG] * 2          # the default: refused, as before the setting
        for bad in (2, -1, 7):
            assert rc_of(lambda: ranks[0].comm_set_ceres(bad)) == B.E_ARG
            assert rc_of(lambda: one.comm_set_ceres(bad)) == B.E_ARG
        assert rc_of(lambda: one.comm_set_ceres(1)) == B.OK                       # any context, any time
        for c in ranks:
            c.comm_set_ceres(1)
        assert [code(x) for x in on_ranks(ranks, call)] == [B.OK] * 2
        for c in ranks:
            c.comm_set_ceres(0)
        assert [code(x) for x in on_ranks(ranks, call)] == [B.E_ARG] * 2
        # a context without a communicator ignores the setting
        one.map_set_points(m)
        p1, s1 = one.scan_to_map(feats, guess, 2, max_num_iter=LM, mode=L.MODE_CERES)
        one.comm_set_ceres(0)
        p0, s0 = one.scan_to_map(feats, guess, 2, max_num_iter=LM, mode=L.MODE_CERES)
        assert p1.tobytes() == p0.tobytes() and [bytes(s) for s in s1] == [bytes(s) for s in s0]
    finally:
        close_all(ranks + [one])


# ---- the scan world of test_gpu_sharded.py at every (nranks, block) of its search list

@pytest.mark.parametrize("nranks,block", SEARCH)
def test_scan_world_every_outer_iteration(oracle, scan_world, nranks, block):
    import liliom_b200 as L
    m, feats, guess = scan_world
    one, pc = single(), single()
    ranks = ceres_ranks(nranks, block)
    try:
        for c in ranks + [one, pc]:
            c.map_set_points(m)
        pose, st = _ceres_on(ranks, lambda r, c: c.scan_to_map(feats, guess, OUTER, max_num_iter=LM, mode=L.MODE_CERES))
        assert np.array_equal(pose, RA.unify(np.array(st[-1].pose7)))
        for k, start in enumerate(RA.start_poses(guess, st)):
            _, s1 = one.scan_to_map(feats, start, 1, max_num_iter=LM, mode=L.MODE_CERES)
            assert st[k].n_corr == s1[0].n_corr, f"outer {k}: {st[k].n_corr} correspondences, one GPU {s1[0].n_corr}"
            np.testing.assert_allclose(RA.sums29(st[k]), RA.sums29(s1[0]), rtol=RA.SUMS_RTOL, atol=RA.SUMS_ATOL)
        pw = sharding.transform_f32(feats[:, :3], guess)
        assert len(set(sharding.owner_of(pw, nranks, block).tolist())) > 1          # the queries straddle owners
        rep = RA.check_ceres(oracle, oracle.KdTree(m), feats, guess, st, LM, 8, f"sharded ceres {nranks}x{block}", probe_of(pc, feats),
                             truncated_on(ranks, feats))
        assert rep.get("bound_over_step", 0.0) < 1e-6, rep
        p1, _ = one.scan_to_map(feats, guess, OUTER, max_num_iter=LM, mode=L.MODE_CERES)
        assert _pose_close(pose, p1), (pose, p1)
        print(f"sharded_ceres {nranks}x{block} " + json.dumps({k: v for k, v in rep.items() if isinstance(v, float)}))
        assert st[0].n_corr > 100
    finally:
        close_all(ranks + [one, pc])


# ---- every adversarial LM world on 2 and 3 ranks

# (2, 8): every world's sites straddle both owners; (3, 64): rank 1 owns no correspondence (and on single_wall rank 0 owns
# them all), so one rank only ever contributes zeros
LM_SHARDS = [(2, 8), (3, 64)]


def _lm_world(oracle, name, nranks, block):
    import liliom_b200 as L
    fn, mni, _, _ = LA.WORLDS[name]
    m, feats, guess = fn()
    tree = oracle.KdTree(m)
    _, v, _, _, _ = oracle.find_surf_corr(tree, feats, guess)
    owned = np.bincount(sharding.owner_of(sharding.transform_f32(feats[:, :3], guess)[v == 1], nranks, block), minlength=nranks)
    pc = single()
    ranks = ceres_ranks(nranks, block)
    try:
        for c in ranks + [pc]:
            c.map_set_points(m)
        pose, st = _ceres_on(ranks, lambda r, c: c.scan_to_map(feats, guess, 1, max_num_iter=mni, mode=L.MODE_CERES))
        rep = RA.check_ceres(oracle, tree, feats, guess, st, mni, 8, f"lm/{name}/{nranks}x{block}", probe_of(pc, feats),
                             truncated_on(ranks, feats))
        return dict(rep=rep, pose=pose, guess=guess, lm_iters=st[0].lm_iters, owned=owned.tolist())
    finally:
        close_all(ranks + [pc])


@pytest.fixture(scope="module")
def lm_runs(oracle):
    return {(name, nr, b): _lm_world(oracle, name, nr, b) for name in LA.WORLDS for nr, b in LM_SHARDS}


@pytest.mark.parametrize("nranks,block", LM_SHARDS)
@pytest.mark.parametrize("name", list(LA.WORLDS))
def test_lm_world_on_ranks(lm_runs, name, nranks, block):
    _, _, stop, branches = LA.WORLDS[name]
    d = lm_runs[(name, nranks, block)]
    rep = d["rep"]
    assert rep.get("bound_over_step", 0.0) < 1e-6, rep
    assert rep.get("open_decisions", 0) == (1 if name == "parameter_edge" else 0), rep
    if stop:
        assert rep["stops"] == [stop], rep["stops"]
    for b in branches:
        assert b in rep["branches"], rep["branches"]
    if name == "zero_residual":
        assert np.array_equal(d["pose"], d["guess"]) and d["lm_iters"] == 0
    if name != "no_corr":
        assert sum(x > 0 for x in d["owned"]) >= (2 if block == 8 else 1), d["owned"]
    print(f"sharded_lm_trace {name} {nranks}x{block} owned {d['owned']} " +
          json.dumps(dict(stops=rep.get("stops"), branches=sorted(set(rep.get("branches", []))), lm_iters=rep["lm_iters"])))


def test_lm_branch_coverage_on_ranks(lm_runs):
    branches, stops = set(), set()
    for d in lm_runs.values():
        branches.update(d["rep"].get("branches", []))
        stops.update(d["rep"].get("stops", []))
    assert {"accepted", "rejected"} <= branches, branches
    assert {"iteration_cap", "function", "parameter", "gradient", "no_correspondences"} <= stops, stops
    # a rank that owns no correspondence, on a world with correspondences
    assert any(0 in d["owned"] and sum(d["owned"]) > 0 for d in lm_runs.values())


# ---- guards: as the sharded GN path, the pose untouched where the solo call leaves it

def test_guards(oracle, scan_world):
    import liliom_b200 as L
    B = L._binding
    m, feats, guess = scan_world
    ceres = lambda mc, mni=LM, f=feats, g=guess: (lambda r, c: c.scan_to_map(f, g, mc, max_num_iter=mni, mode=L.MODE_CERES))  # noqa: E731
    gn = lambda mc, f=feats, g=guess: (lambda r, c: c.scan_to_map(f, g, mc, mode=L.MODE_GN))  # noqa: E731
    # no map
    ranks = ceres_ranks(3, 16)
    try:
        assert [code(x) for x in on_ranks(ranks, ceres(2))] == [B.E_NOMAP] * 3 == [code(x) for x in on_ranks(ranks, gn(2))]
    finally:
        close_all(ranks)
    # a map under 10 points (counted over all ranks)
    rng = np.random.default_rng(5)
    C = S.corner(16, (1e4, -1e4))
    f40 = np.ones((40, 4), np.float32)
    f40[:, :3] = C + rng.uniform(-0.5, 0.5, (40, 3))
    for n_vox, want in ((7, B.E_FEWMAP), (12, B.OK)):
        pts = _pt48(_voxel_map(n_vox, C, rng), rng)
        ranks = ceres_ranks(3, 16)
        try:
            on_ranks(ranks, lambda r, c: c.map_update(pts, IDENT))
            got = [code(x) for x in on_ranks(ranks, ceres(2, f=f40, g=IDENT))]
            assert got == [want] * 3 == [code(x) for x in on_ranks(ranks, gn(2, f=f40, g=IDENT))], (n_vox, got)
        finally:
            close_all(ranks)
    one = single()
    ranks = ceres_ranks(3, 16)
    try:
        one.map_set_points(m)
        for c in ranks:
            c.map_set_points(m)
        # match_cnt 0: nothing runs, the pose comes back as given
        pose, _ = _ceres_on(ranks, ceres(0))
        assert np.array_equal(pose, guess) and np.array_equal(one.scan_to_map(feats, guess, 0, mode=L.MODE_CERES)[0], guess)
        # max_num_iter 0: one round, the iteration cap before any step; the sign-unified start on every rank, as on one GPU
        pose, st = _ceres_on(ranks, ceres(2, 0))
        p1, s1 = one.scan_to_map(feats, guess, 2, max_num_iter=0, mode=L.MODE_CERES)
        assert pose.tobytes() == p1.tobytes() == RA.unify(guess).tobytes() and [s.lm_iters for s in st] == [0, 0]
        assert [s.n_corr for s in st] == [s.n_corr for s in s1]
        # no correspondence anywhere (the count0 <= 0 stop on the global count): every feature 1 km above the map
        far = feats.copy()
        far[:, 2] += 1000.0
        pose, st = _ceres_on(ranks, ceres(2, f=far))
        p1, s1 = one.scan_to_map(far, guess, 2, max_num_iter=LM, mode=L.MODE_CERES)
        assert pose.tobytes() == p1.tobytes() == RA.unify(guess).tobytes()
        assert [(s.n_corr, s.lm_iters) for s in st] == [(0, 0), (0, 0)] == [(s.n_corr, s.lm_iters) for s in s1]
    finally:
        close_all(ranks + [one])


def test_forgotten_rank_fails_within_the_bound(scan_world):
    import time
    import liliom_b200 as L
    B = L._binding
    m, feats, guess = scan_world
    call = lambda r, c: c.scan_to_map(feats, guess, 2, max_num_iter=LM, mode=L.MODE_CERES)  # noqa: E731
    ranks = ceres_ranks(3, 16, ms=300)
    fresh = ceres_ranks(3, 16)
    try:
        for c in ranks + fresh:
            c.map_set_points(m)
        t0 = time.monotonic()
        res = on_ranks(ranks[:2], call, timeout=30.0)
        assert [code(x) for x in res] == [B.E_NCCL] * 2 and "did not gather" in str(res[0])
        assert time.monotonic() - t0 < 10.0
        # the next call on all ranks runs as on ranks that never failed
        pose, st = _ceres_on(ranks, call)
        pose_f, st_f = _ceres_on(fresh, call)
        assert pose.tobytes() == pose_f.tobytes() and [bytes(s) for s in st] == [bytes(s) for s in st_f]
    finally:
        close_all(ranks + fresh)


# ---- odometry on the ranks: the ranks agree bit for bit, and with one context within 1e-4 m / 1e-4 rad

def test_extract_and_odometry_resident(world_small):
    import liliom_b200 as L
    pts, q, guess = world_small["hz"], world_small["q_hz"], world_small["guess"]
    one = single()
    ranks = ceres_ranks(2, 16)
    try:
        for c in ranks + [one]:
            c.map_set_points(world_small["map"])

        def step(r, c):
            c.upload_scan(pts)
            c.extract_resident(q)
            pose, st, _ = c.odometry_resident(guess, OUTER, max_num_iter=LM, mode=L.MODE_CERES)
            return pose, st
        pose, st = _ceres_on(ranks, step)
        p1, s1 = step(0, one)
        assert _pose_close(pose, p1), (pose, p1)
        assert [s.n_corr for s in st][:1] == [s.n_corr for s in s1][:1] and st[0].n_corr > 100
    finally:
        close_all(ranks + [one])


def test_stream_with_map_updates(scan_world):
    import liliom_b200 as L
    m, feats, guess = scan_world
    rng = np.random.default_rng(3)
    one = single()
    ranks = ceres_ranks(3, 16)
    try:
        base = _pt48(m[:, :3], rng)
        one.map_update(base, IDENT)
        on_ranks(ranks, lambda r, c: c.map_update(base, IDENT))
        frame = _pt48(feats[:, :3], rng)
        p_r, p_1 = np.array(guess), np.array(guess)
        for k in range(10):
            pose, _ = _ceres_on(ranks, lambda r, c: c.scan_to_map(feats, p_r, OUTER, max_num_iter=LM, mode=L.MODE_CERES))
            p1, _ = one.scan_to_map(feats, p_1, OUTER, max_num_iter=LM, mode=L.MODE_CERES)
            assert _pose_close(pose, p1), (k, pose, p1)
            res = on_ranks(ranks, lambda r, c: c.map_update(frame, pose))
            assert all(code(x) == 0 for x in res), [str(x) for x in res]
            one.map_update(frame, p1)
            drift = np.array([0, 0, 0, 0, 0.01 * (k + 1), -0.005, 0.002])
            p_r, p_1 = pose + drift, p1 + drift
    finally:
        close_all(ranks + [one])


def test_lidar_odometry_node_on_ranks(oracle, world_small):
    import liliom_b200 as L
    from liliom_b200 import synth
    one = single()
    ranks = ceres_ranks(2, 16)
    nodes = [L.LidarOdometryNode(c, max_num_iter=LM, scan_match_cnt=2, mode=L.MODE_CERES) for c in ranks]
    node1 = L.LidarOdometryNode(one, max_num_iter=LM, scan_match_cnt=2, mode=L.MODE_CERES)
    try:
        T0 = world_small["T"]
        for k in range(4):
            T = np.array(T0); T[4] += 0.12 * k; T[5] += 0.02 * k
            T[:4] = synth.qmul(synth.q_from_axis_angle([0, 0, 1], np.deg2rad(0.6 * k)), T0[:4])
            pts, q = synth.make_horizon_sweep(T, seed=60 + k)
            surf, edge, cut = oracle.extract_horizon(pts, q)

            def run(r, c):
                nodes[r].feed(0.1 * k, edge, surf, cut)
                out, *_ = nodes[r].run(want_clouds=False)
                return np.array(out.abs_pose), out
            res = on_ranks(ranks, run)
            assert all(code(x) == 0 for x in res), [str(x) for x in res]
            node1.feed(0.1 * k, edge, surf, cut)
            out1, *_ = node1.run(want_clouds=False)
            for pose, out in res:
                assert pose.tobytes() == res[0][0].tobytes() and out.initialized == out1.initialized and out.status == 0
                assert out.n_surf_ds == out1.n_surf_ds and out.kf == out1.kf
            if out1.initialized:
                assert _pose_close(res[0][0], np.array(out1.abs_pose)), (k, res[0][0], list(out1.abs_pose))
    finally:
        for n in nodes + [node1]:
            n.close()
        close_all(ranks + [one])
