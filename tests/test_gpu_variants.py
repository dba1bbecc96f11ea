"""The switches of the small-scan GN kernel must not change a single bit:
  LILIOM_GN_SYNC  = 3 counter grid barrier with a release-only arrival and a relaxed poll (default) | 1 release arrival +
                    acquire poll | 0 full fences on both sides
  fused peer exchange of one rank with itself (the whole NVLink protocol on a single GPU)
  LILIOM_KNN_TMA  = 1 the 16-lane search stages every run with one cp.async.bulk into shared memory (mbarrier) instead of
                    batches of 16-byte loads through registers
Same candidate sets, same per-row arithmetic, same summation trees -> identical poses, correspondences and sums."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# mode % 10 = LILIOM_GN_SYNC; +20: fused peer exchange with itself; +30: bulk-copy staging
VARIANTS = [3, 1, 0, 23, 33]


def _ctx(ll):
    import liliom_b200 as L
    keys = ("LILIOM_GN_SYNC", "LILIOM_KNN_TMA")
    old = {k: os.environ.get(k) for k in keys}
    os.environ["LILIOM_GN_SYNC"] = str(ll % 10)
    os.environ["LILIOM_KNN_TMA"] = "1" if 30 <= ll < 40 else "0"
    try:
        c = L.Context(variant=0)             # the switches are read at liliom_create
        if 20 <= ll < 30:                    # one rank exchanging with itself: the whole protocol on a single GPU
            c.comm_peer_attach([c.comm_peer_export()], 0)
        return c
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def test_gn_variants_bit_identical(oracle, world_small):
    import liliom_b200 as L
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    guess = world_small["guess"]
    # scans of different sizes back to back: the grid size changes between launches, the larger ones leave the 16-lane shape
    # 3000: eight lanes per query (sixteen would need more than one block per SM and leave the single launch)
    scans = [ds, ds[: len(ds) // 3], ds[::2], ds[:40], surf[:6000], surf[:3000], ds]
    ref = None
    for ll in VARIANTS:
        c = _ctx(ll)
        c.map_set_points(world_small["map"])
        out = []
        for f in scans:
            for iters in (10, 3):
                pose, st = c.scan_to_map(f, guess, iters, mode=L.MODE_GN)
                out.append((pose.copy(), [np.array(s.jtj_jtr) for s in st], [s.n_corr for s in st], [s.cost for s in st]))
        v, pl, idx, sqd, s29 = c.find_surf_corr(ds, guess)          # k_knn_plane<16> (ticket path)
        out.append((s29.copy(), [pl.copy()], [idx.copy(), v.copy()], [sqd.copy()]))
        c.close()
        if ref is None:
            ref = out
            rc, pose_o, _ = oracle.scan_to_map_gn(oracle.KdTree(world_small["map"]), ds, guess, 10)
            assert np.linalg.norm(out[0][0][4:] - pose_o[4:]) < 1e-4
            rc, pose_o, _ = oracle.scan_to_map_gn(oracle.KdTree(world_small["map"]), surf[:3000], guess, 10)
            assert np.linalg.norm(out[10][0][4:] - pose_o[4:]) < 1e-4 and abs(abs(np.dot(out[10][0][:4], pose_o[:4])) - 1) < 1e-9
            continue
        for k, (a, b) in enumerate(zip(out, ref)):
            assert a[0].tobytes() == b[0].tobytes(), (ll, k, a[0], b[0])
            for x, y in zip(a[1] + a[3], b[1] + b[3]):
                assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), (ll, k)
            for x, y in zip(a[2], b[2]):
                assert np.array_equal(x, y), (ll, k)


def test_gn_variants_resident_pipeline(oracle, world_small):
    """Through the node-facing call (extract -> VoxelGrid -> persistent GN with the device-side query count)."""
    import liliom_b200 as L
    ref = None
    for ll in VARIANTS:
        c = _ctx(ll)
        c.map_set_points(world_small["map"])
        poses = []
        for k in range(4):
            surf, edge, cut = c.extract_horizon(world_small["hz"], world_small["q_hz"])
            pose, st, ds = c.odometry_resident(world_small["guess"], 10, mode=L.MODE_GN, want_ds=True, cap=len(surf))
            poses.append(pose.copy())
        c.close()
        assert all(p.tobytes() == poses[0].tobytes() for p in poses)            # run-to-run deterministic
        if ref is None:
            ref = poses[0]
        assert poses[0].tobytes() == ref.tobytes(), ll


def test_peer_epoch_resync(oracle, world_small):
    """After a lost exchange the application realigns the ranks' epochs (liliom_comm_peer_epoch / _set_epoch): a scan advances the
    epoch by its iteration count, a jump forward changes nothing in the result, a step back is refused."""
    import liliom_b200 as L
    surf, _, _ = oracle.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = oracle.voxelgrid(surf, 0.4)
    c = _ctx(23)                                   # one rank exchanging with itself
    c.map_set_points(world_small["map"])
    e0 = c.comm_peer_epoch()
    p1, _ = c.scan_to_map(ds, world_small["guess"], 10, mode=L.MODE_GN)
    assert c.comm_peer_epoch() == e0 + 10
    c.comm_peer_set_epoch(e0 + 10 + 1001)             # what max-over-ranks + 2 could look like after a loss elsewhere
    p2, _ = c.scan_to_map(ds, world_small["guess"], 10, mode=L.MODE_GN)
    assert p1.tobytes() == p2.tobytes() and c.comm_peer_epoch() == e0 + 10 + 1001 + 10
    with pytest.raises(L.LiliomError):
        c.comm_peer_set_epoch(5)
    c.close()
