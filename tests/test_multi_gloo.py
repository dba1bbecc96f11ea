"""N > 1 host-side logic on CPU with the gloo backend (world_size 2): the shard-ownership rule
(8 m block hash + halo) used by the CUDA kernels, restated in numpy (liliom_b200/sharding.py), and
the per-iteration exchange — partial 29-vectors summed with one all-reduce — give the single-rank
result.  The per-rank partial sums come from the CPU oracle (the checker), not from the product."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import oracle_lib as O
    from liliom_b200 import sharding, synth
    m, _ = synth.make_map(30000)
    T = synth.default_true_pose()
    pts, q = synth.make_horizon_sweep(T, seed=21)
    surf, _, _ = O.extract_horizon(pts, q)
    ds = O.voxelgrid(surf, 0.4)
    feats = np.ones((len(ds), 4), np.float32); feats[:, 0] = ds["x"]; feats[:, 1] = ds["y"]; feats[:, 2] = ds["z"]
    pose = synth.perturbed_pose(T)
    # --- shard the map: this rank keeps the points whose halo box touches a block it owns
    keep = sharding.shard_mask(m[:, :3], world, rank, halo=1.0)
    local = m[keep]
    # --- this rank's queries = those whose transformed position falls in an owned block
    pw = sharding.transform_f32(feats[:, :3], pose)
    mine = sharding.owner_of(pw, world) == rank
    tree = O.KdTree(local)
    cnt, valid, plane, idx, _ = O.find_surf_corr(tree, feats, pose)
    valid = (valid.astype(bool) & mine).astype(np.uint8)
    part = O.normal_equations(feats, valid, plane, pose)
    t = torch.from_numpy(part.copy())
    dist.all_reduce(t, op=dist.ReduceOp.SUM)           # the path's one collective: 29 fp64 scalars
    counts = torch.tensor([int(keep.sum()), int(mine.sum())], dtype=torch.int64)
    gathered = [torch.zeros_like(counts) for _ in range(world)]
    dist.all_gather(gathered, counts)
    if rank == 0:
        full = O.KdTree(m)
        c0, v0, p0, i0, _ = O.find_surf_corr(full, feats, pose)
        ref = O.normal_equations(feats, v0, p0, pose)
        np.save(out, np.concatenate([t.numpy(), ref, np.array([g.tolist() for g in gathered], np.float64).ravel(), [len(m), len(feats)]]))
    dist.destroy_process_group()


def test_sharded_normal_equations_equal_single_rank(tmp_path):
    world = 2
    out = str(tmp_path / "res.npy")
    port = 29500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    r = np.load(out)
    summed, ref = r[:29], r[29:58]
    shard_pts = r[58:58 + 2 * world:2]; shard_q = r[59:59 + 2 * world:2]
    n_map, n_q = r[-2], r[-1]
    assert summed[28] == ref[28] and ref[28] > 100          # same correspondences, each counted once
    np.testing.assert_allclose(summed, ref, rtol=1e-11, atol=1e-11)
    assert shard_q.sum() == n_q                              # every query has exactly one owner
    assert shard_pts.sum() >= n_map and shard_pts.max() < n_map   # halo duplicates some points, no rank holds all


def test_shard_rule_properties():
    sys.path.insert(0, ROOT)
    from liliom_b200 import sharding
    rng = np.random.default_rng(0)
    p = rng.uniform(-100, 100, (20000, 3)).astype(np.float32)
    for world in (2, 4, 8):
        own = sharding.owner_of(p, world)
        assert own.min() == 0 and own.max() == world - 1
        masks = np.stack([sharding.shard_mask(p, world, r, halo=1.0) for r in range(world)])
        assert masks[own, np.arange(len(p))].all()           # a point is always in its owner's shard
        # every point within 1 m of a query is in the query owner's shard
        q = p[:500] + rng.uniform(-0.9, 0.9, (500, 3)).astype(np.float32) / np.sqrt(3)
        qo = sharding.owner_of(q, world)
        assert masks[qo, np.arange(500)].all()


def _maint_worker(rank, world, port, out):
    """Sharded map maintenance (map.cu push_frame_from_device / liliom_map_rebuild with a communicator), restated on the host:
    a rank keeps the frame points within (1 m + one voxel diagonal) of a block it owns, voxel-filters its shard alone, and
    keeps the voxels within 1 m of an owned block."""
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import oracle_lib as O
    import bench
    from liliom_b200 import sharding, synth
    m, _ = synth.make_map(40000)
    frames = bench.make_frames(m, O.PT32)
    leaf = 0.4
    halo_f = np.float32(1.0 + 1.7320508 * leaf + 0.05)
    mine = []
    for f in frames:
        xyz = np.stack([f["x"], f["y"], f["z"]], 1)
        mine.append(f[sharding.shard_mask(xyz, world, rank, halo=float(halo_f))])
    ds = O.voxelgrid(np.concatenate(mine), leaf)
    xyz = np.stack([ds["x"], ds["y"], ds["z"]], 1)
    ds = ds[sharding.shard_mask(xyz, world, rank, halo=1.0)]
    rows = np.stack([ds["x"], ds["y"], ds["z"]], 1).view(np.uint32)
    n = torch.tensor([len(rows)], dtype=torch.int64)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n)
    np.save(f"{out}.{rank}.npy", rows)
    dist.barrier()
    if rank == 0:
        full = O.voxelgrid(np.concatenate(frames), leaf)
        fx = np.stack([full["x"], full["y"], full["z"]], 1)
        np.save(out, np.concatenate([[len(m), sum(len(f) for f in frames), len(full)], [int(s.item()) for s in sizes]]))
        np.save(out + ".full.npy", fx)
    dist.destroy_process_group()


def test_sharded_map_maintenance_equals_full_filter(tmp_path):
    sys.path.insert(0, ROOT)
    from liliom_b200 import sharding
    world = 2
    out = str(tmp_path / "maint.npy")
    port = 31500 + (os.getpid() % 2000)
    mp.spawn(_maint_worker, args=(world, port, out), nprocs=world, join=True)
    head = np.load(out)
    n_map, n_frames_pts, n_full = int(head[0]), int(head[1]), int(head[2])
    assert n_frames_pts == n_map                                   # the frames partition the map
    assert n_full > 0.95 * n_map
    full = np.load(out + ".full.npy")
    full_rows = {r.tobytes() for r in full.view(np.uint32)}
    for rank in range(world):
        rows = np.load(f"{out}.{rank}.npy")
        got = {r.tobytes() for r in rows}
        assert got <= full_rows                                    # a shard never invents or alters a voxel centroid
        need = full[sharding.shard_mask(full, world, rank, halo=1.0)]
        assert {r.tobytes() for r in need.view(np.uint32)} == got  # and holds exactly the voxels its queries can reach
        assert len(got) < n_full
