#!/usr/bin/env python
"""torchrun --nproc-per-node N tools/multi_check.py : sharded scan-to-map (map split by 8 m block hash,
29-scalar NCCL all-reduce per iteration) must give the single-GPU pose.
LILIOM_MODE=ceres adds the Ceres-faithful leg (liliom_comm_set_ceres): every rank must hold the same pose bits, within
1e-4 m / 1e-4 rad of the single-GPU Ceres pose; each scan's time is printed next to the single-GPU Ceres scan's."""
import os, sys, time
import numpy as np
import torch, torch.distributed as dist
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import liliom_b200 as L
from liliom_b200 import synth

rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); lr = int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(lr)
dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
n_map = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
m, _ = synth.make_map(n_map)
T = synth.default_true_pose()
pts, q = synth.make_horizon_sweep(T)
guess = synth.perturbed_pose(T)
ref = L.Context(variant=0, device=lr)
ref.map_set_points(m)
surf, edge, cut = ref.extract_horizon(pts, q)
ds = ref.voxelgrid(surf, 0.4)
pose_ref, st_ref = ref.scan_to_map(ds, guess, 10, mode=L.MODE_GN)
ctx = L.Context(variant=0, device=lr)
uid = [L.comm_get_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
ctx.comm_init(uid[0], world, rank)
if os.environ.get("LILIOM_PEER"):      # fused exchange over peer memory instead of ncclAllReduce + update kernel per iteration
    hs = [None] * world
    dist.all_gather_object(hs, ctx.comm_peer_export())
    ctx.comm_peer_attach(hs, rank)
ctx.map_set_points(m)
dist.barrier()          # collective call below: with the fused exchange a rank's kernel waits (bounded) for its peers' kernels
pose, st = ctx.scan_to_map(ds, guess, 10, mode=L.MODE_GN)
dt = np.linalg.norm(pose[4:] - pose_ref[4:]); dq = 1 - abs(np.dot(pose[:4], pose_ref[:4]))
sizes = [None] * world
dist.all_gather_object(sizes, ctx.map_size())
poses = [None] * world
dist.all_gather_object(poses, pose.tolist())
if rank == 0:
    same = all(np.array_equal(np.array(p), np.array(poses[0])) for p in poses)
    print(f"world={world} shard sizes={sizes} (global {n_map}); pose delta vs single GPU: {dt:.3e} m, 1-|q.q'|={dq:.2e}; "
          f"n_corr {st[0].n_corr} vs {st_ref[0].n_corr}; identical across ranks: {same}")
    assert dt < 1e-6 and dq < 1e-12 and same and st[0].n_corr == st_ref[0].n_corr
# ---- Ceres-faithful leg: the collective LM (every LM evaluation one NCCL all-reduce of the 29 sums)
if os.environ.get("LILIOM_MODE") == "ceres":
    def timed(c, n=5):
        out, ms = None, []
        for _ in range(n):
            dist.barrier(); torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = c.scan_to_map(ds, guess, 2, max_num_iter=15, mode=L.MODE_CERES)
            ms.append(1e3 * (time.perf_counter() - t0))
        return out, float(np.median(ms))
    (pc_ref, sc_ref), ms_ref = timed(ref)
    ctx.comm_set_ceres(1)
    (pc, sc), ms = timed(ctx)
    cposes = [None] * world
    dist.all_gather_object(cposes, pc.tobytes())
    if rank == 0:
        same = all(p == cposes[0] for p in cposes)
        dt = np.linalg.norm(pc[4:] - pc_ref[4:]); da = 2 * np.arccos(min(1.0, abs(float(np.dot(pc[:4], pc_ref[:4])))))
        print(f"ceres: pose delta vs single GPU {dt:.3e} m, {da:.3e} rad; LM iterations {[s.lm_iters for s in sc]} vs "
              f"{[s.lm_iters for s in sc_ref]}; identical across ranks: {same}; scan {ms:.3f} ms on {world} ranks vs {ms_ref:.3f} ms "
              f"on one GPU (median of 5, map {n_map})")
        assert same and dt < 1e-4 and da < 1e-4
# ---- streamed lifecycle with SHARDED map maintenance: every rank runs the same LidarOdometry node on its shard
def run_sequence(c):
    node = L.LidarOdometryNode(c, max_num_iter=15, scan_match_cnt=2, if_to_deskew=False, mode=L.MODE_GN)
    out_poses, maps = [], []
    for k in range(6):
        Tk = np.array(T); Tk[4] += 0.12 * k; Tk[5] += 0.02 * k
        p, qq = synth.make_horizon_sweep(Tk, seed=60 + k)
        s_, e_, c_ = ref.extract_horizon(p, qq)
        node.feed(0.1 * k, e_, s_, c_)
        o, *_ = node.run(want_clouds=False)
        out_poses.append(np.array(o.abs_pose)); maps.append(o.n_map)
    node.close()
    return np.array(out_poses), maps
single = L.Context(variant=0, device=lr)
p_single, m_single = run_sequence(single)
shard = L.Context(variant=0, device=lr)
uid2 = [L.comm_get_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid2, src=0)
shard.comm_init(uid2[0], world, rank)
if os.environ.get("LILIOM_PEER"):
    hs2 = [None] * world
    dist.all_gather_object(hs2, shard.comm_peer_export())
    shard.comm_peer_attach(hs2, rank)
p_shard, m_shard = run_sequence(shard)
d = float(np.abs(p_shard - p_single).max())
allp = [None] * world
dist.all_gather_object(allp, p_shard.tolist())
if rank == 0:
    same = all(np.array_equal(np.array(x), np.array(allp[0])) for x in allp)
    print(f"streamed sharded lifecycle: max |pose - single GPU| = {d:.3e}; local map sizes {m_shard} vs global {m_single}; identical across ranks: {same}")
    assert d < 1e-9 and same
dist.destroy_process_group()
