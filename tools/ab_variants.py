#!/usr/bin/env python
"""A/B of the small-scan GN kernel switches inside ONE process (on the GPU):
for every LILIOM_GN_SYNC value a fresh context is created (the switch is read at liliom_create), the bench's resident step (extract -> VoxelGrid -> 10 GN iterations, L2 flushed between steps) is timed with
CUDA events, and the pose is compared bit-for-bit with the first configuration.  LILIOM_LIB selects a tuning build of the library.
usage: ab_variants.py [steps] [sync ...]"""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import liliom_b200 as L
from liliom_b200 import synth

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 150
cfgs = [int(a) for a in sys.argv[2:]] or [3, 33, 1, 0, 3, 33]      # +30: LILIOM_KNN_TMA=1 (bulk-copy staging of the runs)
m, _ = synth.make_map(1_000_000)
T0 = synth.default_true_pose()
sweeps = []
for k in range(4):
    T = np.array(T0); T[4] += 0.7 * k; T[5] += 0.15 * k
    pts, q = synth.make_horizon_sweep(T, seed=1 + k)
    sweeps.append((pts, q, synth.perturbed_pose(T)))
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
stream = torch.cuda.Stream()
ref = None
print(f"lib: {L.LIB_PATH}")
for sync in cfgs:
    tens = (sync // 10) % 10                      # 3: bulk-copy staging; 4: results by copies (LILIOM_HOST_RESULTS=0); +100: kernel-timing events off
    os.environ["LILIOM_GN_SYNC"] = str(sync % 10); os.environ["LILIOM_KNN_TMA"] = "1" if tens == 3 else "0"
    os.environ["LILIOM_HOST_RESULTS"] = "0" if tens == 4 else "1"
    c = L.Context(variant=0)
    c.set_stream(stream.cuda_stream)
    c.map_set_points(m)
    c.set_kernel_timing(sync < 100)
    poses = []
    tot = 0.0
    with torch.cuda.stream(stream):
        for k in range(steps + 5):
            pts, q, guess = sweeps[k % len(sweeps)]
            c.upload_scan(pts)
            flush.fill_(k & 0xff)
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            c.extract_resident(q)
            pose, st, nds = c.odometry_resident(guess, 10, mode=L.MODE_GN, want_stats=False)
            e1.record(stream); e1.synchronize()
            if k == 4:
                c.counters(reset=True)
            if k >= 5:
                tot += e0.elapsed_time(e1)
            if k < len(sweeps):
                poses.append(pose.copy())
    cnt = c.counters()
    c.close()
    same = "ref" if ref is None else ("bit-identical" if all(a.tobytes() == b.tobytes() for a, b in zip(poses, ref)) else "DIFFERENT POSES")
    if ref is None:
        ref = poses
    print(f"sync={sync}: {steps / (tot * 1e-3):7.0f} scans/s  step {1e3 * tot / steps:6.1f} us  GN {1e3 * cnt.knn_ms / max(cnt.knn_launches, 1):6.2f} us/pass  [{same}]", flush=True)
