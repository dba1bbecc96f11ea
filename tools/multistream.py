#!/usr/bin/env python
"""Throughput of S independent scan streams sharing ONE H100 (one liliom context + CUDA stream + host
thread per scan stream, as S robots' LidarOdometry/Preprocessing node pairs would).  The single-stream
step is latency-bound (~20 % SM activity), so concurrent streams fill the machine.
usage: multistream.py [streams ...]"""
import os, sys, threading, time, json
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import liliom_b200 as L
from liliom_b200 import synth

ITERS = 10
m, _ = synth.make_map(1_000_000)
T0 = synth.default_true_pose()
sweeps = []
for k in range(8):
    T = np.array(T0); T[4] += 0.7 * k; T[5] += 0.15 * k
    pts, q = synth.make_horizon_sweep(T, seed=1 + k)
    sweeps.append(dict(T=T, guess=synth.perturbed_pose(T), pts=pts, q=q))

def run(S, steps_per_stream=60, e2e=False):
    ctxs = []
    for s in range(S):
        c = L.Context(variant=0)
        c.map_set_points(m)
        ctxs.append(c)
    errs = [0.0] * S
    def worker(s, n):
        c = ctxs[s]
        if e2e:
            cap = max(len(w["pts"]) for w in sweeps)
            bufs = [torch.empty(cap * 48, dtype=torch.uint8).pin_memory().numpy().view(L.PT48) for _ in range(4)]
            pins = [torch.from_numpy(w["pts"].view(np.uint8).reshape(-1)).pin_memory().numpy().view(L.PT48) for w in sweeps]
        for k in range(n):
            sw = sweeps[(k + s) % len(sweeps)]
            if e2e:
                surf, edge, cut = c.extract_horizon(pins[(k + s) % len(sweeps)], sw["q"], out=(bufs[0], bufs[1], bufs[2]))
                pose, st, ds = c.odometry(surf, sw["guess"], ITERS, mode=L.MODE_GN, ds_out=bufs[3])
            else:
                c.upload_scan(sw["pts"])
                c.extract_resident(sw["q"])
                pose, st, nds = c.odometry_resident(sw["guess"], ITERS, mode=L.MODE_GN)
            errs[s] = float(np.linalg.norm(pose[4:] - sw["T"][4:]))
    for s in range(S): worker(s, 3)          # warm-up
    torch.cuda.synchronize()
    ths = [threading.Thread(target=worker, args=(s, steps_per_stream)) for s in range(S)]
    t0 = time.perf_counter()
    for t in ths: t.start()
    for t in ths: t.join()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    for c in ctxs: c.close()
    return S * steps_per_stream / dt, max(errs)

for S in [int(x) for x in sys.argv[1:]] or [1, 2, 4, 8]:
    v, e = run(S)
    v2, e2 = run(S, e2e=True)
    print(json.dumps(dict(streams=S, resident_scans_per_s=round(v, 1), e2e_scans_per_s=round(v2, 1), max_pose_err_m=round(max(e, e2), 4))), flush=True)
