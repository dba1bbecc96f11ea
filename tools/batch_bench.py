#!/usr/bin/env python
"""Several odometry sessions on one GPU, three ways: (a) solo calls one after another, (b) one host thread + context stream
per session (as tools/multistream.py), (c) one liliom_odometry_resident_batch call per step.  Headline workload per session:
seeded 24k-point Horizon sweep (extracted on the device), 1 M-point map, 10 GN iterations; the sweeps and poses of
tools/multistream.py.  Every timed scan is the whole resident step: upload of the raw sweep, extraction, VoxelGrid and GN.
Prints the card, its power limit and maximum SM clock, then one JSON line per session count: aggregate scans/s and the median
per-session step latency (the step call: odometry_resident in (a) and (b), the batch call in (c)), and the GN launches one
batch call issues (k_gn_batch / k_gn_persistent / k_knn_plane kernels counted with torch.profiler in a separate call).
usage: batch_bench.py [--sessions 1 2 4 8 16 32] [--steps 30] [--warmup 5]"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import liliom_b200 as L  # noqa: E402
from liliom_b200 import synth  # noqa: E402

ITERS = 10


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", type=int, nargs="*", default=[1, 2, 4, 8, 16, 32])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("batch_bench.py measures on a CUDA device; none is visible")
    print(json.dumps(card()), flush=True)
    m, _ = synth.make_map(1_000_000)
    T0 = synth.default_true_pose()
    sweeps = []
    for k in range(8):
        T = np.array(T0); T[4] += 0.7 * k; T[5] += 0.15 * k
        pts, q = synth.make_horizon_sweep(T, seed=1 + k)
        sweeps.append(dict(T=T, guess=synth.perturbed_pose(T), pts=pts, q=q))

    for B in args.sessions:
        ctxs = []
        for s in range(B):
            c = L.Context(variant=0)
            c.map_set_points(m)
            ctxs.append(c)

        def feed(s, k):
            sw = sweeps[(k + s) % len(sweeps)]
            ctxs[s].upload_scan(sw["pts"])
            ctxs[s].extract_resident(sw["q"])
            return sw

        def solo_step(s, k, lat):
            sw = feed(s, k)
            t = time.perf_counter()
            ctxs[s].odometry_resident(sw["guess"], ITERS, mode=L.MODE_GN, want_stats=False)
            lat.append(time.perf_counter() - t)

        def batch_step(k, lat):
            poses = np.array([feed(s, k)["guess"] for s in range(B)])
            t = time.perf_counter()
            _, status, _, _ = L.odometry_resident_batch(ctxs, poses, ITERS)
            lat.append(time.perf_counter() - t)
            assert (status == 0).all(), status

        def sequential(n):
            lat = []
            for k in range(n):
                for s in range(B):
                    solo_step(s, k, lat)
            return lat

        def threaded(n):
            lats = [[] for _ in range(B)]
            ths = [threading.Thread(target=lambda s=s: [solo_step(s, k, lats[s]) for k in range(n)]) for s in range(B)]
            for t in ths: t.start()
            for t in ths: t.join()
            return [x for v in lats for x in v]

        def batched(n):
            lat = []
            for k in range(n):
                batch_step(k, lat)
            return lat

        row = dict(sessions=B)
        for name, fn in (("a_solo", sequential), ("b_threads", threaded), ("c_batch", batched)):
            fn(args.warmup)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            lat = fn(args.steps)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            row[f"{name}_scans_per_s"] = round(B * args.steps / dt, 1)
            row[f"{name}_step_ms_median"] = round(float(np.median(lat)) * 1e3, 4)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            batched(1)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        row["batch_gn_launches"] = sum(1 for n in names if "k_gn_batch" in n)
        row["batch_solo_gn_launches"] = sum(1 for n in names if "k_gn_persistent" in n or "k_knn_plane" in n)
        print(json.dumps(row), flush=True)
        for c in ctxs:
            c.close()


if __name__ == "__main__":
    main()
