#!/usr/bin/env python
"""Several odometry sessions on one GPU, three ways: (a) solo calls one after another, (b) one host thread + context stream
per session (as tools/multistream.py), (c) one liliom_odometry_resident_batch_ex call per step.  Workload per session:
--variant horizon (default): the headline, a seeded 24k-point Horizon sweep (extracted on the device), 1 M-point map, the
sweeps and poses of tools/multistream.py; --variant rot: bench.py's configs[2], a seeded 130k-point HDL-64E sweep through the
ROT extractor, 2 M-point map.
--mode gn (default): 10 GN iterations; --mode ceres: the reference's configs, scan_match_cnt 2 outer iterations of at most
max_num_iter 15 LM iterations (--match-cnt / --max-num-iter override either).  Every timed scan of (a)-(c) is the whole resident
step: upload of the raw sweep, extraction, VoxelGrid and scan-to-map.  Two more legs time only the scan-to-map call on resident
down-sampled features (the step legs are bound by the host's upload and extraction): (d) solo liliom_scan_to_map_resident calls
one after another, (e) one liliom_scan_to_map_resident_batch_ex call; their *_call_ms_median is the time of all B sessions.
Extraction: (f) on resident raw sweeps, B solo liliom_extract_resident calls then a device synchronise
(f_extract_solo_ms_median) against one liliom_extract_resident_batch call (f_extract_batch_ms_median); (g) the whole step with
batched extraction: the per-session upload, one liliom_extract_resident_batch, one liliom_odometry_resident_batch_ex.
Prints the card, its power limit and maximum SM clock, then one JSON line per session count: aggregate scans/s, the median
per-session step latency (the step call: odometry_resident in (a) and (b), the batch call in (c)), and the scan-to-map kernels
one batched scan-to-map call launches (counted with torch.profiler in a separate call).
usage: batch_bench.py [--sessions 1 2 4 8 16 32] [--steps 30] [--warmup 5] [--mode {gn,ceres}] [--match-cnt N] [--max-num-iter N]
                      [--variant {horizon,rot}]"""
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
    ap.add_argument("--mode", choices=("gn", "ceres"), default="gn")
    ap.add_argument("--match-cnt", type=int, default=None, help="outer iterations (default: 10 in GN mode, 2 in Ceres mode)")
    ap.add_argument("--max-num-iter", type=int, default=15, help="LM iterations per outer iteration (Ceres mode)")
    ap.add_argument("--variant", choices=("horizon", "rot"), default="horizon")
    args = ap.parse_args()
    mode = L.MODE_CERES if args.mode == "ceres" else L.MODE_GN
    iters = args.match_cnt if args.match_cnt is not None else (2 if mode == L.MODE_CERES else 10)
    mni = args.max_num_iter
    if not torch.cuda.is_available():
        raise SystemExit("batch_bench.py measures on a CUDA device; none is visible")
    rot = args.variant == "rot"
    print(json.dumps(dict(card(), variant=args.variant, mode=args.mode, match_cnt=iters, max_num_iter=mni)), flush=True)
    m, _ = synth.make_map(2_000_000 if rot else 1_000_000)
    T0 = synth.default_true_pose()
    sweeps = []
    for k in range(8):
        T = np.array(T0); T[4] += 0.7 * k; T[5] += 0.15 * k
        pts, q = synth.make_hdl64_sweep(T, seed=2 + k) if rot else synth.make_horizon_sweep(T, seed=1 + k)
        sweeps.append(dict(T=T, guess=synth.perturbed_pose(T), pts=pts, q=q))

    for B in args.sessions:
        ctxs = []
        for s in range(B):
            c = L.Context(variant=1 if rot else 0)
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
            ctxs[s].odometry_resident(sw["guess"], iters, max_num_iter=mni, mode=mode, want_stats=False)
            lat.append(time.perf_counter() - t)

        def batch_step(k, lat):
            poses = np.array([feed(s, k)["guess"] for s in range(B)])
            t = time.perf_counter()
            _, status, _, _ = L.odometry_resident_batch_ex(ctxs, poses, iters, mni, mode)
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
        # scan-to-map alone on resident down-sampled features: each session keeps its sweep's DS cloud
        guesses = []
        for s in range(B):
            sw = feed(s, 0)
            _, _, ds = ctxs[s].odometry_resident(sw["guess"], iters, max_num_iter=mni, mode=mode, want_ds=True, cap=len(sw["pts"]),
                                                 want_stats=False)
            ctxs[s].upload_feats(ds)
            guesses.append(sw["guess"])
        guesses = np.array(guesses)

        def s2m_solo(n):
            lat = []
            for _ in range(n):
                t = time.perf_counter()
                for s in range(B):
                    ctxs[s].scan_to_map_resident(guesses[s], iters, max_num_iter=mni, mode=mode)
                lat.append(time.perf_counter() - t)
            return lat

        def s2m_batch(n):
            lat = []
            for _ in range(n):
                t = time.perf_counter()
                _, status, _ = L.scan_to_map_resident_batch_ex(ctxs, guesses, iters, mni, mode)
                lat.append(time.perf_counter() - t)
                assert (status == 0).all(), status
            return lat

        for name, fn in (("d_s2m_solo", s2m_solo), ("e_s2m_batch", s2m_batch)):
            fn(args.warmup)
            torch.cuda.synchronize()
            lat = fn(args.steps)
            row[f"{name}_call_ms_median"] = round(float(np.median(lat)) * 1e3, 4)
        # (f) extraction alone on resident raw sweeps, and (g) the whole step with batched extraction
        for s in range(B):
            ctxs[s].upload_scan(sweeps[s % len(sweeps)]["pts"])
        qs = np.array([sweeps[s % len(sweeps)]["q"] for s in range(B)])

        def ext_solo(n):
            lat = []
            for _ in range(n):
                t = time.perf_counter()
                for s in range(B):
                    ctxs[s].extract_resident(qs[s])
                torch.cuda.synchronize()
                lat.append(time.perf_counter() - t)
            return lat

        def ext_batch(n):
            lat = []
            for _ in range(n):
                t = time.perf_counter()
                _, status = L.extract_resident_batch(ctxs, qs)
                lat.append(time.perf_counter() - t)
                assert (status == 0).all(), status
            return lat

        for name, fn in (("f_extract_solo", ext_solo), ("f_extract_batch", ext_batch)):
            fn(args.warmup)
            torch.cuda.synchronize()
            lat = fn(args.steps)
            row[f"{name}_ms_median"] = round(float(np.median(lat)) * 1e3, 4)

        def batch_step_g(k, lat):
            sws = [sweeps[(k + s) % len(sweeps)] for s in range(B)]
            for s in range(B):
                ctxs[s].upload_scan(sws[s]["pts"])
            t = time.perf_counter()
            _, st_x = L.extract_resident_batch(ctxs, np.array([sw["q"] for sw in sws]))
            _, status, _, _ = L.odometry_resident_batch_ex(ctxs, np.array([sw["guess"] for sw in sws]), iters, mni, mode)
            lat.append(time.perf_counter() - t)
            assert (st_x == 0).all() and (status == 0).all(), (st_x, status)

        def batched_g(n):
            lat = []
            for k in range(n):
                batch_step_g(k, lat)
            return lat

        batched_g(args.warmup)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        lat = batched_g(args.steps)
        torch.cuda.synchronize()
        row["g_batch_extract_scans_per_s"] = round(B * args.steps / (time.perf_counter() - t0), 1)
        row["g_batch_extract_step_ms_median"] = round(float(np.median(lat)) * 1e3, 4)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            s2m_batch(1)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        for key, pat in (("k_gn_batch", "k_gn_batch"), ("k_knn_plane_batch", "k_knn_plane_batch"), ("k_lm_solve_batch", "k_lm_solve_batch"),
                         ("k_gn_persistent", "k_gn_persistent"), ("k_knn_plane", "k_knn_plane<"), ("k_lm_solve", "k_lm_solve(")):
            row[f"s2m_batch_launches_{key}"] = sum(1 for n in names if pat in n)
        print(json.dumps(row), flush=True)
        for c in ctxs:
            c.close()


if __name__ == "__main__":
    main()
